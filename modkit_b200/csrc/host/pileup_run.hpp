// `modkit pileup` orchestration on top of the device C ABI (include/mkp.h).
// Mirrors ModBamPileup::run (src/pileup/subcommand.rs:381-817): same flags, same defaults, same error
// messages where they are observable, same output ordering (feeder order, positions ascending).
#pragma once
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <future>
#include <memory>
#include <filesystem>
#include <set>
#include <unordered_set>

#include "pileup_host.hpp"

namespace mkh {

struct PileupOptions {
    std::string in_bam, out_bed;
    int threads = 4;
    int schedule_threads = 0;          // --threads as the user gave it (the sampling schedule depends on it); 0 = threads
    uint32_t interval_size = 100000, sampling_interval_size = 1000000;
    size_t num_reads = 10042;
    bool have_frac = false; double frac = 0;
    bool no_filtering = false, include_unmapped = false, force_allow = false, cpg = false, mask = false;
    bool traditional = false, combine_mods = false, combine_strands = false, mixed = false, header = false, invert_edge = false;
    float percentile = 0.1f;
    std::vector<std::string> filter_thresholds, mod_thresholds, motif_parts;
    std::string region, sample_region, ignore, ref_fp, edge, stats_json, include_bed;
    int device = 0;
    uint32_t chunk_bp = 16u << 20;     // reference span handed to the GPU per call
    bool host_ingest = false;          // inflate + slice the BAM on the host (zlib) instead of on the GPU
    std::vector<std::string> partition_tags;   // --partition-tag (repeatable): one output file per tag-value combination
    bool bedgraph = false;             // --bedgraph: out path is a directory of <code>_<strand>.bedgraph files
    std::string prefix;                // --prefix for the files of --bedgraph / --partition-tag
    bool quiet = false;
    uint32_t max_depth = 8000;         // --max-depth (src/pileup/subcommand.rs:117-121)
    std::vector<int> devices;          // --devices a,b,...: one interval shard per listed GPU (threads of this process)
    bool hemi = false;                 // `modkit pileup-hemi`: duplex pattern counts at the + strand positions of one palindromic motif
};

// pileup-hemi's motif (src/pileup/subcommand.rs:1242-1272): exactly one, --cpg or --motif, and it must be a palindrome. Checked
// before any device work, so argument errors need no GPU.
inline MotifSpec hemi_motif(const PileupOptions& o) {
    if (o.ref_fp.empty()) throw std::runtime_error("the following required arguments were not provided: --ref <REFERENCE_FASTA>");
    if (o.cpg && !o.motif_parts.empty()) throw std::runtime_error("the argument '--cpg' cannot be used with '--motif <MOTIF> <MOTIF>'");
    if (o.motif_parts.size() > 2) throw std::runtime_error("the argument '--motif <MOTIF> <MOTIF>' cannot be used multiple times");
    if (!o.cpg && o.motif_parts.empty()) throw std::runtime_error("either --cpg or a --motif must be provided for pileup-hemi");
    MotifSpec m;
    if (o.cpg) m = parse_motif("CG", 0);
    else {
        const std::string& off = o.motif_parts[1];
        if (off.empty() || off.find_first_not_of("0123456789") != std::string::npos) throw std::runtime_error("couldn't parse focus position, " + off);
        m = parse_motif(o.motif_parts[0], std::stoi(off));
    }
    if (!m.palindromic) throw std::runtime_error("motif must be palindromic for pileup-hemi");
    return m;
}

struct Region { std::string name; uint32_t start = 0, end = 0; };

inline bool parse_code(const std::string& raw, uint32_t* out) {
    if (raw.size() == 1) { *out = (uint8_t)raw[0]; return true; }
    if (raw.empty()) return false;
    uint64_t v = 0;
    for (char c : raw) { if (c < '0' || c > '9') return false; v = v * 10 + (c - '0'); if (v > 0x7fffffffull) return false; }
    *out = 0x80000000u | (uint32_t)v;
    return true;
}

inline Region parse_region_arg(const std::string& raw, const BamReader& bam) {   // util.rs:475-523
    auto colon = raw.find(':');
    if (colon == std::string::npos) {
        for (size_t i = 0; i < bam.ref_names.size(); i++) if (bam.ref_names[i] == raw) return Region{raw, 0, bam.ref_lens[i]};
        throw std::runtime_error("contig " + raw + " missing from header");
    }
    Region r;
    r.name = raw.substr(0, colon);
    const std::string rest = raw.substr(colon + 1);
    auto dash = rest.find('-');
    if (rest.find(':') != std::string::npos || dash == std::string::npos || rest.find('-', dash + 1) != std::string::npos)
        throw std::runtime_error("invalid region " + raw);
    auto num = [&](std::string s) {
        s.erase(std::remove(s.begin(), s.end(), ','), s.end());
        if (s.empty() || s.size() > 12 || s.find_first_not_of("0123456789") != std::string::npos) throw std::runtime_error("invalid region " + raw);
        const unsigned long long v = std::stoull(s);
        if (v > 0xffffffffull) throw std::runtime_error("invalid region " + raw + " (coordinate does not fit 32 bits)");
        return (uint32_t)v;
    };
    r.start = num(rest.substr(0, dash));
    r.end = num(rest.substr(dash + 1));
    if (r.end <= r.start) throw std::runtime_error("invalid region " + raw);
    return r;
}

inline double secs_between(std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double>(b - a).count(); }

// A fixed set of worker threads for the per-chunk formatting (threads are not created per chunk). Tasks are handed out in increasing
// index order; run() returns when all of them are done; the caller takes part.
class WorkerPool {
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cv_, done_cv_;
    const std::function<void(int)>* fn_ = nullptr;
    int n_tasks_ = 0, next_ = 0, pending_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
    void drain(uint64_t g) {
        for (;;) {
            int i;
            { std::lock_guard<std::mutex> lk(mu_); if (gen_ != g || next_ >= n_tasks_) return; i = next_++; }
            (*fn_)(i);
            { std::lock_guard<std::mutex> lk(mu_); if (--pending_ == 0) done_cv_.notify_all(); }
        }
    }
public:
    explicit WorkerPool(int n_threads) {
        for (int t = 1; t < n_threads; t++) th_.emplace_back([this]() {
            uint64_t seen = 0;
            for (;;) {
                uint64_t g;
                { std::unique_lock<std::mutex> lk(mu_); cv_.wait(lk, [&] { return stop_ || gen_ != seen; }); if (stop_) return; g = seen = gen_; }
                drain(g);
            }
        });
    }
    ~WorkerPool() { { std::lock_guard<std::mutex> lk(mu_); stop_ = true; } cv_.notify_all(); for (auto& t : th_) t.join(); }
    int size() const { return (int)th_.size() + 1; }
    void run(int n_tasks, const std::function<void(int)>& fn) {
        if (n_tasks <= 0) return;
        uint64_t g;
        { std::lock_guard<std::mutex> lk(mu_); fn_ = &fn; n_tasks_ = n_tasks; next_ = 0; pending_ = n_tasks; g = ++gen_; }
        cv_.notify_all();
        drain(g);
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [&] { return pending_ == 0; });
    }
};

inline void trace_mark0(const char* what);
struct DeviceGuard {
    mkp_ctx* ctx = nullptr;
    ~DeviceGuard() { if (ctx) { trace_mark0("host objects released"); mkp_destroy(ctx); trace_mark0("device context destroyed"); } }
};

// ---- threshold estimation: host schedule (reads_sampler/*), device decode + histogram --------------
// MKH_TRACE=1: wall-clock marks of a run's stages on stderr (development); the epoch is set where run_pileup starts
struct TraceClock {
    std::chrono::steady_clock::time_point epoch = std::chrono::steady_clock::now();
    bool on = getenv("MKH_TRACE") != nullptr;
    void mark(int rank, const char* what) const { if (on) fprintf(stderr, "[mkh r%d] %8.3f s  %s\n", rank, std::chrono::duration<double>(std::chrono::steady_clock::now() - epoch).count(), what); }
};
inline TraceClock& trace_clock() { static TraceClock t; return t; }
inline void trace_mark0(const char* what) { trace_clock().mark(0, what); }

struct SamplerConfig {
    int threads = 4;
    int workers = 4;                   // host threads that fetch candidates (not part of the schedule)
    std::shared_ptr<void>* defer_free = nullptr;         // indexed sampler: its candidate buffers (hundreds of MB) are handed over instead of being
                                                         // released before the result is returned; the caller drops them when convenient
    std::shared_future<void>* device_ready = nullptr;    // indexed sampler: the candidates are fetched from the file first (host only); the
                                                         // decode passes wait for this (the device is busy loading the BAM until then)
    uint32_t sampling_interval_size = 1000000;
    bool take_all = false;
    size_t num_reads = 10042;
    const Region* region = nullptr;
    bool include_unmapped = false;
    bool edge_on = false;
    const IncludeBed* include = nullptr;
};

inline bool sampler_flag_ok(const RecRef& r, bool require_mapped) {
    const uint16_t flag = r.flag;
    if (flag & (0x100 | 0x400 | 0x800)) return false;
    if (r.l_seq == 0) return false;
    if (require_mapped && (flag & 0x4)) return false;
    return true;
}

// the sampled reads themselves (summary: a second device pass over them once the thresholds are known)
struct SampledChunk { PackedChunk pc; std::vector<uint8_t> take; uint32_t tid = 0; };

// resident chunk of sampled reads: without coordinates of its own, except with --include-bed (bitmaps of the contig)
inline void upload_sample_chunk(mkp_ctx* ctx, const PackedChunk& pc, uint32_t tid, const IncludeBed* include, std::vector<uint32_t>* fpos, std::vector<uint32_t>* fneg) {
    mkp_chunk ch;
    memset(&ch, 0, sizeof ch);
    ch.start = 0; ch.end = 32;
    if (include) {
        int64_t lo = INT64_MAX, hi = 0;
        for (auto& r : pc.recs) { lo = std::min<int64_t>(lo, r.pos); hi = std::max<int64_t>(hi, r.end); }
        if (lo < 0) lo = 0;
        if (hi <= lo) hi = lo + 1;
        ch.start = (uint32_t)lo; ch.end = (uint32_t)hi;
        include->bitmaps(tid, ch.start, ch.end, fpos, fneg);
        ch.focus_pos = fpos->data(); ch.focus_neg = fneg->data();
    }
    ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
    if (mkp_upload_chunk(ctx, &ch)) throw std::runtime_error(mkp_last_error(ctx));
}

// Fills hist[4][MKP_HIST_BINS]; returns number of reads selected
inline size_t sample_histogram(const BamReader& bam, mkp_ctx* ctx, const SamplerConfig& cfg, uint64_t* hist, uint64_t* inexact, std::vector<SampledChunk>* keep = nullptr) {
    int region_tid = -1;
    if (cfg.region) {
        for (size_t i = 0; i < bam.ref_names.size(); i++) if (bam.ref_names[i] == cfg.region->name) region_tid = (int)i;
        if (region_tid < 0) throw std::runtime_error("did not find target_id for region in header");
    }
    uint64_t total_mapped = 0, total_unmapped = 0;
    std::map<uint32_t, uint64_t> mapped;
    for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
        if (cfg.region && (int)t != region_tid) continue;
        if (!cfg.region && cfg.include && !cfg.include->has_contig(t)) continue;
        mapped[t] = bam.stats.n_mapped[t];
        total_mapped += bam.stats.n_mapped[t];
        total_unmapped += bam.stats.n_unmapped[t];
    }
    if (!cfg.region) total_unmapped += bam.stats.n_no_coor;
    const uint64_t total = cfg.include_unmapped ? total_mapped + total_unmapped : total_mapped;
    if (!total) throw std::runtime_error("zero reads found in bam index");
    std::map<uint32_t, int64_t> quota;   // -1 = all
    for (auto& kv : mapped) {
        if (!kv.second) continue;
        if (cfg.take_all) { quota[kv.first] = -1; continue; }
        const float frac = (float)kv.second / (float)total;
        quota[kv.first] = (int64_t)std::min<uint64_t>((uint64_t)std::ceil((float)cfg.num_reads * frac), kv.second);
    }
    std::vector<RefTarget> contigs;
    std::map<uint32_t, uint32_t> contig_len;
    for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
        if (!quota.count(t)) continue;
        RefTarget c{t, 0, bam.ref_lens[t], bam.ref_names[t]};
        if (cfg.region) { c.start = cfg.region->start; c.length = cfg.region->end - cfg.region->start; }
        contigs.push_back(c);
        contig_len[t] = c.length;
    }
    std::vector<std::vector<size_t>> groups;
    std::vector<RefInterval> ivs;
    if (!contigs.empty()) ivs = reference_intervals(contigs, cfg.sampling_interval_size, false, nullptr, &groups);
    const size_t B = std::max<size_t>(1, (size_t)std::floor((float)cfg.threads * 1.5f));
    const bool only_mapped = !cfg.include_unmapped;
    std::map<uint32_t, size_t> so_far;
    std::unordered_set<uint64_t> selected_ids;     // record identity = offset in the stream
    PackedChunk cand;
    std::vector<uint8_t> contributes, take;
    std::vector<uint32_t> fpos, fneg;
    std::vector<uint64_t> batch_hist(4 * MKP_HIST_BINS);
    memset(hist, 0, 4 * MKP_HIST_BINS * sizeof(uint64_t));
    if (inexact) *inexact = 0;

    // One device pass decides which candidate reads contribute (MODE_HIST without a histogram); a second pass over the
    // same resident chunk adds the values of the newly selected reads to the histogram.
    auto upload = [&](PackedChunk& pc, uint32_t tid) {
        mkp_chunk ch;
        memset(&ch, 0, sizeof ch);
        ch.start = 0; ch.end = 32;
        if (cfg.include) {
            // chunk range = span of the candidates, bitmaps = the include-bed of this contig
            int64_t lo = INT64_MAX, hi = 0;
            for (auto& r : pc.recs) { lo = std::min<int64_t>(lo, r.pos); hi = std::max<int64_t>(hi, r.end); }
            if (lo < 0) lo = 0;
            if (hi <= lo) hi = lo + 1;
            ch.start = (uint32_t)lo; ch.end = (uint32_t)hi;
            cfg.include->bitmaps(tid, ch.start, ch.end, &fpos, &fneg);
            ch.focus_pos = fpos.data(); ch.focus_neg = fneg.data();
        }
        if (bam.on_device) { device_chunk(bam, pc.recs, ch.start, ch.end, ch.focus_pos, ch.focus_neg); return; }
        ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
        if (mkp_upload_chunk(ctx, &ch)) throw std::runtime_error(mkp_last_error(ctx));
    };
    // candidate records: sliced on the host (pack_record) or, with the device ingest, only listed (sliced on the GPU)
    auto add_candidate = [&](const RecRef& r) { if (!bam.on_device) pack_record(bam.rec(r), r.size, &cand); cand.recs.push_back(r); };
    auto decode_contributes = [&](PackedChunk& pc, uint32_t tid) {
        contributes.assign(pc.recs.size(), 0);
        if (pc.recs.empty()) return;
        upload(pc, tid);
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, nullptr, nullptr, contributes.data(), nullptr)) throw std::runtime_error(mkp_last_error(ctx));
    };
    auto add_selected = [&]() {       // histogram of the reads flagged in `take` (resident chunk)
        bool any = false;
        for (uint8_t t : take) any = any || t;
        if (!any) return;
        uint64_t inx = 0;
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, take.data(), batch_hist.data(), nullptr, &inx)) throw std::runtime_error(mkp_last_error(ctx));
        for (int k = 0; k < 4 * MKP_HIST_BINS; k++) hist[k] += batch_hist[k];
        if (inexact) *inexact += inx;
    };

    struct Grp { uint32_t tid, start, end; int64_t n; };
    for (size_t sb = 0; sb < groups.size(); sb += B) {
        std::vector<size_t> coords;
        for (size_t k = sb; k < std::min(groups.size(), sb + B); k++) for (size_t i : groups[k]) coords.push_back(i);
        std::sort(coords.begin(), coords.end(), [&](size_t a, size_t b) { return ivs[a].tid != ivs[b].tid ? ivs[a].tid < ivs[b].tid : ivs[a].start < ivs[b].start; });
        std::map<uint32_t, uint32_t> len_c;
        for (size_t i : coords) len_c[ivs[i].tid] += ivs[i].end - ivs[i].start;
        std::map<uint32_t, int64_t> k_c;
        for (auto& kv : len_c) {
            auto q = quota.find(kv.first);
            if (q == quota.end()) continue;
            if (q->second < 0) { k_c[kv.first] = -1; continue; }
            const size_t done = so_far.count(kv.first) ? so_far[kv.first] : 0;
            if ((size_t)q->second <= done) continue;
            const float f = (float)kv.second / (float)contig_len[kv.first];
            k_c[kv.first] = (int64_t)std::ceil(f * (float)((size_t)q->second - done));
        }
        std::vector<Grp> todo;
        bool have = false;
        Grp slack{};
        for (size_t i : coords) {
            const RefInterval& iv = ivs[i];
            auto kc = k_c.find(iv.tid);
            if (kc == k_c.end()) continue;
            if (kc->second < 0) { todo.push_back({iv.tid, iv.start, iv.end, -1}); continue; }
            const float f = (float)(iv.end - iv.start) / (float)len_c[iv.tid];
            const int64_t x = (int64_t)std::ceil((float)kc->second * f);
            Grp cur{iv.tid, iv.start, iv.end, x};
            if (x < 50) {
                if (!have) { slack = cur; have = true; }
                else if (slack.tid == cur.tid) {
                    Grp m{cur.tid, std::min(slack.start, cur.start), std::max(slack.end, cur.end), slack.n + x};
                    if (m.n < 50) slack = m; else { todo.push_back(m); have = false; }
                } else { todo.push_back(slack); slack = cur; }
            } else if (have) {
                have = false;
                if (slack.tid == cur.tid) todo.push_back({cur.tid, std::min(slack.start, cur.start), std::max(slack.end, cur.end), slack.n + x});
                else { todo.push_back(slack); todo.push_back(cur); }
            } else todo.push_back(cur);
        }
        if (have) todo.push_back(slack);
        // candidates of one interval at a time: first n contributing records in file order; extend while short
        for (const Grp& g : todo) {
            if (cfg.include && !cfg.include->overlaps_any(g.tid, g.start, g.end)) continue;
            std::vector<RecRef> recs;
            bam.ensure_tid(g.tid);          // ranged device ingest: the contig's byte range becomes resident
            bam.for_overlapping(g.tid, g.start, g.end, [&](const RecRef& r) { if (sampler_flag_ok(r, only_mapped || cfg.edge_on)) recs.push_back(r); });
            size_t used = 0, cursor = 0;
            while (cursor < recs.size() && (g.n < 0 || used < (size_t)g.n)) {
                const size_t want = g.n < 0 ? recs.size() : std::min(recs.size(), cursor + (size_t)(g.n - (int64_t)used) * 2 + 32);
                cand.clear();
                for (size_t k = cursor; k < want; k++) add_candidate(recs[k]);
                decode_contributes(cand, g.tid);
                take.assign(cand.recs.size(), 0);
                for (size_t k = 0; k < cand.recs.size() && (g.n < 0 || used < (size_t)g.n); k++) {
                    if (!contributes[k]) continue;
                    used++;
                    if (selected_ids.insert(cand.recs[k].off).second) take[k] = 1;
                }
                add_selected();
                if (keep && !bam.on_device) { bool any = false; for (uint8_t x : take) any = any || x; if (any) keep->push_back({cand, take, g.tid}); }
                cursor = want;
            }
            so_far[g.tid] += used;
        }
    }
    if (!only_mapped) {   // reads without coordinates (reads_sampler/mod.rs:85-129)
        const size_t limit = cfg.take_all ? (size_t)-1 : (cfg.num_reads > selected_ids.size() ? cfg.num_reads - selected_ids.size() : 0);
        cand.clear();
        bam.ensure_unplaced();
        for (auto& r : bam.unplaced) if (sampler_flag_ok(r, cfg.edge_on)) add_candidate(r);
        if (!cand.recs.empty()) {
            decode_contributes(cand, 0);
            take.assign(cand.recs.size(), 0);
            size_t used = 0;
            for (size_t k = 0; k < cand.recs.size() && used < limit; k++) {
                if (!contributes[k]) continue;
                used++;
                if (selected_ids.insert(cand.recs[k].off).second) take[k] = 1;
            }
            add_selected();
            if (keep && !bam.on_device) keep->push_back({cand, take, 0});
        }
    }
    return selected_ids.size();
}

// ---- the same schedule on an indexed file, without the per-group device round trips -----------------------------
// The candidates come straight from the file (BamReader::fetch_*: BAI linear index + zlib on the few members that hold
// them), so the sampler does not depend on what is resident on the device, and the per-contig state of the schedule
// (`so_far`) makes contigs independent: in an interval-sharded run every rank samples the contigs it owns and the
// histograms are summed once (SURVEY 8e). Per contig the schedule is first simulated under the assumption that every group
// finds its quota (true whenever the coverage is not tiny); the candidates of all planned groups are fetched in parallel,
// decoded in ONE device pass, and the real schedule then consumes them in order. A group that deviates from the plan, or
// needs more candidates than were fetched, falls back to fetching and decoding on demand - the result is the same reads
// either way: the first n contributing records of every group, in file order.
struct Collective {          // sum over the ranks of a sharded run (in place); world == 1: nothing to do
    int rank = 0, world = 1;
    int (*allreduce_sum)(uint64_t* buf, size_t n, void* user) = nullptr;
    void* user = nullptr;
    void sum(uint64_t* buf, size_t n) const {
        if (world <= 1) return;
        if (!allreduce_sum || allreduce_sum(buf, n, user) != 0) throw std::runtime_error("collective (all-reduce) failed");
    }
};

inline void append_packed(const PackedChunk& src, PackedChunk* dst) {
    const uint64_t base = (dst->heap.size() + 15) & ~(uint64_t)15;
    dst->heap.resize(base);
    dst->heap.insert(dst->heap.end(), src.heap.begin(), src.heap.end());
    for (auto h : src.hdrs) { h.off += base; dst->hdrs.push_back(h); }
    dst->recs.insert(dst->recs.end(), src.recs.begin(), src.recs.end());
}

inline size_t sample_histogram_indexed(const BamReader& bam, mkp_ctx* ctx, const SamplerConfig& cfg, uint64_t* hist, uint64_t* inexact,
                                       const Collective& coll, double* fetch_s = nullptr, std::vector<SampledChunk>* keep = nullptr) {
    using clk = std::chrono::steady_clock;
    int region_tid = -1;
    if (cfg.region) {
        for (size_t i = 0; i < bam.ref_names.size(); i++) if (bam.ref_names[i] == cfg.region->name) region_tid = (int)i;
        if (region_tid < 0) throw std::runtime_error("did not find target_id for region in header");
    }
    uint64_t total_mapped = 0, total_unmapped = 0;
    std::map<uint32_t, uint64_t> mapped;
    for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
        if (cfg.region && (int)t != region_tid) continue;
        if (!cfg.region && cfg.include && !cfg.include->has_contig(t)) continue;
        mapped[t] = bam.stats.n_mapped[t];
        total_mapped += bam.stats.n_mapped[t];
        total_unmapped += bam.stats.n_unmapped[t];
    }
    if (!cfg.region) total_unmapped += bam.stats.n_no_coor;
    const uint64_t total = cfg.include_unmapped ? total_mapped + total_unmapped : total_mapped;
    if (!total) throw std::runtime_error("zero reads found in bam index");
    std::map<uint32_t, int64_t> quota;   // -1 = all
    for (auto& kv : mapped) {
        if (!kv.second) continue;
        if (cfg.take_all) { quota[kv.first] = -1; continue; }
        const float frac = (float)kv.second / (float)total;
        quota[kv.first] = (int64_t)std::min<uint64_t>((uint64_t)std::ceil((float)cfg.num_reads * frac), kv.second);
    }
    std::vector<RefTarget> contigs;
    std::map<uint32_t, uint32_t> contig_len;
    for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
        if (!quota.count(t)) continue;
        RefTarget c{t, 0, bam.ref_lens[t], bam.ref_names[t]};
        if (cfg.region) { c.start = cfg.region->start; c.length = cfg.region->end - cfg.region->start; }
        contigs.push_back(c);
        contig_len[t] = c.length;
    }
    std::vector<std::vector<size_t>> groups;
    std::vector<RefInterval> ivs;
    if (!contigs.empty()) ivs = reference_intervals(contigs, cfg.sampling_interval_size, false, nullptr, &groups);
    const size_t B = std::max<size_t>(1, (size_t)std::floor((float)cfg.threads * 1.5f));
    const bool only_mapped = !cfg.include_unmapped;
    // super-batch structure: per super-batch and contig, the contig's intervals (position order) and their total length
    struct SbC { std::vector<size_t> iv; uint32_t len = 0; };
    std::vector<std::map<uint32_t, SbC>> sbs;
    for (size_t sb = 0; sb < groups.size(); sb += B) {
        std::vector<size_t> coords;
        for (size_t k = sb; k < std::min(groups.size(), sb + B); k++) for (size_t i : groups[k]) coords.push_back(i);
        std::sort(coords.begin(), coords.end(), [&](size_t a, size_t b) { return ivs[a].tid != ivs[b].tid ? ivs[a].tid < ivs[b].tid : ivs[a].start < ivs[b].start; });
        std::map<uint32_t, SbC> m;
        for (size_t i : coords) { SbC& c = m[ivs[i].tid]; c.iv.push_back(i); c.len += ivs[i].end - ivs[i].start; }
        sbs.push_back(std::move(m));
    }
    struct Grp { uint32_t tid, start, end; int64_t n; };
    // groups of contig t in super-batch s given the reads sampled from the contig so far (sampling_schedule.rs:171-615)
    auto todo_for = [&](size_t s, uint32_t t, size_t done) {
        std::vector<Grp> todo;
        auto sc = sbs[s].find(t);
        auto q = quota.find(t);
        if (sc == sbs[s].end() || q == quota.end()) return todo;
        int64_t kc;
        if (q->second < 0) kc = -1;
        else {
            if ((size_t)q->second <= done) return todo;
            const float f = (float)sc->second.len / (float)contig_len[t];
            kc = (int64_t)std::ceil(f * (float)((size_t)q->second - done));
        }
        bool have = false;
        Grp slack{};
        for (size_t i : sc->second.iv) {
            const RefInterval& iv = ivs[i];
            if (kc < 0) { todo.push_back({iv.tid, iv.start, iv.end, -1}); continue; }
            const float f = (float)(iv.end - iv.start) / (float)sc->second.len;
            const int64_t x = (int64_t)std::ceil((float)kc * f);
            Grp cur{iv.tid, iv.start, iv.end, x};
            if (x < 50) {
                if (!have) { slack = cur; have = true; }
                else {
                    Grp m{cur.tid, std::min(slack.start, cur.start), std::max(slack.end, cur.end), slack.n + x};
                    if (m.n < 50) slack = m; else { todo.push_back(m); have = false; }
                }
            } else if (have) {
                have = false;
                todo.push_back({cur.tid, std::min(slack.start, cur.start), std::max(slack.end, cur.end), slack.n + x});
            } else todo.push_back(cur);
        }
        if (have) todo.push_back(slack);
        return todo;
    };
    // contig -> rank: largest contigs first onto the least loaded rank (identical on every rank)
    std::map<uint32_t, int> owner;
    {
        std::vector<std::pair<uint64_t, uint32_t>> order;
        for (auto& kv : quota) order.push_back({mapped[kv.first], kv.first});
        std::sort(order.begin(), order.end(), [](auto& a, auto& b) { return a.first != b.first ? a.first > b.first : a.second < b.second; });
        std::vector<uint64_t> load(std::max(1, coll.world), 0);
        for (auto& o : order) { int r = 0; for (int k = 1; k < coll.world; k++) if (load[k] < load[r]) r = k; owner[o.second] = r; load[r] += o.first + 1; }
    }
    memset(hist, 0, 4 * MKP_HIST_BINS * sizeof(uint64_t));
    uint64_t inexact_local = 0, n_selected = 0;
    std::vector<uint64_t> batch_hist(4 * MKP_HIST_BINS);
    std::vector<uint32_t> fpos, fneg;
    double t_fetch = 0;
    const bool req_mapped = only_mapped || cfg.edge_on;

    auto upload = [&](PackedChunk& pc, uint32_t tid) {
        mkp_chunk ch;
        memset(&ch, 0, sizeof ch);
        ch.start = 0; ch.end = 32;
        if (cfg.include) {
            int64_t lo = INT64_MAX, hi = 0;
            for (auto& r : pc.recs) { lo = std::min<int64_t>(lo, r.pos); hi = std::max<int64_t>(hi, r.end); }
            if (lo < 0) lo = 0;
            if (hi <= lo) hi = lo + 1;
            ch.start = (uint32_t)lo; ch.end = (uint32_t)hi;
            cfg.include->bitmaps(tid, ch.start, ch.end, &fpos, &fneg);
            ch.focus_pos = fpos.data(); ch.focus_neg = fneg.data();
        }
        ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
        if (mkp_upload_chunk(ctx, &ch)) throw std::runtime_error(mkp_last_error(ctx));
    };
    auto contributes_of = [&](PackedChunk& pc, uint32_t tid, std::vector<uint8_t>* contributes) {
        contributes->assign(pc.recs.size(), 0);
        if (pc.recs.empty()) return;
        upload(pc, tid);
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, nullptr, nullptr, contributes->data(), nullptr)) throw std::runtime_error(mkp_last_error(ctx));
    };
    auto add_taken = [&](const std::vector<uint8_t>& take) {     // histogram of the flagged reads of the resident chunk
        bool any = false;
        for (uint8_t t : take) any = any || t;
        if (!any) return;
        uint64_t inx = 0;
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, take.data(), batch_hist.data(), nullptr, &inx)) throw std::runtime_error(mkp_last_error(ctx));
        for (int k = 0; k < 4 * MKP_HIST_BINS; k++) hist[k] += batch_hist[k];
        inexact_local += inx;
    };
    auto key_of = [](const Grp& g) { return std::to_string(g.tid) + ":" + std::to_string(g.start) + "-" + std::to_string(g.end) + "/" + std::to_string(g.n); };

    struct Planned { Grp g; BamReader::FetchCursor cur; PackedChunk pc; size_t lo = 0, hi = 0; bool used = false; };
    struct ContigPlan { uint32_t tid = 0; std::vector<Planned> plan; size_t bulk = 0; };
    struct Bulk { PackedChunk pc; std::vector<uint8_t> contributes, take; uint32_t tid = 0; };
    struct Heavy { std::vector<ContigPlan> cps; std::vector<Bulk> bulks; };
    auto heavy = std::make_shared<Heavy>();
    std::vector<ContigPlan>& cps = heavy->cps;
    // ---- plan every owned contig under "every group finds its quota"
    for (auto& c : contigs) {
        const uint32_t t = c.tid;
        if (owner[t] != coll.rank) continue;
        ContigPlan cp;
        cp.tid = t;
        size_t done = 0;
        for (size_t s = 0; s < sbs.size(); s++) for (const Grp& g : todo_for(s, t, done)) {
            if (cfg.include && !cfg.include->overlaps_any(g.tid, g.start, g.end)) continue;
            Planned p; p.g = g; cp.plan.push_back(std::move(p));
            if (g.n >= 0) done += (size_t)g.n;
        }
        cps.push_back(std::move(cp));
    }
    // ---- fetch the candidates of all planned groups of all contigs (parallel over groups)
    const auto tf0 = clk::now();
    {
        std::vector<Planned*> all;
        for (auto& cp : cps) for (auto& p : cp.plan) all.push_back(&p);
        std::atomic<size_t> next{0};
        std::exception_ptr err;
        std::mutex mu;
        auto work = [&]() {
            try {
                std::vector<RecRef> recs;
                for (;;) {
                    const size_t i = next.fetch_add(1);
                    if (i >= all.size()) break;
                    Planned& p = *all[i];
                    p.cur = bam.fetch_begin(p.g.tid, p.g.start, p.g.end);
                    const size_t want = p.g.n < 0 ? (size_t)-1 : (size_t)p.g.n * 2 + 32;
                    // packed right after each fetch: record bytes live in the cursor's buffer until the next fetch_more
                    while (!p.cur.done && p.pc.recs.size() < want) {
                        recs.clear();
                        bam.fetch_more(p.cur, std::min<size_t>(want - p.pc.recs.size(), 4096), [&](const RecRef& r) { return sampler_flag_ok(r, req_mapped); }, &recs);
                        for (auto& r : recs) { pack_record(p.cur.bytes(r), r.size, &p.pc); p.pc.recs.push_back(r); }
                    }
                }
            } catch (...) { std::lock_guard<std::mutex> g(mu); if (!err) err = std::current_exception(); }
        };
        const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, cfg.workers), all.size()));
        std::vector<std::thread> th;
        for (int k = 1; k < nt; k++) th.emplace_back(work);
        work();
        for (auto& x : th) x.join();
        if (err) std::rethrow_exception(err);
    }
    // ---- one resident chunk for all of them (one per contig with --include-bed: its bitmaps are per contig), one decode pass each
    std::vector<Bulk>& bulks = heavy->bulks;
    for (auto& cp : cps) {
        if (bulks.empty() || cfg.include) { bulks.emplace_back(); bulks.back().tid = cp.tid; }
        cp.bulk = bulks.size() - 1;
        Bulk& B = bulks.back();
        for (auto& p : cp.plan) { p.lo = B.pc.recs.size(); append_packed(p.pc, &B.pc); p.hi = B.pc.recs.size(); p.pc.clear(); p.pc.heap.shrink_to_fit(); p.pc.hdrs.shrink_to_fit(); }
    }
    t_fetch += secs_between(tf0, clk::now());
    trace_clock().mark(coll.rank, "sampler: candidates fetched + packed");
    if (cfg.device_ready) cfg.device_ready->wait();
    size_t resident_bulk = (size_t)-1;
    for (size_t bi = 0; bi < bulks.size(); bi++) { bulks[bi].take.assign(bulks[bi].pc.recs.size(), 0); contributes_of(bulks[bi].pc, bulks[bi].tid, &bulks[bi].contributes); resident_bulk = bi; }
    trace_clock().mark(coll.rank, "sampler: candidates decoded on the device");
    size_t n_on_demand = 0;
    // ---- the real schedule, contig by contig
    for (auto& cp : cps) {
        const uint32_t t = cp.tid;
        std::vector<Planned>& plan = cp.plan;
        Bulk& B = bulks[cp.bulk];
        std::map<std::string, size_t> by_key;
        for (size_t i = 0; i < plan.size(); i++) by_key.emplace(key_of(plan[i].g), i);
        std::unordered_set<uint64_t> selected;
        size_t done = 0;
        PackedChunk extra;
        std::vector<uint8_t> xcontrib, xtake;
        std::vector<RecRef> recs;
        for (size_t s = 0; s < sbs.size(); s++) for (const Grp& g : todo_for(s, t, done)) {
            if (cfg.include && !cfg.include->overlaps_any(g.tid, g.start, g.end)) continue;
            size_t used = 0;
            BamReader::FetchCursor own;
            BamReader::FetchCursor* curp = &own;
            auto it = by_key.find(key_of(g));
            if (it != by_key.end() && !plan[it->second].used) {
                Planned& p = plan[it->second];
                p.used = true;
                for (size_t k = p.lo; k < p.hi && (g.n < 0 || used < (size_t)g.n); k++) {
                    if (!B.contributes[k]) continue;
                    used++;
                    if (selected.insert(B.pc.recs[k].off).second) B.take[k] = 1;
                }
                curp = &p.cur;             // (stays with the plan: its buffers are released with the rest, see defer_free)
            } else own = bam.fetch_begin(g.tid, g.start, g.end);
            BamReader::FetchCursor& cur = *curp;
            // on demand: the plan did not cover the group, or the group needs more candidates than were fetched
            while (!cur.done && (g.n < 0 || used < (size_t)g.n)) {
                n_on_demand++;
                const size_t want = g.n < 0 ? 4096 : ((size_t)g.n - used) * 2 + 32;
                extra.clear();
                recs.clear();
                bam.fetch_more(cur, want, [&](const RecRef& r) { return sampler_flag_ok(r, req_mapped); }, &recs);
                for (auto& r : recs) { pack_record(cur.bytes(r), r.size, &extra); extra.recs.push_back(r); }
                if (extra.recs.empty()) continue;
                contributes_of(extra, t, &xcontrib);
                resident_bulk = (size_t)-1;
                xtake.assign(extra.recs.size(), 0);
                for (size_t k = 0; k < extra.recs.size() && (g.n < 0 || used < (size_t)g.n); k++) {
                    if (!xcontrib[k]) continue;
                    used++;
                    if (selected.insert(extra.recs[k].off).second) xtake[k] = 1;
                }
                add_taken(xtake);
                if (keep) { bool any = false; for (uint8_t x : xtake) any = any || x; if (any) keep->push_back({extra, xtake, t}); }
            }
            done += used;
        }
        n_selected += selected.size();
    }
    if (trace_clock().on) fprintf(stderr, "[mkh r%d]             sampler: %zu on-demand fetches during the replay\n", coll.rank, n_on_demand);
    trace_clock().mark(coll.rank, "sampler: schedule replayed");
    // ---- histogram of the selected reads of every bulk chunk
    for (size_t bi = 0; bi < bulks.size(); bi++) {
        Bulk& B = bulks[bi];
        bool any = false;
        for (uint8_t x : B.take) any = any || x;
        if (!any) continue;
        if (resident_bulk != bi) { upload(B.pc, B.tid); resident_bulk = bi; }
        add_taken(B.take);
        if (keep) keep->push_back({std::move(B.pc), std::move(B.take), B.tid});
    }
    trace_clock().mark(coll.rank, "sampler: histogram of the selection");
    if (!only_mapped) {   // reads without coordinates (reads_sampler/mod.rs:85-129): the last rank, after the global count is known
        uint64_t cnt[1] = {n_selected};
        coll.sum(cnt, 1);
        if (coll.rank == coll.world - 1) {
            const size_t limit = cfg.take_all ? (size_t)-1 : (cfg.num_reads > cnt[0] ? cfg.num_reads - (size_t)cnt[0] : 0);
            PackedChunk cand;
            BamReader::FetchCursor cur = bam.fetch_unplaced_begin();
            std::vector<RecRef> recs;
            while (!cur.done) {
                recs.clear();
                bam.fetch_more(cur, 4096, [&](const RecRef& r) { return sampler_flag_ok(r, cfg.edge_on); }, &recs);
                for (auto& r : recs) { pack_record(cur.bytes(r), r.size, &cand); cand.recs.push_back(r); }
            }
            if (!cand.recs.empty()) {
                std::vector<uint8_t> contributes, take(cand.recs.size(), 0);
                contributes_of(cand, 0, &contributes);
                size_t used = 0;
                for (size_t k = 0; k < cand.recs.size() && used < limit; k++) { if (!contributes[k]) continue; used++; take[k] = 1; }
                add_taken(take);
                n_selected += used;
                if (keep && used) keep->push_back({std::move(cand), std::move(take), 0});
            }
        }
    }
    // ---- the one exchange of a sharded run: sum of the histograms (+ the inexact-value count and the read count)
    if (coll.world > 1) {
        std::vector<uint64_t> buf(4 * MKP_HIST_BINS + 2);
        memcpy(buf.data(), hist, 4 * MKP_HIST_BINS * sizeof(uint64_t));
        buf[4 * MKP_HIST_BINS] = inexact_local; buf[4 * MKP_HIST_BINS + 1] = n_selected;
        coll.sum(buf.data(), buf.size());
        memcpy(hist, buf.data(), 4 * MKP_HIST_BINS * sizeof(uint64_t));
        inexact_local = buf[4 * MKP_HIST_BINS]; n_selected = buf[4 * MKP_HIST_BINS + 1];
    }
    if (inexact) *inexact = inexact_local;
    if (fetch_s) *fetch_s = t_fetch;
    if (cfg.defer_free) *cfg.defer_free = heavy;
    return (size_t)n_selected;
}

// htslib bam_plp_push with maxcnt (sam.c): the engine drops the reads of its flag mask first (they never count), keeps the
// first read of every start position, and drops a further read of the same start position when its buffer already holds
// `maxcnt` reads. The buffer holds the kept reads whose end lies at or after the current start (a read is released when the
// column at its end position is built). `recs`: the records fetched for ONE interval, file order; filtered in place.
inline void depth_limit_keep(std::vector<RecRef>* recs, uint32_t maxcnt) {
    if (!maxcnt || recs->size() <= maxcnt) return;
    std::vector<int32_t> ends;          // min-heap of the ends of the kept reads still in the buffer
    auto cmp = [](int32_t a, int32_t b) { return a > b; };
    int64_t cur = INT64_MIN;
    size_t w = 0;
    for (size_t i = 0; i < recs->size(); i++) {
        const RecRef& r = (*recs)[i];
        if (r.flag & (0x4 | 0x100 | 0x200 | 0x400)) { (*recs)[w++] = r; continue; }      // masked: never enters the buffer (and is not admitted later either)
        bool keep = true;
        if (r.pos != cur) {
            cur = r.pos;
            while (!ends.empty() && ends.front() < r.pos) { std::pop_heap(ends.begin(), ends.end(), cmp); ends.pop_back(); }
        } else if (ends.size() + 1 > maxcnt) keep = false;
        if (keep) { ends.push_back(r.end); std::push_heap(ends.begin(), ends.end(), cmp); (*recs)[w++] = r; }
    }
    recs->resize(w);
}

struct RunSummary {
    uint64_t positions = 0, rows = 0, reads_packed = 0, algorithmic_bytes = 0, chunks = 0;
    uint64_t rows_total = 0, positions_total = 0;      // over all ranks of a sharded run
    double fetch_s = 0;                                // threshold sampler: host fetch of the candidates
    double slice_s = 0, pass_s = 0, rowcopy_s = 0;     // parts of gpu_s: GPU slicing + upload of focus, kernels, rows to the host
    double load_s = 0, threshold_s = 0, interval_s = 0, pack_s = 0, gpu_s = 0, write_s = 0, total_s = 0, kernel_ms = 0;
    float thresholds[4] = {0, 0, 0, 0};
    bool threshold_set[4] = {false, false, false, false};
};

// Interval-sharded runs (SURVEY 8e): the reference intervals (feeder order) are cut into `world` contiguous ranges of about
// equal weight = compressed BAM bytes under the interval (BAI linear index) plus a small term for its length. Every rank
// computes the same cuts; cuts lie on interval boundaries, so rows and focus sets do not depend on the number of ranks.
inline std::vector<size_t> shard_cuts(const BamReader& bam, const std::vector<RefInterval>& ivs, int world) {
    std::vector<double> cum(ivs.size() + 1, 0.0);
    for (size_t i = 0; i < ivs.size(); i++) {
        double w = (double)(ivs[i].end - ivs[i].start) / 64.0;
        if (bam.have_index()) {
            const uint64_t a = bam.approx_file_offset(ivs[i].tid, ivs[i].start), b = bam.approx_file_offset(ivs[i].tid, ivs[i].end);
            if (b > a) w += (double)(b - a);
        }
        cum[i + 1] = cum[i] + w;
    }
    std::vector<size_t> cuts(world + 1, ivs.size());
    cuts[0] = 0;
    for (int r = 1; r < world; r++) {
        const double want = cum.back() * r / world;
        cuts[r] = (size_t)(std::lower_bound(cum.begin(), cum.end(), want) - cum.begin());
        cuts[r] = std::min(std::max(cuts[r], cuts[r - 1]), ivs.size());
    }
    return cuts;
}

inline int run_pileup(const PileupOptions& o, RunSummary* summary, std::string* error, const Collective* coll_in = nullptr) {
    using clk = std::chrono::steady_clock;
    auto secs = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double>(b - a).count(); };
    const Collective coll = coll_in ? *coll_in : Collective();
    const bool sharded = coll.world > 1;
    try {
        const auto t0 = clk::now();
        trace_clock().epoch = t0;
        auto trace = [&](const char* what) { trace_clock().mark(coll.rank, what); };
        if (o.percentile > 1.0f) throw std::runtime_error("filter percentile must be <= 1.0");
        MotifSpec hemi_m;
        if (o.hemi) hemi_m = hemi_motif(o);
        const int32_t hemi_partner = o.hemi ? hemi_m.rc_offset - hemi_m.offset : 0;     // MotifInfo::negative_strand_position
        // the device comes first: with the device ingest (default) the BAM is inflated and sliced on the GPU
        DeviceGuard dev;
        {
            const int rc = mkp_create(o.device, &dev.ctx);
            if (rc) throw std::runtime_error("no usable CUDA device (mkp_create returned " + std::to_string(rc) + "); this build has no CPU fallback");
        }
        trace("device context created");
        BamReader bam;
        // util.rs:690-712
        for (size_t i = 0; i < o.partition_tags.size(); i++) {
            if (o.partition_tags[i].size() != 2) throw std::runtime_error("illegal tag " + o.partition_tags[i] + " should be length 2");
            for (size_t j = 0; j < i; j++) if (o.partition_tags[j] == o.partition_tags[i]) throw std::runtime_error("cannot repeat partition-tags, got " + o.partition_tags[i] + " twice");
        }
        const bool partitioned = !o.partition_tags.empty();
        const bool to_dir = partitioned || o.bedgraph;     // the output path is a directory (writers.rs:264-381, 1005-1082)
        if (to_dir && o.header) throw std::runtime_error("the argument '--header' cannot be used with '--bedgraph' / '--partition-tag'");
        if (o.bedgraph && o.mixed) throw std::runtime_error("the argument '--mixed-delim' cannot be used with '--bedgraph'");
        if (sharded && (to_dir || o.host_ingest)) throw std::runtime_error("multi-GPU runs write one bedMethyl file through the device ingest: --bedgraph / --partition-tag / --host-ingest need a single device");
        if (sharded && (o.out_bed == "-" || o.out_bed == "stdout")) throw std::runtime_error("multi-GPU runs need an output file (ranks write their slices at their offsets)");
        // (partition keys: the tag values come from the device-resident records, mkp_bam_tags; --host-ingest reads them on the host)
        bool loaded = false;
        if (o.host_ingest) { bam.open(o.in_bam, o.threads); loaded = true; }
        else bam.open_device_index(o.in_bam, dev.ctx);         // header + index; the device load follows once the shard is known
        Region region, sregion;
        const Region* rp = nullptr; const Region* srp = nullptr;
        if (!o.region.empty()) { region = parse_region_arg(o.region, bam); rp = &region; }
        if (!o.sample_region.empty()) { sregion = parse_region_arg(o.sample_region, bam); srp = &sregion; }
        std::vector<RefTarget> targets;
        for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
            if (rp) { if (bam.ref_names[t] == rp->name) targets.push_back({t, rp->start, rp->end - rp->start, rp->name}); }
            else targets.push_back({t, 0, bam.ref_lens[t], bam.ref_names[t]});
        }
        IncludeBed include;
        const IncludeBed* inc = nullptr;
        if (!o.include_bed.empty()) {
            std::map<std::string, uint32_t> name_to_tid;
            for (auto& t : targets) name_to_tid[t.name] = t.tid;
            include.read(o.include_bed, name_to_tid);
            inc = &include;
        }
        bool combine_strands = o.combine_strands || o.hemi;        // pileup-hemi: the feeder runs in combine-strands mode
        if (combine_strands && !(o.cpg || !o.motif_parts.empty())) throw std::runtime_error("need to specify either --motif or --cpg to combine strands");

        mkp_params P;
        memset(&P, 0, sizeof P);
        P.force_allow_implicit = o.force_allow;
        P.max_depth = o.max_depth;
        if (o.traditional) { P.numeric_mode = 2; P.collapse_code = 'h'; combine_strands = true; }
        else if (o.combine_mods) P.numeric_mode = 1;
        else if (!o.ignore.empty()) { uint32_t c; if (!parse_code(o.ignore, &c)) throw std::runtime_error("failed to parse mod code " + o.ignore); P.numeric_mode = 2; P.collapse_code = c; }
        if (!o.edge.empty()) {
            P.edge_filter_on = 1; P.edge_filter_inverted = o.invert_edge;
            auto c = o.edge.find(',');
            if (c == std::string::npos) P.edge_filter_start = P.edge_filter_end = (uint32_t)std::stoul(o.edge);
            else { P.edge_filter_start = (uint32_t)std::stoul(o.edge.substr(0, c)); P.edge_filter_end = (uint32_t)std::stoul(o.edge.substr(c + 1)); }
        }
        // motifs (subcommand.rs:526-539, 592-612)
        std::vector<std::string> parts = o.motif_parts;
        MotifContext mc;
        bool have_motifs = false;
        if (o.hemi) { mc.motifs.push_back(hemi_m); have_motifs = true; }
        else if (!parts.empty()) {
            if (o.traditional) throw std::runtime_error("cannot use presets and motifs together");
            if (parts.size() % 2) throw std::runtime_error("illegal number of parts for motif");
            for (size_t i = 0; i < parts.size(); i += 2) for (size_t j = i + 2; j < parts.size(); j += 2)
                if (parts[i] == parts[j] && parts[i + 1] == parts[j + 1]) throw std::runtime_error("cannot have the same motif more than once");
            bool cg0 = false;
            for (size_t i = 0; i < parts.size(); i += 2) cg0 = cg0 || (parts[i] == "CG" && parts[i + 1] == "0");
            if (o.cpg && !cg0) { parts.push_back("CG"); parts.push_back("0"); }
            for (size_t i = 0; i < parts.size(); i += 2) mc.motifs.push_back(parse_motif(parts[i], std::stoi(parts[i + 1])));
            have_motifs = true;
        } else if (o.traditional || o.cpg) { mc.motifs.push_back(parse_motif("CG", 0)); have_motifs = true; }
        BedFormat fmt;
        fmt.mixed_delim = o.mixed;
        for (auto& m : mc.motifs) fmt.motif_labels.push_back(m.label());
        if (have_motifs) {
            if (o.ref_fp.empty()) throw std::runtime_error("reference fasta is required for using --motif or --cpg options");
            if (combine_strands) for (auto& m : mc.motifs) if (!m.palindromic) throw std::runtime_error("cannot combine strands with a motif that is not a palindrome");
            mc.fasta.open(o.ref_fp);
            mc.keep_case = o.mask;
            mc.include = inc;
            for (auto& m : mc.motifs) mc.longest = std::max<uint64_t>(mc.longest, m.len);
        }
        // ---- reference intervals: boundaries now (cheap), focus positions of this rank's range in the background
        trace("index + fasta opened");
        const auto t_iv0 = clk::now();
        std::vector<RefTarget> iv_targets = targets;
        if (inc) iv_targets = targets_from_include_bed(*inc, iv_targets, o.interval_size);
        std::vector<size_t> iv_owner;
        std::vector<RefInterval> ivs = interval_grid(iv_targets, o.interval_size, combine_strands, have_motifs ? &mc : nullptr, &iv_owner);
        size_t my_i0 = 0, my_i1 = ivs.size();
        if (sharded) { const std::vector<size_t> cuts = shard_cuts(bam, ivs, coll.world); my_i0 = cuts[coll.rank]; my_i1 = cuts[coll.rank + 1]; }
        // ---- threshold estimation starts now when it can run beside the load: its candidates come straight from the file (host
        // fetch through the index), only its decode passes need the device and wait for `dev_ready`
        const bool estimate = o.filter_thresholds.empty() && !o.no_filtering;
        std::vector<uint64_t> bg_hist(4 * MKP_HIST_BINS);
        uint64_t bg_inexact = 0;
        double bg_fetch_s = 0;
        std::exception_ptr bg_err;
        std::promise<void> dev_ready_p;
        std::shared_future<void> dev_ready_f = dev_ready_p.get_future().share();
        bool dev_ready_set = false;
        SamplerConfig bg_sc;
        std::shared_ptr<void> bg_garbage;
        std::promise<void> bg_result_p;
        std::future<void> bg_result_f = bg_result_p.get_future();
        struct BgJoin { std::thread t; std::promise<void>* p; bool* set; ~BgJoin() { if (!*set) { try { p->set_value(); } catch (...) {} *set = true; } if (t.joinable()) t.join(); } } bg_job{std::thread(), &dev_ready_p, &dev_ready_set};
        trace("interval grid + shard cuts");
        const bool sampler_bg = estimate && !loaded && bam.have_index();
        if (sampler_bg) {
            if (o.have_frac && o.frac != 1.0) throw std::runtime_error("only --sampling-frac 1.0 is reproducible without the reference's RNG; use -n or -f 1.0");
            mkp_params PS = P;
            PS.max_depth = 0;           // the sampler looks at reads, not at pileup columns
            if (mkp_set_params(dev.ctx, &PS)) throw std::runtime_error(mkp_last_error(dev.ctx));
            bg_sc.threads = o.schedule_threads > 0 ? o.schedule_threads : o.threads; bg_sc.workers = o.threads; bg_sc.sampling_interval_size = o.sampling_interval_size;
            bg_sc.take_all = o.have_frac;
            bg_sc.num_reads = o.num_reads;
            bg_sc.region = srp ? srp : rp;
            bg_sc.include_unmapped = o.include_unmapped;
            bg_sc.edge_on = P.edge_filter_on;
            bg_sc.include = inc;
            bg_sc.device_ready = &dev_ready_f;
            bg_sc.defer_free = &bg_garbage;
            bg_job.t = std::thread([&]() {
                try { sample_histogram_indexed(bam, dev.ctx, bg_sc, bg_hist.data(), &bg_inexact, coll, &bg_fetch_s); }
                catch (...) { bg_err = std::current_exception(); }
                bg_result_p.set_value();           // the result is out; the candidate buffers are released after that, beside the pileup
                bg_garbage.reset();
            });
        }
        // ---- focus positions of this rank's intervals (reference motif scan), beside the load and the sampler. Every object the
        // job touches is declared above; its joiner is declared after them, so it is destroyed (joined) before they are.
        std::exception_ptr iv_err;
        double iv_secs = 0;
        struct Joiner { std::thread t; void join() { if (t.joinable()) t.join(); } ~Joiner() { join(); } } iv_job;
        iv_job.t = std::thread([&]() {
            try {
                fill_interval_focus(ivs, my_i0, my_i1, iv_targets, iv_owner, combine_strands, have_motifs ? &mc : nullptr, inc, std::max(1, o.threads / 2));
                iv_secs = secs(t_iv0, clk::now());
                trace("interval focus filled (background)");
            } catch (...) { iv_err = std::current_exception(); }
        });
        // ---- device load: everything, or the byte ranges under this rank's intervals
        if (!loaded) {
            if (sharded) {
                std::vector<BamReader::Piece> pieces;
                for (size_t i = my_i0; i < my_i1; i++) {
                    if (!pieces.empty() && pieces.back().tid == ivs[i].tid) pieces.back().hi = std::max(pieces.back().hi, ivs[i].end);
                    else pieces.push_back({ivs[i].tid, ivs[i].start, ivs[i].end});
                }
                bam.load_pieces(pieces);
            } else {
                try { bam.load_default(); }
                catch (const DeviceIngestTooBig& e) {
                    // a front-end choice, not a compute fallback: the reads are sliced on the host and uploaded chunk by chunk
                    if (!o.quiet) fprintf(stderr, "> %s; reading the BAM on the host instead\n", e.what());
                    bam = BamReader();
                    bam.open(o.in_bam, o.threads);
                }
            }
        }
        if (!dev_ready_set) { dev_ready_p.set_value(); dev_ready_set = true; }
        const auto t_load = clk::now();
        trace("device load done");
        if (trace_clock().on) fprintf(stderr, "[mkh r%d]             ingest: h2d %.1f ms, inflate %.1f ms, record walk %.1f ms, total %.1f ms\n", coll.rank, bam.ingest_ms[0], bam.ingest_ms[1], bam.ingest_ms[2], bam.ingest_ms[3]);
        uint64_t any_mapped = 0;
        for (auto& t : targets) if (rp || !inc || inc->has_contig(t.tid)) any_mapped += bam.stats.n_mapped[t.tid];
        if (!any_mapped) throw std::runtime_error("did not find any mapped reads, perform alignment first or use modkit extract and/or modkit summary to inspect unaligned modBAMs");
        // output first, like the reference, so a bad path fails before any work
        FILE* out = nullptr;
        struct Router {          // files of the output directory, created on first use
            std::string dir;
            std::map<std::string, FILE*> files;
            FILE* get(const std::string& name) {
                auto it = files.find(name);
                if (it != files.end()) return it->second;
                FILE* f = fopen((dir + "/" + name).c_str(), "w");
                if (!f) throw std::runtime_error("failed to make output file " + dir + "/" + name);
                files[name] = f;
                return f;
            }
            ~Router() { for (auto& kv : files) fclose(kv.second); }
        } router;
        std::string shard_text;      // sharded: this rank's slice of the output (header; the formatted parts follow in shard_parts), written at its offset at the end
        std::vector<std::string> shard_parts;
        int out_fd = -1;             // single regular output file: the formatting workers write their text at its offset (pwrite)
        uint64_t file_pos = 0;
        if (sharded) {
            if (coll.rank == 0) {
                FILE* f = fopen(o.out_bed.c_str(), "w");     // created (and truncated) by rank 0 before the first exchange
                if (!f) throw std::runtime_error("failed to make output file");
                fclose(f);
                if (o.header) shard_text += bed_header_line();
            }
        } else if (!to_dir) {
            out = (o.out_bed == "-" || o.out_bed == "stdout") ? stdout : fopen(o.out_bed.c_str(), "w");
            if (!out) throw std::runtime_error("failed to make output file");
            if (o.header) fputs(bed_header_line(), out);
            if (out != stdout) {
                fflush(out);
                struct stat sb;
                const off_t at = ftello(out);
                if (at >= 0 && fstat(fileno(out), &sb) == 0 && S_ISREG(sb.st_mode)) { out_fd = fileno(out); file_pos = (uint64_t)at; }
            }
        } else {
            std::error_code ec;
            std::filesystem::create_directories(o.out_bed, ec);
            if (ec) throw std::runtime_error("failed to create output directory " + o.out_bed);
            router.dir = o.out_bed;
        }
        const std::string pfx = o.prefix.empty() ? std::string() : o.prefix + "_";

        // thresholds (subcommand.rs:615-638, command_utils.rs:49-134)
        for (auto& raw : o.mod_thresholds) {
            auto c = raw.find(':');
            uint32_t code;
            if (c == std::string::npos || raw.find(':', c + 1) != std::string::npos || !parse_code(raw.substr(0, c), &code))
                throw std::runtime_error("encountered illegal per-mod threshold: " + raw + ". Should be mod_code:threshold e.g. h:0.8");
            if (P.n_mod_thresholds >= MKP_MAX_MOD_THRESHOLDS) throw std::runtime_error("too many per-mod thresholds");
            P.mod_code[P.n_mod_thresholds] = code;
            P.mod_threshold[P.n_mod_thresholds++] = std::stof(raw.substr(c + 1));
        }
        double fetch_s = 0;
        if (!o.filter_thresholds.empty()) {
            bool have_default = false;
            for (auto& raw : o.filter_thresholds) {
                auto c = raw.find(':');
                if (c == std::string::npos) {
                    if (have_default) throw std::runtime_error("default threshold encountered more than once");
                    P.default_threshold = std::stof(raw); have_default = true;
                } else {
                    const char* B = "ACGT";
                    const char* f = raw.empty() ? nullptr : strchr(B, raw[0]);
                    if (!f || !raw[0]) throw std::runtime_error("failed to parse base " + raw);
                    if (P.base_threshold_set[f - B]) throw std::runtime_error(std::string("repeated threshold for base ") + raw[0]);
                    P.base_threshold_set[f - B] = 1;
                    P.base_threshold[f - B] = std::stof(raw.substr(c + 1));
                }
            }
        } else if (!o.no_filtering && sampler_bg) {
            bg_result_f.wait();
            trace("sampler result");
            if (bg_err) std::rethrow_exception(bg_err);
            fetch_s = bg_fetch_s;
            if (bg_inexact) throw std::runtime_error("sampled probabilities are not multiples of 1/1024 (" + std::to_string(bg_inexact) + " values): exact histogram quantile impossible; pass --filter-threshold");
            for (int b = 0; b < 4; b++) {
                float thr;
                uint64_t n = 0;
                for (int k = 0; k < MKP_HIST_BINS; k++) n += bg_hist[b * MKP_HIST_BINS + k];
                if (!n) continue;
                if (!percentile_from_hist(bg_hist.data() + b * MKP_HIST_BINS, o.percentile, &thr)) throw std::runtime_error("not enough datapoints to estimate a threshold");
                P.base_threshold_set[b] = 1;
                P.base_threshold[b] = thr;
                if (!o.quiet && coll.rank == 0) fprintf(stderr, "> Using filter threshold %.9g for %c.\n", thr, "ACGT"[b]);
            }
        } else if (!o.no_filtering) {
            mkp_params PS = P;
            PS.max_depth = 0;           // the sampler looks at reads, not at pileup columns
            if (mkp_set_params(dev.ctx, &PS)) throw std::runtime_error(mkp_last_error(dev.ctx));
            SamplerConfig sc;
            sc.threads = o.schedule_threads > 0 ? o.schedule_threads : o.threads; sc.workers = o.threads; sc.sampling_interval_size = o.sampling_interval_size;
            if (o.have_frac) { if (o.frac != 1.0) throw std::runtime_error("only --sampling-frac 1.0 is reproducible without the reference's RNG; use -n or -f 1.0"); sc.take_all = true; }
            sc.num_reads = o.num_reads;
            sc.region = srp ? srp : rp;
            sc.include_unmapped = o.include_unmapped;
            sc.edge_on = P.edge_filter_on;
            sc.include = inc;
            std::vector<uint64_t> hist(4 * MKP_HIST_BINS);
            uint64_t inexact = 0;
            if (bam.on_device && bam.have_index()) sample_histogram_indexed(bam, dev.ctx, sc, hist.data(), &inexact, coll, &fetch_s);
            else {
                if (sharded) throw std::runtime_error("interval-sharded runs need a BAM index (.bai)");
                sample_histogram(bam, dev.ctx, sc, hist.data(), &inexact);
            }
            if (inexact) throw std::runtime_error("sampled probabilities are not multiples of 1/1024 (" + std::to_string(inexact) + " values): exact histogram quantile impossible; pass --filter-threshold");
            for (int b = 0; b < 4; b++) {
                float thr;
                uint64_t n = 0;
                for (int k = 0; k < MKP_HIST_BINS; k++) n += hist[b * MKP_HIST_BINS + k];
                if (!n) continue;
                if (!percentile_from_hist(hist.data() + b * MKP_HIST_BINS, o.percentile, &thr)) throw std::runtime_error("not enough datapoints to estimate a threshold");
                P.base_threshold_set[b] = 1;
                P.base_threshold[b] = thr;
                if (!o.quiet && coll.rank == 0) fprintf(stderr, "> Using filter threshold %.9g for %c.\n", thr, "ACGT"[b]);
            }
        }
        if (mkp_set_params(dev.ctx, &P)) throw std::runtime_error(mkp_last_error(dev.ctx));
        if (summary) for (int b = 0; b < 4; b++) { summary->thresholds[b] = P.base_threshold[b]; summary->threshold_set[b] = P.base_threshold_set[b]; }
        const auto t_thr = clk::now();
        trace("thresholds done");

        iv_job.join();
        if (iv_err) std::rethrow_exception(iv_err);
        const auto t_iv = clk::now();
        (void)t_iv;
        RunSummary S;
        S.fetch_s = fetch_s;
        if (sharded) { ivs.erase(ivs.begin() + (ptrdiff_t)my_i1, ivs.end()); ivs.erase(ivs.begin(), ivs.begin() + (ptrdiff_t)my_i0); }
        for (auto& iv : ivs) S.positions += iv.end - iv.start;

        // ---- two stages: a device thread selects the reads of chunk after chunk, slices them on the GPU, runs the pass and takes
        // the rows; this thread turns finished chunks into text (strand combining, formatting: parallel over intervals) and
        // writes them in order. The device works on chunk k + 1 while chunk k is being formatted.
        struct ChunkOut { size_t i0 = 0, i1 = 0; std::string key_name; std::vector<mkp_row> rows; std::vector<mkp_hemi_row> hemi_rows; bool last = false; };
        std::mutex q_mu;
        std::condition_variable q_cv;
        std::deque<ChunkOut> queue;
        std::vector<std::vector<mkp_row>> spare_rows;       // row buffers travel back to the device stage (no fresh pages per chunk)
        std::exception_ptr dev_err;
        bool consumer_gone = false;
        const bool want_alg_bytes = !o.stats_json.empty();
        auto push_out = [&](ChunkOut&& co) {
            std::unique_lock<std::mutex> lk(q_mu);
            q_cv.wait(lk, [&] { return queue.size() < 2 || consumer_gone; });
            queue.push_back(std::move(co));
            q_cv.notify_all();
        };
        auto device_stage = [&]() {
            try {
                PackedChunk pc;
                std::vector<uint32_t> fpos, fneg;
                for (size_t c0 = 0; c0 < ivs.size();) {
                    // a chunk = consecutive intervals of one contig up to chunk_bp
                    size_t c1 = c0 + 1;
                    while (c1 < ivs.size() && ivs[c1].tid == ivs[c0].tid && ivs[c1].start == ivs[c1 - 1].end && ivs[c1].end - ivs[c0].start <= o.chunk_bp) c1++;
                    if (ivs[c1 - 1].end <= ivs[c0].start) { c0 = c1; continue; }
                    // the reads of the chunk
                    std::vector<RecRef> chunk_recs;
                    bam.ensure_tid(ivs[c0].tid);
                    bam.for_overlapping(ivs[c0].tid, ivs[c0].start, ivs[c1 - 1].end, [&](const RecRef& r) { chunk_recs.push_back(r); });
                    if (chunk_recs.empty()) { c0 = c1; continue; }
                    // --max-depth (src/pileup/mod.rs:755-759 -> bam_plp_set_maxcnt): the pileup engine of the reference runs per interval
                    // and drops reads while its buffer is full, so the reads that count can differ from interval to interval. Only a
                    // chunk that holds more reads than the limit can be affected: it is then processed interval by interval, each with
                    // the reads its own engine would keep. (Parity unpinned by the reference's tests; rule restated in depth_limit_keep.)
                    struct Work { size_t a, b; std::vector<RecRef> recs; };
                    std::vector<Work> work;
                    bool split = false;
                    if (o.max_depth && chunk_recs.size() > o.max_depth) {
                        std::vector<Work> per_iv;
                        for (size_t k = c0; k < c1; k++) {
                            Work w{k, k + 1, {}};
                            for (auto& r : chunk_recs) if (r.pos < (int64_t)ivs[k].end && r.end > (int64_t)ivs[k].start) w.recs.push_back(r);
                            const size_t before = w.recs.size();
                            depth_limit_keep(&w.recs, o.max_depth);
                            split = split || w.recs.size() != before;
                            per_iv.push_back(std::move(w));
                        }
                        if (split) work.swap(per_iv);
                    }
                    if (!split) { Work w{c0, c1, {}}; w.recs.swap(chunk_recs); work.push_back(std::move(w)); }
                    for (auto& wk : work) {
                        const size_t i0 = wk.a, i1 = wk.b;
                        const uint32_t cs = ivs[i0].start, ce = ivs[i1 - 1].end;
                        if (ce <= cs || wk.recs.empty()) continue;
                        // pileup-hemi: the call window reaches the partner of every motif position; the reads stay those of the intervals
                        uint32_t wcs = cs, wce = ce;
                        if (hemi_partner < 0) wcs = cs - std::min<uint32_t>(cs, (uint32_t)-hemi_partner);
                        if (hemi_partner > 0) wce = (uint32_t)std::min<uint64_t>((uint64_t)ce + (uint32_t)hemi_partner, std::max(ce, bam.ref_lens[ivs[i0].tid]));
                        std::vector<RecRef>& all_recs = wk.recs;
                        // with --partition-tag one group per key (each an independent pileup: src/pileup/mod.rs:795-830), in key order
                        std::map<std::string, std::vector<RecRef>> groups;
                        if (!partitioned) groups[""].swap(all_recs);
                        else {
                            // only alignments the pileup admits create a key (flag filter of the pileup engine, pileup/mod.rs:783-791)
                            std::vector<RecRef> adm;
                            for (auto& r : all_recs) if (!((r.flag & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)) || r.l_seq == 0)) adm.push_back(r);
                            std::vector<uint8_t> cells;
                            const size_t n_pt = o.partition_tags.size();
                            if (bam.on_device && !adm.empty()) {
                                std::vector<uint32_t> ids(adm.size());
                                for (size_t k = 0; k < adm.size(); k++) ids[k] = adm[k].idx;
                                cells.resize(adm.size() * n_pt * MKP_TAG_CELL);
                                // four tags per call (mkp_bam_tags); the cells of a record are laid side by side in tag order
                                std::vector<uint8_t> part;
                                for (size_t t0 = 0; t0 < n_pt; t0 += 4) {
                                    const size_t nt4 = std::min<size_t>(4, n_pt - t0);
                                    std::string tg;
                                    for (size_t t = t0; t < t0 + nt4; t++) tg += o.partition_tags[t];
                                    part.resize(adm.size() * nt4 * MKP_TAG_CELL);
                                    if (mkp_bam_tags(dev.ctx, ids.data(), (uint32_t)ids.size(), tg.c_str(), (uint32_t)nt4, part.data())) throw std::runtime_error(mkp_last_error(dev.ctx));
                                    for (size_t k = 0; k < adm.size(); k++)
                                        memcpy(cells.data() + (k * n_pt + t0) * MKP_TAG_CELL, part.data() + k * nt4 * MKP_TAG_CELL, nt4 * MKP_TAG_CELL);
                                }
                            }
                            for (size_t k = 0; k < adm.size(); k++) {
                                std::string key;
                                const bool have = bam.on_device ? partition_key_of_cells(cells.data() + k * n_pt * MKP_TAG_CELL, n_pt, &key)
                                                                : partition_key_of(bam.rec(adm[k]), adm[k].size, o.partition_tags, &key);
                                groups[have ? key : std::string("\1")].push_back(adm[k]);
                            }
                        }
                        bool focus_done = false;
                        for (auto& grp : groups) {
                            const auto ta = clk::now();
                            pc.clear();
                            if (bam.on_device) pc.recs = grp.second;
                            else pack_records_mt(bam, grp.second, o.threads, &pc);
                            if (pc.recs.empty()) continue;
                            mkp_chunk ch;
                            memset(&ch, 0, sizeof ch);
                            ch.start = wcs; ch.end = wce; ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
                            if (have_motifs || inc) { if (!focus_done) { focus_bitmaps(ivs, i0, i1, wcs, wce, &fpos, &fneg); focus_done = true; } ch.focus_pos = fpos.data(); ch.focus_neg = fneg.data(); }
                            const auto tb = clk::now();
                            S.pack_s += secs(ta, tb);
                            const mkp_row* rows = nullptr;
                            const mkp_hemi_row* hemi_rows = nullptr;
                            size_t n_rows = 0;
                            mkp_stats st;
                            auto hemi_pass = [&]() {
                                std::vector<uint32_t> starts;
                                for (size_t k = i0; k < i1; k++) starts.push_back(ivs[k].start);
                                if (mkp_hemi_resident(dev.ctx, starts.data(), (uint32_t)starts.size(), hemi_partner, &st)) throw std::runtime_error(mkp_last_error(dev.ctx));
                            };
                            if (bam.on_device) {
                                // slice on the GPU (no packed chunk in host memory), then the same kernels
                                device_chunk(bam, pc.recs, wcs, wce, ch.focus_pos, ch.focus_neg);
                                const auto t_s = clk::now();
                                S.slice_s += secs(tb, t_s);
                                if (o.hemi) hemi_pass();
                                else if (mkp_pileup_resident(dev.ctx, &st)) throw std::runtime_error(mkp_last_error(dev.ctx));
                                const auto t_k = clk::now();
                                S.pass_s += secs(t_s, t_k);
                                if (o.hemi ? mkp_fetch_hemi_rows(dev.ctx, &hemi_rows, &n_rows) : mkp_fetch_rows(dev.ctx, &rows, &n_rows)) throw std::runtime_error(mkp_last_error(dev.ctx));
                                S.rowcopy_s += secs(t_k, clk::now());
                                if (want_alg_bytes) {
                                    pc.hdrs.resize(pc.recs.size());
                                    uint32_t nr = 0;
                                    if (mkp_fetch_chunk(dev.ctx, pc.hdrs.data(), &nr, nullptr, nullptr)) throw std::runtime_error(mkp_last_error(dev.ctx));
                                }
                            } else if (o.hemi) {
                                if (mkp_upload_chunk(dev.ctx, &ch)) throw std::runtime_error(mkp_last_error(dev.ctx));
                                hemi_pass();
                                if (mkp_fetch_hemi_rows(dev.ctx, &hemi_rows, &n_rows)) throw std::runtime_error(mkp_last_error(dev.ctx));
                            } else if (mkp_pileup_chunk(dev.ctx, &ch, &rows, &n_rows, &st)) throw std::runtime_error(mkp_last_error(dev.ctx));
                            ChunkOut co;
                            co.i0 = i0; co.i1 = i1;
                            co.key_name = !partitioned ? std::string() : (grp.first == "\1" ? std::string("ungrouped") : grp.first);
                            { std::lock_guard<std::mutex> lk(q_mu); if (!spare_rows.empty()) { co.rows.swap(spare_rows.back()); spare_rows.pop_back(); } }
                            if (o.hemi) co.hemi_rows.assign(hemi_rows, hemi_rows + n_rows);
                            else co.rows.assign(rows, rows + n_rows);          // the context's row buffer is reused by the next chunk
                            S.gpu_s += secs(tb, clk::now());
                            S.kernel_ms += st.kernel_ms[7];
                            S.reads_packed += pc.recs.size();
                            S.algorithmic_bytes += (want_alg_bytes || !bam.on_device ? pc.algorithmic_bytes() : 0) + (o.hemi ? sizeof(mkp_hemi_row) : sizeof(mkp_row)) * n_rows;
                            S.chunks++;
                            push_out(std::move(co));
                        }
                    }
                    c0 = c1;
                }
            } catch (...) { dev_err = std::current_exception(); }
            trace("device stage done");
            ChunkOut fin;
            fin.last = true;
            push_out(std::move(fin));
        };
        struct DevJoiner { std::thread t; std::mutex* mu; std::condition_variable* cv; bool* gone;
                           ~DevJoiner() { { std::lock_guard<std::mutex> g(*mu); *gone = true; } cv->notify_all(); if (t.joinable()) t.join(); } } dev_job{std::thread(), &q_mu, &q_cv, &consumer_gone};
        dev_job.t = std::thread(device_stage);
        WorkerPool pool(std::max(1, o.threads));
        std::vector<std::string> part_pool;
        for (;;) {
            ChunkOut co;
            {
                std::unique_lock<std::mutex> lk(q_mu);
                q_cv.wait(lk, [&] { return !queue.empty(); });
                co = std::move(queue.front());
                queue.pop_front();
                q_cv.notify_all();
            }
            if (co.last) break;
            const auto tc = clk::now();
            const size_t i0 = co.i0, i1 = co.i1;
            const mkp_row* rows = co.rows.data();
            const size_t n_rows = o.hemi ? co.hemi_rows.size() : co.rows.size();
            auto pos_of = [&](size_t j) { return o.hemi ? co.hemi_rows[j].pos : rows[j].pos; };
            const std::string& key_name = co.key_name;
            // rows are position sorted: every interval gets its slice; intervals are finished and formatted in parallel
            const std::string& chrom = bam.ref_names[ivs[i0].tid];
            const size_t n_iv = i1 - i0;
            std::vector<size_t> rlo(n_iv + 1);
            {
                size_t r0 = 0;
                for (size_t i = i0; i < i1; i++) { while (r0 < n_rows && pos_of(r0) < ivs[i].start) r0++; rlo[i - i0] = r0; }
                size_t r1 = rlo[n_iv - 1];
                while (r1 < n_rows && pos_of(r1) < ivs[i1 - 1].end) r1++;
                rlo[n_iv] = r1;
            }
            const int nt = std::max(1, std::min<int>(o.threads, (int)n_iv));
            std::vector<std::string>& parts = part_pool;
            if ((int)parts.size() < nt) parts.resize(nt);
            for (auto& ps : parts) ps.clear();                               // (capacity kept from the chunks before)
            std::vector<std::map<std::string, std::string>> routed(nt);      // to_dir: file name -> text, per worker
            std::vector<uint64_t> part_rows(nt, 0);
            const bool direct = out_fd >= 0 && !to_dir && !sharded;
            std::unique_ptr<std::atomic<uint64_t>[]> psize(new std::atomic<uint64_t>[nt]);
            for (int t = 0; t < nt; t++) psize[t].store(UINT64_MAX);
            std::atomic<bool> write_failed{false};
            {
                auto work = [&](int t) {
                    struct Publish { std::atomic<uint64_t>* a; ~Publish() { if (a->load() == UINT64_MAX) a->store(0); } } guard{&psize[t]};      // (a worker that leaves early must not block the others)
                    std::vector<OutRow> local;
                    const size_t a = n_iv * t / nt, b = n_iv * (t + 1) / nt;
                    for (size_t k = a; k < b; k++) {
                        const size_t r_end = k + 1 < n_iv ? std::max(rlo[k], rlo[k + 1]) : rlo[n_iv];
                        size_t r1 = rlo[k];
                        while (r1 < r_end && pos_of(r1) < ivs[i0 + k].end) r1++;
                        if (o.hemi) {       // rows are final: one per (position, base, pattern), in output order
                            for (size_t j = rlo[k]; j < r1; j++) format_hemi_row(co.hemi_rows[j], chrom, o.mixed, &parts[t]);
                            part_rows[t] += r1 - rlo[k];
                            continue;
                        }
                        local.clear();
                        finish_interval_rows(ivs[i0 + k], rows + rlo[k], r1 - rlo[k], have_motifs ? &mc.motifs : nullptr, combine_strands, &local);
                        if (!to_dir) for (auto& orow : local) format_bed_row(orow, chrom, fmt, &parts[t]);
                        else if (!o.bedgraph) { std::string& dst = routed[t][pfx + key_name + ".bed"]; for (auto& orow : local) format_bed_row(orow, chrom, fmt, &dst); }
                        else for (auto& orow : local) {
                            std::string label;
                            std::string& dst = routed[t][pfx + key_name + (key_name.empty() ? "" : "_") + bedgraph_label(orow, fmt) + "_" + strand_label(orow.strand) + ".bedgraph"];
                            format_bedgraph_row(orow, chrom, &dst);
                        }
                        part_rows[t] += local.size();
                    }
                    if (direct) {
                        // the text of worker t follows the text of the workers before it: wait for their sizes, then write in place
                        psize[t].store(parts[t].size(), std::memory_order_release);
                        uint64_t at = file_pos;
                        for (int q = 0; q < t; q++) { uint64_t v; while ((v = psize[q].load(std::memory_order_acquire)) == UINT64_MAX) std::this_thread::yield(); at += v; }
                        size_t done = 0;
                        while (done < parts[t].size()) {
                            const ssize_t w = pwrite(out_fd, parts[t].data() + done, parts[t].size() - done, (off_t)(at + done));
                            if (w <= 0) { write_failed = true; break; }
                            done += (size_t)w;
                        }
                    }
                };
                pool.run(nt, work);
            }
            if (write_failed) throw std::runtime_error("failed to write output file " + o.out_bed);
            for (int t = 0; t < nt; t++) {
                if (sharded) { if (!parts[t].empty()) shard_parts.push_back(std::move(parts[t])); }
                else if (direct) file_pos += parts[t].size();
                else if (out) fwrite(parts[t].data(), 1, parts[t].size(), out);
                for (auto& kv : routed[t]) if (!kv.second.empty()) fwrite(kv.second.data(), 1, kv.second.size(), router.get(kv.first));
                S.rows += part_rows[t];
            }
            { std::lock_guard<std::mutex> lk(q_mu); co.rows.clear(); if (spare_rows.size() < 4) spare_rows.push_back(std::move(co.rows)); }
            S.write_s += secs(tc, clk::now());
        }
        trace("last chunk formatted");
        if (dev_job.t.joinable()) dev_job.t.join();
        if (dev_err) std::rethrow_exception(dev_err);
        if (out) { if (out != stdout) fclose(out); else fflush(out); }
        if (sharded) {
            // rank-ordered concatenation (the reference's ordered collect, src/pileup/subcommand.rs:735-799): the slice sizes
            // are exchanged (second and last collective) and every rank writes its slice at its offset
            const auto tw = clk::now();
            std::vector<uint64_t> sizes((size_t)coll.world + 2, 0);
            uint64_t my_bytes = shard_text.size();
            for (auto& sp : shard_parts) my_bytes += sp.size();
            sizes[coll.rank] = my_bytes;
            sizes[coll.world] = S.rows; sizes[(size_t)coll.world + 1] = S.positions;
            coll.sum(sizes.data(), sizes.size());
            uint64_t at = 0;
            for (int r = 0; r < coll.rank; r++) at += sizes[r];
            const int fd = ::open(o.out_bed.c_str(), O_WRONLY);
            if (fd < 0) throw std::runtime_error("failed to open output file " + o.out_bed);
            // the pieces (header, then the formatted parts in order) go to their offsets from several threads
            std::vector<std::pair<const std::string*, uint64_t>> pieces;
            pieces.push_back({&shard_text, at});
            { uint64_t q = at + shard_text.size(); for (auto& sp : shard_parts) { pieces.push_back({&sp, q}); q += sp.size(); } }
            std::atomic<size_t> next_piece{0};
            std::atomic<bool> failed{false};
            auto put = [&]() {
                for (;;) {
                    const size_t k = next_piece.fetch_add(1);
                    if (k >= pieces.size() || failed) break;
                    const std::string& txt = *pieces[k].first;
                    size_t done = 0;
                    while (done < txt.size()) {
                        const ssize_t w = pwrite(fd, txt.data() + done, txt.size() - done, (off_t)(pieces[k].second + done));
                        if (w <= 0) { failed = true; break; }
                        done += (size_t)w;
                    }
                }
            };
            {
                std::vector<std::thread> th;
                const int nw = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, o.threads), pieces.size()));
                for (int t = 1; t < nw; t++) th.emplace_back(put);
                put();
                for (auto& t : th) t.join();
            }
            ::close(fd);
            if (failed) throw std::runtime_error("failed to write output file " + o.out_bed);
            S.rows_total = sizes[coll.world]; S.positions_total = sizes[(size_t)coll.world + 1];
            S.write_s += secs(tw, clk::now());
        } else { S.rows_total = S.rows; S.positions_total = S.positions; }
        const auto t1 = clk::now();
        trace("output written");
        S.load_s = secs(t0, t_load); S.threshold_s = secs(t_load, t_thr); S.interval_s = iv_secs;   /* runs beside ingest + thresholds; wait time = secs(t_thr, t_iv) */ S.total_s = secs(t0, t1);
        for (int b = 0; b < 4; b++) { S.thresholds[b] = P.base_threshold[b]; S.threshold_set[b] = P.base_threshold_set[b]; }
        if (summary) *summary = S;
        if (!o.quiet && (!sharded || coll.rank == 0))
            fprintf(stderr, "> Done, processed %llu rows. positions=%llu reads=%llu chunks=%llu load=%.3fs thresholds=%.3fs intervals=%.3fs pack=%.3fs gpu=%.3fs (kernels %.3f ms) write=%.3fs total=%.3fs\n",
                    (unsigned long long)S.rows, (unsigned long long)S.positions, (unsigned long long)S.reads_packed, (unsigned long long)S.chunks,
                    S.load_s, S.threshold_s, S.interval_s, S.pack_s, S.gpu_s, S.kernel_ms, S.write_s, S.total_s);
        if (!o.stats_json.empty()) {
            FILE* jf = fopen(o.stats_json.c_str(), "w");
            if (jf) {
                fprintf(jf, "{\"positions\": %llu, \"rows\": %llu, \"reads\": %llu, \"chunks\": %llu, \"algorithmic_bytes\": %llu, \"load_s\": %.6f, \"thresholds_s\": %.6f, \"intervals_s\": %.6f, \"pack_s\": %.6f, \"gpu_s\": %.6f, \"kernel_ms\": %.6f, \"write_s\": %.6f, \"total_s\": %.6f, \"ingest\": \"%s\", \"ingest_h2d_ms\": %.3f, \"ingest_inflate_ms\": %.3f, \"ingest_walk_ms\": %.3f, \"sampler_fetch_s\": %.6f, \"slice_s\": %.6f, \"pass_s\": %.6f, \"rowcopy_s\": %.6f}\n",
                        (unsigned long long)S.positions, (unsigned long long)S.rows, (unsigned long long)S.reads_packed, (unsigned long long)S.chunks, (unsigned long long)S.algorithmic_bytes,
                        S.load_s, S.threshold_s, S.interval_s, S.pack_s, S.gpu_s, S.kernel_ms, S.write_s, S.total_s,
                        bam.on_device ? (bam.ranged() ? "device-ranged" : "device") : "host", bam.ingest_ms[0], bam.ingest_ms[1], bam.ingest_ms[2], S.fetch_s, S.slice_s, S.pass_s, S.rowcopy_s);
                fclose(jf);
            }
        }
        if (trace_clock().on) {      // (development: where the release of the run's host objects goes)
            trace("stats written");
            std::vector<RefInterval>().swap(ivs); trace("intervals released");
            part_pool.clear(); part_pool.shrink_to_fit(); shard_parts.clear(); shard_parts.shrink_to_fit(); spare_rows.clear(); spare_rows.shrink_to_fit(); trace("text + row buffers released");
            bam.release_host_tables(); trace("record tables released");
        }
        return 0;
    } catch (const std::exception& e) {
        if (error) *error = e.what();
        return 1;
    }
}

// ---- several GPUs from one process: `--devices a,b,...` runs one interval shard per listed device on its own host thread
// (bound to the device's NUMA node); the two exchanges of a sharded run (histogram sum, slice sizes) are in-process sums.
struct InProcGroup {
    int world = 1;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<uint64_t> acc, result;
    int arrived = 0, gen = 0;
    bool aborted = false;
    void abort() { std::lock_guard<std::mutex> g(mu); aborted = true; cv.notify_all(); }
    int allreduce(uint64_t* buf, size_t n) {
        std::unique_lock<std::mutex> lk(mu);
        if (aborted) return -1;
        if (arrived == 0) acc.assign(n, 0);
        if (acc.size() != n) { aborted = true; cv.notify_all(); return -1; }
        for (size_t i = 0; i < n; i++) acc[i] += buf[i];
        const int my_gen = gen;
        if (++arrived == world) { result = acc; arrived = 0; gen++; cv.notify_all(); }
        else cv.wait(lk, [&] { return gen != my_gen || aborted; });
        if (gen == my_gen) return -1;       // aborted before the round completed
        memcpy(buf, result.data(), n * sizeof(uint64_t));
        return 0;
    }
    static int thunk(uint64_t* buf, size_t n, void* user) { return ((InProcGroup*)user)->allreduce(buf, n); }
};

inline int run_pileup_devices(const PileupOptions& o, RunSummary* summary, std::string* error) {
    const int world = (int)o.devices.size();
    if (world <= 1) { PileupOptions o1 = o; if (world == 1) o1.device = o.devices[0]; return run_pileup(o1, summary, error); }
    InProcGroup grp;
    grp.world = world;
    std::vector<RunSummary> sums(world);
    std::vector<std::string> errs(world);
    std::vector<int> rcs(world, 0);
    std::vector<std::thread> th;
    for (int r = 0; r < world; r++) th.emplace_back([&, r]() {
        mkp_bind_host_thread(o.devices[r]);            // NUMA-local pinned buffers and worker threads
        PileupOptions or_ = o;
        or_.device = o.devices[r];
        or_.schedule_threads = o.schedule_threads > 0 ? o.schedule_threads : o.threads;
        or_.threads = std::max(1, o.threads / world);
        if (r) or_.stats_json.clear();
        Collective c;
        c.rank = r; c.world = world; c.allreduce_sum = &InProcGroup::thunk; c.user = &grp;
        rcs[r] = run_pileup(or_, &sums[r], &errs[r], &c);
        if (rcs[r]) grp.abort();
    });
    for (auto& t : th) t.join();
    for (int r = 0; r < world; r++) if (rcs[r] && errs[r] != "collective (all-reduce) failed") { if (error) *error = errs[r]; return rcs[r]; }
    for (int r = 0; r < world; r++) if (rcs[r]) { if (error) *error = errs[r]; return rcs[r]; }
    if (summary) {
        *summary = sums[0];
        for (int r = 1; r < world; r++) { summary->reads_packed += sums[r].reads_packed; summary->chunks += sums[r].chunks; summary->algorithmic_bytes += sums[r].algorithmic_bytes; summary->kernel_ms = std::max(summary->kernel_ms, sums[r].kernel_ms); }
        summary->rows = sums[0].rows_total; summary->positions = sums[0].positions_total;
    }
    return 0;
}

// clap-compatible subset of the `modkit pileup` flag surface (src/pileup/subcommand.rs:37-379). hemi: `modkit pileup-hemi`
// (src/pileup/subcommand.rs:825-1130): the same flags without --preset, --combine-strands, --bedgraph, --with-header, --prefix
// and --partition-tag, one positional <IN_BAM>, output to -o/--out-bed or stdout.
inline bool parse_pileup_args(int argc, const char* const* argv, PileupOptions* o, std::string* err, bool hemi = false) {
    std::vector<std::string> pos;
    o->hemi = hemi;
    for (int i = 0; i < argc; i++) {
        const std::string a = argv[i];
        auto val = [&]() -> std::string { if (i + 1 >= argc) throw std::runtime_error("a value is required for '" + a + "' but none was supplied"); return argv[++i]; };
        try {
            if (hemi && (a == "--preset" || a == "--combine-strands" || a == "--bedgraph" || a == "--header" || a == "--with-header" ||
                         a == "--include_header" || a == "--prefix" || a == "--partition-tag")) { *err = "unexpected argument '" + a + "' found"; return false; }
            if (hemi && (a == "-o" || a == "--out-bed")) o->out_bed = val();
            else if (a == "-t" || a == "--threads") o->threads = std::stoi(val());
            else if (a == "-i" || a == "--interval-size") o->interval_size = (uint32_t)std::stoul(val());
            else if (a == "--region") o->region = val();
            else if (a == "--sample-region") o->sample_region = val();
            else if (a == "--sampling-interval-size") o->sampling_interval_size = (uint32_t)std::stoul(val());
            else if (a == "-n" || a == "--num-reads") o->num_reads = std::stoul(val());
            else if (a == "-f" || a == "--sampling-frac") { o->have_frac = true; o->frac = std::stod(val()); }
            else if (a == "--max-depth") o->max_depth = (uint32_t)std::stoul(val());
            else if (a == "--devices") { o->devices.clear(); std::string v = val(); for (size_t i = 0; i < v.size();) { size_t j = v.find(',', i); if (j == std::string::npos) j = v.size(); o->devices.push_back(std::stoi(v.substr(i, j - i))); i = j + 1; } if (o->devices.empty()) throw std::runtime_error("--devices needs a list of device indices"); }
            else if (a == "--seed" || a == "--queue-size" || a == "--chunk-size" || a == "--log-filepath" || a == "--log") val();
            else if (a == "--no-filtering") o->no_filtering = true;
            else if (a == "-p" || a == "--filter-percentile") o->percentile = std::stof(val());
            else if (a == "--filter-threshold" || a == "--pass_threshold") o->filter_thresholds.push_back(val());
            else if (a == "--mod-thresholds" || a == "--mod-threshold") o->mod_thresholds.push_back(val());
            else if (a == "--include-unmapped") o->include_unmapped = true;
            else if (a == "--ignore") o->ignore = val();
            else if (a == "--force-allow-implicit") o->force_allow = true;
            else if (a == "--motif") { o->motif_parts.push_back(val()); o->motif_parts.push_back(val()); }
            else if (a == "--cpg") o->cpg = true;
            else if (a == "-r" || a == "--ref" || a == "--reference") o->ref_fp = val();
            else if (a == "-k" || a == "--mask") o->mask = true;
            else if (a == "--preset") { if (val() != "traditional") throw std::runtime_error("invalid value for '--preset'"); o->traditional = true; }
            else if (a == "--combine-mods") o->combine_mods = true;
            else if (a == "--combine-strands") o->combine_strands = true;
            else if (a == "--edge-filter") o->edge = val();
            else if (a == "--invert-edge-filter") o->invert_edge = true;
            else if (a == "--only-tabs" || a == "--suppress-progress") {}
            else if (a == "--mixed-delim" || a == "--mixed-delimiters") o->mixed = true;
            else if (a == "--header" || a == "--with-header" || a == "--include_header") o->header = true;
            else if (a == "--device") o->device = std::stoi(val());
            else if (a == "--gpu-chunk-bp") o->chunk_bp = (uint32_t)std::stoul(val());
            else if (a == "--host-ingest") o->host_ingest = true;
            else if (a == "--stats-json") o->stats_json = val();
            else if (a == "--quiet") o->quiet = true;
            else if (a == "--include-bed" || a == "--include-positions") o->include_bed = val();
            else if (a == "--partition-tag") o->partition_tags.push_back(val());
            else if (a == "--bedgraph") o->bedgraph = true;
            else if (a == "--prefix") o->prefix = val();
            else if (a.size() > 1 && a[0] == '-') { *err = "unexpected argument '" + a + "' found"; return false; }
            else pos.push_back(a);
        } catch (const std::exception& e) { *err = e.what(); return false; }
    }
    if (hemi) {
        if (pos.size() != 1) { *err = pos.empty() ? "the following required arguments were not provided: <IN_BAM>" : "unexpected argument '" + pos[1] + "' found"; return false; }
        o->in_bam = pos[0];
        if (o->out_bed.empty()) o->out_bed = "-";
        return true;
    }
    if (pos.size() != 2) { *err = "the following required arguments were not provided: <IN_BAM> <OUT_BED>"; return false; }
    o->in_bam = pos[0]; o->out_bed = pos[1];
    return true;
}


// ================================================================================================================
// `modkit summary` and `modkit sample-probs` (SURVEY 8f-3; src/commands.rs:549-1190, src/summarize.rs:117-252,
// src/writers.rs:394-684, 692-790): the reads come from the same sampling schedule as the pileup's threshold estimation, the
// decode runs on the GPU (mkp_sample_histogram / mkp_sample_summary). The reference prints its maps in hash order; here rows
// are ordered: canonical bases A C G T, then canonical before modified states, codes in ModCodeRepr order.
// ================================================================================================================
struct SampleOptions {
    std::string in_bam, region, include_bed, ignore, edge, percentiles = "0.1,0.5,0.9";
    std::vector<std::string> filter_thresholds, mod_thresholds;
    int threads = 4, device = 0;
    uint32_t interval_size = 1000000;
    size_t num_reads = 10042;
    bool have_frac = false, no_sampling = false, no_filtering = false, only_mapped = false, invert_edge = false, tsv = false;
    double frac = 0;
    float percentile = 0.1f;
};

struct ModSummaryOut {
    uint64_t reads_with[4] = {0, 0, 0, 0};
    std::map<uint64_t, uint64_t> pass[4], fail[4];     // key: 0 = canonical, else 1 + (code ordering key)
    std::set<uint64_t> observed[4];
    uint64_t total_reads = 0;
    float thresholds[4] = {0, 0, 0, 0};
    bool threshold_set[4] = {false, false, false, false};
};

inline uint64_t state_order_key(uint32_t code) { return 1ull + ((code & 0x80000000u) ? (1ull << 32) + (code & 0x7fffffffu) : (uint64_t)code); }
inline std::string state_label_of_key(uint64_t k) { return k > (1ull << 32) ? std::to_string(k - 1 - (1ull << 32)) : std::string(1, (char)(k - 1)); }
inline std::string f64_display(double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
    char buf[400];
    auto r = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::fixed);
    return std::string(buf, r.ptr);
}

// sampling + thresholds shared by both commands; fills the kept chunks when `keep` is given. `inexact` receives the count of
// sampled values off the histogram's 1/1024 grid: only a quantile of the histogram needs them on it
inline void sample_for_summary(const SampleOptions& o, mkp_ctx* ctx, BamReader& bam, mkp_params* P, Region* region_out, bool* have_region, IncludeBed* include, bool* have_include,
                               std::vector<uint64_t>* hist, std::vector<SampledChunk>* keep, size_t* n_selected, uint64_t* inexact_out) {
    try { bam.open_device_index(o.in_bam, ctx); }
    catch (...) { throw; }
    if (!bam.have_index()) { bam = BamReader(); bam.open(o.in_bam, o.threads); }       // no index: the (small) file is read on the host
    *have_region = false;
    if (!o.region.empty()) { *region_out = parse_region_arg(o.region, bam); *have_region = true; }
    *have_include = false;
    if (!o.include_bed.empty()) {
        std::map<std::string, uint32_t> name_to_tid;
        for (uint32_t t = 0; t < bam.ref_names.size(); t++) if (!*have_region || bam.ref_names[t] == region_out->name) name_to_tid[bam.ref_names[t]] = t;
        include->read(o.include_bed, name_to_tid);
        *have_include = true;
    }
    memset(P, 0, sizeof *P);
    if (!o.ignore.empty()) { uint32_t c; if (!parse_code(o.ignore, &c)) throw std::runtime_error("failed to parse mod code " + o.ignore); P->numeric_mode = 2; P->collapse_code = c; }
    if (!o.edge.empty()) {
        P->edge_filter_on = 1; P->edge_filter_inverted = o.invert_edge;
        auto c = o.edge.find(',');
        if (c == std::string::npos) P->edge_filter_start = P->edge_filter_end = (uint32_t)std::stoul(o.edge);
        else { P->edge_filter_start = (uint32_t)std::stoul(o.edge.substr(0, c)); P->edge_filter_end = (uint32_t)std::stoul(o.edge.substr(c + 1)); }
    }
    P->force_allow_implicit = 1;     // the sampler takes implicit lists as they are (no InvalidImplicitMode check outside the pileup)
    if (mkp_set_params(ctx, P)) throw std::runtime_error(mkp_last_error(ctx));
    SamplerConfig sc;
    sc.threads = o.threads; sc.workers = o.threads; sc.sampling_interval_size = o.interval_size;
    if (o.no_sampling) sc.take_all = true;
    else if (o.have_frac) { if (o.frac != 1.0) throw std::runtime_error("only --sampling-frac 1.0 is reproducible without the reference's RNG; use -n, -f 1.0 or --no-sampling"); sc.take_all = true; }
    sc.num_reads = o.num_reads;
    sc.region = *have_region ? region_out : nullptr;
    sc.include_unmapped = !(o.only_mapped || *have_include);
    sc.edge_on = P->edge_filter_on;
    sc.include = *have_include ? include : nullptr;
    hist->assign(4 * MKP_HIST_BINS, 0);
    uint64_t inexact = 0;
    Collective solo;
    if (bam.on_device && bam.have_index()) *n_selected = sample_histogram_indexed(bam, ctx, sc, hist->data(), &inexact, solo, nullptr, keep);
    else *n_selected = sample_histogram(bam, ctx, sc, hist->data(), &inexact, keep);
    *inexact_out = inexact;
}

inline void require_exact(uint64_t inexact) {
    if (inexact) throw std::runtime_error("sampled probabilities are not multiples of 1/1024 (" + std::to_string(inexact) + " values): exact quantiles impossible");
}

inline int run_summary(const SampleOptions& o, std::string* text, std::string* error) {
    try {
        DeviceGuard dev;
        { const int rc = mkp_create(o.device, &dev.ctx); if (rc) throw std::runtime_error("no usable CUDA device (mkp_create returned " + std::to_string(rc) + "); this build has no CPU fallback"); }
        if (o.percentile > 1.0f) throw std::runtime_error("filter percentile must be <= 1.0");
        BamReader bam;
        mkp_params P;
        Region region; bool have_region = false;
        IncludeBed include; bool have_include = false;
        std::vector<uint64_t> hist;
        std::vector<SampledChunk> keep;
        size_t n_selected = 0;
        uint64_t inexact = 0;
        sample_for_summary(o, dev.ctx, bam, &P, &region, &have_region, &include, &have_include, &hist, &keep, &n_selected, &inexact);
        ModSummaryOut S;
        // thresholds (src/commands.rs:1086-1098, 1147-1160)
        for (auto& raw : o.mod_thresholds) {
            auto c = raw.find(':');
            uint32_t code;
            if (c == std::string::npos || raw.find(':', c + 1) != std::string::npos || !parse_code(raw.substr(0, c), &code))
                throw std::runtime_error("encountered illegal per-mod threshold: " + raw + ". Should be mod_code:threshold e.g. h:0.8");
            if (P.n_mod_thresholds >= MKP_MAX_MOD_THRESHOLDS) throw std::runtime_error("too many per-mod thresholds");
            P.mod_code[P.n_mod_thresholds] = code;
            P.mod_threshold[P.n_mod_thresholds++] = std::stof(raw.substr(c + 1));
        }
        if (!o.filter_thresholds.empty()) {
            bool have_default = false;
            for (auto& raw : o.filter_thresholds) {
                auto c = raw.find(':');
                if (c == std::string::npos) { if (have_default) throw std::runtime_error("default threshold encountered more than once"); P.default_threshold = std::stof(raw); have_default = true; }
                else {
                    const char* B = "ACGT";
                    const char* f = raw.empty() ? nullptr : strchr(B, raw[0]);
                    if (!f || !raw[0]) throw std::runtime_error("failed to parse base " + raw);
                    P.base_threshold_set[f - B] = 1;
                    P.base_threshold[f - B] = std::stof(raw.substr(c + 1));
                }
            }
        } else if (!o.no_filtering) {
            require_exact(inexact);
            for (int b = 0; b < 4; b++) {
                uint64_t n = 0;
                for (int k = 0; k < MKP_HIST_BINS; k++) n += hist[b * MKP_HIST_BINS + k];
                if (!n) continue;
                float thr;
                if (!percentile_from_hist(hist.data() + b * MKP_HIST_BINS, o.percentile, &thr)) throw std::runtime_error("not enough datapoints to estimate a threshold");
                P.base_threshold_set[b] = 1; P.base_threshold[b] = thr;
            }
        }
        for (int b = 0; b < 4; b++) { S.thresholds[b] = P.base_threshold[b]; S.threshold_set[b] = P.base_threshold_set[b]; }
        if (mkp_set_params(dev.ctx, &P)) throw std::runtime_error(mkp_last_error(dev.ctx));
        // ---- second pass over the sampled reads: counts per (base, state, pass / fail)
        std::vector<uint32_t> fpos, fneg;
        const int incl_unal = !(o.only_mapped || have_include) ? 1 : 0;
        for (auto& kc : keep) {
            if (kc.pc.recs.empty()) continue;
            upload_sample_chunk(dev.ctx, kc.pc, kc.tid, have_include ? &include : nullptr, &fpos, &fneg);
            std::vector<uint64_t> table(4 * 2 * 33, 0), states(32, ~0ull);
            uint64_t rw[4] = {0, 0, 0, 0};
            uint32_t obs[4] = {0, 0, 0, 0};
            if (mkp_sample_summary(dev.ctx, incl_unal, kc.take.data(), table.data(), rw, obs, states.data())) throw std::runtime_error(mkp_last_error(dev.ctx));
            for (int b = 0; b < 4; b++) {
                S.reads_with[b] += rw[b];
                for (int f = 0; f < 2; f++) for (int k = 0; k < 33; k++) {
                    const uint64_t n = table[(b * 2 + f) * 33 + k];
                    if (!n) continue;
                    const uint64_t key = k == 0 ? 0 : state_order_key((uint32_t)states[k - 1]);
                    (f == 0 ? S.pass[b] : S.fail[b])[key] += n;
                }
                for (int id = 0; id < 32; id++) if ((obs[b] >> id) & 1u) S.observed[b].insert(state_order_key((uint32_t)states[id]));
            }
            for (uint8_t t : kc.take) S.total_reads += t;
        }
        // ---- text
        std::string& out = *text;
        out.clear();
        std::string bases;
        for (int b = 0; b < 4; b++) if (!S.pass[b].empty() || S.reads_with[b]) { if (!bases.empty()) bases += ","; bases += "ACGT"[b]; }
        if (o.tsv) {
            // TsvWriter<ModSummary> (src/writers.rs:609-684), keys in a fixed order
            out += "mod_bases\t" + bases + "\n";
            for (int b = 0; b < 4; b++) if (S.reads_with[b]) out += std::string("count_reads_") + "ACGT"[b] + "\t" + std::to_string(S.reads_with[b]) + "\n";
            for (int b = 0; b < 4; b++) {
                if (S.pass[b].empty() && !S.reads_with[b]) continue;
                uint64_t total = 0, total_f = 0;
                for (auto& kv : S.pass[b]) total += kv.second;
                for (auto& kv : S.fail[b]) total_f += kv.second;
                const std::string B(1, "ACGT"[b]);
                for (auto& kv : S.pass[b]) {
                    const std::string label = kv.first == 0 ? std::string("unmodified") : "modified_" + state_label_of_key(kv.first);
                    auto fi = S.fail[b].find(kv.first);
                    out += B + "_pass_calls_" + label + "\t" + std::to_string(kv.second) + "\n";
                    out += B + "_pass_frac_" + label + "\t" + f64_display((double)kv.second / (double)total) + "\n";
                    out += B + "_fail_calls_" + label + "\t" + std::to_string(fi == S.fail[b].end() ? 0 : fi->second) + "\n";
                }
                out += B + "_total_mod_calls\t" + std::to_string(total) + "\n";
                out += B + "_total_fail_mod_calls\t" + std::to_string(total_f) + "\n";
            }
            out += "total_reads_used\t" + std::to_string(S.total_reads) + "\n";
        } else {
            // TableWriter<ModSummary> (src/writers.rs:394-560): '#'-prefixed metadata, then base / code / pass_count / pass_frac / all_count / all_frac
            out += "# bases             " + bases + "\n";
            out += "# total_reads_used  " + std::to_string(S.total_reads) + "\n";
            for (int b = 0; b < 4; b++) if (S.reads_with[b]) out += std::string("# count_reads_") + "ACGT"[b] + "     " + std::to_string(S.reads_with[b]) + "\n";
            for (int b = 0; b < 4; b++) if (S.threshold_set[b]) out += std::string("# pass_threshold_") + "ACGT"[b] + "  " + f32_display(S.thresholds[b]) + "\n";
            if (have_region) out += "# region            " + region.name + ":" + std::to_string(region.start) + "-" + std::to_string(region.end) + "\n";
            std::vector<std::vector<std::string>> rows;
            rows.push_back({"base", "code", "pass_count", "pass_frac", "all_count", "all_frac"});
            for (int b = 0; b < 4; b++) {
                uint64_t total_p = 0, total_f = 0;
                for (auto& kv : S.pass[b]) total_p += kv.second;
                for (auto& kv : S.fail[b]) total_f += kv.second;
                const uint64_t total = total_p + total_f;
                std::set<uint64_t> keys;
                for (auto& kv : S.pass[b]) keys.insert(kv.first);
                for (uint64_t k : S.observed[b]) keys.insert(k);
                if (!S.pass[b].empty() || !S.fail[b].empty()) keys.insert(0);           // the canonical row is always shown
                for (uint64_t k : keys) {
                    auto pi = S.pass[b].find(k); auto fi = S.fail[b].find(k);
                    const uint64_t pc = pi == S.pass[b].end() ? 0 : pi->second, fc = fi == S.fail[b].end() ? 0 : fi->second;
                    rows.push_back({std::string(1, "ACGT"[b]), k == 0 ? std::string("-") : state_label_of_key(k), std::to_string(pc),
                                    f32_display((float)pc / (float)total_p), std::to_string(pc + fc), f32_display((float)(pc + fc) / (float)total)});
                }
            }
            std::vector<size_t> w(6, 0);
            for (auto& r : rows) for (size_t i = 0; i < 6; i++) w[i] = std::max(w[i], r[i].size());
            for (auto& r : rows) { for (size_t i = 0; i < 6; i++) { out += " " + r[i] + std::string(w[i] - r[i].size(), ' ') + " "; } out += "\n"; }
        }
        return 0;
    } catch (const std::exception& e) { if (error) *error = e.what(); return 1; }
}

// `modkit sample-probs`: percentiles of the arg-max probabilities per canonical base (thresholds table, src/writers.rs:779-790)
inline int run_sample_probs(const SampleOptions& o, std::string* text, std::string* error) {
    try {
        DeviceGuard dev;
        { const int rc = mkp_create(o.device, &dev.ctx); if (rc) throw std::runtime_error("no usable CUDA device (mkp_create returned " + std::to_string(rc) + "); this build has no CPU fallback"); }
        std::vector<float> qs;
        for (size_t i = 0; i < o.percentiles.size();) {
            size_t j = o.percentiles.find(',', i); if (j == std::string::npos) j = o.percentiles.size();
            const float q = std::stof(o.percentiles.substr(i, j - i));
            if (q > 1.0f || q < 0.0f) throw std::runtime_error("percentiles must be between 0 and 1.0");
            qs.push_back(q);
            i = j + 1;
        }
        BamReader bam;
        mkp_params P;
        Region region; bool have_region = false;
        IncludeBed include; bool have_include = false;
        std::vector<uint64_t> hist;
        size_t n_selected = 0;
        uint64_t inexact = 0;
        sample_for_summary(o, dev.ctx, bam, &P, &region, &have_region, &include, &have_include, &hist, nullptr, &n_selected, &inexact);
        require_exact(inexact);
        std::vector<std::vector<std::string>> rows;
        rows.push_back({"base", "percentile", "threshold"});
        for (int b = 0; b < 4; b++) {
            uint64_t n = 0;
            for (int k = 0; k < MKP_HIST_BINS; k++) n += hist[b * MKP_HIST_BINS + k];
            if (!n) continue;
            for (float q : qs) {
                float v;
                if (!percentile_from_hist(hist.data() + b * MKP_HIST_BINS, q, &v)) throw std::runtime_error("not enough datapoints to calculate percentiles");
                volatile float pct = q * 100.0f;
                rows.push_back({std::string(1, "ACGT"[b]), f32_display(pct), f32_display(v)});
            }
        }
        std::vector<size_t> w(3, 0);
        for (auto& r : rows) for (size_t i = 0; i < 3; i++) w[i] = std::max(w[i], r[i].size());
        text->clear();
        for (auto& r : rows) { for (size_t i = 0; i < 3; i++) { *text += " " + r[i] + std::string(w[i] - r[i].size(), ' ') + " "; } *text += "\n"; }
        return 0;
    } catch (const std::exception& e) { if (error) *error = e.what(); return 1; }
}

inline bool parse_sample_args(int argc, const char* const* argv, bool summary, SampleOptions* o, std::string* out_path, std::string* err) {
    std::vector<std::string> pos;
    for (int i = 0; i < argc; i++) {
        const std::string a = argv[i];
        auto val = [&]() -> std::string { if (i + 1 >= argc) throw std::runtime_error("a value is required for '" + a + "' but none was supplied"); return argv[++i]; };
        try {
            if (a == "-t" || a == "--threads") o->threads = std::stoi(val());
            else if (a == "--region") o->region = val();
            else if (a == "-n" || a == "--num-reads") o->num_reads = std::stoul(val());
            else if (a == "-f" || a == "--sampling-frac") { o->have_frac = true; o->frac = std::stod(val()); }
            else if (a == "--no-sampling") o->no_sampling = true;
            else if (a == "-i" || a == "--interval-size") o->interval_size = (uint32_t)std::stoul(val());
            else if (a == "--include-bed" || a == "--include-positions") o->include_bed = val();
            else if (a == "--only-mapped") o->only_mapped = true;
            else if (a == "--ignore") o->ignore = val();
            else if (a == "--edge-filter") o->edge = val();
            else if (a == "--invert-edge-filter") o->invert_edge = true;
            else if (a == "--seed" || a == "--log-filepath" || a == "--log") val();
            else if (a == "--suppress-progress") {}
            else if (a == "--device") o->device = std::stoi(val());
            else if (a == "--out") *out_path = val();                 // (this build: write the report to a file instead of stdout)
            else if (summary && (a == "--filter-threshold" || a == "--pass_threshold")) o->filter_thresholds.push_back(val());
            else if (summary && (a == "--mod-thresholds" || a == "--mod-threshold")) o->mod_thresholds.push_back(val());
            else if (summary && a == "--no-filtering") o->no_filtering = true;
            else if (summary && (a == "-p" || a == "--filter-percentile")) o->percentile = std::stof(val());
            else if (summary && a == "--tsv") o->tsv = true;
            else if (summary && a == "--table") o->tsv = false;
            else if (!summary && (a == "-p" || a == "--percentiles")) o->percentiles = val();
            else if (!summary && (a == "--hist" || a == "-o" || a == "--out-dir" || a == "--prefix" || a == "--force" || a == "--dna-color" || a == "--mod-color"))
                throw std::runtime_error("histogram / file outputs of sample-probs (" + a + ") are not provided by this build: the percentile table goes to stdout");
            else if (a.size() > 1 && a[0] == '-') { *err = "unexpected argument '" + a + "' found"; return false; }
            else pos.push_back(a);
        } catch (const std::exception& e) { *err = e.what(); return false; }
    }
    if (pos.size() != 1) { *err = "the following required arguments were not provided: <IN_BAM>"; return false; }
    o->in_bam = pos[0];
    return true;
}

}  // namespace mkh
