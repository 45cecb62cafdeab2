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
#include <numeric>
#include <filesystem>
#include <optional>
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

// pileup-hemi's motif (src/pileup/subcommand.rs:1242-1272): exactly one, --cpg or --motif, and it must be a palindrome
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
    std::shared_ptr<void>* defer_free = nullptr;         // the candidate buffers (hundreds of MB with an index) are handed over instead of
                                                         // being released before the result is returned; the caller drops them when convenient
    std::shared_future<void>* device_ready = nullptr;    // the candidates are fetched first (host only); the decode passes wait for this
                                                         // (the device is busy loading the BAM until then)
    uint32_t sampling_interval_size = 1000000;
    bool take_all = false;
    size_t num_reads = 10042;
    const Region* region = nullptr;
    bool include_unmapped = false;
    bool edge_on = false;
    const IncludeBed* include = nullptr;
    bool keep = false;                 // also return the sampled reads (summary's second pass); needs host-packed reads, so not the device-resident source
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

struct SampleResult {
    std::vector<uint64_t> hist = std::vector<uint64_t>(4 * MKP_HIST_BINS, 0);    // [4][MKP_HIST_BINS], summed over the ranks
    uint64_t inexact = 0;              // sampled values off the 1/1024 grid
    size_t n_selected = 0;             // reads selected, all ranks
    double fetch_s = 0;                // host fetch + pack of the planned candidates
    std::vector<SampledChunk> keep;    // SamplerConfig::keep: the selected reads, flagged in `take` of their chunks
};

// Candidate reads of one sampling group (tid < 0: the reads without coordinates) in file order, from one of three sources:
// the index fetch (the reader has a BAI, BamReader::fetch_*: the record bytes come from the file), the records the reader holds
// on the host, or the records it holds on the device (only listed; sliced on the GPU when the chunk is uploaded). A resident
// reader is never loaded range by range (that needs the index), so its records need no ensure_tid.
struct Candidates {
    const BamReader& bam;
    const bool req_mapped;
    BamReader::FetchCursor fc;         // index source
    std::vector<RecRef> recs, got;     // resident sources: the group's candidates, `next` the first not handed out
    size_t next = 0;
    bool done = false;
    Candidates(const BamReader& b, int64_t tid, uint32_t start, uint32_t end, bool req_mapped_) : bam(b), req_mapped(req_mapped_) {
        if (bam.have_index()) { fc = tid < 0 ? bam.fetch_unplaced_begin() : bam.fetch_begin((uint32_t)tid, start, end); done = fc.done; return; }
        auto add = [&](const RecRef& r) { if (sampler_flag_ok(r, req_mapped)) recs.push_back(r); };
        if (tid < 0) for (auto& r : bam.unplaced) add(r);
        else bam.for_overlapping((uint32_t)tid, start, end, add);
        done = recs.empty();
    }
    // appends up to n more candidates to `out` (packed unless the records are on the device)
    void more(size_t n, PackedChunk* out) {
        if (bam.have_index()) {
            got.clear();
            bam.fetch_more(fc, n, [&](const RecRef& r) { return sampler_flag_ok(r, req_mapped); }, &got);
            for (auto& r : got) { pack_record(fc.bytes(r), r.size, out); out->recs.push_back(r); }     // (bytes valid until the next fetch_more)
            done = fc.done;
            return;
        }
        for (const size_t stop = next + std::min(n, recs.size() - next); next < stop; next++) {
            if (!bam.on_device) pack_record(bam.rec(recs[next]), recs[next].size, out);
            out->recs.push_back(recs[next]);
        }
        done = next == recs.size();
    }
};

// Makes a chunk of sampled reads the resident chunk: packed reads are uploaded, device-resident ones sliced on the GPU. The chunk
// has no coordinates of its own, except with --include-bed: then it spans its reads and carries the bitmaps of contig `tid`.
inline void upload_sampled(const BamReader& bam, mkp_ctx* ctx, const PackedChunk& pc, uint32_t tid, const IncludeBed* include) {
    mkp_chunk ch;
    memset(&ch, 0, sizeof ch);
    ch.start = 0; ch.end = 32;
    std::vector<uint32_t> fpos, fneg;
    if (include) {
        int64_t lo = INT64_MAX, hi = 0;
        for (auto& r : pc.recs) { lo = std::min<int64_t>(lo, r.pos); hi = std::max<int64_t>(hi, r.end); }
        if (lo < 0) lo = 0;
        if (hi <= lo) hi = lo + 1;
        ch.start = (uint32_t)lo; ch.end = (uint32_t)hi;
        include->bitmaps(tid, ch.start, ch.end, &fpos, &fneg);
        ch.focus_pos = fpos.data(); ch.focus_neg = fneg.data();
    }
    if (bam.on_device && !bam.have_index()) { device_chunk(bam, pc.recs, ch.start, ch.end, ch.focus_pos, ch.focus_neg); return; }
    ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
    if (mkp_upload_chunk(ctx, &ch)) throw std::runtime_error(mkp_last_error(ctx));
}

// The schedule's unit of selection: the first `limit` contributing reads of recs[lo, hi) count towards the group (`used`); those
// not selected by an earlier group of the contig are flagged in `take`.
inline void select_first(const std::vector<RecRef>& recs, const std::vector<uint8_t>& contributes, size_t lo, size_t hi, size_t limit, size_t* used,
                         std::unordered_set<uint64_t>* selected, std::vector<uint8_t>* take) {
    for (size_t k = lo; k < hi && *used < limit; k++) {
        if (!contributes[k]) continue;
        ++*used;
        if (selected->insert(recs[k].off).second) (*take)[k] = 1;
    }
}

struct Collective {          // sum over the ranks of a sharded run (in place); world == 1: nothing to do
    int rank = 0, world = 1;
    int (*allreduce_sum)(uint64_t* buf, size_t n, void* user) = nullptr;
    void* user = nullptr;
    void sum(uint64_t* buf, size_t n) const {
        if (world <= 1) return;
        if (!allreduce_sum || allreduce_sum(buf, n, user) != 0) throw std::runtime_error("collective (all-reduce) failed");
    }
};

// The files of a sharded run that writes a directory (--partition-tag). Every rank holds, per file name, the text of its own
// intervals; a file is the rank-ordered concatenation of those texts. agree_file_slices gives every rank the union of the names
// (sorted), the total size of each file and this rank's offset in it. Every rank calls it, with whatever map it has (an empty one
// too). It makes up to three sums, each of the same length on every rank (NCCL requires that): the name-list sizes (world words),
// the name lists (each rank fills its own window of a zeroed buffer), and the size matrix (files x world). The last two are left
// out on every rank when no rank has a name.
struct FileSlices { std::vector<std::string> names; std::vector<uint64_t> offset, total; };
inline FileSlices agree_file_slices(const Collective& coll, const std::map<std::string, uint64_t>& mine) {
    const size_t world = (size_t)std::max(1, coll.world), rank = (size_t)coll.rank;
    // a name list in u64 words: per name its length, then its bytes (zero-padded to whole words)
    std::vector<uint64_t> list;
    for (auto& kv : mine) {
        const std::string& nm = kv.first;
        list.push_back(nm.size());
        const size_t at = list.size();
        list.resize(at + (nm.size() + 7) / 8, 0);
        memcpy(list.data() + at, nm.data(), nm.size());
    }
    std::vector<uint64_t> words(world, 0);
    words[rank] = list.size();
    coll.sum(words.data(), words.size());
    std::vector<uint64_t> all(std::accumulate(words.begin(), words.end(), (uint64_t)0), 0);
    std::copy(list.begin(), list.end(), all.begin() + (ptrdiff_t)std::accumulate(words.begin(), words.begin() + (ptrdiff_t)rank, (uint64_t)0));
    if (!all.empty()) coll.sum(all.data(), all.size());           // (every rank knows the size: none sums an empty buffer)
    std::set<std::string> uni;
    for (size_t p = 0; p < all.size();) {
        const size_t len = (size_t)all[p++];
        if (len > (all.size() - p) * 8) throw std::runtime_error("malformed file-name exchange");
        uni.insert(std::string((const char*)(all.data() + p), len));
        p += (len + 7) / 8;
    }
    FileSlices fs;
    fs.names.assign(uni.begin(), uni.end());
    std::vector<uint64_t> sizes(fs.names.size() * world, 0);           // [file][rank]
    for (size_t f = 0; f < fs.names.size(); f++) { auto it = mine.find(fs.names[f]); if (it != mine.end()) sizes[f * world + rank] = it->second; }
    if (!sizes.empty()) coll.sum(sizes.data(), sizes.size());
    for (size_t f = 0; f < fs.names.size(); f++) {
        const uint64_t* row = sizes.data() + f * world;
        fs.offset.push_back(std::accumulate(row, row + rank, (uint64_t)0));
        fs.total.push_back(std::accumulate(row, row + world, (uint64_t)0));
    }
    return fs;
}

inline void append_packed(const PackedChunk& src, PackedChunk* dst) {
    const uint64_t base = (dst->heap.size() + 15) & ~(uint64_t)15;
    dst->heap.resize(base);
    dst->heap.insert(dst->heap.end(), src.heap.begin(), src.heap.end());
    for (auto h : src.hdrs) { h.off += base; dst->hdrs.push_back(h); }
    dst->recs.insert(dst->recs.end(), src.recs.begin(), src.recs.end());
}

// The sampling schedule of the reference (reads_sampler/sampling_schedule.rs:171-615) and the histogram of the reads it selects:
// the first n contributing records of every group, in file order. The schedule's state is per contig (`done`, the reads
// selected so far), and the records of different contigs are disjoint, so walking contig by contig gives the same groups and
// the same reads as the reference's walk over super-batches of all contigs (oracle/driver.hpp:427-500): a slack group never
// spans two contigs. The contigs are therefore independent: in an interval-sharded run every rank samples the contigs it owns
// and the histograms are summed once (SURVEY 8e). Per contig the schedule is first simulated under the assumption that every
// group finds its quota (true whenever the coverage is not tiny); the candidates of all planned groups are fetched in parallel,
// decoded in ONE device pass, and the real schedule then consumes them in order. A group that deviates from the plan, or needs
// more candidates than were fetched, fetches and decodes on demand - the reads are the same either way.
inline SampleResult sample_histogram(const BamReader& bam, mkp_ctx* ctx, const SamplerConfig& cfg, const Collective& coll = Collective()) {
    using clk = std::chrono::steady_clock;
    if (coll.world > 1 && !bam.have_index()) throw std::runtime_error("interval-sharded runs need a BAM index (.bai)");
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
    // groups of contig t in super-batch s given the reads sampled from the contig so far; groups of fewer than 50 reads merge
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
    SampleResult res;
    std::vector<uint64_t> batch_hist(4 * MKP_HIST_BINS);
    const bool req_mapped = !cfg.include_unmapped || cfg.edge_on;

    // one device pass decides which reads of a chunk contribute (MODE_HIST without a histogram); a second pass over the same
    // resident chunk adds the values of the selected reads to the histogram
    auto decode = [&](const PackedChunk& pc, uint32_t tid, std::vector<uint8_t>* contributes) {
        contributes->assign(pc.recs.size(), 0);
        if (pc.recs.empty()) return;
        upload_sampled(bam, ctx, pc, tid, cfg.include);
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, nullptr, nullptr, contributes->data(), nullptr)) throw std::runtime_error(mkp_last_error(ctx));
    };
    auto any = [](const std::vector<uint8_t>& take) { for (uint8_t t : take) if (t) return true; return false; };
    auto add_taken = [&](const std::vector<uint8_t>& take) {     // histogram of the flagged reads of the resident chunk
        if (!any(take)) return;
        uint64_t inx = 0;
        if (mkp_sample_histogram_wide(ctx, cfg.include_unmapped ? 1 : 0, take.data(), batch_hist.data(), nullptr, &inx)) throw std::runtime_error(mkp_last_error(ctx));
        for (int k = 0; k < 4 * MKP_HIST_BINS; k++) res.hist[k] += batch_hist[k];
        res.inexact += inx;
    };
    auto keep = [&](PackedChunk&& pc, std::vector<uint8_t>&& take, uint32_t tid) { if (cfg.keep && any(take)) res.keep.push_back({std::move(pc), std::move(take), tid}); };
    auto key_of = [](const Grp& g) { return std::to_string(g.tid) + ":" + std::to_string(g.start) + "-" + std::to_string(g.end) + "/" + std::to_string(g.n); };

    struct Planned { Grp g; std::optional<Candidates> cur; PackedChunk pc; size_t lo = 0, hi = 0; bool used = false; };
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
            cp.plan.emplace_back();
            cp.plan.back().g = g;
            if (g.n >= 0) done += (size_t)g.n;
        }
        cps.push_back(std::move(cp));
    }
    // ---- fetch the candidates of all planned groups of all contigs (parallel over groups; a copy of RecRefs when resident)
    const auto tf0 = clk::now();
    {
        std::vector<Planned*> all;
        for (auto& cp : cps) for (auto& p : cp.plan) all.push_back(&p);
        std::atomic<size_t> next{0};
        std::exception_ptr err;
        std::mutex mu;
        auto work = [&]() {
            try {
                for (;;) {
                    const size_t i = next.fetch_add(1);
                    if (i >= all.size()) break;
                    Planned& p = *all[i];
                    Candidates& cur = p.cur.emplace(bam, p.g.tid, p.g.start, p.g.end, req_mapped);
                    const size_t want = p.g.n < 0 ? (size_t)-1 : (size_t)p.g.n * 2 + 32;
                    while (!cur.done && p.pc.recs.size() < want) cur.more(std::min<size_t>(want - p.pc.recs.size(), 4096), &p.pc);
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
        Bulk& bk = bulks.back();
        for (auto& p : cp.plan) { p.lo = bk.pc.recs.size(); append_packed(p.pc, &bk.pc); p.hi = bk.pc.recs.size(); p.pc.clear(); p.pc.heap.shrink_to_fit(); p.pc.hdrs.shrink_to_fit(); }
    }
    res.fetch_s = std::chrono::duration<double>(clk::now() - tf0).count();
    trace_clock().mark(coll.rank, "sampler: candidates fetched + packed");
    if (cfg.device_ready) cfg.device_ready->wait();
    size_t resident_bulk = (size_t)-1;
    for (size_t bi = 0; bi < bulks.size(); bi++) { bulks[bi].take.assign(bulks[bi].pc.recs.size(), 0); decode(bulks[bi].pc, bulks[bi].tid, &bulks[bi].contributes); resident_bulk = bi; }
    trace_clock().mark(coll.rank, "sampler: candidates decoded on the device");
    size_t n_on_demand = 0;
    // ---- the real schedule, contig by contig
    for (auto& cp : cps) {
        const uint32_t t = cp.tid;
        std::vector<Planned>& plan = cp.plan;
        Bulk& bk = bulks[cp.bulk];
        std::map<std::string, size_t> by_key;
        for (size_t i = 0; i < plan.size(); i++) by_key.emplace(key_of(plan[i].g), i);
        std::unordered_set<uint64_t> selected;
        size_t done = 0;
        PackedChunk extra;
        std::vector<uint8_t> xcontrib, xtake;
        for (size_t s = 0; s < sbs.size(); s++) for (const Grp& g : todo_for(s, t, done)) {
            if (cfg.include && !cfg.include->overlaps_any(g.tid, g.start, g.end)) continue;
            const size_t limit = g.n < 0 ? (size_t)-1 : (size_t)g.n;
            size_t used = 0;
            std::optional<Candidates> own;
            Candidates* cur;
            auto it = by_key.find(key_of(g));
            if (it != by_key.end() && !plan[it->second].used) {
                Planned& p = plan[it->second];
                p.used = true;
                select_first(bk.pc.recs, bk.contributes, p.lo, p.hi, limit, &used, &selected, &bk.take);
                cur = &*p.cur;             // (stays with the plan: its buffers are released with the rest, see defer_free)
            } else cur = &own.emplace(bam, g.tid, g.start, g.end, req_mapped);
            // on demand: the plan did not cover the group, or the group needs more candidates than were fetched
            while (!cur->done && used < limit) {
                n_on_demand++;
                extra.clear();
                cur->more(g.n < 0 ? 4096 : (limit - used) * 2 + 32, &extra);
                if (extra.recs.empty()) continue;
                decode(extra, t, &xcontrib);
                resident_bulk = (size_t)-1;
                xtake.assign(extra.recs.size(), 0);
                select_first(extra.recs, xcontrib, 0, extra.recs.size(), limit, &used, &selected, &xtake);
                add_taken(xtake);
                keep(PackedChunk(extra), std::vector<uint8_t>(xtake), t);
            }
            done += used;
        }
        res.n_selected += selected.size();
    }
    if (trace_clock().on) fprintf(stderr, "[mkh r%d]             sampler: %zu on-demand fetches during the replay\n", coll.rank, n_on_demand);
    trace_clock().mark(coll.rank, "sampler: schedule replayed");
    // ---- histogram of the selected reads of every bulk chunk
    for (size_t bi = 0; bi < bulks.size(); bi++) {
        Bulk& bk = bulks[bi];
        if (!any(bk.take)) continue;
        if (resident_bulk != bi) { upload_sampled(bam, ctx, bk.pc, bk.tid, cfg.include); resident_bulk = bi; }
        add_taken(bk.take);
        keep(std::move(bk.pc), std::move(bk.take), bk.tid);
    }
    trace_clock().mark(coll.rank, "sampler: histogram of the selection");
    if (cfg.include_unmapped) {   // reads without coordinates (reads_sampler/mod.rs:85-129): the last rank, after the global count is known
        uint64_t cnt[1] = {res.n_selected};
        coll.sum(cnt, 1);
        if (coll.rank == coll.world - 1) {
            const size_t limit = cfg.take_all ? (size_t)-1 : (cfg.num_reads > cnt[0] ? cfg.num_reads - (size_t)cnt[0] : 0);
            PackedChunk cand;
            Candidates cur(bam, -1, 0, 0, cfg.edge_on);
            while (!cur.done) cur.more(4096, &cand);
            if (!cand.recs.empty()) {
                std::vector<uint8_t> contributes, take(cand.recs.size(), 0);
                decode(cand, 0, &contributes);
                size_t used = 0;
                std::unordered_set<uint64_t> none;
                select_first(cand.recs, contributes, 0, cand.recs.size(), limit, &used, &none, &take);
                add_taken(take);
                res.n_selected += used;
                keep(std::move(cand), std::move(take), 0);
            }
        }
    }
    // ---- the one exchange of a sharded run: sum of the histograms (+ the inexact-value count and the read count)
    if (coll.world > 1) {
        std::vector<uint64_t> buf(res.hist);
        buf.push_back(res.inexact);
        buf.push_back(res.n_selected);
        coll.sum(buf.data(), buf.size());
        std::copy(buf.begin(), buf.begin() + 4 * MKP_HIST_BINS, res.hist.begin());
        res.inexact = buf[4 * MKP_HIST_BINS]; res.n_selected = buf[4 * MKP_HIST_BINS + 1];
    }
    if (cfg.defer_free) *cfg.defer_free = heavy;
    return res;
}

// --sampling-frac / --no-sampling and the schedule's other options. Only -f 1.0 is reproducible without the reference's RNG;
// `alternatives` names the command's other ways to choose the reads.
inline SamplerConfig sampler_config(int threads, uint32_t sampling_interval_size, size_t num_reads, bool have_frac, double frac, bool no_sampling, const char* alternatives) {
    if (!no_sampling && have_frac && frac != 1.0) throw std::runtime_error(std::string("only --sampling-frac 1.0 is reproducible without the reference's RNG; use ") + alternatives);
    SamplerConfig sc;
    sc.threads = sc.workers = threads;
    sc.sampling_interval_size = sampling_interval_size;
    sc.take_all = no_sampling || have_frac;
    sc.num_reads = num_reads;
    return sc;
}

// a quantile of the histogram is exact only when every sampled value lies on its 1/1024 grid; `hint` ends the error otherwise
inline void require_exact(uint64_t inexact, const char* hint) {
    if (inexact) throw std::runtime_error("sampled probabilities are not multiples of 1/1024 (" + std::to_string(inexact) + " values): " + hint);
}

// The estimated thresholds (command_utils.rs:74-134, thresholds.rs:118-156): the `percentile` quantile of every base the sample
// has values for. `announce`: print pileup's "> Using filter threshold" lines.
inline void estimated_thresholds(const SampleResult& s, float percentile, const char* inexact_hint, bool announce, mkp_params* P) {
    require_exact(s.inexact, inexact_hint);
    for (int b = 0; b < 4; b++) {
        const uint64_t* h = s.hist.data() + b * MKP_HIST_BINS;
        if (std::all_of(h, h + MKP_HIST_BINS, [](uint64_t v) { return v == 0; })) continue;
        float thr;
        if (!percentile_from_hist(h, percentile, &thr)) throw std::runtime_error("not enough datapoints to estimate a threshold");
        P->base_threshold_set[b] = 1;
        P->base_threshold[b] = thr;
        if (announce) fprintf(stderr, "> Using filter threshold %.9g for %c.\n", thr, "ACGT"[b]);
    }
}

// ---- the filter flags shared by pileup, pileup-hemi, summary and sample-probs (command_utils.rs:18-73, 243-275)
// --edge-filter N | START,END and --invert-edge-filter
inline void parse_edge_filter(const std::string& raw, bool invert, mkp_params* P) {
    if (raw.empty()) return;
    P->edge_filter_on = 1; P->edge_filter_inverted = invert;
    auto c = raw.find(',');
    if (c == std::string::npos) P->edge_filter_start = P->edge_filter_end = (uint32_t)std::stoul(raw);
    else { P->edge_filter_start = (uint32_t)std::stoul(raw.substr(0, c)); P->edge_filter_end = (uint32_t)std::stoul(raw.substr(c + 1)); }
}
// --mod-thresholds CODE:VALUE (repeatable)
inline void parse_mod_thresholds(const std::vector<std::string>& raws, mkp_params* P) {
    for (auto& raw : raws) {
        auto c = raw.find(':');
        uint32_t code;
        if (c == std::string::npos || raw.find(':', c + 1) != std::string::npos || !parse_code(raw.substr(0, c), &code))
            throw std::runtime_error("encountered illegal per-mod threshold: " + raw + ". Should be mod_code:threshold e.g. h:0.8");
        if (P->n_mod_thresholds >= MKP_MAX_MOD_THRESHOLDS) throw std::runtime_error("too many per-mod thresholds");
        P->mod_code[P->n_mod_thresholds] = code;
        P->mod_threshold[P->n_mod_thresholds++] = std::stof(raw.substr(c + 1));
    }
}
// --filter-threshold [BASE:]VALUE (repeatable): one default, one per base
inline void parse_filter_thresholds(const std::vector<std::string>& raws, mkp_params* P) {
    bool have_default = false;
    for (auto& raw : raws) {
        auto c = raw.find(':');
        if (c == std::string::npos) {
            if (have_default) throw std::runtime_error("default threshold encountered more than once");
            P->default_threshold = std::stof(raw); have_default = true;
        } else {
            const char* B = "ACGT";
            const char* f = raw.empty() ? nullptr : strchr(B, raw[0]);
            if (!f || !raw[0]) throw std::runtime_error("failed to parse base " + raw);
            if (P->base_threshold_set[f - B]) throw std::runtime_error(std::string("repeated threshold for base ") + raw[0]);
            P->base_threshold_set[f - B] = 1;
            P->base_threshold[f - B] = std::stof(raw.substr(c + 1));
        }
    }
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
    double slice_s = 0, pass_s = 0, rowcopy_s = 0;     // parts of gpu_s: making the chunk resident (GPU slicing or upload), kernels, rows to the host
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

// the context of CUDA device `device`; this build has no CPU fallback, so a machine without a usable device stops here
inline mkp_ctx* open_device(int device) {
    mkp_ctx* ctx = nullptr;
    if (const int rc = mkp_create(device, &ctx)) throw std::runtime_error("no usable CUDA device (mkp_create returned " + std::to_string(rc) + "); this build has no CPU fallback");
    return ctx;
}
inline void check_mkp(mkp_ctx* ctx, int rc) { if (rc) throw std::runtime_error(mkp_last_error(ctx)); }

// A job on a thread of its own. An exception it throws is kept and rethrown by join(). `release` (optional) runs on the owner's
// thread before the join, to let go a job that may be waiting on the owner. Declare the job after every object it touches, so
// that it is destroyed (joined) before they are.
class BackgroundJob {
    std::function<void()> release_;
    std::exception_ptr err_;
    std::thread t_;
public:
    explicit BackgroundJob(std::function<void()> fn, std::function<void()> release = nullptr)
        : release_(std::move(release)), t_([this, fn = std::move(fn)]() { try { fn(); } catch (...) { err_ = std::current_exception(); } }) {}
    ~BackgroundJob() { if (t_.joinable()) { if (release_) release_(); t_.join(); } }
    void join() { if (release_) release_(); t_.join(); if (err_) std::rethrow_exception(err_); }
};

// What a pileup run needs from its options. The constructor makes every check that needs no device and no file, in the
// reference's order, so argument errors need no GPU; open_inputs and lay_out follow once the BAM header is read.
struct PileupPlan {
    mkp_params P{};                    // the thresholds are added once the output exists (subcommand.rs:615-638)
    MotifContext mc;
    BedFormat fmt;
    bool have_motifs = false, combine_strands = false;
    bool to_dir = false;               // the output path is a directory (writers.rs:264-381, 1005-1082)
    int32_t hemi_partner = 0;          // pileup-hemi: MotifInfo::negative_strand_position
    std::optional<Region> region, sregion;
    std::vector<RefTarget> targets, iv_targets;
    IncludeBed include;
    const IncludeBed* inc = nullptr;
    std::vector<RefInterval> ivs;
    std::vector<size_t> iv_owner;
    size_t my_i0 = 0, my_i1 = 0;       // this rank's intervals
    PileupPlan(const PileupPlan&) = delete;
    PileupPlan(const PileupOptions& o, bool sharded) {
        if (o.percentile > 1.0f) throw std::runtime_error("filter percentile must be <= 1.0");
        MotifSpec hemi_m;
        if (o.hemi) { hemi_m = hemi_motif(o); hemi_partner = hemi_m.rc_offset - hemi_m.offset; }
        // util.rs:690-712
        for (size_t i = 0; i < o.partition_tags.size(); i++) {
            if (o.partition_tags[i].size() != 2) throw std::runtime_error("illegal tag " + o.partition_tags[i] + " should be length 2");
            for (size_t j = 0; j < i; j++) if (o.partition_tags[j] == o.partition_tags[i]) throw std::runtime_error("cannot repeat partition-tags, got " + o.partition_tags[i] + " twice");
        }
        to_dir = !o.partition_tags.empty() || o.bedgraph;
        if (to_dir && o.header) throw std::runtime_error("the argument '--header' cannot be used with '--bedgraph' / '--partition-tag'");
        if (o.bedgraph && o.mixed) throw std::runtime_error("the argument '--mixed-delim' cannot be used with '--bedgraph'");
        if (sharded && (o.bedgraph || o.host_ingest)) throw std::runtime_error("multi-GPU runs write one bedMethyl file through the device ingest, or one per partition: --bedgraph / --host-ingest need a single device");
        if (sharded && (o.out_bed == "-" || o.out_bed == "stdout")) throw std::runtime_error("multi-GPU runs need an output file (ranks write their slices at their offsets)");
        combine_strands = o.combine_strands || o.hemi;        // pileup-hemi: the feeder runs in combine-strands mode
        if (combine_strands && !(o.cpg || !o.motif_parts.empty())) throw std::runtime_error("need to specify either --motif or --cpg to combine strands");
        P.force_allow_implicit = o.force_allow;
        P.max_depth = o.max_depth;
        if (o.traditional) { P.numeric_mode = 2; P.collapse_code = 'h'; combine_strands = true; }
        else if (o.combine_mods) P.numeric_mode = 1;
        else if (!o.ignore.empty()) { uint32_t c; if (!parse_code(o.ignore, &c)) throw std::runtime_error("failed to parse mod code " + o.ignore); P.numeric_mode = 2; P.collapse_code = c; }
        parse_edge_filter(o.edge, o.invert_edge, &P);
        // motifs (subcommand.rs:526-539, 592-612)
        std::vector<std::string> parts = o.motif_parts;
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
        fmt.mixed_delim = o.mixed;
        for (auto& m : mc.motifs) fmt.motif_labels.push_back(m.label());
        if (have_motifs) {
            if (o.ref_fp.empty()) throw std::runtime_error("reference fasta is required for using --motif or --cpg options");
            if (combine_strands) for (auto& m : mc.motifs) if (!m.palindromic) throw std::runtime_error("cannot combine strands with a motif that is not a palindrome");
            mc.keep_case = o.mask;
            for (auto& m : mc.motifs) mc.longest = std::max<uint64_t>(mc.longest, m.len);
        }
    }
    // what the BAM header and the input files decide: the regions, the targets, --include-bed and the FASTA
    void open_inputs(const PileupOptions& o, const BamReader& bam) {
        if (!o.region.empty()) region = parse_region_arg(o.region, bam);
        if (!o.sample_region.empty()) sregion = parse_region_arg(o.sample_region, bam);
        for (uint32_t t = 0; t < bam.ref_names.size(); t++) {
            if (region) { if (bam.ref_names[t] == region->name) targets.push_back({t, region->start, region->end - region->start, region->name}); }
            else targets.push_back({t, 0, bam.ref_lens[t], bam.ref_names[t]});
        }
        if (!o.include_bed.empty()) {
            std::map<std::string, uint32_t> name_to_tid;
            for (auto& t : targets) name_to_tid[t.name] = t.tid;
            include.read(o.include_bed, name_to_tid);
            inc = &include;
        }
        if (have_motifs) { mc.fasta.open(o.ref_fp); mc.include = inc; }
    }
    // the reference intervals: boundaries and shard cuts now (cheap), the focus positions of this rank's range in the background
    void lay_out(const PileupOptions& o, const BamReader& bam, const Collective& coll) {
        iv_targets = inc ? targets_from_include_bed(*inc, targets, o.interval_size) : targets;
        ivs = interval_grid(iv_targets, o.interval_size, combine_strands, have_motifs ? &mc : nullptr, &iv_owner);
        my_i1 = ivs.size();
        if (coll.world > 1) { const std::vector<size_t> cuts = shard_cuts(bam, ivs, coll.world); my_i0 = cuts[coll.rank]; my_i1 = cuts[coll.rank + 1]; }
    }
};

// The records of the pileup: with the device ingest everything, or the byte ranges under this rank's intervals, is loaded on the
// GPU. A BAM too big for it is read on the host: a front-end choice, not a compute fallback (the reads are sliced on the host and
// uploaded chunk by chunk). That reader is one of its own, `host_bam`: the sampler may still be fetching through `bam`.
inline BamReader& load_reads(const PileupOptions& o, const PileupPlan& plan, bool sharded, BamReader& bam, std::optional<BamReader>* host_bam) {
    if (o.host_ingest) return bam;
    if (!sharded) {
        try { bam.load_default(); return bam; }
        catch (const DeviceIngestTooBig& e) {
            if (!o.quiet) fprintf(stderr, "> %s; reading the BAM on the host instead\n", e.what());
            host_bam->emplace();
            (*host_bam)->open(o.in_bam, o.threads);
            return **host_bam;
        }
    }
    std::vector<BamReader::Piece> pieces;
    for (size_t i = plan.my_i0; i < plan.my_i1; i++) {
        if (!pieces.empty() && pieces.back().tid == plan.ivs[i].tid) pieces.back().hi = std::max(pieces.back().hi, plan.ivs[i].end);
        else pieces.push_back({plan.ivs[i].tid, plan.ivs[i].start, plan.ivs[i].end});
    }
    bam.load_pieces(pieces);
    return bam;
}

// a chunk = consecutive intervals [c0, c1) of one contig, up to chunk_bp
inline size_t chunk_end(const std::vector<RefInterval>& ivs, size_t c0, uint32_t chunk_bp) {
    size_t c1 = c0 + 1;
    while (c1 < ivs.size() && ivs[c1].tid == ivs[c0].tid && ivs[c1].start == ivs[c1 - 1].end && ivs[c1].end - ivs[c0].start <= chunk_bp) c1++;
    return c1;
}

struct ChunkWork { size_t i0, i1; std::vector<RecRef> recs; };
// The device work of the chunk [c0, c1) with reads `recs`. --max-depth (src/pileup/mod.rs:755-759 -> bam_plp_set_maxcnt): the
// pileup engine of the reference runs per interval and drops reads while its buffer is full, so the reads that count can differ
// from interval to interval. Only a chunk that holds more reads than the limit can be affected: it is then processed interval by
// interval, each with the reads its own engine would keep. (Parity unpinned by the reference's tests; rule restated in
// depth_limit_keep.)
inline std::vector<ChunkWork> chunk_work(const std::vector<RefInterval>& ivs, size_t c0, size_t c1, std::vector<RecRef>&& recs, uint32_t max_depth) {
    if (max_depth && recs.size() > max_depth) {
        std::vector<ChunkWork> per_iv;
        bool split = false;
        for (size_t k = c0; k < c1; k++) {
            ChunkWork w{k, k + 1, {}};
            for (auto& r : recs) if (r.pos < (int64_t)ivs[k].end && r.end > (int64_t)ivs[k].start) w.recs.push_back(r);
            const size_t before = w.recs.size();
            depth_limit_keep(&w.recs, max_depth);
            split = split || w.recs.size() != before;
            per_iv.push_back(std::move(w));
        }
        if (split) return per_iv;
    }
    std::vector<ChunkWork> whole;
    whole.push_back({c0, c1, std::move(recs)});
    return whole;
}

// With --partition-tag one group of reads per key (each an independent pileup: src/pileup/mod.rs:795-830), in key order, "\1" for
// the reads without a key; otherwise one group "" of all reads. Device-resident records give their tag values on the GPU
// (mkp_bam_tag_values, four tags per call, values of any length); `vals` is the host buffer of those values, kept between calls.
inline std::map<std::string, std::vector<RecRef>> partition_groups(mkp_ctx* ctx, const BamReader& reads, const std::vector<std::string>& tags, std::vector<RecRef>&& recs,
                                                                   std::vector<uint8_t>* vals) {
    std::map<std::string, std::vector<RecRef>> groups;
    if (tags.empty()) { groups[""] = std::move(recs); return groups; }
    // only alignments the pileup admits create a key (flag filter of the pileup engine, pileup/mod.rs:783-791)
    std::vector<RecRef> adm;
    for (auto& r : recs) if (!((r.flag & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)) || r.l_seq == 0)) adm.push_back(r);
    const size_t n_pt = tags.size();
    // per (record, tag), record-major: aux type, value length, value offset in `vals`
    std::vector<uint8_t> types;
    std::vector<uint32_t> lens;
    std::vector<uint64_t> offs;
    if (reads.on_device && !adm.empty()) {
        const size_t n = adm.size();
        std::vector<uint32_t> ids(n);
        for (size_t k = 0; k < n; k++) ids[k] = adm[k].idx;
        types.resize(n * n_pt); lens.resize(n * n_pt); offs.resize(n * n_pt);
        std::vector<uint8_t> pt;
        std::vector<uint32_t> pl, po;
        size_t base = 0;                   // the values of earlier calls (tags t0 - 4 ...) come first in `vals`
        for (size_t t0 = 0; t0 < n_pt; t0 += 4) {
            const size_t nt4 = std::min<size_t>(4, n_pt - t0);
            std::string tg;
            for (size_t t = t0; t < t0 + nt4; t++) tg += tags[t];
            pt.resize(n * nt4); pl.resize(n * nt4); po.resize(n * nt4);
            uint64_t total = 0;
            if (vals->size() < base) vals->resize(base);
            auto call = [&]() {
                check_mkp(ctx, mkp_bam_tag_values(ctx, ids.data(), (uint32_t)n, tg.c_str(), (uint32_t)nt4, pt.data(), pl.data(), po.data(),
                                                  vals->data() + base, vals->size() - base, &total));
            };
            call();
            if (vals->size() - base < total) { vals->resize(base + total); call(); }       // sized by the first call
            for (size_t k = 0; k < n; k++)
                for (size_t t = 0; t < nt4; t++) {
                    const size_t q = k * n_pt + t0 + t, j = k * nt4 + t;
                    types[q] = pt[j]; lens[q] = pl[j]; offs[q] = base + po[j];
                }
            base += total;
        }
    }
    for (size_t k = 0; k < adm.size(); k++) {
        std::string key;
        const bool have = reads.on_device ? partition_key_of_values(types.data() + k * n_pt, lens.data() + k * n_pt, offs.data() + k * n_pt, vals->data(), n_pt, &key)
                                          : partition_key_of(reads.rec(adm[k]), adm[k].size, tags, &key);
        groups[have ? key : std::string("\1")].push_back(adm[k]);
    }
    return groups;
}

struct ChunkOut { size_t i0 = 0, i1 = 0; std::string key_name; std::vector<mkp_row> rows; std::vector<mkp_hemi_row> hemi_rows; bool last = false; };
// From the device stage to the formatting stage: at most two finished chunks wait; row buffers travel back (no fresh pages per chunk)
struct ChunkQueue {
    std::mutex mu;
    std::condition_variable cv;
    std::deque<ChunkOut> q;
    std::vector<std::vector<mkp_row>> spare_rows;
    bool consumer_gone = false;
    void push(ChunkOut&& co) { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return q.size() < 2 || consumer_gone; }); q.push_back(std::move(co)); cv.notify_all(); }
    ChunkOut pop() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return !q.empty(); }); ChunkOut co = std::move(q.front()); q.pop_front(); cv.notify_all(); return co; }
    void take_spare(std::vector<mkp_row>* rows) { std::lock_guard<std::mutex> lk(mu); if (!spare_rows.empty()) { rows->swap(spare_rows.back()); spare_rows.pop_back(); } }
    void recycle(std::vector<mkp_row>&& rows) { std::lock_guard<std::mutex> lk(mu); rows.clear(); if (spare_rows.size() < 4) spare_rows.push_back(std::move(rows)); }
    void leave() { std::lock_guard<std::mutex> lk(mu); consumer_gone = true; cv.notify_all(); }
};

// One group of reads on the device: the chunk made resident (sliced on the GPU from device-resident records, or the packed reads
// uploaded), the pass (pileup, or pileup-hemi over the intervals starting at `starts`), the rows copied into `co`
inline void device_step(mkp_ctx* ctx, const BamReader& reads, const mkp_chunk& ch, bool hemi, const std::vector<uint32_t>& starts, int32_t hemi_partner,
                        bool want_alg_bytes, PackedChunk* pc, ChunkOut* co, RunSummary* S) {
    using clk = std::chrono::steady_clock;
    const auto t0 = clk::now();
    if (reads.on_device) device_chunk(reads, pc->recs, ch.start, ch.end, ch.focus_pos, ch.focus_neg);
    else check_mkp(ctx, mkp_upload_chunk(ctx, &ch));
    const auto t_s = clk::now();
    mkp_stats st;
    check_mkp(ctx, hemi ? mkp_hemi_resident(ctx, starts.data(), (uint32_t)starts.size(), hemi_partner, &st) : mkp_pileup_resident(ctx, &st));
    const auto t_k = clk::now();
    const mkp_row* rows = nullptr;
    const mkp_hemi_row* hemi_rows = nullptr;
    size_t n_rows = 0;
    check_mkp(ctx, hemi ? mkp_fetch_hemi_rows(ctx, &hemi_rows, &n_rows) : mkp_fetch_rows(ctx, &rows, &n_rows));
    S->slice_s += secs_between(t0, t_s); S->pass_s += secs_between(t_s, t_k); S->rowcopy_s += secs_between(t_k, clk::now());
    if (want_alg_bytes && reads.on_device) {     // the headers of the reads the GPU sliced
        pc->hdrs.resize(pc->recs.size());
        uint32_t nr = 0;
        check_mkp(ctx, mkp_fetch_chunk(ctx, pc->hdrs.data(), &nr, nullptr, nullptr));
    }
    if (hemi) co->hemi_rows.assign(hemi_rows, hemi_rows + n_rows);
    else co->rows.assign(rows, rows + n_rows);          // the context's row buffer is reused by the next chunk
    S->kernel_ms += st.kernel_ms[7];
    S->algorithmic_bytes += (want_alg_bytes || !reads.on_device ? pc->algorithmic_bytes() : 0) + (hemi ? sizeof(mkp_hemi_row) : sizeof(mkp_row)) * n_rows;
    S->reads_packed += pc->recs.size();
    S->chunks++;
    S->gpu_s += secs_between(t0, clk::now());
}

// The device stage: the reads of chunk after chunk, each unit of work and partition group through device_step, in output order
inline void device_stage(mkp_ctx* ctx, const BamReader& reads, const PileupOptions& o, const PileupPlan& plan, ChunkQueue* queue, RunSummary* S) {
    using clk = std::chrono::steady_clock;
    const std::vector<RefInterval>& ivs = plan.ivs;
    PackedChunk pc;
    std::vector<uint32_t> fpos, fneg;
    std::vector<uint8_t> tag_vals;
    for (size_t c0 = 0, c1; c0 < ivs.size(); c0 = c1) {
        c1 = chunk_end(ivs, c0, o.chunk_bp);
        if (ivs[c1 - 1].end <= ivs[c0].start) continue;
        std::vector<RecRef> recs;
        reads.ensure_tid(ivs[c0].tid);
        reads.for_overlapping(ivs[c0].tid, ivs[c0].start, ivs[c1 - 1].end, [&](const RecRef& r) { recs.push_back(r); });
        if (recs.empty()) continue;
        for (ChunkWork& wk : chunk_work(ivs, c0, c1, std::move(recs), o.max_depth)) {
            const size_t i0 = wk.i0, i1 = wk.i1;
            const uint32_t cs = ivs[i0].start, ce = ivs[i1 - 1].end;
            if (ce <= cs || wk.recs.empty()) continue;
            // pileup-hemi: the call window reaches the partner of every motif position; the reads stay those of the intervals
            mkp_chunk ch{};
            ch.start = cs - (plan.hemi_partner < 0 ? std::min<uint32_t>(cs, (uint32_t)-plan.hemi_partner) : 0);
            ch.end = plan.hemi_partner > 0 ? (uint32_t)std::min<uint64_t>((uint64_t)ce + (uint32_t)plan.hemi_partner, std::max(ce, reads.ref_lens[ivs[i0].tid])) : ce;
            std::vector<uint32_t> starts;
            if (o.hemi) for (size_t k = i0; k < i1; k++) starts.push_back(ivs[k].start);
            bool focus_done = false;
            for (auto& grp : partition_groups(ctx, reads, o.partition_tags, std::move(wk.recs), &tag_vals)) {
                const auto ta = clk::now();
                pc.clear();
                if (reads.on_device) pc.recs = grp.second;
                else pack_records_mt(reads, grp.second, o.threads, &pc);
                if (pc.recs.empty()) continue;
                ch.hdrs = pc.hdrs.data(); ch.n_reads = (uint32_t)pc.hdrs.size(); ch.heap = pc.heap.data(); ch.heap_bytes = pc.heap.size();
                if (plan.have_motifs || plan.inc) { if (!focus_done) { focus_bitmaps(ivs, i0, i1, ch.start, ch.end, &fpos, &fneg); focus_done = true; } ch.focus_pos = fpos.data(); ch.focus_neg = fneg.data(); }
                S->pack_s += secs_between(ta, clk::now());
                ChunkOut co{i0, i1, grp.first == "\1" ? std::string("ungrouped") : grp.first};
                queue->take_spare(&co.rows);
                device_step(ctx, reads, ch, o.hemi, starts, plan.hemi_partner, !o.stats_json.empty(), &pc, &co, S);
                queue->push(std::move(co));
            }
        }
    }
}

// Where the text goes: a stream (stdout, or a file that is not regular); a regular file, which the formatting workers write in
// place; a directory of files made on first use (--bedgraph / --partition-tag); or, in a sharded run, this rank's slice of the
// one file, written at its offset at the end. The output is made first, like the reference, so a bad path fails before any work.
class PileupWriter {
    const std::string path_;
    const Collective coll_;
    FILE* out_ = nullptr;
    int fd_ = -1;                      // out_ is a regular file: written in place, at pos_
    uint64_t pos_ = 0;
    std::map<std::string, FILE*> files_;
    std::vector<std::string> parts_;                          // per formatting worker (capacity kept from chunk to chunk)
    std::vector<std::map<std::string, std::string>> routed_;  // per formatting worker, to a directory: file name -> text
    std::vector<std::string> slice_;   // sharded: the header (rank 0), then the formatted parts in order
    const bool to_dir_;
    std::map<std::string, std::vector<std::string>> dir_slices_;   // sharded, to a directory: file name -> its formatted parts in order
    static bool pwrite_all(int fd, const std::string& text, uint64_t offset) {
        for (size_t done = 0; done < text.size();) {
            const ssize_t w = pwrite(fd, text.data() + done, text.size() - done, (off_t)(offset + done));
            if (w <= 0) return false;
            done += (size_t)w;
        }
        return true;
    }
    FILE* file(const std::string& name) {
        FILE*& f = files_[name];
        if (!f && !(f = fopen((path_ + "/" + name).c_str(), "w"))) { files_.erase(name); throw std::runtime_error("failed to make output file " + path_ + "/" + name); }
        return f;
    }
public:
    PileupWriter(const PileupOptions& o, bool to_dir, const Collective& coll) : path_(o.out_bed), coll_(coll), to_dir_(to_dir) {
        if (coll.world > 1 && to_dir) {
            if (coll.rank == 0) {             // the files are made at the end, once the ranks agree on them
                std::error_code ec;
                std::filesystem::create_directories(path_, ec);
                if (ec) throw std::runtime_error("failed to create output directory " + path_);
            }
        } else if (coll.world > 1) {
            if (coll.rank == 0) {
                FILE* f = fopen(path_.c_str(), "w");     // created (and truncated) by rank 0 before the first exchange
                if (!f) throw std::runtime_error("failed to make output file");
                fclose(f);
            }
            slice_.push_back(coll.rank == 0 && o.header ? bed_header_line() : "");
        } else if (!to_dir) {
            out_ = (path_ == "-" || path_ == "stdout") ? stdout : fopen(path_.c_str(), "w");
            if (!out_) throw std::runtime_error("failed to make output file");
            if (o.header) fputs(bed_header_line(), out_);
            if (out_ != stdout) {
                fflush(out_);
                struct stat sb;
                const off_t at = ftello(out_);
                if (at >= 0 && fstat(fileno(out_), &sb) == 0 && S_ISREG(sb.st_mode)) { fd_ = fileno(out_); pos_ = (uint64_t)at; }
            }
        } else {
            std::error_code ec;
            std::filesystem::create_directories(path_, ec);
            if (ec) throw std::runtime_error("failed to create output directory " + path_);
        }
    }
    ~PileupWriter() { if (out_ && out_ != stdout) fclose(out_); for (auto& kv : files_) fclose(kv.second); }

    // one chunk, formatted by nt workers of the pool: format(t, text, files) fills worker t's text, or its files of a directory
    void write_chunk(WorkerPool& pool, int nt, const std::function<void(int, std::string*, std::map<std::string, std::string>*)>& format) {
        if ((int)parts_.size() < nt) { parts_.resize(nt); routed_.resize(nt); }
        for (auto& p : parts_) p.clear();
        for (auto& r : routed_) r.clear();
        std::unique_ptr<std::atomic<uint64_t>[]> psize(new std::atomic<uint64_t>[nt]);
        for (int t = 0; t < nt; t++) psize[t].store(UINT64_MAX);
        std::atomic<bool> failed{false};
        pool.run(nt, [&](int t) {
            struct Publish { std::atomic<uint64_t>* a; ~Publish() { if (a->load() == UINT64_MAX) a->store(0); } } guard{&psize[t]};      // (a worker that leaves early must not block the others)
            format(t, &parts_[t], &routed_[t]);
            if (fd_ < 0) return;
            // the text of worker t follows the text of the workers before it: wait for their sizes, then write in place
            psize[t].store(parts_[t].size(), std::memory_order_release);
            uint64_t at = pos_;
            for (int q = 0; q < t; q++) { uint64_t v; while ((v = psize[q].load(std::memory_order_acquire)) == UINT64_MAX) std::this_thread::yield(); at += v; }
            if (!pwrite_all(fd_, parts_[t], at)) failed = true;
        });
        if (failed) throw std::runtime_error("failed to write output file " + path_);
        for (int t = 0; t < nt; t++) {
            if (coll_.world > 1) { if (!parts_[t].empty()) slice_.push_back(std::move(parts_[t])); }
            else if (fd_ >= 0) pos_ += parts_[t].size();
            else if (out_) fwrite(parts_[t].data(), 1, parts_[t].size(), out_);
            for (auto& kv : routed_[t]) {
                if (kv.second.empty()) continue;
                if (coll_.world > 1) dir_slices_[kv.first].push_back(std::move(kv.second));
                else fwrite(kv.second.data(), 1, kv.second.size(), file(kv.first));
            }
        }
    }

    // The end of the output. Sharded: rank-ordered concatenation (the reference's ordered collect, src/pileup/subcommand.rs:735-799):
    // the slice sizes are exchanged (second and last collective) and every rank writes its slice at its offset, on the pool.
    void finish(WorkerPool& pool, RunSummary* S) {
        if (out_) { if (out_ != stdout) fclose(out_); else fflush(out_); out_ = nullptr; }
        if (coll_.world <= 1) { S->rows_total = S->rows; S->positions_total = S->positions; return; }
        const auto tw = std::chrono::steady_clock::now();
        if (to_dir_) { finish_dir(pool, S); S->write_s += secs_between(tw, std::chrono::steady_clock::now()); return; }
        std::vector<uint64_t> sizes((size_t)coll_.world + 2, 0), at(slice_.size());
        for (auto& s : slice_) sizes[coll_.rank] += s.size();
        sizes[coll_.world] = S->rows; sizes[(size_t)coll_.world + 1] = S->positions;
        coll_.sum(sizes.data(), sizes.size());
        uint64_t a = std::accumulate(sizes.begin(), sizes.begin() + coll_.rank, (uint64_t)0);
        for (size_t k = 0; k < slice_.size(); k++) { at[k] = a; a += slice_[k].size(); }
        const int fd = ::open(path_.c_str(), O_WRONLY);
        if (fd < 0) throw std::runtime_error("failed to open output file " + path_);
        std::atomic<bool> failed{false};
        pool.run((int)slice_.size(), [&](int k) { if (!failed && !pwrite_all(fd, slice_[k], at[k])) failed = true; });
        ::close(fd);
        if (failed) throw std::runtime_error("failed to write output file " + path_);
        S->rows_total = sizes[coll_.world]; S->positions_total = sizes[(size_t)coll_.world + 1];
        S->write_s += secs_between(tw, std::chrono::steady_clock::now());
    }
    // Sharded, to a directory: the ranks agree on the files and on every rank's offset in each (agree_file_slices); rank 0 makes
    // (or truncates) every file that gets text, the next exchange holds the others back until that is done, then every rank writes
    // its parts in place. Files no rank has text for are not touched, as with one device.
    void finish_dir(WorkerPool& pool, RunSummary* S) {
        std::map<std::string, uint64_t> mine;
        for (auto& kv : dir_slices_) { uint64_t n = 0; for (auto& part : kv.second) n += part.size(); mine[kv.first] = n; }
        const FileSlices fs = agree_file_slices(coll_, mine);
        uint64_t made_fail = 0;
        if (coll_.rank == 0)
            for (size_t f = 0; f < fs.names.size(); f++) {
                if (!fs.total[f]) continue;
                const int fd = ::open((path_ + "/" + fs.names[f]).c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0666);
                if (fd < 0) { made_fail = 1; break; }
                ::close(fd);
            }
        uint64_t done[3] = {made_fail, S->rows, S->positions};
        coll_.sum(done, 3);
        if (done[0]) throw std::runtime_error("failed to make output files in " + path_);
        struct Job { int fd; const std::string* text; uint64_t at; };
        std::vector<Job> jobs;
        std::vector<int> fds;
        bool open_failed = false;
        for (size_t f = 0; f < fs.names.size() && !open_failed; f++) {
            auto it = dir_slices_.find(fs.names[f]);
            if (it == dir_slices_.end()) continue;
            const int fd = ::open((path_ + "/" + fs.names[f]).c_str(), O_WRONLY);
            if (fd < 0) { open_failed = true; break; }
            fds.push_back(fd);
            uint64_t at = fs.offset[f];
            for (auto& part : it->second) { jobs.push_back({fd, &part, at}); at += part.size(); }
        }
        std::atomic<bool> failed{open_failed};
        if (!open_failed) pool.run((int)jobs.size(), [&](int k) { if (!failed && !pwrite_all(jobs[k].fd, *jobs[k].text, jobs[k].at)) failed = true; });
        for (int fd : fds) ::close(fd);
        if (failed) throw std::runtime_error("failed to write output files in " + path_);
        S->rows_total = done[1]; S->positions_total = done[2];
    }
    void release_buffers() { parts_.clear(); parts_.shrink_to_fit(); slice_.clear(); slice_.shrink_to_fit(); dir_slices_.clear(); }
};

// The rows of one chunk as text (position sorted: every interval gets its slice; intervals are formatted in parallel); row count
inline uint64_t format_chunk(const ChunkOut& co, const PileupOptions& o, const PileupPlan& plan, const std::string& chrom, WorkerPool& pool, PileupWriter* out) {
    const std::vector<RefInterval>& ivs = plan.ivs;
    const size_t i0 = co.i0, n_iv = co.i1 - co.i0;
    const mkp_row* rows = co.rows.data();
    const size_t n_rows = o.hemi ? co.hemi_rows.size() : co.rows.size();
    auto pos_of = [&](size_t j) { return o.hemi ? co.hemi_rows[j].pos : rows[j].pos; };
    std::vector<size_t> rlo(n_iv + 1);
    {
        size_t r0 = 0;
        for (size_t k = 0; k < n_iv; k++) { while (r0 < n_rows && pos_of(r0) < ivs[i0 + k].start) r0++; rlo[k] = r0; }
        size_t r1 = rlo[n_iv - 1];
        while (r1 < n_rows && pos_of(r1) < ivs[co.i1 - 1].end) r1++;
        rlo[n_iv] = r1;
    }
    const int nt = std::max(1, std::min<int>(o.threads, (int)n_iv));
    const std::string pfx = o.prefix.empty() ? std::string() : o.prefix + "_";
    std::vector<uint64_t> part_rows(nt, 0);
    out->write_chunk(pool, nt, [&](int t, std::string* text, std::map<std::string, std::string>* files) {
        std::vector<OutRow> local;
        for (size_t k = n_iv * t / nt; k < n_iv * (t + 1) / nt; k++) {
            const size_t r_end = k + 1 < n_iv ? std::max(rlo[k], rlo[k + 1]) : rlo[n_iv];
            size_t r1 = rlo[k];
            while (r1 < r_end && pos_of(r1) < ivs[i0 + k].end) r1++;
            if (o.hemi) {       // rows are final: one per (position, base, pattern), in output order
                for (size_t j = rlo[k]; j < r1; j++) format_hemi_row(co.hemi_rows[j], chrom, o.mixed, text);
                part_rows[t] += r1 - rlo[k];
                continue;
            }
            local.clear();
            finish_interval_rows(ivs[i0 + k], rows + rlo[k], r1 - rlo[k], plan.have_motifs ? &plan.mc.motifs : nullptr, plan.combine_strands, &local);
            if (!plan.to_dir) for (auto& orow : local) format_bed_row(orow, chrom, plan.fmt, text);
            else if (!o.bedgraph) { std::string& dst = (*files)[pfx + co.key_name + ".bed"]; for (auto& orow : local) format_bed_row(orow, chrom, plan.fmt, &dst); }
            else for (auto& orow : local) {
                std::string& dst = (*files)[pfx + co.key_name + (co.key_name.empty() ? "" : "_") + bedgraph_label(orow, plan.fmt) + "_" + strand_label(orow.strand) + ".bedgraph"];
                format_bedgraph_row(orow, chrom, &dst);
            }
            part_rows[t] += local.size();
        }
    });
    return std::accumulate(part_rows.begin(), part_rows.end(), (uint64_t)0);
}

inline int run_pileup(const PileupOptions& o, RunSummary* summary, std::string* error, const Collective* coll_in = nullptr) {
    using clk = std::chrono::steady_clock;
    const Collective coll = coll_in ? *coll_in : Collective();
    const bool sharded = coll.world > 1;
    try {
        const auto t0 = clk::now();
        trace_clock().epoch = t0;
        auto trace = [&](const char* what) { trace_clock().mark(coll.rank, what); };
        PileupPlan plan(o, sharded);
        // the device comes first: with the device ingest (default) the BAM is inflated and sliced on the GPU
        DeviceGuard dev{open_device(o.device)};
        trace("device context created");
        BamReader bam;
        if (o.host_ingest) bam.open(o.in_bam, o.threads);
        else bam.open_device_index(o.in_bam, dev.ctx);         // header + index; the device load follows once the shard is known
        plan.open_inputs(o, bam);
        trace("index + fasta opened");
        const auto t_iv0 = clk::now();
        plan.lay_out(o, bam, coll);
        // ---- threshold estimation. With the device ingest of an indexed BAM it starts now, beside the load: its candidates come
        // straight from the file (host fetch through the index), only its decode passes need the device and wait for `dev_ready`.
        // Otherwise it runs after the load, on the reads of the pileup.
        const bool estimate = o.filter_thresholds.empty() && !o.no_filtering;
        SamplerConfig sc;
        std::shared_ptr<void> sample_garbage;
        std::promise<SampleResult> sample_p;
        std::future<SampleResult> sample_f = sample_p.get_future();
        auto run_sampler = [&](const BamReader& src) {
            try { sample_p.set_value(sample_histogram(src, dev.ctx, sc, coll)); }
            catch (...) { sample_p.set_exception(std::current_exception()); }
            sample_garbage.reset();              // the result is out; the candidate buffers are released after that, beside the pileup
        };
        std::promise<void> dev_ready_p;
        std::shared_future<void> dev_ready_f = dev_ready_p.get_future().share();
        bool dev_ready_set = false;
        auto set_dev_ready = [&]() { if (!dev_ready_set) { dev_ready_p.set_value(); dev_ready_set = true; } };
        std::optional<BackgroundJob> sampler_job;
        trace("interval grid + shard cuts");
        if (estimate) {
            sc = sampler_config(o.schedule_threads > 0 ? o.schedule_threads : o.threads, o.sampling_interval_size, o.num_reads, o.have_frac, o.frac, false, "-n or -f 1.0");
            sc.workers = o.threads;
            sc.region = plan.sregion ? &*plan.sregion : plan.region ? &*plan.region : nullptr;
            sc.include_unmapped = o.include_unmapped;
            sc.edge_on = plan.P.edge_filter_on;
            sc.include = plan.inc;
            sc.defer_free = &sample_garbage;
            mkp_params PS = plan.P;
            PS.max_depth = 0;           // the sampler looks at reads, not at pileup columns
            check_mkp(dev.ctx, mkp_set_params(dev.ctx, &PS));
            if (!o.host_ingest && bam.have_index()) {
                sc.device_ready = &dev_ready_f;
                sampler_job.emplace([&]() { run_sampler(bam); }, set_dev_ready);
            }
        }
        // ---- focus positions of this rank's intervals (reference motif scan), beside the load and the sampler
        double iv_secs = 0;
        BackgroundJob iv_job([&]() {
            fill_interval_focus(plan.ivs, plan.my_i0, plan.my_i1, plan.iv_targets, plan.iv_owner, plan.combine_strands, plan.have_motifs ? &plan.mc : nullptr, plan.inc, std::max(1, o.threads / 2));
            iv_secs = secs_between(t_iv0, clk::now());
            trace("interval focus filled (background)");
        });
        std::optional<BamReader> host_bam;
        BamReader& reads = load_reads(o, plan, sharded, bam, &host_bam);
        set_dev_ready();
        const auto t_load = clk::now();
        trace("device load done");
        if (trace_clock().on) fprintf(stderr, "[mkh r%d]             ingest: h2d %.1f ms, inflate %.1f ms, record walk %.1f ms, total %.1f ms\n", coll.rank, reads.ingest_ms[0], reads.ingest_ms[1], reads.ingest_ms[2], reads.ingest_ms[3]);
        uint64_t any_mapped = 0;
        for (auto& t : plan.targets) if (plan.region || !plan.inc || plan.inc->has_contig(t.tid)) any_mapped += reads.stats.n_mapped[t.tid];
        if (!any_mapped) throw std::runtime_error("did not find any mapped reads, perform alignment first or use modkit extract and/or modkit summary to inspect unaligned modBAMs");
        PileupWriter out(o, plan.to_dir, coll);

        // thresholds (subcommand.rs:615-638, command_utils.rs:49-134)
        parse_mod_thresholds(o.mod_thresholds, &plan.P);
        parse_filter_thresholds(o.filter_thresholds, &plan.P);
        SampleResult sample;
        if (estimate) {
            if (!sampler_job) run_sampler(reads);
            sample_f.wait();
            trace("sampler result");
            sample = sample_f.get();
            estimated_thresholds(sample, o.percentile, "exact histogram quantile impossible; pass --filter-threshold", !o.quiet && coll.rank == 0, &plan.P);
        }
        check_mkp(dev.ctx, mkp_set_params(dev.ctx, &plan.P));
        const auto t_thr = clk::now();
        trace("thresholds done");

        iv_job.join();
        RunSummary S;
        S.fetch_s = sample.fetch_s;
        std::vector<RefInterval>& ivs = plan.ivs;
        if (sharded) { ivs.erase(ivs.begin() + (ptrdiff_t)plan.my_i1, ivs.end()); ivs.erase(ivs.begin(), ivs.begin() + (ptrdiff_t)plan.my_i0); }
        for (auto& iv : ivs) S.positions += iv.end - iv.start;

        // ---- two stages: a device thread selects the reads of chunk after chunk, slices them on the GPU, runs the pass and takes
        // the rows; this thread turns finished chunks into text (strand combining, formatting: parallel over intervals) and
        // writes them in order. The device works on chunk k + 1 while chunk k is being formatted.
        ChunkQueue queue;
        BackgroundJob dev_job([&]() {
            auto close_queue = [&]() { trace("device stage done"); ChunkOut fin; fin.last = true; queue.push(std::move(fin)); };
            try { device_stage(dev.ctx, reads, o, plan, &queue, &S); }
            catch (...) { close_queue(); throw; }
            close_queue();
        }, [&]() { queue.leave(); });
        WorkerPool pool(std::max(1, o.threads));
        for (ChunkOut co = queue.pop(); !co.last; co = queue.pop()) {
            const auto tc = clk::now();
            S.rows += format_chunk(co, o, plan, reads.ref_names[ivs[co.i0].tid], pool, &out);
            queue.recycle(std::move(co.rows));
            S.write_s += secs_between(tc, clk::now());
        }
        trace("last chunk formatted");
        dev_job.join();
        out.finish(pool, &S);
        const auto t1 = clk::now();
        trace("output written");
        S.load_s = secs_between(t0, t_load); S.threshold_s = secs_between(t_load, t_thr); S.interval_s = iv_secs;   /* runs beside ingest + thresholds */ S.total_s = secs_between(t0, t1);
        for (int b = 0; b < 4; b++) { S.thresholds[b] = plan.P.base_threshold[b]; S.threshold_set[b] = plan.P.base_threshold_set[b]; }
        if (summary) *summary = S;
        if (!o.quiet && coll.rank == 0)
            fprintf(stderr, "> Done, processed %llu rows. positions=%llu reads=%llu chunks=%llu load=%.3fs thresholds=%.3fs intervals=%.3fs pack=%.3fs gpu=%.3fs (kernels %.3f ms) write=%.3fs total=%.3fs\n",
                    (unsigned long long)S.rows, (unsigned long long)S.positions, (unsigned long long)S.reads_packed, (unsigned long long)S.chunks,
                    S.load_s, S.threshold_s, S.interval_s, S.pack_s, S.gpu_s, S.kernel_ms, S.write_s, S.total_s);
        if (FILE* jf = o.stats_json.empty() ? nullptr : fopen(o.stats_json.c_str(), "w")) {
            fprintf(jf, "{\"positions\": %llu, \"rows\": %llu, \"reads\": %llu, \"chunks\": %llu, \"algorithmic_bytes\": %llu, \"load_s\": %.6f, \"thresholds_s\": %.6f, \"intervals_s\": %.6f, \"pack_s\": %.6f, \"gpu_s\": %.6f, \"kernel_ms\": %.6f, \"write_s\": %.6f, \"total_s\": %.6f, \"ingest\": \"%s\", \"ingest_h2d_ms\": %.3f, \"ingest_inflate_ms\": %.3f, \"ingest_walk_ms\": %.3f, \"sampler_fetch_s\": %.6f, \"slice_s\": %.6f, \"pass_s\": %.6f, \"rowcopy_s\": %.6f}\n",
                    (unsigned long long)S.positions, (unsigned long long)S.rows, (unsigned long long)S.reads_packed, (unsigned long long)S.chunks, (unsigned long long)S.algorithmic_bytes,
                    S.load_s, S.threshold_s, S.interval_s, S.pack_s, S.gpu_s, S.kernel_ms, S.write_s, S.total_s,
                    reads.on_device ? (reads.ranged() ? "device-ranged" : "device") : "host", reads.ingest_ms[0], reads.ingest_ms[1], reads.ingest_ms[2], S.fetch_s, S.slice_s, S.pass_s, S.rowcopy_s);
            fclose(jf);
        }
        if (trace_clock().on) {      // (development: where the release of the run's host objects goes)
            trace("stats written");
            std::vector<RefInterval>().swap(ivs); trace("intervals released");
            out.release_buffers(); std::vector<std::vector<mkp_row>>().swap(queue.spare_rows); trace("text + row buffers released");
            reads.release_host_tables(); trace("record tables released");
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
    // sample-probs -o DIR: the report as files (thresholds.tsv; with --hist also probabilities.tsv, counts.html, proportion.html)
    std::string out_dir, prefix;
    bool have_prefix = false, force = false, hist = false;
    std::vector<std::string> dna_colors, mod_colors;    // --dna-color / --mod-color values, two per occurrence
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

// the sampled reads of both commands: the reader (a file without index is read on the host), the filters, the schedule.
// `keep`: also return the sampled reads themselves
inline SampleResult sample_for_summary(const SampleOptions& o, mkp_ctx* ctx, bool keep, BamReader& bam, mkp_params* P, Region* region_out, bool* have_region,
                                       IncludeBed* include, bool* have_include) {
    bam.open_device_index(o.in_bam, ctx);
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
    parse_edge_filter(o.edge, o.invert_edge, P);
    P->force_allow_implicit = 1;     // the sampler takes implicit lists as they are (no InvalidImplicitMode check outside the pileup)
    if (mkp_set_params(ctx, P)) throw std::runtime_error(mkp_last_error(ctx));
    SamplerConfig sc = sampler_config(o.threads, o.interval_size, o.num_reads, o.have_frac, o.frac, o.no_sampling, "-n, -f 1.0 or --no-sampling");
    sc.region = *have_region ? region_out : nullptr;
    sc.include_unmapped = !(o.only_mapped || *have_include);
    sc.edge_on = P->edge_filter_on;
    sc.include = *have_include ? include : nullptr;
    sc.keep = keep;
    return sample_histogram(bam, ctx, sc);
}

inline int run_summary(const SampleOptions& o, std::string* text, std::string* error) {
    try {
        DeviceGuard dev{open_device(o.device)};
        if (o.percentile > 1.0f) throw std::runtime_error("filter percentile must be <= 1.0");
        BamReader bam;
        mkp_params P;
        Region region; bool have_region = false;
        IncludeBed include; bool have_include = false;
        SampleResult sample = sample_for_summary(o, dev.ctx, true, bam, &P, &region, &have_region, &include, &have_include);
        ModSummaryOut S;
        // thresholds (src/commands.rs:1086-1098, 1147-1160)
        parse_mod_thresholds(o.mod_thresholds, &P);
        parse_filter_thresholds(o.filter_thresholds, &P);
        if (o.filter_thresholds.empty() && !o.no_filtering) estimated_thresholds(sample, o.percentile, "exact quantiles impossible", false, &P);
        for (int b = 0; b < 4; b++) { S.thresholds[b] = P.base_threshold[b]; S.threshold_set[b] = P.base_threshold_set[b]; }
        if (mkp_set_params(dev.ctx, &P)) throw std::runtime_error(mkp_last_error(dev.ctx));
        // ---- second pass over the sampled reads: counts per (base, state, pass / fail)
        const int incl_unal = !(o.only_mapped || have_include) ? 1 : 0;
        for (auto& kc : sample.keep) {
            upload_sampled(bam, dev.ctx, kc.pc, kc.tid, have_include ? &include : nullptr);
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

// ---- `sample-probs -o DIR [--hist]` (src/writers.rs:692-993, src/read_ids_to_base_mod_probs.rs:104-187) ----------------------
// Counts of the arg-max values per (canonical base, state) and prob_to_qual bin. Key: (base, 0 = canonical | state_order_key),
// so the map iterates in the reference's (DnaBase, BaseState) order: Canonical first, then Code(char) before ChEbi(u32).
using ModHistogram = std::map<std::pair<int, uint64_t>, std::array<uint64_t, 256>>;

// adds one mkp_sample_mod_histogram result (hist u64[4][33][256], states u64[32]) to H
inline void add_mod_histogram(const uint64_t* hist, const uint64_t* states, ModHistogram* H) {
    for (int b = 0; b < 4; b++) for (int s = 0; s < 33; s++) {
        const uint64_t* h = hist + (b * 33 + s) * 256;
        if (std::all_of(h, h + 256, [](uint64_t v) { return v == 0; })) continue;
        std::array<uint64_t, 256>& dst = (*H)[{b, s == 0 ? 0 : state_order_key((uint32_t)states[s - 1])}];
        for (int q = 0; q < 256; q++) dst[q] += h[q];
    }
}

// probabilities.tsv (ProbHistogram::get_artifacts, src/writers.rs:837-945, csv writer with a tab delimiter): non-zero bins in
// ascending order; frac and percentile_rank in f32, the rank over an f32 running sum of the counts, as the reference folds it
inline std::string probabilities_tsv(const ModHistogram& H) {
    std::string out = "code\tprimary_base\trange_start\trange_end\tcount\tfrac\tpercentile_rank\n";
    for (const auto& kv : H) {
        const std::array<uint64_t, 256>& c = kv.second;
        uint64_t sum = 0;
        for (uint64_t n : c) sum += n;
        const float total = (float)sum;
        const std::string head = (kv.first.second == 0 ? std::string("-") : state_label_of_key(kv.first.second)) + "\t" + "ACGT"[kv.first.first] + "\t";
        float cum = 0.f;
        for (int q = 0; q < 256; q++) {
            if (!c[q]) continue;
            const float n = (float)c[q];
            cum = cum + n;
            const float rank = ((cum - 0.5f * n) / total) * 100.0f;
            out += head + f32_display((float)q / 256.0f) + "\t" + f32_display((float)(q + 1) / 256.0f) + "\t" + std::to_string(c[q]) + "\t" +
                   f32_display(n / total) + "\t" + f32_display(rank) + "\n";
        }
    }
    return out;
}

// JSON string literal, with '<' escaped so that a label or colour cannot close the page's <script>
inline std::string json_str(const std::string& s) {
    std::string o = "\"";
    for (unsigned char ch : s) {
        if (ch == '"' || ch == '\\') { o += '\\'; o += (char)ch; }
        else if (ch < 0x20 || ch == '<') { char b[8]; snprintf(b, sizeof b, "\\u%04x", ch); o += b; }
        else o += (char)ch;
    }
    return o + "\"";
}

// series colours: --dna-color / --mod-color, then the reference's defaults (mod_base_code.rs:94-102); any other label gets a
// fixed colour derived from the label (FNV-1a), where the reference seeds the random_color crate with it
struct HistColors { std::map<int, std::string> dna; std::map<uint32_t, std::string> mod; };

inline HistColors parse_hist_colors(const SampleOptions& o) {
    HistColors hc;
    for (size_t i = 0; i + 1 < o.dna_colors.size(); i += 2) {
        const std::string& b = o.dna_colors[i];
        if (b.size() != 1) throw std::runtime_error("DNA base should be a char, " + b);
        const char* f = strchr("ACGT", b[0]);
        if (!f || !b[0]) throw std::runtime_error("invalid DNA base, should be A, C, G, or T: " + b);
        hc.dna[(int)(f - "ACGT")] = o.dna_colors[i + 1];
    }
    for (size_t i = 0; i + 1 < o.mod_colors.size(); i += 2) {
        uint32_t c;
        if (!parse_code(o.mod_colors[i], &c)) throw std::runtime_error("failed to parse mod code " + o.mod_colors[i]);
        hc.mod[c] = o.mod_colors[i + 1];
    }
    return hc;
}

inline std::string hist_series_color(const HistColors& hc, int base, uint64_t key, const std::string& label) {
    if (key == 0) {
        auto it = hc.dna.find(base);
        if (it != hc.dna.end()) return it->second;
        if (base == 1) return "#0000FF";
        if (base == 0) return "#009600";
    } else if (key < (1ull << 32)) {
        const uint32_t code = (uint32_t)(key - 1);
        auto it = hc.mod.find(code);
        if (it != hc.mod.end()) return it->second;
        if (code == 'm') return "#FF0000";
        if (code == 'h') return "#FF00FF";
        if (code == 'a') return "#0084A9";
    } else {
        auto it = hc.mod.find(0x80000000u | (uint32_t)(key - 1 - (1ull << 32)));
        if (it != hc.mod.end()) return it->second;
    }
    uint32_t h = 2166136261u;
    for (unsigned char ch : label) { h ^= ch; h *= 16777619u; }
    char b[8];
    snprintf(b, sizeof b, "#%06X", h & 0xffffffu);
    return b;
}

// counts.html / proportion.html: one ECharts bar chart (get_blank_chart / get_artifacts, src/writers.rs:799-945) whose option
// object is embedded as JSON, 800 x 800, ECharts loaded by <script src> as charming's HtmlRenderer does
inline std::string histogram_chart_html(const ModHistogram& H, const HistColors& hc, bool proportion) {
    std::vector<int> bins;
    for (int q = 0; q < 256; q++) for (const auto& kv : H) if (kv.second[q]) { bins.push_back(q); break; }
    std::string cats, series, colors;
    for (int q : bins) {
        char a[64], b[64];
        *put_pct2(a, (float)q / 256.0f * 100.0f) = 0;
        *put_pct2(b, (float)(q + 1) / 256.0f * 100.0f) = 0;
        cats += std::string(cats.empty() ? "" : ",") + json_str(std::string("[") + a + ", " + b + ")");
    }
    for (const auto& kv : H) {
        const int base = kv.first.first;
        const std::string label = std::string(1, "ACGT"[base]) + ":" + (kv.first.second == 0 ? std::string("-") : state_label_of_key(kv.first.second));
        int64_t tot = 0;
        for (int q : bins) tot += (int64_t)kv.second[q];
        std::string data;
        for (int q : bins) {
            const int64_t n = (int64_t)kv.second[q];
            data += std::string(data.empty() ? "" : ",") + (proportion ? f32_display((float)n / (float)tot) : std::to_string(n));
        }
        series += std::string(series.empty() ? "" : ",") + "{\"type\":\"bar\",\"name\":" + json_str(label) + ",\"data\":[" + data + "]}";
        colors += std::string(colors.empty() ? "" : ",") + json_str(hist_series_color(hc, base, kv.first.second, label));
    }
    const char* title = proportion ? "Proportion" : "Counts";
    const std::string option = std::string("{\"title\":{\"text\":\"") + title + "\"},\"tooltip\":{\"trigger\":\"axis\",\"axisPointer\":{\"type\":\"shadow\"}},"
        "\"legend\":{},\"toolbox\":{\"feature\":{\"dataZoom\":{\"yAxisIndex\":\"none\"},\"restore\":{},\"saveAsImage\":{}}},"
        "\"dataZoom\":[{\"type\":\"slider\"}],\"xAxis\":{\"type\":\"category\",\"name\":\"bin\",\"data\":[" + cats + "]},"
        "\"yAxis\":{\"type\":\"value\",\"name\":\"" + (proportion ? "proportion" : "counts") + "\"},\"color\":[" + colors + "],\"series\":[" + series + "]}";
    return std::string("<!DOCTYPE html>\n<html lang=\"en\">\n<head>\n  <meta charset=\"utf-8\">\n  <title>") + (proportion ? "Proportions" : "Counts") +
           "</title>\n  <script src=\"https://cdn.jsdelivr.net/npm/echarts@5.4.2/dist/echarts.min.js\"></script>\n</head>\n<body>\n"
           "  <div id=\"chart\" style=\"width:800px;height:800px;\"></div>\n  <script type=\"text/javascript\">\n"
           "    var option = " + option + ";\n"
           "    echarts.init(document.getElementById(\"chart\")).setOption(option);\n  </script>\n</body>\n</html>\n";
}

// the files of `-o DIR` (SampledProbs::get_*_filename*, src/writers.rs:700-725)
inline std::vector<std::string> sample_output_files(const SampleOptions& o) {
    const std::string p = o.have_prefix ? o.prefix + "_" : "";
    std::vector<std::string> v{p + "thresholds.tsv"};
    if (o.hist) for (const char* n : {"probabilities.tsv", "counts.html", "proportion.html"}) v.push_back(p + n);
    return v;
}

// SampledProbs::check_files (src/writers.rs:731-763) and the colour arguments: before any device work or sampling
inline HistColors check_sample_outputs(const SampleOptions& o) {
    if (o.out_dir.empty()) return HistColors();
    for (const std::string& n : sample_output_files(o)) {
        const std::filesystem::path fp = std::filesystem::path(o.out_dir) / n;
        if (std::filesystem::exists(fp) && !o.force) throw std::runtime_error("refusing to overwrite \"" + fp.string() + "\"");
    }
    return parse_hist_colors(o);
}

inline void write_text_file(const std::filesystem::path& fp, const std::string& text) {
    FILE* f = fopen(fp.c_str(), "wb");
    if (!f) throw std::runtime_error("failed to create " + fp.string());
    const bool ok = fwrite(text.data(), 1, text.size(), f) == text.size();
    if (fclose(f) != 0 || !ok) throw std::runtime_error("failed to write " + fp.string());
}

// `modkit sample-probs`: percentiles of the arg-max probabilities per canonical base (thresholds table, src/writers.rs:779-790);
// with -o the table goes to DIR/thresholds.tsv and nothing to stdout, with --hist also the per-state histograms
inline int run_sample_probs(const SampleOptions& o, std::string* text, std::string* error) {
    try {
        const HistColors colors = check_sample_outputs(o);
        DeviceGuard dev{open_device(o.device)};
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
        SampleResult sample = sample_for_summary(o, dev.ctx, o.hist, bam, &P, &region, &have_region, &include, &have_include);
        require_exact(sample.inexact, "exact quantiles impossible");
        const std::vector<uint64_t>& hist = sample.hist;
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
        if (o.out_dir.empty()) return 0;
        // ---- -o DIR: the histograms are a second device pass over the sampled reads (get_per_mod_histograms)
        ModHistogram H;
        if (o.hist) {
            const int incl_unal = !(o.only_mapped || have_include) ? 1 : 0;
            for (auto& kc : sample.keep) {
                upload_sampled(bam, dev.ctx, kc.pc, kc.tid, have_include ? &include : nullptr);
                std::vector<uint64_t> hist(4 * 33 * 256, 0), states(32, ~0ull);
                if (mkp_sample_mod_histogram(dev.ctx, incl_unal, kc.take.data(), hist.data(), states.data())) throw std::runtime_error(mkp_last_error(dev.ctx));
                add_mod_histogram(hist.data(), states.data(), &H);
            }
        }
        const std::filesystem::path dir(o.out_dir);
        std::filesystem::create_directories(dir);
        const std::vector<std::string> files = sample_output_files(o);
        write_text_file(dir / files[0], *text);
        if (o.hist) {
            write_text_file(dir / files[1], probabilities_tsv(H));
            write_text_file(dir / files[2], histogram_chart_html(H, colors, false));
            write_text_file(dir / files[3], histogram_chart_html(H, colors, true));
        }
        text->clear();
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
            else if (!summary && (a == "-o" || a == "--out-dir")) o->out_dir = val();
            else if (!summary && a == "--prefix") { o->prefix = val(); o->have_prefix = true; }
            else if (!summary && a == "--force") o->force = true;
            else if (!summary && a == "--hist") o->hist = true;
            else if (!summary && (a == "--dna-color" || a == "--mod-color")) {
                std::vector<std::string>& v = a == "--dna-color" ? o->dna_colors : o->mod_colors;
                if (i + 2 >= argc) throw std::runtime_error("invalid number of arguments for '" + a + "': 2 values are required");
                v.push_back(argv[++i]);
                v.push_back(argv[++i]);
            }
            else if (a.size() > 1 && a[0] == '-') { *err = "unexpected argument '" + a + "' found"; return false; }
            else pos.push_back(a);
        } catch (const std::exception& e) { *err = e.what(); return false; }
    }
    // the `requires` rules of the output flags (src/commands.rs:573-622); --out is this build's report file, -o the reference's directory
    const char* needs_out_dir = o->have_prefix ? "--prefix" : o->force ? "--force" : o->hist ? "--hist" : nullptr;
    if (needs_out_dir && o->out_dir.empty()) { *err = std::string("the following required arguments were not provided: --out-dir <OUT_DIR> (required by ") + needs_out_dir + ")"; return false; }
    if (!o->hist && !(o->dna_colors.empty() && o->mod_colors.empty())) { *err = "the following required arguments were not provided: --hist (required by --dna-color / --mod-color)"; return false; }
    if (!o->out_dir.empty() && !out_path->empty()) { *err = "the argument '--out <FILE>' cannot be used with '--out-dir <OUT_DIR>'"; return false; }
    if (pos.size() != 1) { *err = "the following required arguments were not provided: <IN_BAM>"; return false; }
    o->in_bam = pos[0];
    return true;
}

}  // namespace mkh
