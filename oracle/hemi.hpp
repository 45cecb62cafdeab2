// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// `modkit_oracle_hemi pileup-hemi [flags] <in.bam> [-o out.bed]` (hemi_main.cpp): CPU restatement of `modkit pileup-hemi` (reference v0.4.4):
//   flags, DuplexModBamPileup::run          src/pileup/subcommand.rs:825-1514
//   process_region_duplex, decode           src/pileup/duplex.rs
//   DuplexReadCache::get_duplex_mod_call    src/read_cache.rs:368-468
//   DuplexModCall, DuplexModCodeRepr        src/mod_bam.rs:1674-1830
//   row format                              src/writers.rs:185-255
//   partner position                        src/find_motifs/motif_bed.rs:119-141
// The read set per interval, the decode of a read and the threshold calls are the pileup's (pileup.hpp). Per + strand motif
// position p and admitted read: a deletion counts n_delete; an ACGT SEQ base pairs the read's call on the + strand at p with
// its call on the - strand at p + (reverse offset - forward offset). A read whose decode fails counts once as NoCall, at the
// first motif position of the interval where it has an ACGT base (the read cache checks its skip set before the first decode
// and then ignores the read).
#pragma once
#include <atomic>
#include <condition_variable>
#include <stdexcept>
#include <memory>
#include <thread>
#include <unordered_map>

#include "driver.hpp"

namespace orc {

constexpr ModCode HEMI_CANONICAL = 0;   // DuplexModCodeRepr::Canonical, '-': sorts before every mod code

struct HemiRow {
    uint32_t pos;
    int base;           // primary base: the read's SEQ base at pos
    ModCode code_pos, code_neg;
    uint32_t count, n_other, n_canon, n_delete, n_fail, n_diff, n_nocall;
};

// A read's decode does not depend on the interval: it is done once per record and shared by the intervals (small -i would
// otherwise decode every read once per interval it overlaps).
struct HemiDecodeCache {
    std::mutex mu;
    std::unordered_map<const BamRecord*, std::unique_ptr<ReadCalls>> by_rec;
    const ReadCalls& get(const BamRecord& r, const PileupParams& P, StateTable& st) {
        {
            std::lock_guard<std::mutex> g(mu);
            auto it = by_rec.find(&r);
            if (it != by_rec.end()) return *it->second;
        }
        std::unique_ptr<ReadCalls> rc(new ReadCalls());
        decode_read_for_pileup(r, P, st, rc.get());
        std::lock_guard<std::mutex> g(mu);
        std::unique_ptr<ReadCalls>& slot = by_rec[&r];
        if (!slot) slot = std::move(rc);
        return *slot;
    }
};

inline void process_interval_hemi(const BamFile& bam, const Interval& iv, const PileupParams& P, StateTable& st, int partner_off,
                                  HemiDecodeCache& cache, std::vector<HemiRow>* rows_out) {
    const uint32_t start = iv.start, end = iv.end;
    if (end <= start || iv.focus.pos_ids.empty()) return;
    std::vector<const BamRecord*> recs;
    {
        std::vector<const BamRecord*> pushed;
        bam.fetch(iv.tid, start, end, [&](const BamRecord& r) { if (!(r.flag() & (0x4 | 0x100 | 0x200 | 0x400))) pushed.push_back(&r); });
        plp_maxcnt_filter(&pushed, P.max_depth);
        for (const BamRecord* r : pushed) if (admitted_for_pileup(*r)) recs.push_back(r);
    }
    if (recs.empty()) return;
    // focus: the + strand motif positions (positive_motifs of FocusPositions::MotifCombineStrands)
    std::vector<uint32_t> focus;
    for (auto& kv : iv.focus.pos_ids) focus.push_back(kv.first);
    std::vector<int32_t> fidx(end - start, -1);
    for (size_t i = 0; i < focus.size(); i++) fidx[focus[i] - start] = (int32_t)i;
    struct PerBase { std::map<std::pair<ModCode, ModCode>, uint32_t> pat; uint32_t filtered = 0, nocall = 0; };
    struct PerPos { uint32_t n_delete = 0; PerBase b[4]; };
    std::vector<PerPos> acc(focus.size());

    std::vector<int64_t> r2q;
    for (const BamRecord* rp : recs) {
        const BamRecord& r = *rp;
        const ReadCalls& rc = cache.get(r, P, st);
        const bool rev = r.is_reverse();
        const int L = r.l_seq();
        // reference position -> query position of the M/=/X bases of the read
        int64_t ref_len = 0;
        for (int ci = 0; ci < r.n_cigar(); ci++) { const uint32_t c = r.cigar_op(ci); const int op = c & 0xf; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ref_len += c >> 4; }
        r2q.assign((size_t)ref_len + 1, -1);
        {
            int64_t x = 0; int q = 0;
            for (int ci = 0; ci < r.n_cigar(); ci++) {
                const uint32_t c = r.cigar_op(ci);
                const int op = c & 0xf, len = (int)(c >> 4);
                if (op == 0 || op == 7 || op == 8) { for (int k = 0; k < len; k++, x++, q++) if (q < L) r2q[x] = q; }
                else if (op == 1 || op == 4) q += len;
                else if (op == 2 || op == 3) x += len;
            }
        }
        const int64_t r0 = r.pos();
        auto query_at = [&](int64_t ref) -> int { const int64_t x = ref - r0; return (x < 0 || x >= ref_len) ? -1 : (int)r2q[(size_t)x]; };
        const std::vector<uint16_t>& pos_tab = rev ? rc.minus : rc.plus;   // calls on the + reference strand
        const std::vector<uint16_t>& neg_tab = rev ? rc.plus : rc.minus;
        bool noted = false;   // skipped read: counted once
        int64_t ref = r0;
        int q = 0;
        for (int ci = 0; ci < r.n_cigar(); ci++) {
            const uint32_t c = r.cigar_op(ci);
            const int op = c & 0xf, len = (int)(c >> 4);
            if (op == 0 || op == 7 || op == 8) {
                for (int k = 0; k < len; k++, q++, ref++) {
                    if (ref < start || ref >= end || q >= L) continue;
                    const int32_t fi = fidx[ref - start];
                    if (fi < 0) continue;
                    const int b = base_idx(r.base_at(q));
                    if (b < 0) continue;
                    PerBase& B = acc[fi].b[b];
                    if (rc.skipped) { if (!noted) { B.nocall++; noted = true; } continue; }
                    const int64_t partner = ref + partner_off;
                    uint16_t vp = pos_tab[q], vn = 0;
                    if (partner >= 0) {
                        // the - strand call is looked up in the table of the complementary base (read_cache.rs:434-454)
                        const int qn = query_at(partner);
                        if (qn >= 0 && base_idx(r.base_at(qn)) == comp_idx(b)) vn = neg_tab[qn];
                    }
                    if (!vp || !vn) { B.nocall++; continue; }
                    if (vp == 1 || vn == 1) { B.filtered++; continue; }
                    ModCode cp = vp == 2 ? HEMI_CANONICAL : st.get(vp - 3).second;
                    ModCode cn = vn == 2 ? HEMI_CANONICAL : st.get(vn - 3).second;
                    if (P.numeric == COMBINE && !(cp == HEMI_CANONICAL && cn == HEMI_CANONICAL)) {   // into_combined
                        if (cp != HEMI_CANONICAL) cp = (ModCode)(uint8_t)BASES[b];
                        if (cn != HEMI_CANONICAL) cn = (ModCode)(uint8_t)BASES[b];
                    }
                    B.pat[{cp, cn}]++;
                }
            } else if (op == 1 || op == 4) {
                q += len;
            } else if (op == 2) {
                for (int k = 0; k < len; k++, ref++) {
                    if (ref < start || ref >= end) continue;
                    const int32_t fi = fidx[ref - start];
                    if (fi >= 0) acc[fi].n_delete++;
                }
            } else if (op == 3) {
                ref += len;
            }
        }
    }
    // DuplexFeatureVector::decode, rows by position, base, pattern
    for (size_t i = 0; i < focus.size(); i++) {
        const PerPos& A = acc[i];
        uint32_t pat_total[4] = {0, 0, 0, 0};
        for (int b = 0; b < 4; b++) for (auto& kv : A.b[b].pat) pat_total[b] += kv.second;
        const uint32_t all = pat_total[0] + pat_total[1] + pat_total[2] + pat_total[3];
        for (int b = 0; b < 4; b++) {
            const PerBase& B = A.b[b];
            auto cc = B.pat.find({HEMI_CANONICAL, HEMI_CANONICAL});
            const uint32_t n_canon = cc == B.pat.end() ? 0 : cc->second;
            for (auto& kv : B.pat)
                rows_out->push_back(HemiRow{focus[i], b, kv.first.first, kv.first.second, kv.second, pat_total[b] - kv.second, n_canon,
                                            A.n_delete, B.filtered, all - pat_total[b], B.nocall});
        }
    }
}

inline void format_hemi_row(const HemiRow& R, const std::string& chrom, bool mixed_delim, std::string* out) {
    const char sp = mixed_delim ? ' ' : '\t';
    auto side = [](ModCode c) { return c == HEMI_CANONICAL ? std::string("-") : code_to_string(c); };
    const std::string name = side(R.code_pos) + "," + side(R.code_neg) + "," + std::string(1, BASES[R.base]);
    const uint32_t cov = R.count + R.n_other;
    float frac = (float)R.count / (float)cov;
    volatile float pct = frac * 100.0f;
    char buf[512];
    int n = snprintf(buf, sizeof buf, "%s\t%u\t%u\t%s\t%u\t.\t%u\t%u\t255,0,0\t%u%c%.2f%c%u%c%u%c%u%c%u%c%u%c%u%c%u\n",
                     chrom.c_str(), R.pos, R.pos + 1, name.c_str(), cov, R.pos, R.pos + 1,
                     cov, sp, (double)pct, sp, R.count, sp, R.n_canon, sp, R.n_other, sp, R.n_delete, sp,
                     R.n_fail, sp, R.n_diff, sp, R.n_nocall);
    out->append(buf, (size_t)n);
}

inline int hemi_main(int argc, char** argv) {
    auto bail = [](const std::string& m) { throw std::runtime_error(m); };
    std::vector<std::string> pos;
    int threads = 4;
    uint32_t interval_size = 100000, sampling_interval_size = 1000000;
    size_t num_reads = 10042;
    bool have_frac = false; double frac = 0;
    bool no_filtering = false, include_unmapped = false, force_allow = false, cpg = false, mask = false;
    bool combine_mods = false, mixed = false, invert_edge = false;
    uint32_t max_depth = 8000;
    float percentile = 0.1f;
    std::vector<std::string> filter_thresholds, mod_thresholds, motif_parts;
    std::string region_s, sample_region_s, ignore_s, ref_fp, edge_s, include_bed, out_fp;
    for (int i = 2; i < argc; i++) {
        std::string a = argv[i];
        auto val = [&]() -> std::string { if (i + 1 >= argc) bail("missing value for " + a); return argv[++i]; };
        if (a == "-t" || a == "--threads") threads = std::stoi(val());
        else if (a == "-o" || a == "--out-bed") out_fp = val();
        else if (a == "-i" || a == "--interval-size") interval_size = (uint32_t)std::stoul(val());
        else if (a == "--region") region_s = val();
        else if (a == "--sample-region") sample_region_s = val();
        else if (a == "--sampling-interval-size") sampling_interval_size = (uint32_t)std::stoul(val());
        else if (a == "-n" || a == "--num-reads") num_reads = std::stoul(val());
        else if (a == "-f" || a == "--sampling-frac") { have_frac = true; frac = std::stod(val()); }
        else if (a == "--max-depth") max_depth = (uint32_t)std::stoul(val());
        else if (a == "--seed" || a == "--queue-size" || a == "--chunk-size" || a == "--log-filepath" || a == "--log") val();
        else if (a == "--no-filtering") no_filtering = true;
        else if (a == "-p" || a == "--filter-percentile") percentile = std::stof(val());
        else if (a == "--filter-threshold" || a == "--pass_threshold") filter_thresholds.push_back(val());
        else if (a == "--mod-thresholds" || a == "--mod-threshold") mod_thresholds.push_back(val());
        else if (a == "--include-unmapped") include_unmapped = true;
        else if (a == "--ignore") ignore_s = val();
        else if (a == "--force-allow-implicit") force_allow = true;
        else if (a == "--motif") { if (!motif_parts.empty()) bail("the argument '--motif' cannot be used multiple times"); motif_parts.push_back(val()); motif_parts.push_back(val()); }
        else if (a == "--cpg") cpg = true;
        else if (a == "-r" || a == "--ref" || a == "--reference") ref_fp = val();
        else if (a == "-k" || a == "--mask") mask = true;
        else if (a == "--combine-mods") combine_mods = true;
        else if (a == "--edge-filter") edge_s = val();
        else if (a == "--invert-edge-filter") invert_edge = true;
        else if (a == "--only-tabs" || a == "--suppress-progress") {}
        else if (a == "--mixed-delim" || a == "--mixed-delimiters") mixed = true;
        else if (a == "--include-bed" || a == "--include-positions") include_bed = val();
        else if (a.size() > 1 && a[0] == '-') bail("unexpected argument '" + a + "' found");
        else pos.push_back(a);
    }
    if (pos.size() != 1) bail("usage: modkit_oracle_hemi pileup-hemi [flags] <in.bam> -r <ref.fa> [-o out.bed]");
    if (ref_fp.empty()) bail("the following required arguments were not provided: --ref <REFERENCE_FASTA>");
    if (cpg && !motif_parts.empty()) bail("the argument '--cpg' cannot be used with '--motif <MOTIF> <MOTIF>'");
    if (combine_mods && !ignore_s.empty()) bail("the argument '--combine-mods' cannot be used with '--ignore <IGNORE>'");
    if (invert_edge && edge_s.empty()) bail("--invert-edge-filter requires --edge-filter");
    BamFile bam;
    bam.load(pos[0], threads);
    Region region, sample_region;
    const Region* rp = nullptr; const Region* srp = nullptr;
    if (!region_s.empty()) { region = parse_region(region_s, bam); rp = &region; }
    if (!sample_region_s.empty()) { sample_region = parse_region(sample_region_s, bam); srp = &sample_region; }
    std::vector<RefRecord> targets = get_targets(bam, rp);
    PositionFilter pfilter;
    const PositionFilter* pf = nullptr;
    if (!include_bed.empty()) {
        std::map<std::string, uint32_t> c2t;
        for (auto& t : targets) c2t[t.name] = t.tid;
        pfilter.load(include_bed, c2t);
        pf = &pfilter;
    }
    {
        uint64_t mapped = 0;
        for (auto& t : targets) if (rp || !pf || pf->has_contig(t.tid)) mapped += bam.n_mapped[t.tid];
        if (!mapped) bail("did not find any mapped reads, perform alignment first or use modkit extract and/or modkit summary to inspect unaligned modBAMs");
    }
    if (percentile > 1.0f) bail("filter percentile must be <= 1.0");
    PileupParams P;
    P.max_depth = max_depth;
    P.force_allow_implicit = force_allow;
    P.combine_strands = true;
    bool threshold_collapse = false;
    if (combine_mods) {
        P.numeric = COMBINE;
    } else if (!ignore_s.empty()) {
        ModCode c;
        if (!parse_mod_code(ignore_s, &c)) bail("failed to parse mod code " + ignore_s);
        P.numeric = COLLAPSE; P.collapse_code = c; threshold_collapse = true;
    }
    if (!edge_s.empty()) {
        P.edge.on = true; P.edge.inverted = invert_edge;
        auto c = edge_s.find(',');
        if (c == std::string::npos) P.edge.start = P.edge.end = std::stoul(edge_s);
        else { P.edge.start = std::stoul(edge_s.substr(0, c)); P.edge.end = std::stoul(edge_s.substr(c + 1)); }
    }
    Motif motif;
    if (cpg) motif = Motif::parse("CG", 0);
    else if (motif_parts.empty()) bail("either --cpg or a --motif must be provided for pileup-hemi");
    else motif = Motif::parse(motif_parts[0], std::stoi(motif_parts[1]));
    if (!motif.palindrome) bail("motif must be palindromic for pileup-hemi");
    const int partner_off = motif.rev_off - motif.fwd_off;
    MotifLookup lookup;
    lookup.fa.open(ref_fp);
    lookup.motifs = {motif};
    lookup.mask = mask;
    lookup.pf = pf;
    lookup.longest = motif.length;
    FILE* out = out_fp.empty() ? stdout : fopen(out_fp.c_str(), "w");
    if (!out) bail("failed to make output file");
    for (auto& raw : mod_thresholds) {
        auto c = raw.find(':');
        ModCode code;
        if (c == std::string::npos || !parse_mod_code(raw.substr(0, c), &code)) bail("illegal per-mod threshold " + raw);
        P.caller.mod_thr.push_back({code, std::stof(raw.substr(c + 1))});
    }
    if (!filter_thresholds.empty()) {
        for (auto& raw : filter_thresholds) {
            auto c = raw.find(':');
            if (c == std::string::npos) { P.caller.default_thr = std::stof(raw); continue; }
            int b = base_idx(raw[0]);
            if (b < 0) bail("failed to parse base " + raw);
            P.caller.base_set[b] = true;
            P.caller.base_thr[b] = std::stof(raw.substr(c + 1));
        }
    } else if (!no_filtering) {
        SampleOptions so;
        so.threads = threads;
        so.sampling_interval_size = sampling_interval_size;
        if (have_frac) { if (frac != 1.0) bail("oracle supports only -f 1.0 (Rust StdRng sampling is not reproducible)"); so.frac_all = true; }
        so.num_reads = num_reads;
        so.region = srp ? srp : rp;
        so.include_unmapped = include_unmapped;
        so.collapse = threshold_collapse;
        so.collapse_code = P.collapse_code;
        so.edge = P.edge;
        so.pf = pf;
        estimate_thresholds(bam, so, percentile, &P.caller);
        for (int b = 0; b < 4; b++) if (P.caller.base_set[b]) fprintf(stderr, "> Using filter threshold %.9g for %c.\n", P.caller.base_thr[b], BASES[b]);
    }
    if (pf) targets = optimize_reference_records(*pf, targets, interval_size);
    std::vector<Interval> ivs = make_intervals(targets, interval_size, true, &lookup, nullptr, pf);

    StateTable st;
    HemiDecodeCache cache;
    std::vector<std::string> results(ivs.size());
    std::vector<char> done(ivs.size(), 0);
    std::atomic<size_t> next{0};
    std::mutex mu;
    std::condition_variable cv;
    auto worker = [&]() {
        while (true) {
            const size_t i = next.fetch_add(1);
            if (i >= ivs.size()) break;
            std::vector<HemiRow> rows;
            process_interval_hemi(bam, ivs[i], P, st, partner_off, cache, &rows);
            std::string text;
            for (auto& R : rows) format_hemi_row(R, bam.ref_names[ivs[i].tid], mixed, &text);
            std::lock_guard<std::mutex> g(mu);
            results[i].swap(text);
            done[i] = 1;
            cv.notify_all();
        }
    };
    std::vector<std::thread> pool;
    for (int t = 0; t < std::max(1, threads); t++) pool.emplace_back(worker);
    for (size_t i = 0; i < ivs.size(); i++) {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return done[i] != 0; });
        std::string text;
        text.swap(results[i]);
        lk.unlock();
        fwrite(text.data(), 1, text.size(), out);
    }
    for (auto& t : pool) t.join();
    if (out != stdout) fclose(out); else fflush(out);
    return 0;
}

}  // namespace orc
