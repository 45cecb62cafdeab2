// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// `modkit_oracle pileup [flags] <in.bam> <out.bed>`: CPU restatement of `modkit pileup`
// (reference v0.4.4, src/pileup/subcommand.rs:381-817) used (a) as the parity checker in tests/
// and (b) as the `cpu_baseline` / `--impl reference` arm of bench.py (the Rust reference cannot be
// built in this image: no cargo/rustc). Parallelised like the reference: one worker per genomic
// interval (src/pileup/mod.rs:696-715), results written in feeder order.
#include <filesystem>
#include <atomic>
#include <chrono>
#include <condition_variable>

#include "driver.hpp"

using namespace orc;

static void die(const std::string& m) { fprintf(stderr, "> Error! %s\n", m.c_str()); exit(1); }

// Known-answer helpers for tests/ (mirror the reference's in-crate unit tests):
//   decode SEQ MM ML_CSV [ignore_code]  -> one line per table entry: strand base pos inferred code:prob[,code:prob] canonical_prob
//   call BASE code:p[,code:p] default [B:thr ...] [mod=c:thr ...] -> filtered | canonical P | modified CODE P
//   percentile Q v0,v1,...
//   endpos IN.BAM -> one line per record in file order: name pos endpos n_cigar (the CIGAR accessors, CG:B,I applied)
static int kat_main(int argc, char** argv) {
    std::string cmd = argv[1];
    if (cmd == "endpos") {
        if (argc < 3) return 2;
        BamFile bam;
        bam.load(argv[2]);
        for (const BamRecord& r : bam.records) printf("%s %d %lld %u\n", r.name(), r.pos(), (long long)r.endpos(), r.n_cigar());
        return 0;
    }
    if (cmd == "decode") {
        if (argc < 5) return 2;
        std::string seq = argv[2], mm = argv[3], mlcsv = argv[4];
        std::vector<uint8_t> ml;
        for (size_t i = 0; i < mlcsv.size();) { size_t j = mlcsv.find(',', i); if (j == std::string::npos) j = mlcsv.size(); if (j > i) ml.push_back((uint8_t)std::stoi(mlcsv.substr(i, j - i))); i = j + 1; }
        std::vector<MmList> lists;
        if (!parse_mm(mm.data(), mm.size(), &lists)) { printf("ERROR parse\n"); return 0; }
        ModBaseInfo info;
        if (!build_mod_base_info(lists, ml.data(), ml.size(), seq, &info)) { printf("ERROR build\n"); return 0; }
        for (int st = 0; st < 2; st++) for (int b = 0; b < 4; b++) {
            if (!info.present[st][b]) continue;
            for (auto& kv : info.tab[st][b].pos) {
                BaseModProbs bmp = kv.second;
                if (argc > 5) { ModCode c; parse_mod_code(argv[5], &c); bmp = redistribute(bmp, c); }
                printf("%c %c %u %d ", st ? '-' : '+', BASES[b], kv.first, bmp.inferred ? 1 : 0);
                bool first = true;
                bmp.probs.for_each([&](ModCode c, float p) { printf("%s%s:%.9g", first ? "" : ",", code_to_string(c).c_str(), p); first = false; });
                printf(" %.9g mode=%d\n", bmp.canonical_prob(), info.tab[st][b].mode);
            }
        }
        return 0;
    }
    if (cmd == "call") {
        if (argc < 5) return 2;
        int b = base_idx(argv[2][0]);
        BaseModProbs bmp;
        std::string ps = argv[3];
        for (size_t i = 0; i < ps.size();) {
            size_t j = ps.find(',', i); if (j == std::string::npos) j = ps.size();
            std::string kv = ps.substr(i, j - i); size_t c = kv.find(':');
            ModCode code; parse_mod_code(kv.substr(0, c), &code);
            *bmp.probs.entry_or_insert(code, 0.f) = std::stof(kv.substr(c + 1));
            i = j + 1;
        }
        Caller caller;
        caller.default_thr = std::stof(argv[4]);
        for (int i = 5; i < argc; i++) {
            std::string a = argv[i];
            if (a.rfind("mod=", 0) == 0) { size_t c = a.find(':'); ModCode code; parse_mod_code(a.substr(4, c - 4), &code); caller.mod_thr.push_back({code, std::stof(a.substr(c + 1))}); }
            else { int bb = base_idx(a[0]); caller.base_set[bb] = true; caller.base_thr[bb] = std::stof(a.substr(2)); }
        }
        Call c = make_call(caller, b, bmp);
        if (c.kind == CALL_FILTERED) printf("filtered\n");
        else if (c.kind == CALL_CANONICAL) printf("canonical %.9g\n", bmp.canonical_prob());
        else printf("modified %s %.9g\n", code_to_string(c.code).c_str(), *bmp.probs.get(c.code));
        return 0;
    }
    if (cmd == "percentile") {
        std::vector<float> xs;
        std::string vs = argv[3];
        for (size_t i = 0; i < vs.size();) { size_t j = vs.find(',', i); if (j == std::string::npos) j = vs.size(); xs.push_back(std::stof(vs.substr(i, j - i))); i = j + 1; }
        std::sort(xs.begin(), xs.end());
        printf("%.9g\n", percentile_linear_interp(xs, std::stof(argv[2])));
        return 0;
    }
    return 2;
}

// modkit_oracle summary|sample-probs [flags] <in.bam>  (src/commands.rs:549-1190): report on stdout
static int sample_main(int argc, char** argv) {
    const bool summary = std::string(argv[1]) == "summary";
    std::vector<std::string> pos, filter_thresholds, mod_thresholds;
    int threads = 4;
    uint32_t interval_size = 1000000;
    size_t num_reads = 10042;
    bool have_frac = false, no_sampling = false, no_filtering = false, only_mapped = false, invert_edge = false, tsv = false;
    double frac = 0;
    float percentile = 0.1f;
    std::string region_s, include_bed, ignore_s, edge_s, percentiles = "0.1,0.5,0.9";
    for (int i = 2; i < argc; i++) {
        std::string a = argv[i];
        auto val = [&]() -> std::string { if (i + 1 >= argc) die("missing value for " + a); return argv[++i]; };
        if (a == "-t" || a == "--threads") threads = std::stoi(val());
        else if (a == "--region") region_s = val();
        else if (a == "-n" || a == "--num-reads") num_reads = std::stoul(val());
        else if (a == "-f" || a == "--sampling-frac") { have_frac = true; frac = std::stod(val()); }
        else if (a == "--no-sampling") no_sampling = true;
        else if (a == "-i" || a == "--interval-size") interval_size = (uint32_t)std::stoul(val());
        else if (a == "--include-bed") include_bed = val();
        else if (a == "--only-mapped") only_mapped = true;
        else if (a == "--ignore") ignore_s = val();
        else if (a == "--edge-filter") edge_s = val();
        else if (a == "--invert-edge-filter") invert_edge = true;
        else if (summary && a == "--filter-threshold") filter_thresholds.push_back(val());
        else if (summary && a == "--mod-thresholds") mod_thresholds.push_back(val());
        else if (summary && a == "--no-filtering") no_filtering = true;
        else if (summary && (a == "-p" || a == "--filter-percentile")) percentile = std::stof(val());
        else if (summary && a == "--tsv") tsv = true;
        else if (!summary && (a == "-p" || a == "--percentiles")) percentiles = val();
        else if (a.size() > 1 && a[0] == '-') die("unexpected argument " + a);
        else pos.push_back(a);
    }
    if (pos.size() != 1) die("usage: modkit_oracle " + std::string(argv[1]) + " [flags] <in.bam>");
    BamFile bam;
    bam.load(pos[0], threads);
    Region region;
    const Region* rp = nullptr;
    if (!region_s.empty()) { region = parse_region(region_s, bam); rp = &region; }
    PositionFilter pfilter;
    const PositionFilter* pf = nullptr;
    if (!include_bed.empty()) {
        std::map<std::string, uint32_t> name_to_tid;
        for (auto& c : get_targets(bam, rp)) name_to_tid[c.name] = c.tid;
        pfilter.load(include_bed, name_to_tid);
        pf = &pfilter;
    }
    SampleOptions so;
    so.threads = threads; so.sampling_interval_size = interval_size;
    if (no_sampling) so.frac_all = true;
    else if (have_frac) { if (frac != 1.0) die("oracle supports only -f 1.0"); so.frac_all = true; }
    so.num_reads = num_reads;
    so.region = rp;
    so.include_unmapped = !(only_mapped || pf);
    if (!ignore_s.empty()) { so.collapse = true; if (!parse_mod_code(ignore_s, &so.collapse_code)) die("failed to parse mod code " + ignore_s); }
    if (!edge_s.empty()) {
        so.edge.on = true; so.edge.inverted = invert_edge;
        auto c = edge_s.find(',');
        if (c == std::string::npos) so.edge.start = so.edge.end = std::stoul(edge_s);
        else { so.edge.start = std::stoul(edge_s.substr(0, c)); so.edge.end = std::stoul(edge_s.substr(c + 1)); }
    }
    so.pf = pf;
    Caller est;
    std::vector<float> vals[4];
    std::vector<const BamRecord*> selected;
    estimate_thresholds(bam, so, percentile, &est, vals, &selected);
    std::string text;
    if (!summary) {
        std::vector<std::vector<std::string>> rows;
        rows.push_back({"base", "percentile", "threshold"});
        std::vector<float> qs;
        for (size_t i = 0; i < percentiles.size();) { size_t j = percentiles.find(',', i); if (j == std::string::npos) j = percentiles.size(); qs.push_back(std::stof(percentiles.substr(i, j - i))); i = j + 1; }
        for (int b = 0; b < 4; b++) {
            if (vals[b].empty()) continue;
            for (float q : qs) { volatile float pct = q * 100.0f; rows.push_back({std::string(1, BASES[b]), f32_display(pct), f32_display(percentile_linear_interp(vals[b], q))}); }
        }
        std::vector<size_t> w(3, 0);
        for (auto& r : rows) for (size_t i = 0; i < 3; i++) w[i] = std::max(w[i], r[i].size());
        for (auto& r : rows) { for (size_t i = 0; i < 3; i++) text += " " + r[i] + std::string(w[i] - r[i].size(), ' ') + " "; text += "\n"; }
    } else {
        Caller caller;
        for (auto& raw : mod_thresholds) {
            auto c = raw.find(':');
            ModCode code;
            if (c == std::string::npos || !parse_mod_code(raw.substr(0, c), &code)) die("encountered illegal per-mod threshold: " + raw);
            caller.mod_thr.push_back({code, std::stof(raw.substr(c + 1))});
        }
        if (!filter_thresholds.empty()) {
            for (auto& raw : filter_thresholds) {
                auto c = raw.find(':');
                if (c == std::string::npos) caller.default_thr = std::stof(raw);
                else { const char* f = strchr(BASES, raw[0]); if (!f || !raw[0]) die("failed to parse base " + raw); caller.base_set[f - BASES] = true; caller.base_thr[f - BASES] = std::stof(raw.substr(c + 1)); }
            }
        } else if (!no_filtering) {
            for (int b = 0; b < 4; b++) { caller.base_set[b] = est.base_set[b]; caller.base_thr[b] = est.base_thr[b]; }
        }
        ModSummaryOut S;
        summarize_reads(selected, so, caller, &S);
        text = summary_text(S, caller, tsv, rp ? rp->name + ":" + std::to_string(rp->start) + "-" + std::to_string(rp->end) : std::string());
    }
    fwrite(text.data(), 1, text.size(), stdout);
    return 0;
}

int main(int argc, char** argv) {
    try {
        if (argc >= 2 && (std::string(argv[1]) == "decode" || std::string(argv[1]) == "call" || std::string(argv[1]) == "percentile" || std::string(argv[1]) == "endpos")) return kat_main(argc, argv);
        if (argc >= 2 && (std::string(argv[1]) == "summary" || std::string(argv[1]) == "sample-probs")) return sample_main(argc, argv);
        if (argc < 2 || std::string(argv[1]) != "pileup") die("usage: modkit_oracle pileup [flags] <in.bam> <out.bed>");
        std::vector<std::string> pos;
        int threads = 4;
        uint32_t interval_size = 100000, sampling_interval_size = 1000000;
        size_t num_reads = 10042;
        bool have_frac = false; double frac = 0;
        bool no_filtering = false, include_unmapped = false, force_allow = false, cpg = false, mask = false;
        uint32_t max_depth = 8000;
        bool traditional = false, combine_mods = false, combine_strands = false, mixed = false, header = false, invert_edge = false;
        float percentile = 0.1f;
        std::vector<std::string> filter_thresholds, mod_thresholds, motif_parts;
        std::string region_s, sample_region_s, ignore_s, ref_fp, edge_s, timing_fp, include_bed, prefix;
        std::vector<std::string> partition_tags;
        bool bedgraph = false;
        for (int i = 2; i < argc; i++) {
            std::string a = argv[i];
            auto val = [&]() -> std::string { if (i + 1 >= argc) die("missing value for " + a); return argv[++i]; };
            if (a == "-t" || a == "--threads") threads = std::stoi(val());
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
            else if (a == "--motif") { motif_parts.push_back(val()); motif_parts.push_back(val()); }
            else if (a == "--cpg") cpg = true;
            else if (a == "-r" || a == "--ref" || a == "--reference") ref_fp = val();
            else if (a == "-k" || a == "--mask") mask = true;
            else if (a == "--preset") { if (val() != "traditional") die("unknown preset"); traditional = true; }
            else if (a == "--combine-mods") combine_mods = true;
            else if (a == "--combine-strands") combine_strands = true;
            else if (a == "--edge-filter") edge_s = val();
            else if (a == "--invert-edge-filter") invert_edge = true;
            else if (a == "--only-tabs" || a == "--suppress-progress") {}
            else if (a == "--mixed-delim" || a == "--mixed-delimiters") mixed = true;
            else if (a == "--header" || a == "--with-header" || a == "--include_header") header = true;
            else if (a == "--timing-json") timing_fp = val();
            else if (a == "--include-bed" || a == "--include-positions") include_bed = val();
            else if (a == "--partition-tag") partition_tags.push_back(val());
            else if (a == "--bedgraph") bedgraph = true;
            else if (a == "--prefix") prefix = val();
            else if (a.size() > 1 && a[0] == '-' && a != "-") die("unsupported flag " + a);
            else pos.push_back(a);
        }
        if (pos.size() != 2) die("expected <in.bam> <out.bed>");
        auto t0 = std::chrono::steady_clock::now();
        BamFile bam;
        bam.load(pos[0], threads);
        auto t_load = std::chrono::steady_clock::now();

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
            if (!mapped) die("did not find any mapped reads, perform alignment first or use modkit extract and/or modkit summary to inspect unaligned modBAMs");
        }
        if (percentile > 1.0f) die("filter percentile must be <= 1.0");
        if (combine_strands && !(cpg || !motif_parts.empty())) die("need to specify either --motif or --cpg to combine strands");

        PileupParams P;
        P.max_depth = max_depth;
        P.force_allow_implicit = force_allow;
        bool threshold_collapse = false;
        if (traditional) {
            P.numeric = COLLAPSE; P.collapse_code = 'h'; combine_strands = true; threshold_collapse = true;
        } else if (combine_mods) {
            P.numeric = COMBINE;
        } else if (!ignore_s.empty()) {
            ModCode c;
            if (!parse_mod_code(ignore_s, &c)) die("failed to parse mod code " + ignore_s);
            P.numeric = COLLAPSE; P.collapse_code = c; threshold_collapse = true;
        }
        P.combine_strands = combine_strands;
        if (!edge_s.empty()) {
            P.edge.on = true; P.edge.inverted = invert_edge;
            auto c = edge_s.find(',');
            if (c == std::string::npos) P.edge.start = P.edge.end = std::stoul(edge_s);
            else { P.edge.start = std::stoul(edge_s.substr(0, c)); P.edge.end = std::stoul(edge_s.substr(c + 1)); }
        }
        // motifs
        std::vector<Motif> motifs;
        bool have_motifs = false;
        if (!motif_parts.empty()) {
            if (traditional) die("cannot use presets and motifs together");
            for (size_t i = 0; i + 1 < motif_parts.size(); i += 2)
                for (size_t j = i + 2; j + 1 < motif_parts.size(); j += 2)
                    if (motif_parts[i] == motif_parts[j] && motif_parts[i + 1] == motif_parts[j + 1]) die("cannot have the same motif more than once");
            bool has_cg0 = false;
            for (size_t i = 0; i + 1 < motif_parts.size(); i += 2) if (motif_parts[i] == "CG" && motif_parts[i + 1] == "0") has_cg0 = true;
            if (cpg && !has_cg0) { motif_parts.push_back("CG"); motif_parts.push_back("0"); }
            for (size_t i = 0; i + 1 < motif_parts.size(); i += 2) motifs.push_back(Motif::parse(motif_parts[i], std::stoi(motif_parts[i + 1])));
            have_motifs = true;
        } else if (traditional || cpg) {
            motifs.push_back(Motif::parse("CG", 0));
            have_motifs = true;
        }
        std::vector<std::string> motif_labels;
        for (auto& m : motifs) motif_labels.push_back(m.label());
        MotifLookup lookup;
        if (have_motifs) {
            if (ref_fp.empty()) die("reference fasta is required for using --motif or --cpg options");
            if (combine_strands) for (auto& m : motifs) if (!m.palindrome) die("cannot combine strands with a motif that is not a palindrome");
            lookup.fa.open(ref_fp);
            lookup.motifs = motifs;
            lookup.mask = mask;
            lookup.pf = pf;
            for (auto& m : motifs) lookup.longest = std::max<uint64_t>(lookup.longest, m.length);
        }
        // thresholds
        auto parse_base_thr = [&](const std::string& raw) {
            auto c = raw.find(':');
            if (c == std::string::npos) { P.caller.default_thr = std::stof(raw); return; }
            int b = base_idx(raw[0]);
            if (b < 0) die("failed to parse base " + raw);
            P.caller.base_set[b] = true;
            P.caller.base_thr[b] = std::stof(raw.substr(c + 1));
        };
        for (auto& raw : mod_thresholds) {
            auto c = raw.find(':');
            ModCode code;
            if (c == std::string::npos || !parse_mod_code(raw.substr(0, c), &code)) die("illegal per-mod threshold " + raw);
            P.caller.mod_thr.push_back({code, std::stof(raw.substr(c + 1))});
        }
        if (!filter_thresholds.empty()) {
            for (auto& raw : filter_thresholds) parse_base_thr(raw);
        } else if (!no_filtering) {
            SampleOptions so;
            so.threads = threads;
            so.sampling_interval_size = sampling_interval_size;
            if (have_frac) { if (frac != 1.0) die("oracle supports only -f 1.0 (Rust StdRng sampling is not reproducible)"); so.frac_all = true; }
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
        auto t_thr = std::chrono::steady_clock::now();

        if (pf) targets = optimize_reference_records(*pf, targets, interval_size);
        std::vector<Interval> ivs = make_intervals(targets, interval_size, combine_strands, have_motifs ? &lookup : nullptr, nullptr, pf);
        uint64_t total_positions = 0;
        for (auto& iv : ivs) total_positions += iv.end - iv.start;
        auto t_ivs = std::chrono::steady_clock::now();

        // util.rs:690-712
        for (size_t i = 0; i < partition_tags.size(); i++) {
            if (partition_tags[i].size() != 2) die("illegal tag " + partition_tags[i] + " should be length 2");
            for (size_t j = 0; j < i; j++) if (partition_tags[j] == partition_tags[i]) die("cannot repeat partition-tags, got " + partition_tags[i] + " twice");
        }
        const bool partitioned = !partition_tags.empty();
        const bool to_dir = partitioned || bedgraph;       // output path is a directory of files (writers.rs:264-381, 1005-1082)
        if (to_dir && header) die("--header cannot be used with --bedgraph / --partition-tag");
        if (bedgraph && mixed) die("--mixed-delim cannot be used with --bedgraph");
        FILE* out = nullptr;
        std::map<std::string, FILE*> files;
        if (!to_dir) {
            out = (pos[1] == "-" || pos[1] == "stdout") ? stdout : fopen(pos[1].c_str(), "w");
            if (!out) die("failed to make output file");
            if (header) fputs(bedmethyl_header(), out);
        } else {
            std::error_code ec;
            std::filesystem::create_directories(pos[1], ec);
            if (ec) die("failed to create output directory");
        }
        auto sink = [&](const std::string& fname) -> FILE* {
            auto it = files.find(fname);
            if (it != files.end()) return it->second;
            FILE* f = fopen((pos[1] + "/" + fname).c_str(), "w");
            if (!f) die("failed to make output file " + fname);
            files[fname] = f;
            return f;
        };

        StateTable st;
        typedef std::vector<std::pair<std::string, std::string>> Routed;      // (file name, text) in a fixed order
        std::vector<std::string> results(ivs.size());
        std::vector<Routed> routed(ivs.size());
        std::vector<char> done(ivs.size(), 0);
        std::atomic<size_t> next{0};
        std::mutex mu;
        std::condition_variable cv;
        size_t n_rows = 0;
        const std::string pfx = prefix.empty() ? std::string() : prefix + "_";
        auto worker = [&]() {
            while (true) {
                size_t i = next.fetch_add(1);
                if (i >= ivs.size()) break;
                const std::string& chrom = bam.ref_names[ivs[i].tid];
                std::string text;
                Routed rt;
                size_t nr = 0;
                if (!to_dir) {
                    std::vector<Row> rows;
                    process_interval(bam, ivs[i], P, st, have_motifs ? &motifs : nullptr, &rows);
                    for (auto& R : rows) format_row(R, chrom, motif_labels, mixed, &text);
                    nr = rows.size();
                } else {
                    // partition keys present among the admitted reads of this interval ("" = no partitioning, "\1" = NoKey)
                    std::set<std::string> keys;
                    if (!partitioned) keys.insert("");
                    else bam.fetch(ivs[i].tid, ivs[i].start, ivs[i].end, [&](const BamRecord& r) {
                        if (!admitted_for_pileup(r)) return;
                        std::string k;
                        keys.insert(partition_key_of(r, partition_tags, &k) ? k : std::string("\1"));
                    });
                    std::map<std::string, std::string> by_file;
                    for (auto& key : keys) {
                        std::function<bool(const BamRecord&)> keep = [&](const BamRecord& r) {
                            std::string k;
                            const bool have = partition_key_of(r, partition_tags, &k);
                            return key == "\1" ? !have : (have && k == key);
                        };
                        std::vector<Row> rows;
                        process_interval(bam, ivs[i], P, st, have_motifs ? &motifs : nullptr, &rows, nullptr, nullptr, partitioned ? &keep : nullptr);
                        nr += rows.size();
                        const std::string key_name = !partitioned ? std::string() : (key == "\1" ? std::string("ungrouped") : key);
                        if (!bedgraph) {
                            std::string& t = by_file[pfx + key_name + ".bed"];
                            for (auto& R : rows) format_row(R, chrom, motif_labels, mixed, &t);
                        } else {
                            for (auto& R : rows) {
                                std::string label, line;
                                format_bedgraph_row(R, chrom, motif_labels, &label, &line);
                                by_file[pfx + key_name + (key_name.empty() ? "" : "_") + label + "_" + strand_label(R.strand) + ".bedgraph"] += line;
                            }
                        }
                    }
                    for (auto& kv : by_file) if (!kv.second.empty()) rt.push_back(kv);
                }
                std::lock_guard<std::mutex> g(mu);
                results[i].swap(text);
                routed[i].swap(rt);
                done[i] = 1;
                n_rows += nr;
                cv.notify_all();
            }
        };
        std::vector<std::thread> pool;
        for (int t = 0; t < std::max(1, threads); t++) pool.emplace_back(worker);
        for (size_t i = 0; i < ivs.size(); i++) {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return done[i] != 0; });
            std::string text;
            Routed rt;
            text.swap(results[i]);
            rt.swap(routed[i]);
            lk.unlock();
            if (out) fwrite(text.data(), 1, text.size(), out);
            for (auto& kv : rt) fwrite(kv.second.data(), 1, kv.second.size(), sink(kv.first));
        }
        for (auto& t : pool) t.join();
        if (out) { if (out != stdout) fclose(out); else fflush(out); }
        for (auto& kv : files) fclose(kv.second);
        auto t1 = std::chrono::steady_clock::now();
        auto sec = [](auto a, auto b) { return std::chrono::duration<double>(b - a).count(); };
        fprintf(stderr, "> Done, processed %zu rows. positions=%llu load=%.3fs thresholds=%.3fs intervals=%.3fs pileup=%.3fs total=%.3fs\n",
                n_rows, (unsigned long long)total_positions, sec(t0, t_load), sec(t_load, t_thr), sec(t_thr, t_ivs), sec(t_ivs, t1), sec(t0, t1));
        if (!timing_fp.empty()) {
            FILE* tf = fopen(timing_fp.c_str(), "w");
            if (tf) {
                fprintf(tf, "{\"positions\": %llu, \"rows\": %zu, \"threads\": %d, \"load_s\": %.6f, \"thresholds_s\": %.6f, \"intervals_s\": %.6f, \"pileup_s\": %.6f, \"total_s\": %.6f}\n",
                        (unsigned long long)total_positions, n_rows, threads, sec(t0, t_load), sec(t_load, t_thr), sec(t_thr, t_ivs), sec(t_ivs, t1), sec(t0, t1));
                fclose(tf);
            }
        }
        return 0;
    } catch (const std::exception& e) {
        die(e.what());
    }
    return 1;
}
