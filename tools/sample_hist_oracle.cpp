// TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// `sample_hist_oracle [sample-probs flags] <in.bam>`: CPU restatement of the probabilities.tsv of `modkit sample-probs --hist`
// (reference v0.4.4, src/read_ids_to_base_mod_probs.rs:104-187, src/writers.rs:837-945), printed to stdout. It builds on the
// oracle's sampler and decode (oracle/driver.hpp: estimate_thresholds, sample_record), so its reads and calls are the ones of
// `modkit_oracle sample-probs`, whose stdout is the thresholds.tsv of the same run. Flags: -t, --region, -n, -f 1.0,
// --no-sampling, -i, --include-bed, --only-mapped, --ignore, --edge-filter, --invert-edge-filter; -p, --prefix and --hist are
// accepted and ignored, so that the product's argument list can be passed as it is.
#include <filesystem>

#include "../oracle/driver.hpp"

using namespace orc;

static void die(const std::string& m) { fprintf(stderr, "> Error! %s\n", m.c_str()); exit(1); }

// every sampled call's arg-max call keyed by (canonical base, BaseState): 0 canonical, else state_order_key; counts per qual
typedef std::map<std::pair<int, uint64_t>, std::map<int, uint64_t>> ProbHistogram;

static int prob_to_qual(float p) {                                 // mod_bam.rs:798-806
    if (p == 1.0f) return 255;
    const float s = std::floor(p * 256.0f);
    return !(s > 0.0f) ? 0 : s >= 255.0f ? 255 : (int)s;           // Rust `as u8`: saturating, NaN -> 0
}

static void mod_histogram_reads(const std::vector<const BamRecord*>& selected, const SampleOptions& o, ProbHistogram* H) {
    for (const BamRecord* rp : selected) {
        std::vector<float> v[4];
        std::vector<BaseModProbs> probs[4];
        if (!sample_record(*rp, o, v, probs)) continue;
        for (int b = 0; b < 4; b++) {
            for (const BaseModProbs& bmp : probs[b]) {
                // argmax_base_mod_call (mod_bam.rs:489-505): the last maximal code, if it beats the canonical probability
                const float cp = bmp.canonical_prob();
                bool have = false; float mp = 0.f; ModCode mc = 0;
                bmp.probs.for_each([&](ModCode c, float p) { if (!have || p >= mp) { have = true; mp = p; mc = c; } });
                if (have && mp > cp) (*H)[{b, state_order_key(mc)}][prob_to_qual(mp)]++;
                else (*H)[{b, 0}][prob_to_qual(cp)]++;
            }
        }
    }
}

// ProbHistogram::get_artifacts: rows by (base, state), non-zero bins ascending; frac and percentile_rank in f32 over an f32
// running sum of the counts
static std::string probabilities_text(const ProbHistogram& H) {
    std::string out = "code\tprimary_base\trange_start\trange_end\tcount\tfrac\tpercentile_rank\n";
    for (const auto& st : H) {
        uint64_t total_n = 0;
        for (const auto& kv : st.second) total_n += kv.second;
        const float total = (float)total_n;
        float cum_sum = 0.f;
        for (const auto& kv : st.second) {
            const float n = (float)kv.second;
            const float f = n / total;
            cum_sum = cum_sum + n;
            volatile float half = 0.5f * n;
            volatile float rank = ((cum_sum - half) / total) * 100.0f;
            out += (st.first.second == 0 ? std::string("-") : state_label_of_key(st.first.second));
            out += std::string("\t") + BASES[st.first.first] + "\t" + f32_display((float)kv.first / 256.0f) + "\t" + f32_display(((float)kv.first + 1.0f) / 256.0f) +
                   "\t" + std::to_string(kv.second) + "\t" + f32_display(f) + "\t" + f32_display(rank) + "\n";
        }
    }
    return out;
}

int main(int argc, char** argv) {
    try {
        std::vector<std::string> pos;
        int threads = 4;
        uint32_t interval_size = 1000000;
        size_t num_reads = 10042;
        bool have_frac = false, no_sampling = false, only_mapped = false, invert_edge = false;
        double frac = 0;
        std::string region_s, include_bed, ignore_s, edge_s;
        for (int i = 1; i < argc; i++) {
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
            else if (a == "-p" || a == "--percentiles" || a == "--prefix") val();
            else if (a == "--hist") {}
            else if (a.size() > 1 && a[0] == '-') die("unexpected argument " + a);
            else pos.push_back(a);
        }
        if (pos.size() != 1) die("usage: sample_hist_oracle [flags] <in.bam>");
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
        estimate_thresholds(bam, so, 0.1f, &est, vals, &selected);
        ProbHistogram H;
        mod_histogram_reads(selected, so, &H);
        const std::string text = probabilities_text(H);
        fwrite(text.data(), 1, text.size(), stdout);
        return 0;
    } catch (const std::exception& e) { die(e.what()); }
    return 1;
}
