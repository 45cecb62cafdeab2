// Host side of the H100 `modkit pileup` path: everything the reference does around
// process_region_batch (src/pileup/subcommand.rs:381-817) that is not the hot loop itself:
//   reference intervals + focus positions   src/interval_chunks.rs:61-297, 563-643; src/fasta.rs:92-226
//   motif search                            src/find_motifs/motif_bed.rs:21-330
//   strand combining / motif labelling      src/pileup/mod.rs:331-363, 469-561
//   bedMethyl text                          src/writers.rs:87-156
// The per-read work (MM/ML decode, CIGAR projection, thresholding, counting) runs on the GPU behind
// include/mkp.h; nothing here computes calls or counts.
#pragma once
#include <cmath>
#include <cstdio>
#include <fstream>
#include <atomic>
#include <exception>
#include <map>
#include <unistd.h>
#include <mutex>
#include <thread>
#include <sstream>

#include "bam_reader.hpp"

namespace mkh {

// ---------------------------------------------------------------- FASTA (.fai) -------------------
class IndexedFasta {
    struct Ent { uint64_t len, off, bases, width; };
    std::map<std::string, Ent> ents_;
    FILE* fh_ = nullptr;
public:
    ~IndexedFasta() { if (fh_) fclose(fh_); }
    void open(const std::string& fa) {
        std::ifstream f(fa + ".fai");
        if (!f) throw std::runtime_error("failed to open FASTA index " + fa + ".fai (a .fai is required)");
        std::string name;
        Ent e;
        std::string line;
        while (std::getline(f, line)) { std::istringstream ss(line); if (ss >> name >> e.len >> e.off >> e.bases >> e.width) ents_[name] = e; }
        fh_ = fopen(fa.c_str(), "rb");
        if (!fh_) throw std::runtime_error("failed to open FASTA " + fa);
    }
    uint64_t length(const std::string& contig) const { auto it = ents_.find(contig); return it == ents_.end() ? 0 : it->second.len; }
    // upper-cased (unless keep_case) bases [b,e)
    void slice(const std::string& contig, uint64_t b, uint64_t e, bool keep_case, std::string* out) {
        out->clear();
        auto it = ents_.find(contig);
        if (it == ents_.end()) throw std::runtime_error("contig " + contig + " missing from FASTA index");
        const Ent& en = it->second;
        e = std::min(e, en.len);
        if (b >= e) return;
        const uint64_t first = en.off + (b / en.bases) * en.width + b % en.bases;
        const uint64_t last = en.off + ((e - 1) / en.bases) * en.width + (e - 1) % en.bases;
        std::string buf(last - first + 1, '\0');
        // pread: slices are taken from several threads at once
        size_t got = 0;
        while (got < buf.size()) {
            const ssize_t r = pread(fileno(fh_), &buf[got], buf.size() - got, (off_t)(first + got));
            if (r <= 0) break;
            got += (size_t)r;
        }
        if (got < buf.size()) throw std::runtime_error("short read from the reference FASTA (truncated file or stale .fai?) for contig " + contig);
        out->reserve(e - b);
        for (size_t i = 0; i < got; i++) { char c = buf[i]; if (c == '\n' || c == '\r') continue; out->push_back(keep_case ? c : (char)toupper((unsigned char)c)); }
    }
};

// ---------------------------------------------------------------- include-bed -----------------------
// `--include-bed` position filter (src/position_filter.rs:20-365): stranded, merged (overlapping or touching)
// half-open intervals per contig.
class IncludeBed {
public:
    struct Span { uint64_t b, e; };
    std::map<uint32_t, std::vector<Span>> plus, minus;

    static void coalesce(std::vector<Span>* v) {
        std::sort(v->begin(), v->end(), [](const Span& x, const Span& y) { return x.b != y.b ? x.b < y.b : x.e < y.e; });
        size_t w = 0;
        for (size_t i = 0; i < v->size(); i++) {
            if (w && (*v)[i].b <= (*v)[w - 1].e) (*v)[w - 1].e = std::max((*v)[w - 1].e, (*v)[i].e);
            else (*v)[w++] = (*v)[i];
        }
        v->resize(w);
    }
    void read(const std::string& path, const std::map<std::string, uint32_t>& name_to_tid) {
        std::ifstream f(path);
        if (!f) throw std::runtime_error("failed to open BED file " + path);
        std::string line, field;
        std::map<std::string, bool> skipped;
        while (std::getline(f, line)) {
            std::vector<std::string> col;
            std::istringstream ss(line);
            while (ss >> field) col.push_back(field);
            if (col.size() < 3 || skipped.count(col[0])) continue;
            auto num = [](const std::string& t, uint64_t* out) { if (t.empty() || t.find_first_not_of("0123456789") != std::string::npos) return false; *out = std::stoull(t); return true; };
            Span sp;
            if (!num(col[1], &sp.b) || !num(col[2], &sp.e)) continue;
            bool fw = true, rv = true;                     // BED3: both strands
            if (col.size() >= 6) {
                if (col[5] == "+") rv = false; else if (col[5] == "-") fw = false; else if (col[5] != ".") continue;
            } else if (col.size() != 3) continue;          // must be BED3 or BED6+
            auto t = name_to_tid.find(col[0]);
            if (t == name_to_tid.end()) { skipped[col[0]] = true; continue; }
            if (fw) plus[t->second].push_back(sp);
            if (rv) minus[t->second].push_back(sp);
        }
        if (plus.empty() && minus.empty()) throw std::runtime_error("zero valid positions parsed from BED file");
        for (auto& kv : plus) coalesce(&kv.second);
        for (auto& kv : minus) coalesce(&kv.second);
    }
    static bool touches(const std::vector<Span>& v, uint64_t a, uint64_t b) {   // some span with span.b < b && span.e > a
        size_t lo = 0, hi = v.size();
        while (lo < hi) { size_t mid = (lo + hi) / 2; if (v[mid].b < b) lo = mid + 1; else hi = mid; }
        return lo > 0 && v[lo - 1].e > a;
    }
    bool has(uint32_t tid, uint64_t p, bool minus_strand) const {
        const auto& m = minus_strand ? minus : plus;
        auto it = m.find(tid);
        return it != m.end() && touches(it->second, p, p + 1);
    }
    bool overlaps_any(uint32_t tid, uint64_t a, uint64_t b) const {
        auto it = plus.find(tid);
        if (it != plus.end() && touches(it->second, a, b)) return true;
        it = minus.find(tid);
        return it != minus.end() && touches(it->second, a, b);
    }
    bool has_contig(uint32_t tid) const { return plus.count(tid) || minus.count(tid); }
    // strand bitmaps of [cs,ce): the sampling-side position filter and FocusPositions::Regions rules
    void bitmaps(uint32_t tid, uint32_t cs, uint32_t ce, std::vector<uint32_t>* fp, std::vector<uint32_t>* fn) const {
        const size_t nw = ((size_t)ce - cs + 31) / 32;
        fp->assign(nw, 0); fn->assign(nw, 0);
        auto paint = [&](const std::map<uint32_t, std::vector<Span>>& m, std::vector<uint32_t>* bits) {
            auto it = m.find(tid);
            if (it == m.end()) return;
            for (auto& sp : it->second) {
                const uint64_t a = std::max<uint64_t>(sp.b, cs), b = std::min<uint64_t>(sp.e, ce);
                for (uint64_t p = a; p < b; p++) (*bits)[(p - cs) >> 5] |= 1u << ((p - cs) & 31);
            }
        };
        paint(plus, fp);
        paint(minus, fn);
    }
};

// ---------------------------------------------------------------- motifs -------------------------
struct MotifSpec {
    std::string raw;
    int offset = 0, rc_offset = 0, len = 0;
    bool palindromic = false;
    std::vector<uint8_t> fwd, rev;   // per position: allowed-base bit set A1 C2 G4 T8
    std::string label() const { return raw + "," + std::to_string(offset); }
};

inline uint8_t iupac_bits(char c) {
    switch (c) {
        case 'A': return 1; case 'C': return 2; case 'G': return 4; case 'T': return 8; case 'U': return 0;
        case 'M': return 3; case 'R': return 5; case 'W': return 9; case 'S': return 6; case 'Y': return 10; case 'K': return 12;
        case 'V': return 7; case 'H': return 11; case 'D': return 13; case 'B': return 14; case 'X': case 'N': return 15;
        default: return 0xff;
    }
}
inline uint8_t comp_bits(uint8_t m) { return (uint8_t)(((m & 1) << 3) | ((m & 2) << 1) | ((m & 4) >> 1) | ((m & 8) >> 3)); }

inline MotifSpec parse_motif(const std::string& raw, int offset) {
    MotifSpec m;
    m.raw = raw; m.len = (int)raw.size(); m.offset = offset;
    if (m.len == 1 && std::string("ACGT").find(raw[0]) == std::string::npos)
        throw std::runtime_error("degenerate bases are not supported as single base motifs, must be 'A', 'C', 'G', or 'T'.");
    if (offset + 1 > m.len) throw std::runtime_error("motif not long enough for offset " + std::to_string(offset));
    m.rc_offset = m.len - (offset + 1);
    for (char c : raw) { uint8_t b = iupac_bits(c); if (b == 0xff) throw std::runtime_error(std::string("Invalid IUPAC code: ") + c); m.fwd.push_back(b); }
    for (int i = m.len - 1; i >= 0; i--) m.rev.push_back(raw[i] == 'U' ? 1 : comp_bits(m.fwd[i]));
    // The reference compares the forward regex text with its reverse complement (motif_bed.rs:217-222). The text of
    // a class such as "[AC]" reverse-complements to "[GT]" with the letters in reversed order, so the texts are equal
    // exactly when the class sets are equal position by position and every class reads the same after that reversal,
    // which holds for all IUPAC classes the reference emits except none: set equality is the criterion.
    m.palindromic = (m.fwd == m.rev);
    for (char c : raw) if (c == 'U') m.palindromic = false;
    return m;
}

inline uint8_t base_bit(char c) { return c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 4 : c == 'T' ? 8 : 0; }

typedef std::map<uint32_t, uint8_t> SiteRules;   // position -> StrandRule bits (1 '+', 2 '-', 3 both)

inline void add_site(SiteRules* s, uint32_t p, uint8_t strand_bit) {
    auto it = s->find(p);
    if (it == s->end()) (*s)[p] = strand_bit; else if (it->second != strand_bit) it->second = 3;
}

// all hits of one motif inside seq (which starts at reference coordinate `origin`)
inline void motif_sites(const std::string& seq, uint64_t origin, const MotifSpec& m, SiteRules* out) {
    const size_t n = seq.size();
    auto hit = [&](size_t i, const std::vector<uint8_t>& cls) {
        if (i + cls.size() > n) return false;
        for (size_t k = 0; k < cls.size(); k++) if (!(base_bit(seq[i + k]) & cls[k])) return false;
        return true;
    };
    if (m.palindromic) {
        for (size_t i = 0; i < n; i++) if (hit(i, m.fwd)) { add_site(out, (uint32_t)(origin + i + m.offset), 1); add_site(out, (uint32_t)(origin + i + m.rc_offset), 2); }
    } else if (m.len == 1) {
        const char fw = m.raw[0], rv = fw == 'A' ? 'T' : fw == 'C' ? 'G' : fw == 'G' ? 'C' : 'A';
        for (size_t i = 0; i < n; i++) { if (seq[i] == fw) add_site(out, (uint32_t)(origin + i), 1); else if (seq[i] == rv) add_site(out, (uint32_t)(origin + i), 2); }
    } else {
        for (size_t i = 0; i < n; i++) {
            if (hit(i, m.fwd)) add_site(out, (uint32_t)(origin + i + m.offset), 1);
            if (hit(i, m.rev)) add_site(out, (uint32_t)(origin + i + m.rc_offset), 2);
        }
    }
}

// ---------------------------------------------------------------- intervals ----------------------
struct RefTarget { uint32_t tid, start, length; std::string name; uint32_t end() const { return start + length; } };

struct RefInterval {
    uint32_t tid = 0, start = 0, end = 0;
    bool all_positions = true;
    SiteRules rule;                                      // focus positions
    std::map<uint32_t, std::vector<int>> plus_ids, minus_ids;   // motif ids per strand
    // single palindromic two-base motif such as CG (the common case): the same information as a flat, position-sorted list
    // (position, StrandRule bits); motif id 0 on the strand(s) of the bits. rule / plus_ids / minus_ids stay empty.
    bool flat_valid = false;
    std::vector<std::pair<uint32_t, uint8_t>> flat;
    uint8_t flat_rule(uint32_t p) const {
        auto it = std::lower_bound(flat.begin(), flat.end(), std::make_pair(p, (uint8_t)0));
        return it != flat.end() && it->first == p ? it->second : 0;
    }
};

struct MotifContext {
    IndexedFasta fasta;
    std::vector<MotifSpec> motifs;
    bool keep_case = false;   // --mask
    uint64_t longest = 0;
    const IncludeBed* include = nullptr;   // motif hits outside the include-bed (strand-wise) are dropped (fasta.rs:55-69)
};

inline void fill_focus(RefInterval* iv, const std::vector<SiteRules>& sites, const std::vector<MotifSpec>& motifs, bool combine) {
    iv->all_positions = false;
    auto inside = [&](uint32_t p) { return p >= iv->start && p < iv->end; };
    if (combine) {   // FocusPositions::new_motif_combine_strands
        for (size_t id = 0; id < sites.size(); id++) for (auto& kv : sites[id]) {
            if (!inside(kv.first)) continue;
            auto it = iv->rule.find(kv.first);
            if (it == iv->rule.end()) iv->rule[kv.first] = kv.second; else if (it->second != kv.second) it->second = 3;
            if (kv.second & 1) iv->plus_ids[kv.first].push_back((int)id); else iv->minus_ids[kv.first].push_back((int)id);
        }
        return;
    }
    bool all_single = true;
    for (auto& m : motifs) all_single = all_single && m.len == 1;
    if (sites.size() == 1) {
        for (auto& kv : sites[0]) {
            if (!inside(kv.first)) continue;
            iv->rule[kv.first] = kv.second;
            if (kv.second & 1) iv->plus_ids[kv.first] = {0};
            if (kv.second & 2) iv->minus_ids[kv.first] = {0};
        }
    } else if (all_single) {
        auto id_of = [&](const char* b) { for (size_t i = 0; i < motifs.size(); i++) if (motifs[i].raw == b) return (int)i; return -1; };
        const char* pairs[2][2] = {{"A", "T"}, {"C", "G"}};
        for (auto& pr : pairs) {
            const int top = id_of(pr[0]), bot = id_of(pr[1]);
            if (top < 0) continue;   // the reference only walks the top base's table (interval_chunks.rs:216)
            for (auto& kv : sites[top]) {
                if (!inside(kv.first)) continue;
                if (bot >= 0) { iv->rule[kv.first] = 3; iv->plus_ids[kv.first] = {top, bot}; iv->minus_ids[kv.first] = {top, bot}; }
                else { iv->rule[kv.first] = kv.second; if (kv.second == 1) iv->plus_ids[kv.first] = {top}; else if (kv.second == 2) iv->minus_ids[kv.first] = {top}; }
            }
        }
    } else {
        for (size_t id = 0; id < sites.size(); id++) for (auto& kv : sites[id]) {
            if (!inside(kv.first)) continue;
            auto it = iv->rule.find(kv.first);
            if (it == iv->rule.end()) iv->rule[kv.first] = kv.second; else if (it->second != kv.second) it->second = 3;
            if (kv.second & 1) iv->plus_ids[kv.first].push_back((int)id);
            if (kv.second & 2) iv->minus_ids[kv.first].push_back((int)id);
        }
    }
}

// Motif sites of [start,end) and the (possibly extended) interval end (src/fasta.rs:92-226)
inline uint32_t motif_interval(MotifContext& mc, const RefTarget& c, uint64_t start, uint64_t end, bool combine, std::vector<SiteRules>* sites) {
    std::string seq;
    auto scan = [&](uint64_t e) {
        mc.fasta.slice(c.name, start, e, mc.keep_case, &seq);
        sites->assign(mc.motifs.size(), SiteRules());
        for (size_t i = 0; i < mc.motifs.size(); i++) motif_sites(seq, start, mc.motifs[i], &(*sites)[i]);
        if (mc.include) for (auto& st : *sites) for (auto it = st.begin(); it != st.end();) {
            uint8_t keep = 0;
            if ((it->second & 1) && mc.include->has(c.tid, it->first, false)) keep |= 1;
            if ((it->second & 2) && mc.include->has(c.tid, it->first, true)) keep |= 2;
            if (!keep) it = st.erase(it); else { it->second = keep; ++it; }
        }
    };
    if (!combine) { scan(end); return (uint32_t)end; }
    const uint64_t ref_end = c.end();
    const uint64_t pad = mc.longest * 5;
    uint64_t cut = end, fetch_end = std::min(end + pad, ref_end);
    for (;;) {
        scan(fetch_end);
        const uint64_t too_close = fetch_end >= mc.longest ? fetch_end - mc.longest : 0;
        // union of [site, site + len - offset) spans; spans that touch are merged (rust-lapper merge_overlaps)
        std::vector<std::pair<uint64_t, uint64_t>> spans;
        for (size_t i = 0; i < sites->size(); i++) {
            const uint64_t adj = mc.motifs[i].len >= mc.motifs[i].offset ? mc.motifs[i].len - mc.motifs[i].offset : mc.motifs[i].len;
            for (auto& kv : (*sites)[i]) spans.push_back({kv.first, kv.first + adj});
        }
        std::sort(spans.begin(), spans.end());
        uint64_t search_end = cut;
        uint64_t cur_b = 0, cur_e = 0;
        bool open = false;
        auto test = [&](uint64_t b, uint64_t e) { return b < cut && e > (cut ? cut - 1 : 0); };
        bool found = false;
        for (auto& s : spans) {
            if (open && s.first <= cur_e) { cur_e = std::max(cur_e, s.second); continue; }
            if (open && test(cur_b, cur_e)) { search_end = cur_e; found = true; break; }
            cur_b = s.first; cur_e = s.second; open = true;
        }
        if (!found && open && test(cur_b, cur_e)) search_end = cur_e;
        if (search_end < too_close || fetch_end >= ref_end) {
            for (auto& s : *sites) for (auto it = s.begin(); it != s.end();) { if (it->first > search_end) it = s.erase(it); else ++it; }
            return (uint32_t)search_end;
        }
        cut = fetch_end;
        fetch_end = std::min(fetch_end + pad, ref_end);
    }
}

// optimize_reference_records (src/position_filter.rs:106-212): the targets become spans that cover runs of include-bed
// intervals (a run is closed once it is longer than interval_size)
inline std::vector<RefTarget> targets_from_include_bed(const IncludeBed& ib, const std::vector<RefTarget>& targets, uint32_t interval_size) {
    std::vector<RefTarget> out;
    std::map<uint32_t, const RefTarget*> by_tid;
    for (auto& t : targets) by_tid[t.tid] = &t;
    std::map<uint32_t, bool> tids;
    for (auto& kv : ib.plus) tids[kv.first] = true;
    for (auto& kv : ib.minus) tids[kv.first] = true;
    for (auto& kv : tids) {
        auto bt = by_tid.find(kv.first);
        if (bt == by_tid.end()) continue;
        std::vector<IncludeBed::Span> all;
        auto a = ib.plus.find(kv.first); if (a != ib.plus.end()) all.insert(all.end(), a->second.begin(), a->second.end());
        auto b = ib.minus.find(kv.first); if (b != ib.minus.end()) all.insert(all.end(), b->second.begin(), b->second.end());
        IncludeBed::coalesce(&all);
        if (all.empty()) continue;
        IncludeBed::Span cur = all[0];
        for (size_t i = 1; i < all.size(); i++) {
            if (cur.e - cur.b > interval_size) { out.push_back({kv.first, (uint32_t)cur.b, (uint32_t)(cur.e - cur.b), bt->second->name}); cur = all[i]; }
            else cur.e = all[i].e;
        }
        out.push_back({kv.first, (uint32_t)cur.b, (uint32_t)(cur.e - cur.b), bt->second->name});
    }
    return out;
}

// End of the combine-strands interval that starts at `start` with nominal end `end` (src/fasta.rs:92-226): the same loop
// as motif_interval(combine = true), but every round only looks at the reference around the cut. The result depends on
// the merged span that covers cut - 1, whose right end is decided by the hits at and to the right of the hits covering
// cut - 1; those start within 2 * longest of the cut, so a window that starts 4 * longest + 8 before it sees all of them
// (a hit straddling the window start ends well before the cut and can neither be nor extend that span's right end).
inline uint32_t combine_interval_end(MotifContext& mc, const RefTarget& c, uint64_t start, uint64_t end) {
    const uint64_t ref_end = c.end();
    const uint64_t pad = mc.longest * 5, W = mc.longest * 4 + 8;
    uint64_t cut = end, fetch_end = std::min(end + pad, ref_end);
    std::string seq;
    std::vector<SiteRules> sites;
    for (;;) {
        const uint64_t ws = cut > start + W ? cut - W : start;
        mc.fasta.slice(c.name, ws, fetch_end, mc.keep_case, &seq);
        sites.assign(mc.motifs.size(), SiteRules());
        for (size_t i = 0; i < mc.motifs.size(); i++) motif_sites(seq, ws, mc.motifs[i], &sites[i]);
        if (mc.include) for (auto& st : sites) for (auto it = st.begin(); it != st.end();) {
            uint8_t keep = 0;
            if ((it->second & 1) && mc.include->has(c.tid, it->first, false)) keep |= 1;
            if ((it->second & 2) && mc.include->has(c.tid, it->first, true)) keep |= 2;
            if (!keep) it = st.erase(it); else { it->second = keep; ++it; }
        }
        const uint64_t too_close = fetch_end >= mc.longest ? fetch_end - mc.longest : 0;
        std::vector<std::pair<uint64_t, uint64_t>> spans;
        for (size_t i = 0; i < sites.size(); i++) {
            const uint64_t adj = mc.motifs[i].len >= mc.motifs[i].offset ? mc.motifs[i].len - mc.motifs[i].offset : mc.motifs[i].len;
            for (auto& kv : sites[i]) spans.push_back({kv.first, kv.first + adj});
        }
        std::sort(spans.begin(), spans.end());
        uint64_t search_end = cut, cur_b = 0, cur_e = 0;
        bool open = false, found = false;
        auto test = [&](uint64_t b, uint64_t e) { return b < cut && e > (cut ? cut - 1 : 0); };
        for (auto& sp : spans) {
            if (open && sp.first <= cur_e) { cur_e = std::max(cur_e, sp.second); continue; }
            if (open && test(cur_b, cur_e)) { search_end = cur_e; found = true; break; }
            cur_b = sp.first; cur_e = sp.second; open = true;
        }
        if (!found && open && test(cur_b, cur_e)) search_end = cur_e;
        if (search_end < too_close || fetch_end >= ref_end) return (uint32_t)search_end;
        cut = fetch_end;
        fetch_end = std::min(fetch_end + pad, ref_end);
    }
}

// ReferenceIntervalsFeeder order (src/interval_chunks.rs:563-643), step 1: the interval boundaries only (cheap: the
// combine-strands chain reads a few bases around every cut). `owner[i]` = index into `targets`.
inline std::vector<RefInterval> interval_grid(const std::vector<RefTarget>& targets, uint32_t interval_size, bool combine, MotifContext* mc,
                                              std::vector<size_t>* owner) {
    std::vector<RefInterval> out;
    for (size_t ti = 0; ti < targets.size(); ti++) {
        const RefTarget& c = targets[ti];
        if (!c.length) continue;
        uint32_t at = c.start;
        for (;;) {
            RefInterval iv;
            iv.tid = c.tid; iv.start = at;
            uint32_t e = (uint32_t)std::min<uint64_t>((uint64_t)at + interval_size, c.end());
            if (mc && combine) e = std::min(combine_interval_end(*mc, c, at, e), c.end());
            iv.end = e;
            if (owner) owner->push_back(ti);
            out.push_back(std::move(iv));
            if (e >= c.end()) break;
            at = e;
        }
    }
    return out;
}

// Step 2: focus positions (motif hits / include-bed positions) of the intervals [i0, i1), in parallel. Identical to what
// motif_interval + fill_focus give interval by interval: hits are searched in [start, end + 5 * longest) (any slice that
// reaches `longest` past the end finds every hit with a site before the end), hits that straddle the interval START are
// not found, sites at or past the end are dropped.
inline void fill_interval_focus(std::vector<RefInterval>& ivs, size_t i0, size_t i1, const std::vector<RefTarget>& targets, const std::vector<size_t>& owner,
                                bool combine, MotifContext* mc, const IncludeBed* include, int threads) {
    if (!(mc || include) || i1 <= i0) return;
    // one palindromic two-base motif at offset 0 (CG): hits cannot share a position, so the focus set is a flat sorted list
    const bool flat_ok = mc && mc->motifs.size() == 1 && mc->motifs[0].len == 2 && mc->motifs[0].palindromic && mc->motifs[0].offset == 0 &&
                         mc->motifs[0].fwd[0] != mc->motifs[0].fwd[1] && __builtin_popcount(mc->motifs[0].fwd[0]) == 1 && __builtin_popcount(mc->motifs[0].fwd[1]) == 1;
    auto fill = [&](RefInterval& iv, const RefTarget& c) {
        if (flat_ok) {
            MotifContext& m = *mc;
            std::string seq;
            // hits are searched in [start, fe): without --combine-strands fe is the interval end (a hit straddling the end is not
            // found, src/fasta.rs:207-227); with it the slice reaches past the end and sites at or past the end are dropped
            const uint64_t fe = combine ? std::min<uint64_t>((uint64_t)iv.end + m.longest * 5, c.end()) : iv.end;
            m.fasta.slice(c.name, iv.start, fe, m.keep_case, &seq);
            const uint8_t b0 = m.motifs[0].fwd[0], b1 = m.motifs[0].fwd[1];
            iv.all_positions = false;
            iv.flat_valid = true;
            iv.flat.clear();
            for (size_t i = 0; i + 1 < seq.size(); i++) {
                if (!(base_bit(seq[i]) & b0) || !(base_bit(seq[i + 1]) & b1)) continue;
                const uint32_t p = (uint32_t)(iv.start + i);
                uint8_t k0 = 1, k1 = 2;
                if (m.include) { if (!m.include->has(c.tid, p, false)) k0 = 0; if (!m.include->has(c.tid, p + 1, true)) k1 = 0; }
                if (k0 && p < iv.end) iv.flat.push_back({p, k0});
                if (k1 && p + 1 < iv.end) iv.flat.push_back({p + 1, k1});
            }
            return;
        }
        if (mc) {
            std::vector<SiteRules> sites;
            if (!combine) motif_interval(*mc, c, iv.start, iv.end, false, &sites);
            else {
                // sites of [start, end): scan a slice that reaches past the end, keep what lies before it
                MotifContext& m = *mc;
                std::string seq;
                const uint64_t fe = std::min<uint64_t>((uint64_t)iv.end + m.longest * 5, c.end());
                m.fasta.slice(c.name, iv.start, fe, m.keep_case, &seq);
                sites.assign(m.motifs.size(), SiteRules());
                for (size_t i = 0; i < m.motifs.size(); i++) motif_sites(seq, iv.start, m.motifs[i], &sites[i]);
                if (m.include) for (auto& st : sites) for (auto it = st.begin(); it != st.end();) {
                    uint8_t keep = 0;
                    if ((it->second & 1) && m.include->has(c.tid, it->first, false)) keep |= 1;
                    if ((it->second & 2) && m.include->has(c.tid, it->first, true)) keep |= 2;
                    if (!keep) it = st.erase(it); else { it->second = keep; ++it; }
                }
                for (auto& st : sites) for (auto it = st.begin(); it != st.end();) { if (it->first > iv.end) it = st.erase(it); else ++it; }
            }
            fill_focus(&iv, sites, mc->motifs, combine);
        } else if (include) {   // FocusPositions::new_regions / check_position (interval_chunks.rs:299-371)
            iv.all_positions = false;
            auto paint = [&](const std::map<uint32_t, std::vector<IncludeBed::Span>>& m, uint8_t bit) {
                auto it = m.find(c.tid);
                if (it == m.end()) return;
                for (auto& sp : it->second) { const uint64_t a = std::max<uint64_t>(sp.b, iv.start), b = std::min<uint64_t>(sp.e, iv.end); for (uint64_t p = a; p < b; p++) iv.rule[(uint32_t)p] |= bit; }
            };
            paint(include->plus, 1);
            paint(include->minus, 2);
        }
    };
    const size_t n = i1 - i0;
    const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, threads), n));
    std::atomic<size_t> next{0};
    std::exception_ptr err;
    std::mutex err_mu;
    auto work = [&]() {
        try { for (;;) { const size_t i = next.fetch_add(1); if (i >= n) break; fill(ivs[i0 + i], targets[owner[i0 + i]]); } }
        catch (...) { std::lock_guard<std::mutex> g(err_mu); if (!err) err = std::current_exception(); }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nt; t++) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    if (err) std::rethrow_exception(err);
}

// both steps for all intervals; `groups` = MultiChromCoordinates membership (sampling schedule)
inline std::vector<RefInterval> reference_intervals(const std::vector<RefTarget>& targets, uint32_t interval_size, bool combine,
                                                    MotifContext* mc, std::vector<std::vector<size_t>>* groups = nullptr,
                                                    const IncludeBed* include = nullptr, int threads = 1) {
    std::vector<size_t> owner;
    std::vector<RefInterval> out = interval_grid(targets, interval_size, combine, mc, &owner);
    fill_interval_focus(out, 0, out.size(), targets, owner, combine, mc, include, threads);
    if (groups) {
        std::vector<size_t> grp;
        uint64_t grp_len = 0;
        for (size_t i = 0; i < out.size(); i++) {
            grp_len += out[i].end - out[i].start;
            grp.push_back(i);
            if (grp_len >= interval_size) { groups->push_back(grp); grp.clear(); grp_len = 0; }
        }
        if (!grp.empty()) groups->push_back(grp);
    }
    return out;
}

// ---------------------------------------------------------------- rows -> bedMethyl --------------
struct OutRow { mkp_row r; int motif_idx; char strand; };

inline std::string code_text(uint32_t code) { return (code & 0x80000000u) ? std::to_string(code & 0x7fffffffu) : std::string(1, (char)code); }

// Expand device rows of one interval into output rows: motif-id replication (pileup/mod.rs:331-363) and
// strand combination (pileup/mod.rs:469-561).
inline void finish_interval_rows(const RefInterval& iv, const mkp_row* rows, size_t n, const std::vector<MotifSpec>* motifs,
                                 bool combine_strands, std::vector<OutRow>* out) {
    if (iv.flat_valid && combine_strands && motifs) {
        // one two-base palindromic motif (CG): the '+' rows at a site and the '-' rows at site + 1 are summed per code, in code
        // order (the BTreeMap of combine_strand_features); rows are position sorted, so one forward walk does it
        size_t i = 0;
        for (const auto& site : iv.flat) {
            if (!(site.second & 1)) continue;
            const uint32_t p = site.first;
            while (i < n && rows[i].pos < p) i++;
            mkp_row acc[40];             // (the device knows at most 32 (base, code) states)
            int na = 0;
            const bool minus_ok = (iv.flat_rule(p + 1) & 2) != 0;
            for (size_t j = i; j < n && rows[j].pos <= p + 1; j++) {
                const mkp_row& r = rows[j];
                if (!((r.pos == p && r.strand == '+') || (r.pos == p + 1 && r.strand == '-' && minus_ok))) continue;
                int k = 0;
                while (k < na && acc[k].code != r.code) k++;
                if (k == na) {
                    if (na == 40) break;
                    memset(&acc[na], 0, sizeof(mkp_row));
                    acc[na].pos = p; acc[na].code = r.code; acc[na].strand = '.'; acc[na].primary_base = r.primary_base;
                    na++;
                }
                mkp_row& A = acc[k];
                A.n_mod += r.n_mod; A.n_canon += r.n_canon; A.n_other += r.n_other; A.n_delete += r.n_delete;
                A.n_filtered += r.n_filtered; A.n_diff += r.n_diff; A.n_nocall += r.n_nocall;
            }
            for (int a = 1; a < na; a++) { const mkp_row key = acc[a]; int b = a; while (b > 0 && acc[b - 1].code > key.code) { acc[b] = acc[b - 1]; b--; } acc[b] = key; }
            for (int a = 0; a < na; a++) out->push_back({acc[a], 0, '.'});
        }
        return;
    }
    std::vector<OutRow> tmp;
    for (size_t i = 0; i < n; i++) {
        const mkp_row& r = rows[i];
        const std::vector<int>* ids = nullptr;
        static const std::vector<int> id0{0};
        if (iv.flat_valid) { if (iv.flat_rule(r.pos) & (r.strand == '+' ? 1 : 2)) ids = &id0; }
        else if (!iv.all_positions) {
            const auto& m = r.strand == '+' ? iv.plus_ids : iv.minus_ids;
            auto it = m.find(r.pos);
            if (it != m.end()) ids = &it->second;
        }
        if (ids) for (int id : *ids) tmp.push_back({r, id, (char)r.strand}); else tmp.push_back({r, -1, (char)r.strand});
    }
    if (!(combine_strands && !iv.all_positions && motifs)) { out->insert(out->end(), tmp.begin(), tmp.end()); return; }
    // rows are position sorted: index by position
    std::map<uint32_t, std::pair<size_t, size_t>> span;
    for (size_t i = 0; i < tmp.size();) { size_t j = i; while (j < tmp.size() && tmp[j].r.pos == tmp[i].r.pos) j++; span[tmp[i].r.pos] = {i, j}; i = j; }
    static const std::vector<int> id0v{0};
    std::vector<std::pair<uint32_t, const std::vector<int>*>> plus_sites;
    if (iv.flat_valid) { for (auto& e : iv.flat) if (e.second & 1) plus_sites.push_back({e.first, &id0v}); }
    else for (auto& kv : iv.plus_ids) plus_sites.push_back({kv.first, &kv.second});
    for (auto& kv : plus_sites) {
        const uint32_t p = kv.first;
        for (int id : *kv.second) {
            const MotifSpec& m = (*motifs)[id];
            if (!m.palindromic) continue;
            const int64_t partner = (int64_t)p + (m.rc_offset - m.offset);
            if (partner < 0) continue;
            std::map<uint32_t, mkp_row> acc;
            auto take = [&](uint32_t at, char strand) {
                auto it = span.find(at);
                if (it == span.end()) return;
                for (size_t i = it->second.first; i < it->second.second; i++) {
                    const OutRow& o = tmp[i];
                    if (o.strand != strand || o.motif_idx != id) continue;
                    auto a = acc.find(o.r.code);
                    if (a == acc.end()) { mkp_row z; memset(&z, 0, sizeof z); z.pos = p; z.code = o.r.code; z.strand = '.'; z.primary_base = o.r.primary_base; a = acc.emplace(o.r.code, z).first; }
                    mkp_row& A = a->second;
                    A.n_mod += o.r.n_mod; A.n_canon += o.r.n_canon; A.n_other += o.r.n_other; A.n_delete += o.r.n_delete;
                    A.n_filtered += o.r.n_filtered; A.n_diff += o.r.n_diff; A.n_nocall += o.r.n_nocall;
                }
            };
            take(p, '+');
            take((uint32_t)partner, '-');
            for (auto& a : acc) out->push_back({a.second, id, '.'});
        }
    }
}

struct BedFormat { bool mixed_delim = false; std::vector<std::string> motif_labels; };

inline char* put_u32(char* p, uint32_t v) {
    if (v < 10) { *p++ = (char)('0' + v); return p; }
    if (v < 100) { *p++ = (char)('0' + v / 10); *p++ = (char)('0' + v % 10); return p; }
    char t[12]; int n = 0; do { t[n++] = (char)('0' + v % 10); v /= 10; } while (v); while (n) *p++ = t[--n]; return p;
}

// printf("%.2f") of a float (writers.rs:140 prints an f32 with {:.2}): the exact binary value rounded to two decimals, ties to even.
// v * 100 is exact in double (24 + 7 significant bits), so are its integer part and the remainder.
inline char* put_pct2(char* p, float v) {
    if (!(v >= 0.0f && v < 1.0e6f)) return p + snprintf(p, 48, "%.2f", (double)v);       // (nan for rows without valid coverage, negatives: never)
    const double x = (double)v * 100.0;
    uint64_t k = (uint64_t)x;
    const double fr = x - (double)k;
    if (fr > 0.5 || (fr == 0.5 && (k & 1))) k++;
    p = put_u32(p, (uint32_t)(k / 100));
    *p++ = '.'; *p++ = (char)('0' + (k / 10) % 10); *p++ = (char)('0' + k % 10);
    return p;
}

inline void format_bed_row(const OutRow& o, const std::string& chrom, const BedFormat& fmt, std::string* out) {
    const mkp_row& r = o.r;
    const uint32_t cov = r.n_mod + r.n_canon + r.n_other;
    const char sp = fmt.mixed_delim ? ' ' : '\t';
    // name column: the code (a letter or a ChEBI number), plus the motif label when there are several motifs
    char name[96];
    size_t n_name = 0;
    if (r.code & 0x80000000u) n_name = (size_t)(put_u32(name, r.code & 0x7fffffffu) - name); else name[n_name++] = (char)r.code;
    const std::string* label = fmt.motif_labels.size() >= 2 && o.motif_idx >= 0 && (size_t)o.motif_idx < fmt.motif_labels.size() ? &fmt.motif_labels[o.motif_idx] : nullptr;
    // one row, one append: the numeric part needs < 200 bytes
    char stack_buf[640];
    std::string big;
    char* b0 = stack_buf;
    const size_t need = chrom.size() + n_name + (label ? label->size() + 1 : 0) + 256;
    if (need > sizeof stack_buf) { big.resize(need); b0 = &big[0]; }
    char* p = b0;
    memcpy(p, chrom.data(), chrom.size()); p += chrom.size();
    *p++ = '\t'; p = put_u32(p, r.pos); *p++ = '\t'; p = put_u32(p, r.pos + 1); *p++ = '\t';
    memcpy(p, name, n_name); p += n_name;
    if (label) { *p++ = ','; memcpy(p, label->data(), label->size()); p += label->size(); }
    *p++ = '\t'; p = put_u32(p, cov); *p++ = '\t'; *p++ = o.strand; *p++ = '\t'; p = put_u32(p, r.pos); *p++ = '\t'; p = put_u32(p, r.pos + 1);
    memcpy(p, "\t255,0,0\t", 9); p += 9;
    p = put_u32(p, cov); *p++ = sp;
    // writers.rs:140: format!("{:.2}", fraction_modified * 100f32) with f32 arithmetic
    const float frac = (float)r.n_mod / (float)cov;
    volatile float pct = frac * 100.0f;
    p = put_pct2(p, pct);
    *p++ = sp; p = put_u32(p, r.n_mod); *p++ = sp; p = put_u32(p, r.n_canon); *p++ = sp; p = put_u32(p, r.n_other);
    *p++ = sp; p = put_u32(p, r.n_delete); *p++ = sp; p = put_u32(p, r.n_filtered); *p++ = sp; p = put_u32(p, r.n_diff);
    *p++ = sp; p = put_u32(p, r.n_nocall); *p++ = '\n';
    out->append(b0, (size_t)(p - b0));
}

// `pileup-hemi` row (src/writers.rs:185-255): name `{pos call},{neg call},{base}` ('-' = canonical), strand '.', percent of the
// pattern among the base's patterns
inline void format_hemi_row(const mkp_hemi_row& r, const std::string& chrom, bool mixed_delim, std::string* out) {
    const uint32_t cov = r.count + r.n_other_pattern;
    const char sp = mixed_delim ? ' ' : '\t';
    char stack_buf[640];
    std::string big;
    char* b0 = stack_buf;
    if (chrom.size() + 256 > sizeof stack_buf) { big.resize(chrom.size() + 256); b0 = &big[0]; }
    char* p = b0;
    auto code = [&](uint32_t c) {
        if (c == MKP_HEMI_CANONICAL) *p++ = '-';
        else if (c & 0x80000000u) p = put_u32(p, c & 0x7fffffffu);
        else *p++ = (char)c;
    };
    memcpy(p, chrom.data(), chrom.size()); p += chrom.size();
    *p++ = '\t'; p = put_u32(p, r.pos); *p++ = '\t'; p = put_u32(p, r.pos + 1); *p++ = '\t';
    code(r.code_pos); *p++ = ','; code(r.code_neg); *p++ = ','; *p++ = "ACGT"[r.primary_base & 3];
    *p++ = '\t'; p = put_u32(p, cov); memcpy(p, "\t.\t", 3); p += 3; p = put_u32(p, r.pos); *p++ = '\t'; p = put_u32(p, r.pos + 1);
    memcpy(p, "\t255,0,0\t", 9); p += 9;
    p = put_u32(p, cov); *p++ = sp;
    // duplex.rs:44-46 and writers.rs:231: format!("{:.2}", count as f32 / valid_coverage as f32 * 100f32)
    const float frac = (float)r.count / (float)cov;
    volatile float pct = frac * 100.0f;
    p = put_pct2(p, pct);
    *p++ = sp; p = put_u32(p, r.count); *p++ = sp; p = put_u32(p, r.n_canonical); *p++ = sp; p = put_u32(p, r.n_other_pattern);
    *p++ = sp; p = put_u32(p, r.n_delete); *p++ = sp; p = put_u32(p, r.n_fail); *p++ = sp; p = put_u32(p, r.n_diff);
    *p++ = sp; p = put_u32(p, r.n_nocall); *p++ = '\n';
    out->append(b0, (size_t)(p - b0));
}

// --bedgraph (src/writers.rs:318-381): `chrom start end fraction coverage`, one file per (partition, strand, code[, motif])
inline const char* strand_label(char s) { return s == '+' ? "positive" : s == '-' ? "negative" : s == '.' ? "combined" : "_unknown"; }
inline std::string bedgraph_label(const OutRow& o, const BedFormat& fmt) {
    std::string label = code_text(o.r.code);
    if (o.motif_idx >= 0 && (size_t)o.motif_idx < fmt.motif_labels.size()) {
        std::string l = fmt.motif_labels[o.motif_idx];
        l.erase(std::remove(l.begin(), l.end(), ','), l.end());
        label += "_" + l;
    }
    return label;
}
inline void format_bedgraph_row(const OutRow& o, const std::string& chrom, std::string* out) {
    const mkp_row& r = o.r;
    const uint32_t cov = r.n_mod + r.n_canon + r.n_other;
    char buf[64];
    char* p = buf;
    out->append(chrom);
    *p++ = '\t'; p = put_u32(p, r.pos); *p++ = '\t'; p = put_u32(p, r.pos + 1); *p++ = '\t';
    out->append(buf, p - buf);
    out->append(f32_display((float)r.n_mod / (float)cov));      // `{}` of the f32 fraction
    p = buf;
    *p++ = '\t'; p = put_u32(p, cov); *p++ = '\n';
    out->append(buf, p - buf);
}

inline const char* bed_header_line() {
    return "chrom\tchromStart\tchromEnd\tname\tscore\tstrand\tthickStart\tthickEnd\tcolor\tvalid_coverage\tpercent_modified\t"
           "count_modified\tcount_canonical\tcount_other_mod\tcount_delete\tcount_fail\tcount_diff\tcount_nocall\n";
}

// focus bitmaps of a chunk [cs,ce) from its intervals
inline void focus_bitmaps(const std::vector<RefInterval>& ivs, size_t i0, size_t i1, uint32_t cs, uint32_t ce,
                          std::vector<uint32_t>* fpos, std::vector<uint32_t>* fneg) {
    const size_t nw = (ce - cs + 31) / 32;
    fpos->assign(nw, 0); fneg->assign(nw, 0);
    for (size_t i = i0; i < i1; i++) if (ivs[i].flat_valid) for (auto& kv : ivs[i].flat) {
        const uint32_t x = kv.first - cs;
        if (kv.second & 1) (*fpos)[x >> 5] |= 1u << (x & 31);
        if (kv.second & 2) (*fneg)[x >> 5] |= 1u << (x & 31);
    }
    for (size_t i = i0; i < i1; i++) if (!ivs[i].flat_valid) for (auto& kv : ivs[i].rule) {
        const uint32_t x = kv.first - cs;
        if (kv.second & 1) (*fpos)[x >> 5] |= 1u << (x & 31);
        if (kv.second & 2) (*fneg)[x >> 5] |= 1u << (x & 31);
    }
}

// thresholds.rs:17-39 on a histogram of MKP_HIST_BINS bins whose bin k holds the exact value k/1024
inline bool percentile_from_hist(const uint64_t* h, float q, float* out) {
    uint64_t n = 0;
    for (int k = 0; k < MKP_HIST_BINS; k++) n += h[k];
    if (n < 2) return false;
    auto value_at = [&](uint64_t idx) { uint64_t acc = 0; for (int k = 0; k < MKP_HIST_BINS; k++) { acc += h[k]; if (idx < acc) return (float)k / 1024.0f; } return (float)(MKP_HIST_BINS - 1) / 1024.0f; };
    if (q == 1.0f) { *out = value_at(n - 1); return true; }
    const float l = (float)(n - 1);
    const float x = l * q;
    const float left = std::floor(x);
    const uint64_t right = (uint64_t)std::ceil(x);
    const float g = x - std::trunc(x);
    const float y0 = value_at((uint64_t)left), y1 = value_at(right);
    volatile float a = y0 * (1.0f - g);
    volatile float b = y1 * g;
    *out = a + b;
    return true;
}

}  // namespace mkh
