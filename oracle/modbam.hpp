// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// CPU restatement of the per-read codecs of `modkit pileup` (reference v0.4.4):
//   MM grammar            src/mod_bam.rs:900-1000  (MmTagInfo::parse / parse_mm_tag)
//   delta -> positions    src/mod_bam.rs:697-767   (DeltaListConverter::to_positions*)
//   ML -> probability     src/mod_bam.rs:808-816   (quals_to_probs)
//   per-list tables       src/mod_bam.rs:1213-1295 (get_base_mod_probs, implicit fill)
//   list merging          src/mod_bam.rs:1037-1054, 629-656 (combine_positions_to_probs)
//   ModBaseInfo           src/mod_bam.rs:1481-1577
//   collapse              src/mod_bam.rs:530-627   (ReDistribute is the only one pileup reaches)
//   edge filter           src/mod_bam.rs:1075-1102, 1635-1672
//   threshold call        src/threshold_mod_caller.rs:28-63
//   argmax                src/mod_bam.rs:489-509
// Hash-map iteration order (rustc-hash 1.1.0 + hashbrown, SURVEY Appendix B.1) is restated in
// FxProbMap: slot = linear probe from (fxhash & mask), iteration = ascending slot.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

namespace orc {

// ModCodeRepr as u32: Code(char) = code point; ChEbi(n) = 0x80000000 | n, so n has 31 bits: a larger ChEBI number is an error
// (a read error in an MM header), where the reference takes any u32.
// Derived Ord (src/mod_base_code.rs:106): Code(_) < ChEbi(_), then by value  == plain u32 order.
typedef uint32_t ModCode;
inline bool code_is_chebi(ModCode c) { return c & 0x80000000u; }
inline std::string code_to_string(ModCode c) {
    if (code_is_chebi(c)) return std::to_string(c & 0x7fffffffu);
    return std::string(1, (char)c);
}
inline bool parse_mod_code(const std::string& raw, ModCode* out) {  // ModCodeRepr::parse
    if (raw.size() == 1) { *out = (uint8_t)raw[0]; return true; }
    if (raw.empty()) return false;
    uint64_t v = 0;
    for (char ch : raw) { if (ch < '0' || ch > '9') return false; v = v * 10 + (ch - '0'); if (v > 0x7fffffffull) return false; }
    *out = 0x80000000u | (uint32_t)v;
    return true;
}

inline int base_idx(char b) { switch (b) { case 'A': return 0; case 'C': return 1; case 'G': return 2; case 'T': return 3; default: return -1; } }
static const char BASES[5] = "ACGT";
inline int comp_idx(int b) { return 3 - b; }

inline uint64_t fx_hash_code(ModCode c) {
    const uint64_t K = 0x517cc1b727220a95ull;
    uint64_t h = 0;
    uint64_t disc = code_is_chebi(c) ? 1 : 0;
    h = (((h << 5) | (h >> 59)) ^ disc) * K;
    uint64_t v = code_is_chebi(c) ? (c & 0x7fffffffu) : c;
    h = (((h << 5) | (h >> 59)) ^ v) * K;
    return h;
}

// FxHashMap<ModCodeRepr, f32> with reproducible iteration order.
struct FxProbMap {
    std::vector<int> slot_to_item;   // size = buckets, -1 empty
    std::vector<ModCode> keys;
    std::vector<float> vals;
    std::vector<char> live;
    int n_live = 0;

    static int cap_of(int buckets) { return buckets < 8 ? buckets - 1 : buckets / 8 * 7; }
    static int buckets_for(int cap) {  // hashbrown capacity_to_buckets
        if (cap < 4) return 4;
        if (cap < 8) return 8;
        int adj = cap * 8 / 7;
        int b = 1;
        while (b < adj) b <<= 1;
        return b;
    }
    void place(int item) {
        int nb = (int)slot_to_item.size();
        int s = (int)(fx_hash_code(keys[item]) & (uint64_t)(nb - 1));
        while (slot_to_item[s] >= 0) s = (s + 1) & (nb - 1);
        slot_to_item[s] = item;
    }
    void reserve_for_insert() {
        if (slot_to_item.empty()) { slot_to_item.assign(4, -1); return; }
        int nb = (int)slot_to_item.size();
        if (n_live + 1 <= cap_of(nb)) return;
        int want = std::max(n_live + 1, cap_of(nb) + 1);
        std::vector<int> old = slot_to_item;
        slot_to_item.assign(buckets_for(want), -1);
        for (int it : old) if (it >= 0) place(it);
    }
    void reserve(int n) {  // from_iter / collect with a size hint
        if (!slot_to_item.empty() || n <= 0) return;
        slot_to_item.assign(buckets_for(n), -1);
    }
    int find(ModCode k) const {
        for (size_t i = 0; i < keys.size(); i++) if (live[i] && keys[i] == k) return (int)i;
        return -1;
    }
    float* get(ModCode k) { int i = find(k); return i < 0 ? nullptr : &vals[i]; }
    float* entry_or_insert(ModCode k, float v) {
        int i = find(k);
        if (i >= 0) return &vals[i];
        reserve_for_insert();
        keys.push_back(k); vals.push_back(v); live.push_back(1); n_live++;
        place((int)keys.size() - 1);
        return &vals.back();
    }
    // iteration in hashbrown order
    template <class F> void for_each(F&& f) const {
        for (int it : slot_to_item) if (it >= 0) f(keys[it], vals[it]);
    }
    size_t size() const { return (size_t)n_live; }
};

struct BaseModProbs {
    FxProbMap probs;
    bool inferred = false;
    float canonical_prob() const {  // mod_bam.rs:507-509 (f32 sum in map order)
        float s = 0.f;
        probs.for_each([&](ModCode, float p) { s += p; });
        return 1.0f - s;
    }
};

enum SkipMode { EXPLICIT = 0, IMPLICIT = 1, DEFAULT_IMPLICIT = 2 };

struct MmList {
    char base;       // A C G T U N
    char strand;     // + -
    int mode;
    std::vector<ModCode> codes;
    std::vector<uint32_t> deltas;
};

// src/mod_bam.rs:900-1000. Returns false on any parse error (read is skipped).
inline bool parse_mm(const char* s, size_t n, std::vector<MmList>* out) {
    size_t i = 0;
    while (i <= n) {
        size_t j = i;
        while (j < n && s[j] != ';') j++;
        if (j > i) {
            const char* part = s + i;
            size_t plen = j - i;
            size_t hlen = 0;
            while (hlen < plen && part[hlen] != ',') hlen++;
            MmList L;
            if (hlen < 1) return false;
            L.base = part[0];
            if (!(L.base == 'A' || L.base == 'C' || L.base == 'G' || L.base == 'T' || L.base == 'U' || L.base == 'N')) return false;
            if (hlen < 2) return false;
            L.strand = part[1];
            if (L.strand != '+' && L.strand != '-') return false;
            size_t k = 2;
            bool seen_chebi = false;
            int mode = -1;
            if (k < hlen && part[k] >= '0' && part[k] <= '9') {
                uint64_t v = 0;
                while (k < hlen && part[k] >= '0' && part[k] <= '9') { v = v * 10 + (part[k] - '0'); if (v > 0x7fffffffull) return false; k++; }
                L.codes.push_back(0x80000000u | (uint32_t)v);
                seen_chebi = true;
            }
            for (; k < hlen; k++) {
                char c = part[k];
                if (c == '?') mode = EXPLICIT;
                else if (c == '.') mode = IMPLICIT;
                else if (c >= '0' && c <= '9') return false;
                else if ((uint8_t)c >= 0x80) return false;  // the reference splits at a character count: the delta text would start off place
                else { if (seen_chebi) return false; L.codes.push_back((uint8_t)c); }
            }
            L.mode = mode < 0 ? DEFAULT_IMPLICIT : mode;
            if (L.codes.empty()) return false;  // reference would panic on a zero stride
            if (hlen + 1 <= plen) {
                // separated_list1(",", ws digit1 ws): at least one number; stop at first failure
                size_t q = hlen + 1;
                bool first = true;
                while (true) {
                    size_t save = q;
                    while (q < plen && (part[q] == ' ' || part[q] == '\t' || part[q] == '\n' || part[q] == '\r')) q++;
                    size_t d0 = q;
                    uint64_t v = 0;
                    while (q < plen && part[q] >= '0' && part[q] <= '9') { v = v * 10 + (part[q] - '0'); if (v > 0xffffffffull) return false; q++; }
                    if (q == d0) { if (first) return false; q = save; break; }
                    while (q < plen && (part[q] == ' ' || part[q] == '\t' || part[q] == '\n' || part[q] == '\r')) q++;
                    L.deltas.push_back((uint32_t)v);
                    first = false;
                    if (q < plen && part[q] == ',') q++; else break;
                }
            }
            out->push_back(std::move(L));
        }
        i = j + 1;
    }
    return true;
}

// One (strand, base) table: forward-read position -> probs
struct SeqPosTable {
    int mode = EXPLICIT;
    std::map<uint32_t, BaseModProbs> pos;   // ordered for determinism; the reference's order is not observable
};

struct ModBaseInfo {
    // [strand 0:+ 1:-][base idx]
    bool present[2][4] = {{false}};
    SeqPosTable tab[2][4];
    bool is_empty() const {
        for (int s = 0; s < 2; s++) for (int b = 0; b < 4; b++) if (present[s][b] && !tab[s][b].pos.empty()) return false;
        return true;
    }
};

const float MAX_PROB = 1.01f;

inline bool fundamental_matches(char fb, char nt) {
    switch (fb) { case 'A': return nt == 'A'; case 'C': return nt == 'C'; case 'G': return nt == 'G';
                  case 'T': case 'U': return nt == 'T'; case 'N': return true; }
    return false;
}

// src/mod_bam.rs:1488-1577 + 1213-1295. fwd = forward-read sequence (as sequenced), ml = ML bytes.
inline bool build_mod_base_info(const std::vector<MmList>& lists, const uint8_t* ml, size_t n_ml,
                                const std::string& fwd, ModBaseInfo* out) {
    size_t pointer = 0;
    std::vector<uint32_t> positions;
    for (const MmList& L : lists) {
        positions.clear();
        // --- to_positions
        if (L.base == 'N') {
            if (!L.deltas.empty()) {
                size_t cur = L.deltas[0];
                positions.push_back((uint32_t)cur);
                for (size_t k = 1; k < L.deltas.size(); k++) {
                    size_t nx = cur + L.deltas[k] + 1;
                    if (nx >= fwd.size()) return false;
                    positions.push_back((uint32_t)nx);
                    cur = nx;
                }
            }
        } else {
            size_t finger = 0;
            uint64_t n_skips = 0;
            uint32_t cum = 0;  // cumulative count at `finger`
            bool have = false;
            for (uint32_t d : L.deltas) {
                if (finger >= fwd.size()) return false;
                if (!have) { cum = fundamental_matches(L.base, fwd[0]) ? 1 : 0; have = true; }
                while ((uint64_t)cum <= (uint64_t)d + n_skips) {
                    finger++;
                    if (finger >= fwd.size()) return false;
                    if (fundamental_matches(L.base, fwd[finger])) cum++;
                }
                positions.push_back((uint32_t)finger);
                n_skips += (uint64_t)d + 1;
            }
        }
        size_t stride = L.codes.size();
        size_t end = pointer + L.deltas.size() * stride;
        if (end > n_ml) return false;
        // --- per-list tables keyed by the actual forward base
        bool lp[4] = {false, false, false, false};
        SeqPosTable lt[4];
        for (size_t k = 0; k < positions.size(); k++) {
            uint32_t p = positions[k];
            if (p >= fwd.size()) return false;  // (reference would panic for an out-of-range first N delta)
            int b = base_idx(fwd[p]);
            if (b < 0) return false;
            if (!lp[b]) { lp[b] = true; lt[b].mode = L.mode; }
            auto it = lt[b].pos.find(p);
            for (size_t c = 0; c < stride; c++) {
                float prob = ((float)ml[pointer + k * stride + c] + 0.5f) / 256.0f;
                if (it == lt[b].pos.end()) {
                    BaseModProbs bmp;
                    bmp.probs.reserve(1);
                    bmp.probs.entry_or_insert(L.codes[c], prob);
                    it = lt[b].pos.emplace(p, std::move(bmp)).first;
                } else {
                    BaseModProbs& bmp = it->second;
                    if (bmp.inferred && prob > 0.f) return false;
                    float* q = bmp.probs.entry_or_insert(L.codes[c], 0.f);
                    if (*q + prob > MAX_PROB) return false;
                    *q += prob;
                }
            }
        }
        if (L.mode != EXPLICIT && L.base != 'N') {
            for (size_t p = 0; p < fwd.size(); p++) {
                if (!fundamental_matches(L.base, fwd[p])) continue;
                int b = base_idx(fwd[p]);
                if (b < 0) return false;
                if (!lp[b]) { lp[b] = true; lt[b].mode = L.mode; }
                auto it = lt[b].pos.find((uint32_t)p);
                if (it != lt[b].pos.end()) {
                    BaseModProbs& bmp = it->second;
                    if (bmp.inferred) {
                        for (ModCode c : L.codes) {
                            float* q = bmp.probs.get(c);
                            bool bad = q && *q > 0.f;
                            *bmp.probs.entry_or_insert(c, 0.f) = 0.f;
                            if (bad) return false;
                        }
                    }
                } else {
                    BaseModProbs bmp;
                    bmp.inferred = true;
                    bmp.probs.reserve((int)L.codes.size());
                    for (ModCode c : L.codes) *bmp.probs.entry_or_insert(c, 0.f) = 0.f;
                    lt[b].pos.emplace((uint32_t)p, std::move(bmp));
                }
            }
        }
        // --- combine into the strand tables
        int s = L.strand == '+' ? 0 : 1;
        for (int b = 0; b < 4; b++) {
            if (!lp[b]) continue;
            SeqPosTable& agg = out->tab[s][b];
            if (!out->present[s][b]) { out->present[s][b] = true; agg.mode = L.mode; }
            if (agg.mode != lt[b].mode) agg.mode = IMPLICIT;
            for (auto& kv : lt[b].pos) {
                auto it = agg.pos.find(kv.first);
                if (it == agg.pos.end()) { agg.pos.emplace(kv.first, std::move(kv.second)); continue; }
                BaseModProbs& a = it->second;
                if (a.inferred != kv.second.inferred) return false;
                kv.second.probs.for_each([&](ModCode c, float p) { *a.probs.entry_or_insert(c, 0.f) += p; });
                float sum = 0.f;
                a.probs.for_each([&](ModCode, float p) { sum += p; });
                if (sum > MAX_PROB) return false;
            }
        }
        pointer += L.deltas.size() * stride;
    }
    return true;
}

// CollapseMethod::ReDistribute (src/mod_bam.rs:558-600)
inline BaseModProbs redistribute(const BaseModProbs& in, ModCode drop) {
    float marginal = 0.f;
    int n_other = 0;
    in.probs.for_each([&](ModCode c, float p) { if (c == drop) marginal += p; else n_other++; });
    float share = marginal / ((float)n_other + 1.0f);
    BaseModProbs out;
    out.inferred = in.inferred;
    in.probs.for_each([&](ModCode c, float p) { if (c != drop) *out.probs.entry_or_insert(c, 0.f) = p + share; });
    return out;
}

struct EdgeFilter {
    bool on = false;
    size_t start = 0, end = 0;
    bool inverted = false;
    bool read_can_be_trimmed(size_t len) const { return !(len <= start || len <= end); }
    bool keep(size_t pos, size_t len) const {
        if (inverted) return pos < start || pos >= len - end;
        return pos >= start && pos < len - end;
    }
};

struct Caller {  // MultipleThresholdModCaller
    bool base_set[4] = {false, false, false, false};
    float base_thr[4] = {0, 0, 0, 0};
    std::vector<std::pair<ModCode, float>> mod_thr;
    float default_thr = 0.f;
    const float* per_mod(ModCode c) const { for (auto& kv : mod_thr) if (kv.first == c) return &kv.second; return nullptr; }
};

enum CallKind : uint8_t { CALL_NONE = 0, CALL_FILTERED = 1, CALL_CANONICAL = 2, CALL_MODIFIED = 3 };
struct Call { uint8_t kind = CALL_NONE; ModCode code = 0; };

// src/threshold_mod_caller.rs:28-63
inline Call make_call(const Caller& caller, int threshold_base, const BaseModProbs& bmp) {
    bool have = false;
    float best_p = 0.f;
    Call best;
    bmp.probs.for_each([&](ModCode c, float p) {
        const float* t = caller.per_mod(c);
        if (!t) t = caller.per_mod((ModCode)(uint8_t)BASES[threshold_base]);
        if (!t && caller.base_set[threshold_base]) t = &caller.base_thr[threshold_base];
        float thr = t ? *t : caller.default_thr;
        if (p >= thr) {
            if (!have || p >= best_p) { have = true; best_p = p; best.kind = CALL_MODIFIED; best.code = c; }
        }
    });
    float cthr = caller.base_set[threshold_base] ? caller.base_thr[threshold_base] : caller.default_thr;
    float cp = bmp.canonical_prob();
    if (cp >= cthr) {
        if (!have || cp >= best_p) { have = true; best_p = cp; best.kind = CALL_CANONICAL; best.code = 0; }
    }
    if (!have) best.kind = CALL_FILTERED;
    return best;
}

// src/mod_bam.rs:489-505: value used by threshold estimation
inline float argmax_prob(const BaseModProbs& bmp) {
    float cp = bmp.canonical_prob();
    bool have = false;
    float mp = 0.f;
    bmp.probs.for_each([&](ModCode, float p) { if (!have || p >= mp) { have = true; mp = p; } });
    if (have && mp > cp) return mp;
    return cp;
}

}  // namespace orc
