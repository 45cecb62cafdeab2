// Device kernels of the H100-native `modkit pileup` hot path (sm_90a), and of pileup-hemi, threshold estimation, `summary` and
// `sample-probs` over the same decode. DESIGN §4.1 describes the pass.
//
// Per chunk, on one stream (intermediates stay in L2/HBM):
//   k_parse       warp per read: admission, reference span, MM list discovery and delta parse, rank/select on the 4-bit SEQ
//                 -> forward position of every list entry, ML length checks, implicit-mode bookkeeping; hands a list table to
//                 k_resolve (src/mod_bam.rs:900-1000, 667-767, 1213-1295, src/read_cache.rs:122-137)
//   k_resolve     warp per read, lane per list entry: CIGAR prefix, list merging, collapse, threshold call (MODE_PILEUP) or
//                 histogram / summary value (MODE_HIST), edge filter, projection to reference coordinates; emits call records,
//                 observed-code masks, implicit tables and hot-bitmap marks (src/mod_bam.rs:530-656, src/read_cache.rs:69-211,
//                 src/threshold_mod_caller.rs:28-63, src/util.rs:122-145, src/summarize.rs:117-252)
//   k_block_popc, k_scan_blocks, k_word_prefix, k_word_record   rank over the hot bitmap -> counter slot per hot position
//   k_count_calls warp per read, lanes over its call records: modcall / canonical / filtered counters (src/pileup/mod.rs:876-937)
//   k_count_bases warp per work item (a window of a read's reference span): base / delete counters under the hot positions and
//                 observed-code masks; counts the call records of reads with one sorted run itself (src/pileup/mod.rs:831-874)
//   k_rows        thread per bitmap word: FeatureVector::decode (src/pileup/mod.rs:283-445) -> mkp_row
//   k_hemi_count, k_hemi_rows   `pileup-hemi`: duplex pattern counters per + strand motif position and
//                 DuplexFeatureVector::decode -> mkp_hemi_row (src/pileup/duplex.rs)
// Integer and indexing work: no tensor cores, and far from bound by HBM bandwidth (DESIGN §11).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mkp.h"

namespace mkp {

constexpr int MAX_LISTS = 16;
constexpr int MAX_LIST_CODES = 4;
constexpr int MAX_MAP = 7;          // codes at one read position
constexpr int MAX_STATES = 32;
constexpr int CUM_CAP = 512;        // 32-base blocks whose occurrence counts fit in shared memory (reads <= 16 kb)
#ifndef MKP_CQ_CAP
#define MKP_CQ_CAP 640
#endif
constexpr int CQ_CAP = MKP_CQ_CAP;  // CIGAR ops whose prefix sums fit in shared memory per warp
constexpr int QT_CAP = 512;         // buckets of the query -> op table
constexpr uint32_t FULL = 0xffffffffu;

// layout (u32 words) of the counter slot of one (position, reference strand) pair; stride SL_MOD + states
constexpr int SL_BASE = 0;    // [b] 4 words, signed
constexpr int SL_DEL = 4;
constexpr int SL_FILT = 5;
constexpr int SL_CANON = 6;   // [pb]
constexpr int SL_OBS = 10;    // observed-code mask
constexpr int SL_MOD = 11;    // [state]

struct DevParams {
    float default_thr;
    float base_thr[4];
    uint32_t base_set[4];
    uint32_t n_mod_thr;
    uint32_t mod_code[MKP_MAX_MOD_THRESHOLDS];
    float mod_thr[MKP_MAX_MOD_THRESHOLDS];
    uint32_t numeric_mode, collapse_code, force_allow_implicit;
    uint32_t edge_on, edge_inv, edge_start, edge_end;
};

struct ReadMeta {       // 40 bytes, written by k_parse and k_resolve
    int32_t ref_end;
    uint32_t flags;     // bit0 admitted, bit1 has mod info (not in skip_set), bit2 call records are one position-sorted run
    uint32_t pos_mask, neg_mask;
    uint32_t n_calls;
    uint32_t n_hist;    // sampling: values contributed
    uint64_t entry_off;
    // implicit ('.'/default mode) tables: imp[s] byte b = 0x80 | state of the inferred-canonical entry of the
    // (mod strand s, forward base b) table (src/mod_bam.rs:1265-1292); 0 = no implicit table
    uint32_t imp[2];
};

struct ReadLists;

struct ChunkDev {
    const mkp_read_hdr* hdrs;
    const uint8_t* heap;
    const uint64_t* entry_off;  // exclusive prefix of len_ml
    uint32_t n_reads;
    uint32_t cs, ce;            // chunk range
    const uint32_t* focus_pos;  // may be null
    const uint32_t* focus_neg;
    ReadMeta* meta;
    uint32_t* P;                // forward positions per raw entry
    uint2* calls;               // (ref_pos, info)
    uint32_t* hot;              // [2][n_words] bitmaps over [cs,ce), per reference strand (+ then -)
    uint32_t* hot_prefix;
    unsigned long long* states; // registry: (pb<<32 | code), ~0 empty
    uint32_t* n_states;
    uint32_t* err;
    // dynamic read queues: +0 k_parse, +1 fast k_resolve, +2 k_count_bases / k_hemi_count, +3 k_count_calls (CountDev::work
    // and HemiDev::work point at +2), +4 length of slow_list, +5 generic k_resolve's cursor in slow_list
    uint32_t* work;
    uint32_t* slow_list;        // reads left to the generic k_resolve instantiation
    unsigned long long* total_calls;
    // per-warp scratch
    uint32_t* scr_cq; uint32_t* scr_cr;
    uint32_t max_ncigar, max_blocks;
    // sampling
    unsigned long long* hist;   // [4][MKP_HIST_BINS]
    unsigned long long* hist_inexact;
    const uint8_t* take;
    uint32_t hist_include_unaligned;
    // `modkit summary` (src/summarize.rs:117-252): with the caller's thresholds in c_par, every value of MODE_HIST is also classed
    // by (thresholded call, arg-max call): summ[((base * 2 + fail) * 33) + s], s = 0 canonical, 1 + state id; then reads per base
    // [4] and, as u32, the states observed per base [4]. nullptr = off.
    unsigned long long* summ;
    // `modkit sample-probs --hist` (src/read_ids_to_base_mod_probs.rs:104-187): every value of MODE_HIST counted under its
    // arg-max call and prob_to_qual bin: qhist[(base * 33 + s) * 256 + qual], s = 0 canonical, 1 + state id. nullptr = off.
    unsigned long long* qhist;
    uint32_t mode;              // MODE_PILEUP / MODE_HIST (admission rules of k_parse)
    struct ReadLists* rl;
    // chunks with focus bitmaps (the hot bitmap is the focus set, ranked at upload, and is not written):
    // 1 = list mode: the reads k_pileup_fused left to the generic kernels; k_parse walks slow_list[0 .. *(work + 4));
    // 2 = every read through the per-stage kernels
    uint32_t list_mode;
    // processing order of the dynamic read queue: longest reads first (a 200 kb read that starts last is the kernel's tail); null = index order
    const uint32_t* order;
};

__constant__ DevParams c_par;

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// --edge-filter (src/util.rs:122-145): a read no longer than either edge has no position the filter keeps
__device__ __forceinline__ bool edge_read_ok(uint32_t L) { return !c_par.edge_on || !(L <= c_par.edge_start || L <= c_par.edge_end); }
// does forward position f of a read of length L pass the filter? Only for a read that passes edge_read_ok (L > edge_end).
// k_count_bases and k_hemi_count call it without that guard: k_resolve gives no such read an implicit table
__device__ __forceinline__ bool edge_keep(uint32_t f, uint32_t L) {
    bool keep = true;
    if (c_par.edge_on) {
        if (c_par.edge_inv) keep = f < c_par.edge_start || f >= L - c_par.edge_end;
        else keep = f >= c_par.edge_start && f < L - c_par.edge_end;
    }
    return keep;
}
// threshold of canonical base tb: its --filter-threshold, else the default one
__device__ __forceinline__ float base_threshold(int tb) { return c_par.base_set[tb] ? c_par.base_thr[tb] : c_par.default_thr; }

// CIGAR op classes: query length, reference length, and M/=/X (a base aligned to the reference)
__device__ __forceinline__ bool cig_is_match(uint32_t op) { return op == 0 || op == 7 || op == 8; }
__device__ __forceinline__ uint32_t cig_qlen(uint32_t op, uint32_t len) { return (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) ? len : 0u; }
__device__ __forceinline__ uint32_t cig_rlen(uint32_t op, uint32_t len) { return (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ? len : 0u; }

// MODE_PILEUP call record (reference position, info): info = mod strand | forward base << 1 | state << 3 | nosub << 11, with
// state 0 filtered, 1 canonical, 2 + id modified, and nosub set on a '-' record whose position a '+' list also holds
__device__ __forceinline__ uint32_t call_info(uint32_t st, uint32_t b, uint32_t state, uint32_t nosub) { return st | (b << 1) | (state << 3) | (nosub << 11); }
__device__ __forceinline__ uint32_t call_strand(uint32_t info) { return info & 1u; }
__device__ __forceinline__ uint32_t call_base(uint32_t info) { return (info >> 1) & 3u; }
__device__ __forceinline__ uint32_t call_state(uint32_t info) { return (info >> 3) & 0xffu; }
__device__ __forceinline__ uint32_t call_nosub(uint32_t info) { return (info >> 11) & 1u; }

// MODE_HIST value record (key, value): key = bin | canonical base << 16 | inexact << 20 | qual << 21. With summ / qhist the
// value is the classification: thresholded kind | its state id << 2 | arg-max kind << 8 | its state id << 10 (kind 0 filtered,
// 1 canonical, 2 modified; a state id is only read with kind 2)
__device__ __forceinline__ uint32_t sample_key(uint32_t bin, uint32_t base, uint32_t inexact, uint32_t qual) { return bin | (base << 16) | (inexact << 20) | (qual << 21); }
__device__ __forceinline__ uint32_t sample_bin(uint32_t key) { return key & 0xffffu; }
__device__ __forceinline__ uint32_t sample_base(uint32_t key) { return (key >> 16) & 3u; }
__device__ __forceinline__ uint32_t sample_inexact(uint32_t key) { return (key >> 20) & 1u; }
__device__ __forceinline__ uint32_t sample_qual(uint32_t key) { return (key >> 21) & 255u; }
__device__ __forceinline__ uint32_t sample_class(uint32_t tk, uint32_t ts, uint32_t ak, uint32_t as) { return tk | (ts << 2) | (ak << 8) | (as << 10); }
__device__ __forceinline__ uint32_t class_tkind(uint32_t c) { return c & 3u; }
__device__ __forceinline__ uint32_t class_tstate(uint32_t c) { return (c >> 2) & 63u; }
__device__ __forceinline__ uint32_t class_akind(uint32_t c) { return (c >> 8) & 3u; }
__device__ __forceinline__ uint32_t class_astate(uint32_t c) { return (c >> 10) & 63u; }

// prob_to_qual (mod_bam.rs:798-806): exactly 1.0 -> 255, else floor(p * 256) in f32 with Rust's saturating `as u8` (NaN and
// negatives -> 0, values from 255/256 up -> 255)
__device__ __forceinline__ uint32_t prob_to_qual(float p) {
    if (p == 1.0f) return 255u;
    const float s = __fmul_rn(p, 256.0f);
    return s >= 255.0f ? 255u : s > 0.0f ? (uint32_t)s : 0u;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(FULL, v, d); if (lane_id() >= d) v += t; }
    return v;
}
__device__ __forceinline__ unsigned long long warp_incl_scan64(unsigned long long v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(FULL, v, d); if (lane_id() >= d) v += t; }
    return v;
}

// count of nibbles equal to X in a 32-bit word of BAM 4-bit sequence
__device__ __forceinline__ uint32_t nib_eq_flags(uint32_t w, uint32_t X) {
    uint32_t x = w ^ (X * 0x11111111u);
    uint32_t t = (x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x11111111u;
    return t ^ 0x11111111u;  // bit 4n set where nibble n == X
}
// flags (bit 4n) -> 8-bit mask in base order (base j <-> nibble j^1 inside a little-endian word)
__device__ __forceinline__ uint32_t nib_flags_to_mask(uint32_t y) {
    y = (y | (y >> 3)) & 0x03030303u;
    y = (y | (y >> 6)) & 0x000F000Fu;
    y = (y | (y >> 12)) & 0xFFu;
    return ((y & 0x55u) << 1) | ((y & 0xAAu) >> 1);
}
__device__ __forceinline__ uint32_t seq_nibble(const uint8_t* seq, uint32_t q) {
    uint32_t b = seq[q >> 1];
    return (q & 1) ? (b & 0xf) : (b >> 4);
}
// BAM nibble -> 0..3 (A C G T) or 4
__device__ __forceinline__ int nib_to_base(uint32_t n) { return n == 1 ? 0 : n == 2 ? 1 : n == 4 ? 2 : n == 8 ? 3 : 4; }
__device__ __forceinline__ uint32_t base_to_nib(int b) { return 1u << b; }

__device__ __forceinline__ bool is_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

// ---- FxHashMap<ModCodeRepr,f32> iteration order (SURVEY Appendix B.1) -------------------------
__device__ __forceinline__ unsigned long long fx_hash_code(uint32_t c) {
    const unsigned long long K = 0x517cc1b727220a95ull;
    unsigned long long disc = (c & 0x80000000u) ? 1ull : 0ull;
    unsigned long long h = disc * K;                       // (rotl(0,5) ^ disc) * K
    unsigned long long v = (c & 0x80000000u) ? (unsigned long long)(c & 0x7fffffffu) : (unsigned long long)c;
    h = (((h << 5) | (h >> 59)) ^ v) * K;
    return h;
}

struct ProbMap {
    uint32_t code[MAX_MAP];
    float p[MAX_MAP];
    int8_t slot[8];   // slot -> item, -1 empty
    int n, nb;
    __device__ void init() { n = 0; nb = 4; for (int i = 0; i < 8; i++) slot[i] = -1; }
    __device__ __noinline__ void place(int item) {
        int s = (int)(fx_hash_code(code[item]) & (unsigned long long)(nb - 1));
        while (slot[s] >= 0) s = (s + 1) & (nb - 1);
        slot[s] = (int8_t)item;
    }
    // returns item index, or -1 on overflow
    __device__ __noinline__ int insert(uint32_t c, float v) {
        if (n >= MAX_MAP) return -1;
        if (nb == 4 && n + 1 > 3) {
            int8_t old[4];
            for (int i = 0; i < 4; i++) old[i] = slot[i];
            nb = 8;
            for (int i = 0; i < 8; i++) slot[i] = -1;
            for (int i = 0; i < 4; i++) if (old[i] >= 0) place(old[i]);
        }
        code[n] = c; p[n] = v;
        place(n);
        return n++;
    }
};

// ---- probabilities of one read position in insertion order (BaseModProbs) ---------------------------------------
struct Items {
    uint32_t code[MAX_MAP];
    float p[MAX_MAP];
    int n;
    __device__ __forceinline__ int find(uint32_t c) const { for (int i = 0; i < n; i++) if (code[i] == c) return i; return -1; }
    __device__ __forceinline__ bool push(uint32_t c, float v) { if (n >= MAX_MAP) return false; code[n] = c; p[n] = v; n++; return true; }
};
// low two bits of the Fx hash: K = 1 (mod 4), rotl(K,5) = 2 (mod 4)
__device__ __forceinline__ uint32_t bucket4(uint32_t c) { return (c & 0x80000000u) ? ((2u ^ c) & 3u) : (c & 3u); }
// ML byte -> probability, (b + 0.5) / 256 (mod_bam.rs). b + 0.5 is exact in float and 256 is a power of two, so the product
// by 2^-8 is the same real number as the quotient and rounds to the same bits, without a division.
__device__ __forceinline__ float ml_prob(uint32_t b) { return __fmul_rn(__fadd_rn((float)b, 0.5f), 0x1p-8f); }
// CollapseMethod::ReDistribute (src/mod_bam.rs:558-600) of at most two codes: the dropped code's probability is shared as
// marginal / (n_other + 1). With two codes that is p / 2, which p * 0.5 gives exactly (the same real number); when no code is
// dropped the share is 0 / k = +0, and p + 0 is p for every p >= 0, so that add is left out.
__device__ __forceinline__ float half_share(float p) { return __fmul_rn(p, 0.5f); }
__device__ __forceinline__ void redistribute2(uint32_t drop, uint32_t& c0, float& p0, uint32_t c1, float p1, int& n2c) {
    if (n2c == 1) { if (c0 == drop) n2c = 0; }
    else if (c0 == drop) { c0 = c1; p0 = __fadd_rn(p1, half_share(p0)); n2c = 1; }
    else if (c1 == drop) { p0 = __fadd_rn(p0, half_share(p1)); n2c = 1; }
}
__device__ __noinline__ void iter_order_slow(const Items& it, int* ord) {
    ProbMap m;
    m.init();
    for (int i = 0; i < it.n; i++) m.insert(it.code[i], it.p[i]);
    int k = 0;
    for (int s = 0; s < 8; s++) if (m.slot[s] >= 0) ord[k++] = m.slot[s];
}
// FxHashMap iteration order of the items (1 and 2 entries in closed form: 4 buckets, linear probing)
__device__ __forceinline__ void iter_order(const Items& it, int* ord) {
    if (it.n <= 1) { ord[0] = 0; return; }
    if (it.n == 2) {
        const uint32_t b0 = bucket4(it.code[0]), b1 = bucket4(it.code[1]);
        const bool swap = b0 != b1 ? (b1 < b0) : (b0 == 3);
        ord[0] = swap ? 1 : 0; ord[1] = swap ? 0 : 1;
        return;
    }
    iter_order_slow(it, ord);
}
__device__ __forceinline__ float items_sum(const Items& it, const int* ord) {
    float s = 0.f;
    for (int k = 0; k < it.n; k++) s = __fadd_rn(s, it.p[ord[k]]);
    return s;
}
// CollapseMethod::ReDistribute (src/mod_bam.rs:558-600)
__device__ __forceinline__ void redistribute_items(const Items& in, const int* ord, uint32_t drop, Items& out) {
    float marginal = 0.f;
    int n_other = 0;
    for (int k = 0; k < in.n; k++) { const int i = ord[k]; if (in.code[i] == drop) marginal = __fadd_rn(marginal, in.p[i]); else n_other++; }
    const float share = __fdiv_rn(marginal, __fadd_rn((float)n_other, 1.0f));
    out.n = 0;
    for (int k = 0; k < in.n; k++) { const int i = ord[k]; if (in.code[i] != drop) out.push(in.code[i], __fadd_rn(in.p[i], share)); }
}
// threshold of mod code c at canonical base tb: the code's own, else the base's any-mod ("C") one, else base_thr
__device__ __forceinline__ float mod_threshold(uint32_t c, int tb, float base_thr) {
    float thr = base_thr;
    if (c_par.n_mod_thr) {
        const uint32_t any_code = (uint32_t)("ACGT"[tb]);
        bool found = false;
        for (uint32_t t = 0; t < c_par.n_mod_thr && !found; t++) if (c_par.mod_code[t] == c) { thr = c_par.mod_thr[t]; found = true; }
        for (uint32_t t = 0; t < c_par.n_mod_thr && !found; t++) if (c_par.mod_code[t] == any_code) { thr = c_par.mod_thr[t]; found = true; }
    }
    return thr;
}
// MultipleThresholdModCaller::call (src/threshold_mod_caller.rs:28-63): 0 filtered, 1 canonical, 2 modified (*code)
__device__ __forceinline__ int make_call_items(const Items& it, const int* ord, int tb, uint32_t* code) {
    bool have = false;
    float best = 0.f;
    int kind = 0;
    const float base_thr = base_threshold(tb);
    for (int k = 0; k < it.n; k++) {
        const int i = ord[k];
        const uint32_t c = it.code[i];
        const float thr = mod_threshold(c, tb, base_thr);
        const float pm = it.p[i];
        if (pm >= thr && (!have || pm >= best)) { have = true; best = pm; kind = 2; *code = c; }
    }
    const float cp = __fsub_rn(1.0f, items_sum(it, ord));
    if (cp >= base_thr && (!have || cp >= best)) { have = true; kind = 1; }
    return have ? kind : 0;
}

// BaseModProbs::argmax_base_mod_call value (src/mod_bam.rs:489-505)
__device__ __forceinline__ float argmax_items(const Items& it, const int* ord) {
    const float cp = __fsub_rn(1.0f, items_sum(it, ord));
    bool have = false;
    float mp = 0.f;
    for (int k = 0; k < it.n; k++) { const float v = it.p[ord[k]]; if (!have || v >= mp) { have = true; mp = v; } }
    return (have && mp > cp) ? mp : cp;
}

// Registry of (primary base, mod code) states. A per-thread 4-entry cache keeps the hot path off the (single,
// heavily shared) global table: every warp asking L2 for the same sector serialises at one slice.
struct StateCache {      // two most recent (key -> id) pairs, in registers
    unsigned long long k0, k1;
    int i0, i1;
    __device__ void init() { k0 = k1 = ~0ull; i0 = i1 = 0; }
};

__device__ __noinline__ int state_id_global(unsigned long long* states, uint32_t* n_states, uint32_t* err, unsigned long long key) {
    for (int i = 0; i < MAX_STATES; i++) {
        unsigned long long v = *((volatile unsigned long long*)&states[i]);
        if (v == key) return i;
        if (v == ~0ull) {
            unsigned long long old = atomicCAS(&states[i], ~0ull, key);
            if (old == ~0ull) { atomicMax(n_states, (uint32_t)i + 1); return i; }
            if (old == key) return i;
        }
    }
    atomicOr(err, MKP_DERR_TOO_MANY_STATES);
    return 0;
}

__device__ __forceinline__ int state_id(const ChunkDev& C, StateCache& sc, int pb, uint32_t code) {
    const unsigned long long key = ((unsigned long long)pb << 32) | code;
    if (sc.k0 == key) return sc.i0;
    if (sc.k1 == key) return sc.i1;
    const int id = state_id_global(C.states, C.n_states, C.err, key);
    sc.k1 = sc.k0; sc.i1 = sc.i0; sc.k0 = key; sc.i0 = id;
    return id;
}

// per-warp parsed MM list table
struct ListTab {
    uint32_t d_start[MAX_LISTS];   // offset of the first delta byte (after the header comma), == d_end when no deltas
    uint32_t d_end[MAX_LISTS];
    uint32_t code[MAX_LISTS][MAX_LIST_CODES];
    uint32_t n_delta[MAX_LISTS];
    uint32_t ent_off[MAX_LISTS];
    uint32_t ml_off[MAX_LISTS];
    uint8_t base[MAX_LISTS];       // fundamental base char
    uint8_t strand[MAX_LISTS];     // 0 '+', 1 '-'
    uint8_t mode[MAX_LISTS];       // 0 '?', 1 '.', 2 default
    uint8_t ncodes[MAX_LISTS];
    uint32_t n;
    uint32_t tot[4];               // occurrences of nibble-base x in SEQ (query order)
};

enum { MODE_PILEUP = 0, MODE_HIST = 1 };

// per-read hand-over between k_parse and k_resolve (global memory; only the used records are touched)
struct ListRec { uint32_t n_delta, ent_off, ml_off; uint32_t code[MAX_LIST_CODES]; uint8_t base, strand, mode, ncodes; };   // 32 bytes
struct ReadLists { uint32_t n, ent, flags, pad; uint16_t imp_lists[8]; ListRec rec[MAX_LISTS]; };

// binary search: first index in sorted P[0..n) with value >= f
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* P, uint32_t n, uint32_t f) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (P[mid] < f) lo = mid + 1; else hi = mid; }
    return lo;
}

// Kernel A: per read, everything that depends only on the read's own bytes: admission, reference span, MM list
// discovery, per-base occurrence counts, MM token parse + select -> forward positions P[] and the list table.
// k_parse: 9 blocks of 128 threads = a limit of 56 registers; it takes 55 and does not spill. At 10 blocks (48 registers) it spills 72 / 100 bytes and takes
// 1.4 % longer on an H100; at 8 (63 registers, 32 warps per SM) it took 2 % longer (profiles/README.md)
#ifndef MKP_MINB_PARSE
#define MKP_MINB_PARSE 9
#endif
// fast k_resolve: 7 blocks of 128 threads = 72 registers, 140 / 80 bytes of spills. Before its loads were issued together, on an
// H100 it took 1.44 ms per pass on the profile chunk at 7 blocks, against 1.76 at 8 (64 registers) and 1.98 at 9
// (profiles/resolve_ptxas.txt, profiles/README.md)
#ifndef MKP_MINB_RESOLVE_FAST
#define MKP_MINB_RESOLVE_FAST 7
#endif
#ifndef MKP_MINB_RESOLVE
#define MKP_MINB_RESOLVE 7
#endif
// k_count_bases: 5 blocks of 256 threads = 48 registers, which leaves 32 bytes of spills (8 before it took work items; the launch
// bounds were not swept again). At 8 blocks (32 registers) its hot loop
// spilled 128 / 152 bytes and the kernel took 1.41x as long on an H100 (profiles/README.md); 4 blocks (64 registers, no spills) is
// slower than 5: the walk is latency bound and wants the warps
#ifndef MKP_MINB_BASES
#define MKP_MINB_BASES 5
#endif
// MKP_PARSE_CLOCKS=1 (measurement builds only): every warp of k_parse sums clock64() deltas per phase over the reads it handles
// and adds them into g_parse_clk at exit: [0] queue + header, [1] CIGAR span, [2] MM list scan, [3] alias compare, [4] delta
// tokenizer, [5] streaming select, [6] hand-over, [7] reads, [8] SEQ rounds of the select. Read back by mkp_debug_parse_clocks.
#ifdef MKP_PARSE_CLOCKS
constexpr int PCLK_N = 9;
__device__ unsigned long long g_parse_clk[PCLK_N];
// (the sums live in shared memory, so the measured kernel keeps the register budget of the default build)
#define PCLK_INIT __shared__ unsigned long long s_pclk[4][PCLK_N]; unsigned long long* pclk = s_pclk[wib]; \
    if (lane < PCLK_N) pclk[lane] = 0; __syncwarp(); unsigned long long pclk_t = clock64()
#define PCLK(k) do { const unsigned long long t_ = clock64(); if (lane == 0) pclk[k] += t_ - pclk_t; pclk_t = t_; } while (0)
#define PCLK_COUNT(k, n) do { if (lane == 0) pclk[k] += (n); } while (0)
#define PCLK_FLUSH do { __syncwarp(); if (lane < PCLK_N) atomicAdd(&g_parse_clk[lane], pclk[lane]); } while (0)
#else
#define PCLK_INIT do {} while (0)
#define PCLK(k) do {} while (0)
#define PCLK_COUNT(k, n) do {} while (0)
#define PCLK_FLUSH do {} while (0)
#endif
// MKP_RESOLVE_CLOCKS=1 (measurement builds only): every warp of the fast k_resolve<MODE_PILEUP> sums clock64() deltas per phase
// over the reads it handles and adds them into g_resolve_clk at exit: [0] queue + header + list table, [1] CIGAR prefix,
// [2] query -> op table, [3] per-entry resolve (ML -> call), [4] projection + emit, [5] commit, [6] reads, [7] list entries.
// Each round of 32 entries splits at the slowest lane's end of the call: lanes run the call and the projection in turn, and the
// warp moves on when its last lane is done. Read back by mkp_debug_resolve_clocks.
#ifdef MKP_RESOLVE_CLOCKS
constexpr int RCLK_N = 8;
__device__ unsigned long long g_resolve_clk[RCLK_N];
#define RCLK_ON (FAST_ONLY && MODE == MODE_PILEUP)
#define RCLK_INIT __shared__ unsigned long long s_rclk[4][RCLK_N]; unsigned long long* rclk = s_rclk[wib]; \
    if (lane < RCLK_N) rclk[lane] = 0; __syncwarp(); unsigned long long rclk_t = clock64(), rclk_mid = 0
#define RCLK(k) do { if (RCLK_ON) { const unsigned long long t_ = clock64(); if (lane == 0) rclk[k] += t_ - rclk_t; rclk_t = t_; } } while (0)
#define RCLK_COUNT(k, n) do { if (RCLK_ON && lane == 0) rclk[k] += (n); } while (0)
#define RCLK_MARK do { if (RCLK_ON) rclk_mid = clock64(); } while (0)
#define RCLK_ROUND do { if (RCLK_ON) { \
    const unsigned long long t_ = clock64(); \
    const uint32_t d_ = __reduce_max_sync(FULL, rclk_mid > rclk_t ? (uint32_t)min(rclk_mid - rclk_t, t_ - rclk_t) : 0u); \
    if (lane == 0) { rclk[3] += d_; rclk[4] += t_ - rclk_t - d_; } rclk_t = t_; rclk_mid = 0; } } while (0)
#define RCLK_FLUSH do { if (RCLK_ON) { __syncwarp(); if (lane < RCLK_N) atomicAdd(&g_resolve_clk[lane], rclk[lane]); } } while (0)
#else
#define RCLK_INIT do {} while (0)
#define RCLK(k) do {} while (0)
#define RCLK_COUNT(k, n) do {} while (0)
#define RCLK_MARK do {} while (0)
#define RCLK_ROUND do {} while (0)
#define RCLK_FLUSH do {} while (0)
#endif
// SEQ per lane and round of k_parse's streaming select, in uint4 (32 bases each). On an H100, 2 took 1.95 ms per pass on the
// profile chunk and 4 took 2.07 (profiles/README.md): wider blocks cost more in the token lookup than they save in rounds.
constexpr int SEL_Q = 2;
__global__ void __launch_bounds__(128, MKP_MINB_PARSE) k_parse(ChunkDev C) {
    __shared__ ListTab s_tab[4];
    __shared__ __align__(16) uint8_t s_txt[4][160];
    __shared__ uint8_t s_tok[4][132];
    __shared__ uint32_t s_cb[4][32], s_tp[4][MAX_LISTS];
    __shared__ uint4 s_fq[SEL_Q][4][32];
    __shared__ uint32_t s_val[4][96];
    const uint32_t lane = lane_id();
    const uint32_t wib = threadIdx.x >> 5;
    ListTab& T = s_tab[wib];
    PCLK_INIT;

    for (;;) {
        // dynamic work distribution: reads differ in length by 2-3 orders of magnitude
        uint32_t ri = 0;
        if (lane == 0) {
            ri = atomicAdd(C.work, 1u);
            if (C.list_mode == 1) ri = ri < C.work[4] ? C.slow_list[ri] : 0xffffffffu;
            else if (C.order && ri < C.n_reads) ri = C.order[ri];
        }
        ri = __shfl_sync(FULL, ri, 0);
        if (ri >= C.n_reads) { PCLK(0); break; }
        PCLK_COUNT(7, 1);
        const mkp_read_hdr h = C.hdrs[ri];
        const uint32_t flag = h.flags & 0xffffu;
        const uint32_t L = h.l_seq;
        const bool rev = flag & 0x10;
        ReadMeta meta;
        meta.ref_end = h.ref_start;
        meta.flags = 0; meta.pos_mask = 0; meta.neg_mask = 0; meta.n_calls = 0; meta.n_hist = 0; meta.imp[0] = 0; meta.imp[1] = 0;
        meta.entry_off = C.entry_off[ri];
        bool admitted;
        if (C.mode == MODE_PILEUP) admitted = !(flag & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)) && L > 0;
        else admitted = !(flag & (0x100 | 0x400 | 0x800)) && L > 0 && (C.take == nullptr || C.take[ri]) &&
                        !((flag & 0x4) && (!C.hist_include_unaligned || c_par.edge_on));
        if (!admitted) { if (lane == 0) { C.meta[ri] = meta; C.rl[ri].n = 0; C.rl[ri].flags = 1; } PCLK(0); continue; }
        PCLK(0);
        meta.flags = 1;
        const uint32_t* cig = (const uint32_t*)(C.heap + h.off);
        const uint8_t* seq = C.heap + h.off + 4ull * h.n_cigar;
        const uint8_t* ml = seq + ((L + 1) >> 1);
        const uint8_t* mm = ml + h.len_ml;
        // ---- phase 0: reference span (k_resolve builds the per-op prefix; here only the end is needed) ----
        {
            uint32_t rsum = 0;
#pragma unroll 4
            for (uint32_t i = lane; i < h.n_cigar; i += 32) {
                const uint32_t c = cig[i];
                rsum += cig_rlen(c & 15, c >> 4);
            }
            meta.ref_end = (int32_t)((uint32_t)h.ref_start + __reduce_add_sync(FULL, rsum));
        }
        PCLK(1);
        bool err = (h.flags & MKP_RF_TAGS_INVALID) != 0;
        // ---- phase 1: list discovery: warp-parallel scan for ';' and the first ',' of each part; the few
        //      header bytes of each part are parsed by lane 0 (src/mod_bam.rs:900-1000) ------------------
        {
            const uint32_t M = h.len_mm;
            uint32_t n = 0, seg = 0, hdr_end = 0xffffffffu;   // uniform across the warp
            bool e0 = false;                                   // lane 0 only
            auto close_part = [&](uint32_t j) {                // part = mm[seg..j)
                if (j > seg) {
                    if (n >= MAX_LISTS) { if (lane == 0) { atomicOr(C.err, MKP_DERR_TOO_MANY_LISTS); e0 = true; } }
                    else if (lane == 0 && !e0) {
                        const uint32_t hl = hdr_end == 0xffffffffu ? j : hdr_end;
                        uint32_t k = seg;
                        const uint8_t fb = mm[k];
                        bool e = !(fb == 'A' || fb == 'C' || fb == 'G' || fb == 'T' || fb == 'U' || fb == 'N');
                        k++;
                        uint8_t st = 0;
                        if (!e) { if (k >= hl) e = true; else { st = mm[k]; if (st != '+' && st != '-') e = true; k++; } }
                        uint32_t nc = 0;
                        bool seen_chebi = false;
                        int mode = 2;
                        if (!e && k < hl && is_digit(mm[k])) {
                            unsigned long long v = 0;
                            while (k < hl && is_digit(mm[k])) { v = v * 10 + (mm[k] - '0'); if (v > 0x7fffffffull) { e = true; break; } k++; }
                            T.code[n][nc++] = 0x80000000u | (uint32_t)v;
                            seen_chebi = true;
                        }
                        for (; !e && k < hl; k++) {
                            const uint8_t c = mm[k];
                            if (c == '?') mode = 0;
                            else if (c == '.') mode = 1;
                            else if (is_digit(c) || seen_chebi || c >= 0x80) e = true;   // (a non-ASCII header is a read error)
                            else if (nc >= MAX_LIST_CODES) { atomicOr(C.err, MKP_DERR_TOO_MANY_CODES); e = true; }
                            else T.code[n][nc++] = c;
                        }
                        if (nc == 0) e = true;
                        T.base[n] = fb; T.strand[n] = st == '-'; T.mode[n] = (uint8_t)mode; T.ncodes[n] = (uint8_t)nc;
                        // delta text mm[d_start..d_end) starts right after the header comma; n_delta = 0xffffffff marks
                        // "a comma follows the header, so at least one number must parse" (nom separated_list1)
                        if (hl < j) { T.d_start[n] = hl + 1; T.d_end[n] = j; T.n_delta[n] = 0xffffffffu; }
                        else { T.d_start[n] = j; T.d_end[n] = j; T.n_delta[n] = 0u; }
                        if (e) e0 = true;
                    }
                    if (n < MAX_LISTS) n++;
                }
                seg = j + 1;
                hdr_end = 0xffffffffu;
            };
            // four text bytes per lane (one aligned word), 128 per round; SWAR byte compare gives a 0x80 flag per
            // matching byte, the first flagged byte at or after a given offset is a warp min-reduction
            const int iM = (int)M;
            for (int c0 = -(int)((uintptr_t)mm & 3u); c0 < iM && !err; c0 += 128) {
                const int g0 = c0 + 4 * (int)lane;
                uint32_t zs = 0, zc = 0;
                if (g0 < iM && g0 + 4 > 0) {
                    const uint32_t w = *(const uint32_t*)(mm + g0);
                    const uint32_t xs = w ^ 0x3b3b3b3bu, xc = w ^ 0x2c2c2c2cu;
                    zs = ~(((xs & 0x7f7f7f7fu) + 0x7f7f7f7fu) | xs | 0x7f7f7f7fu);
                    zc = ~(((xc & 0x7f7f7f7fu) + 0x7f7f7f7fu) | xc | 0x7f7f7f7fu);
                    uint32_t keepm = 0xffffffffu;
                    if (g0 < 0) keepm &= 0xffffffffu << (8 * (-g0));
                    if (g0 + 4 > iM) keepm &= 0xffffffffu >> (8 * (g0 + 4 - iM));
                    zs &= keepm; zc &= keepm;
                }
                if (hdr_end != 0xffffffffu && !__any_sync(FULL, zs != 0)) continue;
                // offset (0..127 in this round, 128 = none) of the first flagged byte at or after offset t
                auto first_from = [&](uint32_t z, uint32_t t) -> uint32_t {
                    const uint32_t lb = 4 * lane;
                    if (t > lb) z = t - lb >= 4 ? 0u : (z & (0xffffffffu << (8 * (t - lb))));
                    const uint32_t cand = z ? lb + (((uint32_t)__ffs(z) - 1u) >> 3) : 128u;
                    return __reduce_min_sync(FULL, cand);
                };
                uint32_t lo = 0;
                while (lo < 128) {
                    const uint32_t sp = first_from(zs, lo);
                    if (hdr_end == 0xffffffffu) { const uint32_t cp = first_from(zc, lo); if (cp < sp) hdr_end = (uint32_t)(c0 + (int)cp); }
                    if (sp == 128) break;
                    close_part((uint32_t)(c0 + (int)sp));
                    lo = sp + 1;
                }
            }
            if (!err && seg < M) close_part(M);
            if (__shfl_sync(FULL, e0 ? 1 : 0, 0)) err = true;
            if (lane == 0) T.n = err ? 0xffffffffu : n;
        }
        __syncwarp();
        if (T.n == 0xffffffffu) err = true;
        const uint32_t nl = err ? 0 : T.n;
        // ---- which bases need rank/select over the SEQ (query-order nibble index x: 0..3 = A C G T as stored) ----
        uint32_t need = 0;
        for (uint32_t l = 0; l < nl; l++) {
            uint8_t fb = T.base[l];
            if (fb == 'N') continue;
            int b = fb == 'A' ? 0 : fb == 'C' ? 1 : fb == 'G' ? 2 : 3;
            int x = rev ? 3 - b : b;
            need |= 1u << x;
        }
        if (lane < 4) T.tot[lane] = 0;
        __syncwarp();
        // ---- phase 3: tokens -> forward positions ------------------------------------------------------
        uint32_t* P = C.P + meta.entry_off;
        uint32_t ent = 0, mlp = 0;
        uint32_t alias_mask = 0;              // lists that share the entries of the list before them
        PCLK(2);
        for (uint32_t l = 0; l < nl && !err; l++) {
            const uint32_t ds = T.d_start[l], de = T.d_end[l];
            const bool must = T.n_delta[l] == 0xffffffffu;
            unsigned long long carry = 0;     // sum of (d+1) so far
            uint32_t ntok = 0;
            // A list whose delta text repeats the previous list's byte for byte, on the same base (basecallers write one
            // delta list per code: C+h?,...;C+m?,...), has the same tokens, occurrence indices and positions: it shares the
            // previous list's entries instead of being tokenised and selected again.
            if (l > 0 && must && de > ds && T.base[l] == T.base[l - 1] && de - ds == T.d_end[l - 1] - T.d_start[l - 1] && T.n_delta[l - 1] > 0) {
                const uint32_t pds = T.d_start[l - 1], len = de - ds;
                bool same = true;
                for (uint32_t c0 = 0; c0 < len && same; c0 += 128) {
                    bool eq = true;
#pragma unroll
                    for (int t = 0; t < 4; t++) { const uint32_t i = c0 + 32 * t + lane; if (i < len && mm[ds + i] != mm[pds + i]) eq = false; }
                    same = __all_sync(FULL, eq);
                }
                if (same) {
                    ntok = T.n_delta[l - 1];
                    const uint32_t shared = T.ent_off[l - 1];
                    __syncwarp();
                    if (lane == 0) { T.n_delta[l] = ntok; T.ent_off[l] = shared; T.ml_off[l] = mlp; }
                    if ((unsigned long long)mlp + (unsigned long long)ntok * T.ncodes[l] > (unsigned long long)h.len_ml) err = true;
                    mlp += ntok * T.ncodes[l];
                    alias_mask |= 1u << l;
                    __syncwarp();
                    PCLK(3);
                    continue;
                }
            }
            PCLK(3);
            // delta values of up to 32 tokens (one per lane, `mine` lanes in token order) -> forward positions P[]
            // delta values of up to 32 tokens (one per lane, `mine` lanes in token order) -> 0-based occurrence index of the
            // list's base in forward-read order (for 'N' lists that already is the forward position); stored in P[] and
            // turned into positions by the streaming pass below
            auto place = [&](unsigned long long val, bool mine, uint32_t keep_mask) {
                const unsigned long long inc = mine ? (val + 1ull) : 0ull;
                const unsigned long long pre = warp_incl_scan64(inc);
                const uint32_t idx = ntok + __popc(keep_mask & ((1u << lane) - 1u));
                bool bad = false;
                if (mine) {
                    const unsigned long long k = carry + pre - 1ull;
                    if (k >= (unsigned long long)L || ent + idx >= h.len_ml) bad = true;   // past the last base whatever the base is; more tokens than ML entries is an error anyway (and P has len_ml slots)
                    else P[ent + idx] = (uint32_t)k;
                }
                if (__any_sync(FULL, bad)) err = true;
                carry += __shfl_sync(FULL, pre, 31);
                ntok += __popc(keep_mask);
            };
            // ---- fast path: the text is exactly digits(,digits)* with <= 9 digits per number. Four text bytes per lane
            //      (one aligned word), 128 per round. The number in progress is an affine map v -> 10 v + d (reset at
            //      ','): every lane composes its four bytes, a TRUNCATED warp scan (distance 1 and 2: three lanes = 12
            //      bytes back) gives the value / digit count entering the lane, which is exact for numbers of <= 9
            //      digits, and any 10th digit is seen by the same window and sends the list to the exact path.
            //      Finished numbers (<= 2 per lane) are compacted into a queue and placed 32 at a time. Anything else
            //      (white space, empty or over-long tokens, other bytes) falls back to the exact path below.
            bool slow = false;
            if (must) {
                uint32_t* qv = s_val[wib];
                uint32_t qn = 0, v_carry = 0, nd_carry = 0;
                const int ids = (int)ds, ide = (int)de;
                for (int c0 = ids - (int)((uintptr_t)(mm + ds) & 3u); c0 < ide && !slow && !err; c0 += 128) {
                    const int g0 = c0 + 4 * (int)lane;
                    const uint32_t w = g0 < ide ? *(const uint32_t*)(mm + g0) : 0u;
                    uint32_t nb = __shfl_down_sync(FULL, w, 1) & 0xffu;
                    if (lane == 31) nb = g0 + 4 < ide ? mm[g0 + 4] : 0u;
                    const uint32_t wn = (w >> 8) | (nb << 24);        // byte j = the byte after byte j of w
                    bool odd = false;
                    uint32_t A = 1, B = 0, R = 1u << 16;              // v_out = A v_in + B; R = carries_in << 16 | digits
                    uint32_t dm = 0, cm = 0, em = 0;                  // per byte: digit, comma, last digit of a number
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int g = g0 + j;
                        const bool in = g >= ids && g < ide, nin = g + 1 < ide;
                        const uint32_t ch = (w >> (8 * j)) & 0xffu, nx = (wn >> (8 * j)) & 0xffu;
                        const bool dig = in && (ch - '0') < 10u, com = in && ch == ',';
                        // anomalies: a byte that is neither digit nor comma; an empty token (comma at the very start,
                        // before another comma, or at the very end)
                        if (in && !dig && !com) odd = true;
                        if (com && (!nin || nx == ',' || g == ids)) odd = true;
                        if (dig) { B = B * 10u + (ch - '0'); A *= 10u; R += 1u; dm |= 1u << j; if (!nin || nx == ',') em |= 1u << j; }
                        if (com) { A = 0; B = 0; R = 0; cm |= 1u << j; }
                    }
                    if (lane == 0) { B = A * v_carry + B; if (R >> 16) R += nd_carry; A = 0; R &= 0xffffu; }   // absorb the carry
#pragma unroll
                    for (int d = 1; d <= 2; d <<= 1) {
                        const uint32_t pA = __shfl_up_sync(FULL, A, d), pB = __shfl_up_sync(FULL, B, d), pR = __shfl_up_sync(FULL, R, d);
                        if (lane >= (uint32_t)d) { B = A * pB + B; A = A * pA; if (R >> 16) R = pR + (R & 0xffffu); }
                    }
                    uint32_t v = __shfl_up_sync(FULL, B, 1), n = __shfl_up_sync(FULL, R, 1) & 0xffffu;   // entering this lane
                    if (lane == 0) { v = v_carry; n = nd_carry; }
                    uint32_t e0 = 0, e1 = 0, ec = 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        if ((dm >> j) & 1u) {
                            v = v * 10u + (((w >> (8 * j)) & 0xffu) - '0'); n++;
                            if (n > 9) odd = true;
                            if ((em >> j) & 1u) { if (ec == 0) e0 = v; else e1 = v; ec++; }
                        } else if ((cm >> j) & 1u) { v = 0; n = 0; }
                    }
                    if (__any_sync(FULL, odd)) { slow = true; break; }
                    const uint32_t m1 = __ballot_sync(FULL, ec >= 1), m2 = __ballot_sync(FULL, ec == 2);
                    const uint32_t lt = (1u << lane) - 1u;
                    const uint32_t at = qn + __popc(m1 & lt) + __popc(m2 & lt);
                    if (ec >= 1) qv[at] = e0;
                    if (ec == 2) qv[at + 1] = e1;
                    qn += __popc(m1) + __popc(m2);
                    v_carry = __shfl_sync(FULL, v, 31); nd_carry = __shfl_sync(FULL, n, 31);
                    __syncwarp();
                    uint32_t qh = 0;
                    while (qn - qh >= 32 && !err) { place(qv[qh + lane], true, FULL); qh += 32; }
                    if (qh) {
                        const uint32_t rest = qn - qh;
                        const uint32_t mv = lane < rest ? qv[qh + lane] : 0;
                        __syncwarp();
                        if (lane < rest) qv[lane] = mv;
                        qn = rest;
                        __syncwarp();
                    }
                }
                if (!slow && !err && qn) { const bool mine = lane < qn; place(mine ? qv[lane] : 0, mine, qn >= 32 ? FULL : ((1u << qn) - 1u)); }
                if (!slow && !err && ntok == 0) slow = true;         // (empty text: let the exact path raise the error)
            }
            if (slow) { carry = 0; ntok = 0; }
            bool stop = false;                // list truncated by a malformed token
            // ---- exact path. Tokens start after every ',' of mm[ds-1 .. de) (mm[ds-1] is the header comma); grammar per
            // token: ws* digit+ ws* (nom separated_list1). 128 text bytes per round are staged in shared memory, the
            // token starts are compacted, then every lane parses one token.
            uint8_t* txt = s_txt[wib];
            uint8_t* tok = s_tok[wib];
            for (uint32_t c0 = ds - 1; must && slow && c0 < de && !stop && !err; c0 += 128) {
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 5; k++) { const uint32_t o = lane + 32 * k, g = c0 + o; txt[o] = g < de ? mm[g] : 0; }
                __syncwarp();
                // commas among the first 128 staged bytes (only those before `de`)
                const uint32_t w4 = ((const uint32_t*)txt)[lane];
                const uint32_t xr = w4 ^ 0x2c2c2c2cu;
                uint32_t zf = ~(((xr & 0x7f7f7f7fu) + 0x7f7f7f7fu) | xr | 0x7f7f7f7fu);   // 0x80 in every byte that is ','
                const uint32_t nvalid = de - c0;                                           // staged bytes that are text
                if (4 * lane + 4 > nvalid) { const uint32_t keepb = nvalid > 4 * lane ? nvalid - 4 * lane : 0; zf &= keepb ? (0xffffffffu >> (8 * (4 - keepb))) : 0u; }
                const uint32_t ncom = __popc(zf);
                const uint32_t incl = warp_incl_scan(ncom);
                uint32_t at = incl - ncom;
                while (zf) { const uint32_t bi = (uint32_t)(__ffs(zf) - 1) >> 3; zf &= zf - 1; tok[at++] = (uint8_t)(4 * lane + bi + 1); }
                const uint32_t nt = __shfl_sync(FULL, incl, 31);
                __syncwarp();
                for (uint32_t g0 = 0; g0 < nt && !stop && !err; g0 += 32) {
                    const bool starts = g0 + lane < nt;
                    unsigned long long val = 0;
                    bool ok_start = false, clean = false;
                    if (starts) {
                        uint32_t k = tok[g0 + lane];                      // offset in the staged text; text ends at nvalid
                        auto chr = [&](uint32_t o) -> uint8_t { return o < 160 ? txt[o] : mm[c0 + o]; };
                        while (k < nvalid && is_ws(chr(k))) k++;
                        const uint32_t d0 = k;
                        while (k < nvalid && is_digit(chr(k))) { val = val * 10 + (chr(k) - '0'); if (val > 0xffffffffull) val = 0x1ffffffffull; k++; }
                        ok_start = k > d0;                                 // a number above u32 keeps its place (clamped to 2^33 - 1): place() fails the read
                        while (k < nvalid && is_ws(chr(k))) k++;
                        clean = (k >= nvalid) || (chr(k) == ',');
                    }
                    const uint32_t m_start = __ballot_sync(FULL, starts);
                    const uint32_t m_badstart = __ballot_sync(FULL, starts && !ok_start);
                    const uint32_t m_dirty = __ballot_sync(FULL, starts && ok_start && !clean);
                    // first terminating token: a bad start excludes itself, a dirty end includes itself
                    const uint32_t first_bad = m_badstart ? (uint32_t)__ffs(m_badstart) - 1 : 32;
                    const uint32_t first_dirty = m_dirty ? (uint32_t)__ffs(m_dirty) - 1 : 32;
                    uint32_t keep_mask = m_start;
                    if (first_bad < 32 || first_dirty < 32) {
                        stop = true;
                        const uint32_t cut = first_bad <= first_dirty ? first_bad : first_dirty + 1;   // lanes < cut are kept
                        keep_mask &= cut >= 32 ? FULL : ((1u << cut) - 1u);
                    }
                    if (ntok == 0 && g0 == 0 && !(keep_mask & 1u)) err = true;             // the first token must parse
                    place(val, (keep_mask >> lane) & 1u, keep_mask);
                }
            }
            if (must && ntok == 0) err = true;
            // N lists: the reference checks only deltas after the first against the sequence length; the first
            // then panics on indexing, which we turn into a read error (handled by `bad` above).
            __syncwarp();
            if (lane == 0) { T.n_delta[l] = ntok; T.ent_off[l] = ent; T.ml_off[l] = mlp; }
            if ((unsigned long long)mlp + (unsigned long long)ntok * T.ncodes[l] > (unsigned long long)h.len_ml) err = true;
            mlp += ntok * T.ncodes[l];
            ent += ntok;
            __syncwarp();
            PCLK(4);
        }
        // ---- streaming select: for every needed base, one pass over the SEQ in forward-read order during which the tokens of
        //      all lists of that base are placed. The SEQ is read in blocks of SEL_Q uint4 (32 SEL_Q bases) of the 16-byte
        //      aligned grid that holds it (block b starts at query base 32 SEL_Q b - 2 a, a = seq & 15), one block per lane and
        //      32 per round; only the first and the last round mask the bytes outside the SEQ. Per lane: the nibble-equality
        //      flags (bit 4n) of its words and a warp scan of their popcounts. A token with occurrence index k lands in the
        //      block whose running count brackets k (5-step search over the 32 counts in shared memory), at the (k - count)-th
        //      match of the block, looked up in the one word that holds it. The pass is bound by instruction issue, not by its
        //      loads, so the blocks are as wide as the registers allow: every round pays one scan and one token placement.
        if (!err && need) {
            const uint32_t a16 = (uint32_t)((uintptr_t)seq & 15u);
            const uint4* seq4 = (const uint4*)(seq - a16);
            const uint32_t s_end = a16 + ((L + 1) >> 1);                 // the SEQ is bytes [a16, s_end) of the grid
            const uint32_t nb = (s_end + 16 * SEL_Q - 1) / (16 * SEL_Q);
            for (int x = 0; x < 4 && !err; x++) {
                if (!(need & (1u << x))) continue;
                const int bfw = rev ? 3 - x : x;                        // forward base of this nibble
                uint32_t lists = 0;                                      // lists whose base is bfw
                for (uint32_t l = 0; l < nl; l++) {
                    const uint8_t fb = T.base[l];
                    const int b = fb == 'A' ? 0 : fb == 'C' ? 1 : fb == 'G' ? 2 : (fb == 'T' || fb == 'U') ? 3 : 4;
                    if (b == bfw) lists |= 1u << l;
                }
                lists &= ~alias_mask;                                    // shared entries are placed once, by their first list
                if (lane < MAX_LISTS) s_tp[wib][lane] = 0;
                __syncwarp();
                // The first list of the base keeps its window of 32 occurrence indices in registers (wv, one per lane) across
                // rounds; P is read again only when a window has been placed. Other lists of the base (their deltas differ from
                // it) read theirs from P every round.
                const uint32_t n0 = lists ? T.n_delta[__ffs(lists) - 1] : 0u;
                uint32_t* K0 = P + (lists ? T.ent_off[__ffs(lists) - 1] : 0u);
                const uint32_t rest = lists & (lists - 1u);
                uint32_t wt = 0, tp0 = 0;                                // the window's first token; tokens placed
                uint32_t wv = lane < n0 ? K0[lane] : 0u;
                uint32_t run = 0;                                        // occurrences in the blocks already streamed
                for (uint32_t i0 = 0; i0 < nb; i0 += 32) {
                    const uint32_t bi = i0 + lane;                       // index in streaming (forward-read) order
                    const uint32_t blk = rev ? nb - 1u - bi : bi;        // block in query order
                    uint4 qv[SEL_Q];                                     // (a uint4 wholly past the SEQ is not read)
#pragma unroll
                    for (int h = 0; h < SEL_Q; h++) qv[h] = bi < nb && 16u * (SEL_Q * blk + h) < s_end ? seq4[SEL_Q * blk + h] : make_uint4(0u, 0u, 0u, 0u);
                    const bool edge = i0 == 0 || i0 + 32 >= nb;          // first / last round: bytes of the grid outside the SEQ
                    uint32_t cnt = 0;
#pragma unroll
                    for (int h = 0; h < SEL_Q; h++) {
                        uint32_t f[4] = {qv[h].x, qv[h].y, qv[h].z, qv[h].w};
                        if (edge) {
#pragma unroll
                            for (int w = 0; w < 4; w++) {
                                const uint32_t g = 16u * (SEL_Q * blk + h) + 4u * w;   // grid offset of the word (lanes past the end hold zeros)
                                if (g < a16) f[w] &= a16 - g >= 4 ? 0u : 0xffffffffu << (8 * (a16 - g));
                                if (g + 4 > s_end) f[w] &= g >= s_end ? 0u : 0xffffffffu >> (8 * (g + 4 - s_end));
                            }
                        }
#pragma unroll
                        for (int w = 0; w < 4; w++) { f[w] = nib_eq_flags(f[w], 1u << x); cnt += __popc(f[w]); }   // a zero nibble matches no base
                        s_fq[h][wib][lane] = make_uint4(f[0], f[1], f[2], f[3]);
                    }
                    const uint32_t incl = warp_incl_scan(cnt);
                    s_cb[wib][lane] = run + incl - cnt;
                    const uint32_t hi = run + __shfl_sync(FULL, incl, 31);      // tokens with index in [run, hi) live here
                    __syncwarp();
                    auto select = [&](uint32_t k) -> uint32_t {          // forward position of occurrence k, run <= k < hi
                        uint32_t lo = 0, hb = 32;                        // largest b with s_cb[b] <= k
#pragma unroll
                        for (int st = 0; st < 5; st++) { const uint32_t mid = (lo + hb) >> 1; if (s_cb[wib][mid] <= k) lo = mid; else hb = mid; }
                        const uint32_t c_lo = s_cb[wib][lo];
                        uint32_t within = k - c_lo;
                        if (rev) within = (lo < 31 ? s_cb[wib][lo + 1] : hi) - c_lo - 1u - within;   // forward order runs down the query
                        uint4 fl = s_fq[0][wib][lo];
                        uint32_t pos = 0;
#pragma unroll
                        for (int h = 1; h < SEL_Q; h++) {                // (once found, within stays below the count)
                            const uint32_t c = __popc(fl.x) + __popc(fl.y) + __popc(fl.z) + __popc(fl.w);
                            if (within >= c) { within -= c; pos += 32; fl = s_fq[h][wib][lo]; }
                        }
                        const uint32_t c0 = __popc(fl.x), c1 = __popc(fl.y), c2 = __popc(fl.z);
                        uint32_t y = fl.x;
                        if (within >= c0) {
                            within -= c0; y = fl.y; pos += 8;
                            if (within >= c1) {
                                within -= c1; y = fl.z; pos += 8;
                                if (within >= c2) { within -= c2; y = fl.w; pos += 8; }
                            }
                        }
                        uint32_t msk = nib_flags_to_mask(y), c;          // the word's 8 bases in base order
                        c = __popc(msk & 0xfu); if (within >= c) { within -= c; pos += 4; msk >>= 4; }
                        c = __popc(msk & 0x3u); if (within >= c) { within -= c; pos += 2; msk >>= 2; }
                        c = msk & 1u;           if (within >= c) { pos += 1; }
                        const uint32_t bq = rev ? nb - 1u - (i0 + lo) : i0 + lo;
                        const uint32_t q = bq * (32u * SEL_Q) + pos - 2u * a16;
                        return rev ? L - 1u - q : q;
                    };
                    while (tp0 < n0) {
                        const uint32_t t = wt + lane;
                        const bool in = t >= tp0 && t < n0 && wv < hi;
                        if (in) K0[t] = select(wv);
                        tp0 += __popc(__ballot_sync(FULL, in));
                        if (tp0 < wt + 32u) break;                       // the rest of the window lies in later rounds
                        wt += 32u;
                        wv = wt + lane < n0 ? K0[wt + lane] : 0u;
                    }
                    uint32_t ls = rest;
                    while (ls) {
                        const uint32_t l = __ffs(ls) - 1;
                        ls &= ls - 1;
                        const uint32_t n = T.n_delta[l];
                        uint32_t* Kp = P + T.ent_off[l];
                        uint32_t tp = s_tp[wib][l];
                        while (tp < n) {
                            const uint32_t t = tp + lane;
                            const uint32_t kv = t < n ? Kp[t] : 0xffffffffu;
                            const bool in = t < n && kv < hi;
                            if (in) Kp[t] = select(kv);
                            const uint32_t c_in = __popc(__ballot_sync(FULL, in));
                            tp += c_in;
                            if (c_in < 32) break;
                        }
                        __syncwarp();
                        if (lane == 0) s_tp[wib][l] = tp;
                    }
                    run = hi;
                    __syncwarp();
                    PCLK_COUNT(8, 1);
                }
                if (lane == 0) T.tot[x] = run;
                // a token left unplaced refers to an occurrence past the end of the read (mod_bam.rs:705-727)
                if (tp0 < n0) err = true;
                uint32_t ls = rest;
                while (ls) { const uint32_t l = __ffs(ls) - 1; ls &= ls - 1; if (s_tp[wib][l] < T.n_delta[l]) err = true; }
                __syncwarp();
            }
        }
        __syncwarp();
        PCLK(5);
        // '.'/default-mode lists (src/read_cache.rs:122-137, src/mod_bam.rs:1041-1043, 1265-1292)
        bool any_entries = ent > 0;
        uint32_t imp_lists[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};   // lists that infer canonical on (strand, base)
        if (!err) {
            for (uint32_t l = 0; l < nl; l++) {
                const uint8_t md = T.mode[l];
                if (md == 0) continue;
                const uint8_t bl = T.base[l] == 'U' ? 'T' : T.base[l];
                bool contributes;
                if (bl == 'N') contributes = T.n_delta[l] > 0;
                else { int b = bl == 'A' ? 0 : bl == 'C' ? 1 : bl == 'G' ? 2 : 3; contributes = T.tot[rev ? 3 - b : b] > 0; }
                if (!contributes) continue;
                // the (strand, base) table keeps the default mode only if every contributing list has it
                bool all_default = md == 2;
                for (uint32_t l2 = 0; l2 < nl && all_default; l2++) {
                    if (l2 == l || T.strand[l2] != T.strand[l]) continue;
                    const uint8_t b2 = T.base[l2] == 'U' ? 'T' : T.base[l2];
                    if (b2 != bl && !(b2 == 'N' && T.n_delta[l2] > 0) && bl != 'N') continue;
                    if (T.mode[l2] != 2 && (T.n_delta[l2] > 0 || T.mode[l2] == 1)) all_default = false;
                }
                if (all_default && !c_par.force_allow_implicit) { err = true; break; }   // InvalidImplicitMode: read skipped
                if (bl == 'N') continue;      // N lists get no implicit fill
                { int b = bl == 'A' ? 0 : bl == 'C' ? 1 : bl == 'G' ? 2 : 3; imp_lists[T.strand[l]][b] |= 1u << l; any_entries = true; }
            }
        }
        // ---- hand-over to k_resolve: list table (only the used records), implicit-table masks, flags -------
        __syncwarp();
        {
            ReadLists* R = C.rl + ri;
            if (lane == 0) {
                R->n = nl; R->ent = ent; R->flags = (err ? 1u : 0u) | (any_entries ? 2u : 0u);
                for (int k = 0; k < 8; k++) R->imp_lists[k] = (uint16_t)imp_lists[k >> 2][k & 3];
                C.meta[ri] = meta;
            }
            if (lane < nl) {
                ListRec rec;
                rec.n_delta = T.n_delta[lane]; rec.ent_off = T.ent_off[lane]; rec.ml_off = T.ml_off[lane];
                for (int c = 0; c < MAX_LIST_CODES; c++) rec.code[c] = T.code[lane][c];
                rec.base = T.base[lane]; rec.strand = T.strand[lane]; rec.mode = T.mode[lane]; rec.ncodes = T.ncodes[lane];
                R->rec[lane] = rec;
            }
        }
        __syncwarp();
        PCLK(6);
    }
    PCLK_FLUSH;
}

// canonical base of implicit table sb (mod strand sb >> 2, forward base sb & 3)
__device__ __forceinline__ int table_base(int sb) { return (sb >> 2) == 0 ? (sb & 3) : 3 - (sb & 3); }

// the read's list table, handed over by k_parse, into the warp's shared copy
__device__ __forceinline__ void load_list_table(ListTab& T, const ReadLists* R, uint32_t nl, uint32_t lane) {
    __syncwarp();
    if (lane < nl) {
        const ListRec rec = R->rec[lane];
        T.n_delta[lane] = rec.n_delta; T.ent_off[lane] = rec.ent_off; T.ml_off[lane] = rec.ml_off;
        for (int c = 0; c < MAX_LIST_CODES; c++) T.code[lane][c] = rec.code[c];
        T.base[lane] = rec.base; T.strand[lane] = rec.strand; T.mode[lane] = rec.mode; T.ncodes[lane] = rec.ncodes;
    }
    __syncwarp();
}

// register-only path: no implicit tables, no 'N' list, and per strand either one list with <= 2 codes or two single-code lists
__device__ __forceinline__ bool fast_shape(const ListTab& T, uint32_t nl, bool imp_any) {
    bool fast = !imp_any;
    uint32_t cnt0 = 0, cnt1 = 0, max0 = 0, max1 = 0;
    for (uint32_t l2 = 0; l2 < nl; l2++) {
        if (T.base[l2] == 'N') fast = false;
        if (!T.n_delta[l2]) continue;
        const uint32_t ncd = T.ncodes[l2];
        if (T.strand[l2]) { cnt1++; max1 = max(max1, ncd); } else { cnt0++; max0 = max(max0, ncd); }
    }
    if (!(cnt0 <= 1 ? max0 <= 2 : (cnt0 == 2 && max0 == 1))) fast = false;
    if (!(cnt1 <= 1 ? max1 <= 2 : (cnt1 == 2 && max1 == 1))) fast = false;
    return fast;
}

// query position -> reference position over the read's CIGAR prefix: cq[i] = 2 * query start of op i + (op i is M/=/X), one
// sentinel cq[nc] = 2 * query length; cr[i] = reference start of op i; qt[t] = the op that holds query base t << qt_shift
struct QueryMap {
    uint32_t* cq;
    uint32_t* cr;
    uint16_t* qt;
    uint32_t nc, q_total, qt_shift;
    bool use_qt;
};

// CIGAR prefix: query / reference start of every op; four ops per lane (one 16-byte load), 128 per round
__device__ __forceinline__ void cigar_prefix(QueryMap& M, const uint32_t* cig, uint32_t ref_start, uint32_t lane) {
    const uint32_t nc = M.nc;
    uint32_t qc = 0, rc = ref_start;
    for (uint32_t b = 0; b < nc; b += 128) {
        const uint32_t i = b + 4 * lane;
        uint4 c4 = make_uint4(0, 0, 0, 0);
        if (i < nc) c4 = *(const uint4*)(cig + i);    // 16-byte aligned; words past nc belong to the read's own block
        const uint32_t cw[4] = {c4.x, c4.y, c4.z, c4.w};
        uint32_t ql[4], rl[4], qs = 0, rs = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t c = i + k < nc ? cw[k] : 0u, op = c & 15, len = c >> 4;
            // (spelled out: through cig_qlen / cig_rlen nvcc evaluates the classes with 16 more instructions in this loop)
            ql[k] = (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) ? len : 0;
            rl[k] = (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ? len : 0;
            qs += ql[k]; rs += rl[k];
        }
        const uint32_t qi = warp_incl_scan(qs), rr = warp_incl_scan(rs);
        uint32_t q0 = qc + qi - qs, r0 = rc + rr - rs;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (i + k < nc) {
                const uint32_t op = cw[k] & 15;
                M.cq[i + k] = 2u * q0 + (cig_is_match(op) ? 1u : 0u);
                M.cr[i + k] = r0;
            }
            q0 += ql[k]; r0 += rl[k];
        }
        qc += __shfl_sync(FULL, qi, 31);
        rc += __shfl_sync(FULL, rr, 31);
    }
    if (lane == 0) M.cq[nc] = 2u * qc;
    M.q_total = qc;
    __syncwarp();
}

// query -> op table: qt[t] = the op that holds query base t << shift (the largest i with cq[i] <= that base)
__device__ __forceinline__ void query_op_table(QueryMap& M, uint32_t lane) {
    const uint32_t nc = M.nc;
    uint32_t qt_shift = 7;
    while (qt_shift < 31 && (M.q_total >> qt_shift) >= (uint32_t)QT_CAP) qt_shift++;
    M.qt_shift = qt_shift;
    M.use_qt = nc > 0 && nc <= 65535u;
    if (M.use_qt) {
        const uint32_t B = 1u << qt_shift;
        for (uint32_t i = lane; i < nc; i += 32) {
            const uint32_t s0 = M.cq[i] >> 1, e0 = M.cq[i + 1] >> 1;
            for (uint32_t m = (s0 + B - 1) & ~(B - 1); m < e0; m += B) M.qt[m >> qt_shift] = (uint16_t)i;
        }
        if (lane == 0) M.qt[(M.q_total + B - 1) >> qt_shift] = (uint16_t)(nc - 1);
    }
    __syncwarp();
}

// reference position of query position q, when an M/=/X op holds it: that op is the largest i with cq[i] >> 1 <= q, narrowed by
// the table
__device__ __forceinline__ bool project(const QueryMap& M, uint32_t q, uint32_t& rpos) {
    bool aligned = false;
    if (M.nc > 0 && q < M.q_total) {
        uint32_t lo = 0, hi = M.nc;
        if (M.use_qt) { const uint32_t t = q >> M.qt_shift; lo = M.qt[t]; hi = (uint32_t)M.qt[t + 1] + 1u; }
        const uint32_t key = 2u * q + 1u;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (M.cq[mid] <= key) lo = mid; else hi = mid; }
        const uint32_t e = M.cq[lo];
        if ((e & 1u) && q < (M.cq[lo + 1] >> 1)) { aligned = true; rpos = M.cr[lo] + (q - (e >> 1)); }
    }
    return aligned;
}

// Implicit tables ('.'/default mode, src/mod_bam.rs:1265-1292): every other occurrence of a table's base is an inferred-canonical
// entry. A table survives the edge filter when some occurrence of its base keeps its forward position. MODE_PILEUP: the table's
// call goes to imp_meta (ReadMeta::imp); MODE_HIST: imp_hist[sb] counts its inferred values that pass, explicit ones off.
template <int MODE>
__device__ __forceinline__ void implicit_tables(const ChunkDev& C, StateCache& scache, const ListTab& T, uint32_t nl, const uint32_t (*imp_lists)[4],
                                                const mkp_read_hdr& h, const uint32_t* cig, const uint8_t* seq, uint32_t L, bool rev, uint32_t lane,
                                                const uint32_t* imp_explicit, uint32_t* sum_obs, uint32_t& pos_mask, uint32_t& neg_mask,
                                                bool& table_survived, uint32_t* imp_meta, unsigned long long* imp_hist) {
    const bool trim_ok = edge_read_ok(L);
    for (uint32_t sb = 0; sb < 8; sb++) {
        const uint32_t s = sb >> 2, b = sb & 3;
        const uint32_t lists = imp_lists[s][b];
        if (!lists || !trim_ok) continue;
        const uint32_t xn = 1u << (rev ? 3 - b : b);          // SEQ nibble of the forward base b
        // survives the edge filter?  (any occurrence of the base with a kept forward position)
        bool any = false;
        for (uint32_t q = lane; q < L && !any; q += 32) {
            if (seq_nibble(seq, q) != xn) continue;
            const uint32_t f = rev ? L - 1u - q : q;
            // (spelled out: through edge_keep, nvcc compiles this loop of k_resolve<MODE_HIST, false> to 296 more SASS lines)
            bool keep = true;
            if (c_par.edge_on) keep = c_par.edge_inv ? (f < c_par.edge_start || f >= L - c_par.edge_end) : (f >= c_par.edge_start && f < L - c_par.edge_end);
            any = keep;
        }
        if (!__any_sync(FULL, any)) continue;
        Items m, mc;
        m.n = 0;
        int ord[MAX_MAP];
        for (uint32_t l = 0; l < nl; l++) if ((lists >> l) & 1u) for (uint32_t c = 0; c < T.ncodes[l]; c++) if (m.find(T.code[l][c]) < 0) m.push(T.code[l][c], 0.f);
        iter_order(m, ord);
        const Items* use = &m;
        if (c_par.numeric_mode == 2) { redistribute_items(m, ord, c_par.collapse_code, mc); iter_order(mc, ord); use = &mc; }
        const int tb = s == 0 ? (int)b : 3 - (int)b;
        table_survived = true;
        if (MODE == MODE_PILEUP) {
            uint32_t mask = 0;
            for (int k = 0; k < use->n; k++) mask |= 1u << state_id(C, scache, tb, use->code[k]);
            if ((s == 0) != rev) pos_mask |= mask; else neg_mask |= mask;
            uint32_t code = 0;
            const int kind = make_call_items(*use, ord, tb, &code);
            const uint32_t state = kind == 0 ? 0u : kind == 1 ? 1u : 2u + (uint32_t)state_id(C, scache, tb, code);
            imp_meta[s] |= (0x80u | state) << (8 * b);
        } else {
            if (C.summ) for (int k = 0; k < use->n; k++) sum_obs[tb] |= 1u << state_id(C, scache, tb, use->code[k]);
            // values: argmax of an all-zero map = canonical probability 1.0 for every passing inferred position
            unsigned long long n_pass = 0;
            if (C.hist_include_unaligned && !C.focus_pos) {
                for (uint32_t q = lane; q < L; q += 32) {
                    if (seq_nibble(seq, q) != xn) continue;
                    const uint32_t f = rev ? L - 1u - q : q;
                    if (edge_keep(f, L)) n_pass++;
                }
            } else {
                uint32_t qc2 = 0, rc2 = (uint32_t)h.ref_start;
                const uint32_t* bm = C.focus_pos ? (((s == 0) == rev) ? C.focus_neg : C.focus_pos) : nullptr;
                for (uint32_t i = 0; i < h.n_cigar; i++) {
                    const uint32_t c = cig[i], op = c & 15, len = c >> 4;
                    if (cig_is_match(op)) {
                        for (uint32_t k = lane; k < len; k += 32) {
                            const uint32_t q = qc2 + k;
                            if (q >= L || seq_nibble(seq, q) != xn) continue;
                            const uint32_t f = rev ? L - 1u - q : q;
                            bool keep = edge_keep(f, L);
                            if (keep && bm) {
                                const uint32_t r = rc2 + k;
                                keep = r >= C.cs && r < C.ce && ((bm[(r - C.cs) >> 5] >> ((r - C.cs) & 31)) & 1u);
                            }
                            if (keep) n_pass++;
                        }
                    }
                    qc2 += cig_qlen(op, len);
                    rc2 += cig_rlen(op, len);
                }
            }
            n_pass = __reduce_add_sync(FULL, (uint32_t)n_pass);
            const uint32_t n_exp = __reduce_add_sync(FULL, imp_explicit[sb]);
            imp_hist[sb] = n_pass > n_exp ? n_pass - n_exp : 0;
        }
    }
}

// Kernel B: per read with mod info: CIGAR prefix, then every list entry -> merged probabilities -> collapse ->
// threshold call -> reference position; call records, observed-code masks, implicit tables, hot-bitmap marks.
// FAST_ONLY = true: handles the reads whose lists fit the register-only path (no implicit tables, no 'N' list, at most
// two codes per position) and queues the others; FAST_ONLY = false: the generic path over the queued reads. Two
// instantiations keep the common case's register and instruction footprint small.
template <int MODE, bool FAST_ONLY>
__global__ void __launch_bounds__(128, FAST_ONLY ? MKP_MINB_RESOLVE_FAST : MKP_MINB_RESOLVE) k_resolve(ChunkDev C) {
    __shared__ ListTab s_tab[4];
    // CIGAR prefix of the current read (global scratch when longer): s_cq = 2 * query start + (op is M/=/X), one
    // sentinel entry 2 * query length at the end; s_cr = reference start; s_qt = op holding every (1 << shift)-th query base
    __shared__ __align__(16) uint32_t s_cq[4][CQ_CAP + 4], s_cr[4][CQ_CAP];
    __shared__ uint16_t s_qt[4][QT_CAP + 2];
    const uint32_t lane = lane_id();
    const uint32_t wib = threadIdx.x >> 5;
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    ListTab& T = s_tab[wib];
    StateCache scache;
    scache.init();
    RCLK_INIT;
    uint32_t* const gcq = C.scr_cq + (size_t)gw * (C.max_ncigar + 4);
    uint32_t* const gcr = C.scr_cr + (size_t)gw * (C.max_ncigar + 4);

    for (;;) {
        uint32_t ri = 0;
        if (FAST_ONLY) {
            if (lane == 0) { ri = atomicAdd(C.work + 1, 1u); if (C.order && ri < C.n_reads) ri = C.order[ri]; }
            ri = __shfl_sync(FULL, ri, 0);
            if (ri >= C.n_reads) break;
        } else {
            if (lane == 0) { ri = atomicAdd(C.work + 5, 1u); ri = ri < C.work[4] ? C.slow_list[ri] : 0xffffffffu; }
            ri = __shfl_sync(FULL, ri, 0);
            if (ri == 0xffffffffu) break;
        }
        ReadMeta meta = C.meta[ri];
        if (!(meta.flags & 1)) continue;
        const ReadLists* R = C.rl + ri;
        const uint32_t nl = R->n;
        bool err = R->flags & 1u;
        const bool any_entries = R->flags & 2u;
        if (err || !any_entries) continue;          // skip_set: counts only as bases (meta already says so)
        const mkp_read_hdr h = C.hdrs[ri];
        const uint32_t L = h.l_seq;
        const bool rev = h.flags & 0x10;
        const uint32_t* cig = (const uint32_t*)(C.heap + h.off);
        const uint8_t* seq = C.heap + h.off + 4ull * h.n_cigar;
        const uint8_t* ml = seq + ((L + 1) >> 1);
        uint32_t imp_lists[2][4];
        for (int k = 0; k < 8; k++) imp_lists[k >> 2][k & 3] = R->imp_lists[k];
        load_list_table(T, R, nl, lane);
        bool imp_any = false;
        for (int k = 0; k < 8; k++) imp_any = imp_any || imp_lists[k >> 2][k & 3];
        const bool fast_read = fast_shape(T, nl, imp_any);
        if (FAST_ONLY && !fast_read) {                 // leave it to the generic instantiation
            if (lane == 0) C.slow_list[atomicAdd(C.work + 4, 1u)] = ri;
            continue;
        }
        RCLK(0);
        RCLK_COUNT(6, 1);
        QueryMap qm;
        qm.nc = h.n_cigar;
        qm.cq = h.n_cigar <= CQ_CAP ? s_cq[wib] : gcq;
        qm.cr = h.n_cigar <= CQ_CAP ? s_cr[wib] : gcr;
        qm.qt = s_qt[wib];
        cigar_prefix(qm, cig, (uint32_t)h.ref_start, lane);
        RCLK(1);
        query_op_table(qm, lane);
        RCLK(2);
        uint32_t* P = C.P + meta.entry_off;
        // ---- phase 4: resolve entries -> calls ---------------------------------------------------
        uint32_t n_calls = 0, n_hist = 0;
        uint32_t n_runs = 0;          // lists that emitted call records (each list's records are sorted by position)
        uint32_t pos_mask = 0, neg_mask = 0;
        bool table_survived = false;
        uint32_t imp_explicit[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // HIST: explicit values on implicit tables (per lane)
        uint32_t sum_obs[4] = {0, 0, 0, 0};                    // summary: states seen per canonical base (per lane)
        uint2* calls = C.calls + meta.entry_off;
        if (!err && any_entries) {
            // (spelled out: through edge_read_ok, ptxas allocates every instantiation differently, and k_resolve<MODE_HIST, false>
            // spills 8 more bytes each way)
            const bool trim_ok = !c_par.edge_on || !(L <= c_par.edge_start || L <= c_par.edge_end);
            uint32_t skip_mask = 0;       // lists whose every entry sits at the same index of an earlier same-strand list
            for (uint32_t l = 0; l < nl && !err; l++) {
                if ((skip_mask >> l) & 1u) continue;    // all its entries are absorbed (basecallers repeat one delta list per code)
                const uint32_t n = T.n_delta[l];
                const uint32_t* Pl = P + T.ent_off[l];
                const uint32_t st = T.strand[l];
                const uint8_t lfb = T.base[l];
                const int lb = lfb == 'A' ? 0 : lfb == 'C' ? 1 : lfb == 'G' ? 2 : (lfb == 'T' || lfb == 'U') ? 3 : 4;
                uint32_t lnext = 0xffffffffu;           // nearest later list of the same strand with entries
                for (uint32_t l2 = nl; l2-- > l + 1;) if (T.strand[l2] == st && T.n_delta[l2]) lnext = l2;
                uint32_t cnt_next = 0;
                const uint32_t calls_before = n_calls;
                RCLK_COUNT(7, n);
                // Register-only path: an entry holds the list's first code c0, and either nothing else ("single") or the
                // pair code pc1 ("pair": the list's second code, or the code of lnext where lnext holds the entry). A pair
                // code equal to c0 adds into c0's probability, so the entry stays single. Whatever depends only on the
                // list is worked out here, once, for both shapes: the codes left after ReDistribute in FxHash order
                // (k-th out code = (sel ^ k) ? pc1 : c0), their thresholds, and (on first use, per lane) their state ids.
                const uint32_t ncl = T.ncodes[l];
                const uint32_t c0 = T.code[l][0];
                const uint32_t pc1 = ncl == 2 ? T.code[l][1] : lnext != 0xffffffffu ? T.code[lnext][0] : c0;
                const uint32_t ml_l = T.ml_off[l];
                const uint32_t nn = lnext != 0xffffffffu ? T.n_delta[lnext] : 0u;      // lnext's entries, offsets
                const uint32_t eo_n = lnext != 0xffffffffu ? T.ent_off[lnext] : 0u, mo_n = lnext != 0xffffffffu ? T.ml_off[lnext] : 0u;
                const int tb_l = st == 0 ? lb : 3 - lb;
                uint32_t plan = 1u | (2u << 4);      // n_out | sel << 2 of the single shape, and of the pair shape << 4
                float thr_s0 = 0.f, thr_p0 = 0.f, thr_p1 = 0.f, base_thr_l = 0.f;
                uint32_t sids = 0xffffffu;           // state ids of the out codes, one byte each: single, pair 0, pair 1;
                                                     // byte 3 bit 0 / 1: the single / pair ids are looked up
                if (MODE == MODE_PILEUP && (FAST_ONLY || fast_read)) {
                    uint32_t ps = 1, pp = 2;
                    if (c_par.numeric_mode == 2) {
                        const uint32_t drop = c_par.collapse_code;
                        if (c0 == drop) ps = 0;
                        pp = c0 == drop ? (1u | 4u) : pc1 == drop ? 1u : 2u;
                    }
                    if (pp == 2 && (bucket4(c0) != bucket4(pc1) ? (bucket4(pc1) < bucket4(c0)) : (bucket4(c0) == 3))) pp |= 4u;
                    plan = ps | (pp << 4);
                    base_thr_l = base_threshold(tb_l);
                    thr_s0 = mod_threshold(c0, tb_l, base_thr_l);
                    thr_p0 = mod_threshold((pp & 4u) ? pc1 : c0, tb_l, base_thr_l);
                    thr_p1 = mod_threshold((pp & 4u) ? c0 : pc1, tb_l, base_thr_l);
                }
                for (uint32_t j0 = 0; j0 < n; j0 += 32) {
                    uint32_t j = j0 + lane;
                    bool active = j < n;
                    bool matched_next = false;
                    bool emit = false;
                    uint32_t rpos = 0, info = 0;
                    bool e2 = false;
                    bool hist_ok = false;
                    float hist_v = 0.f;
                    int hist_base = 0;
                    uint32_t hist_q = 0;
                    if (active) {
                        uint32_t f = Pl[j];
                        // register-only path: the entry's ML byte(s) and lnext's entry at the same index do not depend on f;
                        // loaded beside it, the loads overlap instead of each waiting on the one before
                        uint32_t ma = 0, mb = 0, p2j = 0xffffffffu, qn = 0;
                        if (FAST_ONLY || fast_read) {
                            const uint8_t* mlq = ml + ml_l + (size_t)j * ncl;
                            ma = mlq[0];
                            if (ncl == 2) mb = mlq[1];
                            if (j < nn) { p2j = P[eo_n + j]; qn = ml[mo_n + j]; }
                        }
                        uint32_t q = rev ? L - 1u - f : f;
                        // forward-read base at f: the list's own base (the position was selected as one of its occurrences);
                        // only 'N' lists have to look at the sequence (mod_bam.rs:1245)
                        int b = lb;
                        if (!FAST_ONLY && lb > 3) {
                            const int nb = nib_to_base(seq_nibble(seq, q));
                            b = nb > 3 ? 4 : (rev ? 3 - nb : nb);
                            if (b > 3) e2 = true;
                        }
                        // ExplicitConflictInferred (mod_bam.rs:629-634): an implicit list of this (strand, base) table
                        // that does not list f explicitly holds an inferred entry there
                        if (!FAST_ONLY && b <= 3) {
                            uint32_t others = imp_lists[st][b] & ~(1u << l);
                            while (others && !e2) {
                                const uint32_t l2 = __ffs(others) - 1;
                                others &= others - 1;
                                const uint32_t* P2 = P + T.ent_off[l2];
                                const uint32_t n2 = T.n_delta[l2];
                                if (j < n2 && P2[j] == f) continue;
                                const uint32_t k = lower_bound_u32(P2, n2, f);
                                if (!(k < n2 && P2[k] == f)) e2 = true;
                            }
                        }
                        // absorbed by an earlier list of the same strand?
                        bool owner = true;
                        for (uint32_t l2 = 0; l2 < l && owner; l2++) {
                            if (T.strand[l2] != st || T.n_delta[l2] == 0) continue;
                            const uint32_t* P2 = P + T.ent_off[l2];
                            uint32_t n2 = T.n_delta[l2];
                            if (j < n2 && P2[j] == f) { owner = false; break; }
                            uint32_t k = lower_bound_u32(P2, n2, f);
                            if (k < n2 && P2[k] == f) owner = false;
                        }
                        RCLK_MARK;
                        if (owner && !e2) {
                            const int tb = st == 0 ? b : 3 - b;
                            uint32_t mask = 0, ccode = 0;      // observed states, called code
                            uint32_t csid = 0;                 // state id of the called code (register-only pileup path)
                            int kind = 0;                      // 0 filtered, 1 canonical, 2 modified
                            float hv = 0.f;                    // arg-max value (histogram mode)
                            if (FAST_ONLY || fast_read) {
                                // ---- register-only path: at most two codes at the position (one list with <= 2 codes, or
                                //      two single-code lists of the strand). Same arithmetic as the generic path below.
                                float p0, p1 = 0.f;
                                bool pair = false;
                                {
                                    p0 = ml_prob(ma);
                                    if (ncl == 2) {
                                        const float pb = ml_prob(mb);
                                        if (pc1 == c0) { if (__fadd_rn(p0, pb) > 1.01f) e2 = true; else p0 = __fadd_rn(p0, pb); }
                                        else { p1 = pb; pair = true; }
                                    }
                                }
                                if (lnext != 0xffffffffu && !e2) {       // the strand's other list (single code by construction)
                                    const uint32_t* P2 = P + eo_n;
                                    uint32_t k = j;
                                    const uint8_t* mln = ml + mo_n;
                                    bool found = j < nn && p2j == f;          // same index in the other list: the usual case
                                    if (found) matched_next = true;
                                    else { k = lower_bound_u32(P2, nn, f); found = k < nn && P2[k] == f; if (found) qn = mln[k]; }
                                    if (found) {
                                        const float pn = ml_prob(qn);
                                        if (pc1 == c0) p0 = __fadd_rn(p0, pn);
                                        else { p1 = pn; pair = true; }
                                        if ((pair ? __fadd_rn(p0, p1) : p0) > 1.01f) e2 = true;   // combine_checked
                                    }
                                }
                                if (!e2) {
                                    if (MODE == MODE_PILEUP) {
                                        // the list's plan for the entry's shape: ReDistribute, FxHash order, thresholds
                                        const uint32_t pw = pair ? plan >> 4 : plan;
                                        const uint32_t n_out = pw & 3u;
                                        const bool sel = pw & 4u;
                                        float o0 = sel ? p1 : p0;
                                        const float o1 = sel ? p0 : p1;
                                        if (n_out == 1) o0 = __fadd_rn(o0, half_share(o1));     // single: p1 == 0 adds nothing
                                        const float sum = n_out == 0 ? 0.f : n_out == 1 ? o0 : __fadd_rn(o0, o1);
                                        const float cp = __fsub_rn(1.0f, sum);
                                        bool have = false;
                                        float best = 0.f;
                                        uint32_t called = 0;
                                        if (n_out >= 1 && o0 >= (pair ? thr_p0 : thr_s0)) { have = true; best = o0; kind = 2; }
                                        if (n_out == 2 && o1 >= thr_p1 && (!have || o1 >= best)) { have = true; best = o1; kind = 2; called = 1; }
                                        if (cp >= base_thr_l && (!have || cp >= best)) { have = true; kind = 1; }
                                        if (!have) kind = 0;
                                        // state ids: registered when a lane first meets the shape, as every entry would
                                        if (n_out != 0) {
                                            const uint32_t sh = pair ? 8u : 0u;
                                            if (!((sids >> (24u + (sh >> 3))) & 1u)) {
                                                const uint32_t s0 = (uint32_t)state_id(C, scache, tb_l, sel ? pc1 : c0);
                                                sids = (sids & ~(0xffu << sh)) | (s0 << sh) | (1u << (24u + (sh >> 3)));
                                                if (n_out == 2) sids = (sids & 0xff00ffffu) | ((uint32_t)state_id(C, scache, tb_l, sel ? c0 : pc1) << 16);
                                            }
                                            mask = (1u << ((sids >> sh) & 0xffu)) | (n_out == 2 ? 1u << ((sids >> 16) & 0xffu) : 0u);
                                            csid = (sids >> (sh + 8u * called)) & 0xffu;
                                        }
                                    } else {
                                        uint32_t k0 = c0, k1 = pair ? pc1 : 0u;
                                        int n2c = pair ? 2 : 1;
                                        if (c_par.numeric_mode == 2) redistribute2(c_par.collapse_code, k0, p0, k1, p1, n2c);
                                        // FxHashMap iteration order of the (<= 2) codes
                                        if (n2c == 2) {
                                            const uint32_t b0 = bucket4(k0), b1 = bucket4(k1);
                                            if (b0 != b1 ? (b1 < b0) : (b0 == 3)) { const uint32_t tc = k0; k0 = k1; k1 = tc; const float tp = p0; p0 = p1; p1 = tp; }
                                        }
                                        const float sum = n2c == 0 ? 0.f : n2c == 1 ? __fadd_rn(0.f, p0) : __fadd_rn(__fadd_rn(0.f, p0), p1);
                                        const float cp = __fsub_rn(1.0f, sum);
                                        float mp = 0.f;
                                        bool hm2 = false;
                                        if (n2c >= 1) { mp = p0; hm2 = true; }
                                        if (n2c == 2 && p1 >= mp) mp = p1;
                                        hv = (hm2 && mp > cp) ? mp : cp;
                                        if (C.summ || C.qhist) {
                                            // thresholded call (as in the pileup) and arg-max call (last maximum wins, mod_bam.rs:489-505)
                                            uint32_t s0 = 0, s1 = 0;
                                            if (n2c >= 1) { s0 = (uint32_t)state_id(C, scache, tb, k0); mask |= 1u << s0; }
                                            if (n2c == 2) { s1 = (uint32_t)state_id(C, scache, tb, k1); mask |= 1u << s1; }
                                            const float base_thr = base_threshold(tb);
                                            bool have = false;
                                            float best = 0.f;
                                            uint32_t tk = 0, ts = 0;
                                            for (int k2 = 0; k2 < n2c; k2++) {
                                                const float pp = k2 == 0 ? p0 : p1;
                                                const float thr = mod_threshold(k2 == 0 ? k0 : k1, tb, base_thr);
                                                if (pp >= thr && (!have || pp >= best)) { have = true; best = pp; tk = 2; ts = k2 == 0 ? s0 : s1; }
                                            }
                                            if (cp >= base_thr && (!have || cp >= best)) { have = true; tk = 1; }
                                            if (!have) tk = 0;
                                            const uint32_t as = (n2c == 2 && p1 >= p0) ? s1 : s0;
                                            const uint32_t ak = (hm2 && mp > cp) ? 2u : 1u;
                                            ccode = sample_class(tk, ts, ak, as);     // summary record of this value
                                        }
                                    }
                                }
                            } else {
                            Items m;
                            m.n = 0;
                            int ord[MAX_MAP];
                            const uint8_t* mlq = ml + T.ml_off[l] + (size_t)j * T.ncodes[l];
                            for (uint32_t c = 0; c < T.ncodes[l] && !e2; c++) {
                                const float p = ml_prob(mlq[c]);
                                const int it = m.find(T.code[l][c]);
                                if (it < 0) { if (!m.push(T.code[l][c], p)) { atomicOr(C.err, MKP_DERR_TOO_MANY_CODES); e2 = true; } }
                                else { if (__fadd_rn(m.p[it], p) > 1.01f) e2 = true; else m.p[it] = __fadd_rn(m.p[it], p); }
                            }
                            for (uint32_t l2 = l + 1; l2 < nl && !e2; l2++) {
                                if (T.strand[l2] != st || T.n_delta[l2] == 0) continue;
                                const uint32_t* P2 = P + T.ent_off[l2];
                                const uint32_t n2 = T.n_delta[l2];
                                uint32_t k;
                                if (j < n2 && P2[j] == f) { k = j; if (l2 == lnext) matched_next = true; }
                                else { k = lower_bound_u32(P2, n2, f); if (!(k < n2 && P2[k] == f)) continue; }
                                // per-list table first (add_base_mod_prob), then combine_checked into the aggregate
                                Items t2;
                                t2.n = 0;
                                const uint8_t* ml2 = ml + T.ml_off[l2] + (size_t)k * T.ncodes[l2];
                                for (uint32_t c = 0; c < T.ncodes[l2] && !e2; c++) {
                                    const float p = ml_prob(ml2[c]);
                                    const int it = t2.find(T.code[l2][c]);
                                    if (it < 0) { if (!t2.push(T.code[l2][c], p)) { atomicOr(C.err, MKP_DERR_TOO_MANY_CODES); e2 = true; } }
                                    else { if (__fadd_rn(t2.p[it], p) > 1.01f) e2 = true; else t2.p[it] = __fadd_rn(t2.p[it], p); }
                                }
                                int o2[MAX_MAP];
                                iter_order(t2, o2);
                                for (int s2 = 0; s2 < t2.n && !e2; s2++) {
                                    const int i2 = o2[s2];
                                    const int it = m.find(t2.code[i2]);
                                    if (it < 0) { if (!m.push(t2.code[i2], t2.p[i2])) { atomicOr(C.err, MKP_DERR_TOO_MANY_CODES); e2 = true; } }
                                    else m.p[it] = __fadd_rn(m.p[it], t2.p[i2]);
                                }
                                if (!e2) { iter_order(m, ord); if (items_sum(m, ord) > 1.01f) e2 = true; }
                            }
                            if (!e2) {
                                iter_order(m, ord);
                                Items mc;
                                const Items* use = &m;
                                if (c_par.numeric_mode == 2) { redistribute_items(m, ord, c_par.collapse_code, mc); iter_order(mc, ord); use = &mc; }
                                if (MODE == MODE_PILEUP) {
                                    for (int k2 = 0; k2 < use->n; k2++) mask |= 1u << state_id(C, scache, tb, use->code[k2]);
                                    kind = make_call_items(*use, ord, tb, &ccode);
                                } else {
                                    hv = argmax_items(*use, ord);
                                    if (C.summ || C.qhist) {
                                        uint32_t tcode = 0;
                                        const int tkind = make_call_items(*use, ord, tb, &tcode);
                                        uint32_t ts = 0, as = 0;
                                        if (tkind == 2) ts = (uint32_t)state_id(C, scache, tb, tcode);
                                        const float cp2 = __fsub_rn(1.0f, items_sum(*use, ord));
                                        bool hm = false;
                                        float mp2 = 0.f;
                                        uint32_t acode = 0;
                                        for (int k2 = 0; k2 < use->n; k2++) {
                                            mask |= 1u << state_id(C, scache, tb, use->code[k2]);
                                            const float v = use->p[ord[k2]];
                                            if (!hm || v >= mp2) { hm = true; mp2 = v; acode = use->code[ord[k2]]; }
                                        }
                                        const uint32_t ak = (hm && mp2 > cp2) ? 2u : 1u;
                                        if (ak == 2) as = (uint32_t)state_id(C, scache, tb, acode);
                                        ccode = sample_class((uint32_t)tkind, ts, ak, as);
                                    }
                                }
                            }
                            }
                            RCLK_MARK;
                            if (!e2) {
                                bool keep = trim_ok;
                                if (keep) keep = edge_keep(f, L);
                                if (keep) {
                                    const bool aligned = project(qm, q, rpos);
                                    if (MODE == MODE_PILEUP) {
                                        // (mod strand, read orientation) -> reference strand (read_cache.rs:181-188)
                                        if ((st == 0) != rev) pos_mask |= mask; else neg_mask |= mask;
                                        table_survived = true;
                                        // positions outside the focus set (motif / include-bed) are dropped when the hot bitmap
                                        // is ranked (k_block_popc) and skipped by k_count_calls: no bitmap lookup here
                                        if (aligned && rpos >= C.cs && rpos < C.ce) {
                                            const uint32_t state = kind == 0 ? 0u : kind == 1 ? 1u : 2u + ((FAST_ONLY || fast_read) ? csid : (uint32_t)state_id(C, scache, tb, ccode));
                                            // does a '+' list cover the same position (both pos_call and neg_call present)?
                                            uint32_t nosub = 0;
                                            if (st == 1) {
                                                for (uint32_t l2 = 0; l2 < nl && !nosub; l2++) {
                                                    if (T.strand[l2] != 0 || T.n_delta[l2] == 0) continue;
                                                    const uint32_t* P2 = P + T.ent_off[l2];
                                                    const uint32_t k = lower_bound_u32(P2, T.n_delta[l2], f);
                                                    if (k < T.n_delta[l2] && P2[k] == f) nosub = 1;
                                                }
                                            }
                                            emit = true;
                                            info = call_info(st, (uint32_t)b, state, nosub);
                                        }
                                    } else {
                                        bool pass = aligned || C.hist_include_unaligned;
                                        if (C.focus_pos) {
                                            // --include-bed: keep only aligned positions inside the BED on the matching reference
                                            // strand (read_ids_to_base_mod_probs.rs:1020-1047); chunk bitmaps hold the BED
                                            pass = false;
                                            if (aligned && rpos >= C.cs && rpos < C.ce) {
                                                const uint32_t x = rpos - C.cs;
                                                const uint32_t* bm = ((st == 0) == rev) ? C.focus_neg : C.focus_pos;
                                                pass = (bm[x >> 5] >> (x & 31)) & 1u;
                                            }
                                        }
                                        if (pass) {
                                            hist_ok = true; hist_v = hv; hist_base = tb;
                                            if (C.summ || C.qhist) { hist_q = prob_to_qual(hv); hist_v = __uint_as_float(ccode); }
                                            if (C.summ) sum_obs[tb] |= mask;
                                            if (!FAST_ONLY && imp_lists[st][b]) imp_explicit[st * 4 + b]++;
                                        }
                                    }
                                }
                            }
                        }
                    }
                    err = __any_sync(FULL, e2) || err;
                    cnt_next += __popc(__ballot_sync(FULL, matched_next));
                    if (MODE == MODE_PILEUP) {
                        uint32_t em = __ballot_sync(FULL, emit);
                        if (emit) {
                            calls[n_calls + __popc(em & ((1u << lane) - 1u))] = make_uint2(rpos, info);
                            // marks of a read that fails later stay behind: a hot position without calls yields no rows
                            const uint32_t x = rpos - C.cs;
                            const uint32_t t = call_strand(info) ^ (rev ? 1u : 0u);        // reference strand of the call
                            if (!C.list_mode) atomicOr(&C.hot[t * ((C.ce - C.cs + 31) >> 5) + (x >> 5)], 1u << (x & 31));
                        }
                        n_calls += __popc(em);
                    } else {
                        uint32_t hm = __ballot_sync(FULL, hist_ok);
                        if (hist_ok) {
                            // stash (bin | base<<16 | inexact<<20 | qual<<21) in the call buffer; committed after validation.
                            // Values above 1.0 are legal (ML sums up to 1.01, ReDistribute shares) and get their own bins.
                            // With summ / qhist, y holds the packed classification and the bin is 0
                            float sc = __fmul_rn((C.summ || C.qhist) ? 0.f : hist_v, 1024.0f);
                            int bin = (int)rintf(sc);
                            uint32_t inexact = ((float)bin != sc || bin < 0 || bin >= MKP_HIST_BINS) ? 1u : 0u;
                            if (bin < 0) bin = 0;
                            if (bin >= MKP_HIST_BINS) bin = MKP_HIST_BINS - 1;
                            calls[n_hist + __popc(hm & ((1u << lane) - 1u))] = make_uint2(sample_key((uint32_t)bin, (uint32_t)hist_base, inexact, hist_q), __float_as_uint(hist_v));
                        }
                        n_hist += __popc(hm);
                    }
                    RCLK_ROUND;
                }
                if (n_calls != calls_before) n_runs++;
                if (!imp_any && lnext != 0xffffffffu && T.base[lnext] != 'N' && T.n_delta[lnext] == cnt_next) skip_mask |= 1u << lnext;
            }
        }
        RCLK(3);
        // ---- phase 4b: implicit tables (every other occurrence of the base is an inferred-canonical entry) ----
        uint32_t imp_meta[2] = {0, 0};
        unsigned long long imp_hist[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (!FAST_ONLY && !err)
            implicit_tables<MODE>(C, scache, T, nl, imp_lists, h, cig, seq, L, rev, lane, imp_explicit, sum_obs, pos_mask, neg_mask,
                                  table_survived, imp_meta, imp_hist);
        pos_mask = __reduce_or_sync(FULL, pos_mask);
        neg_mask = __reduce_or_sync(FULL, neg_mask);
        table_survived = __any_sync(FULL, table_survived);
        __syncwarp();
        // ---- phase 5: commit -------------------------------------------------------------------------
        if (MODE == MODE_PILEUP) {
            if (!err && table_survived) {
                meta.flags |= 2;
                if (n_runs <= 1 && !(imp_meta[0] | imp_meta[1])) meta.flags |= 4;     // one sorted run: k_count_bases merges it
                meta.pos_mask = pos_mask; meta.neg_mask = neg_mask; meta.n_calls = n_calls;
                meta.imp[0] = imp_meta[0]; meta.imp[1] = imp_meta[1];
                if (lane == 0 && n_calls) atomicAdd(C.total_calls, (unsigned long long)n_calls);
                if (!FAST_ONLY && (imp_meta[0] | imp_meta[1]) && !C.list_mode) {
                    // every aligned occurrence of an implicit table's base is a call position
                    uint32_t qc2 = 0, rc2 = (uint32_t)h.ref_start;
                    for (uint32_t i = 0; i < h.n_cigar; i++) {
                        const uint32_t c = cig[i], op = c & 15, len = c >> 4;
                        if (cig_is_match(op)) {
                            for (uint32_t k = lane; k < len; k += 32) {
                                const uint32_t q = qc2 + k, r = rc2 + k;
                                if (q >= L || r < C.cs || r >= C.ce) continue;
                                const int nb = nib_to_base(seq_nibble(seq, q));
                                if (nb > 3) continue;
                                const uint32_t b = rev ? 3 - nb : nb;
                                if (!(((imp_meta[0] | imp_meta[1]) >> (8 * b)) & 0x80u)) continue;
                                const uint32_t f = rev ? L - 1u - q : q;
                                if (!edge_keep(f, L)) continue;
                                const uint32_t x = r - C.cs;
                                if (C.focus_pos && !(((C.focus_pos[x >> 5] | C.focus_neg[x >> 5]) >> (x & 31)) & 1u)) continue;
                                // the table of mod strand s counts on reference strand s ^ rev
                                const uint32_t nw = (C.ce - C.cs + 31) >> 5;
                                for (uint32_t s = 0; s < 2; s++)
                                    if ((imp_meta[s] >> (8 * b)) & 0x80u) atomicOr(&C.hot[(s ^ (rev ? 1u : 0u)) * nw + (x >> 5)], 1u << (x & 31));
                            }
                        }
                        qc2 += cig_qlen(op, len);
                        rc2 += cig_rlen(op, len);
                    }
                }
            }
        } else {
            if (!err && any_entries) {
                unsigned long long extra = 0;
                for (int sb = 0; sb < 8; sb++) extra += imp_hist[sb];
                meta.n_hist = n_hist + (uint32_t)(extra < 0x7fffffffull ? extra : 0x7fffffffull);
                if (C.summ) {
                    uint32_t seen = 0;
                    for (uint32_t k = lane; k < n_hist; k += 32) {
                        const uint2 v = calls[k];
                        const uint32_t tb = sample_base(v.x), tk = class_tkind(v.y), ts = class_tstate(v.y), ak = class_akind(v.y), as = class_astate(v.y);
                        seen |= 1u << tb;
                        // pass: the thresholded call; fail: filed under the arg-max call (src/summarize.rs:186-214)
                        if (tk == 1) atomicAdd(&C.summ[(tb * 2 + 0) * 33 + 0], 1ull);
                        else if (tk == 2) atomicAdd(&C.summ[(tb * 2 + 0) * 33 + 1 + ts], 1ull);
                        else if (ak == 1) atomicAdd(&C.summ[(tb * 2 + 1) * 33 + 0], 1ull);
                        else atomicAdd(&C.summ[(tb * 2 + 1) * 33 + 1 + as], 1ull);
                    }
                    seen = __reduce_or_sync(FULL, seen);
                    uint32_t obs[4];
                    for (int b = 0; b < 4; b++) obs[b] = __reduce_or_sync(FULL, sum_obs[b]);
                    if (lane == 0) {
                        for (int sb = 0; sb < 8; sb++) if (imp_hist[sb]) {
                            const int tb = table_base(sb);
                            // an inferred entry is the all-zero map: canonical with probability 1.0
                            atomicAdd(&C.summ[(tb * 2 + (1.0f >= base_threshold(tb) ? 0 : 1)) * 33 + 0], imp_hist[sb]);
                            seen |= 1u << tb;
                        }
                        for (int b = 0; b < 4; b++) {
                            if ((seen >> b) & 1u) atomicAdd(&C.summ[4 * 2 * 33 + b], 1ull);
                            if (obs[b]) atomicOr((uint32_t*)(C.summ + 4 * 2 * 33 + 4) + b, obs[b]);
                        }
                    }
                }
                if (C.qhist) {
                    for (uint32_t k = lane; k < n_hist; k += 32) {
                        const uint2 v = calls[k];
                        const uint32_t tb = sample_base(v.x), q = sample_qual(v.x), ak = class_akind(v.y), as = class_astate(v.y);
                        atomicAdd(&C.qhist[(tb * 33 + (ak == 2 ? 1 + as : 0)) * 256 + q], 1ull);
                    }
                    // an inferred entry is the all-zero map: canonical with probability 1.0, qual 255
                    if (lane == 0) for (int sb = 0; sb < 8; sb++) if (imp_hist[sb]) {
                        const int tb = table_base(sb);
                        atomicAdd(&C.qhist[(tb * 33 + 0) * 256 + 255], imp_hist[sb]);
                    }
                }
                if (C.hist) {
                    for (uint32_t k = lane; k < n_hist; k += 32) {
                        uint32_t v = calls[k].x;
                        atomicAdd(&C.hist[sample_base(v) * MKP_HIST_BINS + sample_bin(v)], 1ull);
                        if (sample_inexact(v)) atomicAdd(C.hist_inexact, 1ull);
                    }
                    if (lane == 0) for (int sb = 0; sb < 8; sb++) if (imp_hist[sb]) {
                        const int tb = table_base(sb);
                        atomicAdd(&C.hist[tb * MKP_HIST_BINS + 1024u], imp_hist[sb]);
                    }
                }
            }
        }
        if (lane == 0) C.meta[ri] = meta;
        __syncwarp();
        RCLK(5);
    }
    RCLK(0);
    RCLK_FLUSH;
}

// ---- rank over the hot bitmap -----------------------------------------------------------------------
// (with focus bitmaps, `bits` is the [2][n_words / 2] per-strand pair: marks outside the strand's focus set, which k_resolve does
// not look at, are cleared here)
__global__ void k_block_popc(uint32_t* __restrict__ bits, uint32_t n_words, uint32_t* __restrict__ block_sums,
                             const uint32_t* __restrict__ focus_pos, const uint32_t* __restrict__ focus_neg) {
    __shared__ uint32_t s[32];
    uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    uint32_t v = 0;
    if (i < n_words) {
        uint32_t word = bits[i];
        if (focus_pos && word) {
            const uint32_t half = n_words >> 1;
            const uint32_t keep = word & (i < half ? focus_pos[i] : focus_neg[i - half]);
            if (keep != word) bits[i] = keep;
            word = keep;
        }
        v = __popc(word);
    }
    uint32_t w = __reduce_add_sync(FULL, v);
    if (lane_id() == 0) s[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x < 32) { uint32_t t = __reduce_add_sync(FULL, s[threadIdx.x]); if (threadIdx.x == 0) block_sums[blockIdx.x] = t; }
}
// single block: exclusive scan of block_sums in place, total -> *total
__global__ void k_scan_blocks(uint32_t* block_sums, uint32_t n, uint32_t* total) {
    __shared__ uint32_t s_carry;
    __shared__ uint32_t s_w[32];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t b = 0; b < n; b += 1024) {
        uint32_t i = b + threadIdx.x;
        uint32_t v = i < n ? block_sums[i] : 0;
        uint32_t inc = warp_incl_scan(v);
        if (lane_id() == 31) s_w[threadIdx.x >> 5] = inc;
        __syncthreads();
        if (threadIdx.x < 32) { uint32_t t = s_w[threadIdx.x]; uint32_t ti = warp_incl_scan(t); s_w[threadIdx.x] = ti - t; }
        __syncthreads();
        uint32_t ex = s_carry + s_w[threadIdx.x >> 5] + inc - v;
        if (i < n) block_sums[i] = ex;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = ex + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_carry;
}
__global__ void k_word_prefix(const uint32_t* __restrict__ bits, uint32_t n_words, const uint32_t* __restrict__ block_sums, uint32_t* __restrict__ prefix) {
    __shared__ uint32_t s_w[32];
    uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    uint32_t v = i < n_words ? __popc(bits[i]) : 0;
    uint32_t inc = warp_incl_scan(v);
    if (lane_id() == 31) s_w[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) { uint32_t t = s_w[threadIdx.x]; uint32_t ti = warp_incl_scan(t); s_w[threadIdx.x] = ti - t; }
    __syncthreads();
    if (i < n_words) prefix[i] = block_sums[blockIdx.x] + s_w[threadIdx.x >> 5] + inc - v;
}

// One 16-byte record per bitmap word, so that a counter update needs one load to find its slot: {+ strand bits, - strand bits,
// slot of the word's first + bit, slot of its first - bit}, from the ranked [2][n_words] per-strand bitmaps (the - strand slots
// follow all + strand slots).
__global__ void k_word_record(const uint32_t* __restrict__ bits, const uint32_t* __restrict__ prefix, uint32_t n_words, uint4* __restrict__ rec) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_words) rec[i] = make_uint4(bits[i], bits[n_words + i], prefix[i], prefix[n_words + i]);
}

// counter slot of (bit `bit` of the word, reference strand t); ~0u: the pair has none
__device__ __forceinline__ uint32_t wslot(const uint4& r, uint32_t t, uint32_t bit) {
    const uint32_t bm = t == 0 ? r.x : r.y;
    if (!((bm >> bit) & 1u)) return 0xffffffffu;
    return (t == 0 ? r.z : r.w) + __popc(bm & ((1u << bit) - 1u));
}

// One work item of k_count_bases: the part [r_lo, r_hi) of a read's reference span inside the chunk, where r_hi is the next
// item's r_lo when that item belongs to the same read, else the chunk end. op is the first CIGAR op whose reference end is past
// r_lo, q and r its query and reference start. A read gets one item per window of S reference bases (k_items_count), and the
// seams between its items lie on the chunk's 32-position word grid, so no bitmap word is split between two items.
struct CountItem { uint32_t read, r_lo, op, q, r; };

// items of a read whose span clipped to the chunk is [cs + a, cs + b), a < b: one if it is at most S long, else one per S
// bases from the word that holds its start (the seams: cs + (a & ~31) + j * S, j >= 1)
__host__ __device__ __forceinline__ uint32_t count_items_of(uint32_t a, uint32_t b, uint32_t S) {
    return b - a <= S ? 1u : (b - 1u - (a & ~31u)) / S + 1u;
}

// warp per read: the read's reference span clipped to [cs, ce) and the number of its items (0 when it misses the chunk)
__global__ void __launch_bounds__(256) k_items_count(const mkp_read_hdr* __restrict__ hdrs, const uint8_t* __restrict__ heap, uint32_t n_reads,
                                                     uint32_t cs, uint32_t ce, uint32_t S, uint32_t* __restrict__ n_items) {
    const uint32_t ri = blockIdx.x * 8 + (threadIdx.x >> 5), lane = lane_id();
    if (ri >= n_reads) return;
    const mkp_read_hdr h = hdrs[ri];
    const uint32_t* cig = (const uint32_t*)(heap + h.off);
    uint32_t rc = (uint32_t)h.ref_start;
    for (uint32_t b0 = 0; b0 < h.n_cigar && rc < ce; b0 += 32) {      // (the part past the chunk end is not needed)
        const uint32_t i = b0 + lane, c = i < h.n_cigar ? cig[i] : 0, op = c & 15;
        rc += __reduce_add_sync(FULL, cig_rlen(op, c >> 4));
    }
    const uint32_t lo = (uint32_t)h.ref_start > cs ? (uint32_t)h.ref_start : cs, hi = rc < ce ? rc : ce;
    if (lane == 0) n_items[ri] = lo < hi ? count_items_of(lo - cs, hi - cs, S) : 0u;
}

// warp per read: the read's items at base[ri] ..; the lane whose op holds a seam writes that item
__global__ void __launch_bounds__(256) k_items_fill(const mkp_read_hdr* __restrict__ hdrs, const uint8_t* __restrict__ heap, uint32_t n_reads,
                                                    uint32_t cs, uint32_t S, const uint32_t* __restrict__ base, CountItem* __restrict__ items) {
    const uint32_t ri = blockIdx.x * 8 + (threadIdx.x >> 5), lane = lane_id();
    if (ri >= n_reads) return;
    const uint32_t n = base[ri + 1] - base[ri];
    if (!n) return;
    const mkp_read_hdr h = hdrs[ri];
    const uint32_t* cig = (const uint32_t*)(heap + h.off);
    const uint32_t lo = (uint32_t)h.ref_start > cs ? (uint32_t)h.ref_start : cs, a0 = (lo - cs) & ~31u;
    const uint32_t last = n == 1 ? lo : cs + a0 + (n - 1) * S;           // the last seam
    CountItem* out = items + base[ri];
    uint32_t qc = 0, rc = (uint32_t)h.ref_start;
    for (uint32_t b0 = 0; b0 < h.n_cigar && rc <= last; b0 += 32) {
        const uint32_t i = b0 + lane, c = i < h.n_cigar ? cig[i] : 0, op = c & 15, len = c >> 4;
        const uint32_t ql = cig_qlen(op, len), rl = cig_rlen(op, len);
        const uint32_t qi = warp_incl_scan(ql), rr = warp_incl_scan(rl);
        const uint32_t q0 = qc + qi - ql, r0 = rc + rr - rl, e = r0 + rl;
        qc += __shfl_sync(FULL, qi, 31);
        rc += __shfl_sync(FULL, rr, 31);
        for (uint32_t j = r0 <= lo ? 0u : (r0 - cs - a0 + S - 1u) / S; rl && j < n; j++) {   // the seams in [r0, e)
            const uint32_t s = j ? cs + a0 + j * S : lo;
            if (s >= e) break;
            CountItem it; it.read = ri; it.r_lo = s; it.op = i; it.q = q0; it.r = r0;
            out[j] = it;
        }
    }
}

struct CountDev {
    const mkp_read_hdr* hdrs;
    const uint8_t* heap;
    const ReadMeta* meta;
    const uint2* calls;
    uint32_t n_reads, cs, ce;
    const uint4* rec;   // per bitmap word (k_word_record)
    uint32_t* slots;
    uint32_t stride;    // words per slot
    uint32_t n_states;
    uint32_t n_words;
    uint32_t* obs_word;   // [2][n_words] observed-code masks of fully covered bitmap words
    uint32_t* work;       // dynamic read / item counter
    const uint32_t* list; // list mode: the reads to count (k_pileup_fused counted the others) and their number
    const uint32_t* list_count;
    const uint32_t* order; // else (k_count_calls): processing order (longest reads first), or null
    const CountItem* items;   // else (k_count_bases): the chunk's work items, in coordinate order
    uint32_t n_items;
};

// MKP_COUNT_CLOCKS=1 (measurement builds only): k_count_bases logs every work item it takes from the queue into
// g_count_clk[queue index] (when below g_count_clk_cap): the SM, %globaltimer at dequeue and at the warp's next dequeue, the read
// and [r_lo, r_hi). %globaltimer, not clock64(): SM clocks are not comparable across SMs. Read back by mkp_debug_count_clocks.
#ifdef MKP_COUNT_CLOCKS
struct CountClk { unsigned long long t0, t1; uint32_t sm, read, r_lo, r_hi; };
__device__ CountClk* g_count_clk;
__device__ uint32_t g_count_clk_cap;
__device__ __forceinline__ unsigned long long global_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// (the pending record lives in shared memory, so the measured kernel keeps the register budget of the default build)
#define CCLK_INIT __shared__ CountClk s_cclk[8]; __shared__ uint32_t s_cclk_i[8]; if (lane == 0) s_cclk_i[wib] = 0xffffffffu
#define CCLK_DEQ(ii) do { if (lane == 0) { const unsigned long long t_ = global_ns(); const uint32_t p_ = s_cclk_i[wib]; \
    if (p_ < g_count_clk_cap) { s_cclk[wib].t1 = t_; g_count_clk[p_] = s_cclk[wib]; } \
    uint32_t sm_; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm_)); s_cclk[wib].t0 = t_; s_cclk[wib].sm = sm_; s_cclk_i[wib] = (ii); } } while (0)
#define CCLK_ITEM(ri, lo, hi) do { if (lane == 0) { s_cclk[wib].read = (ri); s_cclk[wib].r_lo = (lo); s_cclk[wib].r_hi = (hi); } } while (0)
#else
#define CCLK_INIT do {} while (0)
#define CCLK_DEQ(ii) do {} while (0)
#define CCLK_ITEM(ri, lo, hi) do {} while (0)
#endif

// FeatureVector::add_feature + Tally::add_feature (src/pileup/mod.rs:176-193, 238-281) as counter updates, on reference strand t
// at bit `bit` of the word with record r
__device__ __forceinline__ void add_feature(uint32_t* slots, uint32_t stride, const uint4& r, uint32_t bit, uint32_t t, uint32_t pb, uint32_t state, uint32_t delta) {
    const uint32_t k = wslot(r, t, bit);
    if (k == 0xffffffffu) return;
    uint32_t* S = slots + (size_t)k * stride;
    if (state == 0) atomicAdd(&S[SL_FILT], delta);
    else if (state == 1) atomicAdd(&S[SL_CANON + pb], delta);
    else atomicAdd(&S[SL_MOD + (state - 2)], delta);
}

// warp per read, lanes over its call records
__global__ void __launch_bounds__(256) k_count_calls(CountDev D) {
    const uint32_t lane = lane_id();
    for (;;) {
        uint32_t ri = 0;
        if (lane == 0) { ri = atomicAdd(D.work + 1, 1u); if (D.list) ri = ri < *D.list_count ? D.list[ri] : 0xffffffffu; else if (D.order && ri < D.n_reads) ri = D.order[ri]; }
        ri = __shfl_sync(FULL, ri, 0);
        if (ri >= D.n_reads) break;
        const ReadMeta m = D.meta[ri];
        if (!(m.flags & 2) || m.n_calls == 0) continue;
#ifndef MKP_NO_FUSED_CALLS
        if (m.flags & 4) continue;                 // one sorted run of records: counted by k_count_bases while it streams them
#endif
        const uint32_t a = (D.hdrs[ri].flags & 0x10) ? 1u : 0u;
        const uint2* calls = D.calls + m.entry_off;
        for (uint32_t k = lane; k < m.n_calls; k += 32) {
            uint2 c = calls[k];
            uint32_t x = c.x - D.cs;
            uint32_t info = c.y;
            const uint32_t st = call_strand(info), b = call_base(info), state = call_state(info), nosub = call_nosub(info);
            const uint4 r = D.rec[x >> 5];                     // (a pair outside the focus set has no slot)
            const uint32_t bit = x & 31, t = st == 0 ? a : 1u - a, pbb = st == 0 ? b : 3u - b;
            // cancel what k_count_bases adds for this (read, position): the inferred entry of this table if the
            // table is implicit, else the NoCall base on tally[a] (unless the other strand's table is implicit
            // there, in which case no NoCall is counted, or the '+' record of a +/- pair already cancels it)
            const uint32_t imp_own = (m.imp[st] >> (8 * b)) & 0xffu, imp_other = (m.imp[1 - st] >> (8 * b)) & 0xffu;
            if (imp_own & 0x80u) add_feature(D.slots, D.stride, r, bit, t, pbb, imp_own & 0x7fu, 0xffffffffu);
            else if (!(m.flags & 4) && !(imp_other & 0x80u) && !nosub) {
                const uint32_t k = wslot(r, a, bit);
                if (k != 0xffffffffu) atomicAdd(&D.slots[(size_t)k * D.stride + SL_BASE + b], 0xffffffffu);
            }
            add_feature(D.slots, D.stride, r, bit, t, pbb, state, 1u);
        }
    }
}

// warp per work item (the part [r_lo, r_hi) of a read, CountItem; one item per read in list mode): every aligned base / deleted
// position that lands on a hot position, plus the observed-code coverage of the read (src/pileup/mod.rs:831-835: unioned for every
// alignment at the position, deletions included, reference skips excluded).  Coverage is recorded per 32-position bitmap word when
// the read covers the whole word (one coalesced check-then-OR per word) and per hot position only in the partial words at the ends
// of a run. The items keep coordinate order, so that neighbouring warps update neighbouring counter slots, and a long read is
// several items, so that it does not form the kernel's tail when it is dequeued late.
__global__ void __launch_bounds__(256, MKP_MINB_BASES) k_count_bases(CountDev D) {
    __shared__ uint32_t s_op[8][32], s_q[8][32], s_r[8][33];   // the current batch of 32 ops: op|len<<4, query start, reference start
    __shared__ uint32_t s_mask[8][32];                          // positions of the current 32 words where this read has a call
    __shared__ uint32_t s_lim[8][2];                            // the item's [r_lo, r_hi) (kept out of the walk's registers)
    const uint32_t lane = lane_id();
    const uint32_t wib = threadIdx.x >> 5;
    CCLK_INIT;
    for (;;) {
        uint32_t ii = 0;
        if (lane == 0) ii = atomicAdd(D.work, 1u);
        ii = __shfl_sync(FULL, ii, 0);
        CCLK_DEQ(ii);
        uint32_t ri, r_lo, r_hi;
        CountItem it;
        if (D.list) {
            ri = ii < *D.list_count ? D.list[ii] : 0xffffffffu;
            if (ri >= D.n_reads) break;
            r_lo = 0; r_hi = D.ce;                              // (r_lo, the op and its start are the read's, below)
        } else {
            if (ii >= D.n_items) break;
            it = D.items[ii];
            ri = it.read; r_lo = it.r_lo;
            r_hi = D.ce;
            if (ii + 1 < D.n_items) { const CountItem nx = D.items[ii + 1]; if (nx.read == ri) r_hi = nx.r_lo; }
        }
        const ReadMeta m = D.meta[ri];
        if (!(m.flags & 1)) continue;
        const mkp_read_hdr h = D.hdrs[ri];
        if ((uint32_t)m.ref_end <= D.cs || (uint32_t)h.ref_start >= D.ce) continue;
        const uint32_t lo_read = (uint32_t)h.ref_start > D.cs ? (uint32_t)h.ref_start : D.cs;
        if (D.list) { r_lo = lo_read; it.op = 0; it.q = 0; it.r = (uint32_t)h.ref_start; }
        CCLK_ITEM(ri, r_lo, r_hi);
        __syncwarp();
        if (lane == 0) { s_lim[wib][0] = r_lo; s_lim[wib][1] = r_hi; }
        const uint32_t a = (h.flags & 0x10) ? 1u : 0u;
        const uint32_t* cig = (const uint32_t*)(D.heap + h.off);
        const uint8_t* seq = D.heap + h.off + 4ull * h.n_cigar;
        const bool has_mods = m.flags & 2;
        const bool has_imp = (m.imp[0] | m.imp[1]) != 0;
        const uint32_t pm = has_mods ? m.pos_mask : 0u, nm = has_mods ? m.neg_mask : 0u;
        const bool merge = has_mods && (m.flags & 4) && m.n_calls > 0;
        const uint2* rcalls = D.calls + m.entry_off;
        // call records consumed so far (ascending position): on a later item of the read, the first record at or after r_lo
        uint32_t cp = 0;
        if (merge && r_lo > lo_read) {
            uint32_t hi_k = m.n_calls;
            while (cp < hi_k) { const uint32_t mid = (cp + hi_k) >> 1; if (rcalls[a ? m.n_calls - 1u - mid : mid].x < r_lo) cp = mid + 1; else hi_k = mid; }
        }
        // observed-code coverage of one run [ra, rb) of reference positions, inside the item
        auto cover = [&](uint32_t ra, uint32_t rb) {
            if (!(pm | nm)) return;
            if (ra < s_lim[wib][0]) ra = s_lim[wib][0];
            if (rb > s_lim[wib][1]) rb = s_lim[wib][1];
            if (ra >= rb) return;
            const uint32_t wl = (ra - D.cs + 31) >> 5, wh = (rb - D.cs) >> 5;   // words [wl, wh) are fully covered
            for (uint32_t w = wl + lane; w < wh; w += 32) {
                if (pm && (D.obs_word[w] & pm) != pm) atomicOr(&D.obs_word[w], pm);
                if (nm && (D.obs_word[D.n_words + w] & nm) != nm) atomicOr(&D.obs_word[D.n_words + w], nm);
            }
            // partial words: lane = bit
            auto partial = [&](uint32_t pa, uint32_t pb) {     // [pa,pb) lies inside one bitmap word
                if (pa >= pb) return;
                const uint32_t w = (pa - D.cs) >> 5, wbase = D.cs + (w << 5);
                const uint4 r = D.rec[w];
                uint32_t bits = (r.x | r.y) & (FULL << (pa - wbase));
                if (pb < wbase + 32) bits &= (1u << (pb - wbase)) - 1u;
                if ((bits >> lane) & 1u) {
                    const uint32_t kp = pm ? wslot(r, 0, lane) : 0xffffffffu, kn = nm ? wslot(r, 1, lane) : 0xffffffffu;
                    if (kp != 0xffffffffu) { uint32_t* S = D.slots + (size_t)kp * D.stride; if ((S[SL_OBS] & pm) != pm) atomicOr(&S[SL_OBS], pm); }
                    if (kn != 0xffffffffu) { uint32_t* S = D.slots + (size_t)kn * D.stride; if ((S[SL_OBS] & nm) != nm) atomicOr(&S[SL_OBS], nm); }
                }
            };
            if (wl > wh) partial(ra, rb);                       // the run starts and ends inside one word
            else { partial(ra, D.cs + (wl << 5)); partial(D.cs + (wh << 5), rb); }
        };
        uint32_t qc = it.q, rc = it.r;
        uint32_t run_start = rc;                                // start of the current run without reference skips
        for (uint32_t b0 = it.op; b0 < h.n_cigar; b0 += 32) {
            uint32_t i = b0 + lane;
            uint32_t c = i < h.n_cigar ? cig[i] : 0;
            uint32_t op = c & 15, len = c >> 4;
            uint32_t ql = cig_qlen(op, len), rl = cig_rlen(op, len);
            uint32_t qi = warp_incl_scan(ql), rr = warp_incl_scan(rl);
            uint32_t q0 = qc + qi - ql, r0 = rc + rr - rl;
            qc += __shfl_sync(FULL, qi, 31);
            rc += __shfl_sync(FULL, rr, 31);
            // reference skips ('N') end a covered run
            uint32_t skips = __ballot_sync(FULL, op == 3 && len > 0 && i < h.n_cigar);
            while (skips) {
                const int sl = __ffs(skips) - 1;
                skips &= skips - 1;
                const uint32_t sr = __shfl_sync(FULL, r0, sl), slen = __shfl_sync(FULL, len, sl);
                cover(run_start, sr);
                run_start = sr + slen;
            }
            // hot-bitmap words under this batch of ops, one per lane: the word is tested first (most hold no position this
            // read can add to); the op under a hot position is found by one search per word over the batch's reference
            // starts, then by stepping forward. Only M,=,X (a base) and D (a deletion) count.
            const uint32_t R0 = __shfl_sync(FULL, r0, 0), R1 = rc;
            s_op[wib][lane] = op | (len << 4); s_q[wib][lane] = q0; s_r[wib][lane] = r0;
            if (lane == 0) s_r[wib][32] = R1;
            __syncwarp();
            const uint32_t r_lo_ = s_lim[wib][0], r_hi_ = s_lim[wib][1];
            const uint32_t blo = R0 > r_lo_ ? R0 : r_lo_, bhi = R1 < r_hi_ ? R1 : r_hi_;
            if (blo < bhi) {
                const uint32_t w_first = (blo - D.cs) >> 5, w_last = (bhi - 1 - D.cs) >> 5;
                for (uint32_t wt = w_first; wt <= w_last; wt += 32) {
                    const uint32_t w = wt + lane;
                    // reads whose call records form one run sorted by position (flag 4): a position with a call needs no
                    // NoCall (k_count_calls does not cancel one for these reads), so the calls under these 32 words are
                    // streamed in (one cursor per read, ascending positions) and masked out before the per-position work
                    uint32_t called = 0;
                    if (merge) {
                        const uint32_t t_end = D.cs + ((wt + 32) << 5);
                        const uint32_t lim = bhi < t_end ? bhi : t_end;
                        s_mask[wib][lane] = 0;
                        __syncwarp();
                        for (;;) {
                            const uint32_t k = cp + lane;
                            uint32_t x = 0xffffffffu, info = 0;
                            if (k < m.n_calls) { const uint2 c = rcalls[a ? m.n_calls - 1u - k : k]; x = c.x; info = c.y; }
                            const bool take = x < lim;
                            if (take) {
                                const uint32_t rel = x - D.cs;
                                if ((rel >> 5) >= wt) atomicOr(&s_mask[wib][(rel >> 5) - wt], 1u << (rel & 31));
#ifndef MKP_NO_FUSED_CALLS
                                // the record's own counter (k_count_calls leaves these reads alone): modcall / canonical / filtered
                                const uint32_t st = call_strand(info), cb = call_base(info), state = call_state(info);
                                add_feature(D.slots, D.stride, D.rec[rel >> 5], rel & 31, st == 0 ? a : 1u - a, st == 0 ? cb : 3u - cb, state, 1u);
#endif
                            }
                            const uint32_t nt = __popc(__ballot_sync(FULL, take));
                            cp += nt;
                            if (nt < 32) break;
                        }
                        __syncwarp();
                        called = s_mask[wib][lane];
                    }
                    if (w > w_last) continue;
                    const uint4 wr = D.rec[w];
                    const uint32_t word = wr.x | wr.y;
                    if (!word) continue;
                    const uint32_t wbase = D.cs + (w << 5);
                    uint32_t bits = word & ~called;
                    if (blo > wbase) bits &= FULL << (blo - wbase);
                    if (bhi < wbase + 32) bits &= (1u << (bhi - wbase)) - 1u;
                    if (!bits) continue;
                    // positions with a slot on the read's strand (only implicit tables add to the other strand)
                    const uint32_t ok = a == 0 ? wr.x : wr.y, pre = a == 0 ? wr.z : wr.w;
                    if (!has_imp) bits &= ok;
                    if (!bits) continue;
                    // op under the first candidate position: largest j with s_r[j] <= r (ops without reference length share
                    // their start with the next op, so the largest index is the op that holds r)
                    uint32_t j = 0;
                    {
                        const uint32_t r = wbase + (uint32_t)__ffs(bits) - 1u;
#pragma unroll
                        for (int stp = 16; stp >= 1; stp >>= 1) if (s_r[wib][j + stp] <= r) j += stp;
                    }
                    while (bits) {
                        const uint32_t bit = __ffs(bits) - 1;
                        bits &= bits - 1;
                        const uint32_t r = wbase + bit;
                        while (s_r[wib][j + 1] <= r) j++;
                        const uint32_t jc = s_op[wib][j], jop = jc & 15;
                        if (!(cig_is_match(jop) || jop == 2)) continue;       // reference skip
                        if (jop == 2 && !((ok >> bit) & 1u)) continue;
                        uint32_t* S = D.slots + (size_t)(pre + __popc(ok & ((1u << bit) - 1u))) * D.stride;   // (when ok has the bit)
                        if (jop == 2) { atomicAdd(&S[SL_DEL], 1u); continue; }
                        const uint32_t q = s_q[wib][j] + (r - s_r[wib][j]);
                        const int nb = nib_to_base(seq_nibble(seq, q));
                        if (nb > 3) continue;
                        const uint32_t b = a ? 3 - nb : nb;
                        if (!has_imp) { atomicAdd(&S[SL_BASE + b], 1u); continue; }
                        uint32_t ip = (m.imp[0] >> (8 * b)) & 0xffu, in = (m.imp[1] >> (8 * b)) & 0xffu;
                        if ((ip | in) & 0x80u) {
                            // inferred-canonical entries of implicit tables, subject to the edge filter
                            const uint32_t f = a ? h.l_seq - 1u - q : q;
                            if (!edge_keep(f, h.l_seq)) ip = in = 0;
                        }
                        if (!((ip | in) & 0x80u)) { if ((ok >> bit) & 1u) atomicAdd(&S[SL_BASE + b], 1u); continue; }
                        if (ip & 0x80u) add_feature(D.slots, D.stride, wr, bit, a, b, ip & 0x7fu, 1u);
                        if (in & 0x80u) add_feature(D.slots, D.stride, wr, bit, 1u - a, 3u - b, in & 0x7fu, 1u);
                    }
                }
            }
            __syncwarp();
            if (rc >= s_lim[wib][1]) break;                     // the rest of the read is the next item's
        }
        cover(run_start, rc);
    }
}

struct RowDev {
    const uint4* rec;         // per bitmap word (k_word_record)
    uint32_t n_words, cs, ce;
    const uint32_t* slots;
    uint32_t stride, n_states;
    const unsigned long long* states;
    uint32_t numeric_mode;
    const uint32_t* obs_word;
    uint32_t* row_counts;     // per hot-bitmap word
    const uint32_t* row_prefix;
    mkp_row* rows;
    uint32_t rows_cap;        // emit pass: a word whose rows do not fit is skipped (the host grows the buffer and emits again)
};

// rows of the slot S of (pos, strand s), in output order. emit == nullptr => count only
__device__ __forceinline__ uint32_t slot_rows(const RowDev& R, const uint32_t* S, uint32_t pos, uint32_t w, uint32_t s, mkp_row* out) {
    uint32_t n = 0;
    uint32_t mod_by_base[4] = {0, 0, 0, 0};
    for (uint32_t id = 0; id < R.n_states; id++) mod_by_base[(uint32_t)(R.states[id] >> 32) & 3u] += S[SL_MOD + id];
    const uint32_t obs = S[SL_OBS] | R.obs_word[s * R.n_words + w];
    for (uint32_t pb = 0; pb < 4; pb++) {
        uint32_t n_can = S[SL_CANON + pb], total_mod = mod_by_base[pb];
        if (n_can + total_mod == 0) continue;
        uint32_t n_diff = 0;
        for (uint32_t b = 0; b < 4; b++) if (b != pb) n_diff += S[SL_BASE + b] + S[SL_CANON + b] + mod_by_base[b];
        mkp_row r;
        r.pos = pos; r.strand = s == 0 ? '+' : '-'; r.primary_base = (uint8_t)pb; r.reserved = 0;
        r.n_canon = n_can; r.n_delete = S[SL_DEL]; r.n_filtered = S[SL_FILT]; r.n_diff = n_diff; r.n_nocall = S[SL_BASE + pb];
        if (R.numeric_mode == 1) {
            r.code = (uint32_t)("ACGT"[pb]); r.n_mod = total_mod; r.n_other = 0;
            if (out) out[n] = r;
            n++;
        } else {
            for (uint32_t id = 0; id < R.n_states; id++) {
                unsigned long long key = R.states[id];
                if (((uint32_t)(key >> 32) & 3u) != pb || !((obs >> id) & 1u)) continue;
                uint32_t n_mod = S[SL_MOD + id];
                r.code = (uint32_t)key; r.n_mod = n_mod; r.n_other = total_mod - n_mod;
                if (out) out[n] = r;
                n++;
            }
        }
    }
    // stable insertion sort of this strand's rows by code (derived Ord: Code(char) < ChEbi == u32 order)
    if (out) for (uint32_t i = 1; i < n; i++) {
        mkp_row key = out[i];
        uint32_t j = i;
        while (j > 0 && out[j - 1].code > key.code) { out[j] = out[j - 1]; j--; }
        out[j] = key;
    }
    return n;
}

// thread per hot-bitmap word; rows by position, + strand before - strand
template <bool EMIT>
__global__ void __launch_bounds__(256) k_rows(RowDev R) {
    uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= R.n_words) return;
    const uint4 wr = R.rec[w];
    uint32_t bits = wr.x | wr.y;
    if (!bits) { if (!EMIT) R.row_counts[w] = 0; return; }
    uint32_t slot_p = wr.z, slot_n = wr.w;
    uint32_t n = 0;
    if (EMIT && (unsigned long long)R.row_prefix[w] + R.row_counts[w] > (unsigned long long)R.rows_cap) return;
    mkp_row* out = EMIT ? R.rows + R.row_prefix[w] : nullptr;
    while (bits) {
        uint32_t bit = __ffs(bits) - 1;
        bits &= bits - 1;
        const uint32_t pos = R.cs + (w << 5) + bit;
        if ((wr.x >> bit) & 1u) n += slot_rows(R, R.slots + (size_t)slot_p++ * R.stride, pos, w, 0, EMIT ? out + n : nullptr);
        if ((wr.y >> bit) & 1u) n += slot_rows(R, R.slots + (size_t)slot_n++ * R.stride, pos, w, 1, EMIT ? out + n : nullptr);
    }
    if (!EMIT) R.row_counts[w] = n;
}

// exclusive scan of arbitrary u32 array via the same 3-kernel scheme (counts -> prefix)
__global__ void k_block_sum(const uint32_t* __restrict__ v, uint32_t n, uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t s[32];
    uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    uint32_t x = i < n ? v[i] : 0;
    uint32_t w = __reduce_add_sync(FULL, x);
    if (lane_id() == 0) s[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x < 32) { uint32_t t = __reduce_add_sync(FULL, s[threadIdx.x]); if (threadIdx.x == 0) block_sums[blockIdx.x] = t; }
}
__global__ void k_value_prefix(const uint32_t* __restrict__ v, uint32_t n, const uint32_t* __restrict__ block_sums, uint32_t* __restrict__ prefix) {
    __shared__ uint32_t s_w[32];
    uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    uint32_t x = i < n ? v[i] : 0;
    uint32_t inc = warp_incl_scan(x);
    if (lane_id() == 31) s_w[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) { uint32_t t = s_w[threadIdx.x]; uint32_t ti = warp_incl_scan(t); s_w[threadIdx.x] = ti - t; }
    __syncthreads();
    if (i < n) prefix[i] = block_sums[blockIdx.x] + s_w[threadIdx.x >> 5] + inc - x;
}

// ---- pileup-hemi (src/pileup/duplex.rs, src/read_cache.rs:368-468) ---------------------------------------------------------
// Per + strand motif position p (the chunk's focus_pos bitmap) and admitted read: a deletion counts n_delete; an ACGT SEQ base
// pairs the read's call on the + strand at p with its call on the - strand at p + partner, looked up in the table of the
// complementary base. Counter slot of a position = its rank in focus_pos; layout (u32): [0] n_delete, then per primary base
// (SEQ base at p) [filtered, nocall, pattern[pos side][neg side]], side 0 = canonical, 1 + id = mod state id.
struct HemiDev {
    const mkp_read_hdr* hdrs;
    const uint8_t* heap;
    const ReadMeta* meta;
    const uint2* calls;
    uint32_t n_reads, cs, ce;              // call window (the focus bits lie inside it)
    const uint32_t* focus; const uint32_t* focus_prefix;
    const uint32_t* iv_start; uint32_t n_iv;   // starts of the chunk's intervals, non-decreasing
    int32_t partner;                       // reverse offset - forward offset of the motif
    uint32_t* slots;
    uint32_t stride, n_sides;              // n_sides = n_states + 1
    uint32_t* scr_cq; uint32_t* scr_cr; uint32_t scr_stride;   // per-warp CIGAR prefix (query / reference start of every op)
    uint32_t* work;
};

__host__ __device__ __forceinline__ uint32_t hemi_base_words(uint32_t n_sides) { return 2u + n_sides * n_sides; }

// warp per read. The read's call records are one monotone run per MM list (ascending positions on a forward read, descending
// on a reverse one): a lookup is one binary search per run.
__global__ void __launch_bounds__(128) k_hemi_count(HemiDev D) {
    __shared__ uint32_t s_seg[4][MAX_LISTS + 2];
    const uint32_t lane = lane_id();
    const uint32_t wib = threadIdx.x >> 5;
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t* const cq = D.scr_cq + (size_t)gw * D.scr_stride;
    uint32_t* const cr = D.scr_cr + (size_t)gw * D.scr_stride;
    const uint32_t bw = hemi_base_words(D.n_sides);
    for (;;) {
        uint32_t ri = 0;
        if (lane == 0) ri = atomicAdd(D.work, 1u);
        ri = __shfl_sync(FULL, ri, 0);
        if (ri >= D.n_reads) break;
        const ReadMeta m = D.meta[ri];
        if (!(m.flags & 1)) continue;
        const mkp_read_hdr h = D.hdrs[ri];
        if ((uint32_t)m.ref_end <= D.cs || (uint32_t)h.ref_start >= D.ce) continue;
        const uint32_t lo_r = (uint32_t)h.ref_start > D.cs ? (uint32_t)h.ref_start : D.cs;
        const uint32_t hi_r = (uint32_t)m.ref_end < D.ce ? (uint32_t)m.ref_end : D.ce;
        const uint32_t a = (h.flags & 0x10) ? 1u : 0u;
        const bool failed = !(m.flags & 2);           // skip_set: no usable mod info
        const uint32_t* cig = (const uint32_t*)(D.heap + h.off);
        const uint8_t* seq = D.heap + h.off + 4ull * h.n_cigar;
        const uint32_t nc = h.n_cigar;
        __syncwarp();
        {
            uint32_t qc = 0, rc = (uint32_t)h.ref_start;
            for (uint32_t b0 = 0; b0 < nc; b0 += 32) {
                const uint32_t i = b0 + lane;
                const uint32_t c = i < nc ? cig[i] : 0u, op = c & 15, len = c >> 4;
                const uint32_t ql = cig_qlen(op, len), rl = cig_rlen(op, len);
                const uint32_t qi = warp_incl_scan(ql), rr = warp_incl_scan(rl);
                if (i < nc) { cq[i] = qc + qi - ql; cr[i] = rc + rr - rl; }
                qc += __shfl_sync(FULL, qi, 31);
                rc += __shfl_sync(FULL, rr, 31);
            }
        }
        // monotone runs of the records: s_seg[0..n_seg] are their boundaries
        const uint2* rcalls = D.calls + m.entry_off;
        const uint32_t n = failed ? 0u : m.n_calls;
        uint32_t n_seg = 1;
        if (lane == 0) s_seg[wib][0] = 0;
        for (uint32_t k0 = 1; k0 < n; k0 += 32) {
            const uint32_t k = k0 + lane;
            bool brk = false;
            if (k < n) { const uint32_t x1 = rcalls[k].x, x0 = rcalls[k - 1].x; brk = a ? x1 > x0 : x1 < x0; }
            const uint32_t bm = __ballot_sync(FULL, brk);
            if (brk) { const uint32_t at = n_seg + __popc(bm & ((1u << lane) - 1u)); if (at <= MAX_LISTS) s_seg[wib][at] = k; }
            n_seg += __popc(bm);
        }
        if (n_seg > MAX_LISTS) n_seg = MAX_LISTS;     // (one run per MM list, at most MAX_LISTS lists)
        if (lane == 0) s_seg[wib][n_seg] = n;
        __syncwarp();
        // the op under reference position r: 0 none (outside, reference skip), 1 aligned base at query *q, 2 deletion
        auto op_at = [&](uint32_t r, uint32_t* q) -> uint32_t {
            if (nc == 0 || r < cr[0]) return 0;
            uint32_t lo = 0, hi = nc;
            while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (cr[mid] <= r) lo = mid; else hi = mid; }
            const uint32_t c = cig[lo], op = c & 15, len = c >> 4;
            if (r >= cr[lo] + len) return 0;
            if (cig_is_match(op)) { *q = cq[lo] + (r - cr[lo]); return *q < h.l_seq ? 1u : 0u; }
            return op == 2 ? 2u : 0u;
        };
        // the read's call at r on mod strand st, forward base cb: state + 1 (1 filtered, 2 canonical, 3 + id), 0 = none
        auto call_at = [&](uint32_t r, uint32_t q, uint32_t st, uint32_t cb) -> uint32_t {
            for (uint32_t s = 0; s < n_seg; s++) {
                const uint32_t end = s_seg[wib][s + 1];
                uint32_t lo = s_seg[wib][s], hi = end;
                while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; const uint32_t x = rcalls[mid].x; if (a ? x > r : x < r) lo = mid + 1; else hi = mid; }
                for (uint32_t k = lo; k < end; k++) {
                    const uint2 c = rcalls[k];
                    if (c.x != r) break;
                    if (call_strand(c.y) == st && call_base(c.y) == cb) return call_state(c.y) + 1u;
                }
            }
            // implicit table: every other occurrence of its base is an inferred-canonical entry, subject to the edge filter
            const uint32_t imp = (m.imp[st] >> (8 * cb)) & 0xffu;
            if (!(imp & 0x80u)) return 0;
            const uint32_t f = a ? h.l_seq - 1u - q : q;
            if (!edge_keep(f, h.l_seq)) return 0;
            return (imp & 0x7fu) + 1u;
        };
        if (lo_r >= hi_r) continue;
        const uint32_t w0 = (lo_r - D.cs) >> 5, w1 = (hi_r - 1 - D.cs) >> 5;
        auto word_bits = [&](uint32_t w) {
            uint32_t bits = D.focus[w];
            const uint32_t wbase = D.cs + (w << 5);
            if (lo_r > wbase) bits &= FULL << (lo_r - wbase);
            if (hi_r < wbase + 32) bits &= (1u << (hi_r - wbase)) - 1u;
            return bits;
        };
        auto slot = [&](uint32_t w, uint32_t bit) { return D.slots + (size_t)(D.focus_prefix[w] + __popc(D.focus[w] & ((1u << bit) - 1u))) * D.stride; };
        if (!failed) {
            for (uint32_t w = w0 + lane; w <= w1; w += 32) {
                uint32_t bits = word_bits(w);
                while (bits) {
                    const uint32_t bit = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const uint32_t r = D.cs + (w << 5) + bit;
                    uint32_t q = 0;
                    const uint32_t kind = op_at(r, &q);
                    if (!kind) continue;
                    uint32_t* S = slot(w, bit);
                    if (kind == 2) { atomicAdd(&S[0], 1u); continue; }
                    const int nb = nib_to_base(seq_nibble(seq, q));
                    if (nb > 3) continue;
                    uint32_t* B = S + 1 + (uint32_t)nb * bw;
                    const uint32_t cb = a ? 3u - (uint32_t)nb : (uint32_t)nb;
                    const uint32_t vp = call_at(r, q, a, cb);
                    uint32_t vn = 0;
                    const int64_t rn = (int64_t)r + D.partner;
                    if (vp && rn >= 0) {
                        uint32_t qn = 0;
                        if (op_at((uint32_t)rn, &qn) == 1 && nib_to_base(seq_nibble(seq, qn)) == 3 - nb) vn = call_at((uint32_t)rn, qn, 1u - a, 3u - cb);
                    }
                    if (!vp || !vn) atomicAdd(&B[1], 1u);
                    else if (vp == 1 || vn == 1) atomicAdd(&B[0], 1u);
                    else atomicAdd(&B[2 + (vp - 2) * D.n_sides + (vn - 2)], 1u);
                }
            }
        } else {
            // the read cache checks its skip set before the first decode: a read without usable mod info is one NoCall, at its
            // first motif position with an ACGT base in each interval (the reference's cache lives for one interval). Its
            // deletions count like any read's.
            uint32_t iv_done = 0xffffffffu;
            for (uint32_t wt = w0; wt <= w1; wt += 32) {
                const uint32_t w = wt + lane;
                uint32_t ok = 0;
                if (w <= w1) {
                    uint32_t bits = word_bits(w);
                    while (bits) {
                        const uint32_t bit = __ffs(bits) - 1;
                        bits &= bits - 1;
                        uint32_t q = 0;
                        const uint32_t kind = op_at(D.cs + (w << 5) + bit, &q);
                        if (kind == 2) atomicAdd(&slot(w, bit)[0], 1u);
                        else if (kind == 1 && nib_to_base(seq_nibble(seq, q)) <= 3) ok |= 1u << bit;
                    }
                }
                uint32_t lanes = __ballot_sync(FULL, ok != 0);
                while (lanes) {
                    const uint32_t src = __ffs(lanes) - 1;
                    lanes &= lanes - 1;
                    uint32_t bits = __shfl_sync(FULL, ok, src);
                    while (bits) {
                        const uint32_t bit = __ffs(bits) - 1;
                        bits &= bits - 1;
                        const uint32_t r = D.cs + ((wt + src) << 5) + bit;
                        uint32_t lo = 0, hi = D.n_iv;          // interval of r: the last start <= r
                        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (D.iv_start[mid] <= r) lo = mid; else hi = mid; }
                        if (lo == iv_done) continue;
                        iv_done = lo;
                        if (lane == 0) {
                            uint32_t q = 0;
                            op_at(r, &q);
                            const uint32_t nb = (uint32_t)nib_to_base(seq_nibble(seq, q));
                            atomicAdd(&slot(wt + src, bit)[1 + nb * bw + 1], 1u);
                        }
                    }
                }
            }
        }
    }
}

struct HemiRowDev {
    const uint32_t* focus; const uint32_t* focus_prefix;
    uint32_t n_words, cs;
    const uint32_t* slots;
    uint32_t stride, n_sides;
    const unsigned long long* states;   // registry: (pb << 32 | code)
    uint32_t combine;                   // --combine-mods: mod codes -> the base's any-mod code (DuplexModCall::into_combined)
    uint32_t* row_counts;               // per focus word
    const uint32_t* row_prefix;
    mkp_hemi_row* rows;
};

// DuplexFeatureVector::decode (src/pileup/duplex.rs:121-204) of one slot, rows by base then pattern. out == nullptr => count only
__device__ uint32_t hemi_slot_rows(const HemiRowDev& R, const uint32_t* S, uint32_t pos, mkp_hemi_row* out) {
    const uint32_t ns = R.n_sides, bw = hemi_base_words(ns);
    uint32_t tot[4], all = 0;
    for (uint32_t pb = 0; pb < 4; pb++) {
        const uint32_t* B = S + 1 + pb * bw;
        uint32_t t = 0;
        for (uint32_t k = 0; k < ns * ns; k++) t += B[2 + k];
        tot[pb] = t;
        all += t;
    }
    uint32_t n = 0;
    for (uint32_t pb = 0; pb < 4; pb++) {
        if (!tot[pb]) continue;                     // a base without a pattern has no row
        const uint32_t* B = S + 1 + pb * bw;
        mkp_hemi_row r;
        r.pos = pos; r.primary_base = pb;
        r.n_canonical = B[2]; r.n_delete = S[0]; r.n_fail = B[0]; r.n_nocall = B[1]; r.n_diff = all - tot[pb];
        if (R.combine) {
            uint32_t c[2][2] = {{0, 0}, {0, 0}};
            for (uint32_t sp = 0; sp < ns; sp++) for (uint32_t sn = 0; sn < ns; sn++) c[sp > 0][sn > 0] += B[2 + sp * ns + sn];
            const uint32_t any = (uint32_t)("ACGT"[pb]);
            for (uint32_t i = 0; i < 2; i++) for (uint32_t j = 0; j < 2; j++) {
                if (!c[i][j]) continue;
                r.code_pos = i ? any : MKP_HEMI_CANONICAL; r.code_neg = j ? any : MKP_HEMI_CANONICAL;
                r.count = c[i][j]; r.n_other_pattern = tot[pb] - c[i][j];
                if (out) out[n] = r;
                n++;
            }
            continue;
        }
        const uint32_t row0 = n;
        for (uint32_t sp = 0; sp < ns; sp++) for (uint32_t sn = 0; sn < ns; sn++) {
            const uint32_t cnt = B[2 + sp * ns + sn];
            if (!cnt) continue;
            r.code_pos = sp ? (uint32_t)R.states[sp - 1] : MKP_HEMI_CANONICAL;
            r.code_neg = sn ? (uint32_t)R.states[sn - 1] : MKP_HEMI_CANONICAL;
            r.count = cnt; r.n_other_pattern = tot[pb] - cnt;
            if (out) out[n] = r;
            n++;
        }
        // insertion sort by pattern (derived Ord: Canonical < Code(char) < ChEbi, first element then second == u32 order here)
        if (out) for (uint32_t i = row0 + 1; i < n; i++) {
            const mkp_hemi_row key = out[i];
            uint32_t j = i;
            while (j > row0 && (out[j - 1].code_pos > key.code_pos || (out[j - 1].code_pos == key.code_pos && out[j - 1].code_neg > key.code_neg))) { out[j] = out[j - 1]; j--; }
            out[j] = key;
        }
    }
    return n;
}

// thread per focus word: count pass (EMIT = false), then the emit pass at the scanned offsets
template <bool EMIT>
__global__ void __launch_bounds__(256) k_hemi_rows(HemiRowDev R) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= R.n_words) return;
    uint32_t bits = R.focus[w];
    if (!bits) { if (!EMIT) R.row_counts[w] = 0; return; }
    uint32_t slot = R.focus_prefix[w];
    mkp_hemi_row* out = EMIT ? R.rows + R.row_prefix[w] : nullptr;
    uint32_t n = 0;
    while (bits) {
        const uint32_t bit = __ffs(bits) - 1;
        bits &= bits - 1;
        n += hemi_slot_rows(R, R.slots + (size_t)slot * R.stride, R.cs + (w << 5) + bit, EMIT ? out + n : nullptr);
        slot++;
    }
    if (!EMIT) R.row_counts[w] = n;
}

// ---- processing order: reads by descending length class (32 classes by the position of the top bit of l_seq); a counting sort,
//      the order inside a class does not matter (all updates are commutative integer atomics)
__global__ void k_order_hist(const mkp_read_hdr* __restrict__ hdrs, uint32_t n, uint32_t* __restrict__ hist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&hist[31 - (hdrs[i].l_seq ? 31 - __clz(hdrs[i].l_seq) : 0)], 1u);
}
__global__ void k_order_scan(uint32_t* hist) {
    uint32_t acc = 0;
    for (int b = 0; b < 32; b++) { const uint32_t v = hist[b]; hist[b] = acc; acc += v; }
}
__global__ void k_order_scatter(const mkp_read_hdr* __restrict__ hdrs, uint32_t n, uint32_t* __restrict__ hist, uint32_t* __restrict__ order) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) order[atomicAdd(&hist[31 - (hdrs[i].l_seq ? 31 - __clz(hdrs[i].l_seq) : 0)], 1u)] = i;
}

}  // namespace mkp
