// k_pileup_fused: one traversal per read, staged through shared memory by bulk async copies (TMA 1-D, sm_90a).
//
// Used when the chunk carries focus bitmaps (--cpg / --motif / --preset traditional / --include-bed): every position that can
// produce a row is known before the pass, so the counter slot of a position is the rank of its focus bit and a read can be
// decoded, projected, thresholded and counted in ONE pass over its bytes (reference: one traversal per interval,
// src/pileup/mod.rs:718-1020; per-read work: src/mod_bam.rs:900-1577, src/read_cache.rs:69-211,
// src/threshold_mod_caller.rs:28-63, src/util.rs:122-145, src/pileup/mod.rs:238-281, 831-937).
//
// Data movement. A read's block (`CIGAR | SEQ | ML | MM`, 16-byte aligned, contiguous: include/mkp.h) is the unit. One
// producer warp per CTA takes reads in runs of 32 (one coalesced load of their headers), and places every read in a
// FZ_RING-byte shared-memory ring with one `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes` per read,
// signalled on the read's own `full` mbarrier (FZ_SLOTS reads in flight). FZ_WARPS consumer warps take reads in placement
// order (a shared-memory ticket) - reads differ in length by two orders of magnitude, so no warp ever waits for another - and
// hand a read's slot back through its `empty` mbarrier; the producer reclaims ring bytes in placement order. A block longer
// than FZ_MAXBLK is not staged: that read goes to the generic kernels (`slow_list`).
//
// Per read (warp): MM header scan -> tokens -> occurrence select on the 4-bit SEQ (forward positions stay in shared
// memory) -> one walk over the CIGAR in batches of 32 ops; under every batch the read's calls are resolved (ML -> probability,
// collapse, threshold; q -> reference position by a search inside the batch) and counted straight into the slots, then the
// bases / deletions under the remaining focus positions. No P[], calls[], ReadLists or ReadMeta in HBM.
//
// Reads outside the common shape (implicit '.'/default lists, 'N' lists, '-' strand lists, lists of one base that are not
// byte-identical copies, more than two codes at a position) are appended to `slow_list` and go through the generic kernels
// (k_parse / k_resolve / k_count_*) restricted to that list; both paths add into the same slots.
#pragma once
#include "mkp_kernels.cuh"

namespace mkp {

#ifndef MKP_FZ_RING
#define MKP_FZ_RING (160 * 1024)
#endif
#ifndef MKP_FZ_MAXBLK
#define MKP_FZ_MAXBLK (32 * 1024)
#endif
#ifndef MKP_FZ_SLOTS
#define MKP_FZ_SLOTS 64
#endif
#ifndef MKP_FZ_WARPS
#define MKP_FZ_WARPS 16
#endif
#ifndef MKP_FZ_PCAP
#define MKP_FZ_PCAP 384
#endif
constexpr int FZ_RING = MKP_FZ_RING;       // bytes of read blocks resident per CTA
constexpr int FZ_MAXBLK = MKP_FZ_MAXBLK;   // a longer block is not staged: the read goes to the generic kernels
constexpr int FZ_SLOTS = MKP_FZ_SLOTS;     // reads in flight per CTA (staged or being staged); > FZ_WARPS
constexpr int FZ_WARPS = MKP_FZ_WARPS;     // consumer warps per CTA (+ 1 producer warp)
constexpr int FZ_PCAP = MKP_FZ_PCAP;       // forward positions per warp kept in shared memory
constexpr int FZ_THREADS = (FZ_WARPS + 1) * 32;
static_assert(FZ_SLOTS > FZ_WARPS + 1 && FZ_MAXBLK * 4 <= FZ_RING, "ring geometry");

struct FusedDev {
    const mkp_read_hdr* hdrs;
    const uint8_t* heap;
    uint32_t n_reads, cs, ce;
    uint32_t* read_counter;                                 // reads are handed to the CTAs in runs of 32
    const uint4* rec;                                       // per bitmap word: focus bits and slots per strand, built at upload
    uint32_t* slots; uint32_t stride, n_states;             // n_states = state capacity of the slot layout
    uint32_t n_words;
    uint32_t* obs_word;
    unsigned long long* states; uint32_t* n_states_seen; uint32_t* err;
    uint32_t* slow_list; uint32_t* slow_count;
    unsigned long long* total_calls;
    uint32_t* p_scratch; uint32_t p_stride;                 // per-warp global scratch for reads with more than FZ_PCAP entries
};

struct FzSlot { mkp_read_hdr hdr; uint32_t ring_off, ri, kind, bytes; };       // kind: 0 read, 2 end of work
struct __align__(16) FzWarp {
    ListTab tab;
    union {
        struct { __align__(16) uint8_t txt[160]; uint8_t tok[132]; uint32_t cb[32], bm[32], tp[MAX_LISTS], val[96]; } p;
        struct { uint32_t op[32], q[32], r[33], mask[32]; } w;
    } u;
    uint32_t P[FZ_PCAP];
};
struct FzShared {
    __align__(128) uint8_t ring[FZ_RING];
    FzWarp warp[FZ_WARPS];
    FzSlot slot[FZ_SLOTS];
    __align__(8) unsigned long long full[FZ_SLOTS], empty[FZ_SLOTS];
    uint32_t ticket;
};

// ---- mbarrier / bulk copy (PTX ISA 8.x, sm_90+) --------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count)); }
__device__ __forceinline__ void mbar_arrive(unsigned long long* b) { asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* b, uint32_t tx) { asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(smem_u32(b)), "r"(tx) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long* b, uint32_t parity) {
    const uint32_t a = smem_u32(b);
    uint32_t done = 0;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(a), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ int state_id_fz(const FusedDev& F, StateCache& sc, int pb, uint32_t code) {
    const unsigned long long key = ((unsigned long long)pb << 32) | code;
    if (sc.k0 == key) return sc.i0;
    if (sc.k1 == key) return sc.i1;
    const int id = state_id_global(F.states, F.n_states_seen, F.err, key);
    sc.k1 = sc.k0; sc.i1 = sc.i0; sc.k0 = key; sc.i0 = id;
    return id;
}

// one read, one warp
// MM list discovery (src/mod_bam.rs:900-1000), shape classification and tokens -> occurrence indices (src/mod_bam.rs:667-767) of one
// read by one warp. P receives the 0-based occurrence index of every token (per list at T.ent_off[l]); `slow` = the read goes to
// the generic kernels; `err` = the read has no usable mod info (it still counts as bases).
__device__ __forceinline__ void fz_lists_and_tokens(uint32_t* err_flags, FzWarp& W, const mkp_read_hdr& h, const uint8_t* mm, uint32_t* P,
                                                    bool& err, uint32_t& nl, int (&gp)[4], int (&ga)[4], bool& slow, uint32_t& need, uint32_t& ent, uint32_t& alias_mask) {
    const uint32_t lane = lane_id();
    ListTab& T = W.tab;
    const uint32_t L = h.l_seq;
    const bool rev = (h.flags & 0x10u) != 0;
    struct { uint32_t* err; } F{err_flags};
    err = (h.flags & MKP_RF_TAGS_INVALID) != 0;
    // ---- list discovery (src/mod_bam.rs:900-1000): warp scan for ';' and the first ',' of each part, lane 0 parses the headers
    {
        const uint32_t M = h.len_mm;
        uint32_t n = 0, seg = 0, hdr_end = 0xffffffffu;
        bool e0 = false;
        auto close_part = [&](uint32_t j) {
            if (j > seg) {
                if (n >= MAX_LISTS) { if (lane == 0) { atomicOr(F.err, MKP_DERR_TOO_MANY_LISTS); e0 = true; } }
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
                        else if (nc >= MAX_LIST_CODES) { atomicOr(F.err, MKP_DERR_TOO_MANY_CODES); e = true; }
                        else T.code[n][nc++] = c;
                    }
                    if (nc == 0) e = true;
                    T.base[n] = fb; T.strand[n] = st == '-'; T.mode[n] = (uint8_t)mode; T.ncodes[n] = (uint8_t)nc;
                    if (hl < j) { T.d_start[n] = hl + 1; T.d_end[n] = j; T.n_delta[n] = 0xffffffffu; }
                    else { T.d_start[n] = j; T.d_end[n] = j; T.n_delta[n] = 0u; }
                    if (e) e0 = true;
                }
                if (n < MAX_LISTS) n++;
            }
            seg = j + 1;
            hdr_end = 0xffffffffu;
        };
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
    nl = err ? 0 : T.n;
    // ---- shape of the read: per base one list (<= 2 codes) or one list + its byte-identical copy (one code each), '+' strand,
    //      '?' mode. Everything else goes to the generic kernels.
    for (int b = 0; b < 4; b++) { gp[b] = -1; ga[b] = -1; }
    slow = false;
    need = 0;
    for (uint32_t l = 0; l < nl; l++) {
        const uint8_t fb = T.base[l];
        if (fb == 'N' || T.strand[l] || T.mode[l] != 0) { slow = true; break; }
        const int b = fb == 'A' ? 0 : fb == 'C' ? 1 : fb == 'G' ? 2 : 3;
        if (gp[b] < 0) gp[b] = (int)l;
        else if (ga[b] < 0 && (int)l == gp[b] + 1) ga[b] = (int)l;
        else { slow = true; break; }
        need |= 1u << (rev ? 3 - b : b);
    }
    for (int b = 0; b < 4 && !slow; b++) {
        if (gp[b] < 0) continue;
        const uint32_t n0 = T.ncodes[gp[b]];
        if (ga[b] >= 0) { if (n0 != 1 || T.ncodes[ga[b]] != 1 || T.code[gp[b]][0] == T.code[ga[b]][0]) slow = true; }
        else if (n0 > 2 || (n0 == 2 && T.code[gp[b]][0] == T.code[gp[b]][1])) slow = true;
    }
    if (slow) return;
    // ---- tokens -> occurrence indices (src/mod_bam.rs:667-767); same code as k_parse, positions stay on chip
    ent = 0; alias_mask = 0;
    uint32_t mlp = 0;
    for (uint32_t l = 0; l < nl && !err; l++) {
        const uint32_t ds = T.d_start[l], de = T.d_end[l];
        const bool must = T.n_delta[l] == 0xffffffffu;
        unsigned long long carry = 0;
        uint32_t ntok = 0;
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
                continue;
            }
        }
        auto place = [&](unsigned long long val, bool mine, uint32_t keep_mask) {
            const unsigned long long inc = mine ? (val + 1ull) : 0ull;
            const unsigned long long pre = warp_incl_scan64(inc);
            const uint32_t idx = ntok + __popc(keep_mask & ((1u << lane) - 1u));
            bool bad = false;
            if (mine) {
                const unsigned long long k = carry + pre - 1ull;
                if (k >= (unsigned long long)L || ent + idx >= h.len_ml) bad = true;     // (more tokens than ML entries is an error anyway)
                else P[ent + idx] = (uint32_t)k;
            }
            if (__any_sync(FULL, bad)) err = true;
            carry += __shfl_sync(FULL, pre, 31);
            ntok += __popc(keep_mask);
        };
        bool slowtok = false;
        if (must) {
            uint32_t* qv = W.u.p.val;
            uint32_t qn = 0, v_carry = 0, nd_carry = 0;
            const int ids = (int)ds, ide = (int)de;
            for (int c0 = ids - (int)((uintptr_t)(mm + ds) & 3u); c0 < ide && !slowtok && !err; c0 += 128) {
                const int g0 = c0 + 4 * (int)lane;
                const uint32_t w = g0 < ide ? *(const uint32_t*)(mm + g0) : 0u;
                uint32_t nb = __shfl_down_sync(FULL, w, 1) & 0xffu;
                if (lane == 31) nb = g0 + 4 < ide ? mm[g0 + 4] : 0u;
                const uint32_t wn = (w >> 8) | (nb << 24);
                bool odd = false;
                uint32_t A = 1, B = 0, R = 1u << 16;
                uint32_t dm = 0, cm = 0, em = 0;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int g = g0 + j;
                    const bool in = g >= ids && g < ide, nin = g + 1 < ide;
                    const uint32_t ch = (w >> (8 * j)) & 0xffu, nx = (wn >> (8 * j)) & 0xffu;
                    const bool dig = in && (ch - '0') < 10u, com = in && ch == ',';
                    if (in && !dig && !com) odd = true;
                    if (com && (!nin || nx == ',' || g == ids)) odd = true;
                    if (dig) { B = B * 10u + (ch - '0'); A *= 10u; R += 1u; dm |= 1u << j; if (!nin || nx == ',') em |= 1u << j; }
                    if (com) { A = 0; B = 0; R = 0; cm |= 1u << j; }
                }
                if (lane == 0) { B = A * v_carry + B; if (R >> 16) R += nd_carry; A = 0; R &= 0xffffu; }
#pragma unroll
                for (int d = 1; d <= 2; d <<= 1) {
                    const uint32_t pA = __shfl_up_sync(FULL, A, d), pB = __shfl_up_sync(FULL, B, d), pR = __shfl_up_sync(FULL, R, d);
                    if (lane >= (uint32_t)d) { B = A * pB + B; A = A * pA; if (R >> 16) R = pR + (R & 0xffffu); }
                }
                uint32_t v = __shfl_up_sync(FULL, B, 1), n = __shfl_up_sync(FULL, R, 1) & 0xffffu;
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
                if (__any_sync(FULL, odd)) { slowtok = true; break; }
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
            if (!slowtok && !err && qn) { const bool mine = lane < qn; place(mine ? qv[lane] : 0, mine, qn >= 32 ? FULL : ((1u << qn) - 1u)); }
            if (!slowtok && !err && ntok == 0) slowtok = true;
        }
        if (slowtok) { carry = 0; ntok = 0; }
        bool stop = false;
        uint8_t* txt = W.u.p.txt;
        uint8_t* tok = W.u.p.tok;
        for (uint32_t c0 = ds - 1; must && slowtok && c0 < de && !stop && !err; c0 += 128) {
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 5; k++) { const uint32_t o = lane + 32 * k, g = c0 + o; txt[o] = g < de ? mm[g] : 0; }
            __syncwarp();
            const uint32_t w4 = ((const uint32_t*)txt)[lane];
            const uint32_t xr = w4 ^ 0x2c2c2c2cu;
            uint32_t zf = ~(((xr & 0x7f7f7f7fu) + 0x7f7f7f7fu) | xr | 0x7f7f7f7fu);
            const uint32_t nvalid = de - c0;
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
                    uint32_t k = tok[g0 + lane];
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
                const uint32_t first_bad = m_badstart ? (uint32_t)__ffs(m_badstart) - 1 : 32;
                const uint32_t first_dirty = m_dirty ? (uint32_t)__ffs(m_dirty) - 1 : 32;
                uint32_t keep_mask = m_start;
                if (first_bad < 32 || first_dirty < 32) {
                    stop = true;
                    const uint32_t cut = first_bad <= first_dirty ? first_bad : first_dirty + 1;
                    keep_mask &= cut >= 32 ? FULL : ((1u << cut) - 1u);
                }
                if (ntok == 0 && g0 == 0 && !(keep_mask & 1u)) err = true;
                place(val, (keep_mask >> lane) & 1u, keep_mask);
            }
        }
        if (must && ntok == 0) err = true;
        __syncwarp();
        if (lane == 0) { T.n_delta[l] = ntok; T.ent_off[l] = ent; T.ml_off[l] = mlp; }
        if ((unsigned long long)mlp + (unsigned long long)ntok * T.ncodes[l] > (unsigned long long)h.len_ml) err = true;
        mlp += ntok * T.ncodes[l];
        ent += ntok;
        __syncwarp();
    }
    // the second list of a base must be the byte-identical copy of the first (its entries then sit at the same positions)
    if (!err) for (int b = 0; b < 4; b++) if (ga[b] >= 0 && !((alias_mask >> ga[b]) & 1u)) slow = true;
    if (slow) return;
}

__device__ __forceinline__ void fused_read(const FusedDev& F, FzWarp& W, StateCache& scache, uint32_t ri, const mkp_read_hdr& h, const uint8_t* blk, uint32_t* Pg) {
    const uint32_t lane = lane_id();
    ListTab& T = W.tab;
    const uint32_t flag = h.flags & 0xffffu;
    const uint32_t L = h.l_seq;
    const bool rev = flag & 0x10;
    if ((flag & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)) || L == 0) return;          // not admitted (pileup/mod.rs:783-791 + htslib mask)
    const uint32_t* cig = (const uint32_t*)blk;
    const uint8_t* seq = blk + 4ull * h.n_cigar;
    const uint8_t* ml = seq + ((L + 1) >> 1);
    const uint8_t* mm = ml + h.len_ml;
    bool err; uint32_t nl, need, ent, alias_mask; int gp[4], ga[4]; bool slow;
    uint32_t* P = h.len_ml <= (uint32_t)FZ_PCAP ? W.P : Pg;
    fz_lists_and_tokens(F.err, W, h, mm, P, err, nl, gp, ga, slow, need, ent, alias_mask);
    if (slow) { if (lane == 0) F.slow_list[atomicAdd(F.slow_count, 1u)] = ri; return; }
    const uint32_t nblk = (L + 31) >> 5;
    // ---- streaming select: occurrence index -> forward position, one pass over the SEQ per needed base
    if (!err && need) {
        const uint32_t* seqw = (const uint32_t*)seq;
        const uint32_t nbytes = (L + 1) >> 1;
        for (int x = 0; x < 4 && !err; x++) {
            if (!(need & (1u << x))) continue;
            const int bfw = rev ? 3 - x : x;
            uint32_t lists = 0;
            for (uint32_t l = 0; l < nl; l++) {
                const uint8_t fb = T.base[l];
                const int b = fb == 'A' ? 0 : fb == 'C' ? 1 : fb == 'G' ? 2 : 3;
                if (b == bfw) lists |= 1u << l;
            }
            lists &= ~alias_mask;
            if (lane < MAX_LISTS) W.u.p.tp[lane] = 0;
            __syncwarp();
            uint32_t run = 0;
            for (uint32_t i0 = 0; i0 < nblk; i0 += 32) {
                const uint32_t bi = i0 + lane;
                const bool valid = bi < nblk;
                const uint32_t blkq = rev ? nblk - 1u - bi : bi;
                uint32_t bm = 0;
                if (valid) {
#pragma unroll
                    for (int w = 0; w < 4; w++) {
                        const uint32_t byte0 = blkq * 16 + w * 4;
                        if (byte0 >= nbytes) continue;
                        uint32_t word = seqw[blkq * 4 + w];
                        const uint32_t vb = nbytes - byte0;
                        if (vb < 4) word &= (1u << (8 * vb)) - 1u;
                        bm |= nib_flags_to_mask(nib_eq_flags(word, 1u << x)) << (8 * w);
                    }
                }
                const uint32_t cnt = __popc(bm);
                const uint32_t incl = warp_incl_scan(cnt);
                W.u.p.cb[lane] = run + incl - cnt;
                W.u.p.bm[lane] = bm;
                const uint32_t hi = run + __shfl_sync(FULL, incl, 31);
                __syncwarp();
                uint32_t ls = lists;
                while (ls) {
                    const uint32_t l = __ffs(ls) - 1;
                    ls &= ls - 1;
                    const uint32_t n = T.n_delta[l];
                    uint32_t* Kp = P + T.ent_off[l];
                    uint32_t tp = W.u.p.tp[l];
                    while (tp < n) {
                        const uint32_t t = tp + lane;
                        const uint32_t kv = t < n ? Kp[t] : 0xffffffffu;
                        const bool in = t < n && kv < hi;
                        if (in) {
                            uint32_t lo = 0, hb = 32;
#pragma unroll
                            for (int st = 0; st < 5; st++) { const uint32_t mid = (lo + hb) >> 1; if (W.u.p.cb[mid] <= kv) lo = mid; else hb = mid; }
                            uint32_t msk = W.u.p.bm[lo];
                            uint32_t within = kv - W.u.p.cb[lo];
                            if (rev) within = __popc(msk) - 1u - within;
                            uint32_t pos = 0, c;
                            c = __popc(msk & 0xffffu); if (within >= c) { within -= c; pos += 16; msk >>= 16; }
                            c = __popc(msk & 0xffu);   if (within >= c) { within -= c; pos += 8;  msk >>= 8; }
                            c = __popc(msk & 0xfu);    if (within >= c) { within -= c; pos += 4;  msk >>= 4; }
                            c = __popc(msk & 0x3u);    if (within >= c) { within -= c; pos += 2;  msk >>= 2; }
                            c = msk & 1u;              if (within >= c) { pos += 1; }
                            const uint32_t bq = rev ? nblk - 1u - (i0 + lo) : i0 + lo;
                            const uint32_t q = bq * 32 + pos;
                            Kp[t] = rev ? L - 1u - q : q;
                        }
                        const uint32_t c_in = __popc(__ballot_sync(FULL, in));
                        tp += c_in;
                        if (c_in < 32) break;
                    }
                    __syncwarp();
                    if (lane == 0) W.u.p.tp[l] = tp;
                }
                run = hi;
                __syncwarp();
            }
            uint32_t ls = lists;
            while (ls) { const uint32_t l = __ffs(ls) - 1; ls &= ls - 1; if (W.u.p.tp[l] < T.n_delta[l]) err = true; }
            __syncwarp();
        }
    }
    __syncwarp();
    // ---- per base group: codes, observed-code masks, validation of the merged probabilities (src/mod_bam.rs:629-656) -----
    // gc0/gc1: codes in call order after the collapse; gn: codes left (0..2); gmode: 0 one ML byte, 1 two bytes of one list,
    // 2 one byte of the list + one of its copy
    uint32_t gs0[4], gs1[4];
    uint32_t pos_mask = 0, neg_mask = 0;
    bool has_mods = !err && ent > 0;
    if (has_mods) {
        const bool trim_ok = !c_par.edge_on || !(L <= c_par.edge_start || L <= c_par.edge_end);
        bool survived = false;
        for (int b = 0; b < 4; b++) {
            gs0[b] = gs1[b] = 0;
            if (gp[b] < 0) continue;
            const uint32_t lp = (uint32_t)gp[b];
            const uint32_t n = T.n_delta[lp];
            if (!n) continue;
            const uint32_t* Pl = P + T.ent_off[lp];
            uint32_t c0 = T.code[lp][0], c1 = 0, n2c = 1;
            if (T.ncodes[lp] == 2) { c1 = T.code[lp][1]; n2c = 2; }
            else if (ga[b] >= 0) {
                c1 = T.code[ga[b]][0]; n2c = 2;
                // combine_checked: the two lists' probabilities at one position must not sum above 1.01
                const uint8_t* m0 = ml + T.ml_off[lp];
                const uint8_t* m1 = ml + T.ml_off[ga[b]];
                bool bad = false;
                for (uint32_t j = lane; j < n; j += 32) {
                    const float p0 = ml_prob(m0[j]), p1 = ml_prob(m1[j]);
                    if (__fadd_rn(p0, p1) > 1.01f) bad = true;
                }
                if (__any_sync(FULL, bad)) err = true;
            }
            // codes that remain after ReDistribute, in the order the caller sees them
            uint32_t k0 = c0, k1 = c1, kn = n2c;
            if (c_par.numeric_mode == 2) {
                const uint32_t drop = c_par.collapse_code;
                if (n2c == 1) { if (c0 == drop) kn = 0; }
                else if (c0 == drop) { k0 = c1; kn = 1; }
                else if (c1 == drop) { kn = 1; }
            }
            uint32_t mask = 0;
            if (kn >= 1) { gs0[b] = (uint32_t)state_id_fz(F, scache, b, k0); mask |= 1u << gs0[b]; }
            if (kn == 2) { gs1[b] = (uint32_t)state_id_fz(F, scache, b, k1); mask |= 1u << gs1[b]; }
            // does any entry survive the edge filter?  (P is ascending)
            bool any_kept = trim_ok;
            if (any_kept && c_par.edge_on) {
                if (c_par.edge_inv) any_kept = Pl[0] < c_par.edge_start || Pl[n - 1] >= L - c_par.edge_end;
                else { const uint32_t k = lower_bound_u32(Pl, n, c_par.edge_start); any_kept = k < n && Pl[k] < L - c_par.edge_end; }
            }
            if (any_kept) { survived = true; if (!rev) pos_mask |= mask; else neg_mask |= mask; }
        }
        if (err || !survived) { has_mods = false; pos_mask = neg_mask = 0; }
    }
    __syncwarp();
    // ---- the walk: CIGAR in batches of 32 ops; under each batch the calls, then the bases / deletions of what is left -----
    const uint32_t a = rev ? 1u : 0u;
    const uint32_t pm = pos_mask, nm = neg_mask;
    uint32_t cur[4] = {0, 0, 0, 0};          // entries of each group consumed so far, in query order
    uint32_t n_calls = 0;
    auto cover = [&](uint32_t ra, uint32_t rb) {
        if (!(pm | nm)) return;
        if (ra < F.cs) ra = F.cs;
        if (rb > F.ce) rb = F.ce;
        if (ra >= rb) return;
        const uint32_t wl = (ra - F.cs + 31) >> 5, wh = (rb - F.cs) >> 5;
        for (uint32_t w = wl + lane; w < wh; w += 32) {
            const uint4 wr = F.rec[w];
            if (!(wr.x | wr.y)) continue;                   // a word without focus positions produces no rows
            if (pm && (F.obs_word[w] & pm) != pm) atomicOr(&F.obs_word[w], pm);
            if (nm && (F.obs_word[F.n_words + w] & nm) != nm) atomicOr(&F.obs_word[F.n_words + w], nm);
        }
        auto partial = [&](uint32_t pa, uint32_t pb) {
            if (pa >= pb) return;
            const uint32_t w = (pa - F.cs) >> 5, wbase = F.cs + (w << 5);
            const uint4 r = F.rec[w];
            uint32_t bits = (r.x | r.y) & (FULL << (pa - wbase));
            if (pb < wbase + 32) bits &= (1u << (pb - wbase)) - 1u;
            if ((bits >> lane) & 1u) {
                const uint32_t kp = pm ? wslot(r, 0, lane) : 0xffffffffu, kn = nm ? wslot(r, 1, lane) : 0xffffffffu;
                if (kp != 0xffffffffu) { uint32_t* S = F.slots + (size_t)kp * F.stride; if ((S[SL_OBS] & pm) != pm) atomicOr(&S[SL_OBS], pm); }
                if (kn != 0xffffffffu) { uint32_t* S = F.slots + (size_t)kn * F.stride; if ((S[SL_OBS] & nm) != nm) atomicOr(&S[SL_OBS], nm); }
            }
        };
        if (wl > wh) partial(ra, rb);
        else { partial(ra, F.cs + (wl << 5)); partial(F.cs + (wh << 5), rb); }
    };
    // entries of group b with query position below qlim (P ascending in forward-read order)
    auto count_below = [&](int b, uint32_t qlim) -> uint32_t {
        const uint32_t n = T.n_delta[gp[b]];
        const uint32_t* Pl = P + T.ent_off[gp[b]];
        if (!rev) return lower_bound_u32(Pl, n, qlim);                  // f = q < qlim
        if (qlim >= L) return n;
        return n - lower_bound_u32(Pl, n, L - qlim);                    // q = L-1-f < qlim  <=>  f >= L - qlim
    };
    uint32_t qc = 0, rc = (uint32_t)h.ref_start;
    uint32_t run_start = rc;
    for (uint32_t b0 = 0; b0 < h.n_cigar; b0 += 32) {
        const uint32_t i = b0 + lane;
        const uint32_t c = i < h.n_cigar ? cig[i] : 0;
        const uint32_t op = c & 15, len = c >> 4;
        const uint32_t ql = (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) ? len : 0;
        const uint32_t rl = (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ? len : 0;
        const uint32_t qi = warp_incl_scan(ql), rr = warp_incl_scan(rl);
        const uint32_t q0 = qc + qi - ql, r0 = rc + rr - rl;
        const uint32_t Q1 = qc + __shfl_sync(FULL, qi, 31);
        qc = Q1;
        rc += __shfl_sync(FULL, rr, 31);
        uint32_t skips = __ballot_sync(FULL, op == 3 && len > 0 && i < h.n_cigar);
        while (skips) {
            const int sl = __ffs(skips) - 1;
            skips &= skips - 1;
            const uint32_t sr = __shfl_sync(FULL, r0, sl), slen = __shfl_sync(FULL, len, sl);
            cover(run_start, sr);
            run_start = sr + slen;
        }
        const uint32_t R0 = __shfl_sync(FULL, r0, 0), R1 = rc;
        __syncwarp();
        W.u.w.op[lane] = op | (len << 4); W.u.w.q[lane] = q0; W.u.w.r[lane] = r0;
        if (lane == 0) W.u.w.r[32] = R1;
        __syncwarp();
        const uint32_t blo = R0 > F.cs ? R0 : F.cs, bhi = R1 < F.ce ? R1 : F.ce;
        if (blo < bhi) {
            const uint32_t w_first = (blo - F.cs) >> 5, w_last = (bhi - 1 - F.cs) >> 5;
            for (uint32_t wt = w_first; wt <= w_last; wt += 32) {
                const uint32_t w = wt + lane;
                uint32_t called = 0;
                if (has_mods) {
                    // the read's calls under these 32 words: entries are taken in query order while their reference position
                    // (for an unaligned base: the position of the next aligned base) lies before the tile end
                    const unsigned long long t_end = (unsigned long long)F.cs + ((unsigned long long)(wt + 32) << 5);
                    const uint32_t lim = (unsigned long long)bhi < t_end ? bhi : (uint32_t)t_end;
                    W.u.w.mask[lane] = 0;
                    __syncwarp();
                    for (int b = 0; b < 4; b++) {
                        if (gp[b] < 0) continue;
                        const uint32_t lp = (uint32_t)gp[b];
                        const uint32_t n = T.n_delta[lp];
                        if (cur[b] >= n) continue;
                        const uint32_t* Pl = P + T.ent_off[lp];
                        const uint8_t* m0 = ml + T.ml_off[lp];
                        const uint8_t* m1 = ga[b] >= 0 ? ml + T.ml_off[ga[b]] : m0;
                        const uint32_t two = T.ncodes[lp] == 2 ? 2u : 1u;
                        for (;;) {
                            const uint32_t k = cur[b] + lane;
                            bool take = false, aligned = false;
                            uint32_t rpos = 0, f = 0, j = 0;
                            if (k < n) {
                                j = rev ? n - 1u - k : k;
                                f = Pl[j];
                                const uint32_t q = rev ? L - 1u - f : f;
                                if (q < Q1) {
                                    // op holding q: largest t with start <= q (ops without query length share the start of the next op)
                                    uint32_t t = 0;
#pragma unroll
                                    for (int stp = 16; stp >= 1; stp >>= 1) if (t + stp < 32 && W.u.w.q[t + stp] <= q && b0 + t + stp < h.n_cigar) t += stp;
                                    const uint32_t jc = W.u.w.op[t], jop = jc & 15;
                                    aligned = jop == 0 || jop == 7 || jop == 8;
                                    rpos = W.u.w.r[t] + (aligned ? q - W.u.w.q[t] : 0u);
                                    take = rpos < lim;
                                }
                            }
                            const uint32_t tm = __ballot_sync(FULL, take);
                            if (take && aligned && rpos >= F.cs && edge_keep(f, L)) {
                                const uint32_t rel = rpos - F.cs;
                                atomicOr(&W.u.w.mask[(rel >> 5) - wt], 1u << (rel & 31));
                                n_calls++;
                                const uint4 wr = F.rec[rel >> 5];
                                if (((wr.x | wr.y) >> (rel & 31)) & 1u) {
                                    // probabilities -> collapse -> call (src/mod_bam.rs:558-600, src/threshold_mod_caller.rs:28-63)
                                    float p0 = ml_prob(m0[(size_t)j * two]), p1 = 0.f;
                                    uint32_t c0 = T.code[lp][0], c1 = 0;
                                    int n2c = 1;
                                    if (two == 2) { p1 = ml_prob(m0[(size_t)j * 2 + 1]); c1 = T.code[lp][1]; n2c = 2; }
                                    else if (ga[b] >= 0) { p1 = ml_prob(m1[j]); c1 = T.code[ga[b]][0]; n2c = 2; }
                                    uint32_t s0 = gs0[b], s1 = gs1[b];
                                    if (c_par.numeric_mode == 2) redistribute2(c_par.collapse_code, c0, p0, c1, p1, n2c);
                                    if (n2c == 2) {        // FxHashMap iteration order of the two codes
                                        const uint32_t h0 = bucket4(c0), h1 = bucket4(c1);
                                        if (h0 != h1 ? (h1 < h0) : (h0 == 3)) { const uint32_t tc = c0; c0 = c1; c1 = tc; const float tp = p0; p0 = p1; p1 = tp; const uint32_t ts = s0; s0 = s1; s1 = ts; }
                                    }
                                    const float sum = n2c == 0 ? 0.f : n2c == 1 ? __fadd_rn(0.f, p0) : __fadd_rn(__fadd_rn(0.f, p0), p1);
                                    const float cp = __fsub_rn(1.0f, sum);
                                    const int tb = b;
                                    const float base_thr = c_par.base_set[tb] ? c_par.base_thr[tb] : c_par.default_thr;
                                    bool have = false;
                                    float best = 0.f;
                                    uint32_t state = 0;
                                    for (int k2 = 0; k2 < n2c; k2++) {
                                        const uint32_t cc = k2 == 0 ? c0 : c1;
                                        const float pp = k2 == 0 ? p0 : p1;
                                        float thr = base_thr;
                                        if (c_par.n_mod_thr) {
                                            const uint32_t any_code = (uint32_t)("ACGT"[tb]);
                                            bool fnd = false;
                                            for (uint32_t t = 0; t < c_par.n_mod_thr && !fnd; t++) if (c_par.mod_code[t] == cc) { thr = c_par.mod_thr[t]; fnd = true; }
                                            for (uint32_t t = 0; t < c_par.n_mod_thr && !fnd; t++) if (c_par.mod_code[t] == any_code) { thr = c_par.mod_thr[t]; fnd = true; }
                                        }
                                        if (pp >= thr && (!have || pp >= best)) { have = true; best = pp; state = 2u + (k2 == 0 ? s0 : s1); }
                                    }
                                    if (cp >= base_thr && (!have || cp >= best)) { have = true; state = 1; }
                                    if (!have) state = 0;
                                    if (state < 2 || state - 2 < F.n_states)
                                        add_feature(F.slots, F.stride, wr, rel & 31, a, (uint32_t)b, state, 1u);
                                }
                            }
                            const uint32_t nt = __popc(tm);
                            cur[b] += nt;
                            if (nt < 32) break;
                        }
                    }
                    __syncwarp();
                    called = W.u.w.mask[lane];
                    __syncwarp();
                }
                if (w > w_last) continue;
                const uint4 wr = F.rec[w];
                const uint32_t ok = a == 0 ? wr.x : wr.y, pre = a == 0 ? wr.z : wr.w;     // positions with a slot on the read's strand
                if (!ok) continue;
                const uint32_t wbase = F.cs + (w << 5);
                uint32_t bits = ok & ~called;
                if (blo > wbase) bits &= FULL << (blo - wbase);
                if (bhi < wbase + 32) bits &= (1u << (bhi - wbase)) - 1u;
                if (!bits) continue;
                uint32_t j = 0;
                {
                    const uint32_t r = wbase + (uint32_t)__ffs(bits) - 1u;
#pragma unroll
                    for (int stp = 16; stp >= 1; stp >>= 1) if (W.u.w.r[j + stp] <= r) j += stp;
                }
                while (bits) {
                    const uint32_t bit = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const uint32_t r = wbase + bit;
                    while (W.u.w.r[j + 1] <= r) j++;
                    const uint32_t jc = W.u.w.op[j], jop = jc & 15;
                    if (!(jop == 0 || jop == 7 || jop == 8 || jop == 2)) continue;
                    uint32_t* S = F.slots + (size_t)(pre + __popc(ok & ((1u << bit) - 1u))) * F.stride;
                    if (jop == 2) { atomicAdd(&S[SL_DEL], 1u); continue; }
                    const uint32_t q = W.u.w.q[j] + (r - W.u.w.r[j]);
                    const int nb = nib_to_base(seq_nibble(seq, q));
                    if (nb > 3) continue;
                    atomicAdd(&S[SL_BASE + (a ? 3 - nb : nb)], 1u);
                }
            }
        }
        // entries of this batch that were not taken (outside the chunk, or unaligned at the batch end) are dropped
        if (has_mods) for (int b = 0; b < 4; b++) if (gp[b] >= 0) { const uint32_t cb = count_below(b, Q1); if (cb > cur[b]) cur[b] = cb; }
        __syncwarp();
    }
    cover(run_start, rc);
    n_calls = __reduce_add_sync(FULL, n_calls);
    if (lane == 0 && n_calls) atomicAdd(F.total_calls, (unsigned long long)n_calls);
}

__global__ void __launch_bounds__(FZ_THREADS, 1) k_pileup_fused(const FusedDev F) {
    extern __shared__ __align__(128) uint8_t fz_smem_raw[];
    FzShared& S = *reinterpret_cast<FzShared*>(fz_smem_raw);
    const uint32_t lane = lane_id();
    const uint32_t wib = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < FZ_SLOTS; s++) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], 1); }
        S.ticket = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (wib == FZ_WARPS) {
        // ---- producer warp: takes runs of 32 reads, loads their headers (one coalesced load), and lane 0 places every read in
        // the ring: slot k % FZ_SLOTS for the k-th read of this CTA, bytes from the ring's tail. Ring bytes are reclaimed in order
        // (`oldest` = first read not yet known to be released; its consumer arrives on empty[slot] when done).
        uint32_t seq = 0, oldest = 0;          // reads placed / reads known released
        uint32_t tail = 0;                     // next free ring byte
        auto release_oldest = [&]() {          // lane 0
            mbar_wait(&S.empty[oldest % FZ_SLOTS], (oldest / FZ_SLOTS) & 1u);
            oldest++;
        };
        auto place = [&](const mkp_read_hdr& h, uint32_t ri, uint32_t kind) {     // lane 0
            while (seq - oldest >= (uint32_t)FZ_SLOTS) release_oldest();              // the slot's previous read is done
            const unsigned long long size = 4ull * h.n_cigar + ((h.l_seq + 1) >> 1) + h.len_ml + h.len_mm;
            const uint32_t sz = kind == 0 ? (uint32_t)((size + 15ull) & ~15ull) : 0u;
            uint32_t at = tail;
            if (sz) {
                // bytes in use: [head, tail) or, after a wrap, [head, end) + [0, tail); a placement never makes tail meet head
                for (;;) {
                    if (oldest == seq) { at = 0; break; }                            // nothing resident
                    const uint32_t head = S.slot[oldest % FZ_SLOTS].ring_off;        // first byte still in use
                    if (tail > head) {
                        if (tail + sz <= (uint32_t)FZ_RING) { at = tail; break; }
                        if (sz < head) { at = 0; break; }                            // wrap: the bytes up to the ring's end stay unused
                    } else if (tail + sz < head) { at = tail; break; }
                    release_oldest();
                }
            }
            FzSlot& sl = S.slot[seq % FZ_SLOTS];
            sl.hdr = h; sl.ring_off = at; sl.ri = ri; sl.kind = kind; sl.bytes = sz;
            unsigned long long* fb = &S.full[seq % FZ_SLOTS];
            if (sz) {
                mbar_arrive_expect_tx(fb, sz);
                bulk_g2s(S.ring + at, F.heap + h.off, sz, fb);
                tail = at + sz;
            } else mbar_arrive(fb);
            seq++;
        };
        for (;;) {
            uint32_t r0 = 0;
            if (lane == 0) r0 = atomicAdd(F.read_counter, 32u);
            r0 = __shfl_sync(FULL, r0, 0);
            if (r0 >= F.n_reads) break;
            mkp_read_hdr h;
            memset(&h, 0, sizeof h);
            const uint32_t mine = r0 + lane;
            if (mine < F.n_reads) h = F.hdrs[mine];
            const uint32_t cnt = F.n_reads - r0 < 32u ? F.n_reads - r0 : 32u;
            for (uint32_t k = 0; k < cnt; k++) {
                mkp_read_hdr hk;
                hk.ref_start = __shfl_sync(FULL, h.ref_start, k); hk.l_seq = __shfl_sync(FULL, h.l_seq, k); hk.n_cigar = __shfl_sync(FULL, h.n_cigar, k);
                hk.flags = __shfl_sync(FULL, h.flags, k); hk.off = __shfl_sync(FULL, h.off, k); hk.len_ml = __shfl_sync(FULL, h.len_ml, k); hk.len_mm = __shfl_sync(FULL, h.len_mm, k);
                if (lane == 0) {
                    const unsigned long long size = 4ull * hk.n_cigar + ((hk.l_seq + 1) >> 1) + hk.len_ml + hk.len_mm;
                    if (size > (unsigned long long)FZ_MAXBLK) F.slow_list[atomicAdd(F.slow_count, 1u)] = r0 + k;     // too long for the ring
                    else if (size) place(hk, r0 + k, 0u);                            // (a read without bytes has no sequence: not admitted)
                }
            }
        }
        if (lane == 0) {
            mkp_read_hdr z;
            memset(&z, 0, sizeof z);
            for (int w = 0; w < FZ_WARPS; w++) place(z, 0xffffffffu, 2u);           // one end marker per consumer warp
        }
        return;
    }
    // ---- consumers: the k-th ticket of the CTA is the k-th read the producer placed
    FzWarp& W = S.warp[wib];
    StateCache scache;
    scache.init();
    uint32_t* Pg = F.p_scratch + (size_t)(blockIdx.x * FZ_WARPS + wib) * F.p_stride;
    for (;;) {
        uint32_t k = 0;
        if (lane == 0) k = atomicAdd(&S.ticket, 1u);
        k = __shfl_sync(FULL, k, 0);
        const uint32_t sidx = k % FZ_SLOTS;
        mbar_wait(&S.full[sidx], (k / FZ_SLOTS) & 1u);
        const FzSlot& sl = S.slot[sidx];
        const uint32_t kind = sl.kind;
        if (kind == 0) {
            const mkp_read_hdr h = sl.hdr;
            fused_read(F, W, scache, sl.ri, h, S.ring + sl.ring_off, Pg);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.empty[sidx]);
        if (kind == 2) break;
    }
}

}  // namespace mkp
