// k_pileup_tile: the single-traversal pass as CTA-cooperative, lane-parallel phases over shared-memory-resident tiles (sm_90a).
//
// Why (DESIGN.md 4.2): the pass is bound by instruction issue, and warp-per-read code spends most of its issue slots with few
// lanes active (a 1024-position tile holds ~10 calls, a read has ~280 CIGAR ops and ~140 calls: every loop of a warp-per-read
// kernel is short). Here a tile of consecutive reads (their blocks `CIGAR | SEQ | ML | MM` are contiguous in the heap) is brought
// into shared memory by TMA bulk copies (`cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes`, double buffered:
// tile k + 1 lands while tile k is processed) and the whole CTA (16 warps) works on it phase by phase, every phase a flat
// parallel loop over the items of ALL reads of the tile:
//   P1  warp per read     MM list discovery + tokens -> occurrence indices (fz_lists_and_tokens), CIGAR prefix (query / reference
//                         start of every op) into the tile's arena
//   P2  warp per 1024 bases of (read, base)  occurrence masks of the 4-bit SEQ + counts; then THREAD PER TOKEN: occurrence index
//                         -> forward position (search over the chunk counts, popcount walk inside the chunk)
//   P3  warp per read     merged-probability validation, codes after collapse, observed-code masks, edge-filter survival
//   P4  THREAD PER CALL   q -> reference position (search in the CIGAR prefix), collapse, threshold, counter of the focus slot,
//                         called bit in the read's bitmap
//   P5  THREAD PER FOCUS WORD  bases / deletions under the focus positions the read did not call, observed-code coverage
// Reads outside the common shape (see fz_lists_and_tokens), reads with reference skips, blocks that do not end inside the staged
// bytes and reads whose working arrays do not fit the arena go to the generic kernels through `slow_list`.
#pragma once
#include "mkp_fused.cuh"

namespace mkp {

#ifndef MKP_TL_WIN
#define MKP_TL_WIN (32 * 1024)
#endif
#ifndef MKP_TL_STAGE
#define MKP_TL_STAGE (48 * 1024)
#endif
#ifndef MKP_TL_READS
#define MKP_TL_READS 12
#endif
#ifndef MKP_TL_ARENA
#define MKP_TL_ARENA (12 * 1024)
#endif
constexpr int TL_WIN = MKP_TL_WIN;         // heap bytes per tile window (a tile = the reads whose block starts in the window)
constexpr int TL_STAGE = MKP_TL_STAGE;     // bytes staged per tile
constexpr int TL_READS = MKP_TL_READS;     // reads of a tile processed here (further ones -> generic kernels)
constexpr int TL_ARENA = MKP_TL_ARENA;     // u32 words of working arrays per tile
constexpr int TL_WARPS = 16;
constexpr int TL_THREADS = TL_WARPS * 32;
constexpr uint32_t TL_MAXCIG = 2048, TL_MAXENT = 4096;

struct TileInfo { unsigned long long base; uint32_t first; uint32_t pad; };   // entry n_tiles = (heap end, n_reads)

struct TlGroup {
    uint32_t n, ent;            // entries, arena offset of their positions
    uint32_t ml0, ml1, two;     // byte offsets (in the read's block) of the ML bytes of the list / its copy (ml1 = ~0: none); codes per entry of the list
    uint32_t c0, c1, s0, s1, kn;
    uint32_t base;              // 0..3
    uint32_t mask_off, cnt_off, nchunk, tot;   // occurrence masks per 32 bases, occurrences before every 1024-base chunk
};
struct TlRead {
    mkp_read_hdr h;
    uint32_t ri, blk, state;    // state: 0 process, 1 nothing to do, 2 handed to the generic kernels
    uint32_t err, has_mods, ng;
    uint32_t k_off, cq_off, cr_off, called_off, w0, nw;
    uint32_t pm, nm, ref_end, q_total, n_calls;
    TlGroup g[4];
};
struct TlMeta { unsigned long long base; uint32_t first, n, bytes, pad; };
struct TlShared {
    __align__(128) uint8_t stage[2][TL_STAGE];
    __align__(16) mkp_read_hdr hdrs[2][TL_READS];
    uint32_t arena[TL_ARENA];
    TlRead rd[TL_READS];
    FzWarp warp[TL_READS];
    TlMeta meta[2];
    __align__(8) unsigned long long full[2];
    uint32_t arena_top, called_base, called_words;
};

// tile table: tiles[t] = first read whose block starts at or after t * TL_WIN, and that block's offset
__global__ void k_tiles(const mkp_read_hdr* __restrict__ hdrs, uint32_t n_reads, unsigned long long heap_end, TileInfo* __restrict__ tiles, uint32_t n_tiles) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > n_tiles) return;
    TileInfo ti;
    ti.pad = 0;
    if (t == n_tiles) { ti.first = n_reads; ti.base = (heap_end + 15ull) & ~15ull; }
    else {
        const unsigned long long want = (unsigned long long)t * TL_WIN;
        uint32_t lo = 0, hi = n_reads;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (hdrs[mid].off < want) lo = mid + 1; else hi = mid; }
        ti.first = lo;
        ti.base = lo < n_reads ? hdrs[lo].off : ((heap_end + 15ull) & ~15ull);
    }
    tiles[t] = ti;
}

struct TileDev {
    FusedDev F;
    const TileInfo* tiles;
    uint32_t n_tiles;
    uint32_t* tile_counter;
};

__device__ __forceinline__ uint32_t select_bit(uint32_t msk, uint32_t within) {      // position of the within-th set bit
    uint32_t pos = 0, c;
    c = __popc(msk & 0xffffu); if (within >= c) { within -= c; pos += 16; msk >>= 16; }
    c = __popc(msk & 0xffu);   if (within >= c) { within -= c; pos += 8;  msk >>= 8; }
    c = __popc(msk & 0xfu);    if (within >= c) { within -= c; pos += 4;  msk >>= 4; }
    c = __popc(msk & 0x3u);    if (within >= c) { within -= c; pos += 2;  msk >>= 2; }
    c = msk & 1u;              if (within >= c) { pos += 1; }
    return pos;
}

__global__ void __launch_bounds__(TL_THREADS, 1) k_pileup_tile(const TileDev Tl) {
    extern __shared__ __align__(128) uint8_t tl_smem_raw[];
    TlShared& S = *reinterpret_cast<TlShared*>(tl_smem_raw);
    const FusedDev& F = Tl.F;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    StateCache scache;
    scache.init();
    if (tid == 0) {
        mbar_init(&S.full[0], 1); mbar_init(&S.full[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // thread 0: next tile that holds reads -> stage s
    auto prefetch = [&](uint32_t s) {
        uint32_t t, n = 0;
        TileInfo ta, tb;
        for (;;) {
            t = atomicAdd(Tl.tile_counter, 1u);
            if (t >= Tl.n_tiles) break;
            ta = Tl.tiles[t]; tb = Tl.tiles[t + 1];
            n = tb.first - ta.first;
            if (n) break;
        }
        TlMeta& M = S.meta[s];
        if (t >= Tl.n_tiles) { M.n = 0xffffffffu; mbar_arrive(&S.full[s]); return; }
        const unsigned long long span = tb.base - ta.base;
        const uint32_t bytes = span > (unsigned long long)TL_STAGE ? (uint32_t)TL_STAGE : (uint32_t)span;
        const uint32_t nh = n < (uint32_t)TL_READS ? n : (uint32_t)TL_READS;
        M.base = ta.base; M.first = ta.first; M.n = n; M.bytes = bytes;
        mbar_arrive_expect_tx(&S.full[s], bytes + nh * (uint32_t)sizeof(mkp_read_hdr));
        if (bytes) bulk_g2s(S.stage[s], F.heap + ta.base, bytes, &S.full[s]);
        bulk_g2s(S.hdrs[s], F.hdrs + ta.first, nh * (uint32_t)sizeof(mkp_read_hdr), &S.full[s]);
    };
    if (tid == 0) prefetch(0);
    for (uint32_t it = 0;; it++) {
        const uint32_t cur = it & 1u;
        if (tid == 0) prefetch(cur ^ 1u);            // the other stage's tile was finished before the barrier that ended the last round
        mbar_wait(&S.full[cur], (it >> 1) & 1u);
        const TlMeta M = S.meta[cur];
        if (M.n == 0xffffffffu) break;
        const uint32_t nr = M.n < (uint32_t)TL_READS ? M.n : (uint32_t)TL_READS;
        const uint8_t* stage = S.stage[cur];
        // ---- P0: read table, first arena allocation (thread 0), reads that cannot be handled here -> generic kernels
        if (tid == 0) {
            uint32_t top = 0;
            for (uint32_t r = 0; r < M.n; r++) {
                if (r >= nr) { F.slow_list[atomicAdd(F.slow_count, 1u)] = M.first + r; continue; }
                TlRead& R = S.rd[r];
                const mkp_read_hdr h = S.hdrs[cur][r];
                R.h = h; R.ri = M.first + r; R.err = 0; R.has_mods = 0; R.ng = 0; R.n_calls = 0; R.pm = R.nm = 0; R.nw = 0; R.called_off = 0;
                const unsigned long long size = 4ull * h.n_cigar + ((h.l_seq + 1) >> 1) + h.len_ml + h.len_mm;
                const unsigned long long rel = h.off - M.base;
                const uint32_t flag = h.flags & 0xffffu;
                R.blk = (uint32_t)rel;
                if ((flag & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)) || h.l_seq == 0) { R.state = 1; continue; }
                const uint32_t need_w = h.len_ml + 2u * (h.n_cigar + 2u);
                if (rel + size > (unsigned long long)M.bytes || h.n_cigar > TL_MAXCIG || h.len_ml > TL_MAXENT || top + need_w > (uint32_t)TL_ARENA) {
                    R.state = 2; F.slow_list[atomicAdd(F.slow_count, 1u)] = R.ri; continue;
                }
                R.state = 0;
                R.k_off = top; top += h.len_ml;
                R.cq_off = top; top += h.n_cigar + 2u;
                R.cr_off = top; top += h.n_cigar + 2u;
            }
            S.arena_top = top;
        }
        __syncthreads();
        // ---- P1: warp per read: lists, tokens -> occurrence indices; the CIGAR prefix of read r is built by warp 15 - r when that
        //      warp has no read of its own (the two are independent), else by the read's own warp
        auto cigar_prefix = [&](TlRead& R) {
            const mkp_read_hdr h = R.h;
            const uint32_t* cig = (const uint32_t*)(stage + R.blk);
            uint32_t* cq = S.arena + R.cq_off;      // cq[i] = 2 * query start + (op is M/=/X), cr[i] = reference start; sentinels at n_cigar
            uint32_t* cr = S.arena + R.cr_off;
            uint32_t qc = 0, rc = (uint32_t)h.ref_start;
            bool has_skip = false;
            for (uint32_t b0 = 0; b0 < h.n_cigar; b0 += 32) {
                const uint32_t i = b0 + lane;
                const uint32_t c = i < h.n_cigar ? cig[i] : 0;
                const uint32_t op = c & 15, len = c >> 4;
                const uint32_t ql = (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) ? len : 0;
                const uint32_t rl = (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ? len : 0;
                const uint32_t qi = warp_incl_scan(ql), rr = warp_incl_scan(rl);
                if (i < h.n_cigar) { cq[i] = 2u * (qc + qi - ql) + ((op == 0 || op == 7 || op == 8) ? 1u : 0u); cr[i] = rc + rr - rl; }
                if (__any_sync(FULL, op == 3 && len > 0 && i < h.n_cigar)) has_skip = true;
                qc += __shfl_sync(FULL, qi, 31);
                rc += __shfl_sync(FULL, rr, 31);
            }
            if (lane == 0) {
                cq[h.n_cigar] = 2u * qc; cr[h.n_cigar] = rc;
                R.q_total = qc; R.ref_end = rc;
                // reference skips cut the observed-code coverage into runs: generic kernels
                if (has_skip && atomicCAS(&R.state, 0u, 2u) == 0u) F.slow_list[atomicAdd(F.slow_count, 1u)] = R.ri;
            }
        };
        if (wib < nr && S.rd[wib].state != 1 && S.rd[wib].state != 2) {
            TlRead& R = S.rd[wib];
            FzWarp& W = S.warp[wib];
            const mkp_read_hdr h = R.h;
            const uint8_t* blk = stage + R.blk;
            const uint32_t L = h.l_seq;
            const uint8_t* mm = blk + 4ull * h.n_cigar + ((L + 1) >> 1) + h.len_ml;
            bool err, slow; uint32_t nl, need, ent, alias_mask; int gp[4], ga[4];
            fz_lists_and_tokens(F.err, W, h, mm, S.arena + R.k_off, err, nl, gp, ga, slow, need, ent, alias_mask);
            if (lane == 0) {
                if (slow && atomicCAS(&R.state, 0u, 2u) == 0u) F.slow_list[atomicAdd(F.slow_count, 1u)] = R.ri;
                R.err = err ? 1u : 0u;
                uint32_t ng = 0;
                if (!slow && !err && ent > 0) {
                    const ListTab& T = W.tab;
                    const uint32_t ml_base = 4u * h.n_cigar + ((L + 1) >> 1);
                    for (int b = 0; b < 4; b++) {
                        if (gp[b] < 0) continue;
                        const uint32_t lp = (uint32_t)gp[b];
                        if (!T.n_delta[lp]) continue;
                        TlGroup& G = R.g[ng++];
                        G.n = T.n_delta[lp]; G.ent = R.k_off + T.ent_off[lp];
                        G.ml0 = ml_base + T.ml_off[lp]; G.ml1 = ga[b] >= 0 ? ml_base + T.ml_off[ga[b]] : 0xffffffffu;
                        G.two = T.ncodes[lp] == 2 ? 2u : 1u;
                        G.c0 = T.code[lp][0];
                        G.c1 = G.two == 2 ? T.code[lp][1] : (ga[b] >= 0 ? T.code[ga[b]][0] : 0u);
                        G.base = (uint32_t)b; G.s0 = G.s1 = 0; G.kn = 0; G.tot = 0; G.nchunk = (L + 1023) >> 10;
                    }
                }
                R.ng = ng;
            }
            if (15u - wib < nr) cigar_prefix(R);                 // no free warp for this read's CIGAR
        } else if (wib >= nr && 15u - wib < nr) {
            TlRead& R = S.rd[15u - wib];
            if (R.state != 1 && R.state != 2) cigar_prefix(R);
        }
        __syncthreads();
        // ---- second arena allocation: occurrence masks / chunk counts of every group, called bitmap of every read
        if (tid == 0) {
            uint32_t top = S.arena_top;
            for (uint32_t r = 0; r < nr; r++) {
                TlRead& R = S.rd[r];
                if (R.state != 0) continue;
                const uint32_t L = R.h.l_seq;
                uint32_t want = 0;
                for (uint32_t g = 0; g < R.ng; g++) want += ((L + 31) >> 5) + R.g[g].nchunk + 1u;
                if (top + want > (uint32_t)TL_ARENA) { R.state = 2; F.slow_list[atomicAdd(F.slow_count, 1u)] = R.ri; continue; }
                for (uint32_t g = 0; g < R.ng; g++) { R.g[g].mask_off = top; top += (L + 31) >> 5; R.g[g].cnt_off = top; top += R.g[g].nchunk + 1u; }
            }
            S.called_base = top;
            for (uint32_t r = 0; r < nr; r++) {
                TlRead& R = S.rd[r];
                if (R.state != 0) continue;
                const uint32_t ra = (uint32_t)R.h.ref_start > F.cs ? (uint32_t)R.h.ref_start : F.cs, rb = R.ref_end < F.ce ? R.ref_end : F.ce;
                R.nw = 0; R.w0 = 0;
                if (ra < rb) {
                    const uint32_t w0 = (ra - F.cs) >> 5, w1 = (rb - 1 - F.cs) >> 5;
                    if (top + (w1 - w0 + 1) > (uint32_t)TL_ARENA) { R.state = 2; F.slow_list[atomicAdd(F.slow_count, 1u)] = R.ri; continue; }
                    R.w0 = w0; R.nw = w1 - w0 + 1; R.called_off = top; top += R.nw;
                }
            }
            S.called_words = top - S.called_base;
        }
        __syncthreads();
        // ---- P2a: occurrence masks (32 bases per lane) and counts per 1024-base chunk; called bitmaps cleared
        for (uint32_t i = tid; i < S.called_words; i += TL_THREADS) S.arena[S.called_base + i] = 0;
        for (uint32_t r = 0; r < nr; r++) {
            const TlRead& R = S.rd[r];
            if (R.state != 0) continue;
            const uint32_t L = R.h.l_seq, nbytes = (L + 1) >> 1;
            const bool rev = (R.h.flags & 0x10u) != 0;
            const uint32_t* seqw = (const uint32_t*)(stage + R.blk + 4ull * R.h.n_cigar);
            for (uint32_t g = 0; g < R.ng; g++) {
                const TlGroup& G = R.g[g];
                const uint32_t x = rev ? 3u - G.base : G.base;             // SEQ nibble of the list's base as stored
                for (uint32_t c = wib; c < G.nchunk; c += TL_WARPS) {
                    const uint32_t sb = c * 32 + lane;                      // 32-base block in query order
                    uint32_t bm = 0;
                    if (sb * 32 < L) {
#pragma unroll
                        for (int w = 0; w < 4; w++) {
                            const uint32_t byte0 = sb * 16 + w * 4;
                            if (byte0 >= nbytes) continue;
                            uint32_t word = seqw[sb * 4 + w];
                            const uint32_t vb = nbytes - byte0;
                            if (vb < 4) word &= (1u << (8 * vb)) - 1u;
                            bm |= nib_flags_to_mask(nib_eq_flags(word, 1u << x)) << (8 * w);
                        }
                        S.arena[G.mask_off + sb] = bm;
                    }
                    const uint32_t cnt = __reduce_add_sync(FULL, __popc(bm));
                    if (lane == 0) S.arena[G.cnt_off + c] = cnt;
                }
            }
        }
        __syncthreads();
        // ---- P2b: thread per (read, group): occurrences before every chunk
        if (tid < nr * 4) {
            TlRead& R = S.rd[tid >> 2];
            const uint32_t g = tid & 3;
            if (R.state == 0 && g < R.ng) {
                TlGroup& G = R.g[g];
                uint32_t acc = 0;
                for (uint32_t c = 0; c < G.nchunk; c++) { const uint32_t v = S.arena[G.cnt_off + c]; S.arena[G.cnt_off + c] = acc; acc += v; }
                S.arena[G.cnt_off + G.nchunk] = acc;
                G.tot = acc;
            }
        }
        __syncthreads();
        // ---- P2c: thread per token: occurrence index (forward-read order) -> forward position
        for (uint32_t r = 0; r < nr; r++) {
            TlRead& R = S.rd[r];
            if (R.state != 0) continue;
            const uint32_t L = R.h.l_seq;
            const bool rev = (R.h.flags & 0x10u) != 0;
            for (uint32_t g = 0; g < R.ng; g++) {
                const TlGroup& G = R.g[g];
                for (uint32_t j = tid; j < G.n; j += TL_THREADS) {
                    const uint32_t k = S.arena[G.ent + j];
                    if (k >= G.tot) { R.err = 1; continue; }                // an occurrence past the end of the read (mod_bam.rs:705-727)
                    const uint32_t kq = rev ? G.tot - 1u - k : k;           // occurrence index in query order
                    uint32_t lo = 0, hi = G.nchunk;                         // largest chunk with count-before <= kq
                    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (S.arena[G.cnt_off + mid] <= kq) lo = mid; else hi = mid; }
                    uint32_t rem = kq - S.arena[G.cnt_off + lo];
                    uint32_t sb = lo * 32, q = 0xffffffffu;
                    for (const uint32_t sb_end = min(sb + 32u, (L + 31) >> 5); sb < sb_end; sb++) {
                        const uint32_t m = S.arena[G.mask_off + sb];
                        const uint32_t pc = __popc(m);
                        if (rem < pc) { q = sb * 32 + select_bit(m, rem); break; }
                        rem -= pc;
                    }
                    if (q >= L) { R.err = 1; continue; }
                    S.arena[G.ent + j] = rev ? L - 1u - q : q;
                }
            }
        }
        __syncthreads();
        // ---- P3: warp per read: probabilities of merged lists must not sum above 1.01, codes after the collapse, observed-code
        //      masks, does any entry survive the edge filter (src/mod_bam.rs:629-656, 558-600, src/read_cache.rs:151-194)
        if (wib < nr && S.rd[wib].state == 0) {
            TlRead& R = S.rd[wib];
            const uint32_t L = R.h.l_seq;
            const bool rev = (R.h.flags & 0x10u) != 0;
            const uint8_t* blk = stage + R.blk;
            bool err = R.err != 0;
            uint32_t pm = 0, nm = 0;
            bool survived = false;
            const bool trim_ok = !c_par.edge_on || !(L <= c_par.edge_start || L <= c_par.edge_end);
            for (uint32_t g = 0; g < R.ng && !err; g++) {
                TlGroup& G = R.g[g];
                const uint32_t* Pl = S.arena + G.ent;
                uint32_t n2c = 1;
                if (G.two == 2) n2c = 2;
                else if (G.ml1 != 0xffffffffu) {
                    n2c = 2;
                    const uint8_t* m0 = blk + G.ml0;
                    const uint8_t* m1 = blk + G.ml1;
                    bool bad = false;
                    for (uint32_t j = lane; j < G.n; j += 32) {
                        const float p0 = ml_prob(m0[j]), p1 = ml_prob(m1[j]);
                        if (__fadd_rn(p0, p1) > 1.01f) bad = true;
                    }
                    if (__any_sync(FULL, bad)) { err = true; break; }
                }
                uint32_t k0 = G.c0, k1 = G.c1, kn = n2c;
                if (c_par.numeric_mode == 2) {
                    const uint32_t drop = c_par.collapse_code;
                    if (n2c == 1) { if (G.c0 == drop) kn = 0; }
                    else if (G.c0 == drop) { k0 = G.c1; kn = 1; }
                    else if (G.c1 == drop) { kn = 1; }
                }
                uint32_t mask = 0, s0 = 0, s1 = 0;
                if (kn >= 1) { s0 = (uint32_t)state_id_fz(F, scache, (int)G.base, k0); mask |= 1u << s0; }
                if (kn == 2) { s1 = (uint32_t)state_id_fz(F, scache, (int)G.base, k1); mask |= 1u << s1; }
                bool any_kept = trim_ok;
                if (any_kept && c_par.edge_on) {
                    if (c_par.edge_inv) any_kept = Pl[0] < c_par.edge_start || Pl[G.n - 1] >= L - c_par.edge_end;
                    else { const uint32_t k = lower_bound_u32(Pl, G.n, c_par.edge_start); any_kept = k < G.n && Pl[k] < L - c_par.edge_end; }
                }
                if (any_kept) { survived = true; if (!rev) pm |= mask; else nm |= mask; }
                if (lane == 0) { G.s0 = s0; G.s1 = s1; G.kn = kn; }
            }
            if (lane == 0) {
                const bool has = !err && R.ng > 0 && survived;
                R.err = err ? 1u : 0u;
                R.has_mods = has ? 1u : 0u;
                R.pm = has ? pm : 0u; R.nm = has ? nm : 0u;
            }
        }
        __syncthreads();
        // ---- P4: thread per call: project, call, count
        for (uint32_t r = 0; r < nr; r++) {
            TlRead& R = S.rd[r];
            if (R.state != 0 || !R.has_mods) continue;
            const uint32_t L = R.h.l_seq, nc = R.h.n_cigar;
            const bool rev = (R.h.flags & 0x10u) != 0;
            const uint32_t a = rev ? 1u : 0u;
            const uint8_t* blk = stage + R.blk;
            const uint32_t* cq = S.arena + R.cq_off;
            const uint32_t* cr = S.arena + R.cr_off;
            uint32_t my_calls = 0;
            for (uint32_t g = 0; g < R.ng; g++) {
                const TlGroup& G = R.g[g];
                const uint8_t* m0 = blk + G.ml0;
                const uint8_t* m1 = G.ml1 != 0xffffffffu ? blk + G.ml1 : m0;
                for (uint32_t j = tid; j < G.n; j += TL_THREADS) {
                    const uint32_t f = S.arena[G.ent + j];
                    const uint32_t q = rev ? L - 1u - f : f;
                    if (nc == 0 || q >= R.q_total || !edge_keep(f, L)) continue;
                    uint32_t lo = 0, hi = nc;
                    const uint32_t key = 2u * q + 1u;
                    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (cq[mid] <= key) lo = mid; else hi = mid; }
                    const uint32_t e = cq[lo];
                    if (!((e & 1u) && q < (cq[lo + 1] >> 1))) continue;               // inserted or clipped base: no reference position
                    const uint32_t rpos = cr[lo] + (q - (e >> 1));
                    if (rpos < F.cs || rpos >= F.ce) continue;
                    const uint32_t rel = rpos - F.cs;
                    atomicOr(&S.arena[R.called_off + ((rel >> 5) - R.w0)], 1u << (rel & 31));
                    my_calls++;
                    const uint4 wr = F.rec[rel >> 5];
                    if (!(((wr.x | wr.y) >> (rel & 31)) & 1u)) continue;
                    float p0 = ml_prob(m0[(size_t)j * G.two]), p1 = 0.f;
                    uint32_t c0 = G.c0, c1 = 0;
                    int n2c = 1;
                    if (G.two == 2) { p1 = ml_prob(m0[(size_t)j * 2 + 1]); c1 = G.c1; n2c = 2; }
                    else if (G.ml1 != 0xffffffffu) { p1 = ml_prob(m1[j]); c1 = G.c1; n2c = 2; }
                    uint32_t s0 = G.s0, s1 = G.s1;
                    if (c_par.numeric_mode == 2) redistribute2(c_par.collapse_code, c0, p0, c1, p1, n2c);
                    if (n2c == 2) {        // FxHashMap iteration order of the two codes
                        const uint32_t h0 = bucket4(c0), h1 = bucket4(c1);
                        if (h0 != h1 ? (h1 < h0) : (h0 == 3)) { const uint32_t tc = c0; c0 = c1; c1 = tc; const float tp = p0; p0 = p1; p1 = tp; const uint32_t ts = s0; s0 = s1; s1 = ts; }
                    }
                    const float sum = n2c == 0 ? 0.f : n2c == 1 ? __fadd_rn(0.f, p0) : __fadd_rn(__fadd_rn(0.f, p0), p1);
                    const float cp = __fsub_rn(1.0f, sum);
                    const int tb = (int)G.base;
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
                        add_feature(F.slots, F.stride, wr, rel & 31, a, G.base, state, 1u);
                }
            }
            if (my_calls) atomicAdd(&R.n_calls, my_calls);
        }
        __syncthreads();
        // ---- P5: thread per focus word under the read: bases / deletions of what the read did not call; observed-code coverage
        for (uint32_t r = 0; r < nr; r++) {
            const TlRead& R = S.rd[r];
            if (R.state != 0 || !R.nw) continue;
            const uint32_t nc = R.h.n_cigar;
            const bool rev = (R.h.flags & 0x10u) != 0;
            const uint32_t a = rev ? 1u : 0u;
            const uint8_t* seq = stage + R.blk + 4ull * nc;
            const uint32_t* cq = S.arena + R.cq_off;
            const uint32_t* cr = S.arena + R.cr_off;
            const uint32_t ra = (uint32_t)R.h.ref_start > F.cs ? (uint32_t)R.h.ref_start : F.cs, rb = R.ref_end < F.ce ? R.ref_end : F.ce;
            const uint32_t pm = R.pm, nm = R.nm;
            for (uint32_t wi = tid; wi < R.nw; wi += TL_THREADS) {
                const uint32_t w = R.w0 + wi;
                const uint4 wr = F.rec[w];
                const uint32_t word = wr.x | wr.y;
                if (!word) continue;
                const uint32_t wbase = F.cs + (w << 5);
                uint32_t in = FULL;                                   // positions of the word inside [ra, rb)
                if (ra > wbase) in &= FULL << (ra - wbase);
                if (rb < wbase + 32) in &= (1u << (rb - wbase)) - 1u;
                if (pm | nm) {
                    if (in == FULL) {
                        if (pm && (F.obs_word[w] & pm) != pm) atomicOr(&F.obs_word[w], pm);
                        if (nm && (F.obs_word[F.n_words + w] & nm) != nm) atomicOr(&F.obs_word[F.n_words + w], nm);
                    } else {
                        uint32_t ob = word & in;
                        while (ob) {
                            const uint32_t bit = __ffs(ob) - 1;
                            ob &= ob - 1;
                            const uint32_t kp = pm ? wslot(wr, 0, bit) : 0xffffffffu, kn = nm ? wslot(wr, 1, bit) : 0xffffffffu;
                            if (kp != 0xffffffffu) { uint32_t* Sl = F.slots + (size_t)kp * F.stride; if ((Sl[SL_OBS] & pm) != pm) atomicOr(&Sl[SL_OBS], pm); }
                            if (kn != 0xffffffffu) { uint32_t* Sl = F.slots + (size_t)kn * F.stride; if ((Sl[SL_OBS] & nm) != nm) atomicOr(&Sl[SL_OBS], nm); }
                        }
                    }
                }
                const uint32_t ok = a == 0 ? wr.x : wr.y, pre = a == 0 ? wr.z : wr.w;    // positions with a slot on the read's strand
                uint32_t bits = ok & in & ~S.arena[R.called_off + wi];
                while (bits) {
                    const uint32_t bit = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const uint32_t rp = wbase + bit;
                    uint32_t lo = 0, hi = nc;                         // op holding rp: largest i with reference start <= rp
                    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (cr[mid] <= rp) lo = mid; else hi = mid; }
                    if (cr[lo + 1] <= rp) continue;                   // (cannot happen inside [ref_start, ref_end))
                    uint32_t* Sl = F.slots + (size_t)(pre + __popc(ok & ((1u << bit) - 1u))) * F.stride;
                    const uint32_t e = cq[lo];
                    if (!(e & 1u)) { atomicAdd(&Sl[SL_DEL], 1u); continue; }          // a deletion (reference skips were excluded)
                    const uint32_t q = (e >> 1) + (rp - cr[lo]);
                    const int nb = nib_to_base(seq_nibble(seq, q));
                    if (nb > 3) continue;
                    atomicAdd(&Sl[SL_BASE + (a ? 3 - nb : nb)], 1u);
                }
            }
        }
        if (tid < nr && S.rd[tid].state == 0 && S.rd[tid].n_calls) atomicAdd(F.total_calls, (unsigned long long)S.rd[tid].n_calls);
        __syncthreads();
    }
}

}  // namespace mkp
