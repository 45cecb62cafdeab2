// BGZF / BAM ingest on the device (SURVEY §8f-1): the step directly in front of the pileup path.
//
//   k_inflate      one BGZF member per thread: RFC 1951 inflate (stored / fixed / dynamic blocks) into the
//                  inflated BAM stream. Replaces htslib's bgzf_read_block + inflate on the host
//                  (reference: rust-htslib bam::IndexedReader, src/pileup/mod.rs:732-743).
//   k_walk_*       record discovery: the block_size chain is walked from seed offsets (record starts taken from
//                  the BAI linear index / bin chunks) in parallel; builds the record table (tid, pos, end, flag).
//   k_slice_*      the record packer of csrc/host/bam_reader.hpp (pack_record: CIGAR | SEQ | ML | MM, MM/ML/MN tag
//                  resolution of src/mod_bam.rs:1388-1470) on the device, straight into the resident chunk.
//
// Everything is byte/integer work; results are bit-identical to zlib and to the host packer (tests/test_gpu_ingest.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mkp.h"

namespace mkp {

// ---------------------------------------------------------------------------------------------------------------
// inflate
// ---------------------------------------------------------------------------------------------------------------
// Per-decoder tables in shared memory (u16 units). Literal/length and distance codes are kept in canonical form
// (count per length + symbols sorted by code) and fronted by a direct-lookup table on the next INF_LBITS / INF_DBITS
// stream bits; codes longer than that take the bit-by-bit canonical walk.
constexpr int INF_LBITS = 9, INF_DBITS = 6;
// (the sorted symbol lists, needed only by table builds and by codes longer than the lookup, live in local memory: 1.4 KB
// of shared memory per decoder = 5 warps of decoders per SM instead of 3)
constexpr int INF_LCNT = 0, INF_DCNT = 16, INF_OFFS = 32, INF_LFIRST = 48, INF_LINDEX = 64,
              INF_DFIRST = 80, INF_DINDEX = 96, INF_LTAB = 112,
              INF_DTAB = INF_LTAB + (1 << INF_LBITS), INF_WORDS = INF_DTAB + (1 << INF_DBITS);
constexpr int INF_STRIDE = (((INF_WORDS + 1) / 2) | 1) * 2;   // odd number of 32-bit words per decoder: spreads the banks
__constant__ uint8_t c_clord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
constexpr int INF_THREADS = 32;

enum { INF_OK = 0, INF_ERR_BLOCK_TYPE = 1, INF_ERR_STORED = 2, INF_ERR_CODE = 3, INF_ERR_DIST = 4, INF_ERR_OVERRUN = 5, INF_ERR_LENGTHS = 6, INF_ERR_SIZE = 7, INF_ERR_INPUT = 8 };

struct BitReader {
    const uint8_t* p;        // next input byte
    const uint8_t* end;
    unsigned long long bb;   // bit buffer, LSB first
    int nb;                  // valid bits
    uint32_t nxt;            // the aligned word at p, loaded one refill ahead (its latency hides behind a symbol's work)
    bool have_nxt;
    __device__ __forceinline__ void init(const uint8_t* s, const uint8_t* e) { p = s; end = e; bb = 0; nb = 0; nxt = 0; have_nxt = false; }
    // at least 32 valid bits afterwards (zero bits past the end of the input; the caller checks overrun at the end)
    __device__ __forceinline__ void refill() {
        if (nb > 32) return;
#pragma unroll 1
        while (((uintptr_t)p & 3u) && nb <= 56) { const unsigned long long b = p < end ? *p : 0; p++; bb |= b << nb; nb += 8; have_nxt = false; }
        if (nb > 32) return;
        if (p + 4 <= end) {
            const uint32_t w = have_nxt ? nxt : *(const uint32_t*)p;
            bb |= (unsigned long long)w << nb; p += 4; nb += 32;
            have_nxt = p + 4 <= end;
            if (have_nxt) nxt = *(const uint32_t*)p;
            return;
        }
        have_nxt = false;
#pragma unroll 1
        while (nb <= 56) { const unsigned long long b = p < end ? *p : 0; p++; bb |= b << nb; nb += 8; }
    }
    __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)bb & ((1u << n) - 1u); }
    __device__ __forceinline__ void drop(int n) { bb >>= n; nb -= n; }
    __device__ __forceinline__ uint32_t bits(int n) { refill(); const uint32_t v = peek(n); drop(n); return v; }
};

// lens[0..n) -> cnt[16], sym[] (sorted by length, then symbol), tab[1 << tbits] (sym << 4 | len for codes <= tbits),
// first[len] = first canonical code of that length, index[len] = its position in sym[].
// Returns false for an over-subscribed set of lengths.
__device__ bool inf_build(const uint8_t* lens, int n, uint16_t* cnt, uint16_t* sym, uint16_t* offs, uint16_t* tab, int tbits,
                          uint16_t* first, uint16_t* index) {
    for (int i = 0; i < 16; i++) cnt[i] = 0;
    for (int s = 0; s < n; s++) cnt[lens[s]]++;
    cnt[0] = 0;
    int left = 1;
    for (int len = 1; len <= 15; len++) { left <<= 1; left -= cnt[len]; if (left < 0) return false; }
    offs[1] = 0;
    for (int len = 1; len < 15; len++) offs[len + 1] = offs[len] + cnt[len];
    if (first) {
        uint32_t code = 0;
        for (int len = 1; len <= 15; len++) { first[len] = (uint16_t)code; index[len] = offs[len]; code = (code + cnt[len]) << 1; }
    }
    for (int s = 0; s < n; s++) if (lens[s]) sym[offs[lens[s]]++] = (uint16_t)s;
    const int tsz = 1 << tbits;
    for (int i = 0; i < tsz; i++) tab[i] = 0;
    uint32_t code = 0;
    int idx = 0;
    for (int len = 1; len <= tbits; len++) {
        const int c = cnt[len];
        for (int k = 0; k < c; k++, code++) {
            const uint16_t e = (uint16_t)((sym[idx++] << 4) | len);
            const uint32_t rev = __brev(code) >> (32 - len);
            for (uint32_t i = rev; i < (uint32_t)tsz; i += 1u << len) tab[i] = e;
        }
        code <<= 1;
    }
    return true;
}

// codes longer than the lookup table: the next 15 stream bits, most significant first, against the first code of
// every remaining length
__device__ __forceinline__ int inf_decode_long(BitReader& br, int tbits, const uint16_t* cnt, const uint16_t* sym, const uint16_t* first, const uint16_t* index) {
    const uint32_t v = __brev((uint32_t)br.bb) >> 17;          // 15 bits, first stream bit on top
#pragma unroll 1
    for (int len = tbits + 1; len <= 15; len++) {
        const uint32_t c = (v >> (15 - len)) - first[len];
        if (c < cnt[len]) { br.drop(len); return sym[index[len] + c]; }
    }
    return -1;
}

__device__ __forceinline__ int inf_decode(BitReader& br, const uint16_t* tab, int tbits, const uint16_t* cnt, const uint16_t* sym, const uint16_t* first, const uint16_t* index) {
    br.refill();
    const uint16_t e = tab[br.peek(tbits)];
    if (e) { br.drop(e & 15); return e >> 4; }
    return inf_decode_long(br, tbits, cnt, sym, first, index);
}

// One BGZF member (raw deflate payload) per thread, 32 members in flight per warp. The lanes of a warp run a small
// state machine and meet again after every step (one symbol, one block header, one job fetch): without that the
// lanes drift apart for good after the first divergent branch and the warp degenerates into 32 serial threads.
enum { ST_FETCH = 0, ST_HEADER = 1, ST_SYMBOL = 2, ST_FINISH = 3, ST_DONE = 4, ST_COPY = 5 };
constexpr int INF_COPY_STEP = 64;
#ifndef INF_SYMS_PER_STEP
#define INF_SYMS_PER_STEP 4
#endif

#ifndef MKP_INF_MINB
#define MKP_INF_MINB 28
#endif
__global__ void __launch_bounds__(INF_THREADS, MKP_INF_MINB) k_inflate(const uint8_t* __restrict__ in, const mkp_bgzf_member* __restrict__ jobs, uint32_t n_jobs,
                                                        uint8_t* out, uint32_t* status, uint32_t* work, uint32_t job_base, uint16_t* gtab, uint32_t hdr_batch) {
    extern __shared__ uint16_t inf_smem[];
    // decoder tables: shared memory (1.4 KB per decoder: 5 warps of decoders per SM), or - gtab - a per-decoder global scratch that
    // stays in L2: a lookup costs more, but four times as many decoders are resident and the kernel is latency bound
    uint16_t* const my = gtab ? gtab + ((size_t)blockIdx.x * INF_THREADS + threadIdx.x) * INF_STRIDE : inf_smem + (size_t)threadIdx.x * INF_STRIDE;
    uint16_t lsym[288], dsym[32];
    uint16_t* const lcnt = my + INF_LCNT;
    uint16_t* const dcnt = my + INF_DCNT; uint16_t* const offs = my + INF_OFFS; uint16_t* const ltab = my + INF_LTAB;
    uint16_t* const dtab = my + INF_DTAB;
    uint16_t* const lfirst = my + INF_LFIRST; uint16_t* const lindex = my + INF_LINDEX;
    uint16_t* const dfirst = my + INF_DFIRST; uint16_t* const dindex = my + INF_DINDEX;
    uint8_t lens[320];
    int state = ST_FETCH;
    uint32_t cp_len = 0, cp_dist = 0;          // pending match copy (ST_COPY)
    uint32_t j = 0, o = 0, cap = 0;
    uint8_t* dst = nullptr;
    int err = INF_OK;
    bool last = false;
    BitReader br;
    br.init(in, in);
    for (;;) {
        // Block headers are batched: a header (code lengths + two table builds, ~10^4 instructions) run by one lane stalls the 31
        // others, and with ~4 blocks per member that was half of the warp's instructions. A lane that reaches a header now waits
        // until hdr_batch lanes stand at one (or nobody is decoding any more); they then run the header code together.
        const uint32_t at_header = __ballot_sync(0xffffffffu, state == ST_HEADER);
        const uint32_t decoding = __ballot_sync(0xffffffffu, state == ST_SYMBOL || state == ST_COPY);
        const bool header_go = (uint32_t)__popc(at_header) >= hdr_batch || decoding == 0;
        if (state == ST_SYMBOL) {
            // up to INF_SYMS_PER_STEP literals per step; the first symbol that is not a literal ends the step
#pragma unroll 1
            for (int it = 0; it < INF_SYMS_PER_STEP; it++) {
                const int sym = inf_decode(br, ltab, INF_LBITS, lcnt, lsym, lfirst, lindex);
                if (sym < 256) {
                    if (sym < 0) { err = INF_ERR_CODE; state = ST_FINISH; break; }
                    if (o >= cap) { err = INF_ERR_SIZE; state = ST_FINISH; break; }
                    dst[o++] = (uint8_t)sym;
                    continue;
                }
                if (sym == 256) { state = last ? ST_FINISH : ST_HEADER; break; }
                if (sym > 285) { err = INF_ERR_CODE; state = ST_FINISH; break; }
                // length: 257..264 -> 3..10; 265..284 -> 3 + ((4 + (k & 3)) << e) + extra, k = sym - 261, e = k >> 2; 285 -> 258
                uint32_t len;
                if (sym < 265) len = (uint32_t)sym - 254u;
                else if (sym == 285) len = 258;
                else { const uint32_t k = (uint32_t)sym - 261u, e = k >> 2; len = 3u + ((4u + (k & 3u)) << e) + br.bits((int)e); }
                const int ds = inf_decode(br, dtab, INF_DBITS, dcnt, dsym, dfirst, dindex);
                uint32_t dist = 0;
                if (ds < 0 || ds > 29) err = INF_ERR_CODE;
                else if (ds < 4) dist = (uint32_t)ds + 1u;
                else { const uint32_t e = ((uint32_t)ds >> 1) - 1u; dist = 1u + ((2u + ((uint32_t)ds & 1u)) << e) + br.bits((int)e); }
                if (!err && dist > o) err = INF_ERR_DIST;
                if (!err && o + len > cap) err = INF_ERR_SIZE;
                if (err) state = ST_FINISH;
                else { cp_len = len; cp_dist = dist; state = ST_COPY; }
                break;
            }
        }
        if (state == ST_COPY) {
            // at most INF_COPY_STEP bytes per step, so a lane inside a long match does not hold up the lanes decoding symbols
            uint8_t* d = dst + o;
            const uint32_t n = cp_len < (uint32_t)INF_COPY_STEP ? cp_len : (uint32_t)INF_COPY_STEP;
            if (cp_dist >= (uint32_t)INF_COPY_STEP + 8u) {
                // the step's source lies entirely below its destination: every source word is loaded before the first
                // store (one memory latency per step instead of one per word), destination words are assembled with a
                // funnel shift. Head and tail bytes (destination alignment) go bytewise.
                const uint8_t* s0 = d - cp_dist;
                const uint32_t head = min(n, (uint32_t)(-(intptr_t)d & 3));
                const uint32_t nw = (n - head) >> 2, tail = (n - head) & 3u;
                const uint8_t* sp = s0 + head;
                const uint32_t sh = ((uintptr_t)sp & 3u) * 8u;
                const uint32_t* sw = (const uint32_t*)((uintptr_t)sp & ~(uintptr_t)3);
                uint8_t hb[3] = {0, 0, 0}, tb[3] = {0, 0, 0};
#pragma unroll
                for (int q = 0; q < 3; q++) { if ((uint32_t)q < head) hb[q] = s0[q]; if ((uint32_t)q < tail) tb[q] = sp[4 * nw + q]; }
                uint32_t* dw = (uint32_t*)(d + head);
                // two halves of 8 words: short matches (the common case) touch only the first
#pragma unroll
                for (int half = 0; half < 2; half++) {
                    const uint32_t q0 = 8u * half;
                    if (q0 < nw) {
                        uint32_t w[9];
#pragma unroll
                        for (int q = 0; q <= 8; q++) w[q] = q0 + q <= nw ? sw[q0 + q] : 0u;      // (the last one only feeds the shift)
#pragma unroll
                        for (int q = 0; q < 8; q++) if (q0 + q < nw) dw[q0 + q] = __funnelshift_r(w[q], w[q + 1], sh);
                    }
                }
#pragma unroll
                for (int q = 0; q < 3; q++) if ((uint32_t)q < head) d[q] = hb[q];
#pragma unroll
                for (int q = 0; q < 3; q++) if ((uint32_t)q < tail) d[head + 4 * nw + q] = tb[q];
            } else if (cp_dist >= 8) {
                // whole words, one at a time: destination brought to a 4-byte boundary, source words taken with a funnel shift
                // (with a distance of 8 or more every aligned source word is complete before it is loaded)
                const uint8_t* s0 = d - cp_dist;
                uint32_t k = 0;
                while (k < n && ((uintptr_t)(d + k) & 3u)) { d[k] = s0[k]; k++; }
                if (k + 4 <= n) {
                    const uint8_t* sp = s0 + k;
                    const uint32_t sh = ((uintptr_t)sp & 3u) * 8u;
                    const uint32_t* sw = (const uint32_t*)((uintptr_t)sp & ~(uintptr_t)3);
                    uint32_t lo = *sw++;
                    for (; k + 4 <= n; k += 4) {
                        const uint32_t hi = sh ? *sw : 0u;
                        *(uint32_t*)(d + k) = sh ? __funnelshift_r(lo, hi, sh) : lo;
                        lo = sh ? hi : *sw;
                        sw++;
                    }
                }
                for (; k < n; k++) d[k] = s0[k];
            } else if (cp_dist == 1) {
                const uint32_t b = d[-1], w4 = b * 0x01010101u;
                uint32_t k = 0;
                while (k < n && ((uintptr_t)(d + k) & 3u)) d[k++] = (uint8_t)b;
                for (; k + 4 <= n; k += 4) *(uint32_t*)(d + k) = w4;
                for (; k < n; k++) d[k] = (uint8_t)b;
            } else { const uint8_t* s0 = d - cp_dist; for (uint32_t k = 0; k < n; k++) d[k] = s0[k]; }
            o += n; cp_len -= n;
            if (!cp_len) state = ST_SYMBOL;
        } else if (state == ST_HEADER) {
          if (header_go) {
            last = br.bits(1);
            const uint32_t type = br.bits(2);
            if (type == 0) {
                // stored: skip to the byte boundary, LEN, ~LEN, bytes
                br.drop(br.nb & 7);
                br.refill();
                const uint32_t len = br.bits(16);
                const uint32_t nlen = br.bits(16);
                if ((len ^ 0xffffu) != nlen) err = INF_ERR_STORED;
                else if (o + len > cap) err = INF_ERR_SIZE;
                else {
                    // bytes still in the bit buffer first, then straight from the input
                    uint32_t k = 0;
                    while (k < len && br.nb >= 8) { dst[o + k] = (uint8_t)br.bb; br.drop(8); k++; }
                    if (k < len) {
                        br.bb = 0; br.nb = 0; br.have_nxt = false;
                        if (br.p + (len - k) > br.end) err = INF_ERR_INPUT;
                        else for (; k < len; k++) dst[o + k] = *br.p++;
                    }
                    o += len;
                }
                state = (err || last) ? ST_FINISH : ST_HEADER;
            } else if (type == 3) { err = INF_ERR_BLOCK_TYPE; state = ST_FINISH; }
            else {
                if (type == 1) {
                    for (int s2 = 0; s2 < 144; s2++) lens[s2] = 8;
                    for (int s2 = 144; s2 < 256; s2++) lens[s2] = 9;
                    for (int s2 = 256; s2 < 280; s2++) lens[s2] = 7;
                    for (int s2 = 280; s2 < 288; s2++) lens[s2] = 8;
                    inf_build(lens, 288, lcnt, lsym, offs, ltab, INF_LBITS, lfirst, lindex);
                    for (int s2 = 0; s2 < 30; s2++) lens[s2] = 5;
                    inf_build(lens, 30, dcnt, dsym, offs, dtab, INF_DBITS, dfirst, dindex);
                } else {
                    const int nlen = (int)br.bits(5) + 257, ndist = (int)br.bits(5) + 1, ncode = (int)br.bits(4) + 4;
                    if (nlen > 286 || ndist > 30) err = INF_ERR_LENGTHS;
                    if (!err) {
                        for (int s2 = 0; s2 < 19; s2++) lens[s2] = 0;
                        for (int k = 0; k < ncode; k++) lens[c_clord[k]] = (uint8_t)br.bits(3);
                        // the code-length code (<= 7 bits): complete lookup in the not yet used literal table
                        if (!inf_build(lens, 19, dcnt, dsym, offs, ltab, 7, nullptr, nullptr)) err = INF_ERR_LENGTHS;
                    }
                    int idx = 0;
                    while (!err && idx < nlen + ndist) {
                        br.refill();
                        const uint16_t ce = ltab[br.peek(7)];
                        if (!ce) { err = INF_ERR_CODE; break; }
                        br.drop(ce & 15);
                        const int sym = ce >> 4;
                        if (sym < 16) { lens[idx++] = (uint8_t)sym; continue; }
                        int rep, val = 0;
                        if (sym == 16) { if (idx == 0) { err = INF_ERR_LENGTHS; break; } val = lens[idx - 1]; rep = 3 + (int)br.bits(2); }
                        else if (sym == 17) rep = 3 + (int)br.bits(3);
                        else rep = 11 + (int)br.bits(7);
                        if (idx + rep > nlen + ndist) { err = INF_ERR_LENGTHS; break; }
                        while (rep--) lens[idx++] = (uint8_t)val;
                    }
                    if (!err && lens[256] == 0) err = INF_ERR_LENGTHS;
                    // distance lengths follow the literal/length lengths; build distance first (it reads lens[nlen..])
                    if (!err && !inf_build(lens + nlen, ndist, dcnt, dsym, offs, dtab, INF_DBITS, dfirst, dindex)) err = INF_ERR_LENGTHS;
                    if (!err && !inf_build(lens, nlen, lcnt, lsym, offs, ltab, INF_LBITS, lfirst, lindex)) err = INF_ERR_LENGTHS;
                }
                state = err ? ST_FINISH : ST_SYMBOL;
            }
          }
        } else if (state == ST_FETCH) {
            j = atomicAdd(work, 1u);
            if (j >= n_jobs) state = ST_DONE;
            else {
                const mkp_bgzf_member job = jobs[j];
                dst = out + job.out_off; cap = job.out_len; o = 0; err = INF_OK; last = false;
                br.init(in + job.in_off, in + job.in_off + job.in_len);
                state = ST_HEADER;
            }
        } else if (state == ST_FINISH) {
            if (!err && o != cap) err = INF_ERR_SIZE;
            // every input bit consumed lies inside the member (bits still in the buffer are not consumed)
            if (!err && br.p - (br.nb >> 3) > br.end) err = INF_ERR_OVERRUN;
            if (err) atomicCAS(status, 0u, ((uint32_t)err << 24) | ((job_base + j) & 0xffffffu) | 0x80000000u);
            state = ST_FETCH;
        }
        if (__all_sync(0xffffffffu, state == ST_DONE)) break;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// record discovery
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_u32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t ld_u16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

// Walk the block_size chain of one segment [seed[i], seed[i+1]) of the inflated stream.
// pass 0: count records; pass 1: fill the record table at base[i].
template <int PASS>
__global__ void k_walk(const uint8_t* __restrict__ bam, uint64_t total, const uint64_t* __restrict__ seeds, uint32_t n_seeds,
                       uint32_t* counts, const uint32_t* __restrict__ base, mkp_bam_rec* recs, uint32_t* status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_seeds) return;
    uint64_t p = seeds[i];
    const uint64_t stop = i + 1 < n_seeds ? seeds[i + 1] : total;
    uint32_t n = 0;
    mkp_bam_rec* out = PASS ? recs + base[i] : nullptr;
    while (p + 4 <= stop) {
        const uint32_t bs = ld_u32(bam + p);
        if (bs < 32 || p + 4 + bs > total) { atomicCAS(status, 0u, 0x80000000u | 1u); break; }
        if (PASS) {
            const uint8_t* r = bam + p + 4;
            mkp_bam_rec rec;
            rec.off = p + 4; rec.size = bs;
            rec.tid = (int32_t)ld_u32(r); rec.pos = (int32_t)ld_u32(r + 4);
            const uint32_t l_name = r[8], n_cig = ld_u16(r + 12), flag = ld_u16(r + 14);
            rec.flag = flag; rec.l_seq = ld_u32(r + 16);
            // the fixed fields must fit the record (a corrupt or hostile file must not send the slicer out of bounds)
            { const int32_t ls = (int32_t)rec.l_seq; const unsigned long long lq = ls > 0 ? (unsigned long long)ls : 0ull;
              if (32ull + l_name + 4ull * n_cig + (lq + 1) / 2 + lq > bs) { atomicCAS(status, 0u, 0x80000000u | 1u); break; } }
            // htslib bam_endpos: pos + reference length of the CIGAR (1 when unmapped or without CIGAR)
            unsigned long long span = 0;
            if (!(flag & 4) && n_cig && 32ull + l_name + 4ull * n_cig <= bs) {
                const uint8_t* c = r + 32 + l_name;
                for (uint32_t k = 0; k < n_cig; k++) {
                    const uint32_t v = ld_u32(c + 4 * k), op = v & 15;
                    if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += v >> 4;
                }
            }
            rec.end = (int32_t)(rec.pos + (long long)(span ? span : 1));
            out[n] = rec;
        }
        n++;
        p += 4ull + bs;
    }
    if (p != stop) atomicCAS(status, 0u, 0x80000000u | 2u);     // the chain did not land on the next seed
    if (!PASS) counts[i] = n;
}

// ---------------------------------------------------------------------------------------------------------------
// record slicing (pack_record on the device)
// ---------------------------------------------------------------------------------------------------------------
struct SlicePlan { uint64_t cigar, seq, ml, mm; };    // offsets into the inflated stream

struct AuxHitDev { uint32_t type, sub, n; uint64_t p; bool found; };

// first occurrence of tag (a, b); mirrors aux_find of csrc/host/bam_reader.hpp (malformed aux data ends the search)
__device__ AuxHitDev aux_find_dev(const uint8_t* bam, uint64_t aux, uint64_t end, uint8_t a, uint8_t b) {
    AuxHitDev h; h.found = false; h.type = h.sub = h.n = 0; h.p = 0;
    uint64_t p = aux;
    while (p + 3 <= end) {
        const uint8_t t0 = bam[p], t1 = bam[p + 1], ty = bam[p + 2];
        p += 3;
        uint64_t sz; uint32_t n = 0, sub = 0; uint64_t vp = p;
        switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'Z': case 'H': { uint64_t q = p; while (q < end && bam[q]) q++; if (q >= end) return h; n = (uint32_t)(q - p); sz = (uint64_t)n + 1; break; }
            case 'B': {
                if (p + 5 > end) return h;
                sub = bam[p]; n = ld_u32(bam + p + 1);
                const uint64_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                vp = p + 5; sz = 5 + es * (uint64_t)n;
                break;
            }
            default: return h;
        }
        if (p + sz > end) return h;
        if (t0 == a && t1 == b) { h.found = true; h.type = ty; h.sub = sub; h.n = n; h.p = vp; return h; }
        p += sz;
    }
    return h;
}

// ---- one pass over the aux area by a whole warp: the first occurrence of each of K tags, with the same stop rule as aux_find_dev
//      (malformed data ends the walk; what was found before stays found). All lanes follow the same cursor and return the same
//      result; the end of a Z / H value - the MM text is several KB - is searched by the 32 lanes together, 1 KB per round.
//      (reads whole aligned 8-byte words: the inflated stream has 64 bytes of slack behind it, mkp_bam_load)
__device__ __forceinline__ uint64_t warp_find_nul(const uint8_t* bam, uint64_t q, uint64_t end, uint32_t lane) {
    for (uint64_t base = q & ~7ull; base < end; base += 1024) {
        uint64_t w[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { const uint64_t a = base + 256u * k + 8u * lane; w[k] = a < end ? *(const uint64_t*)(bam + a) : ~0ull; }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint64_t a = base + 256u * k + 8u * lane;
            uint64_t v = w[k];
            if (a < q) v |= q - a >= 8 ? ~0ull : (1ull << (8 * (q - a))) - 1ull;                  // bytes in front of the value
            if (a < end && a + 8 > end) v |= ~0ull << (8 * (end - a));                             // bytes behind the record
            const uint64_t z = (v - 0x0101010101010101ull) & ~v & 0x8080808080808080ull;         // lowest set bit = first zero byte
            const uint32_t m = __ballot_sync(0xffffffffu, z != 0);
            if (m) {
                const int src = __ffs(m) - 1;
                const uint64_t zz = __shfl_sync(0xffffffffu, z, src);
                return base + 256u * k + 8u * src + ((__ffsll((long long)zz) - 1) >> 3);
            }
        }
    }
    return end;
}

template <int K>
__device__ __forceinline__ void aux_scan_warp(const uint8_t* bam, uint64_t aux, uint64_t end, const uint16_t (&want)[K], AuxHitDev (&hit)[K], uint32_t lane) {
#pragma unroll
    for (int k = 0; k < K; k++) { hit[k].found = false; hit[k].type = hit[k].sub = hit[k].n = 0; hit[k].p = 0; }
    uint64_t p = aux;
    while (p + 3 <= end) {
        const uint32_t tg = (uint32_t)bam[p] | ((uint32_t)bam[p + 1] << 8), ty = bam[p + 2];
        p += 3;
        uint64_t sz; uint32_t n = 0, sub = 0; uint64_t vp = p;
        switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'Z': case 'H': { const uint64_t q = warp_find_nul(bam, p, end, lane); if (q >= end) return; n = (uint32_t)(q - p); sz = (uint64_t)n + 1; break; }
            case 'B': {
                if (p + 5 > end) return;
                sub = bam[p]; n = ld_u32(bam + p + 1);
                const uint64_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                vp = p + 5; sz = 5 + es * (uint64_t)n;
                break;
            }
            default: return;
        }
        if (p + sz > end) return;
#pragma unroll
        for (int k = 0; k < K; k++) if (tg == want[k] && !hit[k].found) { hit[k].found = true; hit[k].type = ty; hit[k].sub = sub; hit[k].n = n; hit[k].p = vp; }
        p += sz;
    }
}
#define MKP_TAG2(a, b) ((uint16_t)((uint8_t)(a) | ((uint8_t)(b) << 8)))

// warp per selected record: header fields, source offsets, bytes needed
__global__ void __launch_bounds__(256) k_slice_plan(const uint8_t* __restrict__ bam, const mkp_bam_rec* __restrict__ recs, const uint32_t* __restrict__ ids, uint32_t n,
                                                    mkp_read_hdr* hdrs, SlicePlan* plan, uint32_t* need) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const mkp_bam_rec rc = recs[ids[i]];
    const uint8_t* r = bam + rc.off;
    const uint64_t r0 = rc.off, rend = rc.off + rc.size;
    mkp_read_hdr h;
    h.ref_start = (int32_t)ld_u32(r + 4);
    const uint32_t l_name = r[8];
    uint32_t n_cigar = ld_u16(r + 12);
    const uint32_t flag = ld_u16(r + 14);
    const int32_t ls = (int32_t)ld_u32(r + 16);
    h.l_seq = ls > 0 ? (uint32_t)ls : 0u;
    uint64_t cigar = r0 + 32 + l_name;
    const uint64_t seq = cigar + 4ull * n_cigar;
    const uint64_t aux = seq + (h.l_seq + 1) / 2 + h.l_seq;
    const uint16_t want[6] = {MKP_TAG2('C', 'G'), MKP_TAG2('M', 'M'), MKP_TAG2('M', 'm'), MKP_TAG2('M', 'L'), MKP_TAG2('M', 'l'), MKP_TAG2('M', 'N')};
    AuxHitDev hit[6];
    aux_scan_warp<6>(bam, aux, rend, want, hit, lane);
    // long CIGARs (> 65535 ops) live in the CG:B,I tag (SAMv1 4.2.2)
    if (n_cigar == 2) {
        const AuxHitDev cg = hit[0];
        if (cg.found && cg.type == 'B' && cg.sub == 'I') {
            const uint32_t c0 = ld_u32(bam + cigar);
            if ((c0 & 15) == 4 && (c0 >> 4) == h.l_seq) { cigar = cg.p; n_cigar = cg.n; }
        }
    }
    const AuxHitDev mm = hit[1].found ? hit[1] : hit[2];
    bool ok = mm.found && mm.type == 'Z';
    AuxHitDev ml; ml.found = false; ml.n = 0; ml.p = 0; ml.type = ml.sub = 0;
    if (ok) {
        ml = hit[3].found ? hit[3] : hit[4];
        ok = ml.found && ml.type == 'B' && ml.sub == 'C';
    }
    if (ok) {
        const AuxHitDev mn = hit[5];
        if (mn.found) {
            long long v = -1;
            const uint8_t* q = bam + mn.p;
            switch (mn.type) {
                case 'c': v = (int8_t)q[0]; break; case 'C': v = q[0]; break;
                case 's': v = (int16_t)ld_u16(q); break; case 'S': v = ld_u16(q); break;
                case 'i': v = (int32_t)ld_u32(q); break; case 'I': v = ld_u32(q); break;
                default: ok = false;
            }
            if (ok && (unsigned long long)v != (unsigned long long)h.l_seq) ok = false;
        }
    }
    if (lane) return;
    h.n_cigar = n_cigar;
    h.flags = flag | (ok ? 0u : MKP_RF_TAGS_INVALID);
    h.len_ml = ok ? ml.n : 0;
    h.len_mm = ok ? mm.n : 0;
    h.off = 0;
    hdrs[i] = h;
    SlicePlan pl; pl.cigar = cigar; pl.seq = seq; pl.ml = ok ? ml.p : 0; pl.mm = ok ? mm.p : 0;
    plan[i] = pl;
    const unsigned long long nb = 4ull * n_cigar + (h.l_seq + 1) / 2 + h.len_ml + h.len_mm;
    need[i] = (uint32_t)((nb + 15) & ~15ull);      // one read's block is < 4 GiB (BAM block_size is 32 bit)
}

// single block: exclusive u64 prefix sums of need[] (-> hdrs[i].off) and of hdrs[i].len_ml (-> entry_off[]),
// maxima of n_cigar and l_seq; totals[0] = heap bytes (last block unpadded, like the host packer), [1] = entries,
// [2] = max n_cigar, [3] = max l_seq
__global__ void __launch_bounds__(1024) k_slice_scan(mkp_read_hdr* hdrs, const uint32_t* __restrict__ need, uint32_t n, uint64_t* entry_off, uint64_t* totals) {
    __shared__ unsigned long long s_a[32], s_b[32];
    __shared__ unsigned long long c_a, c_b;
    __shared__ uint32_t s_mc[32], s_ml[32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) { c_a = 0; c_b = 0; }
    uint32_t mc = 1, ml = 1;
    unsigned long long last_pad = 0;
    __syncthreads();
    for (uint32_t b = 0; b < n; b += 1024) {
        const uint32_t i = b + threadIdx.x;
        unsigned long long a = 0, e = 0;
        if (i < n) {
            a = need[i]; e = hdrs[i].len_ml; mc = max(mc, hdrs[i].n_cigar); ml = max(ml, hdrs[i].l_seq);
            if (i == n - 1) { const mkp_read_hdr h = hdrs[i]; const unsigned long long nb = 4ull * h.n_cigar + (h.l_seq + 1) / 2 + h.len_ml + h.len_mm; last_pad = a - nb; }
        }
        unsigned long long ia = a, ie = e;
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long ta = __shfl_up_sync(0xffffffffu, ia, d), te = __shfl_up_sync(0xffffffffu, ie, d);
            if (lane >= (uint32_t)d) { ia += ta; ie += te; }
        }
        if (lane == 31) { s_a[wid] = ia; s_b[wid] = ie; }
        __syncthreads();
        if (wid == 0) {
            unsigned long long va = s_a[lane], vb = s_b[lane], xa = va, xb = vb;
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long ta = __shfl_up_sync(0xffffffffu, xa, d), tb = __shfl_up_sync(0xffffffffu, xb, d);
                if (lane >= (uint32_t)d) { xa += ta; xb += tb; }
            }
            s_a[lane] = xa - va; s_b[lane] = xb - vb;
        }
        __syncthreads();
        const unsigned long long exa = c_a + s_a[wid] + ia - a, exb = c_b + s_b[wid] + ie - e;
        if (i < n) { hdrs[i].off = exa; entry_off[i] = exb; }
        __syncthreads();
        if (threadIdx.x == 1023) { c_a = exa + a; c_b = exb + e; }
        __syncthreads();
    }
    // reductions
    for (int d = 16; d >= 1; d >>= 1) { mc = max(mc, __shfl_xor_sync(0xffffffffu, mc, d)); ml = max(ml, __shfl_xor_sync(0xffffffffu, ml, d)); last_pad = max(last_pad, __shfl_xor_sync(0xffffffffu, last_pad, d)); }
    __shared__ unsigned long long s_lp[32];
    if (lane == 0) { s_mc[wid] = mc; s_ml[wid] = ml; s_lp[wid] = last_pad; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t a = 1, b = 1; unsigned long long lp = 0;
        for (int w = 0; w < 32; w++) { a = max(a, s_mc[w]); b = max(b, s_ml[w]); lp = max(lp, s_lp[w]); }
        entry_off[n] = c_b;
        totals[0] = c_a - lp; totals[1] = c_b; totals[2] = a; totals[3] = b;
    }
}

// warp per record: CIGAR | SEQ | ML | MM into the heap block
__global__ void __launch_bounds__(256) k_slice_copy(const uint8_t* __restrict__ bam, const mkp_read_hdr* __restrict__ hdrs, const SlicePlan* __restrict__ plan,
                                                   uint32_t n, uint8_t* heap) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = w; i < n; i += nw) {
        const mkp_read_hdr h = hdrs[i];
        const SlicePlan pl = plan[i];
        uint8_t* d = heap + h.off;
        const uint32_t nc = 4u * h.n_cigar, ns = (h.l_seq + 1) / 2;
        const uint32_t total = nc + ns + h.len_ml + h.len_mm;
        // the four pieces back to back, then zeros up to the 16-byte block boundary (like the host packer); 4 destination
        // bytes per lane and step, sources read bytewise (unaligned)
        const uint32_t padded = (total + 15u) & ~15u;
        for (uint32_t k = 4 * lane; k < padded; k += 128) {
            uint32_t word = 0;
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const uint32_t x = k + t;
                uint8_t b = 0;
                if (x < nc) b = bam[pl.cigar + x];
                else if (x < nc + ns) b = bam[pl.seq + (x - nc)];
                else if (x < nc + ns + h.len_ml) b = bam[pl.ml + (x - nc - ns)];
                else if (x < total) b = bam[pl.mm + (x - nc - ns - h.len_ml)];
                word |= (uint32_t)b << (8 * t);
            }
            *(uint32_t*)(d + k) = word;
        }
    }
}

// ---- --partition-tag on the device front end: the values of up to 4 aux tags of the selected records (src/util.rs:670-688,
//      src/pileup/mod.rs:629-646). Per (record, tag) MKP_TAG_CELL bytes: [0] = aux type (0: tag absent or not stringable), [1] = value
//      length, [2..] = value bytes (Z/H text, or the raw little-endian scalar); a text longer than MKP_TAG_CELL - 3 sets the overflow flag.
__global__ void __launch_bounds__(256) k_tag_values(const uint8_t* __restrict__ bam, const mkp_bam_rec* __restrict__ recs, const uint32_t* __restrict__ ids, uint32_t n,
                                                    uint32_t tags_packed_lo, uint32_t tags_packed_hi, uint32_t n_tags, uint8_t* __restrict__ out, uint32_t* overflow) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const mkp_bam_rec rc = recs[ids[i]];
    const uint8_t* r = bam + rc.off;
    const uint32_t l_name = r[8], n_cigar = ld_u16(r + 12);
    const int32_t ls = (int32_t)ld_u32(r + 16);
    const uint64_t l_seq = ls > 0 ? (uint64_t)ls : 0;
    const uint64_t aux = rc.off + 32 + l_name + 4ull * n_cigar + (l_seq + 1) / 2 + l_seq, rend = rc.off + rc.size;
    // (unused slots ask for a tag no file can hold: 0xffff)
    const uint16_t want[4] = {(uint16_t)(tags_packed_lo & 0xffffu), (uint16_t)(n_tags > 1 ? tags_packed_lo >> 16 : 0xffffu),
                              (uint16_t)(n_tags > 2 ? tags_packed_hi & 0xffffu : 0xffffu), (uint16_t)(n_tags > 3 ? tags_packed_hi >> 16 : 0xffffu)};
    AuxHitDev hit[4];
    aux_scan_warp<4>(bam, aux < rend ? aux : rend, rend, want, hit, lane);
#pragma unroll
    for (uint32_t t = 0; t < 4; t++) {
        if (t >= n_tags) break;
        uint8_t* o = out + ((size_t)i * n_tags + t) * MKP_TAG_CELL;
        const AuxHitDev h = hit[t];
        uint32_t len = 0;
        bool have = h.found;
        if (have) switch (h.type) {
            case 'Z': case 'H': len = h.n; break;
            case 'A': case 'c': case 'C': len = 1; break;
            case 's': case 'S': len = 2; break;
            case 'i': case 'I': case 'f': len = 4; break;
            default: have = false;                               // B arrays are not stringable: the tag counts as missing
        }
        if (len > MKP_TAG_CELL - 3) { if (lane == 0) atomicOr(overflow, 1u); len = MKP_TAG_CELL - 3; }
        if (lane == 0) { o[0] = have ? (uint8_t)h.type : 0; o[1] = have ? (uint8_t)len : 0; }
        for (uint32_t k = lane; have && k < len; k += 32) o[2 + k] = bam[h.p + k];
    }
}

// ---- the same values without a length limit (mkp_bam_tag_values): a warp per selected record finds up to 4 tags and writes,
//      per item k = i * n_tags + t, the aux type (0: absent or a B array), the value length and the value's offset in the
//      inflated stream; the lengths are then scanned and k_tag_value_copy packs the values at their offsets.
__global__ void __launch_bounds__(256) k_tag_value_lens(const uint8_t* __restrict__ bam, const mkp_bam_rec* __restrict__ recs, const uint32_t* __restrict__ ids, uint32_t n,
                                                        uint32_t tags_packed_lo, uint32_t tags_packed_hi, uint32_t n_tags,
                                                        uint8_t* __restrict__ types, uint32_t* __restrict__ lens, uint64_t* __restrict__ src, unsigned long long* total) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const mkp_bam_rec rc = recs[ids[i]];
    const uint8_t* r = bam + rc.off;
    const uint32_t l_name = r[8], n_cigar = ld_u16(r + 12);
    const int32_t ls = (int32_t)ld_u32(r + 16);
    const uint64_t l_seq = ls > 0 ? (uint64_t)ls : 0;
    const uint64_t aux = rc.off + 32 + l_name + 4ull * n_cigar + (l_seq + 1) / 2 + l_seq, rend = rc.off + rc.size;
    const uint16_t want[4] = {(uint16_t)(tags_packed_lo & 0xffffu), (uint16_t)(n_tags > 1 ? tags_packed_lo >> 16 : 0xffffu),
                              (uint16_t)(n_tags > 2 ? tags_packed_hi & 0xffffu : 0xffffu), (uint16_t)(n_tags > 3 ? tags_packed_hi >> 16 : 0xffffu)};
    AuxHitDev hit[4];
    aux_scan_warp<4>(bam, aux < rend ? aux : rend, rend, want, hit, lane);
    if (lane) return;
    uint64_t sum = 0;
#pragma unroll
    for (uint32_t t = 0; t < 4; t++) {
        if (t >= n_tags) break;
        const AuxHitDev h = hit[t];
        uint32_t len = 0;
        uint8_t ty = h.found ? (uint8_t)h.type : 0;
        switch (ty) {
            case 'Z': case 'H': len = h.n; break;
            case 'A': case 'c': case 'C': len = 1; break;
            case 's': case 'S': len = 2; break;
            case 'i': case 'I': case 'f': len = 4; break;
            default: ty = 0;                                     // B arrays are not stringable: the tag counts as missing
        }
        const size_t k = (size_t)i * n_tags + t;
        types[k] = ty; lens[k] = len; src[k] = h.p;
        sum += len;
    }
    if (sum) atomicAdd(total, (unsigned long long)sum);
}

// warp per item: the value bytes to out[offs[k] ..)
__global__ void __launch_bounds__(256) k_tag_value_copy(const uint8_t* __restrict__ bam, const uint32_t* __restrict__ lens, const uint32_t* __restrict__ offs,
                                                        const uint64_t* __restrict__ src, uint32_t m, uint8_t* __restrict__ out) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (k >= m) return;
    const uint32_t len = lens[k];
    const uint8_t* s = bam + src[k];
    uint8_t* o = out + offs[k];
    for (uint32_t b = lane; b < len; b += 32) o[b] = s[b];
}

}  // namespace mkp
