// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// Minimal BGZF/BAM reader for the CPU restatement of `modkit pileup`.
// The reference reaches BAM through rust-htslib 0.46 / htslib (third-party, not in the
// reference tree); this file restates the published SAM/BAM spec (SAMv1 §4) for the
// few things the pileup path touches: BGZF members, header, records, aux tags,
// region fetch (htslib `sam_itr_queryi` semantics: records with pos < end && endpos > beg)
// and per-contig mapped counts (htslib `hts_idx_get_stat`, consumed at
// src/reads_sampler/sampling_schedule.rs:683-722).
#pragma once
#include <zlib.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

namespace orc {

inline uint16_t rd16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline int32_t rdi32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }

struct BamRecord {
    const uint8_t* data = nullptr;  // points at refID (after block_size)
    uint32_t size = 0;              // block_size
    const uint8_t* cg = nullptr;    // the CG:B,I array when the core CIGAR is its placeholder (attach_long_cigar)
    uint32_t n_cg = 0;
    int32_t tid() const { return rdi32(data); }
    int32_t pos() const { return rdi32(data + 4); }
    uint8_t l_name() const { return data[8]; }
    uint16_t n_cigar_core() const { return rd16(data + 12); }   // the ops stored in the record's core (its layout)
    uint32_t n_cigar() const { return cg ? n_cg : n_cigar_core(); }
    uint16_t flag() const { return rd16(data + 14); }
    int32_t l_seq() const { return rdi32(data + 16); }
    const char* name() const { return (const char*)(data + 32); }
    const uint8_t* cigar() const { return data + 32 + l_name(); }
    const uint8_t* seq() const { return cigar() + 4 * (size_t)n_cigar_core(); }
    const uint8_t* qual() const { return seq() + (l_seq() + 1) / 2; }
    const uint8_t* aux() const { return qual() + l_seq(); }
    const uint8_t* end() const { return data + size; }
    bool is_reverse() const { return flag() & 0x10; }
    bool is_unmapped() const { return flag() & 0x4; }
    uint32_t cigar_op(int i) const { return rd32((cg ? cg : cigar()) + 4 * (size_t)i); }
    // reference length consumed (M,D,N,=,X)
    int64_t rlen() const {
        int64_t r = 0;
        for (int i = 0; i < n_cigar(); i++) {
            uint32_t c = cigar_op(i);
            int op = c & 0xf;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) r += c >> 4;
        }
        return r;
    }
    // htslib bam_endpos: pos + (rlen ? rlen : 1); unmapped/no-cigar => pos + 1
    int64_t endpos() const {
        int64_t r = (is_unmapped() || n_cigar() == 0) ? 0 : rlen();
        return (int64_t)pos() + (r ? r : 1);
    }
    char base_at(int q) const {  // 4-bit decode
        static const char* T = "=ACMGRSVTWYHKDBN";
        uint8_t b = seq()[q >> 1];
        return T[(q & 1) ? (b & 0xf) : (b >> 4)];
    }
};

struct AuxField {
    char type = 0;      // 'Z','B','c','C','s','S','i','I', ...
    char subtype = 0;   // for 'B'
    const uint8_t* p = nullptr;
    uint32_t n = 0;     // elements ('B') or strlen ('Z')
};

// Walk aux fields to find `tag`. Returns false when absent (or aux malformed).
inline bool find_aux(const BamRecord& r, const char tag[2], AuxField* out) {
    const uint8_t* p = r.aux();
    const uint8_t* e = r.end();
    while (p + 3 <= e) {
        char t0 = p[0], t1 = p[1], ty = p[2];
        p += 3;
        AuxField f;
        f.type = ty;
        size_t sz = 0;
        switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'Z': case 'H': {
                const uint8_t* q = p;
                while (q < e && *q) q++;
                f.p = p; f.n = (uint32_t)(q - p);
                sz = (q - p) + 1;
                break;
            }
            case 'B': {
                if (p + 5 > e) return false;
                f.subtype = (char)p[0];
                f.n = rd32(p + 1);
                size_t es = (f.subtype == 'c' || f.subtype == 'C') ? 1
                          : (f.subtype == 's' || f.subtype == 'S') ? 2 : 4;
                f.p = p + 5;
                sz = 5 + es * (size_t)f.n;
                break;
            }
            default: return false;
        }
        if (ty != 'Z' && ty != 'H' && ty != 'B') f.p = p;
        if (p + sz > e) return false;
        if (t0 == tag[0] && t1 == tag[1]) { *out = f; return true; }
        p += sz;
    }
    return false;
}

// Long CIGARs (more than 65535 ops, SAMv1 4.2.2): the core holds the placeholder `<l_seq>S <ref_len>N` and the real CIGAR is
// the CG:B,I array. htslib swaps the array in when it reads the record. The rule applied here is the product's packer's: two
// core ops, the first a soft clip of the whole query, and a CG tag of type B,I (DESIGN 7).
inline void attach_long_cigar(BamRecord* r) {
    r->cg = nullptr;
    r->n_cg = 0;
    if (r->n_cigar_core() != 2) return;
    const uint32_t c0 = rd32(r->cigar());
    if ((c0 & 0xf) != 4 || (int64_t)(c0 >> 4) != (int64_t)r->l_seq()) return;
    AuxField f;
    if (find_aux(*r, "CG", &f) && f.type == 'B' && f.subtype == 'I') { r->cg = f.p; r->n_cg = f.n; }
}

struct BamFile {
    std::vector<uint8_t> raw;           // whole decompressed stream
    std::string header_text;
    std::vector<std::string> ref_names;
    std::vector<uint32_t> ref_lens;
    std::vector<BamRecord> records;      // file order
    // per tid: indices into `records` (coordinate sorted), prefix max of endpos
    std::vector<std::vector<uint32_t>> by_tid;
    std::vector<std::vector<int64_t>> prefix_max_end;
    std::vector<uint32_t> unplaced;      // tid < 0
    std::vector<uint64_t> n_mapped, n_unmapped;  // == hts_idx_get_stat
    uint64_t n_no_coor = 0;

    static std::vector<uint8_t> slurp(const std::string& path) {
        FILE* f = fopen(path.c_str(), "rb");
        if (!f) throw std::runtime_error("cannot open " + path);
        fseek(f, 0, SEEK_END);
        long n = ftell(f);
        fseek(f, 0, SEEK_SET);
        std::vector<uint8_t> v((size_t)n);
        if (n && fread(v.data(), 1, (size_t)n, f) != (size_t)n) { fclose(f); throw std::runtime_error("short read " + path); }
        fclose(f);
        return v;
    }

    void load(const std::string& path, int threads = 1) {
        std::vector<uint8_t> comp = slurp(path);
        // pass 1: BGZF member boundaries (BSIZE in the BC extra subfield) + ISIZE
        struct Blk { size_t coff, clen; size_t uoff; uint32_t ulen; };
        std::vector<Blk> blks;
        size_t off = 0, utot = 0;
        while (off + 18 <= comp.size()) {
            const uint8_t* p = comp.data() + off;
            if (p[0] != 31 || p[1] != 139) throw std::runtime_error("not BGZF: " + path);
            uint16_t xlen = rd16(p + 10);
            const uint8_t* x = p + 12;
            const uint8_t* xe = x + xlen;
            int bsize = -1;
            while (x + 4 <= xe) {
                uint16_t slen = rd16(x + 2);
                if (x[0] == 'B' && x[1] == 'C' && slen == 2) bsize = rd16(x + 4);
                x += 4 + slen;
            }
            if (bsize < 0) throw std::runtime_error("BGZF block without BC field");
            size_t clen = (size_t)bsize + 1;
            uint32_t isize = rd32(p + clen - 4);
            blks.push_back({off + 12 + xlen, clen - 12 - xlen - 8, utot, isize});
            utot += isize;
            off += clen;
        }
        raw.resize(utot);
        auto work = [&](size_t b0, size_t b1) {
            for (size_t b = b0; b < b1; b++) {
                if (!blks[b].ulen) continue;
                z_stream zs;
                memset(&zs, 0, sizeof zs);
                if (inflateInit2(&zs, -15) != Z_OK) throw std::runtime_error("inflateInit2");
                zs.next_in = comp.data() + blks[b].coff;
                zs.avail_in = (uInt)blks[b].clen;
                zs.next_out = raw.data() + blks[b].uoff;
                zs.avail_out = blks[b].ulen;
                int rc = inflate(&zs, Z_FINISH);
                inflateEnd(&zs);
                if (rc != Z_STREAM_END) throw std::runtime_error("inflate failed");
            }
        };
        if (threads <= 1 || blks.size() < 8) {
            work(0, blks.size());
        } else {
            std::vector<std::thread> th;
            size_t per = (blks.size() + threads - 1) / threads;
            for (int t = 0; t < threads; t++) {
                size_t b0 = std::min(blks.size(), t * per), b1 = std::min(blks.size(), b0 + per);
                th.emplace_back(work, b0, b1);
            }
            for (auto& t : th) t.join();
        }
        parse();
    }

    void parse() {
        const uint8_t* p = raw.data();
        const uint8_t* e = p + raw.size();
        if (raw.size() < 12 || memcmp(p, "BAM\1", 4)) throw std::runtime_error("bad BAM magic");
        uint32_t l_text = rd32(p + 4);
        header_text.assign((const char*)p + 8, l_text);
        p += 8 + l_text;
        uint32_t n_ref = rd32(p);
        p += 4;
        for (uint32_t i = 0; i < n_ref; i++) {
            uint32_t l_name = rd32(p);
            ref_names.emplace_back((const char*)p + 4, l_name ? l_name - 1 : 0);
            ref_lens.push_back(rd32(p + 4 + l_name));
            p += 8 + l_name;
        }
        by_tid.assign(n_ref, {});
        prefix_max_end.assign(n_ref, {});
        n_mapped.assign(n_ref, 0);
        n_unmapped.assign(n_ref, 0);
        while (p + 4 <= e) {
            uint32_t bs = rd32(p);
            if (p + 4 + bs > e) throw std::runtime_error("truncated BAM record");
            BamRecord r;
            r.data = p + 4;
            r.size = bs;
            attach_long_cigar(&r);
            uint32_t idx = (uint32_t)records.size();
            records.push_back(r);
            int32_t tid = r.tid();
            if (tid >= 0 && (uint32_t)tid < n_ref) {
                by_tid[tid].push_back(idx);
                if (r.is_unmapped()) n_unmapped[tid]++; else n_mapped[tid]++;
            } else {
                unplaced.push_back(idx);
                n_no_coor++;
            }
            p += 4 + bs;
        }
        for (uint32_t t = 0; t < n_ref; t++) {
            int64_t m = -1;
            auto& pm = prefix_max_end[t];
            pm.reserve(by_tid[t].size());
            for (uint32_t idx : by_tid[t]) {
                m = std::max(m, records[idx].endpos());
                pm.push_back(m);
            }
        }
    }

    int tid_of(const std::string& name) const {
        for (size_t i = 0; i < ref_names.size(); i++) if (ref_names[i] == name) return (int)i;
        return -1;
    }

    // records overlapping [beg,end) on tid, in file order
    template <class F>
    void fetch(uint32_t tid, int64_t beg, int64_t end, F&& f) const {
        const auto& ids = by_tid[tid];
        const auto& pm = prefix_max_end[tid];
        size_t lo = std::upper_bound(pm.begin(), pm.end(), beg) - pm.begin();  // first with prefix max end > beg
        for (size_t i = lo; i < ids.size(); i++) {
            const BamRecord& r = records[ids[i]];
            if (r.pos() >= end) break;
            if (r.endpos() > beg) f(r);
        }
    }
};

}  // namespace orc
