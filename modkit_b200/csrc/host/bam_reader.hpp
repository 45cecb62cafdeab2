// Host-side BGZF/BAM/BAI access for the H100 pileup path (no htslib in this image: from scratch on zlib).
// Replaces what the reference gets from rust-htslib: IndexedReader::{from_path, fetch, index_stats}
// (src/pileup/mod.rs:732-743, src/reads_sampler/sampling_schedule.rs:683-722) and aux lookup
// (src/mod_bam.rs:1388-1470).  Records are sliced straight into the device layout of include/mkp.h.
#pragma once
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <charconv>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/mkp.h"

namespace mkh {

template <class T> inline T load_le(const uint8_t* p) { T v; memcpy(&v, p, sizeof(T)); return v; }

struct MappedFile {
    const uint8_t* data = nullptr;
    size_t size = 0;
    int fd = -1;
    void open(const std::string& path) {
        fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) throw std::runtime_error("cannot open " + path);
        struct stat st;
        if (fstat(fd, &st) != 0) throw std::runtime_error("cannot stat " + path);
        size = (size_t)st.st_size;
        if (size) {
            void* p = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
            if (p == MAP_FAILED) throw std::runtime_error("mmap failed for " + path);
            data = (const uint8_t*)p;
        }
    }
    ~MappedFile() { if (data) munmap((void*)data, size); if (fd >= 0) ::close(fd); }
};

// One alignment record, as offsets into the inflated stream
struct RecRef {
    uint64_t off;        // offset of refID field
    uint32_t size;       // block_size
    int32_t pos;
    int32_t end;         // htslib bam_endpos
    uint32_t idx;        // index in file order (record table of the device ingest)
    uint32_t l_seq;
    uint16_t flag;
};

// thrown by BamReader::open_device when file + inflated stream exceed the device memory: callers switch to open()
struct DeviceIngestTooBig : std::runtime_error { using std::runtime_error::runtime_error; };

struct BamIndexStats { std::vector<uint64_t> n_mapped, n_unmapped; uint64_t n_no_coor = 0; bool from_bai = false; };

class BamReader {
public:
    std::vector<uint8_t> raw;                 // inflated stream (whole file; v1 keeps it resident)
    std::vector<std::string> ref_names;
    std::vector<uint32_t> ref_lens;
    std::vector<std::vector<RecRef>> by_tid;  // coordinate order
    std::vector<std::vector<int32_t>> run_max_end;
    std::vector<RecRef> unplaced;
    BamIndexStats stats;

    bool on_device = false;                   // records live in the inflated stream on the GPU (open_device); raw is empty
    mkp_ctx* dev = nullptr;
    // BAI linear index (16 kb windows): smallest virtual offset of a record overlapping the window; empty without an index
    std::vector<std::vector<uint64_t>> lin;
    std::vector<uint64_t> ref_first_voff;     // virtual offset of the first record of every contig (UINT64_MAX: none)
    bool have_index() const { return have_bai_ && file_ != nullptr; }
    float ingest_ms[4] = {0, 0, 0, 0};        // device ingest: H2D, inflate, record walk, total

    struct Member { size_t in_off, in_len, out_off; uint32_t out_len; size_t file_off; };

    static std::vector<Member> scan_members(const MappedFile& mf, const std::string& path, size_t* total_out) {
        std::vector<Member> members;
        size_t off = 0, total = 0;
        while (off + 28 <= mf.size) {
            const uint8_t* p = mf.data + off;
            if (p[0] != 0x1f || p[1] != 0x8b || !(p[3] & 4)) throw std::runtime_error(path + ": not a BGZF file");
            const uint16_t xlen = load_le<uint16_t>(p + 10);
            int bsize = -1;
            for (size_t x = 12; x + 4 <= 12u + xlen;) {
                const uint16_t sl = load_le<uint16_t>(p + x + 2);
                if (p[x] == 'B' && p[x + 1] == 'C' && sl == 2) bsize = load_le<uint16_t>(p + x + 4);
                x += 4 + sl;
            }
            if (bsize < 0) throw std::runtime_error(path + ": BGZF member without BSIZE");
            const size_t mlen = (size_t)bsize + 1;
            if (off + mlen > mf.size) throw std::runtime_error(path + ": truncated BGZF member");
            const uint32_t isize = load_le<uint32_t>(p + mlen - 4);
            members.push_back({off + 12 + xlen, mlen - 20 - xlen, total, isize, off});
            total += isize;
            off += mlen;
        }
        *total_out = total;
        return members;
    }

    // The same chain walked in parallel: `hints` are compressed offsets that should be member starts (the BAI's virtual offsets).
    // A segment starts at a hint and must end exactly on the next segment's start; then the pieces are the chain from offset 0.
    // Anything else (a stale index, a malformed member) falls back to the serial walk, which also produces the error text.
    static std::vector<Member> scan_members_parallel(const MappedFile& mf, const std::string& path, std::vector<uint64_t> hints, int threads, size_t* total_out) {
        std::sort(hints.begin(), hints.end());
        hints.erase(std::unique(hints.begin(), hints.end()), hints.end());
        const size_t n_seg_want = (size_t)std::max(1, threads) * 8;
        std::vector<size_t> starts;
        starts.push_back(0);
        for (size_t k = 1; k < n_seg_want && !hints.empty(); k++) {
            const uint64_t want = (uint64_t)((double)mf.size * (double)k / (double)n_seg_want);
            auto it = std::lower_bound(hints.begin(), hints.end(), want);
            if (it == hints.end()) break;
            if (*it > starts.back() && *it + 28 <= mf.size) starts.push_back((size_t)*it);
        }
        size_t min_bytes = 64u << 20;                     // small files: the serial walk is faster than starting threads
        if (const char* e = getenv("MKH_PARALLEL_SCAN_MIN_BYTES")) min_bytes = (size_t)strtoull(e, nullptr, 10);     // (tests)
        if (starts.size() < 2 || mf.size < min_bytes) return scan_members(mf, path, total_out);
        const size_t n_seg = starts.size();
        std::vector<std::vector<Member>> seg(n_seg);
        std::vector<size_t> seg_total(n_seg, 0);
        std::atomic<size_t> next{0};
        std::atomic<bool> bad{false};
        auto work = [&]() {
            for (;;) {
                const size_t i = next.fetch_add(1);
                if (i >= n_seg || bad) break;
                const size_t stop = i + 1 < n_seg ? starts[i + 1] : mf.size;
                size_t off = starts[i], total = 0;
                std::vector<Member>& out = seg[i];
                while (off + 28 <= mf.size && off < stop) {
                    const uint8_t* p = mf.data + off;
                    if (p[0] != 0x1f || p[1] != 0x8b || !(p[3] & 4)) { bad = true; return; }
                    const uint16_t xlen = load_le<uint16_t>(p + 10);
                    if (off + 12 + xlen > mf.size) { bad = true; return; }
                    int bsize = -1;
                    for (size_t x = 12; x + 4 <= 12u + xlen;) {
                        const uint16_t sl = load_le<uint16_t>(p + x + 2);
                        if (p[x] == 'B' && p[x + 1] == 'C' && sl == 2 && x + 6 <= 12u + xlen) bsize = load_le<uint16_t>(p + x + 4);
                        x += 4 + sl;
                    }
                    const size_t mlen = (size_t)bsize + 1;
                    if (bsize < 0 || mlen < 20u + xlen || off + mlen > mf.size) { bad = true; return; }
                    const uint32_t isize = load_le<uint32_t>(p + mlen - 4);
                    out.push_back({off + 12 + xlen, mlen - 20 - xlen, total, isize, off});
                    total += isize;
                    off += mlen;
                }
                if (i + 1 < n_seg && off != stop) { bad = true; return; }
                seg_total[i] = total;
            }
        };
        {
            std::vector<std::thread> th;
            const int nt = (int)std::min<size_t>((size_t)std::max(1, threads), n_seg);
            for (int t = 1; t < nt; t++) th.emplace_back(work);
            work();
            for (auto& t : th) t.join();
        }
        if (getenv("MKH_SCAN_DEBUG")) fprintf(stderr, "[scan] segments %zu bad %d\n", n_seg, (int)bad.load());
        if (bad) return scan_members(mf, path, total_out);
        size_t n = 0, total = 0;
        for (auto& v : seg) n += v.size();
        std::vector<Member> members;
        members.reserve(n);
        for (size_t i = 0; i < n_seg; i++) {
            for (Member m : seg[i]) { m.out_off += total; members.push_back(m); }
            total += seg_total[i];
        }
        *total_out = total;
        return members;
    }

    void open(const std::string& path, int threads) {
        MappedFile mf;
        mf.open(path);
        size_t total = 0;
        std::vector<Member> members = scan_members(mf, path, &total);
        {   // this front end keeps the whole inflated stream in host memory: say so instead of being killed by the OOM killer
            const long pages = sysconf(_SC_AVPHYS_PAGES), psz = sysconf(_SC_PAGESIZE);
            if (pages > 0 && psz > 0 && (double)total > 0.9 * (double)pages * (double)psz)
                throw std::runtime_error(path + ": the host front end (--host-ingest / --partition-tag) inflates the whole file into memory (" + std::to_string(total >> 20) +
                                         " MiB) and only " + std::to_string(((uint64_t)pages * (uint64_t)psz) >> 20) + " MiB are available; use the GPU ingest (indexed BAM) or --region");
        }
        raw.resize(total + 16);
        std::atomic<size_t> next{0};
        std::atomic<bool> bad{false};
        auto work = [&]() {
            z_stream zs;
            memset(&zs, 0, sizeof zs);
            if (inflateInit2(&zs, -15) != Z_OK) { bad = true; return; }
            for (;;) {
                size_t b = next.fetch_add(16);
                if (b >= members.size()) break;
                for (size_t k = b; k < std::min(members.size(), b + 16); k++) {
                    const Member& m = members[k];
                    if (!m.out_len) continue;
                    inflateReset(&zs);
                    zs.next_in = (Bytef*)(mf.data + m.in_off); zs.avail_in = (uInt)m.in_len;
                    zs.next_out = raw.data() + m.out_off; zs.avail_out = m.out_len;
                    if (inflate(&zs, Z_FINISH) != Z_STREAM_END) bad = true;
                }
            }
            inflateEnd(&zs);
        };
        int nt = std::max(1, threads);
        std::vector<std::thread> th;
        for (int t = 1; t < nt; t++) th.emplace_back(work);
        work();
        for (auto& t : th) t.join();
        if (bad) throw std::runtime_error(path + ": inflate failed");
        index_records(total);
        load_bai(path, nullptr);
    }

    // Device ingest (include/mkp.h, mkp_bam_load): the host walks the BGZF member headers, inflates only the members
    // that hold the BAM header, and turns the BAI's virtual offsets into seed offsets for the record walk.
    // A file whose bytes + inflated stream fit in the device memory is loaded once. A bigger coordinate-sorted, indexed file
    // is loaded range by range (consecutive contigs, mkp_bam_load_range): ensure_tid() switches the resident range.
    void open_device(const std::string& path, mkp_ctx* ctx) {
        open_device_index(path, ctx);
        load_default();
    }

    // Step 1 of the device ingest: map the file, walk the member headers, read the BAM header and the index. Nothing is
    // copied to the device yet: callers either load everything (load_default) or only the byte ranges that hold the reads
    // of some reference pieces (load_pieces: one rank of an interval-sharded run, SURVEY 8e).
    void open_device_index(const std::string& path, mkp_ctx* ctx) {
        path_ = path;
        file_ = std::make_shared<MappedFile>();
        file_->open(path);
        const MappedFile& mf = *file_;
        total_ = 0;
        // ---- BAM header: inflate leading members until it is complete (a short serial walk of the member chain)
        std::vector<uint8_t> head;
        size_t h_off = 0;
        auto more = [&]() {
            if (h_off + 28 > mf.size) throw std::runtime_error(path + ": truncated BAM header");
            const uint8_t* p = mf.data + h_off;
            if (p[0] != 0x1f || p[1] != 0x8b || !(p[3] & 4)) throw std::runtime_error(path + ": not a BGZF file");
            const uint16_t xlen = load_le<uint16_t>(p + 10);
            int bsize = -1;
            for (size_t x = 12; x + 4 <= 12u + xlen && h_off + x + 6 <= mf.size;) {
                const uint16_t sl = load_le<uint16_t>(p + x + 2);
                if (p[x] == 'B' && p[x + 1] == 'C' && sl == 2) bsize = load_le<uint16_t>(p + x + 4);
                x += 4 + sl;
            }
            if (bsize < 0) throw std::runtime_error(path + ": BGZF member without BSIZE");
            const size_t mlen = (size_t)bsize + 1;
            if (mlen < 20u + xlen || h_off + mlen > mf.size) throw std::runtime_error(path + ": truncated BGZF member");
            Member m{h_off + 12 + xlen, mlen - 20 - xlen, 0, load_le<uint32_t>(p + mlen - 4), h_off};
            h_off += mlen;
            const size_t o = head.size();
            head.resize(o + m.out_len);
            if (!m.out_len) return;
            inflate_member(m, head.data() + o);
        };
        auto need = [&](size_t n) { while (head.size() < n) more(); };
        need(12);
        if (memcmp(head.data(), "BAM\1", 4) != 0) throw std::runtime_error("not a BAM stream");
        size_t o = 8 + load_le<uint32_t>(head.data() + 4);
        need(o + 4);
        const uint32_t n_ref = load_le<uint32_t>(head.data() + o);
        o += 4;
        for (uint32_t i = 0; i < n_ref; i++) {
            need(o + 4);
            const uint32_t ln = load_le<uint32_t>(head.data() + o);
            need(o + 8 + ln);
            ref_names.emplace_back((const char*)head.data() + o + 4, ln ? ln - 1 : 0);
            ref_lens.push_back(load_le<uint32_t>(head.data() + o + 4 + ln));
            o += 8 + ln;
        }
        by_tid.assign(n_ref, {});
        run_max_end.assign(n_ref, {});
        stats.n_mapped.assign(n_ref, 0);
        stats.n_unmapped.assign(n_ref, 0);
        // ---- index (also the per-contig read counts), then the member table (walked in parallel from the index's compressed
        // offsets when there is one)
        std::vector<uint64_t> voffs;
        have_bai_ = load_bai(path, &voffs, &ref_first_voff);
        {
            std::vector<uint64_t> hints;
            hints.reserve(voffs.size());
            for (uint64_t v : voffs) hints.push_back(v >> 16);
            members_ = have_bai_ ? scan_members_parallel(mf, path, std::move(hints), 16, &total_) : scan_members(mf, path, &total_);
        }
        const size_t total = total_;
        first_rec_ = o;
        // ---- seeds: virtual offsets of the index -> offsets in the inflated stream
        seeds_.clear();
        seeds_.push_back(first_rec_);
        for (uint64_t v : voffs) { uint64_t x; if (voff_to_offset(v, &x) && x > first_rec_ && x + 36 <= total) seeds_.push_back(x); }
        std::sort(seeds_.begin(), seeds_.end());
        seeds_.erase(std::unique(seeds_.begin(), seeds_.end()), seeds_.end());
        if (first_rec_ >= total) seeds_.clear();
        dev = ctx;
        on_device = true;
    }

    void release_host_tables() { std::vector<std::vector<RecRef>>().swap(by_tid); std::vector<Member>().swap(members_); std::vector<uint64_t>().swap(seeds_); run_max_end.clear(); run_max_end.shrink_to_fit(); }
    // virtual offset -> offset in the inflated stream (false: the compressed offset is not a member start)
    bool voff_to_offset(uint64_t v, uint64_t* x) const {
        const uint64_t coff = v >> 16, uoff = v & 0xffff;
        auto it = std::lower_bound(members_.begin(), members_.end(), coff, [](const Member& m, uint64_t c) { return m.file_off < c; });
        if (it == members_.end() || it->file_off != coff) return false;
        *x = it->out_off + uoff;
        return true;
    }
    size_t member_of_offset(uint64_t off) const {
        return (size_t)(std::upper_bound(members_.begin(), members_.end(), off, [](uint64_t x, const Member& m) { return x < m.out_off; }) - members_.begin()) - 1;
    }
    void inflate_member(const Member& m, uint8_t* dst) const {
        z_stream zs;
        memset(&zs, 0, sizeof zs);
        if (inflateInit2(&zs, -15) != Z_OK) throw std::runtime_error("zlib init failed");
        zs.next_in = (Bytef*)(file_->data + m.in_off); zs.avail_in = (uInt)m.in_len;
        zs.next_out = dst; zs.avail_out = m.out_len;
        const int rc = inflate(&zs, Z_FINISH);
        inflateEnd(&zs);
        if (rc != Z_STREAM_END) throw std::runtime_error(path_ + ": inflate failed");
    }

    // Offset (inflated stream) at or before the first record that overlaps reference position `pos` of contig tid: the
    // linear index entry of the 16 kb window holding pos (entries are non-decreasing; a zero entry means "no record":
    // the nearest earlier entry is used). UINT64_MAX when no record of the contig can overlap [pos, ...).
    uint64_t lower_bound_offset(uint32_t tid, uint64_t pos) const {
        if (tid >= lin.size() || tid >= ref_first_voff.size() || ref_first_voff[tid] == UINT64_MAX) return UINT64_MAX;
        const auto& L = lin[tid];
        size_t w = (size_t)(pos >> 14);
        if (w >= L.size()) return UINT64_MAX;        // beyond the last window that any record overlaps
        uint64_t v = 0;
        for (size_t k = w + 1; k-- > 0;) if (L[k]) { v = L[k]; break; }
        if (!v) v = ref_first_voff[tid];
        uint64_t x;
        if (!voff_to_offset(v, &x)) throw std::runtime_error(path_ + ": index offset is not a BGZF member start (stale index?)");
        return std::max<uint64_t>(x, first_rec_);
    }
    // compressed-file offset near the first record overlapping `pos` (shard weights only: monotone in (tid, pos))
    uint64_t approx_file_offset(uint32_t tid, uint64_t pos) const {
        if (tid >= lin.size() || tid >= ref_first_voff.size() || ref_first_voff[tid] == UINT64_MAX) {
            for (size_t t = (size_t)tid + 1; t < ref_first_voff.size(); t++) if (ref_first_voff[t] != UINT64_MAX) return ref_first_voff[t] >> 16;
            return file_ ? file_->size : 0;
        }
        const auto& L = lin[tid];
        size_t w = (size_t)(pos >> 14);
        if (w >= L.size()) {
            for (size_t t = (size_t)tid + 1; t < ref_first_voff.size(); t++) if (ref_first_voff[t] != UINT64_MAX) return ref_first_voff[t] >> 16;
            return file_ ? file_->size : 0;
        }
        for (size_t k = w + 1; k-- > 0;) if (L[k]) return L[k] >> 16;
        return ref_first_voff[tid] >> 16;
    }
    // offset of the first record of the first contig after tid that has records (or of the unplaced reads / end of stream)
    uint64_t contig_end_offset(uint32_t tid) const {
        for (size_t t = (size_t)tid + 1; t < ref_first_voff.size(); t++) {
            uint64_t x;
            if (ref_first_voff[t] != UINT64_MAX && voff_to_offset(ref_first_voff[t], &x)) return x;
        }
        return total_;      // (the reads without coordinates, if any, travel with the last contig)
    }

    // Step 2a: everything (or, when the file does not fit, contig ranges on demand)
    void load_default() {
        const MappedFile& mf = *file_;
        const size_t total = total_;
        const std::vector<Member>& members = members_;
        const uint32_t n_ref = (uint32_t)ref_names.size();
        const std::vector<uint64_t>& ref_first = ref_first_voff;
        auto to_offset = [&](uint64_t v, uint64_t* x) { return voff_to_offset(v, x); };
        mkp_ctx* ctx = dev;
        // ---- does everything fit at once?
        size_t free_b = 0, total_b = 0;
        const bool have_mem = mkp_device_memory(ctx, &free_b, &total_b) == 0;
        double budget = have_mem ? 0.55 * (double)free_b : 1e18;
        if (const char* e = getenv("MODKIT_B200_INGEST_BUDGET_MB")) budget = atof(e) * 1048576.0;
        auto cost = [](double file_bytes, double inflated) { return file_bytes + 1.6 * inflated; };
        if (cost((double)mf.size, (double)total) <= budget || !have_bai_ || ref_first.size() != n_ref) {
            if (have_mem && cost((double)mf.size, (double)total) + (double)(1ull << 30) > (double)free_b)
                throw DeviceIngestTooBig("BAM does not fit on the device for the GPU ingest (" + std::to_string(total >> 20) + " MiB inflated, " +
                                         std::to_string(free_b >> 20) + " MiB free" + (have_bai_ ? ")" : "; no index for a ranged load)"));
            ranged_ = false;
            if (!seeds_.empty()) load_members(0, members.empty() ? 0 : members.size() - 1, first_rec_, total);
            return;
        }
        // ---- ranged: consecutive contigs per load
        ranged_ = true;
        loaded_ = -1;
        std::vector<std::pair<uint64_t, uint32_t>> firsts;        // (offset of the contig's first record, tid)
        for (uint32_t t = 0; t < n_ref; t++) { uint64_t x; if (ref_first[t] != UINT64_MAX && to_offset(ref_first[t], &x) && x >= first_rec_ && x < total) firsts.push_back({x, t}); }
        for (size_t i = 1; i < firsts.size(); i++) if (firsts[i].first <= firsts[i - 1].first) throw DeviceIngestTooBig("BAM is not coordinate sorted by contig: no ranged GPU ingest");
        if (firsts.empty()) firsts.push_back({first_rec_, n_ref});   // only reads without coordinates
        firsts[0].first = first_rec_;
        batch_of_tid_.assign(n_ref, -1);
        batches_.clear();
        auto member_of = [&](uint64_t off) { return member_of_offset(off); };
        for (size_t i = 0; i < firsts.size();) {
            Batch bt;
            bt.start_off = firsts[i].first;
            bt.m0 = member_of(bt.start_off);
            size_t j = i;
            for (;;) {
                const uint64_t stop = j + 1 < firsts.size() ? firsts[j + 1].first : total;
                const size_t m1 = member_of(stop - 1);
                const double fb = (double)(members[m1].in_off + members[m1].in_len - members[bt.m0].file_off);
                const double ib = (double)(members[m1].out_off + members[m1].out_len - members[bt.m0].out_off);
                if (j > i && cost(fb, ib) > budget) break;
                bt.stop_off = stop; bt.m1 = m1;
                if (firsts[j].second < n_ref) batch_of_tid_[firsts[j].second] = (int)batches_.size();
                j++;
                if (j >= firsts.size()) break;
            }
            batches_.push_back(bt);
            i = j;
        }
        for (auto& bt : batches_) {
            const double fb = (double)(members[bt.m1].in_off + members[bt.m1].in_len - members[bt.m0].file_off);
            const double ib = (double)(members[bt.m1].out_off + members[bt.m1].out_len - members[bt.m0].out_off);
            if (have_mem && cost(fb, ib) + (double)(1ull << 30) > (double)free_b)
                throw DeviceIngestTooBig("one contig of the BAM does not fit on the device for the GPU ingest (" + std::to_string((uint64_t)ib >> 20) + " MiB inflated, " +
                                         std::to_string(free_b >> 20) + " MiB free)");
        }
    }

    // Step 2b: only the reads overlapping the given reference pieces (genome order, at most one piece per contig): the shard of
    // one rank. The byte range of a piece starts at the linear-index offset of its first window and ends where the next contig
    // starts, or - inside a contig - at the index offset of a window `margin` past the piece end; after the load the last record
    // must lie at or past the piece end, otherwise the margin grows and the range is loaded again. Needs the index.
    struct Piece { uint32_t tid, lo, hi; };
    void load_pieces(const std::vector<Piece>& pieces) {
        if (!have_bai_) throw std::runtime_error("interval-sharded runs need a BAM index (.bai)");
        const uint32_t n_ref = (uint32_t)ref_names.size();
        ranged_ = true;
        loaded_ = -1;
        batch_of_tid_.assign(n_ref, -1);
        batches_.clear();
        size_t free_b = 0, total_b = 0;
        const bool have_mem = mkp_device_memory(dev, &free_b, &total_b) == 0;
        double budget = have_mem ? 0.55 * (double)free_b : 1e18;
        if (const char* e = getenv("MODKIT_B200_INGEST_BUDGET_MB")) budget = atof(e) * 1048576.0;
        auto cost = [&](uint64_t a, uint64_t b) {
            const size_t m0 = member_of_offset(a), m1 = member_of_offset(b - 1);
            return (double)(members_[m1].in_off + members_[m1].in_len - members_[m0].file_off) + 1.6 * (double)(members_[m1].out_off + members_[m1].out_len - members_[m0].out_off);
        };
        for (size_t i = 0; i < pieces.size(); i++) {
            const Piece& pc = pieces[i];
            const uint64_t a = lower_bound_offset(pc.tid, pc.lo);
            if (a == UINT64_MAX) continue;                               // no record of the contig reaches the piece
            Batch nb;
            nb.start_off = a;
            nb.tid_last = pc.tid; nb.hi_last = pc.hi; nb.margin = 1u << 19;
            nb.stop_off = piece_stop(nb);
            if (nb.stop_off <= nb.start_off) continue;
            if (!batches_.empty() && cost(batches_.back().start_off, nb.stop_off) <= budget) {     // extend the open batch
                Batch& bt = batches_.back();
                bt.stop_off = std::max(bt.stop_off, nb.stop_off); bt.tid_last = nb.tid_last; bt.hi_last = nb.hi_last; bt.margin = nb.margin;
            } else batches_.push_back(nb);
            batch_of_tid_[pc.tid] = (int)batches_.size() - 1;
        }
        for (auto& bt : batches_) {
            bt.m0 = member_of_offset(bt.start_off); bt.m1 = member_of_offset(bt.stop_off - 1);
            if (have_mem && cost(bt.start_off, bt.stop_off) + (double)(1ull << 30) > (double)free_b)
                throw DeviceIngestTooBig("one contig piece of the BAM does not fit on the device for the GPU ingest");
        }
        if (batches_.size() == 1) load_batch(0);
    }

    // ---- host-side region fetch (BAI linear index + zlib): the equivalent of IndexedReader::fetch for the few thousand
    // records the threshold sampler looks at (src/reads_sampler/sampling_schedule.rs:683-722); independent of what is
    // resident on the device. Records overlapping [beg,end) of tid come out in file order.
    struct FetchCursor {
        uint32_t tid = 0; int64_t beg = 0, end = 0;
        size_t m_next = 0;             // next member to inflate
        uint64_t base_off = 0;         // inflated-stream offset of buf[0]
        std::vector<uint8_t> buf;
        size_t p = 0;                  // parse position in buf
        bool done = true;
        const uint8_t* bytes(const RecRef& r) const { return buf.data() + (r.off - base_off); }   // valid until the next fetch_more
    };
    FetchCursor fetch_begin(uint32_t tid, int64_t beg, int64_t end) const {
        FetchCursor c;
        c.tid = tid; c.beg = beg; c.end = end;
        const uint64_t x = lower_bound_offset(tid, (uint64_t)std::max<int64_t>(0, beg));
        if (x == UINT64_MAX || x >= total_) return c;
        c.m_next = member_of_offset(x);
        c.base_off = members_[c.m_next].out_off;
        c.p = (size_t)(x - c.base_off);
        c.done = false;
        return c;
    }
    // the reads without coordinates (tid -1) follow the last placed record
    FetchCursor fetch_unplaced_begin() const {
        FetchCursor c;
        c.tid = 0xffffffffu; c.beg = INT64_MIN; c.end = INT64_MAX;
        uint64_t x = first_rec_;
        for (size_t t = ref_first_voff.size(); t-- > 0;) {
            if (ref_first_voff[t] == UINT64_MAX || t >= lin.size() || lin[t].empty()) continue;
            const uint64_t y = lower_bound_offset((uint32_t)t, ((uint64_t)lin[t].size() - 1) << 14);
            if (y != UINT64_MAX) { x = y; break; }
        }
        if (x >= total_) return c;
        c.m_next = member_of_offset(x);
        c.base_off = members_[c.m_next].out_off;
        c.p = (size_t)(x - c.base_off);
        c.done = false;
        return c;
    }
    template <class F> size_t fetch_more(FetchCursor& c, size_t n, F&& ok, std::vector<RecRef>* out) const {
        size_t added = 0;
        if (c.p > (1u << 20)) { c.buf.erase(c.buf.begin(), c.buf.begin() + (ptrdiff_t)c.p); c.base_off += c.p; c.p = 0; }
        auto need = [&](size_t upto) {          // make buf hold at least `upto` bytes; false at the end of the stream
            while (c.buf.size() < upto) {
                if (c.m_next >= members_.size()) return false;
                const Member& m = members_[c.m_next++];
                const size_t o = c.buf.size();
                c.buf.resize(o + m.out_len);
                if (m.out_len) inflate_member(m, c.buf.data() + o);
            }
            return true;
        };
        while (!c.done && added < n) {
            if (!need(c.p + 4)) { c.done = true; break; }
            const uint32_t bs = load_le<uint32_t>(c.buf.data() + c.p);
            if (bs < 32) throw std::runtime_error(path_ + ": corrupt BAM record");
            if (!need(c.p + 4 + bs)) { c.done = true; break; }
            const uint8_t* r = c.buf.data() + c.p + 4;
            const int32_t tid = load_le<int32_t>(r), pos = load_le<int32_t>(r + 4);
            if (c.tid == 0xffffffffu) { if (tid >= 0) { c.p += 4 + bs; continue; } }           // reads without coordinates: the tail of the file
            else if (tid != (int32_t)c.tid) { if (tid >= 0 && tid < (int32_t)c.tid) { c.p += 4 + bs; continue; } c.done = true; break; }
            else if (pos >= c.end) { c.done = true; break; }
            const uint32_t l_name = r[8], n_cig = load_le<uint16_t>(r + 12), flag = load_le<uint16_t>(r + 14);
            { const int32_t ls = load_le<int32_t>(r + 16); const uint64_t lq = ls > 0 ? (uint64_t)ls : 0;
              if (32ull + l_name + 4ull * n_cig + (lq + 1) / 2 + lq > bs) throw std::runtime_error(path_ + ": corrupt BAM record"); }
            int64_t span = 0;
            if (!(flag & 4) && n_cig) {
                const uint8_t* cg = r + 32 + l_name;
                for (uint32_t k = 0; k < n_cig; k++) { const uint32_t v = load_le<uint32_t>(cg + 4 * k), op = v & 15; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += v >> 4; }
            }
            RecRef ref;
            ref.off = c.base_off + c.p + 4; ref.size = bs; ref.pos = pos; ref.end = (int32_t)(pos + (span ? span : 1));
            ref.idx = 0xffffffffu; ref.l_seq = load_le<uint32_t>(r + 16); ref.flag = (uint16_t)flag;
            c.p += 4 + bs;
            if (ref.end > c.beg && ok(ref)) { out->push_back(ref); added++; }
        }
        return added;
    }

    // make the records of contig tid resident (ranged device ingest; a no-op otherwise)
    void ensure_tid(uint32_t tid) const {
        if (!ranged_ || tid >= batch_of_tid_.size()) return;
        const int b = batch_of_tid_[tid];
        if (b >= 0 && b != loaded_) const_cast<BamReader*>(this)->load_batch(b);
    }
    // the reads without coordinates live at the end of the file: the last range
    void ensure_unplaced() const { if (ranged_ && !batches_.empty() && loaded_ != (int)batches_.size() - 1) const_cast<BamReader*>(this)->load_batch((int)batches_.size() - 1); }
    bool ranged() const { return ranged_; }
    size_t n_ranges() const { return ranged_ ? batches_.size() : 1; }

    // reads overlapping [beg,end) on tid in file order: half-open record span [pos, endpos)
    template <class F> void for_overlapping(uint32_t tid, int64_t beg, int64_t end, F&& f) const {
        const auto& v = by_tid[tid];
        const auto& rm = run_max_end[tid];
        size_t i = std::upper_bound(rm.begin(), rm.end(), (int32_t)std::min<int64_t>(beg, INT32_MAX)) - rm.begin();
        for (; i < v.size() && v[i].pos < end; i++) if (v[i].end > beg) f(v[i]);
    }
    const uint8_t* rec(const RecRef& r) const { if (on_device) throw std::runtime_error("record bytes are on the device"); return raw.data() + r.off; }

private:
    struct Batch {
        uint64_t start_off = 0, stop_off = 0; size_t m0 = 0, m1 = 0;
        int64_t tid_last = -1; uint32_t hi_last = 0, margin = 0;       // load_pieces: the piece that ends the batch (end check)
    };
    std::string path_;
    std::shared_ptr<MappedFile> file_;
    std::vector<Member> members_;
    std::vector<uint64_t> seeds_;             // known record starts (offsets in the whole inflated stream)
    size_t total_ = 0;
    uint64_t first_rec_ = 0;
    bool have_bai_ = false, ranged_ = false;
    std::vector<Batch> batches_;
    std::vector<int> batch_of_tid_;
    int loaded_ = -1;

    // end of the byte range of a batch that ends inside contig tid_last at hi_last (see load_pieces)
    uint64_t piece_stop(const Batch& bt) const {
        const uint32_t tid = (uint32_t)bt.tid_last;
        const uint64_t cend = contig_end_offset(tid);
        if (bt.hi_last >= ref_lens[tid]) return cend;
        const uint64_t far = (uint64_t)bt.hi_last + bt.margin;
        if (far >= ref_lens[tid]) return cend;
        uint64_t x = lower_bound_offset(tid, far);
        if (x == UINT64_MAX) return cend;
        // the record at x may start inside a member that the walk has to see whole: ranges end on record starts, fine
        return std::min(std::max(x, bt.start_off), cend);
    }

    void load_batch(int b) {
        for (;;) {
            Batch& bt = batches_[b];
            for (auto& v : by_tid) v.clear();
            for (auto& v : run_max_end) v.clear();
            unplaced.clear();
            if (bt.stop_off > bt.start_off) load_members(bt.m0, bt.m1, bt.start_off, bt.stop_off);
            loaded_ = b;
            if (bt.tid_last < 0) return;
            // a range that ends inside a contig must have seen a record starting at or past the piece end
            const uint32_t tid = (uint32_t)bt.tid_last;
            if (bt.stop_off >= contig_end_offset(tid)) return;
            const auto& v = by_tid[tid];
            if (!v.empty() && (uint32_t)std::max(0, v.back().pos) >= bt.hi_last) return;
            if (bt.margin >= (1u << 30)) { bt.stop_off = contig_end_offset(tid); }
            else { bt.margin <<= 2; bt.stop_off = std::max(bt.stop_off, piece_stop(bt)); }
            bt.m1 = member_of_offset(bt.stop_off - 1);
        }
    }

    // inflate members [m0, m1] on the device, walk the records of [start_off, stop_off) and index them
    void load_members(size_t m0, size_t m1, uint64_t start_off, uint64_t stop_off) {
        const MappedFile& mf = *file_;
        const uint32_t n_ref = (uint32_t)ref_names.size();
        const uint64_t fbase = members_[m0].file_off, obase = members_[m0].out_off;
        std::vector<mkp_bgzf_member> jobs;
        jobs.reserve(m1 - m0 + 1);
        for (size_t k = m0; k <= m1; k++) { const Member& m = members_[k]; if (m.out_len) jobs.push_back({(uint64_t)m.in_off - fbase, (uint64_t)m.out_off - obase, (uint32_t)m.in_len, m.out_len}); }
        std::vector<uint64_t> seeds;
        seeds.push_back(start_off - obase);
        for (auto it = std::upper_bound(seeds_.begin(), seeds_.end(), start_off); it != seeds_.end() && *it < stop_off; ++it) seeds.push_back(*it - obase);
        const uint64_t inflated = members_[m1].out_off + members_[m1].out_len - obase;
        const size_t flen = (size_t)(members_[m1].in_off + members_[m1].in_len + 8 - fbase);
        size_t n_rec = 0;
        float ms[4] = {0, 0, 0, 0};
        // the file bytes: copied out of the mapping (default), or - MKH_BAM_PREAD=1 - read with pread into the device layer's pinned
        // staging buffers (no page of the file mapped; slower per thread on tmpfs)
        static const bool use_pread = getenv("MKH_BAM_PREAD") && getenv("MKH_BAM_PREAD")[0] == '1';
        const size_t use_len = std::min(flen, mf.size - (size_t)fbase);
        if (use_pread ? mkp_bam_load_range_fd(dev, mf.fd, fbase, use_len, jobs.data(), jobs.size(), inflated, stop_off - obase, seeds.data(), seeds.size(), &n_rec, ms)
                      : mkp_bam_load_range(dev, mf.data + fbase, use_len, jobs.data(), jobs.size(), inflated, stop_off - obase, seeds.data(), seeds.size(), &n_rec, ms))
            throw std::runtime_error(std::string("device ingest: ") + mkp_last_error(dev));
        for (int i = 0; i < 4; i++) ingest_ms[i] += ms[i];
        std::vector<mkp_bam_rec> recs(n_rec);
        if (n_rec && mkp_bam_records(dev, recs.data())) throw std::runtime_error(std::string("device ingest: ") + mkp_last_error(dev));
        BamIndexStats scan;
        scan.n_mapped.assign(n_ref, 0); scan.n_unmapped.assign(n_ref, 0);
        for (size_t i = 0; i < n_rec; i++) {
            const mkp_bam_rec& d = recs[i];
            RecRef r;
            r.off = d.off + obase;      // identity of the record: offset in the whole inflated stream
            r.size = d.size; r.pos = d.pos; r.end = d.end; r.idx = (uint32_t)i; r.l_seq = d.l_seq; r.flag = (uint16_t)d.flag;
            if (d.tid >= 0 && (uint32_t)d.tid < n_ref) {
                by_tid[d.tid].push_back(r);
                if (d.flag & 4) scan.n_unmapped[d.tid]++; else scan.n_mapped[d.tid]++;
            } else { unplaced.push_back(r); scan.n_no_coor++; }
        }
        if (!have_bai_) stats = scan;
        for (uint32_t t = 0; t < n_ref; t++) {
            if (by_tid[t].empty()) continue;
            int32_t m = INT32_MIN;
            run_max_end[t].clear();
            run_max_end[t].reserve(by_tid[t].size());
            for (auto& r : by_tid[t]) { m = std::max(m, r.end); run_max_end[t].push_back(m); }
        }
    }

    void index_records(size_t total) {
        const uint8_t* p = raw.data();
        if (total < 12 || memcmp(p, "BAM\1", 4) != 0) throw std::runtime_error("not a BAM stream");
        size_t o = 8 + load_le<uint32_t>(p + 4);
        const uint32_t n_ref = load_le<uint32_t>(p + o);
        o += 4;
        for (uint32_t i = 0; i < n_ref; i++) {
            const uint32_t ln = load_le<uint32_t>(p + o);
            ref_names.emplace_back((const char*)p + o + 4, ln ? ln - 1 : 0);
            ref_lens.push_back(load_le<uint32_t>(p + o + 4 + ln));
            o += 8 + ln;
        }
        by_tid.assign(n_ref, {});
        run_max_end.assign(n_ref, {});
        stats.n_mapped.assign(n_ref, 0);
        stats.n_unmapped.assign(n_ref, 0);
        uint32_t n_seen = 0;
        while (o + 4 <= total) {
            const uint32_t bs = load_le<uint32_t>(p + o);
            if (o + 4 + bs > total || bs < 32) throw std::runtime_error("corrupt BAM record");
            const uint8_t* r = p + o + 4;
            RecRef ref;
            ref.off = o + 4; ref.size = bs;
            const int32_t tid = load_le<int32_t>(r);
            ref.pos = load_le<int32_t>(r + 4);
            const uint16_t flag = load_le<uint16_t>(r + 14);
            ref.idx = n_seen++; ref.flag = flag; ref.l_seq = load_le<uint32_t>(r + 16);
            const uint16_t n_cig = load_le<uint16_t>(r + 12);
            { const int32_t ls = load_le<int32_t>(r + 16); const uint64_t lq = ls > 0 ? (uint64_t)ls : 0;
              if (32ull + r[8] + 4ull * n_cig + (lq + 1) / 2 + lq > bs) throw std::runtime_error("corrupt BAM record (fields exceed the record size)"); }
            int64_t span = 0;
            if (!(flag & 4) && n_cig) {
                const uint8_t* c = r + 32 + r[8];
                for (uint16_t k = 0; k < n_cig; k++) {
                    const uint32_t v = load_le<uint32_t>(c + 4 * k);
                    const uint32_t op = v & 15;
                    if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += v >> 4;
                }
            }
            ref.end = (int32_t)(ref.pos + (span ? span : 1));
            if (tid >= 0 && (uint32_t)tid < n_ref) {
                by_tid[tid].push_back(ref);
                if (flag & 4) stats.n_unmapped[tid]++; else stats.n_mapped[tid]++;
            } else {
                unplaced.push_back(ref);
                stats.n_no_coor++;
            }
            o += 4 + bs;
        }
        for (uint32_t t = 0; t < n_ref; t++) {
            int32_t m = INT32_MIN;
            run_max_end[t].reserve(by_tid[t].size());
            for (auto& r : by_tid[t]) { m = std::max(m, r.end); run_max_end[t].push_back(m); }
        }
    }

    // BAI pseudo-bin 37450 (SAMv1 5.2): per-reference mapped/unmapped counts == hts_idx_get_stat
    bool load_bai(const std::string& bam_path, std::vector<uint64_t>* voffs, std::vector<uint64_t>* ref_first = nullptr) {
        std::string cand[2] = {bam_path + ".bai", bam_path.size() > 4 ? bam_path.substr(0, bam_path.size() - 4) + ".bai" : std::string()};
        for (auto& path : cand) {
            if (path.empty()) continue;
            FILE* f = fopen(path.c_str(), "rb");
            if (!f) continue;
            std::vector<uint8_t> b;
            uint8_t buf[65536];
            size_t n;
            while ((n = fread(buf, 1, sizeof buf, f)) > 0) b.insert(b.end(), buf, buf + n);
            fclose(f);
            if (b.size() < 8 || memcmp(b.data(), "BAI\1", 4) != 0) continue;
            size_t o = 4;
            const uint32_t n_ref = load_le<uint32_t>(b.data() + o);
            o += 4;
            if (n_ref != ref_names.size()) continue;
            BamIndexStats s;
            s.n_mapped.assign(n_ref, 0); s.n_unmapped.assign(n_ref, 0);
            if (ref_first) ref_first->assign(n_ref, UINT64_MAX);
            std::vector<std::vector<uint64_t>> lin_local(n_ref);
            auto note = [&](uint32_t r, uint64_t v) { if (ref_first && v && v < (*ref_first)[r]) (*ref_first)[r] = v; };
            bool ok = true;
            for (uint32_t r = 0; r < n_ref && ok; r++) {
                if (o + 4 > b.size()) { ok = false; break; }
                const uint32_t n_bin = load_le<uint32_t>(b.data() + o);
                o += 4;
                for (uint32_t k = 0; k < n_bin; k++) {
                    if (o + 8 > b.size()) { ok = false; break; }
                    const uint32_t bin = load_le<uint32_t>(b.data() + o), n_chunk = load_le<uint32_t>(b.data() + o + 4);
                    o += 8;
                    if (o + 16ull * n_chunk > b.size()) { ok = false; break; }
                    if (bin == 37450 && n_chunk == 2) {
                        s.n_mapped[r] = load_le<uint64_t>(b.data() + o + 16);
                        s.n_unmapped[r] = load_le<uint64_t>(b.data() + o + 24);
                    } else if (voffs) {
                        for (uint32_t c = 0; c < n_chunk; c++) { const uint64_t v = load_le<uint64_t>(b.data() + o + 16ull * c); voffs->push_back(v); note(r, v); }
                    }
                    o += 16ull * n_chunk;
                }
                if (!ok || o + 4 > b.size()) { ok = false; break; }
                const uint32_t n_intv = load_le<uint32_t>(b.data() + o);
                if (o + 4 + 8ull * n_intv > b.size()) { ok = false; break; }
                lin_local[r].resize(n_intv);
                for (uint32_t c = 0; c < n_intv; c++) lin_local[r][c] = load_le<uint64_t>(b.data() + o + 4 + 8ull * c);
                if (voffs) for (uint32_t c = 0; c < n_intv; c++) { const uint64_t v = lin_local[r][c]; voffs->push_back(v); note(r, v); }
                o += 4 + 8ull * n_intv;
            }
            if (!ok) { if (voffs) voffs->clear(); if (ref_first) ref_first->clear(); continue; }
            if (o + 8 <= b.size()) s.n_no_coor = load_le<uint64_t>(b.data() + o);
            s.from_bai = true;
            stats = s;
            lin.swap(lin_local);
            return true;
        }
        // no usable index: keep the counts taken while scanning the records (identical for a consistent index)
        return false;
    }
};

// ---- slicing BAM records into packed read blocks (include/mkp.h) --------------------------------
struct AuxHit { char type = 0, sub = 0; const uint8_t* p = nullptr; uint32_t n = 0; };

inline bool aux_find(const uint8_t* aux, const uint8_t* end, char a, char b, AuxHit* out) {
    const uint8_t* p = aux;
    while (p + 3 <= end) {
        const char t0 = (char)p[0], t1 = (char)p[1], ty = (char)p[2];
        p += 3;
        AuxHit h;
        h.type = ty;
        size_t sz;
        switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; h.p = p; break;
            case 's': case 'S': sz = 2; h.p = p; break;
            case 'i': case 'I': case 'f': sz = 4; h.p = p; break;
            case 'Z': case 'H': { const uint8_t* q = (const uint8_t*)memchr(p, 0, end - p); if (!q) return false; h.p = p; h.n = (uint32_t)(q - p); sz = h.n + 1; break; }
            case 'B': {
                if (p + 5 > end) return false;
                h.sub = (char)p[0];
                h.n = load_le<uint32_t>(p + 1);
                const size_t es = (h.sub == 'c' || h.sub == 'C') ? 1 : (h.sub == 's' || h.sub == 'S') ? 2 : 4;
                h.p = p + 5;
                sz = 5 + es * (size_t)h.n;
                break;
            }
            default: return false;
        }
        if (p + sz > end) return false;
        if (t0 == a && t1 == b) { *out = h; return true; }
        p += sz;
    }
    return false;
}

// Rust `{}` of an f32: shortest round-trip decimal, never in exponent form
inline std::string f32_display(float v) {
    char buf[64];
    auto r = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::fixed);
    return std::string(buf, r.ptr);
}

// --partition-tag: get_stringable_aux (src/util.rs:670-688): the text of one aux value of type `ty` at p (n: the length of a Z/H
// text); false for a type that is not stringable (B arrays)
inline bool aux_value_text(char ty, const uint8_t* p, size_t n, std::string* v) {
    switch (ty) {
        case 'Z': case 'H': v->assign((const char*)p, n); return true;
        case 'A': v->assign(1, (char)p[0]); return true;
        case 'c': *v = std::to_string((int)(int8_t)p[0]); return true;
        case 'C': *v = std::to_string((unsigned)p[0]); return true;
        case 's': *v = std::to_string(load_le<int16_t>(p)); return true;
        case 'S': *v = std::to_string(load_le<uint16_t>(p)); return true;
        case 'i': *v = std::to_string(load_le<int32_t>(p)); return true;
        case 'I': *v = std::to_string(load_le<uint32_t>(p)); return true;
        case 'f': *v = f32_display(load_le<float>(p)); return true;
        default: return false;
    }
}

// parse_tags_from_record (src/pileup/mod.rs:629-646): the values of tags 0 .. n_tags joined by '_', "missing" for absent ones;
// false when none of the tags is present (PartitionKey::NoKey). value(i, &v) is the text of tag i, or false when it is absent.
template <class Value>
inline bool partition_key_join(size_t n_tags, Value&& value, std::string* key) {
    bool any = false;
    std::string k, v;
    for (size_t i = 0; i < n_tags; i++) {
        const bool have = value(i, &v);
        any = any || have;
        if (i) k += "_";
        k += have ? v : std::string("missing");
    }
    if (any) *key = k;
    return any;
}

// the key of a record read on the host
inline bool partition_key_of(const uint8_t* r, uint32_t size, const std::vector<std::string>& tags, std::string* key) {
    const uint32_t l_name = r[8], n_cigar = load_le<uint16_t>(r + 12);
    const uint32_t l_seq = (uint32_t)std::max(0, load_le<int32_t>(r + 16));
    const uint8_t* aux = r + 32 + l_name + 4ull * n_cigar + (l_seq + 1) / 2 + l_seq;
    const uint8_t* end = r + size;
    return partition_key_join(tags.size(), [&](size_t i, std::string* v) {
        AuxHit h;
        return aux < end && aux_find(aux, end, tags[i][0], tags[i][1], &h) && aux_value_text(h.type, h.p, h.n, v);
    }, key);
}

// the same key from the MKP_TAG_CELL-byte (type, length, value) cells of mkp_bam_tags (device front end)
inline bool partition_key_of_cells(const uint8_t* cells, size_t n_tags, std::string* key) {
    return partition_key_join(n_tags, [&](size_t i, std::string* v) {
        const uint8_t* c = cells + (size_t)MKP_TAG_CELL * i;
        return c[0] != 0 && aux_value_text((char)c[0], c + 2, c[1], v);
    }, key);
}

// the same key from the (type, length, offset) items of mkp_bam_tag_values (device front end, values of any length)
inline bool partition_key_of_values(const uint8_t* types, const uint32_t* lens, const uint64_t* offs, const uint8_t* values, size_t n_tags, std::string* key) {
    return partition_key_join(n_tags, [&](size_t i, std::string* v) {
        return types[i] != 0 && aux_value_text((char)types[i], values + offs[i], lens[i], v);
    }, key);
}

struct PackedChunk {
    std::vector<mkp_read_hdr> hdrs;
    std::vector<uint8_t> heap;
    std::vector<RecRef> recs;      // provenance of each packed read
    void clear() { hdrs.clear(); heap.clear(); recs.clear(); }
    size_t algorithmic_bytes() const {
        size_t b = 0;
        for (auto& h : hdrs) b += 32 + 4ull * h.n_cigar + (h.l_seq + 1) / 2 + h.len_mm + h.len_ml;
        return b;
    }
};

// Append one BAM record. Resolves MM/Mm, ML/Ml, MN exactly like parse_raw_mod_tags (src/mod_bam.rs:1457-1470).
inline void pack_record(const uint8_t* r, uint32_t size, PackedChunk* out) {
    mkp_read_hdr h;
    memset(&h, 0, sizeof h);
    h.ref_start = load_le<int32_t>(r + 4);
    const uint32_t l_name = r[8];
    uint32_t n_cigar = load_le<uint16_t>(r + 12);
    const uint32_t flag = load_le<uint16_t>(r + 14);
    h.l_seq = (uint32_t)std::max(0, load_le<int32_t>(r + 16));
    const uint8_t* cigar = r + 32 + l_name;
    const uint8_t* seq = cigar + 4ull * n_cigar;
    const uint8_t* qual = seq + (h.l_seq + 1) / 2;
    const uint8_t* aux = qual + h.l_seq;
    const uint8_t* end = r + size;
    // long CIGARs (> 65535 ops) live in the CG:B,I tag (SAMv1 4.2.2)
    AuxHit cg;
    if (n_cigar == 2 && aux_find(aux, end, 'C', 'G', &cg) && cg.type == 'B' && cg.sub == 'I') {
        const uint32_t c0 = load_le<uint32_t>(cigar);
        if ((c0 & 15) == 4 && (c0 >> 4) == h.l_seq) { cigar = cg.p; n_cigar = cg.n; }
    }
    AuxHit mm, ml, mn;
    bool ok = (aux_find(aux, end, 'M', 'M', &mm) || aux_find(aux, end, 'M', 'm', &mm)) && mm.type == 'Z';
    ok = ok && (aux_find(aux, end, 'M', 'L', &ml) || aux_find(aux, end, 'M', 'l', &ml)) && ml.type == 'B' && ml.sub == 'C';
    if (ok && aux_find(aux, end, 'M', 'N', &mn)) {
        int64_t v = -1;
        switch (mn.type) {
            case 'c': v = (int8_t)mn.p[0]; break; case 'C': v = mn.p[0]; break;
            case 's': v = load_le<int16_t>(mn.p); break; case 'S': v = load_le<uint16_t>(mn.p); break;
            case 'i': v = load_le<int32_t>(mn.p); break; case 'I': v = load_le<uint32_t>(mn.p); break;
            default: ok = false;
        }
        if (ok && (uint64_t)v != (uint64_t)h.l_seq) ok = false;
    }
    h.n_cigar = n_cigar;
    h.flags = flag | (ok ? 0u : MKP_RF_TAGS_INVALID);
    h.len_ml = ok ? ml.n : 0;
    h.len_mm = ok ? mm.n : 0;
    size_t o = (out->heap.size() + 15) & ~(size_t)15;
    h.off = o;
    const size_t need = 4ull * n_cigar + (h.l_seq + 1) / 2 + h.len_ml + h.len_mm;
    out->heap.resize(o + need);
    uint8_t* d = out->heap.data() + o;
    memcpy(d, cigar, 4ull * n_cigar); d += 4ull * n_cigar;
    memcpy(d, seq, (h.l_seq + 1) / 2); d += (h.l_seq + 1) / 2;
    if (ok) { memcpy(d, ml.p, ml.n); d += ml.n; memcpy(d, mm.p, mm.n); }
    out->hdrs.push_back(h);
}

inline void pack_region(const BamReader& bam, uint32_t tid, uint32_t start, uint32_t end, PackedChunk* out) {
    bam.for_overlapping(tid, start, end, [&](const RecRef& r) { pack_record(bam.rec(r), r.size, out); out->recs.push_back(r); });
}

// Multi-threaded variant: records are planned (tag lookup, sizes) and copied in parallel; layout identical to pack_region.
inline void pack_records_mt(const BamReader& bam, const std::vector<RecRef>& recs, int threads, PackedChunk* out);
inline void pack_region_mt(const BamReader& bam, uint32_t tid, uint32_t start, uint32_t end, int threads, PackedChunk* out) {
    std::vector<RecRef> recs;
    bam.for_overlapping(tid, start, end, [&](const RecRef& r) { recs.push_back(r); });
    pack_records_mt(bam, recs, threads, out);
}
// the same for an explicit record list (one partition of a chunk, --partition-tag)
inline void pack_records_mt(const BamReader& bam, const std::vector<RecRef>& recs, int threads, PackedChunk* out) {
    const size_t n = recs.size();
    if (threads <= 1 || n < 512) { for (auto& r : recs) { pack_record(bam.rec(r), r.size, out); out->recs.push_back(r); } return; }
    struct Plan { const uint8_t *cigar, *seq, *ml, *mm; uint32_t n_ml, n_mm; };
    std::vector<Plan> plan(n);
    const size_t h0 = out->hdrs.size();
    out->hdrs.resize(h0 + n);
    std::vector<uint64_t> need(n);
    auto run = [&](auto&& body) {
        std::atomic<size_t> next{0};
        auto work = [&]() { for (;;) { size_t b = next.fetch_add(1024); if (b >= n) break; for (size_t i = b; i < std::min(n, b + 1024); i++) body(i); } };
        std::vector<std::thread> th;
        for (int t = 1; t < threads; t++) th.emplace_back(work);
        work();
        for (auto& t : th) t.join();
    };
    run([&](size_t i) {
        const uint8_t* r = bam.rec(recs[i]);
        const uint32_t size = recs[i].size;
        mkp_read_hdr h;
        memset(&h, 0, sizeof h);
        h.ref_start = load_le<int32_t>(r + 4);
        const uint32_t l_name = r[8];
        uint32_t n_cigar = load_le<uint16_t>(r + 12);
        const uint32_t flag = load_le<uint16_t>(r + 14);
        h.l_seq = (uint32_t)std::max(0, load_le<int32_t>(r + 16));
        const uint8_t* cigar = r + 32 + l_name;
        const uint8_t* seq = cigar + 4ull * n_cigar;
        const uint8_t* aux = seq + (h.l_seq + 1) / 2 + h.l_seq;
        const uint8_t* rend = r + size;
        AuxHit cg;
        if (n_cigar == 2 && aux_find(aux, rend, 'C', 'G', &cg) && cg.type == 'B' && cg.sub == 'I') {
            const uint32_t c0 = load_le<uint32_t>(cigar);
            if ((c0 & 15) == 4 && (c0 >> 4) == h.l_seq) { cigar = cg.p; n_cigar = cg.n; }
        }
        AuxHit mm, ml, mn;
        bool ok = (aux_find(aux, rend, 'M', 'M', &mm) || aux_find(aux, rend, 'M', 'm', &mm)) && mm.type == 'Z';
        ok = ok && (aux_find(aux, rend, 'M', 'L', &ml) || aux_find(aux, rend, 'M', 'l', &ml)) && ml.type == 'B' && ml.sub == 'C';
        if (ok && aux_find(aux, rend, 'M', 'N', &mn)) {
            int64_t v = -1;
            switch (mn.type) {
                case 'c': v = (int8_t)mn.p[0]; break; case 'C': v = mn.p[0]; break;
                case 's': v = load_le<int16_t>(mn.p); break; case 'S': v = load_le<uint16_t>(mn.p); break;
                case 'i': v = load_le<int32_t>(mn.p); break; case 'I': v = load_le<uint32_t>(mn.p); break;
                default: ok = false;
            }
            if (ok && (uint64_t)v != (uint64_t)h.l_seq) ok = false;
        }
        h.n_cigar = n_cigar;
        h.flags = flag | (ok ? 0u : MKP_RF_TAGS_INVALID);
        h.len_ml = ok ? ml.n : 0;
        h.len_mm = ok ? mm.n : 0;
        plan[i] = Plan{cigar, seq, ok ? ml.p : nullptr, ok ? mm.p : nullptr, h.len_ml, h.len_mm};
        need[i] = 4ull * n_cigar + (h.l_seq + 1) / 2 + h.len_ml + h.len_mm;
        out->hdrs[h0 + i] = h;
    });
    uint64_t o = (out->heap.size() + 15) & ~(uint64_t)15;
    for (size_t i = 0; i < n; i++) { out->hdrs[h0 + i].off = o; o = (o + need[i] + 15) & ~(uint64_t)15; }
    // pack_record leaves no padding after the last block: keep the same total size
    const uint64_t total = n ? out->hdrs[h0 + n - 1].off + need[n - 1] : out->heap.size();
    out->heap.resize(total);
    run([&](size_t i) {
        const mkp_read_hdr& h = out->hdrs[h0 + i];
        uint8_t* d = out->heap.data() + h.off;
        memcpy(d, plan[i].cigar, 4ull * h.n_cigar); d += 4ull * h.n_cigar;
        memcpy(d, plan[i].seq, (h.l_seq + 1) / 2); d += (h.l_seq + 1) / 2;
        if (plan[i].n_ml) { memcpy(d, plan[i].ml, plan[i].n_ml); d += plan[i].n_ml; }
        if (plan[i].n_mm) memcpy(d, plan[i].mm, plan[i].n_mm);
    });
    out->recs.insert(out->recs.end(), recs.begin(), recs.end());
}

// Device ingest: the reads overlapping [start,end) become the resident chunk (slicing happens on the GPU).
inline uint32_t device_chunk(const BamReader& bam, const std::vector<RecRef>& recs, uint32_t start, uint32_t end,
                             const uint32_t* focus_pos, const uint32_t* focus_neg) {
    std::vector<uint32_t> ids(recs.size());
    for (size_t i = 0; i < recs.size(); i++) ids[i] = recs[i].idx;
    if (mkp_bam_chunk(bam.dev, start, end, ids.data(), (uint32_t)ids.size(), focus_pos, focus_neg)) throw std::runtime_error(mkp_last_error(bam.dev));
    return (uint32_t)ids.size();
}

}  // namespace mkh
