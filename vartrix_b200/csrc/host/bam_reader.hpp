// bam_reader.hpp -- BGZF + BAM + BAI region reader for the staging host (own DEFLATE decoder, zlib as the
// fallback; htslib is not in this image).  Replaces what rust-htslib 0.36 / C htslib give the reference at
// vartrix src/main.rs:262, 470 (IndexedReader::from_path), 822-829 (fetch + records),
// 742/753 (Record::aux), 793-796 (cigar), 896 (seq).  Region semantics = the htslib iterator: every
// record of the contig with pos < end and bam_endpos > beg, in file order.
#pragma once
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fcntl.h>
#include <functional>
#include <string>
#include <sys/stat.h>
#include <unistd.h>
#include <vector>

#include "../../../include/vartrix_b200.h"
#include "../vtx_record.cuh"
#include "crc32_fast.hpp"
#include "inflate_fast.hpp"

namespace vtxhost {

// thread-seconds the staging threads spend per phase (reported by the CLI at --log-level info)
struct StageClock {
    std::atomic<uint64_t> read_ns{ 0 }, inflate_ns{ 0 }, crc_ns{ 0 }, blocks{ 0 }, inflated_bytes{ 0 }, device_inflate_ns{ 0 };
    static uint64_t now() { return uint64_t(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count()); }
};
inline StageClock& stage_clock() { static StageClock c; return c; }

inline uint16_t rd16(const uint8_t* p) { return uint16_t(p[0] | (p[1] << 8)); }
inline uint32_t rd32(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); }
inline uint64_t rd64(const uint8_t* p) { return uint64_t(rd32(p)) | (uint64_t(rd32(p + 4)) << 32); }

// ---------------------------------------------------------------------------------------------
// BGZF: concatenated gzip members (<= 64 KiB each) addressed by virtual offsets (coffset << 16 | uoffset)
// ---------------------------------------------------------------------------------------------
class Bgzf {
public:
    ~Bgzf() { close(); release_bulk_out(); }
    bool open(const std::string& path, std::string* err)
    {
        close();
        fd_ = ::open(path.c_str(), O_RDONLY);
        if (fd_ < 0) { *err = "cannot open " + path; return false; }
        struct stat st; fstat(fd_, &st); size_ = uint64_t(st.st_size);
        memset(&zs_, 0, sizeof(zs_));
        if (inflateInit2(&zs_, -15) != Z_OK) { *err = "inflateInit2 failed"; return false; }
        zinit_ = true;
        cbuf_.resize((1 << 16) + kInflateInPad);
        for (Slot& c : slots_) { c.coff = ~0ull; c.len = 0; }
        cur_ = nullptr; block_pos_ = 0; eof_ = false; clock_ = 0; err_.clear();
        return true;
    }
    void close()
    {
        if (zinit_) { inflateEnd(&zs_); zinit_ = false; }
        if (fd_ >= 0) { ::close(fd_); fd_ = -1; }
    }
    bool seek(uint64_t voff)
    {
        const uint64_t coff = voff >> 16; const uint32_t uoff = uint32_t(voff & 0xFFFF);
        if (!cur_ || coff != cur_->coff) { if (!load(coff)) return false; }
        if (uoff > cur_->len) return false;
        block_pos_ = uoff;
        return true;
    }
    uint64_t tell()
    {   // htslib convention: at the end of a block the position is the start of the next one
        if (!cur_) return 0;
        if (block_pos_ == cur_->len && cur_->len > 0) return cur_->next << 16;
        return (cur_->coff << 16) | block_pos_;
    }
    // read exactly n bytes; false at EOF / error
    bool read(void* dst, size_t n)
    {
        uint8_t* d = static_cast<uint8_t*>(dst);
        while (n) {
            if (!cur_ || block_pos_ == cur_->len) {
                if (!load(cur_ ? cur_->next : 0)) return false;
                if (cur_->len == 0) { if (eof_) return false; continue; }   // empty (EOF marker) block
            }
            const size_t k = std::min<size_t>(n, cur_->len - block_pos_);
            memcpy(d, cur_->ptr + block_pos_, k);
            d += k; n -= k; block_pos_ += uint32_t(k);
        }
        return true;
    }
    // the next n bytes in place when they lie inside the current block (no copy, position unchanged), else nullptr
    const uint8_t* peek(size_t n)
    {
        if (cur_ && block_pos_ == cur_->len && cur_->len > 0 && !load(cur_->next)) return nullptr;
        if (!cur_ || size_t(cur_->len - block_pos_) < n) return nullptr;
        return cur_->ptr + block_pos_;
    }
    void skip(size_t n) { block_pos_ += uint32_t(n); }     // only after a successful peek(>= n)
    bool at_eof() const { return eof_; }
    // Anything but a clean end of file (bad magic, truncated member, inflate or CRC failure, short read) is an ERROR, not
    // an end of region: the reference aborts on it (`let rec = _rec?`, main.rs:830), so the staging host must too.
    bool bad() const { return !err_.empty(); }
    const std::string& error() const { return err_; }

private:
    // Neighbouring loci fetch overlapping file ranges (every fetch restarts at its 16 kb index window): inflated
    // blocks stay in a small cache and are used in place.  48 x 64 KiB covers the ~10 blocks of a 16 kb window of
    // a deep BAM several times over, so the cyclic re-scan pattern of consecutive loci always hits.
    struct Slot { uint64_t coff = ~0ull, next = 0; uint32_t len = 0; const uint8_t* ptr = nullptr; std::vector<uint8_t> data; };
    static constexpr int kSlots = 48;
    Slot slots_[kSlots];
    Slot end_slot_;
    Slot* cur_ = nullptr;
    int clock_ = 0;

    bool fail(uint64_t coff, const char* what)
    {
        if (err_.empty()) err_ = std::string("BGZF block at file offset ") + std::to_string(coff) + ": " + what;
        return false;
    }
    bool load(uint64_t coff)
    {
        eof_ = false;
        if (!err_.empty()) return false;
        if (coff >= bulk_begin_ && coff < bulk_end_) {              // inflated in bulk on the device (prefetch_bulk)
            auto it = std::lower_bound(bulk_blocks_.begin(), bulk_blocks_.end(), coff, [](const BulkBlock& b, uint64_t c) { return b.coff < c; });
            if (it != bulk_blocks_.end() && it->coff == coff) {
                bulk_slot_.coff = coff; bulk_slot_.next = it->next; bulk_slot_.len = it->len; bulk_slot_.ptr = bulk_out_ + it->out_off;
                cur_ = &bulk_slot_; block_pos_ = 0;
                return true;
            }
        }
        for (Slot& c : slots_)
            if (c.coff == coff) { cur_ = &c; block_pos_ = 0; return true; }
        if (coff >= size_) {            // past the last block: an empty pseudo-block that the cache never serves
            eof_ = true; end_slot_.coff = coff; end_slot_.next = coff; end_slot_.len = 0; cur_ = &end_slot_; block_pos_ = 0;
            return false;
        }
        Slot* v = &slots_[clock_]; clock_ = (clock_ + 1) % kSlots;      // round robin; the outgoing current block is not needed again
        v->coff = ~0ull;
        if (cur_ == v) cur_ = nullptr;
        StageClock& clk = stage_clock();
        const uint64_t t_read = StageClock::now();
        uint8_t hdr[18];
        if (pread(fd_, hdr, 18, off_t(coff)) != 18) return fail(coff, "truncated file (short read of the member header)");
        if (hdr[0] != 31 || hdr[1] != 139 || hdr[2] != 8 || !(hdr[3] & 4)) return fail(coff, "not a BGZF member (bad gzip magic)");
        const uint32_t xlen = rd16(hdr + 10);
        // locate the BC subfield (normally the first and only one)
        uint32_t bsize = 0; bool have_bc = false;
        if (xlen == 6 && hdr[12] == 66 && hdr[13] == 67) { bsize = rd16(hdr + 16); have_bc = true; }
        else {
            std::vector<uint8_t> x(xlen);
            if (pread(fd_, x.data(), xlen, off_t(coff + 12)) != ssize_t(xlen)) return fail(coff, "truncated file (extra field)");
            for (uint32_t q = 0; q + 4 <= xlen;) {
                const uint32_t slen = rd16(x.data() + q + 2);
                if (x[q] == 66 && x[q + 1] == 67 && slen == 2 && q + 6 <= xlen) { bsize = rd16(x.data() + q + 4); have_bc = true; }
                q += 4 + slen;
            }
        }
        if (!have_bc) return fail(coff, "gzip member without the BGZF 'BC' field");
        const uint32_t total = bsize + 1;
        if (total < 12 + xlen + 8) return fail(coff, "BSIZE smaller than the member header");
        const uint32_t clen = total - 12 - xlen - 8;
        if (cbuf_.size() < total + kInflateInPad) cbuf_.resize(total + kInflateInPad);
        if (pread(fd_, cbuf_.data(), clen + 8, off_t(coff + 12 + xlen)) != ssize_t(clen + 8)) return fail(coff, "truncated file (short read of the member body)");
        const uint32_t crc = rd32(cbuf_.data() + clen), isize = rd32(cbuf_.data() + clen + 4);
        if (isize > (1u << 16)) return fail(coff, "ISIZE above 64 KiB");
        const uint64_t t_inf = StageClock::now();
        if (v->data.size() < (size_t(1) << 16) + kInflateOutPad) v->data.resize((size_t(1) << 16) + kInflateOutPad);
        if (isize && !vtx_inflate_raw(cbuf_.data(), clen, v->data.data(), isize)) {
            // the single-pass decoder refused the member: let zlib have the last word before calling the file corrupt
            inflateReset(&zs_);
            zs_.next_in = cbuf_.data(); zs_.avail_in = clen;
            zs_.next_out = v->data.data(); zs_.avail_out = isize;
            if (inflate(&zs_, Z_FINISH) != Z_STREAM_END || zs_.total_out != isize) return fail(coff, "inflate failed (corrupt data)");
        }
        const uint64_t t_crc = StageClock::now();
        if (check_crc_ && vtx_crc::crc32_of(v->data.data(), isize) != crc) return fail(coff, "CRC32 mismatch (corrupt data)");
        const uint64_t t_end = StageClock::now();
        clk.read_ns += t_inf - t_read; clk.inflate_ns += t_crc - t_inf; clk.crc_ns += t_end - t_crc; clk.blocks += 1; clk.inflated_bytes += isize;
        v->coff = coff; v->next = coff + total; v->len = isize; v->ptr = v->data.data();
        cur_ = v; block_pos_ = 0;
        return true;
    }
public:
    void set_check_crc(bool on) { check_crc_ = on; }
    // page-locked memory for the bulk buffer (the device copies straight into it): e.g. vtx_host_alloc / vtx_host_free
    void set_bulk_allocator(std::function<bool(void**, size_t)> a, std::function<void(void*)> f) { release_bulk_out(); bulk_alloc_ = std::move(a); bulk_free_ = std::move(f); }
    // Inflate every BGZF member that starts in [coff_begin, coff_last] in one go through `fn` (the device:
    // vtx_bgzf_inflate) and serve them from that buffer afterwards: the host only reads the compressed bytes and walks
    // the member headers.  Returns false on error (bad() tells whether the file is at fault); a range that cannot be
    // prefetched leaves the reader as it was and the members are inflated one by one on the host as before.
    using BulkInflate = std::function<bool(const vtx_bgzf_block*, uint32_t, const uint8_t*, uint64_t, uint8_t*, uint64_t, std::string*)>;
    bool prefetch_bulk(uint64_t coff_begin, uint64_t coff_last, const BulkInflate& fn)
    {
        if (cur_ == &bulk_slot_) cur_ = nullptr;
        bulk_begin_ = bulk_end_ = 0; bulk_blocks_.clear();
        if (coff_begin >= size_ || coff_last < coff_begin) return true;
        StageClock& clk = stage_clock();
        const uint64_t t0 = StageClock::now();
        // read the compressed range; the last member may reach up to 64 KiB beyond coff_last
        const uint64_t want_end = std::min<uint64_t>(size_, coff_last + (1u << 16) + 64);
        bulk_file_.resize(size_t(want_end - coff_begin));
        if (pread(fd_, bulk_file_.data(), bulk_file_.size(), off_t(coff_begin)) != ssize_t(bulk_file_.size())) return fail(coff_begin, "truncated file (bulk read)");
        bulk_desc_.clear(); bulk_comp_.clear();
        uint64_t pos = 0, out_off = 0;
        while (coff_begin + pos <= coff_last && coff_begin + pos < size_) {
            const uint8_t* h = bulk_file_.data() + pos;
            const uint64_t coff = coff_begin + pos;
            if (pos + 18 > bulk_file_.size()) return fail(coff, "truncated file (short read of the member header)");
            if (h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return fail(coff, "not a BGZF member (bad gzip magic)");
            const uint32_t xlen = rd16(h + 10);
            uint32_t bsize = 0; bool have_bc = false;
            for (uint32_t q = 0; q + 4 <= xlen && pos + 12 + q + 4 <= bulk_file_.size();) {
                const uint32_t slen = rd16(h + 12 + q + 2);
                if (h[12 + q] == 66 && h[12 + q + 1] == 67 && slen == 2 && q + 6 <= xlen) { bsize = rd16(h + 12 + q + 4); have_bc = true; }
                q += 4 + slen;
            }
            if (!have_bc) return fail(coff, "gzip member without the BGZF 'BC' field");
            const uint32_t total = bsize + 1;
            if (total < 12 + xlen + 8) return fail(coff, "BSIZE smaller than the member header");
            if (pos + total > bulk_file_.size()) return fail(coff, "truncated file (short read of the member body)");
            const uint32_t clen = total - 12 - xlen - 8;
            const uint32_t crc = rd32(h + total - 8), isize = rd32(h + total - 4);
            if (isize > (1u << 16)) return fail(coff, "ISIZE above 64 KiB");
            while (bulk_comp_.size() & 7) bulk_comp_.push_back(0);
            vtx_bgzf_block d{};
            d.in_off = bulk_comp_.size(); d.in_len = clen; d.out_len = isize; d.out_off = out_off; d.crc32 = crc;
            bulk_comp_.insert(bulk_comp_.end(), h + 12 + xlen, h + 12 + xlen + clen);
            bulk_desc_.push_back(d);
            bulk_blocks_.push_back({ coff, coff + total, out_off, isize });
            out_off += (uint64_t(isize) + 15) & ~uint64_t(15);
            pos += total;
        }
        bulk_comp_.resize(bulk_comp_.size() + 16, 0);                                   // readable padding behind the last payload
        if (size_t(out_off) + 16 > bulk_out_cap_) {          // grown geometrically; page-locked when the owner supplied such an allocator
            release_bulk_out();
            const size_t want = (size_t(out_off) + 16) * 5 / 4 + (1u << 20);
            if (bulk_alloc_) { void* q = nullptr; if (bulk_alloc_(&q, want)) bulk_out_ = static_cast<uint8_t*>(q); bulk_out_pinned_ = bulk_out_ != nullptr; }
            if (!bulk_out_) { bulk_out_ = static_cast<uint8_t*>(malloc(want)); bulk_out_pinned_ = false; }
            if (!bulk_out_) return fail(coff_begin, "out of memory (bulk inflate buffer)");
            bulk_out_cap_ = want;
        }
        const uint64_t t1 = StageClock::now();
        std::string e;
        if (!bulk_desc_.empty() && !fn(bulk_desc_.data(), uint32_t(bulk_desc_.size()), bulk_comp_.data(), bulk_comp_.size() - 16, bulk_out_, out_off, &e)) {
            bulk_blocks_.clear();
            if (err_.empty()) err_ = "device BGZF inflate: " + e;
            return false;
        }
        clk.read_ns += t1 - t0; clk.device_inflate_ns += StageClock::now() - t1; clk.blocks += bulk_desc_.size(); clk.inflated_bytes += out_off;
        if (!bulk_blocks_.empty()) { bulk_begin_ = bulk_blocks_.front().coff; bulk_end_ = bulk_blocks_.back().next; }
        return true;
    }
    // The members that start in [coff_begin, coff_last], NOT inflated: descriptors with out_off = running sum of ISIZE (one
    // contiguous stream), payloads packed on 8-byte boundaries into `comp` (16 readable bytes behind the last one), and for
    // every member its file offset -> stream offset (`index`, ascending; the last entry is (end of the last member, total)).
    struct MemberRef { uint64_t coff, stream_off; };
    bool read_members(uint64_t coff_begin, uint64_t coff_last, std::vector<vtx_bgzf_block>* desc, std::vector<uint8_t>* comp, std::vector<MemberRef>* index)
    {
        desc->clear(); comp->clear(); index->clear();
        if (coff_begin >= size_ || coff_last < coff_begin) { index->push_back({ coff_begin, 0 }); comp->resize(16, 0); return true; }
        const uint64_t t0 = StageClock::now();
        const uint64_t want_end = std::min<uint64_t>(size_, coff_last + (1u << 16) + 64);
        bulk_file_.resize(size_t(want_end - coff_begin));
        if (pread(fd_, bulk_file_.data(), bulk_file_.size(), off_t(coff_begin)) != ssize_t(bulk_file_.size())) return fail(coff_begin, "truncated file (bulk read)");
        uint64_t pos = 0, out_off = 0;
        while (coff_begin + pos <= coff_last && coff_begin + pos < size_) {
            const uint8_t* h = bulk_file_.data() + pos;
            const uint64_t coff = coff_begin + pos;
            if (pos + 18 > bulk_file_.size()) return fail(coff, "truncated file (short read of the member header)");
            if (h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return fail(coff, "not a BGZF member (bad gzip magic)");
            const uint32_t xlen = rd16(h + 10);
            uint32_t bsize = 0; bool have_bc = false;
            for (uint32_t q = 0; q + 4 <= xlen && pos + 12 + q + 4 <= bulk_file_.size();) {
                const uint32_t slen = rd16(h + 12 + q + 2);
                if (h[12 + q] == 66 && h[12 + q + 1] == 67 && slen == 2 && q + 6 <= xlen) { bsize = rd16(h + 12 + q + 4); have_bc = true; }
                q += 4 + slen;
            }
            if (!have_bc) return fail(coff, "gzip member without the BGZF 'BC' field");
            const uint32_t total = bsize + 1;
            if (total < 12 + xlen + 8) return fail(coff, "BSIZE smaller than the member header");
            if (pos + total > bulk_file_.size()) return fail(coff, "truncated file (short read of the member body)");
            const uint32_t clen = total - 12 - xlen - 8;
            const uint32_t crc = rd32(h + total - 8), isize = rd32(h + total - 4);
            if (isize > (1u << 16)) return fail(coff, "ISIZE above 64 KiB");
            while (comp->size() & 7) comp->push_back(0);
            vtx_bgzf_block d{};
            d.in_off = comp->size(); d.in_len = clen; d.out_len = isize; d.out_off = out_off; d.crc32 = crc;
            comp->insert(comp->end(), h + 12 + xlen, h + 12 + xlen + clen);
            desc->push_back(d);
            index->push_back({ coff, out_off });
            out_off += isize;
            pos += total;
        }
        index->push_back({ coff_begin + pos, out_off });
        comp->resize(comp->size() + 16, 0);
        StageClock& clk = stage_clock();
        clk.read_ns += StageClock::now() - t0; clk.blocks += desc->size(); clk.inflated_bytes += out_off;
        return true;
    }
private:
    struct BulkBlock { uint64_t coff, next, out_off; uint32_t len; };
    std::vector<BulkBlock> bulk_blocks_;
    std::vector<uint8_t> bulk_file_, bulk_comp_;
    uint8_t* bulk_out_ = nullptr;
    size_t bulk_out_cap_ = 0;
    bool bulk_out_pinned_ = false;
    std::function<bool(void**, size_t)> bulk_alloc_;
    std::function<void(void*)> bulk_free_;
    void release_bulk_out()
    {
        if (bulk_out_) { if (bulk_out_pinned_ && bulk_free_) bulk_free_(bulk_out_); else free(bulk_out_); }
        bulk_out_ = nullptr; bulk_out_cap_ = 0;
    }
    std::vector<vtx_bgzf_block> bulk_desc_;
    uint64_t bulk_begin_ = 0, bulk_end_ = 0;
    Slot bulk_slot_;
    std::string err_;
    bool check_crc_ = true;
    int fd_ = -1;
    uint64_t size_ = 0;
    z_stream zs_;
    bool zinit_ = false, eof_ = false;
    std::vector<uint8_t> cbuf_;
    uint32_t block_pos_ = 0;
};

// ---------------------------------------------------------------------------------------------
// BAM record view + BAI index
// ---------------------------------------------------------------------------------------------
struct BamRecord {
    // A view: `p` points at the record (without its block_size prefix) inside the reader's inflated block, or into `own`
    // when the record straddles two blocks.  Valid until the next BamFile::next / fetch on the reader that produced it.
    const uint8_t* p = nullptr;
    uint32_t len = 0;
    std::vector<uint8_t> own;
    uint64_t voff = 0;            // virtual offset of the record (identity of the record inside the file)
    int32_t refid() const { return int32_t(rd32(p)); }
    int32_t pos() const { return int32_t(rd32(p + 4)); }
    uint32_t l_read_name() const { return p[8]; }
    uint32_t mapq() const { return p[9]; }
    uint32_t n_cigar() const { return rd16(p + 12); }
    uint32_t flag() const { return rd16(p + 14); }
    int32_t l_seq() const { return int32_t(rd32(p + 16)); }
    const uint8_t* cigar() const { return p + 32 + l_read_name(); }
    const uint8_t* seq() const { return cigar() + 4 * n_cigar(); }
    const uint8_t* aux() const { return seq() + (l_seq() + 1) / 2 + l_seq(); }
    const uint8_t* end() const { return p + len; }
    // htslib bam_endpos (vtx::stage::ref_end): pos + reference length of the CIGAR; pos + 1 when unmapped / zero length
    int64_t endpos() const { return endpos_of(p); }
    static int64_t endpos_of(const uint8_t* d) { return vtx::stage::ref_end(d); }      // d = the record without its block_size prefix
    // first aux field named `tag`: value bytes when its type is 'Z' (vtx::stage::aux_z), else nullptr
    const uint8_t* aux_z(const char tag[2], uint32_t* len) const
    {
        const uint8_t* a = aux();
        uint32_t off = 0;
        return vtx::stage::aux_z(a, end(), uint8_t(tag[0]), uint8_t(tag[1]), &off, len) ? a + off : nullptr;
    }
};

struct BaiChunk { uint64_t beg, end; };
struct BaiRef {
    std::vector<uint32_t> bin_ids;
    std::vector<std::vector<BaiChunk>> bin_chunks;
    std::vector<uint64_t> linear;
};

class BamFile {
public:
    bool open(const std::string& path, std::string* err)
    {
        path_ = path;
        if (!bg_.open(path, err)) return false;
        uint8_t magic[4];
        if (!bg_.read(magic, 4) || memcmp(magic, "BAM\1", 4) != 0) { *err = path + " is not a BAM file"; return false; }
        uint8_t b4[4];
        if (!bg_.read(b4, 4)) { *err = "truncated BAM header"; return false; }
        std::vector<uint8_t> text(rd32(b4));
        if (!text.empty() && !bg_.read(text.data(), text.size())) { *err = "truncated BAM header"; return false; }
        if (!bg_.read(b4, 4)) { *err = "truncated BAM header"; return false; }
        const uint32_t n_ref = rd32(b4);
        for (uint32_t i = 0; i < n_ref; ++i) {
            if (!bg_.read(b4, 4)) { *err = "truncated BAM header"; return false; }
            std::vector<char> name(rd32(b4));
            if (!bg_.read(name.data(), name.size()) || !bg_.read(b4, 4)) { *err = "truncated BAM header"; return false; }
            ref_names.emplace_back(name.data());
            ref_lens.push_back(rd32(b4));
        }
        return load_index(err);
    }
    int tid_of(const std::string& chrom) const
    {
        for (size_t i = 0; i < ref_names.size(); ++i) if (ref_names[i] == chrom) return int(i);
        return -1;
    }
    std::vector<std::string> ref_names;
    std::vector<uint32_t> ref_lens;

    // htslib-style region iterator: call fetch(), then next() until it returns false
    bool fetch(int tid, int64_t beg, int64_t end)
    {
        chunks_.clear(); cur_ = 0; positioned_ = false; tid_ = tid; beg_ = beg; end_ = end; done_ = false;
        // Resume point of the previous region, valid for this one if it is on the same contig and does not start
        // earlier: the file is coordinate-sorted, so every record before the first record that overlapped
        // [prev_beg, prev_end) (or, if none did, before the record that ended that scan) ends at or before prev_beg
        // <= beg and cannot overlap the new region either.  Sorted VCFs therefore scan each stretch of the file once
        // instead of once per locus from the start of its 16 kb index window.
        const bool resume = hint_valid_ && tid == hint_tid_ && beg >= hint_beg_;
        const uint64_t resume_off = hint_voff_;
        hint_valid_ = false; hint_set_ = false; hint_tid_ = tid; hint_beg_ = beg;
        if (tid < 0 || size_t(tid) >= refs_.size()) { done_ = true; return false; }
        if (beg < 0) beg = 0;
        if (end <= beg) { done_ = true; return true; }
        const BaiRef& r = refs_[tid];
        uint64_t min_off = 0;
        if (!r.linear.empty()) {
            size_t w = size_t(beg >> 14);
            if (w >= r.linear.size()) w = r.linear.size() - 1;
            min_off = r.linear[w];
            // htslib walks back over empty windows; offsets are monotone so the entry itself is a safe lower bound
        }
        if (resume && resume_off > min_off) min_off = resume_off;
        start_off_ = min_off;
        const int64_t e1 = end - 1;
        auto add_bin = [&](uint32_t bin) {
            auto it = std::lower_bound(r.bin_ids.begin(), r.bin_ids.end(), bin);
            if (it == r.bin_ids.end() || *it != bin) return;
            for (const BaiChunk& c : r.bin_chunks[size_t(it - r.bin_ids.begin())]) if (c.end > min_off) chunks_.push_back(c);
        };
        add_bin(0);
        for (int64_t k = 1 + (beg >> 26); k <= 1 + (e1 >> 26); ++k) add_bin(uint32_t(k));
        for (int64_t k = 9 + (beg >> 23); k <= 9 + (e1 >> 23); ++k) add_bin(uint32_t(k));
        for (int64_t k = 73 + (beg >> 20); k <= 73 + (e1 >> 20); ++k) add_bin(uint32_t(k));
        for (int64_t k = 585 + (beg >> 17); k <= 585 + (e1 >> 17); ++k) add_bin(uint32_t(k));
        for (int64_t k = 4681 + (beg >> 14); k <= 4681 + (e1 >> 14); ++k) add_bin(uint32_t(k));
        std::sort(chunks_.begin(), chunks_.end(), [](const BaiChunk& a, const BaiChunk& b) { return a.beg < b.beg; });
        size_t w = 0;                         // merge overlapping / adjacent chunks so no record is visited twice
        for (size_t i = 0; i < chunks_.size(); ++i) {
            if (w && chunks_[i].beg <= chunks_[w - 1].end) chunks_[w - 1].end = std::max(chunks_[w - 1].end, chunks_[i].end);
            else chunks_[w++] = chunks_[i];
        }
        chunks_.resize(w);
        if (chunks_.empty()) done_ = true;
        return true;
    }
    // false = end of the region OR an error: check bad() afterwards (a corrupt or truncated file must abort the run
    // like the reference's `let rec = _rec?` does, main.rs:830, never shorten it silently)
    bool next(BamRecord* rec)
    {
        while (!done_) {
            if (!positioned_) {
                if (cur_ >= chunks_.size()) { done_ = true; break; }
                if (!bg_.seek(std::max(chunks_[cur_].beg, start_off_))) {          // start_off_ is a record boundary
                    if (bg_.bad()) return fail(bg_.error());
                    if (!bg_.at_eof()) return fail("BAM index points outside a BGZF block (index and file do not match)");
                    done_ = true; break;
                }
                positioned_ = true;
            }
            if (bg_.tell() >= chunks_[cur_].end) { ++cur_; positioned_ = false; continue; }
            const uint64_t voff = bg_.tell();
            // records that lie inside one BGZF block are examined in place; only those handed out are copied
            const uint8_t* p = bg_.peek(4);
            uint32_t bs = 0;
            const uint8_t* body = nullptr;
            if (p) { bs = rd32(p); if (bs >= 32) { const uint8_t* q = bg_.peek(4 + size_t(bs)); if (q) body = q + 4; } }
            if (bg_.bad()) return fail(bg_.error());
            if (body) {
                bg_.skip(4 + size_t(bs));
            } else {                                   // straddles a block boundary (or the file ends here): assemble a copy
                uint8_t b4[4];
                if (!bg_.read(b4, 1)) {                // not even one byte: a clean end of file between two records
                    if (bg_.bad()) return fail(bg_.error());
                    done_ = true; break;
                }
                if (!bg_.read(b4 + 1, 3)) return fail(bg_.bad() ? bg_.error() : "truncated BAM record (file ends inside a record)");
                bs = rd32(b4);
                if (bs < 32 || bs > (1u << 28)) return fail("corrupt BAM record (block_size " + std::to_string(bs) + ")");
                rec->own.resize(bs);
                if (!bg_.read(rec->own.data(), bs)) return fail(bg_.bad() ? bg_.error() : "truncated BAM record (file ends inside a record)");
                body = rec->own.data();
            }
            {   // the variable-length fields must lie inside the record: stager and endpos_of index them unchecked
                const int64_t l_seq = int32_t(rd32(body + 16));
                const uint64_t need = 32ull + body[8] + 4ull * rd16(body + 12) + (l_seq < 0 ? 0 : uint64_t(l_seq + 1) / 2 + uint64_t(l_seq));
                if (l_seq < 0 || need > bs) return fail("corrupt BAM record at virtual offset " + std::to_string(voff) + " (fields exceed block_size)");
            }
            if (int32_t(rd32(body)) != tid_ || int64_t(int32_t(rd32(body + 4))) >= end_) {          // sorted file: nothing further can overlap
                if (!hint_set_) { hint_voff_ = voff; hint_set_ = true; }
                hint_valid_ = true;
                done_ = true;
                break;
            }
            if (BamRecord::endpos_of(body) > beg_) {
                if (!hint_set_) { hint_voff_ = voff; hint_set_ = true; }
                rec->p = body; rec->len = bs;
                rec->voff = voff;
                return true;
            }
        }
        // the scan ran off the chunks (or the file) without meeting a record at or beyond `end`: the next region may
        // still resume at the first overlapping record, if there was one
        if (hint_set_) hint_valid_ = true;
        return false;
    }
    bool bad() const { return !err_.empty(); }
    const std::string& error() const { return err_; }
    void set_check_crc(bool on) { bg_.set_check_crc(on); }
    // A virtual offset at or before which every record with pos < end lies (sorted file): the first record the index files under
    // a 16 kb bin whose window starts behind `end` -- that record, and everything after it, starts at or behind `end`.  Chunks of
    // the wide bins (reads that cross 16 kb ... 64 Mb boundaries) reach far beyond a region; a sequential reader stops at the
    // first record with pos >= end, a bulk reader needs this bound instead.  ~0 when the index knows no later 16 kb bin.
    uint64_t upper_clip(int tid, int64_t end) const
    {
        if (tid < 0 || size_t(tid) >= refs_.size() || end <= 0) return ~0ull;
        const BaiRef& r = refs_[size_t(tid)];
        const uint32_t first_bin = 4681u + uint32_t(((end - 1) >> 14) + 1);
        for (auto it = std::lower_bound(r.bin_ids.begin(), r.bin_ids.end(), first_bin); it != r.bin_ids.end(); ++it) {
            const std::vector<BaiChunk>& cs = r.bin_chunks[size_t(it - r.bin_ids.begin())];
            if (cs.empty()) continue;
            uint64_t lo = ~0ull;
            for (const BaiChunk& c : cs) lo = std::min(lo, c.beg);
            return lo;
        }
        return ~0ull;
    }
    // Record boundaries the linear index knows inside (lo, hi): the first record overlapping each 16 kb window of [beg, end).
    // Entry points for a parallel record walk.  Appends to `out`.
    void linear_entries(int tid, int64_t beg, int64_t end, uint64_t lo, uint64_t hi, std::vector<uint64_t>* out) const
    {
        if (tid < 0 || size_t(tid) >= refs_.size() || end <= beg) return;
        const std::vector<uint64_t>& lin = refs_[size_t(tid)].linear;
        if (beg < 0) beg = 0;
        for (size_t w = size_t(beg >> 14); w < lin.size() && int64_t(w) <= ((end - 1) >> 14) + 1; ++w)
            if (lin[w] > lo && lin[w] < hi) out->push_back(lin[w]);
    }
    // Compressed-offset span [first, last] of the BGZF members a fetch(tid, beg, end) may touch (index chunks, before any
    // resume hint).  false when the index has nothing for the region.
    bool region_span(int tid, int64_t beg, int64_t end, uint64_t* c_first, uint64_t* c_last) const
    {
        if (tid < 0 || size_t(tid) >= refs_.size() || end <= beg) return false;
        if (beg < 0) beg = 0;
        const BaiRef& r = refs_[size_t(tid)];
        uint64_t min_off = 0;
        if (!r.linear.empty()) { size_t w = size_t(beg >> 14); if (w >= r.linear.size()) w = r.linear.size() - 1; min_off = r.linear[w]; }
        const int64_t e1 = end - 1;
        const uint64_t max_off = upper_clip(tid, end);
        uint64_t lo = ~0ull, hi = 0;
        auto add_bin = [&](uint32_t bin) {
            auto it = std::lower_bound(r.bin_ids.begin(), r.bin_ids.end(), bin);
            if (it == r.bin_ids.end() || *it != bin) return;
            for (const BaiChunk& c : r.bin_chunks[size_t(it - r.bin_ids.begin())])
                if (c.end > min_off && c.beg < max_off) { lo = std::min(lo, std::max(c.beg, min_off)); hi = std::max(hi, std::min(c.end, max_off)); }
        };
        add_bin(0);
        for (int64_t k = 1 + (beg >> 26); k <= 1 + (e1 >> 26); ++k) add_bin(uint32_t(k));
        for (int64_t k = 9 + (beg >> 23); k <= 9 + (e1 >> 23); ++k) add_bin(uint32_t(k));
        for (int64_t k = 73 + (beg >> 20); k <= 73 + (e1 >> 20); ++k) add_bin(uint32_t(k));
        for (int64_t k = 585 + (beg >> 17); k <= 585 + (e1 >> 17); ++k) add_bin(uint32_t(k));
        for (int64_t k = 4681 + (beg >> 14); k <= 4681 + (e1 >> 14); ++k) add_bin(uint32_t(k));
        if (lo == ~0ull) return false;
        *c_first = lo >> 16; *c_last = hi >> 16;
        return true;
    }
    // The index chunks a fetch(tid, beg, end) walks, as virtual-offset pairs (starts clamped to the linear index like fetch
    // does, ends clamped to upper_clip); every start and end is a record boundary.  Appends to `out`.
    void region_chunks(int tid, int64_t beg, int64_t end, std::vector<BaiChunk>* out) const
    {
        if (tid < 0 || size_t(tid) >= refs_.size() || end <= beg) return;
        if (beg < 0) beg = 0;
        const BaiRef& r = refs_[size_t(tid)];
        uint64_t min_off = 0;
        if (!r.linear.empty()) { size_t w = size_t(beg >> 14); if (w >= r.linear.size()) w = r.linear.size() - 1; min_off = r.linear[w]; }
        const int64_t e1 = end - 1;
        const uint64_t max_off = upper_clip(tid, end);
        auto add_bin = [&](uint32_t bin) {
            auto it = std::lower_bound(r.bin_ids.begin(), r.bin_ids.end(), bin);
            if (it == r.bin_ids.end() || *it != bin) return;
            for (const BaiChunk& c : r.bin_chunks[size_t(it - r.bin_ids.begin())])
                if (c.end > min_off && c.beg < max_off) out->push_back({ std::max(c.beg, min_off), std::min(c.end, max_off) });
        };
        add_bin(0);
        for (int64_t k = 1 + (beg >> 26); k <= 1 + (e1 >> 26); ++k) add_bin(uint32_t(k));
        for (int64_t k = 9 + (beg >> 23); k <= 9 + (e1 >> 23); ++k) add_bin(uint32_t(k));
        for (int64_t k = 73 + (beg >> 20); k <= 73 + (e1 >> 20); ++k) add_bin(uint32_t(k));
        for (int64_t k = 585 + (beg >> 17); k <= 585 + (e1 >> 17); ++k) add_bin(uint32_t(k));
        for (int64_t k = 4681 + (beg >> 14); k <= 4681 + (e1 >> 14); ++k) add_bin(uint32_t(k));
    }
    bool read_members(uint64_t c_first, uint64_t c_last, std::vector<vtx_bgzf_block>* desc, std::vector<uint8_t>* comp, std::vector<Bgzf::MemberRef>* index)
    {
        if (!bg_.read_members(c_first, c_last, desc, comp, index)) { if (bg_.bad()) fail(bg_.error()); return false; }
        return true;
    }
    void set_bulk_allocator(std::function<bool(void**, size_t)> a, std::function<void(void*)> f) { bg_.set_bulk_allocator(std::move(a), std::move(f)); }
    bool prefetch_bulk(uint64_t c_first, uint64_t c_last, const Bgzf::BulkInflate& fn)
    {
        if (!bg_.prefetch_bulk(c_first, c_last, fn)) { if (bg_.bad()) fail(bg_.error()); return false; }
        return true;
    }
    // compressed file offset where the 16 kb window of `pos` starts (BAI linear index; monotone within a contig).
    // Differences of it estimate how much BAM a range of loci spans -- used to balance loci over GPUs before any decode.
    uint64_t linear_offset(int tid, int64_t pos) const
    {
        if (tid < 0 || size_t(tid) >= refs_.size() || refs_[size_t(tid)].linear.empty()) return 0;
        const std::vector<uint64_t>& lin = refs_[size_t(tid)].linear;
        size_t w = pos < 0 ? 0 : size_t(pos >> 14);
        if (w >= lin.size()) w = lin.size() - 1;
        while (w > 0 && lin[w] == 0) --w;           // empty windows carry 0: walk back to the last filled one
        return lin[w] >> 16;
    }

private:
    bool fail(const std::string& what)
    {
        if (err_.empty()) err_ = path_ + ": " + what;
        done_ = true; hint_valid_ = false;
        return false;
    }
    std::string err_;
    bool load_index(std::string* err)
    {
        std::string p = path_ + ".bai";
        FILE* f = fopen(p.c_str(), "rb");
        if (!f) {
            std::string q = path_;
            if (q.size() > 4 && q.substr(q.size() - 4) == ".bam") { q = q.substr(0, q.size() - 4) + ".bai"; f = fopen(q.c_str(), "rb"); }
        }
        if (!f) { *err = "BAM index does not exist. Expecting " + path_ + ".bai (CSI indices are not supported by this reader)"; return false; }
        std::vector<uint8_t> buf;
        fseek(f, 0, SEEK_END); const long sz = ftell(f); fseek(f, 0, SEEK_SET);
        buf.resize(size_t(sz));
        if (sz > 0 && fread(buf.data(), 1, size_t(sz), f) != size_t(sz)) { fclose(f); *err = "cannot read BAM index"; return false; }
        fclose(f);
        if (buf.size() < 8 || memcmp(buf.data(), "BAI\1", 4) != 0) { *err = "bad BAI magic"; return false; }
        size_t o = 4;
        const uint32_t n_ref = rd32(buf.data() + o); o += 4;
        refs_.resize(n_ref);
        for (uint32_t r = 0; r < n_ref; ++r) {
            if (o + 4 > buf.size()) { *err = "truncated BAI"; return false; }
            const uint32_t n_bin = rd32(buf.data() + o); o += 4;
            std::vector<std::pair<uint32_t, std::vector<BaiChunk>>> bins;
            for (uint32_t b = 0; b < n_bin; ++b) {
                if (o + 8 > buf.size()) { *err = "truncated BAI"; return false; }
                const uint32_t bin = rd32(buf.data() + o); const uint32_t n_chunk = rd32(buf.data() + o + 4); o += 8;
                if (o + size_t(n_chunk) * 16 > buf.size()) { *err = "truncated BAI"; return false; }
                std::vector<BaiChunk> cs(n_chunk);
                for (uint32_t c = 0; c < n_chunk; ++c) { cs[c].beg = rd64(buf.data() + o); cs[c].end = rd64(buf.data() + o + 8); o += 16; }
                if (bin != 37450) bins.emplace_back(bin, std::move(cs));      // 37450 = metadata pseudo-bin
            }
            std::sort(bins.begin(), bins.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
            for (auto& b : bins) { refs_[r].bin_ids.push_back(b.first); refs_[r].bin_chunks.push_back(std::move(b.second)); }
            if (o + 4 > buf.size()) { *err = "truncated BAI"; return false; }
            const uint32_t n_intv = rd32(buf.data() + o); o += 4;
            if (o + size_t(n_intv) * 8 > buf.size()) { *err = "truncated BAI"; return false; }
            refs_[r].linear.resize(n_intv);
            for (uint32_t i = 0; i < n_intv; ++i) { refs_[r].linear[i] = rd64(buf.data() + o); o += 8; }
        }
        return true;
    }
    std::string path_;
    Bgzf bg_;
    std::vector<BaiRef> refs_;
    std::vector<BaiChunk> chunks_;
    size_t cur_ = 0;
    bool positioned_ = false, done_ = true;
    int tid_ = -1;
    int64_t beg_ = 0, end_ = 0;
    uint64_t start_off_ = 0;          // lower bound of this region's scan (linear index or resume point)
    bool hint_valid_ = false, hint_set_ = false;
    int hint_tid_ = -1;
    int64_t hint_beg_ = 0;
    uint64_t hint_voff_ = 0;
};

}  // namespace vtxhost
