// inputs.hpp -- FASTA(.fai) windows, VCF records, barcode list, Matrix-Market / label writers for the
// staging host.  Each piece cites the reference lines (vartrix src/main.rs) it stands in for.
#pragma once
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <charconv>
#include <condition_variable>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fcntl.h>
#include <mutex>
#include <string>
#include <thread>
#include <unistd.h>
#include <unordered_map>
#include <vector>

namespace vtxhost {

// ---- whole-file line reader.  Barcodes: gunzip chosen by the ".gz" extension only (open_with_gz, main.rs:721-735).
// VCF (`sniff_gz`): htslib looks at the content, so a gzip/bgzip magic decides whatever the file is called. ----
inline bool read_text_file(const std::string& path, std::string* out, std::string* err, bool sniff_gz = false)
{
    out->clear();
    bool gz = path.size() >= 3 && path.compare(path.size() - 3, 3, ".gz") == 0;
    if (sniff_gz) {
        FILE* f = fopen(path.c_str(), "rb");
        if (!f) { *err = "cannot open " + path; return false; }
        unsigned char m[2] = { 0, 0 };
        const size_t k = fread(m, 1, 2, f);
        fclose(f);
        gz = k == 2 && m[0] == 0x1f && m[1] == 0x8b;
    }
    if (gz) {
        gzFile f = gzopen(path.c_str(), "rb");
        if (!f) { *err = "cannot open " + path; return false; }
        char buf[1 << 16]; int n;
        while ((n = gzread(f, buf, sizeof(buf))) > 0) out->append(buf, size_t(n));
        gzclose(f);
        if (n < 0) { *err = "error reading " + path; return false; }
    } else {
        FILE* f = fopen(path.c_str(), "rb");
        if (!f) { *err = "cannot open " + path; return false; }
        char buf[1 << 16]; size_t n;
        while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
        fclose(f);
    }
    return true;
}

// BufRead::lines(): split on '\n', strip one trailing '\r'; a final empty piece is not a line
inline std::vector<std::string> split_lines(const std::string& s)
{
    std::vector<std::string> v;
    size_t p = 0;
    while (p < s.size()) {
        size_t q = s.find('\n', p);
        if (q == std::string::npos) q = s.size();
        size_t e = q;
        if (e > p && s[e - 1] == '\r') --e;
        v.emplace_back(s, p, e - p);
        p = q + 1;
    }
    return v;
}

// ---- load_barcodes (main.rs:697-718): first-seen order, duplicates keep the first index ----
struct BarcodeList {
    std::vector<std::string> keys;
    std::vector<uint8_t> bytes;
    std::vector<uint32_t> off;
};
inline bool load_barcodes(const std::string& path, BarcodeList* out, std::string* err)
{
    std::string text;
    if (!read_text_file(path, &text, err)) { *err = "error open barcodes file: " + path; return false; }
    std::unordered_map<std::string, uint32_t> seen;
    for (auto& ln : split_lines(text))
        if (seen.emplace(ln, uint32_t(out->keys.size())).second) out->keys.push_back(ln);
    if (out->keys.empty()) { *err = "Loaded 0 barcodes. Is your barcode file gzipped or empty?"; return false; }   // main.rs:712-715
    out->off.push_back(0);
    for (auto& k : out->keys) { out->bytes.insert(out->bytes.end(), k.begin(), k.end()); out->off.push_back(uint32_t(out->bytes.size())); }
    return true;
}

// ---- VCF text records (rust-htslib bcf::Reader over a text VCF, main.rs:221-234, 615-623, 646-659) ----
struct VcfRecord {
    std::string chrom;
    int64_t pos0 = 0;                     // rec.pos(): 0-based
    std::vector<std::string> alleles;     // REF then ALTs; ALT "." -> only REF (main.rs:654-659)
};
inline bool read_vcf(const std::string& path, std::vector<VcfRecord>* out, std::string* err)
{
    std::string text;
    if (!read_text_file(path, &text, err, /*sniff_gz=*/true)) return false;
    if (text.size() >= 3 && memcmp(text.data(), "BCF", 3) == 0) { *err = "binary BCF input is not supported; convert to VCF"; return false; }
    for (auto& ln : split_lines(text)) {
        if (ln.empty() || ln[0] == '#') continue;
        std::vector<std::string> f;
        size_t p = 0;
        while (f.size() < 5) {
            size_t q = ln.find('\t', p);
            if (q == std::string::npos) { f.emplace_back(ln, p); p = ln.size(); break; }
            f.emplace_back(ln, p, q - p); p = q + 1;
        }
        if (f.size() < 5) { *err = "malformed VCF line: " + ln.substr(0, 60); return false; }
        VcfRecord r;
        r.chrom = f[0];
        r.pos0 = std::strtoll(f[1].c_str(), nullptr, 10) - 1;
        r.alleles.push_back(f[3]);
        if (f[4] != ".") {
            size_t a = 0;
            while (true) {
                size_t b = f[4].find(',', a);
                if (b == std::string::npos) { r.alleles.emplace_back(f[4], a); break; }
                r.alleles.emplace_back(f[4], a, b - a); a = b + 1;
            }
        }
        out->push_back(std::move(r));
    }
    return true;
}

// ---- indexed FASTA (bio::io::fasta::IndexedReader over .fai, main.rs:556-572, 936-954) ----
class Fasta {
public:
    ~Fasta() { if (fd_ >= 0) ::close(fd_); }
    bool open(const std::string& path, std::string* err)
    {
        std::string text;
        if (!read_text_file(path + ".fai", &text, err)) { *err = "File " + path + ".fai does not exist"; return false; }   // main.rs:514-518
        for (auto& ln : split_lines(text)) {
            if (ln.empty()) continue;
            Entry e; char name[4096];
            unsigned long long len, off, lb, lw;
            if (sscanf(ln.c_str(), "%4095[^\t]\t%llu\t%llu\t%llu\t%llu", name, &len, &off, &lb, &lw) != 5) { *err = "malformed .fai line"; return false; }
            e.len = len; e.offset = off; e.line_bases = lb; e.line_width = lw;
            index_.emplace(name, entries_.size()); names_.push_back(name); entries_.push_back(e);
        }
        fd_ = ::open(path.c_str(), O_RDONLY);
        if (fd_ < 0) { *err = "error opening fasta file"; return false; }
        return true;
    }
    bool has(const std::string& chrom) const { return index_.count(chrom) != 0; }
    int64_t length(const std::string& chrom) const { auto it = index_.find(chrom); return it == index_.end() ? -1 : int64_t(entries_[it->second].len); }
    // bases [start, end) upper-cased (read_locus, main.rs:944-953); clamps are the caller's business
    bool fetch_upper(const std::string& chrom, int64_t start, int64_t end, std::string* out) const
    {
        out->clear();
        auto it = index_.find(chrom);
        if (it == index_.end()) return false;
        const Entry& e = entries_[it->second];
        if (start < 0) start = 0;
        if (end > int64_t(e.len)) end = int64_t(e.len);
        if (end <= start) return true;
        const uint64_t first = e.offset + uint64_t(start) / e.line_bases * e.line_width + uint64_t(start) % e.line_bases;
        const uint64_t last = e.offset + uint64_t(end - 1) / e.line_bases * e.line_width + uint64_t(end - 1) % e.line_bases + 1;
        std::vector<char> buf(size_t(last - first));
        if (pread(fd_, buf.data(), buf.size(), off_t(first)) != ssize_t(buf.size())) return false;
        out->reserve(size_t(end - start));
        for (char c : buf) {
            if (c == '\n' || c == '\r') continue;
            out->push_back((c >= 'a' && c <= 'z') ? char(c - 32) : c);
        }
        return int64_t(out->size()) == end - start;
    }
private:
    struct Entry { uint64_t len, offset, line_bases, line_width; };
    int fd_ = -1;
    std::vector<Entry> entries_;
    std::vector<std::string> names_;
    std::unordered_map<std::string, size_t> index_;
};

// ---- Rust `{}` for f64: shortest round-trip digits, never an exponent, NaN / inf spelled out ----
inline std::string fmt_f64(double v)
{
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
    char buf[400];
    auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::fixed);
    return std::string(buf, r.ptr);
}

// ---- sprs 0.7.1 write_matrix_market layout (main.rs:381-389; SURVEY.md A.9) ----
// one "row col value\n" line; integral values (consensus / coverage, and 0 or 1 of alt_frac) skip the float formatter
inline char* mtx_line(char* p, uint32_t row, uint32_t col, double v)
{
    p = std::to_chars(p, p + 12, uint64_t(row) + 1).ptr; *p++ = ' ';
    p = std::to_chars(p, p + 12, uint64_t(col) + 1).ptr; *p++ = ' ';
    if (v >= 0.0 && v < 9.0e15 && v == double(uint64_t(v))) p = std::to_chars(p, p + 20, uint64_t(v)).ptr;
    else if (std::isnan(v)) { memcpy(p, "NaN", 3); p += 3; }
    else if (std::isinf(v)) { const char* t = v > 0 ? "inf" : "-inf"; const size_t k = strlen(t); memcpy(p, t, k); p += k; }
    else p = std::to_chars(p, p + 380, v, std::chars_format::fixed).ptr;
    *p++ = '\n';
    return p;
}

// The text of a large matrix is formatted by `threads` workers in blocks of 64 k triplets and written in order
// (a serial formatter takes many times the GPU time of the job).
inline bool write_mtx(const std::string& path, uint64_t n_rows, uint64_t n_cols, uint64_t n, const uint32_t* row,
                      const uint32_t* col, const double* val, std::string* err, unsigned threads = 0)
{
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) { *err = "Error writing " + path; return false; }
    std::string head = "%%MatrixMarket matrix coordinate real general\n% written by sprs\n";
    head += std::to_string(n_rows) + " " + std::to_string(n_cols) + " " + std::to_string(n) + "\n";
    bool ok = fwrite(head.data(), 1, head.size(), f) == head.size();
    constexpr uint64_t kBlock = 1u << 16;
    constexpr size_t kLineMax = 12 + 1 + 12 + 1 + 380 + 1;
    const uint64_t n_blocks = (n + kBlock - 1) / kBlock;
    if (threads == 0) threads = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    threads = unsigned(std::min<uint64_t>(threads, std::max<uint64_t>(n_blocks, 1)));
    auto format_block = [&](uint64_t b, std::vector<char>& buf) -> size_t {
        const uint64_t k0 = b * kBlock, k1 = std::min(n, k0 + kBlock);
        // integral values need at most 12 + 12 + 20 + 3 bytes per line; a block with fractions gets the roomy buffer
        bool frac = false;
        for (uint64_t k = k0; k < k1 && !frac; ++k) frac = !(val[k] >= 0.0 && val[k] < 9.0e15 && val[k] == double(uint64_t(val[k])));
        const size_t need = size_t(k1 - k0) * (frac ? kLineMax : 48);
        if (buf.size() < need) buf.resize(need);
        char* p = buf.data();
        for (uint64_t k = k0; k < k1; ++k) p = mtx_line(p, row[k], col[k], val[k]);
        return size_t(p - buf.data());
    };
    if (threads <= 1) {
        std::vector<char> buf;
        for (uint64_t b = 0; b < n_blocks && ok; ++b) { const size_t len = format_block(b, buf); ok = fwrite(buf.data(), 1, len, f) == len; }
    } else {
        // ring of 2 x threads block buffers: workers claim blocks in order, the writer drains them in order
        const uint64_t ring = uint64_t(threads) * 2;
        std::vector<std::vector<char>> bufs(ring);
        std::vector<size_t> lens(ring, 0);
        std::vector<uint64_t> ready(ring, ~0ull);          // block number held by the slot
        std::mutex mu; std::condition_variable cv;
        std::atomic<uint64_t> next{ 0 };
        uint64_t written = 0;                               // guarded by mu
        auto worker = [&]() {
            for (;;) {
                const uint64_t b = next.fetch_add(1);
                if (b >= n_blocks) return;
                { std::unique_lock<std::mutex> g(mu); cv.wait(g, [&] { return b < written + ring; }); }
                const size_t len = format_block(b, bufs[b % ring]);
                { std::lock_guard<std::mutex> g(mu); lens[b % ring] = len; ready[b % ring] = b; }
                cv.notify_all();
            }
        };
        std::vector<std::thread> pool;
        for (unsigned t = 0; t < threads; ++t) pool.emplace_back(worker);
        for (uint64_t b = 0; b < n_blocks; ++b) {
            { std::unique_lock<std::mutex> g(mu); cv.wait(g, [&] { return ready[b % ring] == b; }); }
            if (ok) ok = fwrite(bufs[b % ring].data(), 1, lens[b % ring], f) == lens[b % ring];
            { std::lock_guard<std::mutex> g(mu); written = b + 1; }
            cv.notify_all();
        }
        for (auto& t : pool) t.join();
    }
    ok = (fclose(f) == 0) && ok;
    if (!ok) *err = "Error writing " + path;
    return ok;
}

}  // namespace vtxhost
