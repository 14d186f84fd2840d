// stager.hpp -- the host half of evaluate_rec / evaluate_alns (vartrix src/main.rs:610-695,
// 809-894): per VCF record build the haplotype windows, fetch the overlapping BAM records, apply the
// four record filters and stage the survivors as one `vtx_batch` shard.  Alignment, barcode lookup, UMI
// gate and aggregation happen on the GPU behind include/vartrix_b200.h.
#pragma once
#include <algorithm>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/vartrix_b200.h"
#include "../vtx_record.cuh"
#include "bam_reader.hpp"
#include "inputs.hpp"

namespace vtxhost {

struct HostMetrics {             // the host-side share of main.rs:449-459
    uint64_t num_reads = 0, num_low_mapq = 0, num_non_primary = 0, num_duplicates = 0, num_not_useful = 0,
             num_invalid_recs = 0, num_multiallelic_recs = 0,
             num_low_base_quality = 0;      // --min-base-quality: not a counter of the reference
    void add(const HostMetrics& o)
    {
        num_reads += o.num_reads; num_low_mapq += o.num_low_mapq; num_non_primary += o.num_non_primary;
        num_duplicates += o.num_duplicates; num_not_useful += o.num_not_useful; num_invalid_recs += o.num_invalid_recs;
        num_multiallelic_recs += o.num_multiallelic_recs; num_low_base_quality += o.num_low_base_quality;
    }
    void add(const uint32_t (&c)[vtx::stage::kNumCounters])       // one locus's record counters
    {
        using namespace vtx::stage;
        num_reads += c[kFetched]; num_low_mapq += c[kLowMapq]; num_non_primary += c[kNonPrimary];
        num_duplicates += c[kDuplicate]; num_not_useful += c[kNotUseful]; num_low_base_quality += c[kLowBaseQuality];
    }
};

struct StageArgs : vtx::stage::RecordFilters {     // --mapq, --primary-alignments, --no-duplicates, --min-base-quality
    int64_t padding = 100;       // --padding
    char bam_tag[2] = { 'C', 'B' };
    bool valid[256] = {};        // --valid-chars
    bool with_umi = true;        // stage the UB keys (--umi, or a dump for the tests); without --umi nobody reads them
    bool name_keys = false;      // --collapse-mates: the staged key is the QNAME (per-shard interner), not the UB tag
    bool locus_filters = false;  // --out-variant-stats: keep the record-filter counters per locus (StagedShard::locus_filters)
    // --gpu-inflate: the BGZF members of a shard's loci are inflated in one device call (vtx_bgzf_inflate) instead of one
    // by one on the staging thread; empty = host inflate
    Bgzf::BulkInflate bulk_inflate;
};

// the tag bytes of a vtx::stage::pack_cb code
inline std::string unpack_cb(uint64_t key)
{
    const uint32_t n = uint32_t(key >> 7) & 31u, suffix = uint32_t(key & 127u);
    std::string s(n, 'A');
    uint64_t k = key >> 12;
    for (uint32_t i = n; i-- > 0;) { s[i] = "ACGT"[k & 3]; k >>= 2; }
    if (suffix) { s += '-'; s += std::to_string(suffix); }
    return s;
}

// One shard in the slim staging layout (vtx_batch2): reads back to back on 4-byte boundaries, u16 lengths, cell tags as
// codes (+ the few that have none as bytes), UMI keys only when asked for, candidate list only when a read serves two loci.
struct StagedShard {
    std::vector<uint32_t> locus_row, ref_off, ref_len, alt_off, alt_len, cand_read, cb_off;
    std::vector<uint64_t> cand_start, read_cb_key, read_umi_key;
    std::vector<uint16_t> read_len;
    std::vector<uint8_t> hap_bytes, read_nib, cb_bytes;
    bool identity = true;        // candidate c is read c so far (no read shared between loci)
    bool with_umi = true;        // read_umi_key is filled
    HostMetrics met;
    // per staged locus: the vtx::stage::kNumCounters record counters (--out-variant-stats; the device counts the rest of
    // vtx_locus_stats)
    std::vector<uint32_t> locus_filters;

    void clear()          // keeps the capacity: shards are recycled so steady-state staging does not page-fault
    {
        locus_row.clear(); ref_off.clear(); ref_len.clear(); alt_off.clear(); alt_len.clear(); read_len.clear(); read_cb_key.clear();
        cand_read.clear(); cand_start.clear(); cb_off.clear(); read_umi_key.clear(); hap_bytes.clear();
        read_nib.clear(); cb_bytes.clear(); met = HostMetrics(); identity = true; locus_filters.clear();
    }
    size_t bytes() const
    {
        return (locus_row.size() * 5 + cand_read.size() + cb_off.size()) * 4 + (cand_start.size() + read_cb_key.size() + read_umi_key.size()) * 8 +
               read_len.size() * 2 + hap_bytes.size() + read_nib.size() + cb_bytes.size() + 16 * 16;
    }
    void fill(vtx_batch2* b) const
    {
        memset(b, 0, sizeof(*b));
        b->n_loci = uint32_t(locus_row.size()); b->locus_row = locus_row.data();
        b->hap_bytes = hap_bytes.data(); b->hap_bytes_len = hap_bytes.size();
        b->ref_off = ref_off.data(); b->ref_len = ref_len.data(); b->alt_off = alt_off.data(); b->alt_len = alt_len.data();
        b->cand_start = cand_start.data();
        b->n_reads = uint32_t(read_len.size()); b->read_nib = read_nib.data(); b->read_nib_len = read_nib.size();
        b->read_off4 = nullptr; b->read_len = read_len.data(); b->read_cb_key = read_cb_key.data();
        b->n_exotic_cb = cb_off.empty() ? 0 : uint32_t(cb_off.size() - 1); b->cb_bytes = cb_bytes.data(); b->cb_off = cb_off.data();
        b->read_umi_key = with_umi ? read_umi_key.data() : nullptr;
        b->n_cand = cand_read.size(); b->cand_read = identity ? nullptr : cand_read.data();
    }
};

// UB strings that do not fit vtx_pack_umi's alphabet/length get a process-wide interned id
class UmiInterner {
public:
    uint64_t key(const uint8_t* s, uint32_t len)
    {
        const uint64_t k = vtx::stage::pack_umi(s, len);
        if (k != VTX_NO_UMI) return k;
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.emplace(std::string(reinterpret_cast<const char*>(s), len), map_.size()).first;
        return (1ull << 61) | it->second;
    }
private:
    std::mutex mu_;
    std::unordered_map<std::string, uint64_t> map_;
};

// --collapse-mates: QNAME -> key, first-seen order, for one shard at a time.  Keys only meet inside one locus, so a table per
// shard (owned by the staging thread) is enough; a name of "*" (SAM: no name) gets a fresh key every time.
class NameInterner {
public:
    void clear() { map_.clear(); next_ = 0; }
    uint64_t key(const uint8_t* s, uint32_t len)
    {
        if (len == 1 && s[0] == '*') return next_++;
        auto it = map_.emplace(std::string(reinterpret_cast<const char*>(s), len), next_);
        if (it.second) ++next_;
        return it.first->second;
    }
private:
    std::unordered_map<std::string, uint64_t> map_;
    uint64_t next_ = 0;
};

inline void pad16(std::vector<uint8_t>& v) { while (v.size() & 15) v.push_back(0); }

// record virtual offset -> staged read id of the current shard: open addressing, linear probing, grows at 50 % load.
// (One lookup per candidate; a node-based std::unordered_map spends more time allocating than hashing here.)
class ReadIndex {
public:
    ReadIndex() { keys_.assign(1 << 12, kEmpty); vals_.resize(1 << 12); }
    void clear() { std::fill(keys_.begin(), keys_.end(), kEmpty); n_ = 0; }
    // id of `voff`; `fresh` tells whether it was inserted now (with id = next_id)
    uint32_t find_or_insert(uint64_t voff, uint32_t next_id, bool* fresh)
    {
        if ((n_ + 1) * 2 > keys_.size()) grow();
        size_t i = slot(voff);
        while (keys_[i] != kEmpty) {
            if (keys_[i] == voff) { *fresh = false; return vals_[i]; }
            i = (i + 1) & (keys_.size() - 1);
        }
        keys_[i] = voff; vals_[i] = next_id; ++n_;
        *fresh = true;
        return next_id;
    }
private:
    static constexpr uint64_t kEmpty = ~0ull;          // no BAM record lives at virtual offset 2^64 - 1
    size_t slot(uint64_t k) const { return size_t((k * 0x9E3779B97F4A7C15ull) >> 20) & (keys_.size() - 1); }
    void grow()
    {
        std::vector<uint64_t> ok; std::vector<uint32_t> ov;
        ok.swap(keys_); ov.swap(vals_);
        keys_.assign(ok.size() * 2, kEmpty); vals_.resize(ok.size() * 2);
        for (size_t j = 0; j < ok.size(); ++j)
            if (ok[j] != kEmpty) {
                size_t i = slot(ok[j]);
                while (keys_[i] != kEmpty) i = (i + 1) & (keys_.size() - 1);
                keys_[i] = ok[j]; vals_[i] = ov[j];
            }
    }
    std::vector<uint64_t> keys_;
    std::vector<uint32_t> vals_;
    size_t n_ = 0;
};

enum class Window { kScored, kMultiallelic, kInvalidAlt, kFastaError };

// VCF record `row` at the locus [start, end) -> its haplotype windows (construct_haplotypes, main.rs:619-684, 958-994).  One
// read of the reference window; its two flanks are the alt haplotype's flanks (same FASTA bytes).  A scored record appends its
// row and both windows to the shard (StagedShard or DeviceShard); a multi-allelic or invalid-ALT one is counted in its metrics.
template <class Shard>
inline Window stage_windows(const VcfRecord& v, uint32_t row, int64_t start, int64_t end, const Fasta& fa, const StageArgs& a,
                            Shard* out, std::string* err)
{
    if (v.alleles.size() > 2) { out->met.num_multiallelic_recs++; return Window::kMultiallelic; }        // main.rs:646-653
    const int64_t L = fa.length(v.chrom);
    if (L < 0) { *err = "Requested chromosome " + v.chrom + " was not found in fasta"; return Window::kFastaError; }
    static thread_local std::string ref_hap, alt_hap;
    const int64_t w0 = std::max<int64_t>(start - a.padding, 0), w1 = std::min(end + a.padding, L);
    if (end > L || !fa.fetch_upper(v.chrom, w0, w1, &ref_hap)) {
        *err = "FASTA fetch failed at " + v.chrom + ":" + std::to_string(v.pos0);
        return Window::kFastaError;
    }
    alt_hap.assign(ref_hap, 0, size_t(start - w0));                    // FASTA[max(start - pad, 0), start)
    if (v.alleles.size() == 2) alt_hap += v.alleles[1];                 // main.rs:656-659: no ALT allele is an empty one
    alt_hap.append(ref_hap, size_t(end - w0), std::string::npos);       // FASTA[end, min(end + pad, L))
    for (unsigned char c : alt_hap)
        if (!a.valid[c]) { out->met.num_invalid_recs++; return Window::kInvalidAlt; }                  // main.rs:675-684
    out->locus_row.push_back(row);
    pad16(out->hap_bytes); out->ref_off.push_back(uint32_t(out->hap_bytes.size())); out->ref_len.push_back(uint32_t(ref_hap.size()));
    out->hap_bytes.insert(out->hap_bytes.end(), ref_hap.begin(), ref_hap.end());
    pad16(out->hap_bytes); out->alt_off.push_back(uint32_t(out->hap_bytes.size())); out->alt_len.push_back(uint32_t(alt_hap.size()));
    out->hap_bytes.insert(out->hap_bytes.end(), alt_hap.begin(), alt_hap.end());
    return Window::kScored;
}

// What the host keeps doing when the device stages the reads itself (vtx_submit_bam): windows from the FASTA, the compressed
// byte range of the loci's index chunks, the BGZF member table, the record boundaries the index knows.
struct DeviceShard {
    std::vector<uint32_t> locus_row, ref_off, ref_len, alt_off, alt_len;
    std::vector<int64_t> locus_start, locus_end;
    std::vector<uint8_t> hap_bytes, comp;
    std::vector<vtx_bgzf_block> members;
    std::vector<uint64_t> entry_off;
    int32_t tid = -1;
    HostMetrics met;             // only the per-record counters the host still owns: multi-allelic / invalid records
    void fill(vtx_bam_shard* b, const StageArgs& a) const
    {
        memset(b, 0, sizeof(*b));
        b->n_loci = uint32_t(locus_row.size()); b->locus_row = locus_row.data(); b->locus_start = locus_start.data(); b->locus_end = locus_end.data();
        b->hap_bytes = hap_bytes.data(); b->hap_bytes_len = hap_bytes.size();
        b->ref_off = ref_off.data(); b->ref_len = ref_len.data(); b->alt_off = alt_off.data(); b->alt_len = alt_len.data();
        b->tid = tid; b->n_members = uint32_t(members.size()); b->members = members.data(); b->comp = comp.data(); b->comp_len = comp.empty() ? 0 : comp.size() - 16;
        b->n_entry = uint32_t(entry_off.size()); b->entry_off = entry_off.data();
        b->mapq = a.mapq_min; b->primary_only = a.primary_only; b->no_duplicates = a.no_duplicates; b->bam_tag[0] = a.bam_tag[0]; b->bam_tag[1] = a.bam_tag[1];
    }
};

// Records [lo, hi) of the VCF -> the host's share of a device-staged shard.  `*supported` = false (and nothing else done) when
// the loci are not ascending on one contig: such shards are staged on the host.
inline bool stage_loci_device(const std::vector<VcfRecord>& recs, size_t lo, size_t hi, const Fasta& fa, BamFile& bam,
                              const StageArgs& a, DeviceShard* out, bool* supported, std::string* err)
{
    *supported = true;
    for (size_t i = lo + 1; i < hi; ++i)
        if (recs[i].chrom != recs[lo].chrom || recs[i].pos0 < recs[i - 1].pos0) { *supported = false; return true; }
    *out = DeviceShard();
    if (hi <= lo) return true;
    out->tid = bam.tid_of(recs[lo].chrom);
    std::vector<BaiChunk> chunks;
    for (size_t i = lo; i < hi; ++i) {
        const VcfRecord& v = recs[i];
        const int64_t start = v.pos0, end = v.pos0 + int64_t(v.alleles[0].size());      // main.rs:619-623
        const Window w = stage_windows(v, uint32_t(i), start, end, fa, a, out, err);
        if (w == Window::kFastaError) return false;
        if (w != Window::kScored) continue;
        out->locus_start.push_back(start); out->locus_end.push_back(end);
        bam.region_chunks(out->tid, start, end, &chunks);
    }
    pad16(out->hap_bytes);
    if (chunks.empty()) return true;                                  // no locus has any indexed read: nothing to inflate
    uint64_t v_first = ~0ull, v_last = 0;
    for (const BaiChunk& c : chunks) { v_first = std::min(v_first, c.beg); v_last = std::max(v_last, c.end); }
    std::vector<Bgzf::MemberRef> index;
    if (!bam.read_members(v_first >> 16, v_last >> 16, &out->members, &out->comp, &index)) { *err = bam.error(); return false; }
    // virtual offset -> offset in the inflated stream
    auto stream_of = [&](uint64_t voff, uint64_t* so) -> bool {
        const uint64_t coff = voff >> 16, uoff = voff & 0xFFFF;
        auto it = std::lower_bound(index.begin(), index.end(), coff, [](const Bgzf::MemberRef& m, uint64_t c) { return m.coff < c; });
        if (it == index.end() || it->coff != coff) return false;
        *so = it->stream_off + uoff;
        return *so <= index.back().stream_off;
    };
    std::vector<uint64_t>& e = out->entry_off;
    // more places to start walking from: the first record of every 16 kb window (linear index) -- one walker per entry point
    std::vector<uint64_t> lin;
    bam.linear_entries(out->tid, out->locus_start.front(), *std::max_element(out->locus_end.begin(), out->locus_end.end()), v_first, v_last, &lin);
    for (uint64_t v : lin) chunks.push_back({ v, v });
    for (const BaiChunk& c : chunks) {
        uint64_t so;
        if (!stream_of(c.beg, &so)) { *err = "BAM index points outside a BGZF member (index and file do not match)"; return false; }
        e.push_back(so);
    }
    uint64_t s_end;
    if (!stream_of(v_last, &s_end)) { *err = "BAM index points outside a BGZF member (index and file do not match)"; return false; }
    e.push_back(s_end);
    std::sort(e.begin(), e.end());
    e.erase(std::unique(e.begin(), e.end()), e.end());
    while (!e.empty() && e.back() > s_end) e.pop_back();
    if (e.size() < 2) e.clear();
    return true;
}

// Records [lo, hi) of the VCF -> one shard.  Mirrors evaluate_rec + the head of evaluate_alns.
inline bool stage_loci(const std::vector<VcfRecord>& recs, size_t lo, size_t hi, const Fasta& fa, BamFile& bam,
                       const StageArgs& a, UmiInterner& umis, StagedShard* out, std::string* err)
{
    out->with_umi = a.with_umi;
    out->cb_off.push_back(0);
    if (a.bulk_inflate && hi > lo) {
        // one compressed range for the whole shard when its loci sit on one contig (the usual case: sorted VCF)
        uint64_t c0 = ~0ull, c1 = 0;
        bool one_contig = true;
        for (size_t i = lo; i < hi && one_contig; ++i) one_contig = recs[i].chrom == recs[lo].chrom;
        if (one_contig) {
            const int tid = bam.tid_of(recs[lo].chrom);
            for (size_t i = lo; i < hi; ++i) {
                uint64_t f = 0, l = 0;
                const int64_t start = recs[i].pos0, end = recs[i].pos0 + int64_t(recs[i].alleles[0].size());
                if (bam.region_span(tid, start, end, &f, &l)) { c0 = std::min(c0, f); c1 = std::max(c1, l); }
            }
            if (c0 != ~0ull && c1 - c0 < (uint64_t(1) << 30)) {
                if (!bam.prefetch_bulk(c0, c1, a.bulk_inflate)) { *err = bam.error().empty() ? "device BGZF inflate failed" : bam.error(); return false; }
            }
        }
    }
    static thread_local ReadIndex read_index;               // record virtual offset -> staged read id (table reused across shards)
    read_index.clear();
    static thread_local NameInterner names;                 // --collapse-mates: this shard's QNAME keys
    names.clear();
    BamRecord rec;
    out->cand_start.push_back(0);
    for (size_t i = lo; i < hi; ++i) {
        const VcfRecord& v = recs[i];
        const int64_t start = v.pos0, end = v.pos0 + int64_t(v.alleles[0].size());      // main.rs:619-623
        const Window w = stage_windows(v, uint32_t(i), start, end, fa, a, out, err);
        if (w == Window::kFastaError) return false;
        if (w != Window::kScored) continue;

        uint32_t c[vtx::stage::kNumCounters] = {};
        const int tid = bam.tid_of(v.chrom);
        if (tid >= 0 && bam.fetch(tid, start, end)) {                                    // main.rs:822-826
            while (bam.next(&rec)) {
                ++c[vtx::stage::kFetched];                                               // 831
                if (const int drop = vtx::stage::drop_reason(rec.flag(), rec.mapq(), rec.p, start, end, a)) { ++c[drop]; continue; }
                bool fresh = false;
                const uint32_t rid = read_index.find_or_insert(rec.voff, uint32_t(out->read_len.size()), &fresh);
                if (fresh) {
                    const int32_t ls = rec.l_seq() < 0 ? 0 : rec.l_seq();
                    if (ls > 0xFFFF) { *err = "read longer than 65535 bases at " + v.chrom + ":" + std::to_string(rec.pos()); return false; }
                    while (out->read_nib.size() & 3) out->read_nib.push_back(0);                              // every read starts on a 4-byte boundary
                    out->read_len.push_back(uint16_t(ls));
                    out->read_nib.insert(out->read_nib.end(), rec.seq(), rec.seq() + (ls + 1) / 2);
                    uint32_t n = 0;
                    const uint8_t* cb = rec.aux_z(a.bam_tag, &n);                                             // main.rs:737-750
                    uint64_t key = VTX_NO_CB_KEY;
                    if (cb && n <= 0xFFFF) {
                        key = vtx::stage::pack_cb(cb, n);
                        if (key == VTX_NO_CB_KEY) {        // a tag the code cannot express travels as bytes
                            key = VTX_CB_EXOTIC | uint64_t(out->cb_off.size() - 1);
                            out->cb_bytes.insert(out->cb_bytes.end(), cb, cb + n);
                            out->cb_off.push_back(uint32_t(out->cb_bytes.size()));
                        }
                    }
                    out->read_cb_key.push_back(key);
                    if (a.name_keys) {
                        n = rec.l_read_name() ? rec.l_read_name() - 1 : 0;                                    // without the NUL
                        out->read_umi_key.push_back(names.key(rec.p + 32, n));
                    } else if (a.with_umi) {
                        const uint8_t* ub = rec.aux_z("UB", &n);                                              // main.rs:752-757
                        out->read_umi_key.push_back(ub ? umis.key(ub, n) : VTX_NO_UMI);
                    }
                }
                if (rid != out->cand_read.size()) out->identity = false;
                out->cand_read.push_back(rid);
            }
            if (bam.bad()) { *err = bam.error(); return false; }            // corrupt / truncated BAM: abort (main.rs:830)
        }
        out->cand_start.push_back(out->cand_read.size());
        out->met.add(c);
        if (a.locus_filters) out->locus_filters.insert(out->locus_filters.end(), c, c + vtx::stage::kNumCounters);
    }
    while (out->read_nib.size() & 3) out->read_nib.push_back(0);
    pad16(out->hap_bytes);
    return true;
}

}  // namespace vtxhost
