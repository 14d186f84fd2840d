// vtx_stage.cuh -- the host half of evaluate_alns on the device: BAM records of a shard of loci, straight from the inflated
// BGZF stream (vtx_inflate.cuh), turned into the engine's candidate lists.
//
// Replaces, for a host that only reads the compressed file, what csrc/host/stager.hpp + bam_reader.hpp do on staging
// threads and the reference does through rust-htslib (vartrix src/main.rs:822-865, 737-757, 790-806):
//   fetch          every record of the contig with pos < end and bam_endpos > start, in file order   (main.rs:822-829)
//   record filters mapq, --primary-alignments, --no-duplicates, useful_alignment, in that order      (main.rs:833-865)
//                  then, with --min-base-quality, the judged bases' qualities (vtx_base_quality.cuh)
//   tags           CB (or --bam-tag) and UB: first aux field of that name, type Z                      (main.rs:737-757)
//                  or, with --collapse-mates, the QNAME as the molecule key instead of UB (name_key below)
// The record stream is walked from the BAI chunk starts that fall into the shard's range (record boundaries by
// construction of the index), one thread per segment; everything after that is one thread per record or per locus.
// Nothing is copied: reads and tag bytes are referenced inside the inflated stream.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "vtx_base_quality.cuh"

namespace vtx {
namespace stage {

constexpr uint32_t kNoCb = 0xFFFFFFFFu;
constexpr uint64_t kNoUmi = 0xFFFFFFFFFFFFFFFFull;

struct Params {
    const uint8_t* s;            // inflated stream: the members' outputs back to back
    uint64_t s_len;
    int32_t tid;                 // contig of every locus of the shard
    uint32_t mapq_min;
    int32_t primary_only, no_duplicates, want_umi;
    uint8_t tag0, tag1;          // --bam-tag
    uint32_t min_base_quality;   // --min-base-quality (0: off)
};

// error bits (first word of `err`): the shard is then re-staged on the host, which produces the message
enum : uint32_t { kErrWalk = 1, kErrRecord = 2, kErrExoticUmi = 4, kErrLongRead = 8 };

__host__ __device__ inline uint32_t ld32(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); }
__host__ __device__ inline uint32_t ld16(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8); }

// The per-item bodies below are __host__ __device__: the kernels at the end of the file are one-line wrappers, and
// tests/stage_dev_shim.cpp runs the same bodies serially on the CPU against the host stager (tests/test_host_staging_cpu.py).
__host__ __device__ inline void flag_or(uint32_t* p, uint32_t v)
{
#ifdef __CUDA_ARCH__
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
__host__ __device__ inline void take_max(uint32_t* p, uint32_t v)
{
#ifdef __CUDA_ARCH__
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
__host__ __device__ inline void add_u64(unsigned long long* p, unsigned long long v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

// ---- 1. record boundaries: one walker per segment [seg_off[k], seg_off[k + 1]) of the stream ----------------------------
// pass 0 counts the records of the segment, pass 1 writes their offsets at rec_first[k]..
// `Fetch` hands out the 24 header bytes of the record at p: straight from memory (CPU tests), or from a shared-memory window
// that a warp refills together (the kernel: the walk is a chain of dependent loads, ~30 cycles from shared memory instead
// of an L2 round trip per record).  Every lane of the warp runs the same walk; `writer()` is true on one of them.
struct DirectFetch {
    const uint8_t* s;
    __host__ __device__ void ensure(uint64_t) {}
    __host__ __device__ const uint8_t* at(uint64_t p) const { return s + p; }
    __host__ __device__ bool writer() const { return true; }
};

template <class Fetch>
__host__ __device__ inline void walk_segment(const Params& P, uint32_t k, const uint64_t* seg_off, int pass, uint32_t* seg_count,
                                             const uint32_t* rec_first, uint64_t* rec_off, uint32_t* err, Fetch& F)
{
    uint64_t p = seg_off[k];
    const uint64_t end = seg_off[k + 1];
    uint32_t n = 0;
    const uint32_t base = pass ? rec_first[k] : 0;
    while (p < end) {
        if (p + 36 > P.s_len) { if (F.writer()) flag_or(err, kErrWalk); break; }
        F.ensure(p);
        const uint8_t* h = F.at(p);                          // block_size, then the fixed fields of the record
        const uint32_t bs = ld32(h);
        const uint8_t* b = h + 4;
        const int64_t l_seq = int32_t(ld32(b + 16));
        const uint64_t need = 32ull + b[8] + 4ull * ld16(b + 12) + (l_seq < 0 ? 0 : uint64_t(l_seq + 1) / 2 + uint64_t(l_seq));
        if (bs < 32 || bs > (1u << 28) || l_seq < 0 || need > bs || p + 4 + bs > P.s_len) { if (F.writer()) flag_or(err, kErrRecord); break; }
        if (pass && F.writer()) rec_off[base + n] = p;
        ++n;
        p += 4 + uint64_t(bs);
    }
    if (p > end && F.writer()) flag_or(err, kErrWalk);    // the walk must land exactly on the next entry point
    if (!pass && F.writer()) seg_count[k] = n;
}

// ---- 2. one thread per record: position, end position (htslib bam_endpos), flag | mapq, longest reference span ---------
__host__ __device__ inline void parse_record(const Params& P, uint32_t i, const uint64_t* rec_off, int32_t* rec_tid, int32_t* rec_pos,
                                             int32_t* rec_end, uint32_t* rec_fm, uint32_t* max_span /* longest reference span of a record */)
{
    const uint8_t* b = P.s + rec_off[i] + 4;
    const int32_t pos = int32_t(ld32(b + 4));
    const uint32_t flag = ld16(b + 14), nc = ld16(b + 12);
    int64_t rlen = 0;
    if (!(flag & 4)) {
        const uint8_t* c = b + 32 + b[8];
        for (uint32_t q = 0; q < nc; ++q) {
            const uint32_t v = ld32(c + 4 * q), op = v & 0xF;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += v >> 4;
        }
    }
    const int64_t e = int64_t(pos) + (rlen > 0 ? rlen : 1);
    const int32_t tid = int32_t(ld32(b));
    rec_tid[i] = tid;
    // a range of the shard's contig holds only its records; should the index ever hand out a tail of the next contig (or of
    // unplaced reads), those sort last and keep the position array monotone for the per-locus binary searches
    rec_pos[i] = tid == P.tid ? pos : 0x7fffffff;
    rec_end[i] = int32_t(e > 0x7fffffff ? 0x7fffffff : e);
    rec_fm[i] = (flag << 8) | b[9];
    if (tid == P.tid) take_max(max_span, uint32_t(e - pos > 0xFFFFFFFFll ? 0xFFFFFFFFu : uint32_t(e - pos)));
}

// rust-htslib 0.36 CigarStringView::read_pos(p, include_softclips = false, include_dels = true) folded into
// useful_alignment (main.rs:790-806): is there a p in start..=end with an aligned base or a deletion?
__host__ __device__ inline bool useful_alignment(const uint8_t* b, int64_t start, int64_t end)
{
    const uint8_t* cg = b + 32 + b[8];
    const uint32_t nc = ld16(b + 12);
    const int64_t pos0 = int32_t(ld32(b + 4));
    uint32_t i0 = 0;
    while (i0 < nc) {            // leading section: first of M,=,X,I,S starts the walk; leading D/N or an interior H is an error
        const uint32_t op = ld32(cg + 4 * i0) & 0xF;
        if (op == 0 || op == 7 || op == 8 || op == 1 || op == 4) break;
        if (op == 2 || op == 3) return false;
        if (op == 5 && i0 != 0 && i0 != nc - 1) return false;
        ++i0;
    }
    if (i0 >= nc) return false;
    for (int64_t p = start; p <= end; ++p) {          // inclusive end, main.rs:794
        int64_t rpos = pos0;
        for (uint32_t i = i0; i < nc && rpos <= p; ++i) {
            const uint32_t v = ld32(cg + 4 * i), op = v & 0xF; const int64_t len = int64_t(v >> 4);
            if (op == 0 || op == 7 || op == 8 || op == 2) { if (p >= rpos && p < rpos + len) return true; rpos += len; }
            else if (op == 3) rpos += len;
            else if (op == 5) { if (i != nc - 1) return false; break; }
        }
    }
    return false;
}

// the first five counters are vtx_bam_metrics' layout; num_low_base_quality has its own getter (vtx_bam_low_base_quality)
struct LocusMetrics { unsigned long long num_reads, num_low_mapq, num_non_primary, num_duplicates, num_not_useful, num_low_base_quality; };

// ---- 3. one thread per locus: the records it fetches, the four filters (and the base-quality floor); pass 0 counts, pass 1 lists
__host__ __device__ inline void locus_cands(const Params& P, uint32_t l, const int64_t* l_start, const int64_t* l_end, uint32_t n_rec,
                                            const uint64_t* rec_off, const int32_t* rec_tid, const int32_t* rec_pos, const int32_t* rec_end,
                                            const uint32_t* rec_fm, const uint32_t* max_span, uint32_t* max_read, int pass, uint32_t* cand_count,
                                            const uint32_t* cand_first, uint32_t* cand_rec, uint32_t* used, LocusMetrics* met,
                                            uint32_t* lfilt = nullptr /* pass 0, vtx_set_locus_stats: [l][6] the counters below */)
{
    const int64_t start = l_start[l], end = l_end[l];
    // records are coordinate-sorted: candidates lie in [first pos > start - max_span, first pos >= end)
    const int64_t lo_pos = start - int64_t(*max_span);
    uint32_t lo = 0, hi = n_rec;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (int64_t(rec_pos[mid]) <= lo_pos) lo = mid + 1; else hi = mid; }
    const uint32_t first = lo;
    hi = n_rec;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (int64_t(rec_pos[mid]) < end) lo = mid + 1; else hi = mid; }
    const uint32_t last = lo;
    uint32_t n = 0, longest = 0;
    unsigned long long fetched = 0, low = 0, nonprim = 0, dup = 0, notuse = 0, lowbq = 0;
    const uint32_t base = pass ? cand_first[l] : 0;
    for (uint32_t i = first; i < last; ++i) {
        if (rec_tid[i] != P.tid || int64_t(rec_end[i]) <= start) continue;
        ++fetched;                                                                        // main.rs:831
        const uint32_t fm = rec_fm[i], fl = fm >> 8;
        if ((fm & 0xFF) < P.mapq_min) { ++low; continue; }                                // 833
        if (P.primary_only && (fl & 0x900)) { ++nonprim; continue; }                      // 841
        if (P.no_duplicates && (fl & 0x400)) { ++dup; continue; }                         // 849
        if (!useful_alignment(P.s + rec_off[i] + 4, start, end)) { ++notuse; continue; }  // 857
        if (P.min_base_quality && !base_quality_ok(P.s + rec_off[i] + 4, start, end, P.min_base_quality)) { ++lowbq; continue; }
        if (pass) { cand_rec[base + n] = i; used[i] = 1u; }
        else { const uint32_t ls = ld32(P.s + rec_off[i] + 4 + 16); if (ls > longest) longest = ls; }                       // l_seq of a read that will be scored
        ++n;
    }
    if (!pass) {
        cand_count[l] = n;
        if (longest) take_max(max_read, longest);
        if (fetched) add_u64(&met->num_reads, fetched);
        if (low) add_u64(&met->num_low_mapq, low);
        if (nonprim) add_u64(&met->num_non_primary, nonprim);
        if (dup) add_u64(&met->num_duplicates, dup);
        if (notuse) add_u64(&met->num_not_useful, notuse);
        if (lowbq) add_u64(&met->num_low_base_quality, lowbq);
        if (lfilt) {                     // the per-locus split of the same counters (vtx_locus_stats.cuh)
            uint32_t* f = lfilt + size_t(l) * 6;
            f[0] = uint32_t(fetched); f[1] = uint32_t(low); f[2] = uint32_t(nonprim); f[3] = uint32_t(dup); f[4] = uint32_t(notuse); f[5] = uint32_t(lowbq);
        }
    }
}

// first aux field named (t0, t1): its value bytes when the type is Z (Record::aux -> Aux::String), else nothing
__host__ __device__ inline bool aux_z(const uint8_t* p, const uint8_t* e, uint8_t t0, uint8_t t1, uint32_t* off_from_p, uint32_t* len)
{
    const uint8_t* base = p;
    while (p + 3 <= e) {
        const bool hit = p[0] == t0 && p[1] == t1;
        const uint8_t ty = p[2];
        p += 3;
        if (ty == 'Z' || ty == 'H') {
            const uint8_t* q = p;
            while (q < e && *q) ++q;
            if (q >= e) return false;
            if (hit) { if (ty == 'Z') { *off_from_p = uint32_t(p - base); *len = uint32_t(q - p); return true; } return false; }
            p = q + 1;
        } else {
            size_t sz;
            switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'B': {
                if (p + 5 > e) return false;
                const uint8_t sub = p[0]; const uint32_t cnt = ld32(p + 1);
                const size_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                sz = 5 + size_t(cnt) * es; break;
            }
            default: return false;
            }
            if (hit) return false;
            p += sz;
        }
    }
    return false;
}

// vtx_pack_umi on the device: strings over {A,C,G,T,N} up to 18 bases; anything else cannot be keyed here
__host__ __device__ inline uint64_t pack_umi(const uint8_t* s, uint32_t len)
{
    if (len > 18) return kNoUmi;
    uint64_t k = 0;
    for (uint32_t i = 0; i < len; ++i) {
        uint64_t c;
        switch (s[i]) { case 'A': c = 0; break; case 'C': c = 1; break; case 'G': c = 2; break; case 'T': c = 3; break; case 'N': c = 4; break; default: return kNoUmi; }
        k = (k << 3) | c;
    }
    return (k << 5) | len;
}

// ---- 4. one thread per record: the read arrays of the engine -----------------------------------------------------------------
// read id = record index (nothing is copied or compacted: bases and tag bytes stay where they are in the stream); records
// that are no locus's candidate get an empty entry
__host__ __device__ inline void read_emit(const Params& P, uint32_t i, const uint64_t* rec_off, const uint32_t* used, uint64_t* read_off,
                                          uint32_t* read_len, uint32_t* read_cb_off, uint16_t* read_cb_len, uint64_t* read_umi, uint32_t* err)
{
    const uint32_t r = i;
    if (!used[i]) { read_off[r] = 0; read_len[r] = 0; read_cb_off[r] = kNoCb; read_cb_len[r] = 0; if (P.want_umi) read_umi[r] = kNoUmi; return; }
    const uint64_t ro = rec_off[i];
    const uint8_t* b = P.s + ro + 4;
    const uint32_t bs = ld32(P.s + ro);
    const int32_t l_seq = int32_t(ld32(b + 16));
    const uint64_t seq_off = ro + 4 + 32 + b[8] + 4ull * ld16(b + 12);
    if (l_seq > 16000) flag_or(err, kErrLongRead);
    read_off[r] = seq_off;
    read_len[r] = uint32_t(l_seq);
    const uint8_t* aux = P.s + seq_off + uint64_t(l_seq + 1) / 2 + uint64_t(l_seq);
    const uint8_t* e = b + bs;
    uint32_t off = 0, len = 0;
    if (aux_z(aux, e, P.tag0, P.tag1, &off, &len) && len <= 0xFFFF && uint64_t(aux - P.s) + off < 0xFFFFFFFFull) {      // main.rs:737-750
        read_cb_off[r] = uint32_t(uint64_t(aux - P.s) + off); read_cb_len[r] = uint16_t(len);
    } else { read_cb_off[r] = kNoCb; read_cb_len[r] = 0; }
    if (P.want_umi) {
        uint64_t key = kNoUmi;
        if (aux_z(aux, e, 'U', 'B', &off, &len)) {                                                                        // main.rs:752-757
            key = pack_umi(aux + off, len);
            if (key == kNoUmi) flag_or(err, kErrExoticUmi);          // needs the host's interner: the shard goes back to the host path
        }
        read_umi[r] = key;
    }
}

// ---- 5. --collapse-mates (VTX_F_NAME_KEYS): one thread per record, the read's molecule key is its QNAME --------------------
// Open addressing over record indices: `tab` has a power-of-two size >= 2 * n_rec and starts out all kEmptySlot.  A record walks
// its probe chain and either claims the first empty slot (key = its own index) or meets an occupant with the same name bytes
// (key = the occupant's index).  Slots only ever go from empty to occupied, so all records of one name walk the same chain up
// to the first of them to claim a slot, and meet it there.  A QNAME of "*" (no name) is never inserted and keeps its own index,
// which no occupant can hold: the keys stay injective.  Keys are compared only inside one locus, so the values do not matter.
constexpr uint32_t kEmptySlot = 0xFFFFFFFFu;

__host__ __device__ inline uint32_t claim_slot(uint32_t* p, uint32_t v)      // -> the slot's value before the call
{
#ifdef __CUDA_ARCH__
    return atomicCAS(p, kEmptySlot, v);
#else
    const uint32_t old = *p;
    if (old == kEmptySlot) *p = v;
    return old;
#endif
}

struct NameHash {                // FNV-1a over the name bytes, folded to 32 bits
    __host__ __device__ uint32_t operator()(const uint8_t* s, uint32_t n) const
    {
        uint64_t h = 0xcbf29ce484222325ull;
        for (uint32_t i = 0; i < n; ++i) { h ^= s[i]; h *= 0x100000001b3ull; }
        return uint32_t(h ^ (h >> 32));
    }
};

__host__ __device__ inline const uint8_t* qname_of(const uint8_t* s, const uint64_t* rec_off, uint32_t i, uint32_t* len)
{
    const uint8_t* b = s + rec_off[i] + 4;
    *len = b[8] ? uint32_t(b[8]) - 1u : 0u;          // l_read_name counts the trailing NUL
    return b + 32;
}

template <class Hash>
__host__ __device__ inline void name_key(const Params& P, uint32_t i, const uint64_t* rec_off, const uint32_t* used, uint32_t* tab,
                                         uint32_t tab_mask, uint64_t* read_umi, const Hash& hash)
{
    if (!used[i]) { read_umi[i] = kNoUmi; return; }
    uint32_t n = 0;
    const uint8_t* name = qname_of(P.s, rec_off, i, &n);
    if (n == 1 && name[0] == '*') { read_umi[i] = i; return; }
    for (uint32_t h = hash(name, n) & tab_mask;; h = (h + 1) & tab_mask) {
        const uint32_t occ = claim_slot(&tab[h], i);
        if (occ == kEmptySlot) { read_umi[i] = i; return; }
        uint32_t m = 0;
        const uint8_t* other = qname_of(P.s, rec_off, occ, &m);
        bool same = m == n;
        for (uint32_t k = 0; same && k < n; ++k) same = other[k] == name[k];
        if (same) { read_umi[i] = occ; return; }
    }
}

#ifdef __CUDACC__
constexpr int kWalkWarps = 4, kWalkWindow = 4096;          // bytes of the stream a warp keeps in shared memory
struct WindowFetch {
    const uint8_t* s;            // 16-byte aligned, readable up to the next multiple of 16 behind s_len (the engine pads its buffers)
    uint8_t* win;
    uint64_t base;
    int lane;
    __device__ void ensure(uint64_t p)
    {
        if (p >= base && p + 24 <= base + kWalkWindow) return;            // warp-uniform: every lane walks the same p
        base = p & ~uint64_t(15);
        __syncwarp();
        for (int i = lane; i < kWalkWindow / 16; i += 32)
            reinterpret_cast<uint4*>(win)[i] = __ldcg(reinterpret_cast<const uint4*>(s + base) + i);
        __syncwarp();
    }
    __device__ const uint8_t* at(uint64_t p) const { return win + (p - base); }
    __device__ bool writer() const { return lane == 0; }
};
// one warp per segment
__global__ void __launch_bounds__(kWalkWarps * 32) vtx_k_walk(Params P, uint32_t n_seg, const uint64_t* __restrict__ seg_off, int pass,
                                                              uint32_t* __restrict__ seg_count, const uint32_t* __restrict__ rec_first,
                                                              uint64_t* __restrict__ rec_off, uint32_t* __restrict__ err)
{
    __shared__ __align__(16) uint8_t windows[kWalkWarps][kWalkWindow];
    const uint32_t k = blockIdx.x * kWalkWarps + (threadIdx.x >> 5);
    if (k >= n_seg) return;
    WindowFetch F{ P.s, windows[threadIdx.x >> 5], ~uint64_t(0) - kWalkWindow, int(threadIdx.x & 31) };
    walk_segment(P, k, seg_off, pass, seg_count, rec_first, rec_off, err, F);
}
__global__ void vtx_k_parse(Params P, uint32_t n_rec, const uint64_t* __restrict__ rec_off, int32_t* __restrict__ rec_tid,
                            int32_t* __restrict__ rec_pos, int32_t* __restrict__ rec_end, uint32_t* __restrict__ rec_fm,
                            uint32_t* __restrict__ max_span)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rec) parse_record(P, i, rec_off, rec_tid, rec_pos, rec_end, rec_fm, max_span);
}
__global__ void vtx_k_locus_cands(Params P, uint32_t n_loci, const int64_t* __restrict__ l_start, const int64_t* __restrict__ l_end,
                                  uint32_t n_rec, const uint64_t* __restrict__ rec_off, const int32_t* __restrict__ rec_tid,
                                  const int32_t* __restrict__ rec_pos, const int32_t* __restrict__ rec_end, const uint32_t* __restrict__ rec_fm,
                                  const uint32_t* __restrict__ max_span, uint32_t* __restrict__ max_read, int pass, uint32_t* __restrict__ cand_count,
                                  const uint32_t* __restrict__ cand_first, uint32_t* __restrict__ cand_rec, uint32_t* __restrict__ used,
                                  LocusMetrics* __restrict__ met, uint32_t* __restrict__ lfilt)
{
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l < n_loci) locus_cands(P, l, l_start, l_end, n_rec, rec_off, rec_tid, rec_pos, rec_end, rec_fm, max_span, max_read, pass, cand_count,
                                cand_first, cand_rec, used, met, lfilt);
}
__global__ void vtx_k_read_emit(Params P, uint32_t n_rec, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ used,
                                uint64_t* __restrict__ read_off, uint32_t* __restrict__ read_len,
                                uint32_t* __restrict__ read_cb_off, uint16_t* __restrict__ read_cb_len, uint64_t* __restrict__ read_umi,
                                uint32_t* __restrict__ err)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rec) read_emit(P, i, rec_off, used, read_off, read_len, read_cb_off, read_cb_len, read_umi, err);
}

__global__ void vtx_k_name_key(Params P, uint32_t n_rec, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ used,
                               uint32_t* __restrict__ tab, uint32_t tab_mask, uint64_t* __restrict__ read_umi)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rec) name_key(P, i, rec_off, used, tab, tab_mask, read_umi, NameHash{});
}

// cand_start (u64, what the pipeline expects) from the u32 exclusive scan of the per-locus counts
__global__ void vtx_k_widen(uint32_t n, const uint32_t* __restrict__ in, uint64_t* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}
#endif   // __CUDACC__

}  // namespace stage
}  // namespace vtx
