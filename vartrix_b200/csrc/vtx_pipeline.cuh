// vtx_pipeline.cuh -- the integer/byte kernels either side of Smith-Waterman (sm_90a).
// HBM-bound scatter/gather work: one thread per element, coalesced 4/8-byte accesses, no host
// synchronisation between stages (every size that depends on data stays on the device).
//
//   vtx_k_cb_lookup     get_cell_barcode + HashMap<Vec<u8>,u32>     main.rs:737-750, 697-718
//   vtx_k_cand_filter   CB miss / --umi gate + metric counters      main.rs:867-894
//   vtx_k_compact       Scores{cell_index, umi, ..} push order      main.rs:923-930
//   vtx_k_locus_prep    tile classes (haplotype width / alphabet)   (scheduler, replaces main.rs:250-254)
//   vtx_k_slots         sort_by_key(cell_index) + group_by          main.rs:932, 1044, 1047-1057
//   vtx_k_umi_collapse  per-UMI 0.75 consensus                      main.rs:1058-1082
//   vtx_k_finalize      consensus_scoring / alt_frac / coverage     main.rs:1111-1164
//   vtx_k_emit          TriMat::add_triplet in row-major order      main.rs:320-348
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "vtx_sw.cuh"
#include "vtx_sw_split.cuh"
#include "vtx_sw_fold.cuh"
#include "vtx_record.cuh"

namespace vtx {

constexpr uint32_t kNoCb = 0xFFFFFFFFu;
constexpr uint64_t kNoUmi = 0xFFFFFFFFFFFFFFFFull;
constexpr uint32_t kInvalid = 0xFFFFFFFFu;

__host__ __device__ inline uint64_t fnv1a64(const uint8_t* p, uint32_t n)
{
    uint64_t h = 1469598103934665603ull;
    for (uint32_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

struct BarcodeTable {
    const int32_t* slot;      // [cap] barcode index or -1
    uint32_t cap_mask;        // cap - 1 (cap is a power of two >= 2 n)
    const uint8_t* bytes;
    const uint32_t* off;      // [n + 1]
};

// exact byte-string lookup of a CB tag in the barcode list: column id or -1
__device__ __forceinline__ int32_t cb_lookup_bytes(const BarcodeTable& t, const uint8_t* __restrict__ key, uint32_t len)
{
    uint32_t h = uint32_t(fnv1a64(key, len)) & t.cap_mask;
    for (;;) {
        const int32_t s = t.slot[h];
        if (s < 0) return -1;
        const uint32_t o = t.off[s], l2 = t.off[s + 1] - o;
        if (l2 == len) {
            bool eq = true;
            for (uint32_t i = 0; i < len; ++i) eq &= (t.bytes[o + i] == key[i]);
            if (eq) return s;
        }
        h = (h + 1) & t.cap_mask;
    }
}

// one thread per read: exact byte-string lookup of the CB tag in the barcode list
__global__ void vtx_k_cb_lookup(BarcodeTable t, uint32_t n_reads, const uint8_t* __restrict__ cb_bytes,
                                const uint32_t* __restrict__ read_cb_off, const uint16_t* __restrict__ read_cb_len,
                                int32_t* __restrict__ read_col)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const uint32_t off = read_cb_off[r];
    read_col[r] = off != kNoCb ? cb_lookup_bytes(t, cb_bytes + off, read_cb_len[r]) : -1;
}

// ---- slim layout (vtx_batch2): cell tags travel as one injective u64 code per read -------------------------------
using stage::kNoCbKey;                          // what stage::pack_cb returns for a tag it cannot code
constexpr uint64_t kCbExotic = 0x8000000000000000ull;

__host__ __device__ inline uint64_t mix64(uint64_t x)
{
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31;
    return x;
}

struct BarcodeKeyTable {      // the barcodes that have a code: open addressing on the code itself
    const uint64_t* key;      // [cap] code or kNoCbKey (empty)
    const uint32_t* idx;      // [cap] column id
    uint32_t cap_mask;
};

// one thread per read: one or two 8-byte probes instead of a byte-wise string compare
__global__ void vtx_k_cb_lookup_key(BarcodeTable t, BarcodeKeyTable kt, uint32_t n_reads, const uint64_t* __restrict__ read_cb_key,
                                    const uint8_t* __restrict__ cb_bytes, const uint32_t* __restrict__ cb_off,
                                    int32_t* __restrict__ read_col)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const uint64_t key = read_cb_key[r];
    int32_t col = -1;
    if (key == kNoCbKey) {
    } else if (key & kCbExotic) {
        const uint32_t i = uint32_t(key & 0xFFFFFFFFu);
        col = cb_lookup_bytes(t, cb_bytes + cb_off[i], cb_off[i + 1] - cb_off[i]);
    } else {
        uint32_t h = uint32_t(mix64(key)) & kt.cap_mask;
        for (;;) {
            const uint64_t k = kt.key[h];
            if (k == key) { col = int32_t(kt.idx[h]); break; }
            if (k == kNoCbKey) break;
            h = (h + 1) & kt.cap_mask;
        }
    }
    read_col[r] = col;
}

// slim layout -> the engine's internal read arrays.  Dense pools: 4-byte units per read first, offsets after a scan.
__global__ void vtx_k_read_units(uint32_t n_reads, const uint16_t* __restrict__ read_len, uint32_t* __restrict__ units)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_reads) units[r] = ((uint32_t(read_len[r]) + 1) / 2 + 3) / 4;
}
__global__ void vtx_k_expand_reads(uint32_t n_reads, const uint16_t* __restrict__ read_len, const uint32_t* __restrict__ off4,
                                   uint64_t* __restrict__ read_off, uint32_t* __restrict__ read_len32)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    read_off[r] = uint64_t(off4[r]) * 4;
    read_len32[r] = read_len[r];
}

// one thread per candidate: keep flag (for the compaction scan) + metric counters, warp-aggregated
__global__ void vtx_k_cand_filter(uint64_t n_cand, const uint32_t* __restrict__ cand_read,
                                  const int32_t* __restrict__ read_col, const uint64_t* __restrict__ read_umi_key,
                                  int use_umi, uint32_t* __restrict__ keep, unsigned long long* __restrict__ metrics)
{
    const uint64_t c = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    bool miss_cb = false, miss_umi = false, ok = false;
    if (c < n_cand) {
        const uint32_t r = cand_read ? cand_read[c] : uint32_t(c);           // NULL: candidate c is read c
        if (read_col[r] < 0) miss_cb = true;                                 // main.rs:868-876
        else if (use_umi && read_umi_key[r] == kNoUmi) miss_umi = true;      // main.rs:880-888
        else ok = true;
        keep[c] = ok ? 1u : 0u;
    }
    // metric counters: warp ballots -> shared memory -> one atomic per counter per block (three hot addresses
    // would otherwise serialise ~half a million warp-level atomics in L2)
    __shared__ uint32_t s_cnt[3];
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t b0 = __ballot_sync(0xffffffffu, miss_cb), b1 = __ballot_sync(0xffffffffu, miss_umi),
                   b2 = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) {
        if (b0) atomicAdd(&s_cnt[0], uint32_t(__popc(b0)));
        if (b1) atomicAdd(&s_cnt[1], uint32_t(__popc(b1)));
        if (b2) atomicAdd(&s_cnt[2], uint32_t(__popc(b2)));
    }
    __syncthreads();
    if (threadIdx.x < 3 && s_cnt[threadIdx.x]) atomicAdd(metrics + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

// largest l with cand_start[l] <= c
__device__ __forceinline__ uint32_t locus_of_cand(const uint64_t* __restrict__ cand_start, uint32_t n_loci, uint64_t c)
{
    uint32_t lo = 0, hi = n_loci;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cand_start[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

// kept candidates -> dense pair arrays (order preserved: locus-major, file order)
__global__ void vtx_k_compact(uint64_t n_cand, const uint32_t* __restrict__ cand_read,
                              const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pidx,
                              const int32_t* __restrict__ read_col, const uint64_t* __restrict__ read_umi_key,
                              int use_umi, uint32_t* __restrict__ pair_read, uint32_t* __restrict__ pair_col,
                              uint64_t* __restrict__ pair_umi)
{
    const uint64_t c = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (c >= n_cand || !keep[c]) return;
    const uint32_t p = pidx[c], r = cand_read ? cand_read[c] : uint32_t(c);
    pair_read[p] = r;
    pair_col[p] = uint32_t(read_col[r]);
    if (use_umi) pair_umi[p] = read_umi_key[r];
}

__global__ void vtx_k_pair_start(uint32_t n_loci, const uint64_t* __restrict__ cand_start,
                                 const uint32_t* __restrict__ pidx, uint32_t* __restrict__ pair_start)
{
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l <= n_loci) pair_start[l] = pidx[cand_start[l]];
}

// pairs given explicitly (vtx_score_pairs): pair_start from a locus-sorted pair_locus array
__global__ void vtx_k_pair_start_explicit(uint32_t n_loci, uint32_t n_pairs, const uint32_t* __restrict__ pair_locus,
                                          uint32_t* __restrict__ pair_start)
{
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l > n_loci) return;
    uint32_t lo = 0, hi = n_pairs;                 // first p with pair_locus[p] >= l
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (pair_locus[mid] < l) lo = mid + 1; else hi = mid; }
    pair_start[l] = lo;
}

// one warp per locus: tile class from haplotype width and alphabet, tiles per class
__global__ void vtx_k_locus_prep(uint32_t n_loci, const uint8_t* __restrict__ hap_bytes,
                                 const uint32_t* __restrict__ ref_off, const uint32_t* __restrict__ ref_len,
                                 const uint32_t* __restrict__ alt_off, const uint32_t* __restrict__ alt_len,
                                 const uint32_t* __restrict__ pair_start, const uint32_t* __restrict__ pair_read,
                                 const uint32_t* __restrict__ read_len, int force_slow, int allow_split, int allow_multi, int allow_fold,
                                 uint32_t max_read, uint32_t max_hap, unsigned long long* __restrict__ bounds_violated,
                                 uint32_t* __restrict__ tcount /* [kNumClasses][n_loci + 1] */)
{
    const uint32_t l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (l >= n_loci) return;
    const uint32_t nr = ref_len[l], na = alt_len[l];
    const uint8_t* rh = hap_bytes + ref_off[l];
    const uint8_t* ah = hap_bytes + alt_off[l];
    bool exotic = false;
    // bytes that a decoded read base other than A/C/G/T could equal: "=MRSVWYHKDBN"
    auto is_exotic = [](uint8_t b) {
        return b == '=' || b == 'M' || b == 'R' || b == 'S' || b == 'V' || b == 'W' || b == 'Y' || b == 'H' ||
               b == 'K' || b == 'D' || b == 'B' || b == 'N';
    };
    for (uint32_t j = lane; j < nr; j += 32) exotic |= is_exotic(rh[j]);
    for (uint32_t j = lane; j < na; j += 32) exotic |= is_exotic(ah[j]);
    exotic = __any_sync(0xffffffffu, exotic);
    // is the first kSplitP-column prefix common to both haplotypes?  (construct_haplotypes: same left flank)
    bool same = nr >= uint32_t(kSplitP) && na >= uint32_t(kSplitP);
    if (same) for (uint32_t j = lane; j < uint32_t(kSplitP); j += 32) same &= (rh[j] == ah[j]);
    same = __all_sync(0xffffffffu, same);
    // ... and the last kFoldP columns (same right flank)?  Then neither flank needs a per-haplotype DP (vtx_sw_fold.cuh).
    bool fold = same && allow_fold && min(nr, na) > uint32_t(2 * kFoldP) && max(nr, na) <= uint32_t(2 * kFoldP + kFoldMaxMid);
    if (fold) for (uint32_t j = lane; j < uint32_t(kFoldP); j += 32) fold &= (rh[nr - 1 - j] == ah[na - 1 - j]);
    fold = __all_sync(0xffffffffu, fold);
    uint32_t longest = 0;
    for (uint32_t p = pair_start[l] + lane; p < pair_start[l + 1]; p += 32) longest = max(longest, read_len[pair_read[p]]);
    longest = __reduce_max_sync(0xffffffffu, longest);
    // the folded kernel keeps 8 x 19 read rows in registers: every read of the locus must fit
    fold = fold && longest <= uint32_t(kFoldMaxRead);
    if (lane != 0) return;
    const uint32_t nmax = max(nr, na);
    // Buffers and kernel shapes were sized from max_read / max_hap (exact for host batches, the caller's promise for
    // device batches).  A locus that breaks the promise gets no tiles -- nothing is read or written out of bounds --
    // and the next vtx_finish reports the violation.
    if (longest > max_read || nmax > max_hap) {
        atomicAdd(bounds_violated, 1ull);
#pragma unroll
        for (int c = 0; c < kNumClasses; ++c) tcount[size_t(c) * (n_loci + 1) + l] = 0u;
        return;
    }
    int cls = kSlowClass;
    if (!exotic && !force_slow) {
#pragma unroll
        for (int c = kNumFastClasses - 1; c >= 0; --c) if (nmax <= uint32_t(class_max_n(c))) cls = c;
        if (cls == kSlowClass && allow_multi) cls = kMultiClass;        // wider than 320 columns: several passes
        if (same && allow_split) {
#pragma unroll
            for (int c = kNumSplitClasses - 1; c >= 0; --c) if (nmax <= uint32_t(split_max_n(c))) cls = kSplitClass0 + c;
        }
        if (fold) cls = kFoldClass;
    }
    const uint32_t np = pair_start[l + 1] - pair_start[l];
#pragma unroll
    for (int c = 0; c < kNumClasses; ++c) {
        const uint32_t ppw = (c == kSlowClass) ? uint32_t(kSlowPairsPerWarp) : (c == kFoldClass ? uint32_t(kFoldPPW) : (c > kSlowClass ? uint32_t(kSplitPPW) : 4u));
        tcount[size_t(c) * (n_loci + 1) + l] = (c == cls) ? (np + ppw - 1) / ppw : 0u;
    }
}

// One CTA per locus: rank every pair's cell (and, with --umi, its (cell, UMI)) among the distinct keys
// of the locus.  slot = pair_start[locus] + rank, so slots of a locus are col-ascending and the final
// triplets come out row-major sorted without a global sort.  O(d^2) compares per locus of depth d
// (d ~ 50 here); keys staged through shared memory in chunks.
constexpr int kSlotThreads = 128;
constexpr int kSlotChunk = 1024;
constexpr uint32_t kSlotSmallMax = 2048;      // deeper loci are enlisted for vtx_k_slots_big
constexpr int kSlotBigThreads = 1024;
constexpr int kSlotBigWords = 7;              // scratch words per pair for vtx_k_slots_big
__global__ void __launch_bounds__(kSlotThreads) vtx_k_slots(
    uint32_t n_loci, const uint32_t* __restrict__ pair_start, const uint32_t* __restrict__ pair_col,
    const uint64_t* __restrict__ pair_umi, int use_umi, uint8_t* __restrict__ pair_first,
    uint32_t* __restrict__ pair_cslot, uint32_t* __restrict__ pair_uslot, uint32_t* __restrict__ cslot_col,
    uint32_t* __restrict__ cslot_locus, uint32_t* __restrict__ uslot_cslot, uint32_t* __restrict__ big_list /* [0] = count */)
{
    __shared__ uint32_t s_col[kSlotChunk];
    __shared__ uint64_t s_umi[kSlotChunk];
    __shared__ uint8_t s_first[kSlotChunk];
    for (uint32_t l = blockIdx.x; l < n_loci; l += gridDim.x) {
        const uint32_t ps = pair_start[l], d = pair_start[l + 1] - ps;
        if (d == 0) continue;
        if (d > kSlotSmallMax) {                  // O(d^2) would be too slow: hand over to the hash + sort kernel
            if (threadIdx.x == 0) big_list[1 + atomicAdd(big_list, 1u)] = l;
            continue;
        }
        // pass 1: is this pair the first occurrence of its cell / of its (cell, umi)?
        for (uint32_t base = 0; base < d; base += kSlotThreads) {
            const uint32_t p = base + threadIdx.x;
            uint32_t colp = 0; uint64_t umip = 0; bool fc = true, fu = true;
            if (p < d) { colp = pair_col[ps + p]; if (use_umi) umip = pair_umi[ps + p]; }
            const uint32_t q_end = min(d, base + kSlotThreads);     // only q < p matter
            for (uint32_t q0 = 0; q0 < q_end; q0 += kSlotChunk) {
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < kSlotChunk && q0 + i < q_end; i += kSlotThreads) {
                    s_col[i] = pair_col[ps + q0 + i];
                    if (use_umi) s_umi[i] = pair_umi[ps + q0 + i];
                }
                __syncthreads();
                if (p < d) {
                    const uint32_t lim = min(uint32_t(kSlotChunk), min(q_end, p) > q0 ? min(q_end, p) - q0 : 0u);
                    for (uint32_t i = 0; i < lim; ++i) {
                        if (s_col[i] == colp) { fc = false; if (!use_umi || s_umi[i] == umip) fu = false; }
                    }
                }
            }
            if (p < d) pair_first[ps + p] = uint8_t((fc ? 1 : 0) | (fu ? 2 : 0));
        }
        __syncthreads();
        // pass 2: rank = number of distinct smaller keys
        for (uint32_t base = 0; base < d; base += kSlotThreads) {
            const uint32_t p = base + threadIdx.x;
            uint32_t colp = 0; uint64_t umip = 0; uint32_t cs = 0, us = 0;
            if (p < d) { colp = pair_col[ps + p]; if (use_umi) umip = pair_umi[ps + p]; }
            for (uint32_t q0 = 0; q0 < d; q0 += kSlotChunk) {
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < kSlotChunk && q0 + i < d; i += kSlotThreads) {
                    s_col[i] = pair_col[ps + q0 + i];
                    s_first[i] = pair_first[ps + q0 + i];
                    if (use_umi) s_umi[i] = pair_umi[ps + q0 + i];
                }
                __syncthreads();
                if (p < d) {
                    const uint32_t lim = min(uint32_t(kSlotChunk), d - q0);
                    for (uint32_t i = 0; i < lim; ++i) {
                        const uint32_t cq = s_col[i]; const uint8_t fq = s_first[i];
                        cs += ((fq & 1) && cq < colp) ? 1u : 0u;
                        if (use_umi) us += ((fq & 2) && (cq < colp || (cq == colp && s_umi[i] < umip))) ? 1u : 0u;
                    }
                }
            }
            if (p < d) {
                const uint8_t fp = pair_first[ps + p];
                pair_cslot[ps + p] = ps + cs;
                if (fp & 1) { cslot_col[ps + cs] = colp; cslot_locus[ps + cs] = l; }
                if (use_umi) {
                    pair_uslot[ps + p] = ps + us;
                    if (fp & 2) uslot_cslot[ps + us] = ps + cs;
                }
            }
        }
        __syncthreads();
    }
}

// Deep loci (d > kSlotSmallMax pairs, e.g. a variant in a highly expressed gene): one 1024-thread CTA per
// locus, O(d log^2 d).  Distinct cells through a hash set in global scratch, sorted with a bitonic network,
// rank by binary search; (cell, UMI) slots only need to be distinct, so they get dense ids in hash-table order.
// scratch region of a locus = kSlotBigWords * pair_start[l] words: ctab[2d] | dcols[d] | utab[2d] | uid[2d].
__device__ __forceinline__ uint32_t mix32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }

__global__ void __launch_bounds__(kSlotBigThreads) vtx_k_slots_big(
    const uint32_t* __restrict__ big_list, const uint32_t* __restrict__ pair_start, const uint32_t* __restrict__ pair_col,
    const uint64_t* __restrict__ pair_umi, int use_umi, uint32_t* __restrict__ scratch, uint32_t* __restrict__ pair_cslot,
    uint32_t* __restrict__ pair_uslot, uint32_t* __restrict__ cslot_col, uint32_t* __restrict__ cslot_locus,
    uint32_t* __restrict__ uslot_cslot)
{
    __shared__ uint32_t s_count;
    const uint32_t n_big = big_list[0];
    const uint32_t tid = threadIdx.x;
    for (uint32_t bi = blockIdx.x; bi < n_big; bi += gridDim.x) {
        const uint32_t l = big_list[1 + bi];
        const uint32_t ps = pair_start[l], d = pair_start[l + 1] - ps;
        const uint32_t cap = 2 * d;
        uint32_t* ctab = scratch + size_t(kSlotBigWords) * ps;
        uint32_t* dcols = ctab + cap;
        uint32_t* utab = dcols + d;
        uint32_t* uid = utab + cap;
        for (uint32_t i = tid; i < cap; i += kSlotBigThreads) { ctab[i] = kInvalid; if (use_umi) utab[i] = kInvalid; }
        if (tid == 0) s_count = 0;
        __syncthreads();
        // distinct cells
        for (uint32_t p = tid; p < d; p += kSlotBigThreads) {
            const uint32_t col = pair_col[ps + p];
            uint32_t h = mix32(col) % cap;
            for (;;) {
                const uint32_t old = atomicCAS(&ctab[h], kInvalid, col);
                if (old == kInvalid || old == col) break;
                h = h + 1 == cap ? 0 : h + 1;
            }
        }
        __syncthreads();
        for (uint32_t i = tid; i < cap; i += kSlotBigThreads)
            if (ctab[i] != kInvalid) dcols[atomicAdd(&s_count, 1u)] = ctab[i];
        __syncthreads();
        const uint32_t D = s_count;
        uint32_t P = 1;
        while (P < D) P <<= 1;                       // P < 2 D <= cap: the hash-set region doubles as the sort buffer
        __syncthreads();
        for (uint32_t i = tid; i < P; i += kSlotBigThreads) ctab[i] = i < D ? dcols[i] : kInvalid;
        __syncthreads();
        for (uint32_t k = 2; k <= P; k <<= 1)
            for (uint32_t j = k >> 1; j > 0; j >>= 1) {
                for (uint32_t i = tid; i < P; i += kSlotBigThreads) {
                    const uint32_t q = i ^ j;
                    if (q > i) {
                        const uint32_t a = ctab[i], b = ctab[q];
                        const bool up = (i & k) == 0;
                        if ((a > b) == up) { ctab[i] = b; ctab[q] = a; }
                    }
                }
                __syncthreads();
            }
        // cell slots: rank among the sorted distinct cells
        for (uint32_t p = tid; p < d; p += kSlotBigThreads) {
            const uint32_t col = pair_col[ps + p];
            uint32_t lo = 0, hi = D;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ctab[mid] < col) lo = mid + 1; else hi = mid; }
            pair_cslot[ps + p] = ps + lo;
            cslot_col[ps + lo] = col;             // every pair of the cell writes the same values
            cslot_locus[ps + lo] = l;
        }
        if (use_umi) {
            if (tid == 0) s_count = 0;
            __syncthreads();
            // claim one table entry per distinct (cell, UMI); the entry remembers its first pair
            for (uint32_t p = tid; p < d; p += kSlotBigThreads) {
                const uint32_t col = pair_col[ps + p]; const uint64_t umi = pair_umi[ps + p];
                uint32_t h = mix32(col ^ mix32(uint32_t(umi) ^ mix32(uint32_t(umi >> 32)))) % cap;
                for (;;) {
                    uint32_t cur = utab[h];
                    if (cur == kInvalid) { cur = atomicCAS(&utab[h], kInvalid, p); if (cur == kInvalid) break; }
                    if (pair_col[ps + cur] == col && pair_umi[ps + cur] == umi) break;
                    h = h + 1 == cap ? 0 : h + 1;
                }
            }
            __syncthreads();
            for (uint32_t i = tid; i < cap; i += kSlotBigThreads)
                if (utab[i] != kInvalid) uid[i] = atomicAdd(&s_count, 1u);
            __syncthreads();
            for (uint32_t p = tid; p < d; p += kSlotBigThreads) {
                const uint32_t col = pair_col[ps + p]; const uint64_t umi = pair_umi[ps + p];
                uint32_t h = mix32(col ^ mix32(uint32_t(umi) ^ mix32(uint32_t(umi >> 32)))) % cap;
                for (;;) {
                    const uint32_t cur = utab[h];
                    if (pair_col[ps + cur] == col && pair_umi[ps + cur] == umi) break;
                    h = h + 1 == cap ? 0 : h + 1;
                }
                const uint32_t us = ps + uid[h];
                pair_uslot[ps + p] = us;
                uslot_cslot[us] = pair_cslot[ps + p];
            }
        }
        __syncthreads();
    }
}

// one thread per UMI slot: collapse the reads of one (locus, cell, UMI) -- main.rs:1058-1082.
// ref_frac/alt_frac >= 0.75 in f64 is exactly 4*count >= 3*total for these integer ranges.
__global__ void vtx_k_umi_collapse(uint32_t n_slots_ub, const uint32_t* __restrict__ n_pairs_ptr,
                                   const uint32_t* __restrict__ uslot_cslot, const uint32_t* __restrict__ ucnt,
                                   uint32_t* __restrict__ ccnt)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_slots_ub || q >= *n_pairs_ptr) return;
    const uint32_t cs = uslot_cslot[q];
    if (cs == kInvalid) return;
    const uint4 c = reinterpret_cast<const uint4*>(ucnt)[q];
    const uint32_t r = c.x, a = c.y, u = c.z, t = r + a + u;
    if (t == 0) return;                               // every read of this UMI evaluated to None
    uint32_t k;
    if (4ull * a >= 3ull * t) k = 1;                  // ALT
    else if (4ull * r >= 3ull * t) k = 0;             // REF
    else k = 2;                                       // UNKNOWN
    atomicAdd(ccnt + size_t(cs) * 4 + k, 1u);
}

// one thread per cell slot: mode value + keep flag
__global__ void vtx_k_finalize(uint32_t n_slots_ub, const uint32_t* __restrict__ n_pairs_ptr, int mode,
                               const uint32_t* __restrict__ cslot_col, const uint32_t* __restrict__ ccnt,
                               uint32_t* __restrict__ keep)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_slots_ub) return;
    uint32_t k = 0;
    if (q < *n_pairs_ptr && cslot_col[q] != kInvalid) {
        if (mode == 0) {                               // consensus drops cells without ref/alt evidence, main.rs:1120-1126
            const uint4 c = reinterpret_cast<const uint4*>(ccnt)[q];
            k = (c.x > 0 || c.y > 0) ? 1u : 0u;
        } else k = 1u;                                 // alt_frac / coverage emit every present cell
    }
    keep[q] = k;
}

struct ResultArrays {
    uint32_t* row; uint32_t* col; uint32_t* ref_cnt; uint32_t* alt_cnt; uint32_t* unk_cnt;
    double* val; double* val2;
};

__global__ void vtx_k_emit(uint32_t n_slots_ub, int mode, const uint32_t* __restrict__ keep,
                           const uint32_t* __restrict__ oidx, const unsigned long long* __restrict__ res_base,
                           const uint32_t* __restrict__ cslot_col, const uint32_t* __restrict__ cslot_locus,
                           const uint32_t* __restrict__ locus_row, const uint32_t* __restrict__ ccnt, ResultArrays out)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_slots_ub || !keep[q]) return;
    const uint64_t o = *res_base + oidx[q];
    const uint4 c = reinterpret_cast<const uint4*>(ccnt)[q];
    const uint32_t r = c.x, a = c.y, u = c.z;
    out.row[o] = locus_row[cslot_locus[q]];
    out.col[o] = cslot_col[q];
    out.ref_cnt[o] = r; out.alt_cnt[o] = a; out.unk_cnt[o] = u;
    double v = 0.0, v2 = 0.0;
    if (mode == 0) v = (r > 0 && a > 0) ? 3.0 : (a > 0 ? 2.0 : 1.0);                 // main.rs:1120-1126
    else if (mode == 2) v = double(a) / (double(r) + double(a) + double(u));        // main.rs:1140-1141 (0/0 = NaN)
    else { v = double(a); v2 = double(r); }                                           // main.rs:1160-1161
    out.val[o] = v; out.val2[o] = v2;
}

__global__ void vtx_k_add_u64(unsigned long long* dst, const unsigned long long* __restrict__ src, int n)
{
    if (blockIdx.x == 0 && int(threadIdx.x) < n) dst[threadIdx.x] += src[threadIdx.x];
}

// res_n += total; the running count also goes to a host-mapped slot so that vtx_finish can start copying the
// triplets of this submit while later submits are still computing
__global__ void vtx_k_bump(unsigned long long* res_n, const uint32_t* __restrict__ total, unsigned long long* cum_host)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const unsigned long long n = *res_n + (total ? *total : 0u);
        *res_n = n;
        if (cum_host) *cum_host = n;
    }
}

// ---------------------------------------------------------------------------------------------
// exclusive scan of uint32 (out has n + 1 entries; out[n] = total).  Three small kernels.
// ---------------------------------------------------------------------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total)
{
    __shared__ uint32_t warp_sums[kScanThreads / 32];
    __shared__ uint32_t s_total;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
        uint32_t s = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
        if (lane < kScanThreads / 32) warp_sums[lane] = s;
        if (lane == kScanThreads / 32 - 1) s_total = s;
    }
    __syncthreads();
    const uint32_t prefix = (w ? warp_sums[w - 1] : 0) + x - v;
    *total = s_total;
    __syncthreads();
    return prefix;
}

__global__ void __launch_bounds__(kScanThreads) vtx_k_scan_tiles(const uint32_t* __restrict__ in, uint64_t n,
                                                                 uint32_t* __restrict__ out, uint32_t* __restrict__ sums)
{
    const uint64_t base = uint64_t(blockIdx.x) * kScanTile + uint64_t(threadIdx.x) * kScanItems;
    uint32_t v[kScanItems], s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) { v[i] = (base + i < n) ? in[base + i] : 0; s += v[i]; }
    uint32_t total;
    uint32_t p = block_exclusive_scan(s, &total);
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) { if (base + i < n) out[base + i] = p; p += v[i]; }
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) vtx_k_scan_sums(uint32_t* __restrict__ sums, uint32_t n_blocks,
                                                                uint32_t* __restrict__ total_out)
{
    uint32_t carry = 0;
    for (uint32_t base = 0; base < n_blocks; base += kScanThreads) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < n_blocks ? sums[i] : 0;
        uint32_t total;
        const uint32_t p = block_exclusive_scan(v, &total);
        if (i < n_blocks) sums[i] = carry + p;
        carry += total;
    }
    if (threadIdx.x == 0) *total_out = carry;
}

// one CTA per row: exclusive scan of `rows` short arrays (the per-class tile counts) in a single launch
__global__ void __launch_bounds__(kScanThreads) vtx_k_scan_rows(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                                uint32_t n, uint32_t stride)
{
    const uint32_t* src = in + size_t(blockIdx.x) * stride;
    uint32_t* dst = out + size_t(blockIdx.x) * stride;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < n; base += kScanTile) {
        const uint32_t i0 = base + threadIdx.x * kScanItems;
        uint32_t v[kScanItems], sum = 0;
#pragma unroll
        for (int k = 0; k < kScanItems; ++k) { v[k] = (i0 + k < n) ? src[i0 + k] : 0; sum += v[k]; }
        uint32_t total;
        uint32_t p = carry + block_exclusive_scan(sum, &total);
#pragma unroll
        for (int k = 0; k < kScanItems; ++k) { if (i0 + k < n) dst[i0 + k] = p; p += v[k]; }
        carry += total;
    }
    if (threadIdx.x == 0) dst[n] = carry;
}

__global__ void __launch_bounds__(kScanThreads) vtx_k_scan_add(uint32_t* __restrict__ out, uint64_t n,
                                                               const uint32_t* __restrict__ sums)
{
    const uint64_t base = uint64_t(blockIdx.x) * kScanTile + uint64_t(threadIdx.x) * kScanItems;
    const uint32_t add = sums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) if (base + i < n) out[base + i] += add;
}

}  // namespace vtx
