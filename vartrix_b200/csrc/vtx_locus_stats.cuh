// vtx_locus_stats.cuh -- per-locus summary of one shard (vtx_set_locus_stats / vtx_locus_stats_get, the CLI's
// --out-variant-stats): why a matrix row holds what it holds.
//
// Every number is already on the device after vtx_k_umi_collapse; this is a per-locus reduction of it:
//   candidates  [cand_start[l], cand_start[l + 1])  -> no_cell_barcode / no_umi (the test of vtx_k_cand_filter)
//   UMI slots   [pair_start[l], pair_start[l + 1])  -> reads_* (ucnt: per-read calls; with use_umi or name keys)
//   cell slots  [pair_start[l], pair_start[l + 1])  -> calls_* and the cell categories (ccnt: the counts the matrix is built
//                                                       from), and reads_* without use_umi (then ccnt holds per-read calls)
// Slots of a locus are locus-contiguous by construction (slot = pair_start[locus] + rank, vtx_k_slots); unused slots hold zero
// counts and kInvalid cells.  The record-filter counters come from locus_cands (vtx_stage.cuh) for vtx_submit_bam shards and
// are 0 for host batches, whose caller counts them while staging.
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): the kernel is a CTA-wide sum over them, and tests/locus_stats_shim.cpp runs the
// same bodies serially on the CPU (tests/test_variant_stats_cpu.py).
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define VTX_LS_HD __host__ __device__
#else
#define VTX_LS_HD
#endif

namespace vtx {
namespace lstats {

// the fields of vtx_locus_stats (include/vartrix_b200.h), in its order
enum : int {
    kRow = 0, kFetched, kLowMapq, kNonPrimary, kDuplicate, kNotUseful, kLowBaseQuality, kNoCellBarcode, kNoUmi, kScored,
    kReadsRef, kReadsAlt, kReadsUnknown, kReadsNone, kCallsRef, kCallsAlt, kCallsUnknown,
    kCells, kCellsRefOnly, kCellsAltOnly, kCellsBoth, kCellsMultiUnknown, kFields
};
constexpr int kFilters = 6;             // kFetched .. kLowBaseQuality: what locus_cands stores per locus
// the summed counters
enum : int { sNoCb = 0, sNoUmi, sReadsRef, sReadsAlt, sReadsUnk, sCallsRef, sCallsAlt, sCallsUnk, sCells, sRefOnly, sAltOnly, sBoth, sMultiUnk, kSums };

constexpr uint64_t kNoUmiKey = 0xFFFFFFFFFFFFFFFFull;
constexpr uint32_t kNoCell = 0xFFFFFFFFu;

struct Inputs {
    const uint64_t* cand_start;     // [n_loci + 1]
    const uint32_t* cand_read;      // [n_cand], nullptr: candidate c is read c
    const int32_t* read_col;        // [n_reads] barcode column or -1
    const uint64_t* read_umi;       // [n_reads] with use_umi, else nullptr
    const uint32_t* pair_start;     // [n_loci + 1], nullptr: no pair of the shard reached Smith-Waterman
    const uint32_t* ucnt;           // [slot][4] per-read calls of a (cell, UMI) slot, nullptr without use_umi
    const uint32_t* ccnt;           // [slot][4] calls of a cell slot (after the collapse with use_umi)
    const uint32_t* cslot_col;      // [slot] column or kNoCell
    const uint32_t* locus_row;      // [n_loci]
    const uint32_t* filters;        // [n_loci][kFilters] from locus_cands, nullptr: host batch
};

VTX_LS_HD inline void add_candidate(const Inputs& in, uint64_t c, uint32_t* s)
{
    const uint32_t r = in.cand_read ? in.cand_read[c] : uint32_t(c);
    if (in.read_col[r] < 0) ++s[sNoCb];                                        // main.rs:868-876
    else if (in.read_umi && in.read_umi[r] == kNoUmiKey) ++s[sNoUmi];          // main.rs:880-888
}

VTX_LS_HD inline void add_slot(const Inputs& in, uint32_t q, uint32_t* s)
{
    const uint32_t* rd = (in.ucnt ? in.ucnt : in.ccnt) + 4 * size_t(q);
    s[sReadsRef] += rd[0]; s[sReadsAlt] += rd[1]; s[sReadsUnk] += rd[2];
    if (in.cslot_col[q] == kNoCell) return;
    const uint32_t* cc = in.ccnt + 4 * size_t(q);
    const uint32_t r = cc[0], a = cc[1], u = cc[2];
    s[sCallsRef] += r; s[sCallsAlt] += a; s[sCallsUnk] += u;
    s[sCells] += 1;
    s[sRefOnly] += (r > 0 && a == 0) ? 1u : 0u;         // consensus value 1 (main.rs:1120-1126)
    s[sAltOnly] += (a > 0 && r == 0) ? 1u : 0u;         // 2
    s[sBoth] += (r > 0 && a > 0) ? 1u : 0u;             // 3
    s[sMultiUnk] += u > 1 ? 1u : 0u;                    // "Check this locus manually" (main.rs:1116-1118)
}

VTX_LS_HD inline void write_entry(const Inputs& in, uint32_t l, const uint32_t* s, uint32_t* out)
{
    out[kRow] = in.locus_row[l];
    for (int f = 0; f < kFilters; ++f) out[kFetched + f] = in.filters ? in.filters[size_t(l) * kFilters + f] : 0u;
    out[kNoCellBarcode] = s[sNoCb]; out[kNoUmi] = s[sNoUmi];
    const uint32_t scored = in.pair_start ? in.pair_start[l + 1] - in.pair_start[l] : 0u;
    out[kScored] = scored;
    out[kReadsRef] = s[sReadsRef]; out[kReadsAlt] = s[sReadsAlt]; out[kReadsUnknown] = s[sReadsUnk];
    out[kReadsNone] = scored - (s[sReadsRef] + s[sReadsAlt] + s[sReadsUnk]);      // evaluate_scores gave None (main.rs:1019-1030)
    out[kCallsRef] = s[sCallsRef]; out[kCallsAlt] = s[sCallsAlt]; out[kCallsUnknown] = s[sCallsUnk];
    out[kCells] = s[sCells]; out[kCellsRefOnly] = s[sRefOnly]; out[kCellsAltOnly] = s[sAltOnly]; out[kCellsBoth] = s[sBoth];
    out[kCellsMultiUnknown] = s[sMultiUnk];
}

// one locus, serially (the CPU tests)
VTX_LS_HD inline void locus_serial(const Inputs& in, uint32_t l, uint32_t* out)
{
    uint32_t s[kSums] = {};
    for (uint64_t c = in.cand_start[l]; c < in.cand_start[l + 1]; ++c) add_candidate(in, c, s);
    if (in.pair_start)
        for (uint32_t q = in.pair_start[l]; q < in.pair_start[l + 1]; ++q) add_slot(in, q, s);
    write_entry(in, l, s, out);
}

#ifdef __CUDACC__
// One CTA per locus (grid-stride): a locus of 100 000 pairs is summed by 128 threads, a shallow one costs one short pass.
constexpr int kStatsThreads = 128;
__global__ void __launch_bounds__(kStatsThreads) vtx_k_locus_stats(Inputs in, uint32_t n_loci, uint32_t* __restrict__ out)
{
    __shared__ uint32_t s_sum[kSums];
    for (uint32_t l = blockIdx.x; l < n_loci; l += gridDim.x) {
        uint32_t acc[kSums] = {};
        const uint64_t c0 = in.cand_start[l], c1 = in.cand_start[l + 1];
        for (uint64_t c = c0 + threadIdx.x; c < c1; c += kStatsThreads) add_candidate(in, c, acc);
        if (in.pair_start) {
            const uint32_t q1 = in.pair_start[l + 1];
            for (uint32_t q = in.pair_start[l] + threadIdx.x; q < q1; q += kStatsThreads) add_slot(in, q, acc);
        }
        if (threadIdx.x < kSums) s_sum[threadIdx.x] = 0;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kSums; ++k) {
            const uint32_t v = __reduce_add_sync(0xffffffffu, acc[k]);
            if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_sum[k], v);
        }
        __syncthreads();
        if (threadIdx.x == 0) write_entry(in, l, s_sum, out + size_t(l) * kFields);
        __syncthreads();
    }
}
#endif   // __CUDACC__

}  // namespace lstats
}  // namespace vtx
