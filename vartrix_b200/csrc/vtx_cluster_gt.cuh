// vtx_cluster_gt.cuh -- genotypes of genotype-free clusters against the pool's ambient RNA, and their match to a VCF's samples
// (vtx_cluster_genotypes, the CLI's --out-cluster-genotypes / --out-cluster-matches).
//
// Model (DESIGN.md §5i).  Inputs are vtx_cluster_cells' final sums A_kv / T_kv (x 2^16; R_kv = T_kv - A_kv) and §5h's row sums
// A_v / T_v.  At rho = m / 1000 a diploid dosage g in {0, 1, 2} expects §5h's q_vs for s = 2g (epsilon, 0.5 and 1 - epsilon
// mixed with the pool fraction f_v, in row_logs' expressions), with int32 logs La_g / Lr_g, and
//   LL_vkg = floor((A_kv La_g + R_kv Lr_g) / 2^16)            exact: a 128-bit product, an arithmetic shift, int64 x 2^24 nats
// The estimate maximises J(m) = sum over used rows and all k of max_g LL_vkg on §5h's grid.  At the chosen m every (v, k) with
// T_kv > 0 gets GT = argmax_g LL (ties: the lowest g), PL_g = floor((10 (LL_max - LL_g) + floor(L10 / 2)) / L10) saturated at
// 2^31 - 1 (L10 = log(10) x 2^24) and GQ = min(99, the second-smallest PL).  Against S sample dosages, over the rows where
// every sample has one: M_ks = sum_v LL_{v,k,g_sv}, and the rows with GQ >= 20 where GT differs from g_sv.
// A per-cluster rho is not identifiable (with a free theta per cluster and row, (1 - rho) theta + rho f only reparametrises
// theta); tying each cluster's fraction to a dosage is what makes one shared rho identifiable.
//
// Kernels (one warp per item; lane k owns cluster k, K <= 32):
//   vtx_k_cg_fit     one warp per (m of the batch, fitted row): lanes 0-5 compute the six logs and shuffle them, lane k the
//                    max over g; the warp's sum goes to J(m) by an integer atomic
//   vtx_k_cg_call    one warp per touched row at the chosen m: LL [touched][K][3] (kept on the device), GT and PL
//   vtx_k_cg_match   a 2-D grid of (row chunk, sample chunk) CTAs: a tile of rows' LL / GT / called flags and dosages in shared
//                    memory, each thread owns up to kPairs (k, s) pairs in registers; one integer atomic per pair per CTA
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/cluster_gt_shim.cpp runs them serially on the CPU
// (tests/test_cluster_genotypes_cpu.py).
#pragma once
#include <cstddef>
#include <cstdint>

#include "vtx_ambient.cuh"

#if defined(__CUDACC__)
#define VTX_CG_HD __host__ __device__
#else
#define VTX_CG_HD
#endif

namespace vtx {
namespace cluster_gt {

constexpr uint32_t kMaxSamples = 1024;
constexpr int64_t kMaxDepthW = int64_t(1) << 51;        // T_kv: the LL products stay below 2^79 and LL in int64
constexpr uint64_t kMaxTotalDepthW = 1ull << 51;        // the sum of T_kv over every row and cluster: J and M_ks stay in int64
constexpr int64_t kL10 = 38630967;                      // llrint(log(10) 2^24)
constexpr uint32_t kMaxPl = 0x7FFFFFFFu;
constexpr uint32_t kMaxGq = 99;
constexpr uint32_t kMinGq = 20;                         // a genotype is "called" at GQ >= 20
constexpr int64_t kMinLlr = int64_t(5) << 24;           // 5 nats between the best and the second sample
constexpr uint8_t kMissing = 0xFF;                      // VTX_GT_MISSING

// log j of the three genotype fractions at (m, row): j = 2g is La_g, j = 2g + 1 is Lr_g (row_logs' entries for s = 2g)
VTX_CG_HD inline int32_t gt_log(const ambient::Fractions& fr, uint32_t m, uint64_t A, uint64_t T, uint32_t j)
{
    return ambient::row_log(fr, m, A, T, int(2 * (j >> 1)), (j & 1u) == 0);
}

// LL_vkg: floor((a La + (t - a) Lr) / 2^16); |a La + (t - a) Lr| < 2^79, the shift of a signed 128-bit value is the floor
VTX_CG_HD inline int64_t gt_ll(int64_t a, int64_t t, int32_t la, int32_t lr)
{
    const __int128 p = (__int128)a * la + (__int128)(t - a) * lr;
    return int64_t(p >> 16);
}

// one (row, cluster) against the six logs L: ll[3] and its maximum
VTX_CG_HD inline int64_t fit_row(const int32_t* L, int64_t a, int64_t t, int64_t* ll)
{
    int64_t mx = 0;
    for (int g = 0; g < 3; ++g) {
        ll[g] = gt_ll(a, t, L[2 * g], L[2 * g + 1]);
        mx = g == 0 || ll[g] > mx ? ll[g] : mx;
    }
    return mx;
}

// floor((10 d + floor(L10 / 2)) / L10) saturated at 2^31 - 1, for d = LL_max - LL_g >= 0.  The 128-bit quotient saturates
// whenever d >= 2^54 (10 x 2^54 / L10 > 2^32); below that 10 d + L10 / 2 < 2^58 and 64 bits hold it.
VTX_CG_HD inline uint32_t phred(int64_t d)
{
    const uint64_t u = uint64_t(d);
    if (u >= (1ull << 54)) return kMaxPl;
    const uint64_t q = (10 * u + uint64_t(kL10 / 2)) / uint64_t(kL10);
    return q > kMaxPl ? kMaxPl : uint32_t(q);
}

// GT and PL of one (row, cluster); a cluster that no molecule reached (T_kv = 0) is missing with PL 0
VTX_CG_HD inline void call_row(const int64_t* ll, bool reached, uint8_t* gt, uint32_t* pl)
{
    if (!reached) { *gt = kMissing; pl[0] = pl[1] = pl[2] = 0; return; }
    uint32_t best = 0;
    for (uint32_t g = 1; g < 3; ++g) if (ll[g] > ll[best]) best = g;
    *gt = uint8_t(best);
    for (int g = 0; g < 3; ++g) pl[g] = phred(ll[best] - ll[g]);
}

// min(99, the second-smallest PL)
VTX_CG_HD inline uint32_t gq_of(const uint32_t* pl)
{
    const uint32_t lo = pl[0] < pl[1] ? pl[0] : pl[1], hi = pl[0] < pl[1] ? pl[1] : pl[0];
    const uint32_t second = pl[2] < lo ? lo : pl[2] < hi ? pl[2] : hi;
    return second < kMaxGq ? second : kMaxGq;
}

// one compared row's contribution to (cluster k, sample s) with dosage g: M_ks and discordant_ks
VTX_CG_HD inline void match_row(const int64_t* ll, uint8_t gt, bool called, uint8_t g, int64_t* M, uint32_t* disc)
{
    *M += ll[g];
    *disc += called && gt != g;
}

// ---- the assignment of one cluster from its match sums (host: the CLI and the tests) ------------------------------------------
struct Assignment {
    uint32_t best, second;      // second = best when S = 1
    int64_t llr;                // M_best - M_second (0 when S = 1)
    bool assigned;
};

// M [S], disc [S] of one cluster; ties go to the lowest sample
inline Assignment assign(const int64_t* M, const uint64_t* disc, uint64_t called, uint32_t S)
{
    Assignment a{ 0, 0, 0, false };
    for (uint32_t s = 1; s < S; ++s) if (M[s] > M[a.best]) a.best = s;
    if (S > 1) {
        a.second = a.best == 0 ? 1 : 0;
        for (uint32_t s = a.second + 1; s < S; ++s) if (s != a.best && M[s] > M[a.second]) a.second = s;
        a.llr = M[a.best] - M[a.second];
    } else {
        a.second = a.best;
    }
    a.assigned = S > 0 && disc[a.best] * 10 <= called && (S == 1 || a.llr >= kMinLlr);
    return a;
}

#ifdef __CUDACC__
constexpr int kCgThreads = 256;
constexpr uint32_t kMatchRows = 32;                     // rows per shared-memory tile of vtx_k_cg_match
constexpr uint32_t kMatchSamples = 64;                  // samples per CTA column of vtx_k_cg_match
constexpr uint32_t kPairs = (clusters::kMaxK * kMatchSamples + kCgThreads - 1) / kCgThreads;     // (k, s) pairs per thread

// the six logs of a row at m, computed by lanes 0-5 and handed to every lane (j unrolled: a constant index into fr keeps the
// fractions in registers, not in a local copy)
__device__ __forceinline__ void warp_logs(const ambient::Fractions& fr, uint32_t m, uint64_t A, uint64_t T, uint32_t lane, int32_t* L)
{
    int32_t x = 0;
#pragma unroll
    for (uint32_t j = 0; j < 6; ++j)
        if (lane == j) x = gt_log(fr, m, A, T, j);
#pragma unroll
    for (int j = 0; j < 6; ++j) L[j] = __shfl_sync(0xffffffffu, x, j);
}

// One warp per (m of the batch, fitted row), m-major.  fit_t lists touched indices; A / T [touched][K], rowA / rowT [touched].
__global__ void __launch_bounds__(kCgThreads) vtx_k_cg_fit(ambient::Batch bt, ambient::Fractions fr, uint32_t K, uint32_t n_fit,
                                                           const uint32_t* __restrict__ fit_t, const unsigned long long* __restrict__ rowA,
                                                           const unsigned long long* __restrict__ rowT, const int64_t* __restrict__ A,
                                                           const int64_t* __restrict__ T, unsigned long long* __restrict__ J)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    const uint64_t total = uint64_t(bt.n) * n_fit;
    for (uint64_t wi = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; wi < total; wi += n_warps) {
        const uint32_t b = uint32_t(wi / n_fit), t = fit_t[wi % n_fit];
        int32_t L[6];
        warp_logs(fr, bt.m[b], rowA[t], rowT[t], lane, L);
        int64_t mx = 0;
        if (lane < K) {
            int64_t ll[3];
            mx = fit_row(L, A[size_t(t) * K + lane], T[size_t(t) * K + lane], ll);
        }
        const uint64_t sum = clusters::warp_sum_u64(uint64_t(mx));     // two's complement: exact while J fits int64
        if (lane == 0) atomicAdd(&J[b], (unsigned long long)sum);
    }
}

// One warp per touched row at m: LL [touched][K][3], GT [touched][K], PL [touched][K][3]
__global__ void __launch_bounds__(kCgThreads) vtx_k_cg_call(uint32_t m, ambient::Fractions fr, uint32_t K, uint32_t n_t,
                                                            const unsigned long long* __restrict__ rowA, const unsigned long long* __restrict__ rowT,
                                                            const int64_t* __restrict__ A, const int64_t* __restrict__ T,
                                                            int64_t* __restrict__ LL, uint8_t* __restrict__ gt, uint32_t* __restrict__ pl)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    for (uint64_t t = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; t < n_t; t += n_warps) {
        int32_t L[6];
        warp_logs(fr, m, rowA[t], rowT[t], lane, L);
        if (lane < K) {
            const size_t o = size_t(t) * K + lane;
            int64_t ll[3];
            uint32_t p[3];
            uint8_t g;
            fit_row(L, A[o], T[o], ll);
            call_row(ll, T[o] > 0, &g, p);
            gt[o] = g;
#pragma unroll
            for (int j = 0; j < 3; ++j) { LL[o * 3 + j] = ll[j]; pl[o * 3 + j] = p[j]; }
        }
    }
}

// CTA (x, y): compared rows [x rows_per_cta, (x + 1) rows_per_cta), samples [y kMatchSamples, (y + 1) kMatchSamples).  cmp_t maps a
// compared row to its touched index, dos [compared][S].  Thread i owns the pairs p = i + kCgThreads j (k = p / 64, s = p % 64):
// a warp reads 32 consecutive dosages of one row and one cluster's LL (a broadcast).  M / disc [K][S], rows / called [K] (the
// y = 0 CTAs count those).
__global__ void __launch_bounds__(kCgThreads) vtx_k_cg_match(uint32_t K, uint32_t S, uint32_t n_cmp, uint32_t rows_per_cta,
                                                             const uint32_t* __restrict__ cmp_t, const uint8_t* __restrict__ dos,
                                                             const int64_t* __restrict__ LL, const uint8_t* __restrict__ gt,
                                                             const uint32_t* __restrict__ pl, unsigned long long* __restrict__ M,
                                                             unsigned long long* __restrict__ disc, unsigned long long* __restrict__ rows,
                                                             unsigned long long* __restrict__ called)
{
    __shared__ int64_t s_ll[kMatchRows][clusters::kMaxK][3];
    __shared__ uint8_t s_gt[kMatchRows][clusters::kMaxK], s_called[kMatchRows][clusters::kMaxK];
    __shared__ uint8_t s_dos[kMatchRows][kMatchSamples];
    const uint32_t tid = threadIdx.x, s0 = blockIdx.y * kMatchSamples;
    const uint64_t r0 = uint64_t(blockIdx.x) * rows_per_cta, r1 = r0 + rows_per_cta < n_cmp ? r0 + rows_per_cta : n_cmp;
    int64_t acc[kPairs];
    uint32_t dis[kPairs];
#pragma unroll
    for (uint32_t j = 0; j < kPairs; ++j) { acc[j] = 0; dis[j] = 0; }
    uint64_t n_rows = 0, n_called = 0;
    for (uint64_t tile = r0; tile < r1; tile += kMatchRows) {
        const uint32_t nr = uint32_t(r1 - tile < kMatchRows ? r1 - tile : kMatchRows);
        __syncthreads();
        for (uint32_t i = tid; i < nr * K * 3; i += kCgThreads) {
            const uint32_t r = i / (K * 3), e = i % (K * 3);
            s_ll[r][e / 3][e % 3] = LL[size_t(cmp_t[tile + r]) * K * 3 + e];
        }
        for (uint32_t i = tid; i < nr * K; i += kCgThreads) {
            const uint32_t r = i / K, k = i % K;
            const size_t o = size_t(cmp_t[tile + r]) * K + k;
            s_gt[r][k] = gt[o];
            s_called[r][k] = gq_of(pl + o * 3) >= kMinGq;
        }
        for (uint32_t i = tid; i < nr * kMatchSamples; i += kCgThreads) {
            const uint32_t r = i / kMatchSamples, sl = i % kMatchSamples;
            s_dos[r][sl] = s0 + sl < S ? dos[size_t(tile + r) * S + s0 + sl] : 0;
        }
        __syncthreads();
        for (uint32_t r = 0; r < nr; ++r) {
#pragma unroll
            for (uint32_t j = 0; j < kPairs; ++j) {
                const uint32_t p = tid + kCgThreads * j, k = p / kMatchSamples, sl = p % kMatchSamples;
                if (k < K) match_row(s_ll[r][k], s_gt[r][k], s_called[r][k], s_dos[r][sl], &acc[j], &dis[j]);
            }
        }
        if (blockIdx.y == 0 && tid < K)
            for (uint32_t r = 0; r < nr; ++r) { n_rows += s_gt[r][tid] != kMissing; n_called += s_called[r][tid]; }
    }
#pragma unroll
    for (uint32_t j = 0; j < kPairs; ++j) {
        const uint32_t p = tid + kCgThreads * j, k = p / kMatchSamples, s = s0 + p % kMatchSamples;
        if (k < K && s < S) {
            atomicAdd(&M[size_t(k) * S + s], (unsigned long long)acc[j]);
            atomicAdd(&disc[size_t(k) * S + s], (unsigned long long)dis[j]);
        }
    }
    if (blockIdx.y == 0 && tid < K) { atomicAdd(&rows[tid], (unsigned long long)n_rows); atomicAdd(&called[tid], (unsigned long long)n_called); }
}
#endif   // __CUDACC__

}  // namespace cluster_gt
}  // namespace vtx
