// vtx_cluster_refine.cuh -- the cells of a genotype-free pool called against their clusters' fitted genotypes and the pool's
// ambient RNA, with the clusters refit from their singlets (vtx_cluster_refine, the CLI's --out-cluster-calls).
//
// Model (DESIGN.md §5j).  Round 0 fits §5i's genotypes and rho on vtx_cluster_cells' sums; every later round first rebuilds the
// sums from the previous round's labels (§5g's final M-step with W_ck = 2^16 on the label's cluster, 0 elsewhere), then fits.
// At the round's m each (touched row, cluster) gets a code: GT when GQ >= 20, else P ("no called genotype: expect the pool's
// fraction").  A row with at least one called code is scored; a hypothesis (i, j) expects at row v
//   both called     §5h's q_vs for s = g_i + g_j (ambient::row_logs)                                  entries 0..4
//   one P           (1 - rho) ((q_2g + f_v) / 2) + rho f_v, g the called one's GT; 1 - q from the complements  entries 5..7
//   both P          f_v                                                                               entry 8
// with int32 logs (log_fixed); a cell adds r Lr + a La at each scored row (int64) and is called by donors::call_of.  A cell
// called singlet on k is labelled k, every other cell is unlabelled and adds nothing to the next round's sums.  The loop stops
// when a round's labels equal the previous round's or after max_rounds rounds after round 0.
//
// Kernels (the by-cell index is §5g's; the hard sums are vtx_k_cl_final; the fit and call are §5i's vtx_k_cg_fit / vtx_k_cg_call):
//   vtx_k_cr_touch     one thread per row: touched (T_kv > 0 for some k) and fitted (touched and used) flags
//   vtx_k_cr_gather    one thread per row: the touched rows' sums, compacted by the scans of those flags
//   vtx_k_cr_codes     one thread per touched row: its K codes and the scored flag
//   vtx_k_cr_tables    one thread per touched row: a scored row's codes, row -> scored index and the nine-entry table (72 B)
//   vtx_k_cr_score     one warp per cell, lane l owns hypotheses l + 32j: log-likelihoods, counts, call and label
//   vtx_k_cr_weights   one thread per cell: the next round's hard weights and the changed-label count
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/cluster_refine_shim.cpp runs them serially on the
// CPU (tests/test_cluster_refine_cpu.py).
#pragma once
#include <cstddef>
#include <cstdint>

#include "vtx_cluster_gt.cuh"

#if defined(__CUDACC__)
#define VTX_CR_HD __host__ __device__
#else
#define VTX_CR_HD
#endif

namespace vtx {
namespace cluster_refine {

constexpr uint8_t kP = 3;                               // no called genotype: the pool's fraction
constexpr uint32_t kNone = 0xFFFFFFFFu;                 // no label / not a scored row (VTX_NO_LABEL)
constexpr uint32_t kMaxRounds = 32;
constexpr uint32_t kEntries = 9;                        // table entries per scored row
constexpr uint64_t kMaxTotalMolecules = cluster_gt::kMaxTotalDepthW >> 16;     // 2^16 sum(r + a) <= 2^51 bounds every round's sums

// the code of one (touched row, cluster) from its GT and PL
VTX_CR_HD inline uint8_t code_of(uint8_t gt, const uint32_t* pl)
{
    return cluster_gt::gq_of(pl) >= cluster_gt::kMinGq ? gt : kP;
}

// the table entry of a hypothesis whose clusters have codes c1, c2
VTX_CR_HD inline uint32_t entry_of(uint32_t c1, uint32_t c2)
{
    return c1 != kP && c2 != kP ? c1 + c2 : c1 != kP ? 5 + c1 : c2 != kP ? 5 + c2 : 8;
}

// the nine-entry table of one row at m: out[2 i] = La_i, out[2 i + 1] = Lr_i
VTX_CR_HD inline void row_logs9(const ambient::Fractions& fr, uint32_t m, uint64_t A, uint64_t T, int32_t* out)
{
    using namespace clusters;
    ambient::row_logs(fr, m, A, T, out);
    const double den = double(T + 2);
    const double f = d_div(double(A + 1), den), of = d_div(double(T - A + 1), den);
    const double rho = d_div(double(m), 1000.0), orho = d_div(double(1000 - m), 1000.0);
    for (int g = 0; g < 3; ++g) {
        out[10 + 2 * g] = ambient::mix_log(d_mul(d_add(fr.q[2 * g], f), 0.5), rho, orho, f);
        out[11 + 2 * g] = ambient::mix_log(d_mul(d_add(fr.oq[2 * g], of), 0.5), rho, orho, of);
    }
    out[16] = log_fixed(f);
    out[17] = log_fixed(of);
}

// ---- serial body (tests/cluster_refine_shim.cpp): vtx_k_cr_score computes the same integers with one lane per hypothesis ------
// cell c against the scored rows: sidx maps a row to its scored index (kNone: skipped), code [scored][K], tab [scored][9][2]:
// ll[H], cnt[3] = scored rows, ref, alt
VTX_CR_HD inline void score_cell(const clusters::CellEntries& ce, uint32_t c, uint32_t K, const uint32_t* sidx, const uint8_t* code,
                                 const int32_t* tab, int64_t* ll, uint64_t* cnt)
{
    const uint32_t H = donors::n_hyp(K);
    for (uint32_t h = 0; h < H; ++h) ll[h] = 0;
    cnt[0] = cnt[1] = cnt[2] = 0;
    for (uint32_t i = ce.start[c]; i < ce.start[c + 1]; ++i) {
        const uint32_t s = sidx[ce.row[i]];
        if (s == kNone) continue;
        const uint8_t* cs = code + size_t(s) * K;
        for (uint32_t h = 0; h < H; ++h) {
            uint32_t d1, d2;
            donors::hyp_donors(h, K, &d1, &d2);
            const int32_t* x = tab + (size_t(s) * kEntries + entry_of(cs[d1], cs[d2])) * 2;
            ll[h] += int64_t(ce.r[i]) * x[1] + int64_t(ce.a[i]) * x[0];
        }
        cnt[0] += 1; cnt[1] += ce.r[i]; cnt[2] += ce.a[i];
    }
}

#ifdef __CUDACC__
constexpr int kCrThreads = 256;

__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_touch(uint64_t n_rows, uint32_t K, const int64_t* __restrict__ T,
                                                             const uint8_t* __restrict__ used, uint32_t* __restrict__ tflag,
                                                             uint32_t* __restrict__ fflag)
{
    for (uint64_t v = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; v < n_rows; v += uint64_t(gridDim.x) * blockDim.x) {
        bool reached = false;
        for (uint32_t k = 0; k < K; ++k) reached = reached || T[v * K + k] > 0;
        tflag[v] = reached;
        fflag[v] = reached && used[v];
    }
}

// A / T [n_rows][K], rowA / rowT [n_rows] -> cA / cT [touched][K], crow [touched] (A_v, then T_v at + n_t), trow [touched],
// fit [fitted] (touched indices)
__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_gather(uint64_t n_rows, uint32_t K, uint32_t n_t, const int64_t* __restrict__ A,
                                                              const int64_t* __restrict__ T, const unsigned long long* __restrict__ rowA,
                                                              const unsigned long long* __restrict__ rowT, const uint32_t* __restrict__ tflag,
                                                              const uint32_t* __restrict__ tpos, const uint32_t* __restrict__ fflag,
                                                              const uint32_t* __restrict__ fpos, int64_t* __restrict__ cA,
                                                              int64_t* __restrict__ cT, unsigned long long* __restrict__ crow,
                                                              uint32_t* __restrict__ trow, uint32_t* __restrict__ fit)
{
    for (uint64_t v = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; v < n_rows; v += uint64_t(gridDim.x) * blockDim.x) {
        if (!tflag[v]) continue;
        const uint32_t t = tpos[v];
        for (uint32_t k = 0; k < K; ++k) { cA[size_t(t) * K + k] = A[v * K + k]; cT[size_t(t) * K + k] = T[v * K + k]; }
        crow[t] = rowA[v];
        crow[size_t(n_t) + t] = rowT[v];
        trow[t] = uint32_t(v);
        if (fflag[v]) fit[fpos[v]] = t;
    }
}

// gt [touched][K], pl [touched][K][3] -> code [touched][K], sflag [touched]
__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_codes(uint32_t n_t, uint32_t K, const uint8_t* __restrict__ gt,
                                                             const uint32_t* __restrict__ pl, uint8_t* __restrict__ code,
                                                             uint32_t* __restrict__ sflag)
{
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_t; t += gridDim.x * blockDim.x) {
        bool any = false;
        for (uint32_t k = 0; k < K; ++k) {
            const size_t o = size_t(t) * K + k;
            const uint8_t c = code_of(gt[o], pl + o * 3);
            code[o] = c;
            any = any || c != kP;
        }
        sflag[t] = any;
    }
}

// the scored rows: sidx [row] = s (preset to kNone), scode [s][K], tab [s][9][2] at m
__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_tables(uint32_t m, ambient::Fractions fr, uint32_t n_t, uint32_t K,
                                                              const uint32_t* __restrict__ trow, const unsigned long long* __restrict__ crow,
                                                              const uint8_t* __restrict__ code, const uint32_t* __restrict__ sflag,
                                                              const uint32_t* __restrict__ spos, uint32_t* __restrict__ sidx,
                                                              uint8_t* __restrict__ scode, int32_t* __restrict__ tab)
{
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_t; t += gridDim.x * blockDim.x) {
        if (!sflag[t]) continue;
        const uint32_t s = spos[t];
        sidx[trow[t]] = s;
        for (uint32_t k = 0; k < K; ++k) scode[size_t(s) * K + k] = code[size_t(t) * K + k];
        row_logs9(fr, m, crow[t], crow[size_t(n_t) + t], tab + size_t(s) * kEntries * 2);
    }
}

// One warp per cell.  The lanes load 32 entries of the cell at once and hand them round with shuffles; an entry at a scored row
// has lane k < K load cluster k's code, and three ballots (GT bit 0, GT bit 1, called) hand every lane all K codes.  The nine
// table values are picked by selects.  Writes ll [c][H], cnt [c][3], label [c]; adds the call to calls[3].
template <int KH>
__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_score(clusters::CellEntries ce, uint32_t n_cols, uint32_t K,
                                                             const uint32_t* __restrict__ sidx, const uint8_t* __restrict__ scode,
                                                             const int32_t* __restrict__ tab, int64_t* __restrict__ ll,
                                                             uint64_t* __restrict__ cnt, uint32_t* __restrict__ label,
                                                             unsigned long long* __restrict__ calls)
{
    using clusters::warp_max_i64;
    using clusters::warp_sum_u64;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t H = donors::n_hyp(K);
    uint32_t pair[KH];
#pragma unroll
    for (int j = 0; j < KH; ++j) {
        uint32_t d1 = 0, d2 = 0;
        if (lane + 32u * j < H) donors::hyp_donors(lane + 32u * j, K, &d1, &d2);
        pair[j] = d1 | d2 << 8;
    }
    const int2* tb = reinterpret_cast<const int2*>(tab);
    for (uint32_t c = warp; c < n_cols; c += n_warps) {
        const uint32_t i0 = ce.start[c], i1 = ce.start[c + 1];
        int64_t acc[KH];
#pragma unroll
        for (int j = 0; j < KH; ++j) acc[j] = 0;
        uint64_t n_v = 0, sum_r = 0, sum_a = 0;
        for (uint32_t base = i0; base < i1; base += 32) {
            const uint32_t i = base + lane;
            uint32_t s = kNone, r = 0, a = 0;
            if (i < i1) { s = sidx[ce.row[i]]; r = ce.r[i]; a = ce.a[i]; }
            if (s != kNone) { n_v += 1; sum_r += r; sum_a += a; }
            const uint32_t n = min(32u, i1 - base);
            for (uint32_t e = 0; e < n; ++e) {
                const uint32_t se = __shfl_sync(0xffffffffu, s, e), re = __shfl_sync(0xffffffffu, r, e), ae = __shfl_sync(0xffffffffu, a, e);
                if (se == kNone) continue;                      // warp-uniform
                const uint32_t cd = lane < K ? scode[size_t(se) * K + lane] : uint32_t(kP);
                const uint32_t b0 = __ballot_sync(0xffffffffu, cd & 1u), b1 = __ballot_sync(0xffffffffu, cd & 2u);
                const uint32_t bc = __ballot_sync(0xffffffffu, cd != kP);
                int64_t v[kEntries];
#pragma unroll
                for (uint32_t x = 0; x < kEntries; ++x) {
                    const int2 t = tb[size_t(se) * kEntries + x];
                    v[x] = int64_t(re) * t.y + int64_t(ae) * t.x;
                }
#pragma unroll
                for (int j = 0; j < KH; ++j) {
                    const uint32_t d1 = pair[j] & 0xFF, d2 = pair[j] >> 8;
                    const uint32_t c1 = bc >> d1 & 1u ? (b0 >> d1 & 1u) | (b1 >> d1 & 1u) << 1 : kP;
                    const uint32_t c2 = bc >> d2 & 1u ? (b0 >> d2 & 1u) | (b1 >> d2 & 1u) << 1 : kP;
                    const uint32_t x = entry_of(c1, c2);
                    int64_t y = v[0];                           // selects, not an indexed (local-memory) array
                    y = x == 1 ? v[1] : y; y = x == 2 ? v[2] : y; y = x == 3 ? v[3] : y; y = x == 4 ? v[4] : y;
                    y = x == 5 ? v[5] : y; y = x == 6 ? v[6] : y; y = x == 7 ? v[7] : y; y = x == 8 ? v[8] : y;
                    acc[j] += y;
                }
            }
        }
        n_v = warp_sum_u64(n_v); sum_r = warp_sum_u64(sum_r); sum_a = warp_sum_u64(sum_a);
        const int64_t best = warp_max_i64(lane < K ? acc[0] : INT64_MIN);
        const uint32_t first = __ffs(__ballot_sync(0xffffffffu, lane < K && acc[0] == best)) - 1;
        const int64_t second = warp_max_i64(lane < K && lane != first ? acc[0] : INT64_MIN);
        int64_t pm = INT64_MIN;
#pragma unroll
        for (int j = 0; j < KH; ++j) {
            const uint32_t h = lane + 32u * j;
            if (h >= K && h < H) pm = acc[j] > pm ? acc[j] : pm;
        }
        const int64_t pbest = warp_max_i64(pm);
        int64_t* out = ll + size_t(c) * H;
#pragma unroll
        for (int j = 0; j < KH; ++j)
            if (lane + 32u * j < H) out[lane + 32u * j] = acc[j];
        if (lane == 0) {
            const uint32_t call = donors::call_of(n_v, best, second, pbest);
            atomicAdd(&calls[call], 1ull);
            label[c] = call == 0 ? first : kNone;
            cnt[3 * size_t(c)] = n_v; cnt[3 * size_t(c) + 1] = sum_r; cnt[3 * size_t(c) + 2] = sum_a;
        }
    }
}

// label [c] -> w [c][K] (2^16 on the label's cluster), prev [c] <- label [c], changed += the labels that differ from prev
__global__ void __launch_bounds__(kCrThreads) vtx_k_cr_weights(uint32_t n_cols, uint32_t K, const uint32_t* __restrict__ label,
                                                               uint32_t* __restrict__ prev, uint32_t* __restrict__ w,
                                                               unsigned long long* __restrict__ changed)
{
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cols; c += gridDim.x * blockDim.x) {
        const uint32_t l = label[c];
        for (uint32_t k = 0; k < K; ++k) w[size_t(c) * K + k] = l == k ? uint32_t(clusters::kW) : 0u;
        if (l != prev[c]) { atomicAdd(changed, 1ull); prev[c] = l; }
    }
}
#endif   // __CUDACC__

}  // namespace cluster_refine
}  // namespace vtx
