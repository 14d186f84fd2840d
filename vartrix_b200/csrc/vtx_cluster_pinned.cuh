// vtx_cluster_pinned.cuh -- clustering of a pool where some donors are genotyped (vtx_cluster_cells_pinned, the CLI's
// --known-donors): §5g's allele-fraction EM with the first J clusters pinned to the VCF's genotypes of J samples.
//
// Model (DESIGN.md §5k).  §5g's model, except that EM cluster j < J at a row v where sample j has a dosage g is not fitted: it
// expects §5h's contaminated fraction of s = 2g,
//   theta_jv = (1 - rho) q_2g + rho f_v,   1 - theta_jv = (1 - rho)(1 - q_2g) + rho (1 - f_v)
// with f_v = (A_v + 1) / (T_v + 2) over every entry at row v and rho = m / 1000 given.  Its La / Lr are ambient::row_log's
// entries s = 2g at m, written over §5g's init and again after every M-step; where sample j has no dosage, cluster j is an
// ordinary §5g cluster.  The final scoring forms the pinned theta_jv in row_log's expressions and feeds it to §5g's pair_logs;
// every other (row, cluster) takes theta(A, T).  The same correctly rounded operations as §5g and §5h, so
// tests/cluster_pinned_oracle.py reproduces the result bit for bit.  With J = 0 (Pins{}) the scoring is §5g's, so
// vtx_cluster_cells scores with vtx_k_cl_score_pinned too.
//
// Kernels (the rest is §5g's: vtx_k_cl_count / scan / scatter / init / estep / mstep / final, and §5h's vtx_k_am_rowsum):
//   vtx_k_cp_pin             one thread per (active restart, used row, pinned sample): the pinned La / Lr where there is a dosage
//   vtx_k_cl_score_pinned    one warp per cell, lane l owning hypotheses l + 32j: the singlet / doublet log-likelihoods, with
//                            lane j < J forming the pinned theta where sample j has a dosage at the row
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/cluster_pinned_shim.cpp runs them serially on the
// CPU (tests/test_cluster_pinned_cpu.py).
#pragma once
#include <cstddef>
#include <cstdint>

#include "vtx_donors.cuh"
#include "vtx_clusters.cuh"
#include "vtx_ambient.cuh"

#if defined(__CUDACC__)
#define VTX_CP_HD __host__ __device__
#else
#define VTX_CP_HD
#endif

namespace vtx {
namespace cluster_pinned {

constexpr uint8_t kMissing = donors::kMissing;

// La / Lr of a pinned sample of dosage g at a row of sums A, T: §5h's table entries s = 2g at m
VTX_CP_HD inline void pinned_logs(const ambient::Fractions& fr, uint32_t m, uint64_t A, uint64_t T, uint32_t g, int32_t* la, int32_t* lr)
{
    // a constant s per branch: the device then reads the fractions straight from the kernel's parameters, not from a local copy
    switch (g) {
    case 0: *la = ambient::row_log(fr, m, A, T, 0, true); *lr = ambient::row_log(fr, m, A, T, 0, false); break;
    case 1: *la = ambient::row_log(fr, m, A, T, 2, true); *lr = ambient::row_log(fr, m, A, T, 2, false); break;
    default: *la = ambient::row_log(fr, m, A, T, 4, true); *lr = ambient::row_log(fr, m, A, T, 4, false); break;
    }
}

// theta and 1 - theta of a pinned sample of dosage g at a row of sums A, T: the fractions whose logs pinned_logs takes, in
// row_log's expressions
VTX_CP_HD inline void pinned_theta(const ambient::Fractions& fr, uint32_t m, uint64_t A, uint64_t T, uint32_t g, double* th, double* om)
{
    using namespace clusters;
    const double den = double(T + 2);
    const double f = d_div(double(A + 1), den), of = d_div(double(T - A + 1), den);
    const double rho = d_div(double(m), 1000.0), orho = d_div(double(1000 - m), 1000.0);
    const double q = g == 0 ? fr.q[0] : g == 1 ? fr.q[2] : fr.q[4], oq = g == 0 ? fr.oq[0] : g == 1 ? fr.oq[2] : fr.oq[4];
    *th = d_add(d_mul(orho, q), d_mul(rho, f));
    *om = d_add(d_mul(orho, oq), d_mul(rho, of));
}

// The pinned samples' side of the model: J samples, dos [n_rows][J], the row sums A_v / T_v, error rate (in fr) and m
struct Pins {
    uint32_t J, m;
    ambient::Fractions fr;
    const uint8_t* dos;
    const unsigned long long* rowA;
    const unsigned long long* rowT;
};

// theta and 1 - theta of canonical cluster j at row v for the final scoring (A, T [n_rows][K], canonical order)
VTX_CP_HD inline void cluster_theta(const Pins& p, uint32_t K, size_t v, uint32_t j, const int64_t* A, const int64_t* T, double* th, double* om)
{
    const uint32_t g = j < p.J ? p.dos[v * p.J + j] : kMissing;
    if (g != kMissing) pinned_theta(p.fr, p.m, p.rowA[v], p.rowT[v], g, th, om);
    else clusters::theta(A[v * K + j], T[v * K + j], th, om);
}

// ---- serial body (tests/cluster_pinned_shim.cpp): vtx_k_cl_score_pinned computes the same integers with one lane per cluster
// final scoring of cell c: ll[H], cnt[3] = variants, ref, alt (clusters::score_cell with cluster_theta)
inline void score_cell(const clusters::CellEntries& ce, uint32_t c, uint32_t K, const Pins& p, const int64_t* A, const int64_t* T,
                       int64_t* ll, uint64_t* cnt)
{
    clusters::score_cell_by(ce, c, K, [&](size_t v, uint32_t j, double* th, double* om) { cluster_theta(p, K, v, j, A, T, th, om); },
                            ll, cnt);
}

#ifdef __CUDACC__
constexpr int kCpThreads = 256;

// One thread per (active restart, used row, pinned sample): restart s's La / Lr of cluster j at row v, where j has a dosage
__global__ void __launch_bounds__(kCpThreads) vtx_k_cp_pin(clusters::Active act, Pins p, uint32_t n_used, const uint32_t* __restrict__ used_rows,
                                                           uint32_t K, uint64_t n_rows, int32_t* __restrict__ la, int32_t* __restrict__ lr)
{
    const uint64_t total = uint64_t(act.n) * n_used * p.J;
    for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < total; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint32_t j = uint32_t(i % p.J);
        const uint64_t v = used_rows[(i / p.J) % n_used];
        const uint32_t s = act.s[i / (uint64_t(p.J) * n_used)];
        const uint32_t g = p.dos[v * p.J + j];
        if (g == kMissing) continue;
        const size_t o = (size_t(s) * n_rows + v) * K + j;
        pinned_logs(p.fr, p.m, p.rowA[v], p.rowT[v], g, la + o, lr + o);
    }
}

// One warp per cell.  Lane k < K forms its cluster's theta and 1 - theta at the entry's row (cluster_theta); lane l then takes
// the two clusters of each of its hypotheses h = l + 32j (j < KH = ceil(H / 32)) by shuffle.
template <int KH>
__global__ void __launch_bounds__(kCpThreads) vtx_k_cl_score_pinned(clusters::CellEntries ce, uint32_t n_cols, uint32_t K, Pins p,
                                                                    const int64_t* __restrict__ A, const int64_t* __restrict__ T,
                                                                    int64_t* __restrict__ ll, uint64_t* __restrict__ cnt)
{
    using namespace clusters;
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
    for (uint32_t c = warp; c < n_cols; c += n_warps) {
        const uint32_t i0 = ce.start[c], i1 = ce.start[c + 1];
        int64_t acc[KH];
#pragma unroll
        for (int j = 0; j < KH; ++j) acc[j] = 0;
        uint64_t sum_r = 0, sum_a = 0;
        for (uint32_t base = i0; base < i1; base += 32) {
            const uint32_t i = base + lane;
            uint32_t v = 0, r = 0, a = 0;
            if (i < i1) { v = ce.row[i]; r = ce.r[i]; a = ce.a[i]; }
            const uint32_t n = min(32u, i1 - base);
            for (uint32_t e = 0; e < n; ++e) {
                const uint32_t ve = __shfl_sync(0xffffffffu, v, e), re = __shfl_sync(0xffffffffu, r, e), ae = __shfl_sync(0xffffffffu, a, e);
                double th = 0.5, om = 0.5;
                if (lane < K) cluster_theta(p, K, ve, lane, A, T, &th, &om);
#pragma unroll
                for (int j = 0; j < KH; ++j) {
                    const uint32_t d1 = pair[j] & 0xFF, d2 = pair[j] >> 8;
                    const double ti = __shfl_sync(0xffffffffu, th, d1), oi = __shfl_sync(0xffffffffu, om, d1);
                    const double tj = __shfl_sync(0xffffffffu, th, d2), oj = __shfl_sync(0xffffffffu, om, d2);
                    if (lane + 32u * j < H) {
                        int32_t la, lr;
                        pair_logs(ti, oi, tj, oj, &la, &lr);
                        acc[j] += int64_t(re) * lr + int64_t(ae) * la;
                    }
                }
            }
            sum_r += r; sum_a += a;
        }
        sum_r = warp_sum_u64(sum_r); sum_a = warp_sum_u64(sum_a);
        int64_t* out = ll + size_t(c) * H;
#pragma unroll
        for (int j = 0; j < KH; ++j)
            if (lane + 32u * j < H) out[lane + 32u * j] = acc[j];
        if (lane == 0) { cnt[3 * size_t(c)] = i1 - i0; cnt[3 * size_t(c) + 1] = sum_r; cnt[3 * size_t(c) + 2] = sum_a; }
    }
}
#endif   // __CUDACC__

}  // namespace cluster_pinned
}  // namespace vtx
