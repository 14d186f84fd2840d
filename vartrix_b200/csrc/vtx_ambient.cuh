// vtx_ambient.cuh -- genotype demultiplexing against allele fractions contaminated by ambient RNA (vtx_donors_ambient, the CLI's
// --ambient-rna): §5f's donor model with the pool's own ALT fraction mixed into every hypothesis, and the estimate of the mix.
//
// Model (DESIGN.md §5h).  §5f's donors, hypotheses, usable rows, counts, call rule and T = 5 nats; at row v a hypothesis of
// index s expects
//   q_vs = (1 - rho) q_s + rho f_v,   1 - q_vs = (1 - rho)(1 - q_s) + rho (1 - f_v)
// with q_s §5f's five fractions (make_tables' expressions), f_v = (A_v + 1) / (T_v + 2) and 1 - f_v = (T_v - A_v + 1) / (T_v + 2)
// (A_v / T_v the sums of a / r + a over every entry at row v), rho = m / 1000 and 1 - rho = (1000 - m) / 1000 for m in 0..500.
// La_vs / Lr_vs = log_fixed(q_vs) / log_fixed(1 - q_vs): §5g's ll_log x 2^24, llrint, int32.  Every + x / is a correctly rounded
// double operation (d_add / d_mul / d_div: the _rn intrinsics on the device), so tests/ambient_oracle.py reproduces the tables
// bit for bit, and everything after them is int64 addition.
// The estimate: J(m) = sum over cells with variants of max_h LL_ch(m) on m = 0, 10, ..., 500, then every m within 9 of the
// coarse winner; the largest J wins (ties: the smallest m).
//
// Kernels (the by-cell index is §5g's vtx_k_cl_count / scan_u32 / vtx_k_cl_scatter with `used` = usable rows):
//   vtx_k_am_rowsum   one thread per entry: A_v, T_v (integer atomics)
//   vtx_k_am_tables   one thread per (m of the batch, touched row): La, Lr of the five fractions
//   vtx_k_am_score    one warp per (m of the batch, cell), lane l owns hypotheses l + 32j: J(m) and the cell's call by integer
//                     atomics; with one m, the cell's log-likelihoods and counts
// Only the usable rows that some kept entry touches get tables ("touched" rows, compacted): a donor VCF may have millions.
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/ambient_shim.cpp runs them serially on the CPU
// (tests/test_ambient_cpu.py).
#pragma once
#include <cstddef>
#include <cstdint>

#include "vtx_donors.cuh"
#include "vtx_clusters.cuh"

#if defined(__CUDACC__)
#define VTX_AM_HD __host__ __device__
#else
#define VTX_AM_HD
#endif

namespace vtx {
namespace ambient {

constexpr int32_t kMaxPermille = 500;
constexpr uint32_t kCoarseStep = 10;                    // the coarse grid m = 0, 10, ..., 500
constexpr uint32_t kFineReach = 9;                      // the fine pass: every m within this of the coarse winner
constexpr uint32_t kMaxBatch = 64;                      // m values per launch
constexpr uint64_t kMaxRowDepth = (1ull << 53) - 3;     // T_v + 2 stays below 2^53

struct Fractions {              // §5f's q_s and 1 - q_s, in make_tables' expressions (host)
    double q[5], oq[5];
};

inline Fractions fractions(double e)
{
    Fractions f;
    const double q[5] = { e, (e + 0.5) / 2, 0.5, (1.5 - e) / 2, 1 - e };
    for (int s = 0; s < 5; ++s) { f.q[s] = q[s]; f.oq[s] = 1 - q[s]; }
    return f;
}

// log_fixed of (1 - rho) q + rho f: La_vs with q = q_s, f = f_v; Lr_vs with their complements
VTX_AM_HD inline int32_t mix_log(double q, double rho, double orho, double f)
{
    using namespace clusters;
    return log_fixed(d_add(d_mul(orho, q), d_mul(rho, f)));
}

// the tables of one row at m: out[2 s] = La_vs, out[2 s + 1] = Lr_vs
VTX_AM_HD inline void row_logs(const Fractions& fr, uint32_t m, uint64_t A, uint64_t T, int32_t* out)
{
    using namespace clusters;
    const double den = double(T + 2);
    const double f = d_div(double(A + 1), den), of = d_div(double(T - A + 1), den);
    const double rho = d_div(double(m), 1000.0), orho = d_div(double(1000 - m), 1000.0);
    for (int s = 0; s < 5; ++s) {
        out[2 * s] = mix_log(fr.q[s], rho, orho, f);
        out[2 * s + 1] = mix_log(fr.oq[s], rho, orho, of);
    }
}

// one entry of row_logs: La_vs (alt) or Lr_vs
VTX_AM_HD inline int32_t row_log(const Fractions& fr, uint32_t m, uint64_t A, uint64_t T, int s, bool alt)
{
    using namespace clusters;
    const double den = double(T + 2);
    const double f = alt ? d_div(double(A + 1), den) : d_div(double(T - A + 1), den);
    return mix_log(alt ? fr.q[s] : fr.oq[s], d_div(double(m), 1000.0), d_div(double(1000 - m), 1000.0), f);
}

// ---- serial body (tests/ambient_shim.cpp): vtx_k_am_score computes the same integers with one lane per hypothesis ----------
// cell c against one m's tables tab [touched][5][2]; tix maps a row to its touched index, dos [touched][D]: ll[H], cnt[3]
inline void score_cell(const clusters::CellEntries& ce, uint32_t c, uint32_t D, const uint32_t* tix, const uint8_t* dos,
                       const int32_t* tab, int64_t* ll, uint64_t* cnt)
{
    const uint32_t H = donors::n_hyp(D);
    for (uint32_t h = 0; h < H; ++h) ll[h] = 0;
    cnt[0] = cnt[1] = cnt[2] = 0;
    for (uint32_t i = ce.start[c]; i < ce.start[c + 1]; ++i) {
        const size_t t = tix[ce.row[i]];
        const uint8_t* g = dos + t * D;
        for (uint32_t h = 0; h < H; ++h) {
            uint32_t d1, d2;
            donors::hyp_donors(h, D, &d1, &d2);
            const int32_t* x = tab + (t * 5 + donors::s_index(g[d1], g[d2])) * 2;
            ll[h] += int64_t(ce.r[i]) * x[1] + int64_t(ce.a[i]) * x[0];
        }
        cnt[0] += 1; cnt[1] += ce.r[i]; cnt[2] += ce.a[i];
    }
}

#ifdef __CUDACC__
constexpr int kAmThreads = 256;

struct Batch {                  // the m values a launch covers
    uint32_t n;
    uint16_t m[kMaxBatch];
};

__global__ void __launch_bounds__(kAmThreads) vtx_k_am_rowsum(uint32_t n, const uint32_t* __restrict__ row, const uint32_t* __restrict__ r,
                                                              const uint32_t* __restrict__ a, unsigned long long* __restrict__ A,
                                                              unsigned long long* __restrict__ T)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        atomicAdd(&A[row[i]], (unsigned long long)a[i]);
        atomicAdd(&T[row[i]], (unsigned long long)r[i] + a[i]);
    }
}

// tab [b][touched][5][2]
__global__ void __launch_bounds__(kAmThreads) vtx_k_am_tables(Batch bt, Fractions fr, uint32_t n_t, const uint32_t* __restrict__ touched,
                                                              const unsigned long long* __restrict__ A, const unsigned long long* __restrict__ T,
                                                              int32_t* __restrict__ tab)
{
    const uint64_t total = uint64_t(bt.n) * n_t;
    for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < total; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint32_t v = touched[i % n_t];
        row_logs(fr, bt.m[i / n_t], A[v], T[v], tab + i * 10);
    }
}

// One warp per (m of the batch, cell), m-major so that the warps of one m share its tables in L2.  The lanes load 32 entries of
// the cell at once and hand them round with shuffles; lane d < D loads donor d's dosage and two ballots hand every lane all D
// (vtx_k_donor_ll's pattern).  The warp reduces the best singlet (ties: the lowest donor), the best other singlet and the best
// doublet, then adds max_h LL to J[b] and the call to calls[b][.].  ll / cnt (when not null, with one m) get the cell's rows.
template <int KH>
__global__ void __launch_bounds__(kAmThreads) vtx_k_am_score(Batch bt, clusters::CellEntries ce, uint32_t n_cols, uint32_t D,
                                                             const uint32_t* __restrict__ tix, const uint8_t* __restrict__ dos,
                                                             const int32_t* __restrict__ tab, uint32_t n_t,
                                                             unsigned long long* __restrict__ J, unsigned long long* __restrict__ calls,
                                                             int64_t* __restrict__ ll, uint64_t* __restrict__ cnt)
{
    using clusters::warp_max_i64;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    const uint32_t H = donors::n_hyp(D);
    uint32_t pair[KH];
#pragma unroll
    for (int k = 0; k < KH; ++k) {
        uint32_t d1 = 0, d2 = 0;
        if (lane + 32u * k < H) donors::hyp_donors(lane + 32u * k, D, &d1, &d2);
        pair[k] = d1 | d2 << 8;
    }
    const uint64_t total = uint64_t(bt.n) * n_cols;
    for (uint64_t wi = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; wi < total; wi += n_warps) {
        const uint32_t b = uint32_t(wi / n_cols), c = uint32_t(wi % n_cols);
        const int2* tb = reinterpret_cast<const int2*>(tab) + size_t(b) * n_t * 5;
        const uint32_t i0 = ce.start[c], i1 = ce.start[c + 1];
        int64_t acc[KH];
#pragma unroll
        for (int k = 0; k < KH; ++k) acc[k] = 0;
        uint64_t sum_r = 0, sum_a = 0;
        for (uint32_t base = i0; base < i1; base += 32) {
            const uint32_t i = base + lane;
            uint32_t t = 0, r = 0, a = 0;
            if (i < i1) { t = tix[ce.row[i]]; r = ce.r[i]; a = ce.a[i]; }
            const uint32_t n = min(32u, i1 - base);
            for (uint32_t e = 0; e < n; ++e) {
                const uint32_t te = __shfl_sync(0xffffffffu, t, e), re = __shfl_sync(0xffffffffu, r, e), ae = __shfl_sync(0xffffffffu, a, e);
                const uint32_t g = lane < D ? dos[size_t(te) * D + lane] : 0u;
                const uint32_t b0 = __ballot_sync(0xffffffffu, g & 1u), b1 = __ballot_sync(0xffffffffu, g & 2u);
                int64_t v[5];
#pragma unroll
                for (int s = 0; s < 5; ++s) {
                    const int2 x = tb[size_t(te) * 5 + s];
                    v[s] = int64_t(re) * x.y + int64_t(ae) * x.x;
                }
#pragma unroll
                for (int k = 0; k < KH; ++k) {
                    const uint32_t d1 = pair[k] & 0xFF, d2 = pair[k] >> 8;
                    const uint32_t s = donors::s_index((b0 >> d1 & 1u) | (b1 >> d1 & 1u) << 1, (b0 >> d2 & 1u) | (b1 >> d2 & 1u) << 1);
                    int64_t x = v[0];                   // selects, not an indexed (local-memory) array
                    x = s == 1 ? v[1] : x; x = s == 2 ? v[2] : x; x = s == 3 ? v[3] : x; x = s == 4 ? v[4] : x;
                    acc[k] += x;
                }
            }
            sum_r += r; sum_a += a;
        }
        const int64_t best = warp_max_i64(lane < D ? acc[0] : INT64_MIN);
        const uint32_t first = __ffs(__ballot_sync(0xffffffffu, lane < D && acc[0] == best)) - 1;
        const int64_t second = warp_max_i64(lane < D && lane != first ? acc[0] : INT64_MIN);
        int64_t pm = INT64_MIN;
#pragma unroll
        for (int k = 0; k < KH; ++k) {
            const uint32_t h = lane + 32u * k;
            if (h >= D && h < H) pm = acc[k] > pm ? acc[k] : pm;
        }
        const int64_t pbest = warp_max_i64(pm);
        if (lane == 0) {
            atomicAdd(&calls[3 * size_t(b) + donors::call_of(i1 - i0, best, second, pbest)], 1ull);
            if (i1 > i0) atomicAdd(&J[b], (unsigned long long)(best > pbest ? best : pbest));
        }
        if (ll) {
            sum_r = clusters::warp_sum_u64(sum_r); sum_a = clusters::warp_sum_u64(sum_a);
            int64_t* out = ll + size_t(c) * H;
#pragma unroll
            for (int k = 0; k < KH; ++k)
                if (lane + 32u * k < H) out[lane + 32u * k] = acc[k];
            if (lane == 0) { cnt[3 * size_t(c)] = i1 - i0; cnt[3 * size_t(c) + 1] = sum_r; cnt[3 * size_t(c) + 2] = sum_a; }
        }
    }
}
#endif   // __CUDACC__

}  // namespace ambient
}  // namespace vtx
