// vtx_clusters.cuh -- genotype-free clustering of pooled cells (vtx_cluster_cells, the CLI's --out-clusters): an allele-fraction
// EM over the finished result's REF / ALT counts, K clusters, R restarts, then the singlet / doublet scoring of --out-donors.
//
// Model (DESIGN.md §5g).  Only non-negative integers and correctly rounded IEEE double operations, so the result does not
// depend on entry order or launch shape and tests/cluster_oracle.py reproduces it bit for bit:
//   used row        at least kMinCells cells with r > 0 and at least kMinCells with a > 0
//   theta_kv        (A_kv + 2^16) / (T_kv + 2^17), and 1 - theta_kv as its own quotient (T_kv - A_kv + 2^16) / (T_kv + 2^17)
//   La_kv / Lr_kv   llrint(ll_log(theta) 2^24) / llrint(ll_log(1 - theta) 2^24), int32
//   E-step          LL_ck = sum r Lr + a La (int64), m_c = max_k LL_ck, E_ck = llrint(ll_exp((LL_ck - m_c) 2^-24) 2^40),
//                   W_ck = floor(E_ck 2^16 / sum_k E_ck); the restart's score is sum_c m_c
//   M-step          A_kv = sum_c W_ck a_cv, T_kv = sum_c W_ck (r_cv + a_cv), int64
// ll_log / ll_exp are built from +, -, x, / (the _rn intrinsics on the device, so that nothing is contracted into an FMA),
// frexp / ldexp and constants: libdevice's log / exp are not correctly rounded, and a 1-ulp difference that crosses an llrint
// boundary would make the result differ from the restatement.
//
// Kernels (one warp per item; lane k owns cluster k, K <= 32):
//   vtx_k_cl_count / scan_u32 / vtx_k_cl_scatter   the entries at used rows with r + a > 0, grouped by cell
//   vtx_k_cl_init      the restarts' first tables from splitmix64
//   vtx_k_cl_estep     one warp per (cell, active restart): W, the restart's "changed" flag and score
//   vtx_k_cl_mstep     one warp per (used row, active restart): the next La / Lr, no atomics
//   vtx_k_cl_final     one warp per row (every row), the best restart: A, T in the canonical cluster order
// The singlet / doublet scoring is vtx_cluster_pinned.cuh's vtx_k_cl_score_pinned with no pinned sample (J = 0).
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/cluster_shim.cpp runs them serially on the CPU
// (tests/test_clusters_cpu.py).  That build must not contract either (g++ does not on x86-64 without -mfma).
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "vtx_donors.cuh"

#if defined(__CUDACC__)
#define VTX_CL_HD __host__ __device__
#else
#define VTX_CL_HD
#endif

namespace vtx {
namespace clusters {

constexpr uint32_t kMinK = 2, kMaxK = 32;
constexpr uint32_t kMaxRestarts = 64;
constexpr uint32_t kMaxIters = 200;
constexpr uint32_t kMinCells = 4;                       // a used row has this many cells with REF and this many with ALT
constexpr int64_t kW = 65536;                           // 2^16: the weight scale (W_ck, A, T)
constexpr double kLogScale = 16777216.0;                // 2^24 (VTX_DONOR_LL_SCALE)
constexpr double kExpScale = 1099511627776.0;           // 2^40
constexpr double kExpFloor = -40.0;                     // ll_exp(x) = 0 below

VTX_CL_HD inline double d_add(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
VTX_CL_HD inline double d_sub(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
VTX_CL_HD inline double d_mul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
VTX_CL_HD inline double d_div(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// fdlibm's split of ln 2: e * kLn2Hi is exact for |e| < 2^20
constexpr double kLn2Hi = 6.93147180369123816490e-01, kLn2Lo = 1.90821492927058770002e-10;
constexpr double kInvLn2 = 1.44269504088896338700e+00, kSqrtHalf = 0.70710678118654752440;

// log(x) for x in (0, 1] (any positive normal x works): x = m 2^e with m in [sqrt(1/2), sqrt(2)), s = (m - 1) / (m + 1),
// log m = 2s + 2s z p(z), z = s^2, p the atanh series 1/3 + z/5 + ... + z^9/21 (|s| < 0.172: the tail is below 1e-17)
VTX_CL_HD inline double ll_log(double x)
{
    int e = 0;
    double m = frexp(x, &e);
    if (m < kSqrtHalf) { m = ldexp(m, 1); e -= 1; }
    const double s = d_div(d_sub(m, 1.0), d_add(m, 1.0));
    const double z = d_mul(s, s);
    double p = 1.0 / 21;
    p = d_add(1.0 / 19, d_mul(z, p));
    p = d_add(1.0 / 17, d_mul(z, p));
    p = d_add(1.0 / 15, d_mul(z, p));
    p = d_add(1.0 / 13, d_mul(z, p));
    p = d_add(1.0 / 11, d_mul(z, p));
    p = d_add(1.0 / 9, d_mul(z, p));
    p = d_add(1.0 / 7, d_mul(z, p));
    p = d_add(1.0 / 5, d_mul(z, p));
    p = d_add(1.0 / 3, d_mul(z, p));
    const double s2 = d_mul(2.0, s);
    const double lm = d_add(s2, d_mul(s2, d_mul(z, p)));
    const double de = double(e);
    return d_add(d_mul(de, kLn2Hi), d_add(d_mul(de, kLn2Lo), lm));
}

// exp(x) for x <= 0, 0 below -40: n = trunc(x / ln2 - 1/2), r = x - n ln2 (|r| < 0.35), exp r by its Taylor series to r^13 / 13!
// (the tail is below 1e-17); ll_exp(0) = 1 exactly
VTX_CL_HD inline double ll_exp(double x)
{
    if (x < kExpFloor) return 0.0;
    const int n = int(d_sub(d_mul(x, kInvLn2), 0.5));
    const double dn = double(n);
    const double r = d_sub(d_sub(x, d_mul(dn, kLn2Hi)), d_mul(dn, kLn2Lo));
    double p = 1.0 / 6227020800.0;
    p = d_add(1.0 / 479001600.0, d_mul(r, p));
    p = d_add(1.0 / 39916800.0, d_mul(r, p));
    p = d_add(1.0 / 3628800.0, d_mul(r, p));
    p = d_add(1.0 / 362880.0, d_mul(r, p));
    p = d_add(1.0 / 40320.0, d_mul(r, p));
    p = d_add(1.0 / 5040.0, d_mul(r, p));
    p = d_add(1.0 / 720.0, d_mul(r, p));
    p = d_add(1.0 / 120.0, d_mul(r, p));
    p = d_add(1.0 / 24.0, d_mul(r, p));
    p = d_add(1.0 / 6.0, d_mul(r, p));
    p = d_add(0.5, d_mul(r, p));
    p = d_add(1.0, d_mul(r, p));
    p = d_add(1.0, d_mul(r, p));
    return ldexp(p, n);
}

VTX_CL_HD inline uint64_t splitmix64(uint64_t x)
{
    uint64_t z = x + 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

VTX_CL_HD inline int32_t log_fixed(double x) { return int32_t(llrint(d_mul(ll_log(x), kLogScale))); }

// the first tables of restart s: theta = 0.05 + 0.9 u, u uniform from the matrix row v
VTX_CL_HD inline void init_logs(uint64_t seed, uint32_t s, uint32_t k, uint64_t v, int32_t* la, int32_t* lr)
{
    const uint64_t z = splitmix64(seed ^ (uint64_t(s) << 48) ^ (uint64_t(k) << 40) ^ v);
    const double u = d_mul(double(z >> 11), 1.0 / 9007199254740992.0);
    const double th = d_add(0.05, d_mul(0.9, u));
    *la = log_fixed(th);
    *lr = log_fixed(d_sub(1.0, th));
}

// theta and 1 - theta of sums A, T (x 2^16), each its own quotient of exactly representable integers
VTX_CL_HD inline void theta(int64_t a, int64_t t, double* th, double* om)
{
    const double den = double(t + 2 * kW);
    *th = d_div(double(a + kW), den);
    *om = d_div(double(t - a + kW), den);
}

// the M-step's tables of one (cluster, row)
VTX_CL_HD inline void row_logs(int64_t a, int64_t t, int32_t* la, int32_t* lr)
{
    double th, om;
    theta(a, t, &th, &om);
    *la = log_fixed(th);
    *lr = log_fixed(om);
}

// the scoring's tables of hypothesis (i, j) (a singlet is (k, k): (x + x) / 2 = x exactly)
VTX_CL_HD inline void pair_logs(double th_i, double om_i, double th_j, double om_j, int32_t* la, int32_t* lr)
{
    *la = log_fixed(d_mul(d_add(th_i, th_j), 0.5));
    *lr = log_fixed(d_mul(d_add(om_i, om_j), 0.5));
}

// E_ck of a cluster whose LL lies d = LL - m_c <= 0 below the cell's maximum (x 2^40; the maximum gets 2^40)
VTX_CL_HD inline uint64_t e_weight(int64_t d)
{
    return uint64_t(llrint(d_mul(ll_exp(d_mul(double(d), 1.0 / kLogScale)), kExpScale)));
}

VTX_CL_HD inline uint32_t w_weight(uint64_t e, uint64_t sum_e) { return uint32_t((e << 16) / sum_e); }

// An entry (row, col, r, a) of the input in cell-major order, after the used-row filter
struct CellEntries {
    const uint32_t* start;      // [n_cols + 1]
    const uint32_t* row;        // [m]
    const uint32_t* r;
    const uint32_t* a;
};

// ---- serial bodies (tests/cluster_shim.cpp): the kernels below compute the same integers with one lane per cluster -------
// E-step of cell c against one restart's tables la / lr [n_rows][K]: w[K]; returns m_c
inline int64_t estep_cell(const CellEntries& ce, uint32_t c, uint32_t K, const int32_t* la, const int32_t* lr, uint32_t* w)
{
    int64_t ll[kMaxK] = {};
    for (uint32_t i = ce.start[c]; i < ce.start[c + 1]; ++i)
        for (uint32_t k = 0; k < K; ++k)
            ll[k] += int64_t(ce.r[i]) * lr[size_t(ce.row[i]) * K + k] + int64_t(ce.a[i]) * la[size_t(ce.row[i]) * K + k];
    int64_t m = ll[0];
    for (uint32_t k = 1; k < K; ++k) m = ll[k] > m ? ll[k] : m;
    uint64_t e[kMaxK], sum = 0;
    for (uint32_t k = 0; k < K; ++k) sum += e[k] = e_weight(ll[k] - m);
    for (uint32_t k = 0; k < K; ++k) w[k] = w_weight(e[k], sum);
    return m;
}

// M-step sums of row v over its entries [i0, i1) of the row-major input; w [n_cols][K], clusters map[j] for j < K
inline void mstep_row(const uint32_t* col, const uint32_t* r, const uint32_t* a, uint32_t i0, uint32_t i1, const uint32_t* w,
                      uint32_t K, const uint32_t* map, int64_t* sum_a, int64_t* sum_t)
{
    for (uint32_t j = 0; j < K; ++j) { sum_a[j] = 0; sum_t[j] = 0; }
    for (uint32_t i = i0; i < i1; ++i)
        for (uint32_t j = 0; j < K; ++j) {
            const int64_t x = w[size_t(col[i]) * K + map[j]];
            sum_a[j] += x * a[i];
            sum_t[j] += x * (int64_t(r[i]) + a[i]);
        }
}

// final scoring of cell c: ll[H], cnt[3] = variants, ref, alt; theta_of(v, k, &th, &om) gives canonical cluster k's theta and
// 1 - theta at row v (vtx_cluster_pinned.cuh's score_cell passes its pinned theta)
template <typename ThetaOf>
inline void score_cell_by(const CellEntries& ce, uint32_t c, uint32_t K, ThetaOf theta_of, int64_t* ll, uint64_t* cnt)
{
    const uint32_t H = donors::n_hyp(K);
    for (uint32_t h = 0; h < H; ++h) ll[h] = 0;
    cnt[0] = cnt[1] = cnt[2] = 0;
    for (uint32_t i = ce.start[c]; i < ce.start[c + 1]; ++i) {
        const size_t v = ce.row[i];
        for (uint32_t h = 0; h < H; ++h) {
            uint32_t d1, d2;
            donors::hyp_donors(h, K, &d1, &d2);
            double ti, oi, tj, oj;
            theta_of(v, d1, &ti, &oi);
            theta_of(v, d2, &tj, &oj);
            int32_t la, lr;
            pair_logs(ti, oi, tj, oj, &la, &lr);
            ll[h] += int64_t(ce.r[i]) * lr + int64_t(ce.a[i]) * la;
        }
        cnt[0] += 1; cnt[1] += ce.r[i]; cnt[2] += ce.a[i];
    }
}

// final scoring of cell c from A, T [n_rows][K] (canonical order): what vtx_k_cl_score_pinned computes with no pinned sample
inline void score_cell(const CellEntries& ce, uint32_t c, uint32_t K, const int64_t* A, const int64_t* T, int64_t* ll, uint64_t* cnt)
{
    score_cell_by(ce, c, K, [&](size_t v, uint32_t k, double* th, double* om) { theta(A[v * K + k], T[v * K + k], th, om); }, ll, cnt);
}

#ifdef __CUDACC__
constexpr int kClThreads = 256;

struct Active {                 // the restarts a launch covers
    uint32_t n;
    uint8_t s[kMaxRestarts];
};

struct Perm { uint8_t k[kMaxK]; };      // canonical cluster j -> EM cluster k[j]

__device__ __forceinline__ bool cl_keep(const uint8_t* used, uint32_t row, uint32_t r, uint32_t a)
{
    return used[row] && uint64_t(r) + a > 0;
}

// the kept entries per cell
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_count(uint32_t n, const uint32_t* __restrict__ row, const uint32_t* __restrict__ col,
                                                             const uint32_t* __restrict__ r, const uint32_t* __restrict__ a,
                                                             const uint8_t* __restrict__ used, uint32_t* __restrict__ cell_count)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (cl_keep(used, row[i], r[i], a[i])) atomicAdd(&cell_count[col[i]], 1u);
}

// the kept entries grouped by cell (any order inside a cell: every sum over them is an integer sum)
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_scatter(uint32_t n, const uint32_t* __restrict__ row, const uint32_t* __restrict__ col,
                                                               const uint32_t* __restrict__ r, const uint32_t* __restrict__ a,
                                                               const uint8_t* __restrict__ used, const uint32_t* __restrict__ cell_start,
                                                               uint32_t* __restrict__ cell_fill, uint32_t* __restrict__ c_row,
                                                               uint32_t* __restrict__ c_r, uint32_t* __restrict__ c_a)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!cl_keep(used, row[i], r[i], a[i])) continue;
        const uint32_t c = col[i], q = cell_start[c] + atomicAdd(&cell_fill[c], 1u);
        c_row[q] = row[i]; c_r[q] = r[i]; c_a[q] = a[i];
    }
}

// one thread per (restart, used row, cluster)
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_init(uint64_t seed, uint32_t R, uint32_t K, uint32_t n_used,
                                                            const uint32_t* __restrict__ used_rows, uint64_t n_rows,
                                                            int32_t* __restrict__ la, int32_t* __restrict__ lr)
{
    const uint64_t total = uint64_t(R) * n_used * K;
    for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < total; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint32_t k = uint32_t(i % K);
        const uint64_t vi = (i / K) % n_used;
        const uint32_t s = uint32_t(i / (uint64_t(K) * n_used));
        const uint64_t v = used_rows[vi];
        const size_t o = (size_t(s) * n_rows + v) * K + k;
        init_logs(seed, s, k, v, la + o, lr + o);
    }
}

__device__ __forceinline__ int64_t warp_max_i64(int64_t x)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) { const int64_t y = __shfl_xor_sync(0xffffffffu, x, o); x = y > x ? y : x; }
    return x;
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t x)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// One warp per (cell, active restart), restart-major so that the warps of one restart share its tables in L2.  The lanes
// load 32 entries of the cell at once and hand them round with shuffles; lane k < K adds r Lr_kv + a La_kv.
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_estep(Active act, CellEntries ce, uint32_t n_cols, uint64_t n_rows, uint32_t K,
                                                             const int32_t* __restrict__ la, const int32_t* __restrict__ lr,
                                                             uint32_t* __restrict__ w, uint32_t* __restrict__ changed,
                                                             unsigned long long* __restrict__ score)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    const uint64_t total = uint64_t(act.n) * n_cols;
    for (uint64_t wi = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; wi < total; wi += n_warps) {
        const uint32_t s = act.s[wi / n_cols], c = uint32_t(wi % n_cols);
        const int32_t* tla = la + size_t(s) * n_rows * K;
        const int32_t* tlr = lr + size_t(s) * n_rows * K;
        const uint32_t i0 = ce.start[c], i1 = ce.start[c + 1];
        int64_t acc = 0;
        for (uint32_t base = i0; base < i1; base += 32) {
            const uint32_t i = base + lane;
            uint32_t v = 0, r = 0, a = 0;
            if (i < i1) { v = ce.row[i]; r = ce.r[i]; a = ce.a[i]; }
            const uint32_t cnt = min(32u, i1 - base);
            for (uint32_t j = 0; j < cnt; ++j) {
                const uint32_t vj = __shfl_sync(0xffffffffu, v, j), rj = __shfl_sync(0xffffffffu, r, j), aj = __shfl_sync(0xffffffffu, a, j);
                if (lane < K) acc += int64_t(rj) * tlr[size_t(vj) * K + lane] + int64_t(aj) * tla[size_t(vj) * K + lane];
            }
        }
        const int64_t m = warp_max_i64(lane < K ? acc : INT64_MIN);
        const uint64_t e = lane < K ? e_weight(acc - m) : 0;
        const uint64_t sum = warp_sum_u64(e);
        bool diff = false;
        if (lane < K) {
            const uint32_t wn = w_weight(e, sum);
            uint32_t* p = w + (size_t(s) * n_cols + c) * K + lane;
            diff = *p != wn;
            if (diff) *p = wn;
        }
        if (lane == 0) atomicAdd(&score[s], (unsigned long long)m);
        if (__any_sync(0xffffffffu, diff) && lane == 0) changed[s] = 1;
    }
}

// the sums of one row (entries [i0, i1) of the row-major input) for lane j < K, which owns EM cluster k
__device__ __forceinline__ void row_sums(const uint32_t* __restrict__ col, const uint32_t* __restrict__ r, const uint32_t* __restrict__ a,
                                         uint32_t i0, uint32_t i1, const uint32_t* __restrict__ w, uint32_t K, uint32_t lane, uint32_t k,
                                         int64_t* sum_a, int64_t* sum_t)
{
    int64_t sa = 0, st = 0;
    for (uint32_t base = i0; base < i1; base += 32) {
        const uint32_t i = base + lane;
        uint32_t c = 0, ri = 0, ai = 0;
        if (i < i1) { c = col[i]; ri = r[i]; ai = a[i]; }
        const uint32_t cnt = min(32u, i1 - base);
        for (uint32_t j = 0; j < cnt; ++j) {
            const uint32_t cj = __shfl_sync(0xffffffffu, c, j), rj = __shfl_sync(0xffffffffu, ri, j), aj = __shfl_sync(0xffffffffu, ai, j);
            if (lane < K) {
                const int64_t x = w[size_t(cj) * K + k];
                sa += x * aj;
                st += x * (int64_t(rj) + aj);
            }
        }
    }
    *sum_a = sa; *sum_t = st;
}

// One warp per (used row, active restart): the next tables
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_mstep(Active act, uint32_t n_used, const uint32_t* __restrict__ used_rows,
                                                             const uint32_t* __restrict__ row_start, const uint32_t* __restrict__ col,
                                                             const uint32_t* __restrict__ r, const uint32_t* __restrict__ a,
                                                             const uint32_t* __restrict__ w, uint32_t n_cols, uint64_t n_rows, uint32_t K,
                                                             int32_t* __restrict__ la, int32_t* __restrict__ lr)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    const uint64_t total = uint64_t(act.n) * n_used;
    for (uint64_t wi = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; wi < total; wi += n_warps) {
        const uint32_t s = act.s[wi / n_used], v = used_rows[wi % n_used];
        int64_t sa, st;
        row_sums(col, r, a, row_start[v], row_start[v + 1], w + size_t(s) * n_cols * K, K, lane, lane, &sa, &st);
        if (lane < K) {
            const size_t o = (size_t(s) * n_rows + v) * K + lane;
            row_logs(sa, st, la + o, lr + o);
        }
    }
}

// One warp per row, every row: the best restart's A, T, lane j holding canonical cluster j
__global__ void __launch_bounds__(kClThreads) vtx_k_cl_final(Perm perm, uint64_t n_rows, const uint32_t* __restrict__ row_start,
                                                             const uint32_t* __restrict__ col, const uint32_t* __restrict__ r,
                                                             const uint32_t* __restrict__ a, const uint32_t* __restrict__ w, uint32_t K,
                                                             int64_t* __restrict__ A, int64_t* __restrict__ T)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = (uint64_t(gridDim.x) * blockDim.x) >> 5;
    const uint32_t k = lane < K ? perm.k[lane] : 0;
    for (uint64_t v = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; v < n_rows; v += n_warps) {
        int64_t sa, st;
        row_sums(col, r, a, row_start[v], row_start[v + 1], w, K, lane, k, &sa, &st);
        if (lane < K) { A[v * K + lane] = sa; T[v * K + lane] = st; }
    }
}
#endif   // __CUDACC__

}  // namespace clusters
}  // namespace vtx
