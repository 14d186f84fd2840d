// vtx_donors.cuh -- per-cell donor log-likelihoods from the donors' VCF genotypes (vtx_set_donors / vtx_donor_ll_get, the
// CLI's --out-donors): genotype demultiplexing of pooled cells.
//
// Model (DESIGN.md §5f).  D donors, H = D + D(D-1)/2 hypotheses: h < D the singlet of donor h, then the doublets (0,1), (0,2),
// ..., (D-2, D-1).  At row v a hypothesis has the index s = g_d1 + g_d2 (a singlet d is the pair (d, d): s = 2 g_d), g the ALT
// dosage 0..2, and the expected ALT fraction q_s = {e, (e + 0.5)/2, 0.5, (1.5 - e)/2, 1 - e}.  A cell slot with r REF and a ALT
// molecules (ccnt after vtx_k_umi_collapse: the counts the matrix is built from) adds r Lr[s] + a La[s] to hypothesis h, where
// Lr[s] = llrint(log(1 - q_s) 2^24) and La[s] = llrint(log(q_s) 2^24) are computed once on the host.  Everything after those
// ten constants is int64 addition, so the result does not depend on summation order, shard size or device count.
//
// A slot takes part ("qualifies") when its column is a listed barcode, its row is in the table and usable (every donor has a
// dosage there) and r + a > 0.  Per submit, after the UMI collapse:
//   vtx_k_donor_count    qualifying slots per column (and rows outside the table, which are skipped and reported)
//   scan_u32             column starts
//   vtx_k_donor_scatter  the qualifying slot indices grouped by column (any order inside a column: the sums are integers)
//   vtx_k_donor_ll       one warp per column: lane owns h = lane + 32k, sums in registers, adds its row of the accumulator
// One warp owns a column within a submit and submits are stream-ordered, so the accumulator needs no atomics.
//
// The per-item bodies are __host__ __device__ (plain C++ without nvcc): tests/donor_shim.cpp runs them serially on the CPU
// (tests/test_donors_cpu.py).
#pragma once
#include <cstddef>
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define VTX_DN_HD __host__ __device__
#else
#define VTX_DN_HD
#endif

namespace vtx {
namespace donors {

constexpr uint32_t kMaxDonors = 32;
constexpr uint32_t kMinDonors = 2;
constexpr uint8_t kMissing = 0xFF;                      // VTX_GT_MISSING
constexpr double kScale = 16777216.0;                   // VTX_DONOR_LL_SCALE = 2^24
constexpr uint32_t kNoCol = 0xFFFFFFFFu;

VTX_DN_HD inline uint32_t n_hyp(uint32_t d) { return d + d * (d - 1) / 2; }

// hypothesis h of D donors -> its two donors (a singlet is (h, h)); doublets in the order (0,1), (0,2), ..., (D-2, D-1)
VTX_DN_HD inline void hyp_donors(uint32_t h, uint32_t d, uint32_t* d1, uint32_t* d2)
{
    if (h < d) { *d1 = *d2 = h; return; }
    uint32_t rem = h - d, a = 0;
    while (rem >= d - 1 - a) { rem -= d - 1 - a; ++a; }
    *d1 = a; *d2 = a + 1 + rem;
}

// the index s of a hypothesis whose donors have dosages g1, g2 (a singlet passes its dosage twice)
VTX_DN_HD inline uint32_t s_index(uint32_t g1, uint32_t g2) { return g1 + g2; }

// the log-likelihood tables, x 2^24
struct Tables {
    int64_t lr[5];      // log(1 - q_s)
    int64_t la[5];      // log(q_s)
};

// what one (cell, row) pair with r REF and a ALT molecules adds to a hypothesis of index s
VTX_DN_HD inline int64_t contribution(const Tables& t, uint32_t s, uint32_t r, uint32_t a)
{
    return int64_t(r) * t.lr[s] + int64_t(a) * t.la[s];
}

VTX_DN_HD inline bool row_usable(const uint8_t* dosage_row, uint32_t d)
{
    for (uint32_t k = 0; k < d; ++k)
        if (dosage_row[k] > 2) return false;
    return true;
}

struct Inputs {
    const uint32_t* cslot_col;      // [slot] column or kNoCol
    const uint32_t* cslot_locus;    // [slot] locus of the shard
    const uint32_t* locus_row;      // [n_loci]
    const uint32_t* ccnt;           // [slot][4] REF, ALT, UNKNOWN calls of the cell slot
    const uint8_t* dosage;          // [n_rows][n_donors]
    const uint8_t* usable;          // [n_rows]
    uint64_t n_rows;
    uint32_t n_cols, n_donors, n_hyp;
    Tables t;
};

// the row of slot q when it qualifies, else -1 (its column is not a listed barcode, its row is outside the table or not
// usable, or it has no REF or ALT molecule)
VTX_DN_HD inline int64_t qualifying_row(const Inputs& in, uint32_t q)
{
    const uint32_t col = in.cslot_col[q];
    if (col >= in.n_cols) return -1;
    const uint32_t row = in.locus_row[in.cslot_locus[q]];
    if (row >= in.n_rows || !in.usable[row]) return -1;
    if (uint64_t(in.ccnt[4 * size_t(q)]) + in.ccnt[4 * size_t(q) + 1] == 0) return -1;
    return int64_t(row);
}

// one qualifying slot of a column, serially over every hypothesis: ll[h] += ..., cnt = {variants, ref, alt}
VTX_DN_HD inline void add_slot(const Inputs& in, uint32_t q, int64_t* ll, uint64_t* cnt)
{
    const uint32_t row = in.locus_row[in.cslot_locus[q]];
    const uint32_t r = in.ccnt[4 * size_t(q)], a = in.ccnt[4 * size_t(q) + 1];
    const uint8_t* g = in.dosage + size_t(row) * in.n_donors;
    for (uint32_t h = 0; h < in.n_hyp; ++h) {
        uint32_t d1, d2;
        hyp_donors(h, in.n_donors, &d1, &d2);
        ll[h] += contribution(in.t, s_index(g[d1], g[d2]), r, a);
    }
    cnt[0] += 1; cnt[1] += r; cnt[2] += a;
}

// the call of a cell with `variants` rows from its best singlet, best other singlet and best doublet log-likelihoods:
// 0 singlet, 1 doublet, 2 unassigned, with the threshold T = 5 nats in the integer scale
VTX_DN_HD inline uint32_t call_of(uint64_t variants, int64_t best, int64_t second, int64_t pair)
{
    const int64_t T = 5 * int64_t(kScale);
    return variants == 0 ? 2u : pair - best >= T ? 1u : best - second >= T ? 0u : 2u;
}

// Lr / La from the error rate: host code only (vtx_set_donors), in the exact double expressions of the model
inline Tables make_tables(double e)
{
    const double q[5] = { e, (e + 0.5) / 2, 0.5, (1.5 - e) / 2, 1 - e };
    Tables t;
    for (int s = 0; s < 5; ++s) { t.lr[s] = llrint(log(1 - q[s]) * kScale); t.la[s] = llrint(log(q[s]) * kScale); }
    return t;
}

#ifdef __CUDACC__
constexpr int kDonorThreads = 256;

// qualifying slots per column; every thread below n_loci also checks that locus's row against the table
__global__ void __launch_bounds__(kDonorThreads) vtx_k_donor_count(Inputs in, uint32_t n_slots_ub, const uint32_t* __restrict__ n_slots,
                                                                   uint32_t n_loci, uint32_t* __restrict__ col_count,
                                                                   unsigned long long* __restrict__ bad_rows)
{
    const uint32_t ns = n_slots ? *n_slots : 0u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_slots_ub || i < n_loci; i += gridDim.x * blockDim.x) {
        if (i < n_loci && in.locus_row[i] >= in.n_rows) atomicAdd(bad_rows, 1ull);
        if (i < ns && qualifying_row(in, i) >= 0) atomicAdd(&col_count[in.cslot_col[i]], 1u);
    }
}

// the qualifying slot indices grouped by column: list[col_start[c] ...) (col_fill zeroed before)
__global__ void __launch_bounds__(kDonorThreads) vtx_k_donor_scatter(Inputs in, uint32_t n_slots_ub, const uint32_t* __restrict__ n_slots,
                                                                     const uint32_t* __restrict__ col_start, uint32_t* __restrict__ col_fill,
                                                                     uint32_t* __restrict__ list)
{
    const uint32_t ns = min(*n_slots, n_slots_ub);
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < ns; q += gridDim.x * blockDim.x) {
        if (qualifying_row(in, q) < 0) continue;
        const uint32_t c = in.cslot_col[q];
        list[col_start[c] + atomicAdd(&col_fill[c], 1u)] = q;
    }
}

// One warp per column (grid-stride).  Lane d < D loads the row's dosage of donor d; two ballots hand every lane the dosages of
// all D donors (bit d of b0 / b1 = bit 0 / 1 of g_d).  Lane l owns hypotheses h = l + 32k, k < KH (KH = ceil(H / 32)).
template <int KH>
__global__ void __launch_bounds__(kDonorThreads) vtx_k_donor_ll(Inputs in, const uint32_t* __restrict__ col_start,
                                                                const uint32_t* __restrict__ list, int64_t* __restrict__ ll,
                                                                uint64_t* __restrict__ cnt)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t H = in.n_hyp, D = in.n_donors;
    uint32_t pair[KH];          // d1 | d2 << 8 of hypothesis lane + 32k
#pragma unroll
    for (int k = 0; k < KH; ++k) {
        uint32_t d1 = 0, d2 = 0;
        if (lane + 32u * k < H) hyp_donors(lane + 32u * k, D, &d1, &d2);
        pair[k] = d1 | d2 << 8;
    }
    for (uint32_t c = warp; c < in.n_cols; c += n_warps) {
        const uint32_t i0 = col_start[c], i1 = col_start[c + 1];
        if (i0 == i1) continue;
        int64_t acc[KH];
#pragma unroll
        for (int k = 0; k < KH; ++k) acc[k] = 0;
        uint64_t sum_r = 0, sum_a = 0;
        for (uint32_t i = i0; i < i1; ++i) {
            const uint32_t q = list[i];
            const uint32_t row = in.locus_row[in.cslot_locus[q]];
            const uint32_t r = in.ccnt[4 * size_t(q)], a = in.ccnt[4 * size_t(q) + 1];
            const uint32_t g = lane < D ? in.dosage[size_t(row) * D + lane] : 0u;
            const uint32_t b0 = __ballot_sync(0xffffffffu, g & 1u), b1 = __ballot_sync(0xffffffffu, g & 2u);
            int64_t v[5];
#pragma unroll
            for (int s = 0; s < 5; ++s) v[s] = contribution(in.t, s, r, a);
#pragma unroll
            for (int k = 0; k < KH; ++k) {
                const uint32_t d1 = pair[k] & 0xFF, d2 = pair[k] >> 8;
                const uint32_t s = s_index((b0 >> d1 & 1u) | (b1 >> d1 & 1u) << 1, (b0 >> d2 & 1u) | (b1 >> d2 & 1u) << 1);
                int64_t x = v[0];                       // selects, not an indexed (local-memory) array
                x = s == 1 ? v[1] : x; x = s == 2 ? v[2] : x; x = s == 3 ? v[3] : x; x = s == 4 ? v[4] : x;
                acc[k] += x;
            }
            sum_r += r; sum_a += a;
        }
        int64_t* out = ll + size_t(c) * H;
#pragma unroll
        for (int k = 0; k < KH; ++k)
            if (lane + 32u * k < H) out[lane + 32u * k] += acc[k];
        if (lane == 0) { cnt[3 * size_t(c)] += i1 - i0; cnt[3 * size_t(c) + 1] += sum_r; cnt[3 * size_t(c) + 2] += sum_a; }
    }
}
#endif   // __CUDACC__

}  // namespace donors
}  // namespace vtx
