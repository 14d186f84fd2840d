// vtx_sw_split.cuh -- two-phase Smith-Waterman that does not compute the shared left flank twice.
//
// The ref and alt haplotypes of a locus are identical up to the variant (construct_haplotypes,
// vartrix src/main.rs:958-994: same left flank), so in the first kSplitP columns the two int16
// halves of vtx_k_sw_pairs carry the same numbers.  Here a warp tile is 8 pairs of one locus:
//
//   phase 1  columns [0, 96): the two halves hold two DIFFERENT READS (A, B) against the common prefix.
//            4 units x 8 lanes, 12 columns per lane.  The substitution word is s_A + (s_B << 16), formed
//            with an IMAD so that it stays off the DPX pipe (PRMT/LOP3 share it).  The last column of every row
//            (H + gap, E) is parked in shared memory, the prefix maximum per read too.
//   phase 2  columns [96, n): halves are (ref, alt) of ONE read again.  8 reads x 4 lanes, C2 columns per
//            lane; lane 0 of a read picks its half of the parked boundary and duplicates it (PRMT).
//
// Same recurrence, sentinels and exactness argument as vtx_sw.cuh; per pair it issues ~3 400 DPX
// instructions instead of ~4 600 (prefix computed once per two reads, shorter pipeline drain).
#pragma once
#include "vtx_sw.cuh"

namespace vtx {

constexpr int kSplitC1 = 12;            // phase 1: 8 lanes x 12 columns = kSplitP
constexpr int kSplitPPW = 8;           // pairs per warp tile

template <int SCLS> struct SplitClass;
#ifndef VTX_SPLIT0_THREADS
#define VTX_SPLIT0_THREADS 320
#endif
#ifndef VTX_SPLIT1_THREADS
#define VTX_SPLIT1_THREADS 256
#endif
template <> struct SplitClass<0> { static constexpr int C2 = 27, CS2 = 28, THREADS = VTX_SPLIT0_THREADS, MINB = 2; };   // n <= 96 + 108 = 204 (SNV, pad 100)
template <> struct SplitClass<1> { static constexpr int C2 = 34, CS2 = 36, THREADS = VTX_SPLIT1_THREADS, MINB = 2; };   // n <= 96 + 136 = 232 (indels <= 30)
static_assert(8 * kSplitC1 == kSplitP && kSplitPPW == int(pairs_per_tile(kSplitClass0)) && kSplitPPW == int(pairs_per_tile(kSplitClass0 + 1)),
              "vtx_tile_class.cuh: prefix columns and pairs per tile of the two-phase classes");
static_assert(kSplitP + 4 * SplitClass<0>::C2 == split_max_n(0) && kSplitP + 4 * SplitClass<1>::C2 == split_max_n(1),
              "vtx_tile_class.cuh: widest window of the two-phase classes");

template <int SCLS>
__host__ __device__ constexpr size_t split_warp_bytes(int mcap)
{
    using SC = SplitClass<SCLS>;
    constexpr int RS2 = (4 * SC::CS2 + 31) / 32 * 32;
    size_t b = size_t(5 * kSplitP) * 4;                         // prof1
    b += size_t(5 * RS2 + 16) * 4;                               // prof2 and 16 spare words
    b += size_t(4) * (mcap + 8) * 8;                             // boundary column, per unit and row
    b += 16;                                                     // prefix maxima
    b += size_t(kSplitPPW) * (mcap + 16);                        // row codes (u8)
    return (b + 15) & ~size_t(15);
}

template <int SCLS>
__global__ void __launch_bounds__(SplitClass<SCLS>::THREADS, SplitClass<SCLS>::MINB) vtx_k_sw_split(const SwArgs a)
{
    using SC = SplitClass<SCLS>;
    constexpr int C1 = kSplitC1, C2 = SC::C2, CS2 = SC::CS2, P = kSplitP;
    constexpr int RS1 = P;                                       // 96 words: 3 x 32 banks
    constexpr int RS2 = (4 * CS2 + 31) / 32 * 32;
    constexpr int M = 8;
    static_assert(CS2 % 4 == 0 && ((CS2 / 4) & 1) == 1 && CS2 >= C2, "phase-2 stride");

    extern __shared__ __align__(16) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int code_stride = a.mcap + 2 * M;
    uint8_t* wbase = smem_raw + warp * split_warp_bytes<SCLS>(a.mcap);
    uint32_t* prof1 = reinterpret_cast<uint32_t*>(wbase);
    uint32_t* prof2 = prof1 + 5 * RS1;
    uint2* bnd = reinterpret_cast<uint2*>(prof2 + 5 * RS2 + 16);
    uint32_t* p1best = reinterpret_cast<uint32_t*>(bnd + 4 * (a.mcap + 8));
    uint8_t* codes = reinterpret_cast<uint8_t*>(p1best + 4);
    const int bnd_stride = a.mcap + 8;

    const uint32_t n_tiles = __ldg(a.tile_start + a.n_loci);
    uint32_t cached_locus = 0xFFFFFFFFu;
    // tiles grabbed per atomic: up to kTileChunk for locality of the per-locus profile, fewer when the shard is
    // small so that every warp still gets >= ~16 grabs (tail balance)
    const uint32_t tile_chunk = max(1u, min(uint32_t(kTileChunk), n_tiles / (gridDim.x * (blockDim.x >> 5) * 16u)));
    const uint32_t k64k = a.k64k;                                // 65536, opaque to ptxas so the merge stays an IMAD

    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(a.tile_counter, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        const uint32_t t_begin = chunk * tile_chunk;
        if (t_begin >= n_tiles) break;
        const uint32_t t_end = min(t_begin + tile_chunk, n_tiles);
        uint32_t locus = upper_locus(a.tile_start, a.n_loci, t_begin);
        for (uint32_t tile = t_begin; tile < t_end; ++tile) {
            while (tile >= __ldg(a.tile_start + locus + 1)) ++locus;
            const uint32_t p0 = __ldg(a.pair_start + locus) + kSplitPPW * (tile - __ldg(a.tile_start + locus));
            const uint32_t p_end = __ldg(a.pair_start + locus + 1);
            __syncwarp();
            // ---- profiles of the locus ----
            if (locus != cached_locus) {
                cached_locus = locus;
                const uint8_t* rh = a.hap_bytes + __ldg(a.ref_off + locus);
                const uint8_t* ah = a.hap_bytes + __ldg(a.alt_off + locus);
                const int n_ref = int(__ldg(a.ref_len + locus)), n_alt = int(__ldg(a.alt_len + locus));
                for (int j = lane; j < P; j += 32) {             // prefix: ref == alt here (checked by vtx_k_locus_prep)
                    const uint32_t rb = hap_code(__ldg(rh + j));
#pragma unroll
                    for (uint32_t r = 0; r < 5; ++r) {
                        prof1[r * RS1 + j] = uint32_t(r == rb ? kProfMatch : kProfMis);      // low half only: merged per step
                    }
                }
                for (int idx = lane; idx < 4 * CS2; idx += 32) {
                    const int gg = idx / CS2, k = idx - gg * CS2;
                    const int j = P + gg * C2 + k;
                    uint32_t rb = 5, ab = 5;
                    if (k < C2) {
                        if (j < n_ref) rb = hap_code(__ldg(rh + j));
                        if (j < n_alt) ab = hap_code(__ldg(ah + j));
                    }
#pragma unroll
                    for (uint32_t r = 0; r < 5; ++r)
                        prof2[r * RS2 + idx] = pack2(r == rb ? kProfMatch : kProfMis, r == ab ? kProfMatch : kProfMis);
                }
            }
            // ---- row codes: lane l helps read (l / 4) ----
            int mmax = 0;
            {
                const int r = lane >> 2, q = lane & 3;
                const uint32_t pair = p0 + r;
                int m = 0;
                const uint8_t* nib = nullptr;
                if (pair < p_end) {
                    const uint32_t rd = __ldg(a.pair_read + pair);
                    m = int(__ldg(a.read_len + rd));
                    nib = a.read_nib + __ldg(a.read_off + rd);
                }
                uint8_t* cr = codes + r * code_stride;
                for (int e = q; e < code_stride; e += 4)
                    if (e < M || e >= M + m) cr[e] = 4;
                for (int b = q; 2 * b < m; b += 4) {
                    const uint32_t by = __ldg(nib + b);
                    cr[M + 2 * b] = uint8_t(nib_code(by >> 4));
                    if (2 * b + 1 < m) cr[M + 2 * b + 1] = uint8_t(nib_code(by & 0xF));
                }
                mmax = m;
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) mmax = max(mmax, __shfl_xor_sync(0xffffffffu, mmax, o));
            }
            __syncwarp();

            // =========================== phase 1: two reads against the common prefix ===========================
            {
                const int u = lane >> 3, g = lane & 7;
                uint32_t hg[C1], f[C1];
#pragma unroll
                for (int c = 0; c < C1; ++c) { hg[c] = kGOE2; f[c] = kNEG2; }
                uint32_t hg_last = kGOE2, e_last = kNEG2, diag_save = kGOE2, best = kBIAS2;
                const uint8_t* cA = codes + (2 * u) * code_stride + M - g;
                const uint8_t* cB = codes + (2 * u + 1) * code_stride + M - g;
                const uint32_t* lane_prof = prof1 + g * C1;
                uint2* my_bnd = bnd + u * bnd_stride;
                const int steps = mmax + 7;
                for (int t = 0; t < steps; ++t) {
                    uint32_t hl = __shfl_up_sync(0xffffffffu, hg_last, 1, 8);
                    uint32_t el = __shfl_up_sync(0xffffffffu, e_last, 1, 8);
                    if (g == 0) { hl = kGOE2; el = kNEG2; }
                    const uint4* pa = reinterpret_cast<const uint4*>(lane_prof + uint32_t(cA[t]) * RS1);
                    const uint4* pb = reinterpret_cast<const uint4*>(lane_prof + uint32_t(cB[t]) * RS1);
                    uint32_t diag = diag_save;
                    diag_save = hl;
                    uint32_t e = el, eg = hl, hleft = hl;
#pragma unroll
                    for (int q = 0; q < C1 / 4; ++q) {
                        const uint4 a4 = pa[q], b4 = pb[q];
                        // {s_A, s_B} = s_A + (s_B << 16) as an IMAD (FMA pipe): PRMT / LEA would compete with the DPX pipe
                        const uint32_t sv[4] = { b4.x * k64k + a4.x, b4.y * k64k + a4.y, b4.z * k64k + a4.z, b4.w * k64k + a4.w };
                        uint32_t hh[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const int c = 4 * q + k;
                            const uint32_t fc = __viaddmax_s16x2(f[c], kGE2, hg[c]);
                            e = __viaddmax_s16x2(e, kGE2, eg);
                            const uint32_t h = sw_h(diag, sv[k], fc, e);
                            hh[k] = h;
                            diag = hg[c];
                            hleft = h + kGoeAdd;
                            eg = hleft;
                            hg[c] = hleft;
                            f[c] = fc;
                        }
                        best = __vimax3_s16x2(best, hh[0], hh[1]);
                        best = __vimax3_s16x2(best, hh[2], hh[3]);
                    }
                    hg_last = hleft;
                    e_last = e;
                    if (g == 7 && t >= 7) my_bnd[t - 7] = make_uint2(hleft, e);     // column P-1 of row t-7
                }
#pragma unroll
                for (int o = 4; o >= 1; o >>= 1) best = __vmaxs2(best, __shfl_xor_sync(0xffffffffu, best, o));
                if (g == 0) p1best[u] = best;
            }
            __syncwarp();

            // =========================== phase 2: (ref, alt) of one read beyond the prefix ===========================
            {
                const int r = lane >> 2, g = lane & 3, u = r >> 1, w = r & 1;
                const uint32_t pair = p0 + r;
                const bool active = pair < p_end;
                const uint32_t sel = w ? 0x3232u : 0x1010u;
                uint32_t hg[C2], f[C2];
#pragma unroll
                for (int c = 0; c < C2; ++c) { hg[c] = kGOE2; f[c] = kNEG2; }
                uint32_t hg_last = kGOE2, e_last = kNEG2, diag_save = kGOE2;
                uint32_t best = __byte_perm(p1best[u], 0, sel);              // the prefix maximum counts for ref and alt
                const uint8_t* cR = codes + r * code_stride + M - g;
                const uint32_t* lane_prof = prof2 + g * CS2;
                const uint2* my_bnd = bnd + u * bnd_stride;
                const int steps = mmax + 3;
                for (int t = 0; t < steps; ++t) {
                    uint32_t hl = __shfl_up_sync(0xffffffffu, hg_last, 1, 4);
                    uint32_t el = __shfl_up_sync(0xffffffffu, e_last, 1, 4);
                    if (g == 0) {
                        if (t < mmax) {
                            const uint2 b = my_bnd[t];
                            hl = __byte_perm(b.x, 0, sel);
                            el = __byte_perm(b.y, 0, sel);
                        } else { hl = kGOE2; el = kNEG2; }
                    }
                    const uint4* prow = reinterpret_cast<const uint4*>(lane_prof + uint32_t(cR[t]) * RS2);
                    uint32_t diag = diag_save;
                    diag_save = hl;
                    uint32_t e = el, eg = hl, hleft = hl;
#pragma unroll
                    for (int q = 0; q < (C2 + 3) / 4; ++q) {
                        const uint4 s4 = prow[q];
                        const uint32_t sv[4] = { s4.x, s4.y, s4.z, s4.w };
                        uint32_t hh[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const int c = 4 * q + k;
                            if (c < C2) {
                                const uint32_t fc = __viaddmax_s16x2(f[c], kGE2, hg[c]);
                                e = __viaddmax_s16x2(e, kGE2, eg);
                                const uint32_t h = sw_h(diag, sv[k], fc, e);
                                hh[k] = h;
                                diag = hg[c];
                                hleft = h + kGoeAdd;
                                eg = hleft;
                                hg[c] = hleft;
                                f[c] = fc;
                            } else {
                                hh[k] = kBIAS2;
                            }
                        }
                        best = __vimax3_s16x2(best, hh[0], hh[1]);
                        if (4 * q + 2 < C2) best = __vimax3_s16x2(best, hh[2], hh[3]);
                    }
                    hg_last = hleft;
                    e_last = e;
                }
#pragma unroll
                for (int o = 2; o >= 1; o >>= 1) best = __vmaxs2(best, __shfl_xor_sync(0xffffffffu, best, o));
                if (active && g == 0) call_and_scatter(a, pair, best - kBIAS2);       // un-bias (no borrow: halves >= kBias)
            }
        }
    }
}

}  // namespace vtx
