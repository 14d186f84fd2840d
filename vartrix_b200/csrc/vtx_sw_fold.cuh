// vtx_sw_fold.cuh -- "folded" Smith-Waterman: neither shared flank of a locus is computed per haplotype.
//
// construct_haplotypes (vartrix src/main.rs:958-994) gives the ref and the alt window the SAME left
// flank and the SAME right flank; only the allele columns in between differ.  The local-alignment maximum
// decomposes exactly (oracle/vtx_oracle.c::vtxo_sw_fold pins this on the CPU against the full matrix):
//
//   best = max( max H over the prefix columns,                                 -- forward DP, shared
//               max Hr over the suffix columns,                                -- DP of the REVERSED read against
//                                                                                 the reversed suffix, shared
//               max H over the allele ("middle") columns,                      -- forward DP continued, per haplotype
//               max_i  H(i, last) + Hr(i + 1),  E(i, last) + Er(i + 1) - go )  -- junction, per haplotype
//
// (E = horizontal-gap state; a gap that runs across the junction was opened on both sides, hence "- go").
// A warp tile is 4 reads of one locus, one read per 8-lane unit:
//
//   main pass   kFoldP = 96 columns, 12 per lane, rows skewed by one step per lane exactly like the other
//               kernels -- but the two int16 halves are (forward DP over hap[0, 96), reversed DP over
//               hap[n - 96, n) reversed) of the SAME read.  Forward row i and reversed row i are read rows i and
//               m - 1 - i, so the per-locus profile is pre-merged over the pair of their codes (25 rows): per
//               step a lane loads one pair code and its 12 substitution words (3 LDS.128), nothing to merge.
//               The last column (H + gap, E) of every row goes to shared memory.
//   extension   the flanks of a window usually reach past 96 columns (--padding 100: 100 on either side of an SNV),
//               so the columns between the main pass and the allele columns are common to ref and alt too.  The
//               table builder picks x (both sides the same, 0 when nothing more is shared): the halves stay
//               (forward, reversed), continued over hap[96, 96 + x) and reversed hap[n - 96 - x, n - 96) once for
//               both haplotypes, column-synchronously like the allele columns below.  Its reversed boundary
//               replaces the parked one.  An SNV with --padding 100 has 4 + 1 such column steps instead of 9.
//   middle      the remaining n - 192 - 2 x allele columns (up to 40): halves are (ref, alt) again.  Lane g owns
//               the 19 read rows [19 g, 19 g + 19), whose (H + gap, E) start from the forward boundary, and the 8
//               lanes of a unit walk over the columns together, one column per step: F down a column is a running
//               maximum, so it crosses the lanes as one exclusive max-scan.
//   junction    after the last allele column of a haplotype every lane adds the parked reverse boundary of the
//               partner rows (reversed row m - 2 - r for forward row r).
//
// Per pair this is 2 x (96 + x) + (n - 192 - 2 x) column-passes in "one read per word" units instead of
// 96 / 2 + (n - 96): ~25 % fewer DPX instructions than vtx_k_sw_split for an SNV window.  Reads up to kFoldMaxRead
// bases, windows with both flanks >= 96 columns in common and at most kFoldMaxMid allele columns.
#pragma once
#include <cuda/atomic>
#include "vtx_sw.cuh"
#include "vtx_fold_ring.cuh"

namespace vtx {

constexpr int kFoldC1 = 12;            // main-pass columns per lane: 8 x 12 = kFoldP
constexpr int kFoldPPW = 4;            // pairs per warp tile
constexpr int kFoldR = 19;             // read rows per lane in the middle (8 x 19 = 152)
static_assert(8 * kFoldC1 == kFoldP && 8 * kFoldR == kFoldMaxRead && kFoldPPW == int(pairs_per_tile(kFoldClass)),
              "vtx_tile_class.cuh: flank columns, longest read and pairs per tile of the folded class");
// boundary rows kept per read; 156 (not 152) so that the four reads of a tile start 8, 16 and 24 banks apart
// (152 rows x 8 bytes put reads 0/2 and 1/3 on the same banks: a 2-way conflict on every boundary store and load)
constexpr int kFoldRows = kFoldMaxRead + 4;
constexpr int kFoldCodeStride = kFoldMaxRead + 16;   // row codes per read and kind (8 sentinels either side)
constexpr int kFoldPairRows = 25;                    // merged profile rows: 5 x forward code + reverse code
#ifndef VTX_FOLD_UNROLL
#define VTX_FOLD_UNROLL 4
#endif
// CTA shapes (one CTA per SM).  A shard with at least kFoldDeepDepth candidates per locus runs kFoldDeepWarps warps
// sharing kFoldDeepSlots slots of per-locus tables (vtx_fold_ring.cuh).  A shallower shard, whose loci are mostly a
// single tile, would have at most kFoldDeepSlots of those warps busy and has little to share: it runs kFoldShallowWarps
// warps with one table each.
constexpr int kFoldDeepWarps = 20, kFoldDeepSlots = 9;
constexpr int kFoldShallowWarps = 13;
#ifndef VTX_FOLD_DEEP_DEPTH
#define VTX_FOLD_DEEP_DEPTH 6
#endif
constexpr uint32_t kFoldDeepDepth = VTX_FOLD_DEEP_DEPTH;
constexpr int kFoldUnroll = VTX_FOLD_UNROLL;         // row-loop unrolling of the main pass
#ifndef VTX_FOLD_MID_UNROLL
#define VTX_FOLD_MID_UNROLL 1
#endif
constexpr int kFoldMidUnroll = VTX_FOLD_MID_UNROLL;  // column-loop unrolling of the allele pass

// per-locus slot: merged profile [pair code][column], then kFoldMidTabBytes for the shared-extension table
// [column][pair code] (kFoldExtColBytes per column) followed by the allele-column table [column][read code] (32 bytes)
constexpr int kFoldMidTabBytes = kFoldMaxMid * 32, kFoldExtColBytes = kFoldPairRows * 4;
constexpr size_t kFoldSlotBytes = size_t(kFoldPairRows) * kFoldP * 4 + kFoldMidTabBytes;
// per warp: boundary column (forward | reverse) per read and row, then the row codes (forward, and pair (row i, row m - 1 - i))
constexpr size_t kFoldWarpBytes = size_t(kFoldPPW) * kFoldRows * 8 + 32 + size_t(2 * kFoldPPW) * kFoldCodeStride;
static_assert(kFoldSlotBytes % 16 == 0 && kFoldWarpBytes % 16 == 0, "slots and warp areas stay 16-byte aligned");
template <int S> __host__ __device__ constexpr size_t fold_ring_bytes() { return (sizeof(FoldRing<S>) + 15) & ~size_t(15); }
// shared memory of a CTA of W warps sharing S slots: ring control | S slots | W warp areas
template <int W, int S> __host__ __device__ constexpr size_t fold_cta_bytes()
{
    return fold_ring_bytes<S>() + S * kFoldSlotBytes + W * kFoldWarpBytes;
}

// the atomic policy of vtx_fold_ring.cuh on the GPU: block-scope atomics on shared memory, one lane per warp
struct FoldSyncDev {
    using ref = cuda::atomic_ref<uint32_t, cuda::thread_scope_block>;
    __device__ static bool try_lock(uint32_t* p)
    {
        uint32_t z = 0;
        return ref(*p).compare_exchange_strong(z, 1u, cuda::memory_order_acquire, cuda::memory_order_relaxed);
    }
    __device__ static void unlock(uint32_t* p) { ref(*p).store(0u, cuda::memory_order_release); }
    __device__ static uint32_t grab(uint32_t* cursor) { return atomicAdd(cursor, 1u); }
    __device__ static uint32_t load_relaxed(uint32_t* p) { return ref(*p).load(cuda::memory_order_relaxed); }
    __device__ static uint32_t load_acquire(uint32_t* p) { return ref(*p).load(cuda::memory_order_acquire); }
    __device__ static void store_relaxed(uint32_t* p, uint32_t v) { ref(*p).store(v, cuda::memory_order_relaxed); }
    __device__ static void store_release(uint32_t* p, uint32_t v) { ref(*p).store(v, cuda::memory_order_release); }
    __device__ static void add(uint32_t* p, uint32_t v) { ref(*p).fetch_add(v, cuda::memory_order_relaxed); }
    __device__ static void sub_release(uint32_t* p, uint32_t v) { ref(*p).fetch_sub(v, cuda::memory_order_release); }
    __device__ static void pause() { __nanosleep(100); }      // leave the issue slots to the warps doing DP work
};

// Largest l in [lo, n) with ts[l] <= t, given ts[lo] <= t (ts ascending), by the whole warp: first the 32 loci after lo
// (lo is the locus of a recently booked tile, so one coalesced load usually settles it), then a 32-ary search.
__device__ __forceinline__ uint32_t fold_locate(const uint32_t* __restrict__ ts, uint32_t n, uint32_t lo, uint32_t t,
                                                int lane)
{
    uint32_t hi = n, step = 1;                                   // invariant: ts[lo] <= t, and the answer is < hi
    for (;;) {
        const uint32_t i = lo + uint32_t(lane + 1) * step;
        const uint32_t k = __popc(__ballot_sync(0xffffffffu, i < hi && __ldg(ts + i) <= t));   // a prefix of the lanes
        lo += k * step;
        if (k < 32) hi = min(hi, lo + step);
        if (hi - lo <= 1) return lo;
        step = (hi - lo + 31) / 32;
    }
}

// junction constants: (H_f + goe + B) + (H_r + goe + B) -> H_f + H_r + B, and (E_f + B) + (E_r + B) - go -> ... + B;
// the sum of two biased halves is >= 2 * (B + goe), so adding the negative constant always carries exactly once
constexpr int kJuncH = -2 * kGoe - kBias, kJuncE = -kGapOpen - kBias;
constexpr uint32_t kJuncH2 = (uint32_t(uint16_t(int16_t(kJuncH - 1))) << 16) | uint32_t(uint16_t(int16_t(kJuncH)));
constexpr uint32_t kJuncE2 = (uint32_t(uint16_t(int16_t(kJuncE - 1))) << 16) | uint32_t(uint16_t(int16_t(kJuncE)));

// allele-pass constants (row c of a strip): y = a - c ge, F = P + goe + (c - 1) ge, H + goe = max(y, P + go) + goe + c ge
static_assert(kGapExtend < 0 && kGapOpen <= 0, "the vertical gap is a running maximum only if go <= 0");
constexpr uint32_t kFoldRowY2 = uint32_t(-kGapExtend) * 0x10001u;   // + (-ge, -ge): positive, never carries
constexpr uint32_t kGO2 = pack2(kGapOpen, kGapOpen);                 // per-half add inside VIADDMNMX
// P above row 0: a biased "minus infinity" that the packed adds and subtracts applied to P cannot borrow from
constexpr uint32_t kScanNeg2 = pack2(kBias - 1024, kBias - 1024);
// + (v, v) with v = goe + c ge < 0 onto halves >= kBias: the low half always carries exactly once (as kGoeAdd)
__host__ __device__ constexpr uint32_t fold_row_hg_add(int c)
{
    return (uint32_t(uint16_t(int16_t(kGoe + c * kGapExtend - 1))) << 16) | uint32_t(uint16_t(int16_t(kGoe + c * kGapExtend)));
}
static_assert(fold_row_hg_add(0) == kGoeAdd, "row 0 adds plain goe");

// W warps per CTA (one CTA per SM) and S slots of per-locus tables.  SHARED: the warps share the slots and
// vtx_fold_ring.cuh hands out the tiles and slots.  Otherwise (S == W) slot w is warp w's own table and each warp takes
// chunks of consecutive tiles from the global cursor, rebuilding its table when the locus changes.
template <int W, int S, bool SHARED>
__global__ void __launch_bounds__(W * 32, 1) vtx_k_sw_fold(const SwArgs a)
{
    constexpr int C1 = kFoldC1, P = kFoldP, R = kFoldR, M = 8;
    constexpr int RS1 = P;                                       // 96 words: rows stay on their banks

    extern __shared__ __align__(16) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u = lane >> 3, g = lane & 7;                       // unit = read of the tile, lane within the unit
    FoldRing<S>& ring = *reinterpret_cast<FoldRing<S>*>(smem_raw);
    uint8_t* const slots = smem_raw + fold_ring_bytes<S>();
    uint2* bnd = reinterpret_cast<uint2*>(slots + S * kFoldSlotBytes + warp * kFoldWarpBytes);
    uint8_t* codes = reinterpret_cast<uint8_t*>(bnd + kFoldPPW * kFoldRows + 4);

    const uint32_t n_tiles = __ldg(a.tile_start + a.n_loci);
    static_assert(SHARED || S == W, "per-warp tables: one slot per warp");
    const uint32_t run_len = SHARED ? fold_run_len(n_tiles, gridDim.x, W, kTileChunk)
                                    : max(1u, min(uint32_t(kTileChunk), n_tiles / (gridDim.x * W * 16u)));
    uint32_t w_next = 0, w_end = 0, w_locus = 0, w_cached = kFoldNoTile;   // per-warp tables: the warp's chunk
    if (threadIdx.x == 0) ring_init(ring);
    __syncthreads();                                             // the only CTA-wide barrier (see vtx_fold_ring.cuh)

    for (;;) {
        __syncwarp();
        uint32_t tile, locus, slot;
        bool build;
        if constexpr (SHARED) {
            FoldTake tk{};
            if (lane == 0) tk = ring_take<FoldSyncDev>(ring, a.tile_counter, run_len, n_tiles);
            tile = __shfl_sync(0xffffffffu, tk.tile, 0);
            if (tile == kFoldNoTile) break;
            locus = fold_locate(a.tile_start, a.n_loci, __shfl_sync(0xffffffffu, tk.hint, 0), tile, lane);
            FoldBook bk{};
            if (lane == 0) bk = ring_book<FoldSyncDev>(ring, tk.ticket, locus);
            slot = __shfl_sync(0xffffffffu, bk.slot, 0);
            build = __shfl_sync(0xffffffffu, bk.build, 0);
        } else {
            if (w_next == w_end) {
                uint32_t chunk = 0;
                if (lane == 0) chunk = atomicAdd(a.tile_counter, 1u);
                chunk = __shfl_sync(0xffffffffu, chunk, 0);
                w_next = chunk * run_len;
                if (w_next >= n_tiles) break;
                w_end = min(w_next + run_len, n_tiles);
                w_locus = upper_locus(a.tile_start, a.n_loci, w_next);
            }
            tile = w_next++;
            while (tile >= __ldg(a.tile_start + w_locus + 1)) ++w_locus;
            locus = w_locus;
            slot = warp;
            build = locus != w_cached;
            w_cached = locus;
        }
        const uint32_t p0 = __ldg(a.pair_start + locus) + kFoldPPW * (tile - __ldg(a.tile_start + locus));
        const uint32_t p_end = __ldg(a.pair_start + locus + 1);
        uint32_t* prof = reinterpret_cast<uint32_t*>(slots + slot * kFoldSlotBytes);
        uint32_t* midtab = prof + kFoldPairRows * RS1;
        // ---- per-locus tables: built by the warp that claimed the locus's first tile in this CTA ----
        if (build) {
            const uint8_t* rh = a.hap_bytes + __ldg(a.ref_off + locus);
            const uint8_t* ah = a.hap_bytes + __ldg(a.alt_off + locus);
            const int n_ref = int(__ldg(a.ref_len + locus)), n_alt = int(__ldg(a.alt_len + locus));
            const int mid_ref = n_ref - 2 * P, mid_alt = n_alt - 2 * P;
            // row 5 a + b, column c: {s(a, hap[c]), s(b, hap[n - 1 - c])}; both flanks are common to ref and alt
            // (vtx_k_locus_prep).  Lane j < 24 fills columns [4 j, 4 j + 4) of every row with one STS.128 each.
            if (lane < P / 4) {
                uint32_t fb[4], sb[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    fb[k] = hap_code(__ldg(rh + 4 * lane + k));
                    sb[k] = hap_code(__ldg(rh + (n_ref - 1 - 4 * lane - k)));
                }
#pragma unroll
                for (uint32_t ra = 0; ra < 5; ++ra)
#pragma unroll
                    for (uint32_t rb = 0; rb < 5; ++rb) {
                        uint32_t w[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            w[k] = pack2(ra == fb[k] ? kProfMatch : kProfMis, rb == sb[k] ? kProfMatch : kProfMis);
                        reinterpret_cast<uint4*>(prof + (5 * ra + rb) * RS1)[lane] = make_uint4(w[0], w[1], w[2], w[3]);
                    }
            }
            // x: the columns P + j (left) and n - 1 - P - j (right) that ref and alt still share, j < x.  Both halves
            // extend by the same x (a half cannot be padded with sentinel columns without changing its boundary), every
            // allele keeps at least one column of its own (the junction follows them), and both tables fit the slot.
            const int lmax = max(mid_ref, mid_alt), lmin = min(mid_ref, mid_alt);
            const int x_cap = min((lmin - 1) / 2, (kFoldMidTabBytes - 32 * lmax) / (kFoldExtColBytes - 64));
            const bool shared = lane < x_cap && __ldg(rh + P + lane) == __ldg(ah + P + lane) &&
                                __ldg(rh + (n_ref - 1 - P - lane)) == __ldg(ah + (n_alt - 1 - P - lane));
            const int x = __ffs(~__ballot_sync(0xffffffffu, shared)) - 1;
            const int am_ref = mid_ref - 2 * x, am_alt = mid_alt - 2 * x;
            if (lane == 0) ring.mids[slot] = uint32_t(am_ref) | uint32_t(am_alt) << 8 | uint32_t(x) << 16;
            // shared extension [column][pair code]: the main pass's merged profile continued over columns P + j, lane j
            // filling column j
            if (lane < x) {
                const uint32_t fb = hap_code(__ldg(rh + P + lane)), sb = hap_code(__ldg(rh + (n_ref - 1 - P - lane)));
#pragma unroll
                for (uint32_t ra = 0; ra < 5; ++ra)
#pragma unroll
                    for (uint32_t rb = 0; rb < 5; ++rb)
                        midtab[lane * kFoldPairRows + 5 * ra + rb] = pack2(ra == fb ? kProfMatch : kProfMis, rb == sb ? kProfMatch : kProfMis);
            }
            uint32_t* alltab = midtab + x * kFoldPairRows;
            for (int idx = lane; idx < (lmax - 2 * x) * 8; idx += 32) {
                const int k = idx >> 3;
                const uint32_t r = uint32_t(idx & 7);
                const uint32_t rb = k < am_ref ? hap_code(__ldg(rh + P + x + k)) : 5u;   // past the shorter allele: sentinel
                const uint32_t ab = k < am_alt ? hap_code(__ldg(ah + P + x + k)) : 5u;
                alltab[idx] = pack2(r == rb ? kProfMatch : kProfMis, r == ab ? kProfMatch : kProfMis);
            }
            __syncwarp();
            if (SHARED && lane == 0) ring_publish<FoldSyncDev>(ring, slot);
        } else if (SHARED) {
            ring_wait<FoldSyncDev>(ring, slot);                          // every lane acquires the builder's tables
        }
        // ---- row codes: the 8 lanes of a unit fill their read's forward codes, then the pair codes from them ----
        const uint32_t pair = p0 + u;
        const bool active = pair < p_end;
        int m = 0;
        uint8_t* cf = codes + (2 * u) * kFoldCodeStride;                 // forward code of row e - M (the middle's rows)
        uint8_t* cp = cf + kFoldCodeStride;                               // 5 x code(row e - M) + code(row m - 1 - (e - M))
        {
            const uint8_t* nib = nullptr;
            if (active) {
                const uint32_t rd = __ldg(a.pair_read + pair);
                m = int(__ldg(a.read_len + rd));
                nib = a.read_nib + __ldg(a.read_off + rd);
            }
            for (int e = g; e < kFoldCodeStride; e += 8)
                if (e < M || e >= M + m) cf[e] = 4;
            for (int b = g; 2 * b < m; b += 8) {
                const uint32_t by = __ldg(nib + b);
                cf[M + 2 * b] = uint8_t(nib_code(by >> 4));
                if (2 * b + 1 < m) cf[M + 2 * b + 1] = uint8_t(nib_code(by & 0xF));
            }
            __syncwarp();
            for (int e = g; e < kFoldCodeStride; e += 8)                 // sentinel rows: (4, 4), all mismatch
                cp[e] = (e < M || e >= M + m) ? uint8_t(5 * 4 + 4) : uint8_t(5 * cf[e] + cf[2 * M + m - 1 - e]);
        }
        int mmax = m;
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) mmax = max(mmax, __shfl_xor_sync(0xffffffffu, mmax, o));
        __syncwarp();

        // The boundary of row r lives at entry r + 7: lane 7 stores at entry t in EVERY step (no `t >= 7` test in the
        // loop); its first 7 stores are scratch.  Entries 156..158 of a read (rows 149..151) fall on the scratch entries
        // 0..2 of the next read, which that read wrote 150 steps earlier and nobody reads; the last read has 4 spare.
        uint2* my_bnd = bnd + u * kFoldRows;
        const uint2* row_bnd = my_bnd + 7;
        uint32_t best;
        // =========================== main pass: forward prefix | reversed suffix ===========================
        {
            uint32_t hg[C1], f[C1];
#pragma unroll
            for (int c = 0; c < C1; ++c) { hg[c] = kGOE2; f[c] = kNEG2; }
            uint32_t hg_last = kGOE2, e_last = kNEG2, diag_save = kGOE2;
            best = kBIAS2;
            const uint8_t* cA = cp + M - g;
            const uint32_t* lane_p = prof + g * C1;
            const int steps = mmax + 7;
#pragma unroll kFoldUnroll
            for (int t = 0; t < steps; ++t) {
                uint32_t hl = __shfl_up_sync(0xffffffffu, hg_last, 1, 8);
                uint32_t el = __shfl_up_sync(0xffffffffu, e_last, 1, 8);
                if (g == 0) { hl = kGOE2; el = kNEG2; }
                const uint4* pa = reinterpret_cast<const uint4*>(lane_p + uint32_t(cA[t]) * RS1);
                uint32_t diag = diag_save;
                diag_save = hl;
                uint32_t e = el, eg = hl, hleft = hl;
#pragma unroll
                for (int q = 0; q < C1 / 4; ++q) {
                    const uint4 a4 = pa[q];                                      // {s_fwd, s_rev}
                    const uint32_t sv[4] = { a4.x, a4.y, a4.z, a4.w };
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
                if (g == 7) my_bnd[t] = make_uint2(hleft, e);                    // columns P-1 (fwd) / n-P (rev) of row t-7
            }
#pragma unroll
            for (int o = 4; o >= 1; o >>= 1) best = __vmaxs2(best, __shfl_xor_sync(0xffffffffu, best, o));
            best = __vmaxs2(best, __byte_perm(best, 0, 0x1032));                 // both halves: max(prefix, suffix)
        }
        __syncwarp();

        // ============ shared extension: (forward, reversed) again; middle: (ref, alt) over the allele columns ============
        {
            const uint32_t mids = ring.mids[slot];                               // read here: nothing held across the main pass
            uint32_t hg[R], e[R], rc[R];
            const uint8_t* cpm = cp + M + R * g;
            const uint8_t* cfm = cf + M + R * g;
#pragma unroll
            for (int c = 0; c < R; ++c) {
                const int row = R * g + c;
                uint2 b = make_uint2(kGOE2, kNEG2);
                if (row < mmax) b = row_bnd[row];
                hg[c] = b.x;                                                     // (forward, reversed) as parked
                e[c] = b.y;
                rc[c] = uint32_t(cpm[c]) * 4u;                                   // pair code of forward row r, reversed row r
            }
            // junction of the halves in `mask`: forward row r meets reversed row m - 2 - r
            // (one base register and the row's constant offset, not one row index per c held across the allele pass)
            const int jlim = m - 2 - R * g;
            const uint2* jbnd = row_bnd + jlim;
            auto junction = [&](uint32_t mask) {
                uint32_t cross = kBIAS2;
#pragma unroll
                for (int c = 0; c < R; ++c) {
                    uint2 b = make_uint2(kGOE2, kGOE2);                          // Hr = 0; Er such that E + Er - go < H
                    if (c <= jlim) b = jbnd[-c];                                 // reversed row m - 2 - (R g + c)
                    const uint32_t ph = __byte_perm(b.x, 0, 0x3232), pe = __byte_perm(b.y, 0, 0x3232);
                    const uint32_t x1 = hg[c] + ph + kJuncH2;
                    const uint32_t x2 = e[c] + pe + kJuncE2;
                    cross = __vimax3_s16x2(cross, x1, x2);
                }
                best = __vmaxs2(best, (cross & mask) | (kBIAS2 & ~mask));
            };
            // All 8 lanes of a unit work on the same column k.  With a(r) = max(H(r-1, k-1) + s, E(r, k), 0), F runs
            // down the column as F(r) = max(F(r-1) + ge, H(r-1) + goe), and H(r-1) = max(a(r-1), F(r-1)); the branch
            // F(r-1) + goe never wins (go <= 0), so
            //     F(r) = max over r' < r of a(r') + goe + (r-1-r') ge = P(r) + goe + (r-1) ge,  P(r) = max_{r' < r} y(r'),
            // with y(r') = a(r') - r' ge.  Pass 1 computes a and y of the lane's 19 rows (y goes into hg[c], whose old
            // value has already served as the diagonal of row c + 1); an exclusive max-scan over the unit's lanes gives
            // P at the top of each strip; pass 2 turns y back into H + goe.  The lane keeps y relative to its first row
            // (y(c) = a - c ge) and adds its offset -19 g ge only for the scan.  max H over a column is max a (F(r) <
            // a(r') for some r' < r), so `best` takes a.
            // Ranges: a is biased in [kBias, kBias + 152], y in [kBias, kBias + 152 + 151] once offset, P never below
            // kScanNeg2 - 19 * 7: all halves stay far inside int16 and above every negative constant added to them below.
            // One column of both halves; trow is the column's table row, indexed by rc.
            auto column = [&](const uint8_t* trow) {
                // H(19 g - 1, k - 1) + goe: the last row of the lane above, before pass 1 overwrites it (at the first
                // column the parked boundary); row -1 of the matrix is H = 0
                uint32_t diag = __shfl_up_sync(0xffffffffu, hg[R - 1], 1, 8);
                if (g == 0) diag = kGOE2;
                uint32_t aa[2], yy[2], ymax = kBIAS2;                            // y >= kBias: the floor changes nothing
#pragma unroll
                for (int c = 0; c < R; ++c) {                                    // pass 1: E, a, y
                    const uint32_t sv = *reinterpret_cast<const uint32_t*>(trow + rc[c]);
                    const uint32_t ec = __viaddmax_s16x2(e[c], kGE2, hg[c]);          // E(r, k)
                    const uint32_t av = __vimax3_s16x2(diag + sv, ec, kBIAS2);       // a(r): positive add, no carry
                    const uint32_t yv = av + kFoldRowY2 * uint32_t(c);
                    diag = hg[c];
                    hg[c] = yv;
                    e[c] = ec;
                    aa[c & 1] = av;
                    yy[c & 1] = yv;
                    if (c & 1) {
                        best = __vimax3_s16x2(best, aa[0], aa[1]);
                        ymax = __vimax3_s16x2(ymax, yy[0], yy[1]);
                    }
                }
                if (R & 1) {
                    best = __vmaxs2(best, aa[0]);
                    ymax = __vmaxs2(ymax, yy[0]);
                }
                // P at row 19 g: the max of y over the lanes above (shfl_up returns a lane's own value below its offset)
                const uint32_t lane_ofs = uint32_t(-kGapExtend * R * g) * 0x10001u;
                uint32_t p = __shfl_up_sync(0xffffffffu, ymax + lane_ofs, 1, 8);
                if (g == 0) p = kScanNeg2;
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) p = __vmaxs2(p, __shfl_up_sync(0xffffffffu, p, o, 8));
                p -= lane_ofs;                                                   // halves >= 19 * 7: no borrow
#pragma unroll
                for (int c = 0; c < R; ++c) {                                    // pass 2: H = max(a, F), stored as H + goe
                    const uint32_t yv = hg[c];
                    // max(y, P + go) = H - c ge; adding goe + c ge (negative) carries exactly once from halves >= kBias
                    hg[c] = __viaddmax_s16x2(p, kGO2, yv) + fold_row_hg_add(c);
                    if (c + 1 < R) p = __vmaxs2(p, yv);
                }
            };
            // Shared extension: columns [P, P + x) forward and [n - P - x, n - P) reversed, common to ref and alt, so
            // scored once for both (the table builder chose x).  Forward row r and reversed row r are read rows r and
            // m - 1 - r, so the table is indexed by pair code like the main pass's profile.
            const uint8_t* tab = reinterpret_cast<const uint8_t*>(midtab);
            for (int k = int(mids >> 16); k > 0; --k, tab += kFoldExtColBytes) column(tab);
            best = __vmaxs2(best, __byte_perm(best, 0, 0x1032));                 // both halves count for ref and alt
            // park the extended reversed boundary for the junction; the allele columns continue the forward half.  Rows
            // 149..151 land on scratch entries (see above), so every row is stored.
            uint2* park = my_bnd + 7 + R * g;
#pragma unroll
            for (int c = 0; c < R; ++c) {
                park[c] = make_uint2(hg[c], e[c]);
                hg[c] = __byte_perm(hg[c], 0, 0x1010);
                e[c] = __byte_perm(e[c], 0, 0x1010);
                rc[c] = uint32_t(cfm[c]) * 4u;
            }
            __syncwarp();                                                        // the junction reads other lanes' rows
            const int mid_ref = int(mids & 0xFFu), mid_alt = int((mids >> 8) & 0xFFu);
            const int lmax = max(mid_ref, mid_alt), lmin = min(mid_ref, mid_alt);
            // the half whose allele ends first, and its last column (none for equal alleles)
            const uint32_t short_mask = mid_ref < mid_alt ? 0x0000FFFFu : mid_alt < mid_ref ? 0xFFFF0000u : 0u;
            const int k_short = lmin != lmax ? lmin - 1 : -1;
#pragma unroll kFoldMidUnroll
            for (int k = 0; k < lmax; ++k) {
                column(tab + 32 * k);                                            // allele table [k][*]
                if (k == k_short) junction(short_mask);                          // the shorter allele ends here (indels only)
            }
            junction(~short_mask);                                                // every lane has finished column lmax - 1
#pragma unroll
            for (int o = 4; o >= 1; o >>= 1) best = __vmaxs2(best, __shfl_xor_sync(0xffffffffu, best, o));
            // every lane is done with the allele table; release before the scatter, whose global atomics the release
            // fence would otherwise wait for
            __syncwarp();
            if (SHARED && lane == 0) ring_release<FoldSyncDev>(ring, slot);
            if (active && g == 0) call_and_scatter(a, pair, best - kBIAS2);
        }
    }
}

}  // namespace vtx
