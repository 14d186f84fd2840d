// vtx_sw_band.cuh -- VTX_BAND_MODEL: Smith-Waterman restricted to a k-mer-chain band (optional, slow path).
//
// The reference aligns with bio 0.30.0's banded::Aligner::new(GAP_OPEN, GAP_EXTEND, score, K = 6, W = 20).local(read, hap)
// (vartrix src/main.rs:27-38, 898-901).  The crate's source is not available to this project; SURVEY.md
// Appendix B restates its band from documentation and memory ("model B", the variant consistent with every golden of the
// reference), and this kernel computes exactly that model:
//   1. every exact k-mer hit (i, j): read[i .. i+k) == hap[j .. j+k), in (i, j) order            (byte equality)
//   2. best chain of hits: a hit starts at k; the hit one step down the same diagonal adds 1; a hit at least k further in
//      both sequences adds k, minus go + ge * |diagonal change| when the diagonal changes; first best wins all ties
//   3. band = every DP column's row range widened by +-w around each cell of each chained hit, around a straight-then-
//      diagonal walk between consecutive chained hits, and around 2k more diagonal cells beyond both ends
//   4. affine local DP over the band only (cells outside are minus infinity); no hit at all -> the full matrix
// The full-matrix score (VTX_BAND_FULL, the default, what reproduces the reference's golden matrices) is an upper bound of
// this one and equal to it whenever the optimal alignment stays inside the band; tools/band_exposure.py measures where it
// does not (short tandem repeats, indels above w).  One warp per alignment; work buffers live in global scratch.
#pragma once
#include "vtx_sw.cuh"

namespace vtx {

constexpr int kBandThreads = 128;                 // 4 warps per CTA
constexpr int32_t kBandNegInf = -(1 << 29);
constexpr int kBandJ = 8;                         // window k-mers per lane kept in registers while hits are enumerated (windows <= 256 + k)

struct BandArgs {
    SwArgs sw;                  // batch, pair lists, epilogue (tile fields unused)
    uint32_t n_pairs_ub;        // pairs are [0, pair_start[n_loci])
    int32_t k, w;
    uint32_t max_read, max_hap; // scratch sizing (exact for host batches)
    uint32_t hit_cap;           // hits per alignment the scratch can hold
    uint8_t* scratch;           // [warps][band_warp_bytes]
    unsigned long long* overflow;   // alignments whose hits did not fit (reported by the next finish)
    unsigned long long* bounds_violated;   // pairs longer / wider than the sizes the scratch was cut for (device batches)
    uint32_t* cursor;           // work cursor over 2 * n_pairs alignments
};

__host__ __device__ inline size_t band_warp_bytes(uint32_t max_read, uint32_t max_hap, uint32_t hit_cap)
{
    size_t b = 0;
    b += (size_t(max_read) + 8) & ~size_t(7);                    // read as ASCII bytes
    b += (size_t(max_read) + size_t(max_hap) + 2) * 8;           // 6-byte k-mer codes of both sequences (u64)
    b += size_t(hit_cap) * 4;                                    // hits (i, j) as u16 pairs
    b += size_t(hit_cap) * 4 * 2;                                // chain score, predecessor
    b += (size_t(max_hap) + 1) * 4 * 2;                          // band: lo / hi row per column
    b += (size_t(max_read) + 1) * 4 * 4;                         // DP columns: S, D (previous | current)
    return (b + 255) & ~size_t(255);
}

__device__ __forceinline__ int32_t warp_max(int32_t v)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// one alignment by one warp; returns the banded (or, without hits, full) local score
__device__ int32_t band_align(const BandArgs& a, uint8_t* ws, const uint8_t* nib, int32_t m, const uint8_t* hap, int32_t n, bool* overflowed)
{
    const int lane = threadIdx.x & 31;
    const int32_t k = a.k, w = a.w;
    uint8_t* x = ws;
    uint64_t* xk = reinterpret_cast<uint64_t*>(ws + ((size_t(a.max_read) + 8) & ~size_t(7)));
    uint64_t* yk = xk + a.max_read + 1;
    uint32_t* hits = reinterpret_cast<uint32_t*>(yk + a.max_hap + 1);
    int32_t* sc = reinterpret_cast<int32_t*>(hits + a.hit_cap);
    int32_t* pr = sc + a.hit_cap;
    int32_t* lo = pr + a.hit_cap;
    int32_t* hi = lo + a.max_hap + 1;
    int32_t* S0 = hi + a.max_hap + 1;
    int32_t* D0 = S0 + a.max_read + 1;
    int32_t* S1 = D0 + a.max_read + 1;
    int32_t* D1 = S1 + a.max_read + 1;

    for (int32_t i = lane; i < m; i += 32) {
        const uint32_t by = __ldg(nib + (i >> 1));
        x[i] = uint8_t("=ACMGRSVTWYHKDBN"[(i & 1) ? (by & 0xF) : (by >> 4)]);               // main.rs:896
    }
    __syncwarp();
    bool banded = m >= k && n >= k && k >= 1 && k <= 8;
    uint32_t nh = 0;
    if (banded) {
        // 1. k-mer codes (k bytes packed: equality of codes == equality of the byte strings), then all hits in (i, j) order
        for (int32_t i = lane; i + k <= m; i += 32) { uint64_t c = 0; for (int32_t t = 0; t < k; ++t) c = (c << 8) | x[i + t]; xk[i] = c; }
        for (int32_t j = lane; j + k <= n; j += 32) { uint64_t c = 0; for (int32_t t = 0; t < k; ++t) c = (c << 8) | __ldg(hap + j + t); yk[j] = c; }
        __syncwarp();
        const int32_t ni = m - k + 1, nj = n - k + 1;
        if (nj <= 32 * kBandJ) {
            // the window's k-mers stay in registers (lane l holds j = l, l + 32, ...): per read position one broadcast load
            // and kBandJ compares; the (q, lane) order of the ballots is ascending j
            uint64_t yr[kBandJ];
#pragma unroll
            for (int q = 0; q < kBandJ; ++q) { const int32_t j = lane + 32 * q; yr[q] = j < nj ? yk[j] : ~0ull; }       // ~0 is no k-mer code (k <= 8 bytes of ASCII)
            for (int32_t i = 0; i < ni; ++i) {
                const uint64_t xi = xk[i];
                uint32_t mine = 0;
#pragma unroll
                for (int q = 0; q < kBandJ; ++q) mine |= uint32_t(yr[q] == xi) << q;
                if (!__any_sync(0xffffffffu, mine != 0)) continue;
#pragma unroll
                for (int q = 0; q < kBandJ; ++q) {
                    const bool hit = (mine >> q) & 1u;
                    const uint32_t mask = __ballot_sync(0xffffffffu, hit);
                    if (hit) {
                        const uint32_t slot = nh + __popc(mask & ((1u << lane) - 1u));
                        if (slot < a.hit_cap) hits[slot] = (uint32_t(i) << 16) | uint32_t(lane + 32 * q);
                    }
                    nh += __popc(mask);
                }
            }
        } else {
            for (int32_t i = 0; i < ni; ++i) {
                const uint64_t xi = xk[i];
                for (int32_t j0 = 0; j0 < nj; j0 += 32) {
                    const int32_t j = j0 + lane;
                    const bool hit = j < nj && yk[j] == xi;
                    const uint32_t mask = __ballot_sync(0xffffffffu, hit);
                    if (hit) {
                        const uint32_t slot = nh + __popc(mask & ((1u << lane) - 1u));
                        if (slot < a.hit_cap) hits[slot] = (uint32_t(i) << 16) | uint32_t(j);
                    }
                    nh += __popc(mask);
                }
            }
        }
        __syncwarp();
        if (nh > a.hit_cap) { *overflowed = true; nh = 0; banded = false; }          // reported; scored with the full matrix
        if (nh == 0) banded = false;                                                  // no hits -> full matrix
    }
    if (banded) {
        // 2. chain: sc[a] = best chain score ending in hit a; the earliest best predecessor wins (strict > over ascending b)
        int32_t best = -1; uint32_t best_idx = 0;
        for (uint32_t ia = 0; ia < nh; ++ia) {
            const int32_t ai = int32_t(hits[ia] >> 16), aj = int32_t(hits[ia] & 0xFFFFu);
            int32_t my = k, my_b = 0x7fffffff;                // (score, predecessor); predecessor "none" sorts last
            for (uint32_t ib = lane; ib < ia; ib += 32) {
                const int32_t di = ai - int32_t(hits[ib] >> 16), dj = aj - int32_t(hits[ib] & 0xFFFFu);
                int32_t cand;
                if (di == 1 && dj == 1) cand = sc[ib] + 1;
                else if (di >= k && dj >= k) { const int32_t dd = abs(di - dj); cand = sc[ib] + k + (dd ? kGapOpen + kGapExtend * dd : 0); }
                else continue;
                if (cand > my) { my = cand; my_b = int32_t(ib); }
            }
            // warp arg-max with ties to the smallest predecessor index; a candidate equal to k never replaces "start here"
            if (nh <= 0xFFFFu && m < 32000) {              // (score, 0xFFFF - index) fits one word: a single REDUX
                const uint32_t key = (uint32_t(my) << 16) | (my_b == 0x7fffffff ? 0u : 0xFFFFu - uint32_t(my_b));     // "none" sorts last
                const uint32_t top = __reduce_max_sync(0xffffffffu, key);
                my = int32_t(top >> 16); my_b = (top & 0xFFFFu) ? int32_t(0xFFFFu - (top & 0xFFFFu)) : 0x7fffffff;
            } else {
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) {
                    const int32_t os = __shfl_xor_sync(0xffffffffu, my, o), ob = __shfl_xor_sync(0xffffffffu, my_b, o);
                    if (os > my || (os == my && ob < my_b)) { my = os; my_b = ob; }
                }
            }
            if (lane == 0) { sc[ia] = my; pr[ia] = my_b == 0x7fffffff ? -1 : my_b; }
            if (my > best) { best = my; best_idx = ia; }
            __syncwarp();
        }
        // 3. band
        for (int32_t c = lane; c <= n; c += 32) { lo[c] = m + 1; hi[c] = -1; }
        __syncwarp();
        auto add_box = [&](int32_t bi, int32_t bj) {            // cell (bi, bj): widen every column within +-w
            const int32_t j0 = max(bj - w, 0), j1 = min(bj + w, n), i0 = max(bi - w, 0), i1 = min(bi + w, m);
            for (int32_t c = j0 + lane; c <= j1; c += 32) { if (i0 < lo[c]) lo[c] = i0; if (i1 > hi[c]) hi[c] = i1; }
            __syncwarp();
        };
        int32_t cur = int32_t(best_idx), last_i = -1, last_j = -1, first_i = 0, first_j = 0;
        while (cur >= 0) {
            const int32_t hi_i = int32_t(hits[cur] >> 16), hi_j = int32_t(hits[cur] & 0xFFFFu);
            // the later hit one step down the diagonal already boxed this hit's cells 1..k
            const int32_t t_end = (last_i == hi_i + 1 && last_j == hi_j + 1) ? 0 : k;
            for (int32_t t = 0; t <= t_end; ++t) add_box(hi_i + t, hi_j + t);
            if (last_i >= 0) {              // between this hit's end and the later hit's start: straight run, then diagonal
                int32_t ai = hi_i + k, aj = hi_j + k;
                while (ai < last_i || aj < last_j) {
                    if (last_i - ai > last_j - aj) ++ai;
                    else if (last_j - aj > last_i - ai) ++aj;
                    else { ++ai; ++aj; }
                    add_box(ai, aj);
                }
            }
            last_i = hi_i; last_j = hi_j; first_i = hi_i; first_j = hi_j;
            cur = pr[cur];
        }
        const int32_t end_i = int32_t(hits[best_idx] >> 16), end_j = int32_t(hits[best_idx] & 0xFFFFu);
        for (int32_t t = 1; t <= 2 * k; ++t) {                 // lazy extension beyond both ends
            int32_t ai = first_i - t, aj = first_j - t;
            if (ai >= 0 && aj >= 0) add_box(ai, aj);
            ai = end_i + k + t; aj = end_j + k + t;
            if (ai <= m && aj <= n) add_box(ai, aj);
        }
    } else {
        for (int32_t c = lane; c <= n; c += 32) { lo[c] = 0; hi[c] = m; }        // full matrix, same DP
        __syncwarp();
    }
    // 4. DP over the band, column by column; rows of a column in chunks of 32 lanes.  The vertical-gap state of a column
    //    is a max-plus prefix scan of S without its vertical-gap term (a gap opened from a gap is never better than
    //    extending it), so the rows of a column are computed together:  I(i) = max_{i' < i} S0(i') + go + ge (i - i').
    for (int32_t i = lane; i <= m; i += 32) { S0[i] = kBandNegInf; D0[i] = kBandNegInf; S1[i] = kBandNegInf; D1[i] = kBandNegInf; }
    __syncwarp();
    int32_t ans = 0;
    const int32_t go = kGapOpen, ge = kGapExtend;
    int32_t prev_lo = 1, prev_hi = 0;                              // band of the previous column (empty before column 0)
    for (int32_t j = 0; j <= n; ++j) {
        int32_t* Sc = (j & 1) ? S1 : S0; int32_t* Dc = (j & 1) ? D1 : D0;
        const int32_t* Sp = (j & 1) ? S0 : S1; const int32_t* Dp = (j & 1) ? D0 : D1;
        const int32_t cl = lo[j], ch = hi[j];
        // the column two back used this buffer: clear exactly its band rows (they are the only non-minus-infinity entries)
        // -- done at the end of this iteration for the *previous* column's buffer; here Sc / Dc are all minus infinity.
        if (ch >= 0) {
            const uint8_t yj = j > 0 ? __ldg(hap + j - 1) : 0;
            int32_t carry = kBandNegInf;                            // max over the rows above of S0(i') - ge * i'  (+ go later)
            for (int32_t base = cl; base <= ch; base += 32) {
                const int32_t i = base + lane;
                const bool on = i <= ch;
                int32_t s = 0, del = kBandNegInf;
                if (on) {
                    if (i > 0 && j > 0) { const int32_t d = Sp[i - 1]; if (d > kBandNegInf / 2) s = max(s, d + (x[i - 1] == yj ? kMatch : kMismatch)); }
                    if (j > 0) {
                        const int32_t dp = Dp[i], sp = Sp[i];
                        if (dp > kBandNegInf / 2) del = dp + ge;
                        if (sp > kBandNegInf / 2) del = max(del, sp + go + ge);
                    }
                    s = max(s, del);
                }
                // inclusive max-scan of t(i) = s(i) - ge * i over the chunk's lanes
                int32_t tv = on ? s - ge * i : kBandNegInf;
                int32_t incl = tv;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int32_t up = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl = max(incl, up); }
                int32_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
                if (lane == 0) excl = kBandNegInf;
                excl = max(excl, carry);                            // rows above, this chunk and the earlier ones
                if (on) {
                    const int32_t ins = excl > kBandNegInf / 2 ? excl + go + ge * i : kBandNegInf;    // = max S0(i') + go + ge (i - i')
                    s = max(s, ins);
                    Sc[i] = s; Dc[i] = del;
                    ans = max(ans, s);
                }
                carry = max(carry, __shfl_sync(0xffffffffu, incl, 31));
            }
        }
        __syncwarp();
        // clear the previous column's buffer (it becomes the current one at j + 1): only its band rows were written
        {
            int32_t* So = (j & 1) ? S0 : S1; int32_t* Do = (j & 1) ? D0 : D1;
            for (int32_t i = prev_lo + lane; i <= prev_hi; i += 32) { So[i] = kBandNegInf; Do[i] = kBandNegInf; }
        }
        prev_lo = ch >= 0 ? cl : 1; prev_hi = ch >= 0 ? ch : 0;
        __syncwarp();
    }
    return warp_max(ans);
}

// One warp per (pair, haplotype): work item 2 p + h.  Ref and alt scores meet in shared memory for the epilogue.
__global__ void __launch_bounds__(kBandThreads) vtx_k_sw_band(const BandArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint8_t* ws = a.scratch + size_t(gwarp) * band_warp_bytes(a.max_read, a.max_hap, a.hit_cap);
    const uint32_t n_pairs = __ldg(a.sw.pair_start + a.sw.n_loci);
    for (;;) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(a.cursor, 1u);
        p = __shfl_sync(0xffffffffu, p, 0);
        if (p >= n_pairs) break;
        const uint32_t locus = upper_locus(a.sw.pair_start, a.sw.n_loci, p);
        const uint32_t r = __ldg(a.sw.pair_read + p);
        const int32_t m = int32_t(__ldg(a.sw.read_len + r));
        const uint8_t* nib = a.sw.read_nib + __ldg(a.sw.read_off + r);
        const uint32_t nr = __ldg(a.sw.ref_len + locus), na = __ldg(a.sw.alt_len + locus);
        if (uint32_t(m) > a.max_read || nr > a.max_hap || na > a.max_hap) {         // a device batch broke its promised bounds
            if (lane == 0) atomicAdd(a.bounds_violated, 1ull);
            continue;
        }
        bool over = false;
        const int32_t rs = band_align(a, ws, nib, m, a.sw.hap_bytes + __ldg(a.sw.ref_off + locus), int32_t(__ldg(a.sw.ref_len + locus)), &over);
        __syncwarp();
        const int32_t as = band_align(a, ws, nib, m, a.sw.hap_bytes + __ldg(a.sw.alt_off + locus), int32_t(__ldg(a.sw.alt_len + locus)), &over);
        __syncwarp();
        if (lane == 0) {
            if (over) atomicAdd(a.overflow, 1ull);
            call_and_scatter(a.sw, p, pack2(rs, as));
        }
    }
}

}  // namespace vtx
