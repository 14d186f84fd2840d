// vtx_tile_class.cuh -- which Smith-Waterman kernel scores a locus (its tile class), and which kernels a batch launches.
// vtx_k_locus_prep gives every locus its class on the device; run_sw launches the kernels of the classes that can get
// tiles.  Both follow the rule written here once: a class that gets tiles but is not launched would drop its pairs
// without an error.  The kernel headers keep their layouts and static_assert that they agree with the limits below.
// Plain C++ when compiled without nvcc: the CPU tests build it with g++.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include "../../include/vartrix_b200.h"

#if defined(__CUDACC__)
#define VTX_TC_HD __host__ __device__
#else
#define VTX_TC_HD
#endif

namespace vtx {

// The classes, in the order vtx_last_tile_counts reports them
constexpr int kNumFastClasses = 4;                 // 0..3: single-phase vtx_k_sw_pairs<c> (vtx_sw.cuh)
constexpr int kSlowClass = kNumFastClasses;        // 4: generic kernel vtx_k_sw_generic
constexpr int kNumSplitClasses = 2;                // 5, 6: two-phase vtx_k_sw_split<s> (vtx_sw_split.cuh)
constexpr int kSplitClass0 = kSlowClass + 1;
constexpr int kFoldClass = kSplitClass0 + kNumSplitClasses;   // 7: folded kernel (vtx_sw_fold.cuh)
constexpr int kNumClasses = kFoldClass + 1;
// Class 3 also takes windows wider than class_max_n(3), in several passes of class_max_n(3) columns
constexpr int kMultiClass = 3;

// Widest window of single-phase class c: LPP * C of TileClass<c>
VTX_TC_HD constexpr int class_max_n(int cls)
{
    return cls == 0 ? 208 : cls == 1 ? 232 : cls == 2 ? 256 : cls == 3 ? 320 : 0x7fffffff;
}
constexpr int kMultiMaxRead = 256;       // longest read the multi-pass class takes
constexpr int kSplitP = 96;              // columns the two-phase kernels score once for both haplotypes
// Widest window of two-phase class s: kSplitP + 4 * C2 of SplitClass<s>
VTX_TC_HD constexpr int split_max_n(int scls) { return scls == 0 ? 204 : 232; }
constexpr int kSplitMaxRead = 256;       // longest read the two-phase kernels take (shared-memory budget)
constexpr int kFoldP = 96;               // flank columns of the folded kernel's main pass, on either side
constexpr int kFoldMaxMid = 40;          // most columns between the two flanks
constexpr int kFoldMaxRead = 152;        // longest read the folded kernel takes: 8 lanes x kFoldR rows in registers

// Pairs per warp tile of each class
VTX_TC_HD constexpr uint32_t pairs_per_tile(int cls)
{
    return cls == kSlowClass ? 16u : cls == kFoldClass ? 4u : cls > kSlowClass ? 8u : 4u;
}

// The kernel families a batch may use: the flags, and the longest read and widest window of the batch
struct SwAllow { bool split, multi, fold; };
VTX_TC_HD inline SwAllow allowed_kernels(uint32_t flags, uint32_t max_read, uint32_t max_hap)
{
    SwAllow a;
    a.split = max_read <= uint32_t(kSplitMaxRead) && !(flags & VTX_F_NO_SPLIT);
    a.multi = max_read <= uint32_t(kMultiMaxRead) && max_hap > uint32_t(class_max_n(kNumFastClasses - 1));
    a.fold = !(flags & (VTX_F_NO_SPLIT | VTX_F_NO_FOLD));
    return a;
}

// What the class of a locus depends on, besides its longest read
struct LocusShape {
    bool exotic;       // a window byte that a read base other than A/C/G/T decodes to: only the generic kernel compares bytes
    bool prefix;       // the windows share their first kSplitP columns (needs prefix_possible)
    bool fold;         // ... and their last kFoldP columns (needs fold_possible)
    uint32_t width;    // the wider window
};
VTX_TC_HD constexpr bool is_exotic(uint8_t b)   // "=MRSVWYHKDBN"
{
    return b == '=' || b == 'M' || b == 'R' || b == 'S' || b == 'V' || b == 'W' || b == 'Y' || b == 'H' ||
           b == 'K' || b == 'D' || b == 'B' || b == 'N';
}
VTX_TC_HD constexpr bool prefix_possible(uint32_t nr, uint32_t na) { return nr >= uint32_t(kSplitP) && na >= uint32_t(kSplitP); }
VTX_TC_HD constexpr bool fold_possible(uint32_t nr, uint32_t na)
{
    return (nr < na ? nr : na) > uint32_t(2 * kFoldP) && (nr < na ? na : nr) <= uint32_t(2 * kFoldP + kFoldMaxMid);
}

// The class of a locus (DESIGN.md section 4): the most specialised kernel that takes it
VTX_TC_HD inline int tile_class(const LocusShape& s, const SwAllow& allow, uint32_t longest_read)
{
    if (s.exotic) return kSlowClass;
    if (s.fold && allow.fold && longest_read <= uint32_t(kFoldMaxRead)) return kFoldClass;
    if (s.prefix && allow.split) {
        for (int c = 0; c < kNumSplitClasses; ++c)
            if (s.width <= uint32_t(split_max_n(c))) return kSplitClass0 + c;
    }
    for (int c = 0; c < kNumFastClasses; ++c)
        if (s.width <= uint32_t(class_max_n(c))) return c;
    return allow.multi ? kMultiClass : kSlowClass;
}

// Classes a device batch or vtx_score_pairs launches.  Their loci are not looked at on the host, so every class that
// a window of at most max_hap columns can get, the folded kernel whenever it is allowed, and the generic kernel.
VTX_TC_HD inline uint32_t device_class_mask(const SwAllow& allow, uint32_t max_hap)
{
    uint32_t mask = 1u << kSlowClass;
    for (int c = 0; c < kNumFastClasses; ++c)
        if (c == 0 || max_hap > uint32_t(class_max_n(c - 1))) mask |= 1u << c;
    for (int c = 0; allow.split && c < kNumSplitClasses; ++c)
        if (c == 0 || max_hap > uint32_t(split_max_n(c - 1))) mask |= 1u << (kSplitClass0 + c);
    if (allow.fold) mask |= 1u << kFoldClass;
    return mask;
}

// ---- host batches: the shapes of the loci, recorded while the batch is validated ----

// The shape of a locus from its windows.  Exotic bytes are left to the device: a byte-wise scan of every window would
// cost more than the launch it could save, so the generic kernel is always launched.
inline LocusShape window_shape(const uint8_t* rh, uint32_t nr, const uint8_t* ah, uint32_t na)
{
    LocusShape s{};
    s.prefix = prefix_possible(nr, na) && memcmp(rh, ah, kSplitP) == 0;
    s.fold = s.prefix && fold_possible(nr, na) && memcmp(rh + nr - kFoldP, ah + na - kFoldP, kFoldP) == 0;
    s.width = std::max(nr, na);
    return s;
}
// A shape as one of kNumShapeKeys keys: the three flags, and the window widths at which tile_class changes its answer
// that lie below the width.  Every width with the same key gets the same class.
constexpr uint32_t kWidthSteps[] = { uint32_t(split_max_n(0)), uint32_t(class_max_n(0)), uint32_t(split_max_n(1)),
                                     uint32_t(class_max_n(1)), uint32_t(class_max_n(2)), uint32_t(class_max_n(3)) };
constexpr int kNumWidthSteps = int(sizeof(kWidthSteps) / sizeof(kWidthSteps[0]));
static_assert(kWidthSteps[0] <= kWidthSteps[1] && kWidthSteps[1] <= kWidthSteps[2] && kWidthSteps[2] <= kWidthSteps[3] &&
              kWidthSteps[3] <= kWidthSteps[4] && kWidthSteps[4] <= kWidthSteps[5], "ascending");
constexpr int kNumShapeKeys = 8 * (kNumWidthSteps + 1);
static_assert(kNumShapeKeys <= 64, "a host batch keeps the keys it saw in one 64-bit word");
inline uint32_t shape_key(const LocusShape& s)
{
    uint32_t w = 0;
    while (w < uint32_t(kNumWidthSteps) && s.width > kWidthSteps[w]) ++w;
    return uint32_t(s.exotic) | uint32_t(s.prefix) << 1 | uint32_t(s.fold) << 2 | w << 3;
}
inline LocusShape key_shape(uint32_t k)
{
    const uint32_t w = k >> 3;
    return LocusShape{ bool(k & 1), bool(k & 2), bool(k & 4), w < uint32_t(kNumWidthSteps) ? kWidthSteps[w] : kWidthSteps[kNumWidthSteps - 1] + 1 };
}
// Classes a host batch launches: those of the shape keys seen, and the generic kernel.  A fold-shaped locus goes to
// another class when one of its reads is longer than kFoldMaxRead; only the batch's longest read tells whether it can.
inline uint32_t host_class_mask(uint64_t seen, const SwAllow& allow, uint32_t max_read)
{
    uint32_t mask = 1u << kSlowClass;
    for (uint32_t k = 0; k < uint32_t(kNumShapeKeys); ++k) {
        if (!(seen >> k & 1u)) continue;
        const LocusShape s = key_shape(k);
        mask |= 1u << tile_class(s, allow, 0) | 1u << tile_class(s, allow, max_read);
    }
    return mask;
}

}  // namespace vtx
