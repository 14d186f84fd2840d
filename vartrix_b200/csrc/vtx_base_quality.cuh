// vtx_base_quality.cuh -- --min-base-quality: the one decision body that the host stager (csrc/host/stager.hpp) and the
// device stager (vtx_stage.cuh, locus_cands) both call, so that the two paths cannot drift apart.  Plain C++ when compiled
// without nvcc: the CLI's host build includes it without the CUDA headers.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define VTX_BQ_HD __host__ __device__
#else
#define VTX_BQ_HD
#endif

namespace vtx {
namespace stage {

constexpr uint32_t kMaxBaseQuality = 93;     // Phred + 33 must stay printable ('~'): SAM's largest quality

// Does the record keep its (read, locus) pair at quality floor `min_q`?  `b` is the record without its block_size prefix;
// the locus covers the reference positions [start, end) = [rec.pos(), rec.pos() + len(REF)).  The CIGAR is walked from the
// record's pos; a read base is *judged* when it is
//   M / = / X : aligned to a reference position p with start <= p < end,
//   I         : inserted right after a reference base inside [start, end) (VCF insertions are anchored on the REF base),
// and S, H, D, N, P judge nothing.  The pair is dropped when a judged base has quality < min_q.  It is kept when no base is
// judged (a deletion over the whole REF span) and when the record carries no qualities (first quality byte 0xFF, as samtools
// writes them).  Query positions at or beyond l_seq (a CIGAR longer than SEQ, or SEQ "*") judge nothing.
VTX_BQ_HD inline bool base_quality_ok(const uint8_t* b, int64_t start, int64_t end, uint32_t min_q)
{
    auto ld32 = [](const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); };
    const int64_t l_seq = int32_t(ld32(b + 16));
    if (min_q == 0 || l_seq <= 0) return true;
    const uint32_t nc = uint32_t(b[12]) | (uint32_t(b[13]) << 8);
    const uint8_t* cg = b + 32 + b[8];
    const uint8_t* qual = cg + 4 * nc + (l_seq + 1) / 2;
    if (qual[0] == 0xFF) return true;                       // qualities absent
    int64_t rpos = int32_t(ld32(b + 4)), qpos = 0;
    for (uint32_t i = 0; i < nc && rpos <= end && qpos < l_seq; ++i) {      // past `end` nothing can be judged any more
        const uint32_t v = ld32(cg + 4 * i), op = v & 0xF;
        const int64_t len = int64_t(v >> 4);
        if (op == 0 || op == 7 || op == 8) {
            // the block's bases on [max(start, rpos), min(end, rpos + len)), clipped to the sequence
            const int64_t r0 = start > rpos ? start : rpos, r1 = end < rpos + len ? end : rpos + len;
            for (int64_t r = r0; r < r1 && qpos + (r - rpos) < l_seq; ++r)
                if (qual[qpos + (r - rpos)] < min_q) return false;
            rpos += len; qpos += len;
        } else if (op == 1) {
            if (rpos - 1 >= start && rpos - 1 < end)
                for (int64_t k = 0; k < len && qpos + k < l_seq; ++k)
                    if (qual[qpos + k] < min_q) return false;
            qpos += len;
        } else if (op == 4) qpos += len;
        else if (op == 2 || op == 3) rpos += len;
    }
    return true;
}

}  // namespace stage
}  // namespace vtx

#undef VTX_BQ_HD
