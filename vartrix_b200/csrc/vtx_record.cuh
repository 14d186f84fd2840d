// vtx_record.cuh -- the reference's rules for one BAM record: the record filters, the end position, the tag parsing and the
// key packing.  Both stagers apply them to every record: the host stager (csrc/host/stager.hpp, bam_reader.hpp) and the
// device stager (vtx_stage.cuh).  There is one body per rule, so that the two paths cannot drift apart.  Plain C++ when
// compiled without nvcc: the CLI's host build includes it without the CUDA headers.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define VTX_REC_HD __host__ __device__
#else
#define VTX_REC_HD
#endif

namespace vtx {
namespace stage {

constexpr uint64_t kNoCbKey = 0xFFFFFFFFFFFFFFFFull;     // VTX_NO_CB_KEY
constexpr uint64_t kNoUmi = 0xFFFFFFFFFFFFFFFFull;       // VTX_NO_UMI
constexpr uint32_t kMaxBaseQuality = 93;     // Phred + 33 must stay printable ('~'): SAM's largest quality

VTX_REC_HD inline uint32_t ld32(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); }
VTX_REC_HD inline uint32_t ld16(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8); }

// In every function below, `b` is a record without its block_size prefix.

// htslib bam_endpos: pos + the reference length of the CIGAR (M, D, N, =, X); pos + 1 when unmapped or of zero length
VTX_REC_HD inline int64_t ref_end(const uint8_t* b)
{
    int64_t rlen = 0;
    if (!(ld16(b + 14) & 4)) {
        const uint8_t* c = b + 32 + b[8];
        const uint32_t nc = ld16(b + 12);
        for (uint32_t i = 0; i < nc; ++i) {
            const uint32_t v = ld32(c + 4 * i), op = v & 0xF;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += v >> 4;
        }
    }
    return int64_t(int32_t(ld32(b + 4))) + (rlen > 0 ? rlen : 1);
}

// rust-htslib 0.36 CigarStringView::read_pos(p, include_softclips = false, include_dels = true) folded into
// useful_alignment (main.rs:790-806): is there a p in start..=end with an aligned base or a deletion?
VTX_REC_HD inline bool useful_alignment(const uint8_t* b, int64_t start, int64_t end)
{
    const uint8_t* cg = b + 32 + b[8];
    const uint32_t nc = ld16(b + 12);
    const int64_t pos0 = int32_t(ld32(b + 4));
    uint32_t i0 = 0;
    while (i0 < nc) {            // leading section: first of M,=,X,I,S starts the walk; leading D/N or an interior H is an error
        const uint32_t op = ld32(cg + 4 * i0) & 0xF;
        if (op == 0 || op == 7 || op == 8 || op == 1 || op == 4) break;
        if (op == 2 || op == 3) return false;
        if (op == 5 && i0 != 0 && i0 != nc - 1) return false;
        ++i0;
    }
    if (i0 >= nc) return false;
    for (int64_t p = start; p <= end; ++p) {          // inclusive end, main.rs:794
        int64_t rpos = pos0;
        for (uint32_t i = i0; i < nc && rpos <= p; ++i) {
            const uint32_t v = ld32(cg + 4 * i), op = v & 0xF; const int64_t len = int64_t(v >> 4);
            if (op == 0 || op == 7 || op == 8 || op == 2) { if (p >= rpos && p < rpos + len) return true; rpos += len; }
            else if (op == 3) rpos += len;
            else if (op == 5) { if (i != nc - 1) return false; break; }
        }
    }
    return false;
}

// Does the record keep its (read, locus) pair at quality floor `min_q`?  The locus covers the reference positions
// [start, end) = [rec.pos(), rec.pos() + len(REF)).  The CIGAR is walked from the record's pos; a read base is *judged* when it is
//   M / = / X : aligned to a reference position p with start <= p < end,
//   I         : inserted right after a reference base inside [start, end) (VCF insertions are anchored on the REF base),
// and S, H, D, N, P judge nothing.  The pair is dropped when a judged base has quality < min_q.  It is kept when no base is
// judged (a deletion over the whole REF span) and when the record carries no qualities (first quality byte 0xFF, as samtools
// writes them).  Query positions at or beyond l_seq (a CIGAR longer than SEQ, or SEQ "*") judge nothing.
VTX_REC_HD inline bool base_quality_ok(const uint8_t* b, int64_t start, int64_t end, uint32_t min_q)
{
    const int64_t l_seq = int32_t(ld32(b + 16));
    if (min_q == 0 || l_seq <= 0) return true;
    const uint32_t nc = ld16(b + 12);
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

// The per-locus record counters, in the order the reference counts them (main.rs:831-865); vtx_bam_metrics, the first
// entries of vtx_locus_stats and the CLI's --out-variant-stats columns use this order.
enum RecordCounter : int { kFetched = 0, kLowMapq, kNonPrimary, kDuplicate, kNotUseful, kLowBaseQuality, kNumCounters };

// The record filter settings.  stage::Params and the host's StageArgs derive from it, so that both stagers read the same
// four fields and a call of drop_reason passes either of them.
struct RecordFilters {
    uint32_t mapq_min = 0;           // --mapq
    bool primary_only = false;       // --primary-alignments
    bool no_duplicates = false;      // --no-duplicates
    uint32_t min_base_quality = 0;   // --min-base-quality (0: off)
};

// The record filters of main.rs:833-865, then the base-quality floor, for a record fetched at the locus [start, end): 0 when
// the record is kept, else the counter of the first filter that drops it.  `flag` and `mapq` come from the caller (the device
// keeps them in a compact per-record array); the record bytes are read only once the flag tests have passed.
VTX_REC_HD inline int drop_reason(uint32_t flag, uint32_t mapq, const uint8_t* b, int64_t start, int64_t end, const RecordFilters& f)
{
    if (mapq < f.mapq_min) return kLowMapq;                                 // 833
    if (f.primary_only && (flag & 0x900)) return kNonPrimary;           // 841: secondary or supplementary
    if (f.no_duplicates && (flag & 0x400)) return kDuplicate;           // 849
    if (!useful_alignment(b, start, end)) return kNotUseful;            // 857
    if (f.min_base_quality && !base_quality_ok(b, start, end, f.min_base_quality)) return kLowBaseQuality;
    return 0;
}

// first aux field named (t0, t1) in [p, e): its value bytes at p + *off_from_p when the type is Z (Record::aux -> Aux::String,
// main.rs:737-757), else nothing
VTX_REC_HD inline bool aux_z(const uint8_t* p, const uint8_t* e, uint8_t t0, uint8_t t1, uint32_t* off_from_p, uint32_t* len)
{
    const uint8_t* base = p;
    while (p + 3 <= e) {
        const bool hit = p[0] == t0 && p[1] == t1;
        const uint8_t ty = p[2];
        p += 3;
        if (ty == 'Z' || ty == 'H') {
#ifdef __CUDA_ARCH__
            const uint8_t* q = p;
            while (q < e && *q) ++q;
#else
            const uint8_t* q = static_cast<const uint8_t*>(memchr(p, 0, size_t(e - p)));     // a byte loop doubles the host's time per tag
            if (!q) q = e;
#endif
            if (q >= e) return false;
            if (hit) { if (ty == 'Z') { *off_from_p = uint32_t(p - base); *len = uint32_t(q - p); return true; } return false; }
            p = q + 1;
        } else {
            size_t sz;
            switch (ty) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'B': {
                if (p + 5 > e) return false;
                const uint8_t sub = p[0]; const uint32_t cnt = ld32(p + 1);
                const size_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                sz = 5 + size_t(cnt) * es; break;
            }
            default: return false;
            }
            if (hit) return false;
            p += sz;
        }
    }
    return false;
}

// vtx_pack_cb: [ACGT]{1,24}(-N)?, N = 1..99 without a leading zero -> bases (2 bits each) << 12 | n_bases << 7 | N; an
// injective code.  kNoCbKey for anything else.
VTX_REC_HD inline uint64_t pack_cb(const uint8_t* s, uint32_t len)
{
    uint32_t n = 0;
    uint64_t k = 0;
    while (n < len && n < 25) {
        uint64_t c;
        const uint8_t b = s[n];
        if (b == 'A') c = 0; else if (b == 'C') c = 1; else if (b == 'G') c = 2; else if (b == 'T') c = 3; else break;
        if (n == 24) return kNoCbKey;
        k = (k << 2) | c;
        ++n;
    }
    if (n == 0) return kNoCbKey;
    uint64_t suffix = 0;
    if (n < len) {
        if (s[n] != '-') return kNoCbKey;
        const uint32_t d = len - n - 1;
        if (d < 1 || d > 2 || s[n + 1] < '1' || s[n + 1] > '9') return kNoCbKey;
        suffix = uint64_t(s[n + 1] - '0');
        if (d == 2) { if (s[n + 2] < '0' || s[n + 2] > '9') return kNoCbKey; suffix = suffix * 10 + uint64_t(s[n + 2] - '0'); }
    }
    return (k << 12) | (uint64_t(n) << 7) | suffix;
}

// vtx_pack_umi: strings over {A,C,G,T,N} up to 18 bases -> 3 bits per base << 5 | length, an injective code; kNoUmi for
// anything else
VTX_REC_HD inline uint64_t pack_umi(const uint8_t* s, uint32_t len)
{
    if (len > 18) return kNoUmi;
    uint64_t k = 0;
    for (uint32_t i = 0; i < len; ++i) {
        uint64_t c;
        switch (s[i]) { case 'A': c = 0; break; case 'C': c = 1; break; case 'G': c = 2; break; case 'T': c = 3; break; case 'N': c = 4; break; default: return kNoUmi; }
        k = (k << 3) | c;
    }
    return (k << 5) | len;      // < 2^59: bits 59..61 stay clear for caller-interned ids
}

}  // namespace stage
}  // namespace vtx

#undef VTX_REC_HD
