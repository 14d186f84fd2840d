// vtx_inflate.cuh -- raw DEFLATE (RFC 1951) decoder for BGZF members on the device: one warp per member.
//
// Replaces, for the staging path, what htslib's bgzf_read_block -> inflate does for the reference
// (vartrix src/main.rs:822-829 through rust-htslib; SURVEY.md section 8(f)-1).  BGZF members are independent,
// <= 64 KiB of output each, with the uncompressed size in the gzip trailer -- thousands of them per shard of loci.
//
// A warp owns one member.  Lane 0 walks the bit stream (64-bit bit buffer refilled from 4-byte words, two-level lookup
// tables in shared memory, the same entry layout as the host decoder csrc/host/inflate_fast.hpp) and decodes up to 32
// symbols into a batch; then the whole warp applies the batch: an exclusive scan of the symbol lengths gives every symbol
// its output position, the literals are stored in one instruction, and every match is copied by all lanes together
// (source index taken modulo the distance, so overlapping matches need no intra-copy ordering).  The symbol decode and the
// table builders are __host__ __device__ so that the bit-stream logic is also pinned on the CPU against zlib
// (tests/test_inflate_cpu.py); the warp-level apply step is checked on the GPU against the host decoder.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace vtx {
namespace inflate {

constexpr int kLitBits = 10, kDistBits = 8;
constexpr int kLitTab = (1 << kLitBits) + 512, kDistTab = (1 << kDistBits) + 512;      // main + second-level entries
constexpr uint32_t kTypeLiteral = 0u << 30, kTypeBase = 1u << 30, kTypeEnd = 2u << 30, kTypeSub = 3u << 30, kTypeMask = 3u << 30;
// entry: [31:30] type  [29:13] payload (literal / base value / subtable offset)  [12:8] extra bits (or subtable bits)  [7:0] code length
__host__ __device__ inline uint32_t make_entry(uint32_t type, uint32_t payload, uint32_t extra, uint32_t len) { return type | (payload << 13) | (extra << 8) | len; }

enum Status : int32_t { kOk = 0, kBadStream = 1, kBadTable = 2, kOverrun = 3, kBadSize = 4, kBadStored = 5, kBadDistance = 6 };

struct Tables {
    uint32_t lit[kLitTab];
    uint32_t dist[kDistTab];
};

__host__ __device__ inline uint32_t reverse_bits(uint32_t v, int n)
{
    uint32_t r = 0;
    for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1); v >>= 1; }
    return r;
}

__host__ __device__ inline uint32_t litlen_entry(int s)
{
    const uint16_t base[29] = { 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258 };
    const uint8_t extra[29] = { 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0 };
    if (s < 256) return make_entry(kTypeLiteral, uint32_t(s), 0, 0);
    if (s == 256) return make_entry(kTypeEnd, 0, 0, 0);
    if (s > 285) return make_entry(kTypeEnd, 1, 0, 0);        // 286, 287: invalid in data (payload 1 marks the error)
    return make_entry(kTypeBase, base[s - 257], extra[s - 257], 0);
}
__host__ __device__ inline uint32_t dist_entry(int s)
{
    const uint16_t base[30] = { 1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                4097, 6145, 8193, 12289, 16385, 24577 };
    const uint8_t extra[30] = { 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13 };
    if (s > 29) return make_entry(kTypeEnd, 1, 0, 0);          // 30, 31: invalid
    return make_entry(kTypeBase, base[s], extra[s], 0);
}
__host__ __device__ inline uint32_t plain_entry(int s) { return make_entry(kTypeLiteral, uint32_t(s), 0, 0); }

// Canonical Huffman code lengths -> two-level lookup table indexed by the next bits of the stream (LSB first).
// KIND: 0 literal/length alphabet, 1 distance alphabet, 2 code-length alphabet.  Returns false for over-subscribed codes,
// incomplete ones (except the single-code case zlib also accepts) and tables that do not fit `tab_cap`.
template <int KIND>
__host__ __device__ inline bool build_table(const uint8_t* lens, int n_sym, int main_bits, uint32_t* tab, int tab_cap)
{
    int count[16];
    for (int i = 0; i < 16; ++i) count[i] = 0;
    for (int s = 0; s < n_sym; ++s) count[lens[s]]++;
    count[0] = 0;
    int max_len = 15;
    while (max_len > 0 && count[max_len] == 0) --max_len;
    const uint32_t main_size = 1u << main_bits;
    for (uint32_t i = 0; i < main_size; ++i) tab[i] = 0;
    if (max_len == 0) return true;               // no codes at all: every lookup is an error
    uint32_t code = 0, next_code[16];
    int left = 1, n_codes = 0;
    next_code[0] = 0;
    for (int l = 1; l <= 15; ++l) {
        left <<= 1; left -= count[l];
        if (left < 0) return false;              // over-subscribed
        code = (code + uint32_t(count[l - 1])) << 1;
        next_code[l] = code;
        n_codes += count[l];
    }
    if (left > 0 && n_codes != 1) return false;  // incomplete
    // second-level tables: one per main-table prefix that has longer codes, sized by the longest code under it.
    // Pass 1 records the largest excess length per prefix in the (still unused) main entries.
    if (max_len > main_bits) {
        uint32_t nc[16];
        for (int l = 0; l < 16; ++l) nc[l] = next_code[l];
        for (int s = 0; s < n_sym; ++s) {
            const int l = lens[s];
            if (l == 0) continue;
            const uint32_t c = nc[l]++;
            if (l > main_bits) {
                const uint32_t prefix = reverse_bits(c >> (l - main_bits), main_bits);
                if (uint32_t(l - main_bits) > tab[prefix]) tab[prefix] = uint32_t(l - main_bits);
            }
        }
        int off = int(main_size);
        for (uint32_t p = 0; p < main_size; ++p) {
            const uint32_t sb = tab[p];
            if (!sb) continue;
            if (off + (1 << sb) > tab_cap) return false;
            tab[p] = make_entry(kTypeSub, uint32_t(off), sb, uint32_t(main_bits));
            for (int i = 0; i < (1 << sb); ++i) tab[off + i] = 0;
            off += 1 << sb;
        }
    }
    for (int s = 0; s < n_sym; ++s) {
        const int l = lens[s];
        if (l == 0) continue;
        const uint32_t c = next_code[l]++;
        const uint32_t rev = reverse_bits(c, l);
        const uint32_t e = (KIND == 0 ? litlen_entry(s) : KIND == 1 ? dist_entry(s) : plain_entry(s)) | uint32_t(l);
        if (l <= main_bits) {
            for (uint32_t i = rev; i < main_size; i += 1u << l) tab[i] = e;
        } else {
            const uint32_t sub = tab[rev & (main_size - 1)];
            const uint32_t off = (sub >> 13) & 0x1FFFF, sb = (sub >> 8) & 31;
            for (uint32_t i = rev >> main_bits; i < (1u << sb); i += 1u << (l - main_bits)) tab[off + i] = e;
        }
    }
    return true;
}

// A decoded symbol of a batch: literal byte, or a match (length 3..258, distance 1..32768), or `n` bytes of a stored block
// to copy verbatim from the input.
struct Sym {
    uint32_t len;       // bytes this symbol produces
    uint32_t arg;       // literal: the byte; match: the distance; stored run: byte offset in the input
    uint32_t kind;      // 0 literal, 1 match, 2 stored run
};

struct State {
    const uint32_t* in32;       // payload, 4-byte aligned, readable 8 bytes beyond in_len
    uint32_t in_len;            // bytes
    uint32_t word;              // next 32-bit word to load
    uint64_t bitbuf;
    int bitcnt;
    uint32_t out_len, op;       // expected output size, bytes produced so far
    int phase;                  // 0 block header next, 1 inside a Huffman block, 2 inside a stored block, 3 done
    int final_block;
    uint32_t stored_left, stored_pos;
    int drop;                   // bits to discard after the next refill (byte position behind a stored block)
    int status;
};

__host__ __device__ inline void state_init(State& s, const uint8_t* in, uint32_t in_len, uint32_t out_len)
{
    s.in32 = reinterpret_cast<const uint32_t*>(in); s.in_len = in_len; s.word = 0; s.bitbuf = 0; s.bitcnt = 0;
    s.out_len = out_len; s.op = 0; s.phase = 0; s.final_block = 0; s.stored_left = 0; s.stored_pos = 0; s.drop = 0; s.status = kOk;
}
__host__ __device__ inline void refill(State& s)
{
    while (s.bitcnt <= 32) {
        const uint32_t max_word = (s.in_len + 3) / 4 + 1;                        // last byte read <= in_len + 6: inside the promised padding
        const uint32_t w = s.word < max_word ? s.in32[s.word] : 0u;
        s.bitbuf |= uint64_t(w) << s.bitcnt; s.bitcnt += 32; ++s.word;
    }
    if (s.drop) { s.bitbuf >>= s.drop; s.bitcnt -= s.drop; s.drop = 0; }       // <= 24 bits of >= 64: still > 32 valid bits
}
__host__ __device__ inline bool overrun(const State& s)
{
    // bits consumed so far = 32 * word - bitcnt; they must lie inside the input
    return uint64_t(s.word) * 32 - uint64_t(s.bitcnt) > uint64_t(s.in_len) * 8;
}

// Header of the next DEFLATE block; builds the tables of a Huffman block.  Returns false on error (s.status set).
__host__ __device__ inline bool next_block(State& s, Tables& T, uint8_t* lens /* >= 320 + 140 bytes of scratch */)
{
    refill(s);
    s.final_block = int(s.bitbuf & 1);
    const uint32_t type = uint32_t((s.bitbuf >> 1) & 3);
    s.bitbuf >>= 3; s.bitcnt -= 3;
    if (type == 0) {                                         // stored: LEN / NLEN on the next byte boundary
        const int drop = s.bitcnt & 7;
        s.bitbuf >>= drop; s.bitcnt -= drop;
        refill(s);
        const uint32_t len = uint32_t(s.bitbuf & 0xFFFF), nlen = uint32_t((s.bitbuf >> 16) & 0xFFFF);
        s.bitbuf >>= 32; s.bitcnt -= 32;
        if ((len ^ 0xFFFFu) != nlen) { s.status = kBadStored; return false; }
        const uint64_t pos_bits = uint64_t(s.word) * 32 - uint64_t(s.bitcnt);           // byte aligned here
        s.stored_pos = uint32_t(pos_bits >> 3); s.stored_left = len;
        if (uint64_t(s.stored_pos) + len > s.in_len || uint64_t(s.op) + len > s.out_len) { s.status = kBadStored; return false; }
        // skip the stored bytes in the bit reader; the words behind them are only touched by the next refill (the kernel may
        // have to move its input window first)
        const uint32_t after = s.stored_pos + len;
        s.word = after / 4; s.bitbuf = 0; s.bitcnt = 0; s.drop = int(after & 3) * 8;
        s.phase = 2;
        return true;
    }
    if (type == 3) { s.status = kBadStream; return false; }
    if (type == 1) {                                         // fixed code
        for (int i = 0; i < 144; ++i) lens[i] = 8;
        for (int i = 144; i < 256; ++i) lens[i] = 9;
        for (int i = 256; i < 280; ++i) lens[i] = 7;
        for (int i = 280; i < 288; ++i) lens[i] = 8;
        build_table<0>(lens, 288, kLitBits, T.lit, kLitTab);
        for (int i = 0; i < 32; ++i) lens[i] = 5;
        build_table<1>(lens, 32, kDistBits, T.dist, kDistTab);
        s.phase = 1;
        return true;
    }
    const uint32_t hlit = uint32_t(s.bitbuf & 31) + 257, hdist = uint32_t((s.bitbuf >> 5) & 31) + 1, hclen = uint32_t((s.bitbuf >> 10) & 15) + 4;
    s.bitbuf >>= 14; s.bitcnt -= 14;
    if (hlit > 286 || hdist > 30) { s.status = kBadTable; return false; }
    const uint8_t order[19] = { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };
    uint8_t pl[19];
    for (int i = 0; i < 19; ++i) pl[i] = 0;
    for (uint32_t i = 0; i < hclen; ++i) {
        refill(s);
        pl[order[i]] = uint8_t(s.bitbuf & 7);
        s.bitbuf >>= 3; s.bitcnt -= 3;
    }
    uint32_t* pre = T.dist;                                  // the code-length table (128 entries) borrows the distance table
    if (!build_table<2>(pl, 19, 7, pre, 1 << 7)) { s.status = kBadTable; return false; }
    uint32_t n = 0;
    while (n < hlit + hdist) {
        refill(s);
        const uint32_t e = pre[s.bitbuf & 127];
        const uint32_t l = e & 0xFF;
        if (l == 0) { s.status = kBadTable; return false; }
        s.bitbuf >>= l; s.bitcnt -= int(l);
        const uint32_t sym = (e >> 13) & 0x1FFFF;
        if (sym < 16) { lens[n++] = uint8_t(sym); continue; }
        uint32_t rep, val = 0;
        if (sym == 16) { if (n == 0) { s.status = kBadTable; return false; } val = lens[n - 1]; rep = 3 + uint32_t(s.bitbuf & 3); s.bitbuf >>= 2; s.bitcnt -= 2; }
        else if (sym == 17) { rep = 3 + uint32_t(s.bitbuf & 7); s.bitbuf >>= 3; s.bitcnt -= 3; }
        else { rep = 11 + uint32_t(s.bitbuf & 127); s.bitbuf >>= 7; s.bitcnt -= 7; }
        if (n + rep > hlit + hdist) { s.status = kBadTable; return false; }
        for (uint32_t i = 0; i < rep; ++i) lens[n + i] = uint8_t(val);
        n += rep;
    }
    if (lens[256] == 0) { s.status = kBadTable; return false; }                  // no end-of-block code
    // distance lengths first (they sit behind the literal/length ones), into their own 32-slot array
    uint8_t* dl = lens + 320;
    for (uint32_t i = 0; i < 32; ++i) dl[i] = i < hdist ? lens[hlit + i] : 0;
    for (uint32_t i = hlit; i < 288; ++i) lens[i] = 0;
    if (!build_table<0>(lens, 288, kLitBits, T.lit, kLitTab)) { s.status = kBadTable; return false; }
    if (!build_table<1>(dl, 32, kDistBits, T.dist, kDistTab)) { s.status = kBadTable; return false; }
    s.phase = 1;
    return true;
}

// Decode up to `cap` (<= 32) symbols; a call that meets a block header decodes the header and returns.  Returns the number of
// symbols decoded (0 is progress too when the phase or the input position moved); s.phase == 3 when the stream has ended,
// s.status != 0 on error.
constexpr uint32_t kMaxInputPerCall = 1024;        // bytes a call may read beyond the position it starts at (see above), with margin
__host__ __device__ inline int decode_batch(State& s, Tables& T, uint8_t* lens, Sym* batch, int cap)
{
    int n = 0;
    if (s.status != kOk || s.phase == 3) return 0;
    if (s.phase == 0) {
        // one header per call, and nothing after it: a call then reads less than kMaxInputPerCall bytes of input (header
        // <= 563 bytes, 32 symbols <= 192), and a stored block's jump ahead is followed by a return
        next_block(s, T, lens);
    } else if (s.phase == 2) {                               // stored run: at most 256 bytes per symbol keeps the apply step balanced
        while (n < cap && s.stored_left) {
            const uint32_t take = s.stored_left < 256u ? s.stored_left : 256u;
            batch[n].kind = 2; batch[n].len = take; batch[n].arg = s.stored_pos; ++n;
            s.stored_pos += take; s.stored_left -= take; s.op += take;
        }
        if (s.stored_left == 0) s.phase = s.final_block ? 3 : 0;
    } else {
        // Huffman block: the bit reader lives in registers for the whole batch (the State may sit in local memory)
        uint64_t bitbuf = s.bitbuf;
        int bitcnt = s.bitcnt;
        uint32_t word = s.word, op = s.op;
        const uint32_t* in32 = s.in32;
        const uint32_t max_word = (s.in_len + 3) / 4 + 1, out_len = s.out_len;     // last byte read <= in_len + 6: inside the promised padding
        int drop = s.drop, status = kOk, phase = 1;
#define VTX_REFILL()                                                                                              \
        do {                                                                                                      \
            while (bitcnt <= 32) { const uint32_t w_ = word < max_word ? in32[word] : 0u; bitbuf |= uint64_t(w_) << bitcnt; bitcnt += 32; ++word; } \
            if (drop) { bitbuf >>= drop; bitcnt -= drop; drop = 0; }                                              \
        } while (0)
        while (n < cap) {
            VTX_REFILL();                                        // > 32 valid bits: one literal/length code (<= 15 + 5)
            uint32_t e = T.lit[uint32_t(bitbuf) & ((1u << kLitBits) - 1)];
            if ((e & kTypeMask) == kTypeSub) e = T.lit[((e >> 13) & 0x1FFFF) + (uint32_t(bitbuf >> kLitBits) & ((1u << ((e >> 8) & 31)) - 1))];
            uint32_t l = e & 0xFF;
            if (l == 0) { status = kBadStream; break; }
            bitbuf >>= l; bitcnt -= int(l);
            const uint32_t type = e & kTypeMask;
            if (type == kTypeLiteral) {
                if (op >= out_len) { status = kBadSize; break; }
                batch[n].kind = 0; batch[n].len = 1; batch[n].arg = (e >> 13) & 0xFF; ++n; ++op;
                continue;
            }
            if (type == kTypeEnd) {
                if ((e >> 13) & 0x1FFFF) { status = kBadStream; break; }           // symbols 286 / 287
                phase = s.final_block ? 3 : 0;                                      // the next call reads the next header
                break;
            }
            const uint32_t xb = (e >> 8) & 31;
            const uint32_t length = ((e >> 13) & 0x1FFFF) + (uint32_t(bitbuf) & ((1u << xb) - 1));
            bitbuf >>= xb; bitcnt -= int(xb);
            VTX_REFILL();                                        // distance code (<= 15) + extra bits (<= 13)
            uint32_t d = T.dist[uint32_t(bitbuf) & ((1u << kDistBits) - 1)];
            if ((d & kTypeMask) == kTypeSub) d = T.dist[((d >> 13) & 0x1FFFF) + (uint32_t(bitbuf >> kDistBits) & ((1u << ((d >> 8) & 31)) - 1))];
            l = d & 0xFF;
            if (l == 0 || (d & kTypeMask) != kTypeBase) { status = kBadStream; break; }
            bitbuf >>= l; bitcnt -= int(l);
            const uint32_t db = (d >> 8) & 31;
            const uint32_t distance = ((d >> 13) & 0x1FFFF) + (uint32_t(bitbuf) & ((1u << db) - 1));
            bitbuf >>= db; bitcnt -= int(db);
            if (distance > op) { status = kBadDistance; break; }
            if (uint64_t(op) + length > out_len) { status = kBadSize; break; }
            batch[n].kind = 1; batch[n].len = length; batch[n].arg = distance; ++n; op += length;
        }
#undef VTX_REFILL
        s.bitbuf = bitbuf; s.bitcnt = bitcnt; s.word = word; s.op = op; s.drop = drop; s.status = status; s.phase = phase;
        if (status == kOk && phase != 1 && overrun(s)) s.status = kOverrun;      // at the end of a block the bits consumed lie inside the input
    }
    if (s.phase == 3 && s.status == kOk) {
        if (overrun(s)) s.status = kOverrun;
        else if (s.op != s.out_len) s.status = kBadSize;
    }
    return n;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------------------------
// the warp-level kernel
// ---------------------------------------------------------------------------------------------------------------
// Output goes straight to global memory: a match copy is a dependent L2 round trip and lane 0's symbol decode a chain of
// dependent ALU and shared-memory operations, so a warp takes milliseconds per 64 KB member -- and what buys throughput is
// the number of members in flight: 20 warps per SM hide each other's latencies.  The alternative, the member's output
// assembled in 64 KB of shared memory by a lone warp per CTA, is faster per member but fits only 2 CTAs on an SM.
#ifndef VTX_INFLATE_PIPELINE
#define VTX_INFLATE_PIPELINE 1
#endif
constexpr int kInflateWarps = 4;                  // per CTA
constexpr int kBatch = 32;

struct BlockDesc {                 // one BGZF member
    uint64_t in_off;               // byte offset of its DEFLATE payload in `comp` (multiple of 4; 8 readable bytes behind it)
    uint32_t in_len;
    uint32_t out_len;              // ISIZE from the gzip trailer (<= 65536)
    uint64_t out_off;              // byte offset of its output in `out`
    uint32_t crc32;                // expected CRC-32 of the output (gzip trailer)
    uint32_t pad;
};

constexpr int kInWords = 512;                     // input window per warp: 2 KB of the member's payload in shared memory
static_assert(kMaxInputPerCall % 4 == 0 && kInWords * 4 >= 2 * int(kMaxInputPerCall), "a call must fit behind any start inside the first half");

struct WarpShared {
    Tables T;
    uint8_t lens[512];
#if VTX_INFLATE_PIPELINE
    Sym batch2[2][kBatch];         // decoded by lane 0 while the other lanes apply the previous one
    int n2[2], done2[2];
#else
    Sym batch[kBatch];
#endif
    uint32_t in_win[kInWords];     // payload words [win_first, win_first + kInWords): the bit reader's refills never leave it
    int n, status, done;
    uint32_t reload;               // first word of the window to load next, or ~0
};
__host__ __device__ constexpr size_t inflate_smem_bytes() { return sizeof(WarpShared) * kInflateWarps + 256 * 4; }

// CRC-32 (IEEE, reflected) of a member's output by the whole warp: every lane takes a contiguous slice, the slices are
// combined with x^(8 len) mod P multiplications (the classic crc32_combine, done as 32 shift/xor steps per power).
__device__ __forceinline__ uint32_t crc_mul(uint32_t a, uint32_t b)       // a * b mod P in the reflected representation
{
    uint32_t p = 0;
    for (int i = 0; i < 32; ++i) {
        if (a & 0x80000000u) p ^= b;
        a <<= 1;
        b = (b >> 1) ^ ((b & 1u) ? 0xEDB88320u : 0u);
    }
    return p;
}
__device__ __forceinline__ uint32_t crc_xpow8n(uint32_t n_bytes)           // x^(8 n) mod P
{
    uint32_t r = 0x80000000u;              // x^0
    uint32_t sq = 0x00800000u;             // x^8
    while (n_bytes) {
        if (n_bytes & 1) r = crc_mul(r, sq);
        sq = crc_mul(sq, sq);
        n_bytes >>= 1;
    }
    return r;
}
__device__ uint32_t warp_crc32(const uint8_t* p, uint32_t n, const uint32_t* table /* 256 entries, shared */)
{
    const int lane = threadIdx.x & 31;
    const uint32_t per = (n + 31) / 32;
    const uint32_t b0 = min(n, per * uint32_t(lane)), b1 = min(n, b0 + per);
    uint32_t c = 0;                                     // raw register value without the 0xFFFFFFFF pre/post conditioning
    for (uint32_t i = b0; i < b1; ++i) c = table[(c ^ __ldcg(p + i)) & 0xFF] ^ (c >> 8);
    // combine left to right: crc(A || B) = crc(A) * x^(8 |B|) + crc(B) for the linear part; the conditioning is added at the end
    // tree combine: at each level a lane absorbs its right neighbour's slice
    uint32_t len = b1 - b0;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t oc = __shfl_down_sync(0xffffffffu, c, o);
        const uint32_t ol = __shfl_down_sync(0xffffffffu, len, o);
        if ((lane & (2 * o - 1)) == 0) { c = crc_mul(c, crc_xpow8n(ol)) ^ oc; len += ol; }
    }
    // conditioning: crc = raw(init = 0xFFFFFFFF) ^ 0xFFFFFFFF, and raw(init) = raw(0) ^ 0xFFFFFFFF * x^(8 n)
    uint32_t full = c ^ crc_mul(0xFFFFFFFFu, crc_xpow8n(n)) ^ 0xFFFFFFFFu;
    return __shfl_sync(0xffffffffu, full, 0);
}

__global__ void __launch_bounds__(kInflateWarps * 32) vtx_k_bgzf_inflate(const BlockDesc* __restrict__ blocks, uint32_t n_blocks,
                                                                          const uint8_t* __restrict__ comp, uint8_t* __restrict__ out,
                                                                          int32_t* __restrict__ status, uint32_t* __restrict__ cursor, int check_crc)
{
    extern __shared__ __align__(16) uint8_t inflate_smem[];
    WarpShared* ws_all = reinterpret_cast<WarpShared*>(inflate_smem);
    uint32_t* crc_table = reinterpret_cast<uint32_t*>(inflate_smem + sizeof(WarpShared) * kInflateWarps);
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ ((c & 1u) ? 0xEDB88320u : 0u);
        crc_table[i] = c;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpShared& ws = ws_all[warp];
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(cursor, 1u);
        b = __shfl_sync(0xffffffffu, b, 0);
        if (b >= n_blocks) break;
        const BlockDesc bd = blocks[b];
        uint8_t* o = out + bd.out_off;
        State st;
        const uint32_t* in_g = reinterpret_cast<const uint32_t*>(comp + bd.in_off);
        const uint32_t max_word = (bd.in_len + 3) / 4 + 1;           // as in refill(): words behind it read as zero
        uint32_t win_first = 0;
        if (lane == 0) {
            state_init(st, comp + bd.in_off, bd.in_len, bd.out_len);
            if (bd.out_len > 65536u || (bd.in_off & 3)) st.status = kBadSize;
            ws.done = 0; ws.reload = 0;
        }
#if VTX_INFLATE_PIPELINE
        // Lane 0 decodes batch k + 1 while lanes 1..31 apply batch k: the two are latency chains of different kinds (ALU /
        // shared-memory lookups there, L2 round trips of the match copies here) and the divergent halves of the warp are
        // scheduled independently, so they hide each other.  Batches hold at most 31 symbols: one per applying lane.
        uint32_t op = 0;
        constexpr uint32_t kApply = 0xFFFFFFFEu;
        auto load_window = [&]() {                       // all 32 lanes
            __syncwarp();
            const uint32_t reload = ws.reload;
            if (reload != 0xFFFFFFFFu) {
                for (int i = lane; i < kInWords; i += 32) ws.in_win[i] = reload + i < max_word ? __ldg(in_g + reload + i) : 0u;
                win_first = reload;
            }
            __syncwarp();
        };
        auto decode_into = [&](int buf) {                // lane 0
            st.in32 = ws.in_win - win_first;             // in32[word] for word in [win_first, win_first + kInWords)
            ws.n2[buf] = st.status == kOk ? decode_batch(st, ws.T, ws.lens, ws.batch2[buf], kBatch - 1) : 0;
            ws.status = st.status; ws.done2[buf] = (st.phase == 3 || st.status != kOk) ? 1 : 0;
            // refills of the next call touch words [st.word, st.word + kMaxInputPerCall / 4 + 2)
            ws.reload = (st.word < win_first || st.word + kMaxInputPerCall / 4 + 2 > win_first + kInWords) ? st.word : 0xFFFFFFFFu;
        };
        load_window();
        if (lane == 0) decode_into(0);
        for (int cur = 0;; cur ^= 1) {
            load_window();                               // also publishes batch `cur` and its flags to every lane
            const int last = ws.done2[cur];
            if (lane == 0) {
                if (!last) decode_into(cur ^ 1);
            } else {
                const int n = ws.n2[cur], idx = lane - 1;
                Sym sy{ 0, 0, 0 };
                if (idx < n) sy = ws.batch2[cur][idx];
                uint32_t incl = sy.len;                  // exclusive scan of the symbol lengths over lanes 1..31
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(kApply, incl, d); if (idx >= d) incl += up; }
                const uint32_t my_pos = op + incl - sy.len;
                const uint32_t total = __shfl_sync(kApply, incl, 31);
                if (idx < n && sy.kind == 0) o[my_pos] = uint8_t(sy.arg);                    // all literals of the batch at once
                __syncwarp(kApply);
                uint32_t heavy = __ballot_sync(kApply, idx < n && sy.kind != 0);             // matches and stored runs, in stream order
                while (heavy) {
                    const int src_lane = __ffs(heavy) - 1;
                    heavy &= heavy - 1;
                    const uint32_t len = __shfl_sync(kApply, sy.len, src_lane), arg = __shfl_sync(kApply, sy.arg, src_lane);
                    const uint32_t kind = __shfl_sync(kApply, sy.kind, src_lane), pos = __shfl_sync(kApply, my_pos, src_lane);
                    if (kind == 1) {
                        const uint8_t* srcp = o + pos - arg;
                        if (arg >= len) { for (uint32_t i = idx; i < len; i += 31) o[pos + i] = __ldcg(srcp + i); }
                        else { for (uint32_t i = idx; i < len; i += 31) o[pos + i] = __ldcg(srcp + (i % arg)); }
                    } else {
                        const uint8_t* srcp = comp + bd.in_off + arg;
                        for (uint32_t i = idx; i < len; i += 31) o[pos + i] = __ldg(srcp + i);
                    }
                    __syncwarp(kApply);
                }
                op += total;
            }
            if (last) break;
        }
        __syncwarp();
#else
        uint32_t op = 0;
        for (;;) {
            // the dependent chain of the bit reader runs on shared memory: the warp moves the window when the next call could
            // leave it (an L2 round trip per ~1 KB of input instead of one per 4 bytes)
            __syncwarp();
            const uint32_t reload = ws.reload;
            if (reload != 0xFFFFFFFFu) {
                for (int i = lane; i < kInWords; i += 32) ws.in_win[i] = reload + i < max_word ? __ldg(in_g + reload + i) : 0u;
                win_first = reload;
            }
            __syncwarp();
            if (lane == 0) {
                st.in32 = ws.in_win - win_first;                   // in32[word] for word in [win_first, win_first + kInWords)
                ws.n = st.status == kOk ? decode_batch(st, ws.T, ws.lens, ws.batch, kBatch) : 0;
                ws.status = st.status; ws.done = (st.phase == 3 || st.status != kOk) ? 1 : 0;
                // refills of the next call touch words [st.word, st.word + kMaxInputPerCall / 4 + 2)
                ws.reload = (st.word < win_first || st.word + kMaxInputPerCall / 4 + 2 > win_first + kInWords) ? st.word : 0xFFFFFFFFu;
            }
            __syncwarp();
            const int n = ws.n;
            // positions: exclusive scan of the symbol lengths
            Sym sy{ 0, 0, 0 };
            if (lane < n) sy = ws.batch[lane];
            uint32_t incl = sy.len;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += up; }
            const uint32_t my_pos = op + incl - sy.len;
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            if (lane < n && sy.kind == 0) o[my_pos] = uint8_t(sy.arg);                   // all literals of the batch at once
            __syncwarp();
            uint32_t heavy = __ballot_sync(0xffffffffu, lane < n && sy.kind != 0);       // matches and stored runs, in stream order
            while (heavy) {
                const int src_lane = __ffs(heavy) - 1;
                heavy &= heavy - 1;
                const uint32_t len = __shfl_sync(0xffffffffu, sy.len, src_lane), arg = __shfl_sync(0xffffffffu, sy.arg, src_lane);
                const uint32_t kind = __shfl_sync(0xffffffffu, sy.kind, src_lane), pos = __shfl_sync(0xffffffffu, my_pos, src_lane);
                if (kind == 1) {
                    const uint8_t* srcp = o + pos - arg;
                    if (arg >= len) { for (uint32_t i = lane; i < len; i += 32) o[pos + i] = __ldcg(srcp + i); }
                    else { for (uint32_t i = lane; i < len; i += 32) o[pos + i] = __ldcg(srcp + (i % arg)); }
                } else {
                    const uint8_t* srcp = comp + bd.in_off + arg;
                    for (uint32_t i = lane; i < len; i += 32) o[pos + i] = __ldg(srcp + i);
                }
                __syncwarp();
            }
            op += total;
            if (ws.done) break;
            __syncwarp();
        }
#endif
        int stt = ws.status;
        if (stt == kOk && check_crc) {
            __syncwarp();
            if (warp_crc32(o, bd.out_len, crc_table) != bd.crc32) stt = 7;               // CRC mismatch
        }
        if (lane == 0) status[b] = stt;
        __syncwarp();
    }
}
#endif   // __CUDACC__

}  // namespace inflate
}  // namespace vtx
