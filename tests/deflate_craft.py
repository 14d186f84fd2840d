"""Raw DEFLATE (RFC 1951) written by hand, for the decoder tests.

zlib's compressor only ever writes the stream shapes its own heuristics choose.  This module writes any shape a test asks
for: stored, fixed and dynamic blocks from an explicit list of literals and matches, dynamic headers with given code
lengths (with or without the run-length codes 16 / 17 / 18), a chosen length symbol for 258, blocks cut wherever the test
wants them.  `corpus()` is the set of streams the CPU and GPU inflate tests share; every valid stream in it is checked
against zlib before use, and every invalid one is checked to be refused by zlib.
"""
from __future__ import annotations

import random
import zlib

# RFC 1951 3.2.5: length symbols 257..285 and distance symbols 0..29 -> (base, extra bits)
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def bits(self, v: int, n: int):
        """n bits of v, least significant first"""
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def code(self, c: int, n: int):
        """a Huffman code: most significant bit first"""
        self.bits(int(format(c, f"0{n}b")[::-1], 2) if n else 0, n)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def getvalue(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lengths):
    """code lengths -> canonical codes (RFC 1951 3.2.2); 0 = unused"""
    mx = max(lengths, default=0)
    count = [0] * (mx + 1)
    for l in lengths:
        if l:
            count[l] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lengths:
        if l:
            out.append(nxt[l]); nxt[l] += 1
        else:
            out.append(None)
    return out


def limited_lengths(freq, maxlen: int):
    """Huffman code lengths for `freq` (symbols with freq 0 get length 0), at most `maxlen` bits, complete whenever two or
    more symbols are used"""
    import heapq
    used = [i for i, f in enumerate(freq) if f > 0]
    L = [0] * len(freq)
    if len(used) == 1:
        L[used[0]] = 1
        return L
    if not used:
        return L
    h = [(freq[i], k, [i]) for k, i in enumerate(used)]
    heapq.heapify(h)
    tick = len(h)
    while len(h) > 1:
        f1, _, a = heapq.heappop(h); f2, _, b = heapq.heappop(h)
        for i in a + b:
            L[i] += 1
        tick += 1
        heapq.heappush(h, (f1 + f2, tick, a + b))
    for i in used:
        L[i] = min(L[i], maxlen)
    one = 1 << maxlen
    kraft = sum(one >> L[i] for i in used)
    while kraft > one:                               # over-subscribed after clamping: lengthen the longest short code
        i = max((i for i in used if L[i] < maxlen), key=lambda i: L[i])
        kraft -= one >> (L[i] + 1); L[i] += 1
    while kraft < one:                               # incomplete: shorten a longest code whose step still fits
        i = max((i for i in used if (one >> L[i]) <= one - kraft and L[i] > 1), key=lambda i: L[i])
        kraft += one >> L[i]; L[i] -= 1
    return L


def len_symbol(length: int, sym258: int = 285):
    """-> (symbol, extra value, extra bits); 258 as symbol 285 (no extra bits) or as 284 with extra 31"""
    if length == 258 and sym258 == 284:
        return 284, 31, 5
    for s in range(28, -1, -1):
        if LEN_BASE[s] <= length and (s == 28 or length < 258):
            if s == 28 and length != 258:
                continue
            return 257 + s, length - LEN_BASE[s], LEN_EXTRA[s]
    raise ValueError(length)


def dist_symbol(d: int):
    for s in range(29, -1, -1):
        if DIST_BASE[s] <= d:
            return s, d - DIST_BASE[s], DIST_EXTRA[s]
    raise ValueError(d)


def lit(data: bytes):
    return [("L", b) for b in data]


def match(length: int, dist: int, sym258: int = 285):
    return [("M", length, dist, sym258)]


def expand(tokens, prefix: bytes = b"") -> bytes:
    """the bytes a token list produces behind `prefix` (the output so far)"""
    out = bytearray(prefix)
    for t in tokens:
        if t[0] == "L":
            out.append(t[1])
        else:
            _, n, d, _ = t
            for _ in range(n):
                out.append(out[-d])
    return bytes(out[len(prefix):])


def _symbols(tokens):
    for t in tokens:
        if t[0] == "L":
            yield t[1], None
        else:
            s, ev, eb = len_symbol(t[1], t[3])
            yield s, (ev, eb, dist_symbol(t[2]))


def _write_tokens(w, tokens, lcodes, llens, dcodes, dlens):
    for s, ext in _symbols(tokens):
        w.code(lcodes[s], llens[s])
        if ext:
            ev, eb, (ds, dv, db) = ext
            w.bits(ev, eb)
            w.code(dcodes[ds], dlens[ds])
            w.bits(dv, db)
    w.code(lcodes[256], llens[256])


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def stored(w: BitWriter, data: bytes, final: bool, nlen_xor: int = 0xFFFF):
    w.bits(int(final), 1); w.bits(0, 2); w.align()
    w.bits(len(data), 16); w.bits(len(data) ^ nlen_xor, 16)
    for b in data:
        w.bits(b, 8)


def fixed(w: BitWriter, tokens, final: bool):
    w.bits(int(final), 1); w.bits(1, 2)
    _write_tokens(w, tokens, canonical(FIXED_LIT), FIXED_LIT, canonical(FIXED_DIST), FIXED_DIST)


def _rle(lengths, use_repeats: bool):
    """code-length sequence -> list of (symbol, extra value, extra bits)"""
    out, i = [], 0
    while i < len(lengths):
        v = lengths[i]
        run = 1
        while i + run < len(lengths) and lengths[i + run] == v:
            run += 1
        if not use_repeats:
            out.append((v, 0, 0)); i += 1
            continue
        if v == 0 and run >= 3:
            k = min(run, 138)
            out.append((18, k - 11, 7) if k >= 11 else (17, k - 3, 3)); i += k
        elif v != 0 and run >= 4:
            out.append((v, 0, 0))
            k = min(run - 1, 6)
            out.append((16, k - 3, 2)); i += 1 + k
        else:
            out.append((v, 0, 0)); i += 1
    return out


def dynamic(w: BitWriter, tokens, final: bool, lit_lens=None, dist_lens=None, use_repeats: bool = True, all_hclen: bool = False,
            hlit: int | None = None, hdist: int | None = None):
    """A dynamic block.  Code lengths default to Huffman lengths of the tokens (<= 15 bits); `hlit` / `hdist` pad the
    length lists with zeros."""
    lf = [0] * 286; df = [0] * 30
    for s, ext in _symbols(tokens):
        lf[s] += 1
        if ext:
            df[ext[2][0]] += 1
    lf[256] += 1
    if lit_lens is None:
        lit_lens = limited_lengths(lf, 15)
    if dist_lens is None:
        dist_lens = limited_lengths(df, 15)
        if not any(dist_lens):
            dist_lens = [0]
    nl = hlit or max(257, max(i for i, l in enumerate(lit_lens) if l) + 1)
    nd = hdist or max(1, max((i for i, l in enumerate(dist_lens) if l), default=0) + 1)
    ll = (list(lit_lens) + [0] * 286)[:nl]; dl = (list(dist_lens) + [0] * 30)[:nd]
    seq = _rle(ll + dl, use_repeats)
    cf = [0] * 19
    for s, _, _ in seq:
        cf[s] += 1
    cl_lens = limited_lengths(cf, 7)
    nc = 19 if all_hclen else max(4, max(k for k in range(19) if cl_lens[CL_ORDER[k]]) + 1)
    w.bits(int(final), 1); w.bits(2, 2)
    w.bits(nl - 257, 5); w.bits(nd - 1, 5); w.bits(nc - 4, 4)
    for k in range(nc):
        w.bits(cl_lens[CL_ORDER[k]], 3)
    cc = canonical(cl_lens)
    for s, ev, eb in seq:
        w.code(cc[s], cl_lens[s]); w.bits(ev, eb)
    _write_tokens(w, tokens, canonical(ll + [0] * (288 - nl)), ll + [0] * (288 - nl), canonical(dl + [0] * (30 - nd)), dl + [0] * (30 - nd))


def build(blocks) -> tuple[bytes, bytes]:
    """blocks: list of ("stored", data) / ("fixed", tokens) / ("dynamic", tokens, kwargs); the last block is
    final.  -> (stream, expected output)"""
    w = BitWriter()
    out = bytearray()
    for k, b in enumerate(blocks):
        final = k == len(blocks) - 1
        if b[0] == "stored":
            stored(w, b[1], final); out += b[1]
        elif b[0] == "fixed":
            fixed(w, b[1], final); out += expand(b[1], bytes(out))
        elif b[0] == "dynamic":
            dynamic(w, b[1], final, **(b[2] if len(b) > 2 else {})); out += expand(b[1], bytes(out))
        else:
            raise ValueError(b[0])
    return w.getvalue(), bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# the corpus
# ---------------------------------------------------------------------------------------------------------------------
def _rand(rng, n):
    return bytes(rng.randrange(256) for _ in range(n))


def largest_header_lengths(seed: int = 3):
    """complete code lengths over all 286 literal/length and all 30 distance symbols, spread over many lengths (up to 15 bits)
    so that the code-length code is deep: written with HLIT 286, HDIST 30, HCLEN 19 and no repeat codes, the largest header"""
    rng = random.Random(seed)
    return (limited_lengths([1 + rng.randrange(1 << rng.randrange(15)) for _ in range(286)], 15),
            limited_lengths([1 + rng.randrange(1 << rng.randrange(15)) for _ in range(30)], 15))


def batches(tokens, cap: int = 31):
    """the symbol batches the device decoder forms inside one Huffman block (the block header is a call of its own)"""
    return [tokens[i:i + cap] for i in range(0, len(tokens), cap)]


def corpus(seed: int = 7):
    """-> list of (name, stream, expected bytes or None when zlib must refuse it, facts dict)"""
    rng = random.Random(seed)
    cases = []

    def add(name, blocks, **facts):
        s, out = build(blocks)
        huff = [b[1] for b in blocks if b[0] != "stored"]
        facts["match_batch31"] = any(len(bt) == 31 and all(t[0] == "M" for t in bt) for toks in huff for bt in batches(toks))
        cases.append((name, s, out, facts))

    # ---- batch seams: symbols per batch (<= 31 per decode call), lane 0 one batch ahead, match copies of stride 31
    for nlit in range(29, 34):
        base = _rand(rng, nlit)
        for kind in ("fixed", "dynamic"):
            add(f"lits{nlit}_then_match_{kind}", [(kind, lit(base) + match(40, nlit) + lit(b"xyz"))])
    for nm in (30, 31, 32, 33, 62, 63):
        toks = lit(_rand(rng, 300))
        for k in range(nm):
            toks += match(3 + (k * 7) % 256, 1 + (k * 37) % 290)
        add(f"matches{nm}_consecutive", [("dynamic", toks)], consecutive_matches=nm)
    for d in list(range(1, 34)) + [255, 256, 257, 32767, 32768]:
        for L in (3, 4, 5, 30, 31, 32, 33, 62, 63, 64, 100, 257, 258):
            if d < 34 and L not in (3, 31, 32, 33, 63, 258) and d not in (1, 2, 3, 7, 31, 32, 33):
                continue
            if d >= 34 and L not in (3, 258):
                continue
            pre = _rand(rng, max(d, 5))
            toks = match(L, d) + (match(258, d, 284) if L == 258 else [])        # 258 also as symbol 284 + extra 31
            # long distances take their source from a stored block, short ones from literals of the same block
            add(f"dist{d}_len{L}", [("stored", pre), ("dynamic", toks)] if d > 1000 else [("dynamic", lit(pre) + toks)])
    # a match whose source is a literal of the same batch, and one whose source lies in the previous batch
    for lead in (1, 10, 29, 30):
        pre = _rand(rng, lead)
        add(f"match_src_same_batch_{lead}", [("fixed", lit(pre) + match(20, lead) + lit(_rand(rng, 40)) + match(45, 41))])
    toks = lit(_rand(rng, 31)) + lit(_rand(rng, 31)) + match(200, 40) + lit(b"q") * 31 + match(258, 250)
    add("match_src_previous_batch", [("fixed", toks)])

    # ---- window seams: the largest dynamic header at every payload offset near 1024 and 2048
    big_ll, big_dl = largest_header_lengths()
    body = lit(_rand(rng, 50)) + match(30, 7) + lit(b"end")
    for target in (1024, 2048):
        for delta in range(-64, 65):
            start = target + delta
            # stored block lead-in: 5 bytes of header per stored block (header bits sit at byte `start` once we are aligned)
            lead = _rand(rng, start - 5)
            blocks = [("stored", lead), ("dynamic", body, dict(lit_lens=big_ll, dist_lens=big_dl, use_repeats=False, all_hclen=True))]
            s, out = build(blocks)
            cases.append((f"big_header_at_{start}", s, out, dict(header_at=start)))
    # stored blocks of every small length with their payload at every input offset mod 4, and of 65 535 bytes; empty blocks in
    # front move the payload without adding output (a member stays within 64 KiB)
    prefixes = {}
    for pre in [[("fixed", [])] * k for k in range(5)] + [[("stored", b"")] + [("fixed", [])] * k for k in range(4)]:
        s, _ = build(pre + [("stored", b"xyz")])
        prefixes.setdefault((len(s) - 3) % 4, pre)
    assert sorted(prefixes) == [0, 1, 2, 3]
    for n in (0, 1, 2, 3, 4, 255, 256, 257, 65535):
        for align in range(4):
            data = _rand(rng, n)
            blocks = prefixes[align] + [("stored", data)] + ([("fixed", lit(b"ab"))] if n < 65535 else [])
            add(f"stored{n}_align{align}", blocks, payload_mod4=align)
    add("stored_fixed_dynamic_stored", [("stored", _rand(rng, 777)), ("fixed", lit(b"hello") + match(100, 3)),
                                        ("dynamic", lit(_rand(rng, 300)) + match(258, 301)), ("stored", _rand(rng, 333))])
    add("fixed_blocks_2000", [("fixed", lit(bytes([rng.randrange(256)]))) for _ in range(2000)])
    add("empty_final_block_fixed", [("fixed", lit(_rand(rng, 100))), ("fixed", [])])
    add("empty_final_block_stored", [("fixed", lit(_rand(rng, 100))), ("stored", b"")])
    add("empty_stream_fixed", [("fixed", [])])
    add("empty_stream_dynamic", [("dynamic", [])])

    # ---- table seams
    # 15-bit codes in both alphabets: literal/length lengths 1..7 then 256 codes of 15 bits; distances 1..14, 15, 15
    ll = [0] * 286
    order = list(range(256)) + [256] + list(range(257, 286))
    rng.shuffle(order)
    order.remove(256); order = [256] + order
    for k, s in enumerate(order[:7]):
        ll[s] = k + 1
    for s in order[7:263]:
        ll[s] = 15
    dl = [0] * 30
    dorder = list(range(30)); rng.shuffle(dorder)
    for k, s in enumerate(dorder[:14]):
        dl[s] = k + 1
    dl[dorder[14]] = 15; dl[dorder[15]] = 15
    lits = [s for s in range(256) if ll[s]]
    toks = lit(bytes(rng.choice(lits) for _ in range(600)))
    lens_ok = [L for L in range(3, 259) if ll[len_symbol(L)[0]]]
    for k in range(200):
        L = rng.choice(lens_ok)
        dsyms = [s for s in range(30) if dl[s] and DIST_BASE[s] <= 600]
        ds = rng.choice(dsyms)
        d = DIST_BASE[ds] + rng.randrange(1 << DIST_EXTRA[ds]) if DIST_EXTRA[ds] else DIST_BASE[ds]
        toks += match(L, min(d, 600))
    toks = [t for t in toks if t[0] == "L" or dl[dist_symbol(t[2])[0]]]
    add("codes15_both_alphabets", [("dynamic", toks, dict(lit_lens=ll, dist_lens=dl))], long_codes=True)
    add("single_distance_code", [("dynamic", lit(_rand(rng, 20)) + match(10, 4) + match(77, 4))])
    add("no_distance_codes", [("dynamic", lit(_rand(rng, 500)), dict(dist_lens=[0]))])
    # every distance code, maximal extra bits
    pre = _rand(rng, 32768)
    toks = []
    for s in range(30):
        toks += match(258, DIST_BASE[s] + (1 << DIST_EXTRA[s]) - 1)
    add("all_distance_codes_max_extra", [("stored", pre), ("dynamic", toks)])
    # repeat codes 16 / 17 / 18 at the start and at the end of the length lists
    ll = [0] * 20 + [8] * 256 + [0] * 10                        # 18 first; the zeros at the end run into the distance list
    dl = [0] * 26 + [2] * 4                                     # ... which ends with 2 and a 16
    usable = [s for s in range(256) if ll[s]]
    add("repeat_codes_18_first_16_last", [("dynamic", lit(bytes(rng.choice(usable) for _ in range(300))), dict(lit_lens=ll, dist_lens=dl))])
    ll = [0] * 5 + [8] * 256 + [0] * 25                         # 17 first
    dl = [1, 1, 0, 0, 0]                                        # 17 last
    usable = [s for s in range(256) if ll[s]]
    add("repeat_codes_17_first_17_last", [("dynamic", lit(bytes(rng.choice(usable) for _ in range(300))) + match(5, 2), dict(lit_lens=ll, dist_lens=dl, hdist=5))])
    add("len258_as_285_and_284", [("fixed", lit(b"Z") + match(258, 1) + match(258, 1, 284) + match(227, 1) + match(258, 1, 284))])

    # ---- invalid streams (one flaw each); expected None: zlib must refuse them
    def bad(name, s):
        cases.append((name, s, None, {}))

    w = BitWriter(); fixed(w, lit(b"abc") + match(5, 4), True); bad("distance_beyond_output", w.getvalue())
    for sym in (286, 287):
        w = BitWriter(); w.bits(1, 1); w.bits(1, 2)
        c = canonical(FIXED_LIT)
        for b in b"ab":
            w.code(c[b], FIXED_LIT[b])
        w.code(c[sym], 8); w.bits(0, 16)
        bad(f"litlen_symbol_{sym}", w.getvalue())
    for ds in (30, 31):
        w = BitWriter(); w.bits(1, 1); w.bits(1, 2)
        c = canonical(FIXED_LIT)
        for b in b"abcd":
            w.code(c[b], FIXED_LIT[b])
        w.code(c[257], 7); w.code(ds, 5); w.bits(0, 16)
        bad(f"distance_symbol_{ds}", w.getvalue())
    w = BitWriter(); stored(w, b"hello", True, nlen_xor=0xFFFE); bad("stored_len_nlen_mismatch", w.getvalue())
    w = BitWriter(); dynamic(w, lit(b"abc"), True, lit_lens=[8] * 256 + [7] + [0] * 29, dist_lens=[1]); bad("oversubscribed_litlen", w.getvalue())
    w = BitWriter(); dynamic(w, lit(b"abc"), True, lit_lens=[9] * 256 + [9] + [0] * 29, dist_lens=[1]); bad("incomplete_litlen", w.getvalue())
    w = BitWriter(); dynamic(w, lit(b"abc") + match(3, 3), True, dist_lens=[1, 1, 1]); bad("oversubscribed_dist", w.getvalue())
    w = BitWriter(); dynamic(w, lit(b"abc") + match(3, 3), True, dist_lens=[2, 2, 2]); bad("incomplete_dist", w.getvalue())
    s, _ = build([("dynamic", lit(_rand(rng, 200)) + match(50, 100), dict(lit_lens=big_ll, dist_lens=big_dl, use_repeats=False, all_hclen=True))])
    bad("truncated_in_header", s[:100])
    w = BitWriter(); fixed(w, lit(b"abc"), False); bad("no_final_block", w.getvalue())
    for name, s, out, facts in cases:
        if out is None:
            try:
                zlib.decompress(s, -15)
            except zlib.error:
                continue
            raise AssertionError(f"{name}: zlib accepts a stream meant to be invalid")
        assert zlib.decompress(s, -15) == out, name
    return cases


def too_long(cases):
    """valid streams, announced one byte shorter than they decode (output longer than ISIZE)"""
    return [(n + "_isize_short", s, len(o) - 1) for n, s, o, _ in cases if o]
