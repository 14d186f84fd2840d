"""Planted-seam cases for the Smith-Waterman kernels (CPU only: numpy and tests/sw_ref.py, no GPU import).

Every tiled kernel cuts the DP matrix into pieces and hands state from one piece to the next: lane seams (__shfl_up of
(H + gap, E)), the pass seams of the multi-pass class, the phase seam of the two-phase kernel, the forward boundary,
the 19-row lane blocks and the junction of the folded kernel, and the row blocks of reads longer than 1 024 bases.
A dropped or mis-indexed carry only changes a score when the optimal alignment crosses that seam in that way, so
random reads rarely see it.  Here every read is planted across a named seam of the kernel family it is routed to:

    "del"         a 2-6 base deletion across the seam (a horizontal gap, E, crosses it)
    "run"         an exact run of the haplotype spanning the seam (the diagonal and H cross it)
    "ins"         a 2-6 base insertion in the read at the seam (a vertical gap, F, crosses a row seam; at a column
                  seam the gap sits right next to it)
    "del_allele"  (folded kernel) a deletion of the whole allele region: E crosses the forward boundary and the
                  junction

with random bases around the planted part and enough matched bases on both sides that the crossing path wins.  Each
case keeps its WITNESS: for the ablations of tests/sw_ref.py ("gap" and "cut" at the seam, or a maximum restricted
to one side for the "*_max" seams), the haplotype halves (ref, alt) whose ablated score differs from the true score.
A kernel that loses that carry gets that half wrong.  Cases without a witness are dropped and planted again.

build(name) returns the loci of a family: windows, reads, and one Case per read; reads of a locus are consecutive
pairs, so the cases land on every pair slot of a tile, and read lengths are ragged inside tiles.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

import sw_ref

ACGT = np.frombuffer(b"ACGT", np.uint8)
KINDS = ("gap", "cut")
HALVES = ("ref", "alt", "both")


@dataclass(frozen=True)
class Seam:
    name: str
    axis: str                      # "col", "row" or "max"
    pos: object                    # col: n -> column; row: read row (int); max: n -> (lo, hi) columns kept
    styles: tuple
    cols: object = None            # row seams: n -> (lo, hi), the columns whose carry crosses this row
    kinds: tuple = KINDS           # witness kinds this seam must show (each at least once)


@dataclass
class Case:
    seam: str
    style: str
    witness: dict                  # kind -> "ref" / "alt" / "both"  (only kinds that hold)
    read: bytes = b""


@dataclass
class Locus:
    ref: bytes
    alt: bytes
    reads: list = field(default_factory=list)
    cases: list = field(default_factory=list)


@dataclass(frozen=True)
class Family:
    name: str
    kernel: str                    # kernel named in failure messages
    engine: dict                   # Engine flags that route the family to the kernel
    cls: int                       # tile class of vtx_last_tile_counts
    ppw: int                       # pairs per warp tile
    window: object                 # rng -> (ref, alt)
    seams: tuple
    m_lo: int
    m_hi: int
    n_loci: int = 24               # at least this many loci
    min_dup: int = 1               # every (seam, kind) at least this often


def _rand(rng, n):
    return ACGT[rng.integers(0, 4, n)].tobytes()


def _edit(rng, seq: bytes, rate: float, indel: bool = True) -> bytes:
    """substitutions at `rate` (always a different base) and, sometimes, one short indel"""
    s = bytearray(seq)
    for j in np.nonzero(rng.random(len(s)) < rate)[0]:
        s[j] = int(ACGT[(int(np.nonzero(ACGT == s[j])[0][0]) + int(rng.integers(1, 4))) % 4]) if s[j] in b"ACGT" else s[j]
    if indel and len(s) > 20 and rng.random() < 0.3:
        j = int(rng.integers(5, len(s) - 5)); k = int(rng.integers(1, 6))
        if rng.random() < 0.5: del s[j:j + k]
        else: s[j:j] = _rand(rng, k)
    return bytes(s)


def _alt_of(rng, ref: bytes) -> bytes:
    """an alt window for the single-phase families: one SNV (most of the window common) or a dense rewrite"""
    u = rng.random()
    if u < 0.4:
        a = bytearray(ref); j = int(rng.integers(0, len(a))); a[j] = int(ACGT[(int(np.nonzero(ACGT == a[j])[0][0]) + 1) % 4]); return bytes(a)
    return _edit(rng, ref, 0.06 if u < 0.7 else 0.25, indel=False)


def _plain_window(n_lo, n_hi):
    def w(rng):
        ref = _rand(rng, int(rng.integers(n_lo, n_hi + 1)))
        return ref, _alt_of(rng, ref)
    return w


def _split_window(n_lo, n_hi):
    def w(rng):
        n = int(rng.integers(n_lo, n_hi + 1))
        ref = _rand(rng, n)
        u = rng.random()
        if u < 0.4:                                   # SNV / short indel right of the common prefix
            a = bytearray(ref); j = int(rng.integers(96, n)); a[j] = int(ACGT[(int(np.nonzero(ACGT == a[j])[0][0]) + 1) % 4])
            alt = bytes(a)
        else:
            alt = ref[:96] + _edit(rng, ref[96:], 0.06 if u < 0.7 else 0.25)
        return ref, alt[:n_hi]
    return w


def _fold_window(rng):
    left, right = _rand(rng, 96), _rand(rng, 96)
    lr = int(rng.integers(1, 41)); u = rng.random()
    mr = _rand(rng, lr)
    if u < 0.4:                                       # SNV-like: same length, one base differs
        a = bytearray(mr); j = int(rng.integers(0, lr)); a[j] = int(ACGT[(int(np.nonzero(ACGT == a[j])[0][0]) + 1) % 4]); ma = bytes(a)
    elif u < 0.7:                                     # indel-like
        ma = _edit(rng, mr, 0.05)
        ma = ma[:40] if ma else _rand(rng, 1)
    else:                                             # unrelated allele
        ma = _rand(rng, int(rng.integers(1, 41)))
    return left + mr + right, left + ma + right


# ---------------------------------------------------------------------------------------------------------------
# families
# ---------------------------------------------------------------------------------------------------------------
COL = ("del", "run", "ins")


def _lanes(C, k_hi, base=0):
    return tuple(Seam(f"lane {base + k * C}", "col", (lambda n, c=base + k * C: c), COL) for k in range(1, k_hi + 1))


def _class_family(cls, C, n_lo, n_hi):
    return Family(f"class{cls}", f"vtx_k_sw_pairs<{cls}>", dict(no_split=True), cls, 4, _plain_window(n_lo, n_hi),
                  _lanes(C, 7), 30, 256)


def _rowblock_seams():
    out = []
    for base in (1024, 2048):
        for g in range(8):
            out.append(Seam(f"row block {base} lane {g}", "row", base - g, ("ins", "run"),
                            cols=(lambda n, g=g: (26 * g, min(n, 26 * (g + 1))))))
    return tuple(out)


def _split_family(scls, C2, n_lo, n_hi):
    seams = _lanes(12, 7) + (Seam("phase 96", "col", lambda n: 96, COL),) + _lanes(C2, 3, base=96) + \
        (Seam("prefix max", "max", lambda n: (96, n), ("run",), kinds=("max",)),)
    return Family(f"split{scls}", f"vtx_k_sw_split<{scls}>", dict(no_fold=True), 5 + scls, 8, _split_window(n_lo, n_hi), seams, 30, 256)


def _fold_seams():
    mid = lambda n: (96, n - 96)
    return (_lanes(12, 7)
            + tuple(Seam(f"suffix lane n-{12 * k}", "col", (lambda n, k=k: n - 12 * k), COL) for k in range(1, 8))
            + (Seam("forward boundary 96", "col", lambda n: 96, COL + ("del_allele",)),)
            + tuple(Seam(f"allele rows {19 * k}", "row", 19 * k, ("ins", "run"), cols=mid) for k in range(1, 8))
            + (Seam("junction n-96", "col", lambda n: n - 96, COL + ("del_allele",)),
               Seam("suffix max", "max", lambda n: (0, n - 96), ("run",), kinds=("max",))))


FAMILIES = {f.name: f for f in (
    _class_family(0, 26, 150, 208),
    _class_family(1, 29, 209, 232),
    _class_family(2, 32, 233, 256),
    _class_family(3, 40, 257, 320),
    Family("multi", "vtx_k_sw_pairs<3> multi-pass", dict(), 3, 4, _plain_window(700, 960),
           (Seam("pass 320", "col", lambda n: 320, COL), Seam("pass 640", "col", lambda n: 640, COL))
           + _lanes(40, 7, base=320) + _lanes(40, 1, base=640), 30, 256),
    Family("rowblock", "vtx_k_sw_pairs<0> row blocks", dict(), 0, 4, _plain_window(190, 208), _rowblock_seams(), 1030, 2300,
           n_loci=8),
    _split_family(0, 27, 150, 204),
    _split_family(1, 34, 205, 232),
    Family("fold", "vtx_k_sw_fold", dict(), 7, 4, _fold_window, _fold_seams(), 30, 152),
)}


# ---------------------------------------------------------------------------------------------------------------
# planting
# ---------------------------------------------------------------------------------------------------------------
def _plant(rng, fam: Family, seam: Seam, style: str, T: bytes, m: int):
    """a read of length about m whose best alignment against T crosses `seam` in the way `style` says (None: no room)"""
    n = len(T)
    k = int(rng.integers(2, 7))
    L1, L2 = int(rng.integers(14, 45)), int(rng.integers(14, 45))
    if seam.axis == "max":
        lo, hi = seam.pos(n)
        if hi - lo < 30:
            return None
        ln = int(rng.integers(25, min(hi - lo, 60) + 1)); a = int(rng.integers(lo, hi - ln + 1))
        core, A = _edit(rng, T[a:a + ln], 0.03, indel=False), int(rng.integers(0, max(1, m - ln)))
    elif seam.axis == "col":
        c = seam.pos(n)
        if style == "del_allele":
            if fam.name != "fold":
                return None
            lo, hi = 96, n - 96
            L1, L2 = min(L1 + 20, 96), min(L2 + 20, 96)
            core = T[lo - L1:lo] + T[hi:hi + L2]
        elif style == "del":
            d1 = int(rng.integers(1, k))
            a, b = c - d1, c - d1 + k
            L1, L2 = min(L1, a), min(L2, n - b)
            if L1 < 10 or L2 < 10:
                return None
            core = T[a - L1:a] + T[b:b + L2]
        elif style == "run":
            L1, L2 = min(L1, c), min(L2, n - c)
            if L1 < 4 or L2 < 4:
                return None
            core = T[c - L1:c + L2]
        else:                                         # ins
            L1, L2 = min(L1, c), min(L2, n - c)
            if L1 < 10 or L2 < 10:
                return None
            core = T[c - L1:c] + _rand(rng, k) + T[c:c + L2]
        A = int(rng.integers(0, max(1, min(30, m - len(core)))))
    else:                                             # row seam r, crossing inside the columns seam.cols(n)
        r = seam.pos
        lo, hi = seam.cols(n)
        if hi - lo < 2:
            return None
        p = int(rng.integers(lo + 1, hi))             # crossing between columns p - 1 and p
        if style == "ins":                            # insertion after column p - 1, covering read rows r - 1 and r
            q = r - int(rng.integers(1, k))               # read row of the first inserted base
            L1 = min(L1, p, q)
            L2 = min(L2, n - p)
            if L1 < 8 or L2 < 8:
                return None
            core = T[p - L1:p] + _rand(rng, k) + T[p:p + L2]
            A = q - L1
        else:                                         # run: read row r meets column p
            L1 = min(L1, p, r); L2 = min(L2, n - p)
            if L1 < 6 or L2 < 6:
                return None
            core = T[p - L1:p + L2]
            A = r - L1
        if A + len(core) > m:
            return None
    Z = m - A - len(core)
    if Z < 0:
        core = core[:m - A] if m - A >= 20 else None
        if core is None:
            return None
        Z = 0
    return _rand(rng, A) + core + _rand(rng, Z)


def _ablations(seam: Seam, n: int):
    """witness kind -> sw_ref.score keyword arguments for a haplotype of n columns"""
    if seam.axis == "max":
        return {"max": dict(max_cols=seam.pos(n))}
    if seam.axis == "col":
        c = seam.pos(n)
        return {"gap": dict(col_gap=[c]), "cut": dict(col_cut=[c])}
    lo, hi = seam.cols(n)
    return {"gap": dict(row_gap=[(seam.pos, lo, hi)]), "cut": dict(row_cut=[(seam.pos, lo, hi)])}


def witness(seam: Seam, read: bytes, ref: bytes, alt: bytes, true=None) -> dict:
    """kind -> "ref" / "alt" / "both" for the ablations of `seam` whose score differs from the true one"""
    if true is None:
        true = sw_ref.score([read, read], [ref, alt])
    out = {}
    abl_r, abl_a = _ablations(seam, len(ref)), _ablations(seam, len(alt))
    for kind in abl_r:
        if abl_r[kind] == abl_a[kind]:
            got = sw_ref.score([read, read], [ref, alt], **abl_r[kind])
        else:
            got = [sw_ref.score_pair(read, ref, **abl_r[kind]), sw_ref.score_pair(read, alt, **abl_a[kind])]
        hit = [h for h, t, g in zip(("ref", "alt"), true, got) if t != g]
        if hit:
            out[kind] = "both" if len(hit) == 2 else hit[0]
    return out


def _seam_applies(fam: Family, seam: Seam, ref: bytes, alt: bytes) -> bool:
    n = min(len(ref), len(alt))
    if seam.axis == "col":
        return 0 < seam.pos(len(ref)) < len(ref) and 0 < seam.pos(len(alt)) < len(alt)
    if seam.axis == "row":
        return seam.cols(n)[1] - seam.cols(n)[0] >= 2
    return True


@functools.lru_cache(maxsize=None)
def build(name: str, seed: int = 0) -> tuple:
    """The loci of one family (a tuple of Locus).  Deterministic for a given seed."""
    fam = FAMILIES[name]
    rng = np.random.default_rng(seed * 1000 + sum(map(ord, name)))
    need = {(s.name, kind): fam.min_dup for s in fam.seams for kind in s.kinds}
    need_halves = {(kind, h): 1 for kind in KINDS for h in HALVES}
    loci = []
    for _it in range(4000):
        if len(loci) >= fam.n_loci and not any(need.values()) and not any(need_halves.values()):
            break
        ref, alt = fam.window(rng)
        loc = Locus(ref, alt)
        n_reads = int(rng.integers(1, 2 * fam.ppw + 2))
        # a quarter of the folded kernel's loci: every read 149-152 bases (the last boundary rows of each unit)
        long_fold = fam.name == "fold" and rng.random() < 0.25
        for _slot in range(n_reads):
            open_seams = [s for s in fam.seams if any(need.get((s.name, k), 0) for k in s.kinds)] or list(fam.seams)
            open_seams = [s for s in open_seams if _seam_applies(fam, s, ref, alt)] or \
                [s for s in fam.seams if _seam_applies(fam, s, ref, alt)]
            for _try in range(8):
                seam = open_seams[int(rng.integers(0, len(open_seams)))]
                style = seam.styles[int(rng.integers(0, len(seam.styles)))]
                want = [h for (kind, h), v in need_halves.items() if v]
                src = alt if (want and want[int(rng.integers(0, len(want)))] == "alt") or rng.random() < 0.3 else ref
                m = int(rng.integers(149, 153)) if long_fold else int(rng.integers(fam.m_lo, fam.m_hi + 1))
                if seam.axis == "row" and fam.m_lo > 1024:    # long reads: just past the row block the seam is in
                    m = seam.pos + int(rng.integers(40, 250))
                read = _plant(rng, fam, seam, style, src, m)
                if read is None:
                    continue
                w = witness(seam, read, ref, alt)
                if w:
                    break
            else:
                continue
            loc.reads.append(read)
            loc.cases.append(Case(seam.name, style, w, read))
            for kind, h in w.items():
                if need.get((seam.name, kind), 0):
                    need[(seam.name, kind)] -= 1
                if need_halves.get((kind, h), 0):
                    need_halves[(kind, h)] -= 1
        if loc.reads:
            loci.append(loc)
    return tuple(loci)


def required(name: str):
    """(seam, kind) pairs the family must witness, and the (kind, halves) pairs"""
    fam = FAMILIES[name]
    return ({(s.name, k) for s in fam.seams for k in s.kinds}, {(k, h) for k in KINDS for h in HALVES})


def pairs(loci):
    """-> (ref windows, alt windows, reads, pair_read, pair_locus, cases) with reads numbered locus by locus"""
    reads, pr, pl, cases = [], [], [], []
    for l, loc in enumerate(loci):
        for rd, c in zip(loc.reads, loc.cases):
            pr.append(len(reads)); pl.append(l); reads.append(rd); cases.append(c)
    return ([l.ref for l in loci], [l.alt for l in loci], reads, np.array(pr, np.uint32), np.array(pl, np.uint32), cases)


def staged_batch(vb, refs, alts, reads):
    """A vartrix_b200.StagedBatch (module passed in: this file imports nothing of the GPU side) holding the windows
    refs[l] / alts[l] of locus l and the reads (bytes) -> the batch; pairs are given separately to score_pairs."""
    haps, ref_off, alt_off = bytearray(), [], []
    for r, a in zip(refs, alts):
        for h, offs in ((r, ref_off), (a, alt_off)):
            haps.extend(b"\0" * (-len(haps) % 16)); offs.append(len(haps)); haps.extend(h)
    haps.extend(b"\0" * (-len(haps) % 16))          # batches may be concatenated: keep every offset a multiple of 16
    nibs, read_off = bytearray(), []
    for rd in reads:
        codes = sw_ref.encode(rd)
        if len(codes) & 1:
            codes = np.concatenate([codes, np.zeros(1, np.uint8)])
        nibs.extend(b"\0" * (-len(nibs) % 16)); read_off.append(len(nibs))
        nibs.extend(((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes())
    nibs.extend(b"\0" * (-len(nibs) % 16))
    n_loci, n_reads = len(refs), len(reads)
    return vb.StagedBatch(
        locus_row=np.arange(n_loci), hap_bytes=np.frombuffer(bytes(haps), np.uint8), ref_off=ref_off,
        ref_len=[len(r) for r in refs], alt_off=alt_off, alt_len=[len(a) for a in alts],
        cand_start=np.zeros(n_loci + 1, np.uint64), read_nib=np.frombuffer(bytes(nibs), np.uint8), read_off=read_off,
        read_len=[len(r) for r in reads], cb_bytes=np.zeros(0, np.uint8), read_cb_off=np.full(n_reads, 0xFFFFFFFF),
        read_cb_len=np.zeros(n_reads), read_umi_key=np.full(n_reads, 0xFFFFFFFFFFFFFFFF, np.uint64),
        cand_read=np.zeros(0, np.uint32), n_rows=n_loci)


BARCODES = [b"ACGTACGTAC-1", b"CCGTACGTAC-1", b"GCGTACGTAC-1", b"TCGTACGTAC-1", b"AAGTACGTAC-1"]


def whole_path_batch(vb, loci, n_reads_n: int = 50):
    """A shard for the whole path (cell tags, candidates) from planted loci: every locus also gets one read of
    n_reads_n N bases (scores 0 / 0), and reads cycle through the five BARCODES and one unlisted tag."""
    refs, alts, reads, cand_start = [], [], [], [0]
    for loc in loci:
        refs.append(loc.ref); alts.append(loc.alt)
        reads.extend(loc.reads); reads.append(b"N" * n_reads_n)
        cand_start.append(len(reads))
    sb = staged_batch(vb, refs, alts, reads)
    tags = BARCODES + [b"TTTTTTTTTT-1"]
    pick = np.arange(len(reads)) % len(tags)
    offs = np.concatenate([[0], np.cumsum([len(t) for t in tags])])
    sb.cb_bytes = np.frombuffer(b"".join(tags), np.uint8).copy()
    sb.read_cb_off = offs[pick].astype(np.uint32)
    sb.read_cb_len = np.array([len(tags[i]) for i in pick], np.uint16)
    sb.cand_start = np.array(cand_start, np.uint64)
    sb.cand_read = np.arange(len(reads), dtype=np.uint32)
    return sb
