"""Shards that cross the seams of the matrix-assembly kernels (vtx_k_slots, vtx_k_slots_big, vtx_k_umi_collapse,
vtx_k_finalize, vtx_k_emit in vartrix_b200/csrc/vtx_pipeline.cuh).

Reads come from a few templates with known calls, so a shard of millions of pairs needs only eight scored reads.
Every candidate is its own read (it carries its own CB and UB) whose bases are one of the templates, shared by
offset.  Two window families:
  * "short": a 61-column SNV window and 40-base reads (single-phase class 0);
  * "prod": a --padding 100 SNV window (201 columns) and 150-base reads (the folded kernel).
Templates per family: REF and ALT (exact across the variant), TIE (30 bases inside the left flank: 30 against both
haplotypes, UNKNOWN) and NONE (20 bases inside the right flank: both scores below 25, None).

A shard is flat per-pair arrays; `fields()` stages it as the vtx_batch layout and `expected_scores()` maps the eight
template scores onto its candidates, which is all matrix_ref needs."""
import functools
from dataclasses import dataclass, field

import numpy as np

import sw_ref

TEMPLATES = ("REF", "ALT", "TIE", "NONE")
T_REF, T_ALT, T_TIE, T_NONE = range(4)
FAMILIES = ("short", "prod")
SHORT, PROD = 0, 1
TAG_LEN = 18
UNLISTED, NO_TAG = -1, -2                         # values of Shard.cb besides a column id
NO_UMI = 0xFFFFFFFFFFFFFFFF
NO_CB_OFF = 0xFFFFFFFF
UMI_KEY_MAX = (1 << 62) - 1                       # VTX_UMI_KEY_MAX
# more than 2^17 columns (ids above 16 bits, D = 100 000 fits), and enough that every deep locus of the ladder, up to
# d = 100 000 (cap 200 000), finds two columns whose bucket is cap - 1
N_BARCODES = 450_000
SLOT_CHUNK, SMALL_MAX = 1024, 2048                # kSlotChunk, kSlotSmallMax
MANY_LOCI = 65_535 * 8 + 1_000                    # more loci than vtx_k_slots launches CTAs

_BASE = 0x0123_4567
# keys that differ only in bits 32-61, only in bits 0-31, keys with bit 61 set (interned UB strings) and the largest
# valid key
UMI_POOL = np.array([_BASE, _BASE | 1 << 32, _BASE | 2 << 32, _BASE | 0x3FFF_FFFF << 32,
                     _BASE + 1, _BASE ^ 0x8000_0000, 1 << 61 | 5, 1 << 61 | 1 << 32 | 5,
                     UMI_KEY_MAX, UMI_KEY_MAX ^ 1 << 32, UMI_KEY_MAX ^ 1], np.uint64)


def mix32(x):
    """vtx_pipeline.cuh mix32, on uint32 arrays"""
    x = np.asarray(x, np.uint32).copy()
    x ^= x >> np.uint32(16); x *= np.uint32(0x7feb352d)
    x ^= x >> np.uint32(15); x *= np.uint32(0x846ca68b)
    x ^= x >> np.uint32(16)
    return x


def cell_bucket(col, cap):
    return mix32(col) % np.uint32(cap)


def umi_bucket(col, umi, cap):
    umi = np.asarray(umi, np.uint64)
    lo, hi = (umi & np.uint64(0xFFFF_FFFF)).astype(np.uint32), (umi >> np.uint64(32)).astype(np.uint32)
    return mix32(np.asarray(col, np.uint32) ^ mix32(lo ^ mix32(hi))) % np.uint32(cap)


def _windows(seed=11):
    """(ref, alt, [REF, ALT, TIE, NONE reads]) per family"""
    rng = np.random.default_rng(seed)
    out = []
    for n, v, m in ((61, 30, 40), (201, 100, 150)):
        ref = bytes(rng.choice(list(b"ACGT"), n).astype(np.uint8))
        alt = bytearray(ref); alt[v] = b"ACGT"[(b"ACGT".index(ref[v]) + 1) % 4]; alt = bytes(alt)
        s = v - m // 2
        out.append((ref, alt, [ref[s:s + m], alt[s:s + m], ref[:30], ref[n - 20:]]))
    return out


WINDOWS = _windows()


def barcode_tags(n):
    """n distinct 16-base tags + '-1' as an [n, 18] uint8 array"""
    shifts = np.arange(15, -1, -1, dtype=np.uint64) * np.uint64(2)
    v = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFF_FFFF)
    tags = np.empty((n, TAG_LEN), np.uint8)
    tags[:, :16] = np.frombuffer(b"ACGT", np.uint8)[((v[:, None] >> shifts[None, :]) & np.uint64(3)).astype(np.int64)]
    tags[:, 16:] = np.frombuffer(b"-1", np.uint8)
    return tags


@dataclass
class Shard:
    name: str
    fam: np.ndarray                 # [n_loci] window family
    cand_start: np.ndarray          # [n_loci + 1]
    tmpl: np.ndarray                # [n_pairs] template
    cb: np.ndarray                  # [n_pairs] column id, UNLISTED or NO_TAG
    umi: np.ndarray                 # [n_pairs] UMI key or NO_UMI
    n_barcodes: int = N_BARCODES
    notes: dict = field(default_factory=dict)

    @property
    def n_loci(self): return int(self.fam.size)
    @property
    def n_pairs(self): return int(self.tmpl.size)
    def depth(self): return np.diff(self.cand_start)


class _Builder:
    def __init__(self, name):
        self.name, self.fam, self.depth, self.tmpl, self.cb, self.umi = name, [], [], [], [], []

    def add(self, fam, tmpl, cb, umi):
        tmpl = np.asarray(tmpl, np.int8)
        self.fam.append(fam); self.depth.append(tmpl.size); self.tmpl.append(tmpl)
        self.cb.append(np.broadcast_to(np.asarray(cb, np.int64), tmpl.shape))
        self.umi.append(np.broadcast_to(np.asarray(umi, np.uint64), tmpl.shape))

    def shard(self, **notes):
        cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
        return Shard(self.name, np.array(self.fam, np.int8), np.concatenate([[0], np.cumsum(self.depth)]).astype(np.int64),
                     cat(self.tmpl, np.int8), cat(self.cb, np.int64), cat(self.umi, np.uint64), notes=notes)


def _calls(rng, n, p=(0.35, 0.35, 0.2, 0.1)):
    return rng.choice(4, n, p=p).astype(np.int8)


def _cells(rng, d, D):
    """cell rank (0 = first seen) of each of d pairs, D distinct; for 1025 <= d <= 2048 and 2 < D < d - 1 the pair at
    p = 1024 has exactly one twin, at p = 1023"""
    if D == d:
        seq = np.arange(d)
    else:
        seq = np.concatenate([np.arange(D), rng.integers(0, D, d - D)])
        rng.shuffle(seq)
        if SLOT_CHUNK < d <= SMALL_MAX and 2 < D < d - 1:
            v, w = seq[SLOT_CHUNK], seq[SLOT_CHUNK - 1]
            if v == w:                               # choose another value for the pair: one seen at least twice more
                cnt = np.bincount(seq, minlength=D)
                v = int(np.nonzero(cnt >= 3)[0][0]) if (cnt >= 3).any() else v
            others = np.nonzero(seq == v)[0]
            others = others[(others != SLOT_CHUNK) & (others != SLOT_CHUNK - 1)]
            seq[others] = w if w != v else seq[0]
            seq[SLOT_CHUNK - 1] = seq[SLOT_CHUNK] = v
            missing = np.setdiff1d(np.arange(D), seq)
            cnt = np.bincount(seq, minlength=D)
            for m in missing:                        # put back any cell the planting removed, over a repeated one
                q = next(i for i in range(d) if i not in (SLOT_CHUNK - 1, SLOT_CHUNK) and cnt[seq[i]] > 1 and seq[i] != v)
                cnt[seq[q]] -= 1; seq[q] = m; cnt[m] += 1
    # relabel so that ranks follow first appearance
    _, first = np.unique(seq, return_index=True)
    rank = np.empty(D, np.int64); rank[np.argsort(first)] = np.arange(D)
    return rank[seq]


@functools.lru_cache(maxsize=None)
def _last_bucket(cap, n_bc):
    """the columns whose bucket in a table of cap entries is cap - 1"""
    return np.nonzero(cell_bucket(np.arange(n_bc), cap) == cap - 1)[0]


def _columns(rng, D, d, n_bc):
    """D distinct columns, descending in first-seen order.  A deep locus gets up to four columns whose bucket is
    cap - 1 (cap = 2 d): two distinct keys there make linear probing wrap to bucket 0 whatever the insertion order"""
    cols = _last_bucket(2 * d, n_bc)[:min(D, 4)] if d > SMALL_MAX else np.zeros(0, np.int64)
    pick = rng.choice(n_bc, D + cols.size, replace=False)
    pick = pick[~np.isin(pick, cols)][:D - cols.size]
    return np.sort(np.concatenate([cols, pick]))[::-1]


def _deep_locus(rng, d, D, fam, n_bc, umi_pool):
    rank = _cells(rng, d, D)
    col = _columns(rng, D, d, n_bc)[rank]
    umi = umi_pool[rng.integers(0, umi_pool.size, d)]
    if d > SMALL_MAX:                                # (cell, UMI) keys planted in the last bucket of utab
        cap = 2 * d
        for p in rng.choice(d, min(d, 4), replace=False):
            hi = umi[p] >> np.uint64(32)
            lo = rng.integers(0, 1 << 32, 20 * cap, dtype=np.uint64)
            keys = (hi << np.uint64(32)) | lo
            hit = np.nonzero(umi_bucket(np.full(keys.size, col[p]), keys, cap) == cap - 1)[0]
            if hit.size:
                umi[p] = keys[hit[0]]
    return fam, _calls(rng, d), col, umi


LADDER = (1, 127, 128, 129, 1023, 1024, 1025, 1152, 1153, 2047, 2048, 2049, 2050, 4096, 4097, 100_000)


def ladder_pairs(d):
    """(d, D) of the depth ladder: D in {1, 2, d/2, d} and the bitonic sizes 1024, 1025, 2048, 2049, 70 000"""
    ds = {1, 2, d // 2, d} | {x for x in (1024, 1025, 2048, 2049, 70_000) if x <= d}
    return sorted(x for x in ds if 1 <= x <= d)


def ladder(depths=LADDER, seed=1):
    rng = np.random.default_rng(seed)
    b = _Builder("ladder")
    i = 0
    for d in depths:
        for D in ladder_pairs(d):
            b.add(*_deep_locus(rng, d, D, i % 2, N_BARCODES, UMI_POOL))
            i += 1
    return b.shard()


def umi_groups():
    """(r, a, u, n_none) of every UMI group of the grid"""
    g = [(r, a, u, nn) for r in range(9) for a in range(9 - r) for u in range(9 - r - a) for nn in (0, 2)]
    g = [x for x in g if sum(x[:3]) or x[3]]
    g += [(0, 0, 0, k) for k in (1, 2, 3)]
    for k in range(1, 51):
        for top in (3 * k, 3 * k - 1):
            rest = 4 * k - top
            g += [(rest // 2, top, rest - rest // 2, 0), (top, rest // 2, rest - rest // 2, 0)]
    return g


def _grid_loci(rng, groups, n_cells, fam_of, split):
    """the groups spread over n_cells cells, in loci of at most `split` pairs (one locus when split is None)"""
    loci, cur = [], []
    size = 0
    for gi, (r, a, u, nn) in enumerate(groups):
        t = [T_REF] * r + [T_ALT] * a + [T_TIE] * u + [T_NONE] * nn
        if split and size + len(t) > split:
            loci.append(cur); cur, size = [], 0
        cur.append((gi, t)); size += len(t)
    loci.append(cur)
    out = []
    for li, loc in enumerate(loci):
        tm = np.concatenate([np.array(t, np.int8) for _gi, t in loc])
        gid = np.concatenate([np.full(len(t), gi) for gi, t in loc])
        col = 100_003 + 7 * (gid % n_cells)
        umi = UMI_POOL[gid % UMI_POOL.size] ^ (gid.astype(np.uint64) << np.uint64(8))
        perm = rng.permutation(tm.size)
        out.append((fam_of(li), tm[perm], col[perm], umi[perm]))
    return out


def umi_grid(seed=2):
    """the 0.75 rule at every small (r, a, u), with and without None reads, and at (3k, 4k) / (3k - 1, 4k) up to
    k = 50: once in shallow loci, once in one deep locus"""
    rng = np.random.default_rng(seed)
    b = _Builder("umi_grid")
    g = umi_groups()
    for loc in _grid_loci(rng, g, 23, lambda li: li % 2, 2000):
        b.add(*loc)
    for loc in _grid_loci(rng, g, 29, lambda li: SHORT, None):
        b.add(*loc)
    return b.shard(n_groups=len(g))


def modes(seed=3):
    """cells whose reads are all None, cells with only UNKNOWN calls, consensus 1, 2 and 3, next to unlisted and
    missing tags and reads without a UMI"""
    rng = np.random.default_rng(seed)
    b = _Builder("modes")
    kinds = {"none": [T_NONE], "unknown": [T_TIE], "ref": [T_REF, T_TIE], "alt": [T_ALT, T_NONE],
             "both": [T_REF, T_ALT, T_TIE, T_NONE]}
    for li in range(40):
        tm, cb, um = [], [], []
        for ci, (k, pool) in enumerate(kinds.items()):
            n = int(rng.integers(1, 6))
            t = np.array(pool, np.int8)[rng.integers(0, len(pool), n)]
            if k in ("ref", "alt"):
                t[0] = pool[0]
            if k == "both":
                t[:2] = [T_REF, T_ALT] if n > 1 else t[:2]
            tm.append(t); cb.append(np.full(n, 5 * li + ci)); um.append(UMI_POOL[rng.integers(0, 4, n)])
        n = 6                                        # unlisted, missing tags, missing UMIs
        tm.append(_calls(rng, n)); cb.append(np.array([UNLISTED, NO_TAG, 7, 7, 9, UNLISTED]))
        um.append(np.array([5, 5, NO_UMI, 5, NO_UMI, NO_UMI], np.uint64))
        tm, cb, um = np.concatenate(tm), np.concatenate(cb), np.concatenate(um)
        perm = rng.permutation(tm.size)
        b.add(li % 2, tm[perm], cb[perm], um[perm])
    return b.shard()


def crowd(n_sm, seed=4):
    """2 n_SM + 1 loci of depth 2049-2100 (every vtx_k_slots_big CTA takes more than one), in runs of adjacent deep loci
    between shallow ones, deep loci first and last"""
    rng = np.random.default_rng(seed)
    b = _Builder("crowd")
    n_deep = 2 * n_sm + 1
    done = 0
    while done < n_deep:
        run = min(int(rng.integers(1, 4)), n_deep - done)
        for _ in range(run):
            d = int(rng.integers(SMALL_MAX + 1, 2101))
            b.add(*_deep_locus(rng, d, int(rng.integers(d // 4, d + 1)), int(rng.integers(0, 2)), N_BARCODES, UMI_POOL))
        done += run
        if done < n_deep:
            for _ in range(int(rng.integers(1, 3))):
                d = int(rng.integers(1, 60))
                b.add(*_deep_locus(rng, d, int(rng.integers(1, d + 1)), int(rng.integers(0, 2)), N_BARCODES, UMI_POOL))
    return b.shard(n_deep=n_deep)


def many_loci(n_loci=MANY_LOCI, seed=5):
    """more loci of 1-3 pairs than vtx_k_slots has CTAs"""
    rng = np.random.default_rng(seed)
    depth = rng.integers(1, 4, n_loci)
    n = int(depth.sum())
    fam = (rng.random(n_loci) < 0.1).astype(np.int8)
    cb = rng.integers(0, N_BARCODES, n)
    dup = rng.random(n) < 0.3                       # a third of the pairs repeat the cell of the pair before
    cb[1:][dup[1:]] = cb[:-1][dup[1:]]
    return Shard("many_loci", fam, np.concatenate([[0], np.cumsum(depth)]), _calls(rng, n), cb,
                 UMI_POOL[rng.integers(0, 3, n)])


def counters():
    """one cell at one locus with 2^21 + 1 ALT, 2^21 + 1 UNKNOWN and 3 REF calls, all under one UMI: the alt and
    unknown counts need 22 bits"""
    rng = np.random.default_rng(6)
    k = (1 << 21) + 1
    tm = np.concatenate([np.full(k, T_ALT), np.full(k, T_TIE), np.full(3, T_REF)]).astype(np.int8)
    rng.shuffle(tm)
    b = _Builder("counters")
    b.add(SHORT, tm, 77_777, UMI_POOL[3])
    return b.shard()


# ---- staging -----------------------------------------------------------------------------------------------------
def _pack(read: bytes):
    codes = sw_ref.encode(read)
    if codes.size & 1:
        codes = np.concatenate([codes, np.zeros(1, np.uint8)])
    return ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8)


def _layout():
    """hap_bytes, ref/alt offsets per family, read_nib, offsets/lengths per (family, template)"""
    haps, hoff = bytearray(), []
    nibs, toff, tlen = bytearray(), np.zeros((2, 4), np.int64), np.zeros((2, 4), np.int64)
    for f, (ref, alt, reads) in enumerate(WINDOWS):
        o = []
        for h in (ref, alt):
            haps.extend(b"\0" * (-len(haps) % 16)); o.append(len(haps)); haps.extend(h)
        hoff.append(o)
        for t, rd in enumerate(reads):
            nibs.extend(b"\0" * (-len(nibs) % 16)); toff[f, t] = len(nibs); tlen[f, t] = len(rd)
            nibs.extend(_pack(rd).tobytes())
    haps.extend(b"\0" * (-len(haps) % 16)); nibs.extend(b"\0" * (-len(nibs) % 16))
    return np.frombuffer(bytes(haps), np.uint8), np.array(hoff), np.frombuffer(bytes(nibs), np.uint8), toff, tlen


def barcodes(n=N_BARCODES):
    """the barcode list every shard's columns index"""
    return [bytes(t) for t in barcode_tags(n)]


def fields(shard, loci=None):
    """the shard (or its loci `loci`, keeping their rows) as vtx_batch fields; every candidate is its own read"""
    if loci is None:
        loci = np.arange(shard.n_loci)
    loci = np.asarray(loci, np.int64)
    d = shard.depth()[loci]
    pidx = (np.repeat(shard.cand_start[loci], d) + np.arange(int(d.sum())) - np.repeat(np.cumsum(d) - d, d)).astype(np.int64)
    hap, hoff, nib, toff, tlen = _layout()
    fam = shard.fam[loci].astype(np.int64)
    pfam = np.repeat(fam, d)
    tm = shard.tmpl[pidx].astype(np.int64)
    cb = shard.cb[pidx]
    n = pidx.size
    # the barcode list's tags, then one unlisted tag
    cb_bytes = np.concatenate([barcode_tags(shard.n_barcodes).reshape(-1), np.frombuffer(b"NNNNAAAACCCCGGGG-1", np.uint8)])
    cb_off = np.where(cb >= 0, cb * TAG_LEN, np.where(cb == UNLISTED, shard.n_barcodes * TAG_LEN, NO_CB_OFF))
    return dict(
        locus_row=loci.astype(np.uint32), hap_bytes=hap, ref_off=hoff[fam, 0].astype(np.uint32),
        ref_len=np.array([len(w[0]) for w in WINDOWS], np.uint32)[fam], alt_off=hoff[fam, 1].astype(np.uint32),
        alt_len=np.array([len(w[1]) for w in WINDOWS], np.uint32)[fam],
        cand_start=np.concatenate([[0], np.cumsum(d)]).astype(np.uint64), read_nib=nib,
        read_off=toff[pfam, tm].astype(np.uint64), read_len=tlen[pfam, tm].astype(np.uint32), cb_bytes=cb_bytes,
        read_cb_off=cb_off.astype(np.uint32), read_cb_len=np.where(cb == NO_TAG, 0, TAG_LEN).astype(np.uint16),
        read_umi_key=shard.umi[pidx].copy(), cand_read=np.arange(n, dtype=np.uint32), n_rows=shard.n_loci)



def template_batch():
    """the eight template reads as a score_pairs batch: (fields, pair_read, pair_locus); pair f * 4 + t"""
    hap, hoff, nib, toff, tlen = _layout()
    z = np.zeros(8, np.int64)
    f = dict(locus_row=np.arange(2, dtype=np.uint32), hap_bytes=hap, ref_off=hoff[:, 0].astype(np.uint32),
             ref_len=np.array([len(w[0]) for w in WINDOWS], np.uint32), alt_off=hoff[:, 1].astype(np.uint32),
             alt_len=np.array([len(w[1]) for w in WINDOWS], np.uint32), cand_start=np.zeros(3, np.uint64),
             read_nib=nib, read_off=toff.reshape(-1).astype(np.uint64), read_len=tlen.reshape(-1).astype(np.uint32),
             cb_bytes=np.zeros(0, np.uint8), read_cb_off=np.full(8, NO_CB_OFF, np.uint32), read_cb_len=z.astype(np.uint16),
             read_umi_key=np.full(8, NO_UMI, np.uint64), cand_read=np.zeros(0, np.uint32), n_rows=2)
    return f, np.arange(8, dtype=np.uint32), np.repeat(np.arange(2), 4).astype(np.uint32)


def expected_scores(shard, tmpl_ref, tmpl_alt, loci=None):
    """(ref, alt) score of every candidate of fields(shard, loci) from the eight template scores"""
    if loci is None:
        loci = np.arange(shard.n_loci)
    loci = np.asarray(loci, np.int64)
    d = shard.depth()[loci]
    pidx = (np.repeat(shard.cand_start[loci], d) + np.arange(int(d.sum())) - np.repeat(np.cumsum(d) - d, d)).astype(np.int64)
    k = np.repeat(shard.fam[loci].astype(np.int64), d) * 4 + shard.tmpl[pidx]
    return np.asarray(tmpl_ref)[k], np.asarray(tmpl_alt)[k]


# ---- what a shard reaches ------------------------------------------------------------------------------------------
def locus_facts(shard, l, umi=False):
    """depth, distinct cells D, bitonic size P, and the chunk / twin / wrap facts of locus l"""
    s, e = int(shard.cand_start[l]), int(shard.cand_start[l + 1])
    d = e - s
    cb = shard.cb[s:e]
    D = int(np.unique(cb).size)
    P = 1
    while P < D:
        P <<= 1
    f = dict(d=d, D=D, P=P)
    if SLOT_CHUNK < d <= SMALL_MAX:
        _, first = np.unique(cb, return_index=True)
        first_at = first[np.searchsorted(np.unique(cb), cb)]
        p = np.arange(d)
        rep = p != first_at
        f["first_and_repeat_in_chunk1"] = bool((rep & (first_at >= SLOT_CHUNK)).any())
        # first seen in chunk 0, and every repeat in chunk 1
        c0 = np.unique(cb[(first_at < SLOT_CHUNK)])
        only1 = [c for c in c0 if (np.nonzero(cb == c)[0][1:] >= SLOT_CHUNK).all() and (cb == c).sum() > 1]
        f["chunk0_repeats_only_in_chunk1"] = len(only1) > 0
        f["twin_1023_1024"] = bool(cb[SLOT_CHUNK] == cb[SLOT_CHUNK - 1] and (cb[:SLOT_CHUNK - 1] != cb[SLOT_CHUNK]).all())
    if d > SMALL_MAX:
        cap = 2 * d
        f["cell_wraps"] = int((cell_bucket(np.unique(cb[cb >= 0]), cap) == cap - 1).sum())
        if umi:
            f["umi_wraps"] = int((umi_bucket(cb, shard.umi[s:e], cap) == cap - 1).sum())
    return f
