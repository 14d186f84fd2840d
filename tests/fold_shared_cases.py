"""The folded kernel's shared extension (vartrix_b200/csrc/vtx_sw_fold.cuh), restated in NumPy, and loci that test it.

After the main pass (forward DP over hap[:96], reversed DP over hap[n - 96:]) the kernel continues both halves over x
more columns that ref and alt still share, once for both, and scores only the columns in between per haplotype:

    prefix [0, 96) | shared extension [96, 96 + x) | allele columns | shared extension [n - 96 - x, n - 96) | suffix

`shared_columns` restates how the table builder picks x.  `split_scores` restates the (ref, alt) scores of that split
with the shared parts computed once, from the ref window, and the allele columns continued per haplotype from them;
the tests pin it against the full matrix.  `window` builds VCF-like windows (flanks of `pad` bases around an SNV, an
insertion or a deletion, with or without a shared anchor base) and `reads` plants reads whose gaps cross the seams."""
from __future__ import annotations

import numpy as np

P, MAX_MID = 96, 40
MID_TAB_BYTES, EXT_COL_BYTES = MAX_MID * 32, 25 * 4      # a slot's allele area; one extension column (25 pair codes)
MATCH, MISMATCH, GAP_OPEN, GAP_EXTEND = 1, -5, -5, -1
GOE = GAP_OPEN + GAP_EXTEND
NEG = -(1 << 40)
ACGT = np.frombuffer(b"ACGT", np.uint8)


def shared_columns(ref: bytes, alt: bytes) -> int:
    """x of a folded window pair: columns 96 + j and n - 97 - j common to ref and alt for every j < x, at least one
    allele column per haplotype left over, extension (100 B per column) and allele table (32 B) within 1280 B"""
    mid_ref, mid_alt = len(ref) - 2 * P, len(alt) - 2 * P
    lmax, lmin = max(mid_ref, mid_alt), min(mid_ref, mid_alt)
    assert 1 <= lmin and lmax <= MAX_MID
    cap = min((lmin - 1) // 2, (MID_TAB_BYTES - 32 * lmax) // (EXT_COL_BYTES - 64))
    x = 0
    while x < cap and ref[P + x] == alt[P + x] and ref[len(ref) - 1 - P - x] == alt[len(alt) - 1 - P - x]:
        x += 1
    return x


def _pad(seqs) -> np.ndarray:
    out = np.full((len(seqs), max(len(s) for s in seqs)), -1, np.int64)
    for i, s in enumerate(seqs):
        out[i, :len(s)] = np.frombuffer(bytes(s), np.uint8)
    return out


def _columns(X, cols, H, E, best):
    """the local-alignment DP of the reads X [B, m] (bytes, -1 = past the read) continued over the haplotype bytes
    `cols` from the column before, (H, E) [B, m] -> (H, E) of the last column and the running maximum of H"""
    r = np.arange(X.shape[1])
    for h in cols:
        diag = np.concatenate([np.zeros((X.shape[0], 1), np.int64), H[:, :-1]], 1)
        E = np.maximum(E + GAP_EXTEND, H + GOE)
        a = np.maximum(np.maximum(diag + np.where(X == h, MATCH, MISMATCH), E), 0)
        # the vertical gap: F(r) = max over r' < r of a(r') + goe + (r - 1 - r') ge
        run = np.maximum.accumulate(a - r * GAP_EXTEND, axis=1)
        F = np.full_like(a, NEG)
        F[:, 1:] = run[:, :-1] + GOE + (r[1:] - 1) * GAP_EXTEND
        H = np.maximum(a, F)
        best = np.maximum(best, H.max(1))
    return H, E, best


def split_scores(reads, ref: bytes, alt: bytes, x: int):
    """(ref scores, alt scores) [B] of the split at 96 + x on both sides, the shared parts scored once"""
    S = P + x
    assert ref[:S] == alt[:S] and ref[len(ref) - S:] == alt[len(alt) - S:] and len(ref) > 2 * S and len(alt) > 2 * S
    X, Xr = _pad(reads), _pad([r[::-1] for r in reads])
    B, m = X.shape
    lens = np.array([len(r) for r in reads])
    edge = (np.zeros((B, m), np.int64), np.full((B, m), NEG, np.int64))
    zero = np.zeros(B, np.int64)
    Hf, Ef, bf = _columns(X, ref[:S], *edge, zero)                       # prefix and extension, forward
    Hr, Er, br = _columns(Xr, ref[::-1][:S], *edge, zero)                # suffix and extension, reversed
    # forward row i meets reversed row len - 2 - i (read row i + 1)
    j = lens[:, None] - 2 - np.arange(m)[None, :]
    ok = j >= 0
    jr = np.clip(j, 0, m - 1)
    Hj, Ej = np.take_along_axis(Hr, jr, 1), np.take_along_axis(Er, jr, 1)
    out = []
    for hap in (ref, alt):
        H, E, b = _columns(X, hap[S:len(hap) - S], Hf, Ef, np.maximum(bf, br))
        cross = np.where(ok, np.maximum(H + Hj, E + Ej - GAP_OPEN), NEG).max(1)
        out.append(np.maximum(b, cross))
    return out


def _base_other(rng, b: int) -> int:
    return int(ACGT[(int(np.nonzero(ACGT == b)[0][0]) + int(rng.integers(1, 4))) % 4])


def _rand(rng, n: int) -> bytes:
    return ACGT[rng.integers(0, 4, n)].tobytes()


KINDS = ("snv", "ins_anchor", "del_anchor", "ins_bare", "del_bare", "mnp")


def window(rng, pad: int, kind: str, alen: int = 1):
    """(ref, alt) windows: `pad` bases either side of a variant, as construct_haplotypes builds them.  Anchored
    indels share their first base (VCF style); bare ones differ from their first base on"""
    left, right = _rand(rng, pad), _rand(rng, pad)
    if kind == "snv":
        ra = _rand(rng, 1); aa = bytes([_base_other(rng, ra[0])])
    elif kind == "mnp":
        ra = _rand(rng, alen); aa = bytes(_base_other(rng, b) for b in ra)
    elif kind in ("ins_anchor", "del_anchor"):
        ra = _rand(rng, 1); aa = ra + _rand(rng, alen)
        if kind == "del_anchor":
            ra, aa = aa, ra
    else:
        ra = _rand(rng, 1); aa = bytes([_base_other(rng, ra[0])]) + _rand(rng, alen)
        if kind == "del_bare":
            ra, aa = aa, ra
    return left + ra + right, left + aa + right


def _mutate(rng, s: bytearray, rate: float):
    for j in np.nonzero(rng.random(len(s)) < rate)[0]:
        s[j] = _base_other(rng, s[j])


def reads(rng, ref: bytes, alt: bytes, x: int, count: int, lengths):
    """`count` reads of the given lengths (cycled) from ref or alt around the variant; most carry a gap or a
    substitution at one of the seams 96 + x (forward) and n - 96 - x (reversed), some are random"""
    out = []
    for k in range(count):
        m = int(lengths[k % len(lengths)])
        hap = ref if rng.random() < 0.5 else alt
        n = len(hap)
        seam = P + x if rng.random() < 0.5 else n - P - x
        style = rng.integers(0, 5)
        if style == 0:                                      # random bases
            out.append(_rand(rng, m)); continue
        g = int(rng.integers(1, 12))
        if style == 1:                                      # hap bases [seam - a, seam + b) skipped: a deletion across the seam
            a = int(rng.integers(1, g + 1)); src = hap[:seam - a] + hap[seam - a + g:]
            c = seam - a
        elif style == 2:                                    # inserted bases at the seam
            src = hap[:seam] + _rand(rng, g) + hap[seam:]
            c = seam
        else:                                               # plain substring, substitutions near the seam
            src = hap; c = seam
        lo = int(np.clip(c - int(rng.integers(0, m + 1)), 0, max(0, len(src) - m)))
        r = bytearray(src[lo:lo + m])
        _mutate(rng, r, 0.02 if style != 4 else 0.15)
        out.append(bytes(r) if r else _rand(rng, m))
    return out
