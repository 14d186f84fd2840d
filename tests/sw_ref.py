"""Independent reference for the engine's Smith-Waterman score, with seam ablations (plain NumPy, no GPU, no oracle).

Affine local alignment (Gotoh) with the engine's constants: match +1, mismatch -5, a gap of length k costs -5 - k.
Rows are read bases (BAM nibbles, decoded through "=ACMGRSVTWYHKDBN"), columns are haplotype bytes, compared by exact
byte equality like vtx_k_sw_generic and oracle/vtx_oracle.c.  Values are int64; a batch of pairs is scored at once,
one DP row at a time:

    F[i][j] = max(F[i-1][j] - 1, H[i-1][j] - 6)                      vertical gap (consumes read bases)
    G[i][j] = max(0, H[i-1][j-1] + s(i, j), F[i][j])                  H without the horizontal gap
    E[i][j] = max_{k < j} G[i][k] - 6 - (j - 1 - k)                   horizontal gap (consumes haplotype bytes)
    H[i][j] = max(G[i][j], E[i][j])                                   answer = max H

E can be taken from G instead of H because opening a gap costs more than extending one: a gap that starts from a
cell whose H came from E scores less than that E continued.  So E is a running maximum along the row.

Ablations remove what one piece of a tiled kernel hands to the next.  A seam is a position, and its kind says what is
lost there:

    column seam c (between haplotype columns c - 1 and c)
        "gap": E entering column c is -inf: no horizontal gap runs from column c - 1 into column c
               (a gap may still open from H of column c - 1);
        "cut": column c sees nothing of column c - 1: H is 0 and E is -inf for both the left and the diagonal
               neighbour (the score becomes the better of the two halves);
    row seam r (between read rows r - 1 and r): the same with F and the upper neighbours.

A kernel that drops a carry computes the ablated score, so a planted case whose true score differs from the ablated
one (its "witness") fails on such a kernel.
"""
from __future__ import annotations

import numpy as np

MATCH, MISMATCH, GAP_OPEN, GAP_EXTEND = 1, -5, -5, -1
GOE = GAP_OPEN + GAP_EXTEND
NEG = -(1 << 40)
DECODE = np.frombuffer(b"=ACMGRSVTWYHKDBN", np.uint8)
NIB = {ord(c): i for i, c in enumerate("=ACMGRSVTWYHKDBN")}


def decode(codes) -> np.ndarray:
    """BAM nibble codes (one per base) -> read bytes."""
    return DECODE[np.asarray(codes, np.uint8)]


def encode(seq: bytes) -> np.ndarray:
    """Read bytes -> BAM nibble codes."""
    return np.array([NIB[b] for b in seq], np.uint8)


def _pad(seqs, fill):
    n = max([len(s) for s in seqs] + [0])
    out = np.full((len(seqs), n), fill, np.int64)
    for i, s in enumerate(seqs):
        out[i, :len(s)] = np.frombuffer(bytes(s), np.uint8)
    return out


def _rows(seams):
    """row seams: r (every column) or (r, lo, hi) (columns [lo, hi) only) -> {r: [(lo, hi), ...]}"""
    out = {}
    for s in seams:
        r, lo, hi = (s, 0, None) if np.isscalar(s) else s
        out.setdefault(int(r), []).append((int(lo), hi))
    return out


def score(reads, haps, col_gap=(), col_cut=(), row_gap=(), row_cut=(), max_cols=None) -> np.ndarray:
    """Scores of the pairs (reads[i] as bytes, haps[i] as bytes), int64 [len(reads)].  The seam lists apply to every
    pair of the call; a row seam is r or (r, lo, hi) to ablate it in columns [lo, hi) only (what row r - 1 hands down
    from those columns: F and H to the same column, H to the diagonal neighbour one column to the right).  max_cols = (lo, hi) takes
    the maximum over those columns only (the DP itself is unchanged).  Reads and haplotypes of different lengths are
    padded with bytes that match nothing; a path through padding only loses score, so the maximum is unchanged."""
    B = len(reads)
    if B == 0:
        return np.zeros(0, np.int64)
    x = _pad(reads, -1)                     # [B, m]
    y = _pad(haps, -2)                      # [B, n]
    m, n = x.shape[1], y.shape[1]
    best = np.zeros(B, np.int64)
    if m == 0 or n == 0:
        return best
    col_gap, col_cut = set(col_gap), set(col_cut)
    row_gap, row_cut = _rows(row_gap), _rows(row_cut)
    mlo, mhi = (0, n) if max_cols is None else max_cols
    # segments of the row: E restarts at every column seam; a segment [c0, c1) takes E only from columns >= c0 - 1
    seams = sorted(c for c in col_gap | col_cut if 0 < c < n)
    bounds = [0] + seams + [n]
    cols = np.arange(n, dtype=np.int64)
    H = np.zeros((B, n), np.int64)          # row i - 1
    F = np.full((B, n), NEG, np.int64)
    cut_cols = np.array(sorted(c for c in col_cut if 0 < c < n), np.int64)
    for i in range(m):
        diag = np.empty_like(H)
        diag[:, 0] = 0
        diag[:, 1:] = H[:, :-1]
        if cut_cols.size:
            diag[:, cut_cols] = 0
        for lo, hi in row_cut.get(i, ()):
            # row i - 1 is hidden in columns [lo, hi): the upper neighbour of columns [lo, hi), the diagonal one of
            # columns [lo + 1, hi + 1)
            H = H.copy(); F = F.copy()
            H[:, lo:hi] = 0; F[:, lo:hi] = NEG; diag[:, lo + 1:None if hi is None else hi + 1] = 0
        Fn = np.maximum(F + GAP_EXTEND, H + GOE)
        for lo, hi in row_gap.get(i, ()):
            Fn[:, lo:hi] = H[:, lo:hi] + GOE
        s = np.where(x[:, i:i + 1] == y, MATCH, MISMATCH)
        G = np.maximum(np.maximum(diag + s, Fn), 0)
        Hn = G.copy()
        for c0, c1 in zip(bounds[:-1], bounds[1:]):
            # left source of the segment: the boundary (H = 0) for c0 = 0, column c0 - 1 for a "gap" seam (its final H),
            # nothing useful for a "cut" seam (H = 0 there: any gap from it scores below 0)
            left = np.zeros(B, np.int64) if c0 == 0 or c0 in col_cut else Hn[:, c0 - 1]
            # E[j] = max(left + GOE + GE * (j - c0), max_{c0 <= k < j} G[k] + GOE + GE * (j - 1 - k))
            k = cols[c0:c1]
            w = G[:, c0:c1] - GAP_EXTEND * k                          # G[k] - GE * k
            run = np.maximum.accumulate(w, axis=1)
            E = np.empty((B, c1 - c0), np.int64)
            E[:, 0] = left + GOE
            if c1 - c0 > 1:
                E[:, 1:] = np.maximum(left[:, None] + GOE + GAP_EXTEND * (k[1:] - c0)[None, :],
                                      run[:, :-1] + GOE + GAP_EXTEND * (k[1:] - 1)[None, :])
            Hn[:, c0:c1] = np.maximum(G[:, c0:c1], E)
        best = np.maximum(best, Hn[:, mlo:mhi].max(axis=1, initial=0))
        H, F = Hn, Fn
    return best


def score_pair(read: bytes, hap: bytes, **seams) -> int:
    return int(score([read], [hap], **seams)[0])
