"""Synthetic inputs for vtx_cluster_refine at the engine level: count entries of a pool of K donors, and a clusters dict as
vtx_cluster_cells returns it.

Each row has a dosage per donor; a cell is a singlet of one donor (or a 50/50 doublet of two) with molecules at random rows,
ALT drawn from the donor's fraction mixed with 10 % pool fraction.  The clusters dict holds each donor's hard sums over a share
of its singlets (x 2^16), so round 0 starts from clusters that are right but shallow, and rows_used marks the rows with at least
four cells on each allele, as §5g does."""
from __future__ import annotations

import numpy as np

import cluster_oracle as CO


def pool(n_rows, n_cols, k, seed, molecules=(5, 400), doublets=0.05, share=0.6):
    """-> (row, col, ref, alt) sorted by (row, col), clusters dict, donor [n_cols] (-1 for doublets)"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, k))
    q = np.array([0.01, 0.5, 0.99])[g]
    f = q.mean(axis=1)
    donor = rng.integers(0, k, n_cols)
    other = (donor + 1 + rng.integers(0, k - 1, n_cols)) % k
    dbl = rng.random(n_cols) < doublets
    ent = {}
    for c in range(n_cols):
        m = int(rng.integers(molecules[0], molecules[1] + 1))
        rows = rng.integers(0, n_rows, m)
        qq = q[rows, donor[c]] if not dbl[c] else (q[rows, donor[c]] + q[rows, other[c]]) / 2
        alt = rng.random(m) < 0.9 * qq + 0.1 * f[rows]
        for v, a in zip(rows.tolist(), alt.tolist()):
            x = ent.setdefault((v, c), [0, 0])
            x[int(a)] += 1
    keys = sorted(ent)
    row = np.array([v for v, _ in keys], np.int64)
    col = np.array([c for _, c in keys], np.int64)
    ref = np.array([ent[x][0] for x in keys], np.int64)
    alt = np.array([ent[x][1] for x in keys], np.int64)
    lab = np.where(~dbl & (rng.random(n_cols) < share), donor, -1)
    w = np.zeros((n_cols, k), np.int64)
    w[np.flatnonzero(lab >= 0), lab[lab >= 0]] = CO.W1
    A, T = CO.msums((row, col, ref, alt), w, n_rows)
    used = CO.used_rows(row, ref, alt, n_rows)
    return (row, col, ref, alt), dict(alt_w=A, depth_w=T, row_used=used.astype(np.uint8)), np.where(dbl, -1, donor)
