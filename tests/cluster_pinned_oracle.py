"""A restatement of `--known-donors` / vtx_cluster_cells_pinned (DESIGN.md §5k) on top of cluster_oracle and ambient_oracle.

§5g's EM (cluster_oracle) with the first J clusters pinned: where pinned sample j has a dosage g at row v, cluster j's La / Lr
are §5h's table entries s = 2g at m (ambient_oracle.tables), written over the init and again after every M-step, and the final
scoring takes its theta in the same expressions.  Free clusters are relabelled among themselves.  Every float64 operation is
one correctly rounded IEEE operation and everything after the logs is int64, so the engine matches this bit for bit; with
J = 0 this is cluster_oracle.cluster."""
from __future__ import annotations

import numpy as np

import ambient_oracle as AO
import cluster_oracle as CO
import donor_oracle as DO

MISSING = DO.MISSING


def _s(g):
    """§5h's fraction index s = 2g of a dosage table (0 where missing; those entries are never used)"""
    return 2 * np.where(g == MISSING, 0, g).astype(np.int64)


def pinned_logs(g, m: int, row_alt, row_depth, eps: float):
    """-> La, Lr int64 [rows, J] of dosage table g [rows, J] at rows of sums A_v, T_v"""
    la5, lr5 = AO.tables(m, row_alt, row_depth, eps)
    s = _s(g)
    return np.take_along_axis(la5, s, axis=1), np.take_along_axis(lr5, s, axis=1)


def pinned_theta(g, m: int, row_alt, row_depth, eps: float):
    """-> theta, 1 - theta float64 [rows, J]: the fractions whose logs pinned_logs takes, in ambient_oracle.tables' expressions"""
    q, oq = AO.fractions(eps)
    f, of = AO.row_fraction(row_alt, row_depth)
    rho, orho = m / 1000.0, (1000 - m) / 1000.0
    s = _s(g)
    return orho * q[s] + rho * f[:, None], orho * oq[s] + rho * of[:, None]


def score(cells, A, T, k, n_cols, g, m, row_alt, row_depth, eps):
    """-> ll int64 [n_cols, H], counts [n_cols, 3]: cluster_oracle.score with the pinned clusters' theta where they have a dosage"""
    row, col, r, a = cells
    th, om = CO.theta(A, T)
    J = g.shape[1]
    if J:
        pth, pom = pinned_theta(g, m, row_alt, row_depth, eps)
        has = g != MISSING
        th[:, :J] = np.where(has, pth, th[:, :J])
        om[:, :J] = np.where(has, pom, om[:, :J])
    hyp = np.asarray(DO.hypotheses(k))
    la = CO.fixed((th[:, hyp[:, 0]] + th[:, hyp[:, 1]]) * 0.5)
    lr = CO.fixed((om[:, hyp[:, 0]] + om[:, hyp[:, 1]]) * 0.5)
    ll = CO._segment_sum(r[:, None] * lr[row] + a[:, None] * la[row], col, n_cols)
    cnt = CO._segment_sum(np.stack([np.ones_like(r), r, a], 1), col, n_cols)
    return ll, cnt


def row_sums(row, ref, alt, n_rows):
    """A_v, T_v over every entry"""
    A = np.zeros(n_rows, np.int64)
    np.add.at(A, np.asarray(row, np.int64), np.asarray(alt, np.int64))
    T = np.zeros(n_rows, np.int64)
    np.add.at(T, np.asarray(row, np.int64), np.asarray(ref, np.int64) + np.asarray(alt, np.int64))
    return A, T


def cluster_pinned(row, col, ref, alt, n_rows, n_cols, k, dosage, rho_permille=0, error_rate=0.01, restarts=8, seed=0):
    """-> dict with the fields of vtx_clusters (NumPy arrays); dosage uint8 [n_rows, J] (J = 0: cluster_oracle.cluster)"""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    r, a = np.asarray(ref, np.int64), np.asarray(alt, np.int64)
    g = np.asarray(dosage, np.uint8).reshape(n_rows, -1)
    J, m, eps = g.shape[1], int(rho_permille), float(error_rate)
    assert 0 <= J < k
    o = np.lexsort((col, row))
    row, col, r, a = row[o], col[o], r[o], a[o]
    rowA, rowT = row_sums(row, r, a, n_rows)
    used = CO.used_rows(row, r, a, n_rows)
    keep = used[row] & (r + a > 0)
    cells = (row[keep], col[keep], r[keep], a[keep])
    urows = np.flatnonzero(used)
    entries_used = tuple(x[used[row]] for x in (row, col, r, a))
    gu = g[urows]
    has = gu != MISSING
    pla, plr = pinned_logs(gu, m, rowA[urows], rowT[urows], eps)

    def pin(la, lr):
        la[urows, :J] = np.where(has, pla, la[urows, :J])
        lr[urows, :J] = np.where(has, plr, lr[urows, :J])

    scores, iters, finals = [], [], []
    for s in range(restarts):
        la = np.zeros((n_rows, k), np.int64)
        lr = np.zeros((n_rows, k), np.int64)
        la[urows], lr[urows] = CO.init_logs(seed, s, k, urows)
        pin(la, lr)
        prev = np.full((n_cols, k), -1, np.int64)
        for it in range(1, CO.MAX_ITERS + 1):
            w, mc = CO.estep(cells, la, lr, n_cols)
            changed = bool((w != prev).any())
            prev = w
            if not changed or it == CO.MAX_ITERS:
                break
            A, T = CO.msums(entries_used, w, n_rows)
            la[urows], lr[urows] = CO.row_logs(A[urows], T[urows])
            pin(la, lr)
        scores.append(int(mc.sum()))
        iters.append(it)
        finals.append(w)
    best = max(range(restarts), key=lambda s: (scores[s], -s))
    w = finals[best]
    tot = w.sum(axis=0)
    perm = list(range(J)) + sorted(range(J, k), key=lambda j: (-int(tot[j]), j))
    A, T = CO.msums((row, col, r, a), w[:, perm], n_rows)
    ll, cnt = score(cells, A, T, k, n_cols, g, m, rowA, rowT, eps)
    return dict(k=k, n_hyp=k + k * (k - 1) // 2, best_restart=best, rows_used=int(used.sum()), ll=ll, counts=cnt,
                row_used=used.astype(np.uint8), alt_w=A, depth_w=T, restart_score=np.asarray(scores, np.int64),
                restart_iters=np.asarray(iters, np.uint32))


# ---- the CLI's two files --------------------------------------------------------------------------------------------------
def names(known, k):
    """the known samples, then C0 .. C{k - J - 1}"""
    return list(known) + [f"C{j}" for j in range(k - len(known))]


def clusters_text(barcodes, res, known) -> str:
    return DO.text(names(known, res["k"]), barcodes, res["ll"].tolist(), res["counts"].tolist())


def alleles_text(labels, res, known) -> str:
    """cluster_oracle.alleles_text with the clusters' names in the header"""
    text = CO.alleles_text(labels, res)
    head, rest = text.split("\n", 1)
    nm = names(known, res["k"])
    return "\t".join(["variant", "used"] + [x for n in nm for x in (f"ref_{n}", f"alt_{n}")]) + "\n" + rest


def expected(vcf, bam, fasta, barcodes, k, known, rho_permille=0, restarts=8, seed=0, error_rate=0.01, **kw):
    """-> (clusters text, alleles text, result) that the CLI's --out-clusters / --out-cluster-alleles should write with
    --known-donors KNOWN (and --ambient-rna rho_permille / 1000)"""
    samples, dosage = DO.read_genotypes(vcf)
    _, table = DO.select(samples, dosage, list(known))
    keys, row, col, alt, ref = DO.coverage_counts(vcf, bam, fasta, barcodes, **kw)
    labels = CO.variant_labels(vcf)
    res = cluster_pinned(row, col, ref, alt, len(labels), len(keys), k, table, rho_permille, error_rate, restarts, seed)
    return clusters_text(keys, res, known), alleles_text(labels, res, known), res
