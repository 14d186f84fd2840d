"""A restatement of `--out-clusters` / vtx_cluster_cells (DESIGN.md §5g) in NumPy integers and float64 basic operations.

ll_log / ll_exp are written op for op as in vtx_clusters.cuh: NumPy evaluates every +, -, *, / of a float64 array as one
correctly rounded IEEE operation (no contraction), and frexp / ldexp / trunc are exact, so the tables, weights and scores
equal the engine's bit for bit.  Everything after the logs is int64 arithmetic.  The counts of a pooled data set come from
the C oracle in coverage mode (donor_oracle.coverage_counts): the REF / ALT counts the matrix is built from in every -s mode."""
from __future__ import annotations

import numpy as np

import donor_oracle as DO

SCALE = 1 << 24
W1 = 1 << 16
MIN_CELLS = 4
MAX_ITERS = 200
LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
INV_LN2, SQRT_HALF = 1.44269504088896338700e+00, 0.70710678118654752440
M64 = (1 << 64) - 1


def ll_log(x):
    x = np.asarray(x, np.float64)
    m, e = np.frexp(x)
    small = m < SQRT_HALF
    m = np.where(small, np.ldexp(m, 1), m)
    e = np.where(small, e - 1, e)
    s = (m - 1.0) / (m + 1.0)
    z = s * s
    p = np.full_like(s, 1.0 / 21)
    for d in (19, 17, 15, 13, 11, 9, 7, 5, 3):
        p = 1.0 / d + z * p
    s2 = 2.0 * s
    lm = s2 + s2 * (z * p)
    de = e.astype(np.float64)
    return de * LN2_HI + (de * LN2_LO + lm)


def ll_exp(x):
    x = np.asarray(x, np.float64)
    n = np.trunc(x * INV_LN2 - 0.5)
    n = np.where(x < -40.0, 0.0, n)
    r = (x - n * LN2_HI) - n * LN2_LO
    p = np.full_like(r, 1.0 / 6227020800.0)
    for f in (479001600.0, 39916800.0, 3628800.0, 362880.0, 40320.0, 5040.0, 720.0, 120.0, 24.0, 6.0):
        p = 1.0 / f + r * p
    for c in (0.5, 1.0, 1.0):
        p = c + r * p
    return np.where(x < -40.0, 0.0, np.ldexp(p, n.astype(np.int32)))


def fixed(x):
    """llrint(ll_log(x) 2^24): round half to even"""
    return np.rint(ll_log(x) * float(SCALE)).astype(np.int64)


def splitmix64(x: int) -> int:
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def splitmix64_np(x):
    """splitmix64 of a uint64 array (wrapping arithmetic)"""
    with np.errstate(over="ignore"):
        z = x + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def init_logs(seed: int, s: int, k: int, rows):
    """restart s's first La / Lr [len(rows), k]"""
    key = np.uint64(seed ^ (s << 48)) ^ (np.arange(k, dtype=np.uint64)[None, :] << np.uint64(40)) ^ np.asarray(rows, np.uint64)[:, None]
    u = (splitmix64_np(key) >> np.uint64(11)).astype(np.float64)
    th = 0.05 + 0.9 * (u * (1.0 / 9007199254740992.0))
    return fixed(th), fixed(1.0 - th)


def theta(A, T):
    den = (T + 2 * W1).astype(np.float64)
    return (A + W1).astype(np.float64) / den, (T - A + W1).astype(np.float64) / den


def row_logs(A, T):
    th, om = theta(A, T)
    return fixed(th), fixed(om)


def _segment_sum(vals, key, n):
    """int64 sums of vals [m, K] grouped by key (any order), [n, K]"""
    out = np.zeros((n, vals.shape[1]), np.int64)
    if len(key):
        order = np.argsort(key, kind="stable")
        k = key[order]
        starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
        out[k[starts]] = np.add.reduceat(vals[order], starts, axis=0)
    return out


def estep(cells, la, lr, n_cols):
    """-> W int64 [n_cols, K], m [n_cols]; cells = (row, col, r, a) of the used entries"""
    row, col, r, a = cells
    ll = _segment_sum(r[:, None] * lr[row] + a[:, None] * la[row], col, n_cols)
    m = ll.max(axis=1)
    e = np.rint(ll_exp((ll - m[:, None]).astype(np.float64) * (1.0 / SCALE)) * float(1 << 40)).astype(np.int64)
    w = (e << 16) // e.sum(axis=1)[:, None]
    return w, m


def msums(entries, w, n_rows):
    """-> A, T int64 [n_rows, K] over the given entries"""
    row, col, r, a = entries
    return _segment_sum(w[col] * a[:, None], row, n_rows), _segment_sum(w[col] * (r + a)[:, None], row, n_rows)


def used_rows(row, r, a, n_rows):
    return (np.bincount(row[r > 0], minlength=n_rows) >= MIN_CELLS) & (np.bincount(row[a > 0], minlength=n_rows) >= MIN_CELLS)


def score(cells, A, T, k, n_cols):
    """-> ll int64 [n_cols, H] (canonical A, T) and counts [n_cols, 3]"""
    row, col, r, a = cells
    hyp = np.asarray(DO.hypotheses(k))
    th, om = theta(A, T)
    la = fixed((th[:, hyp[:, 0]] + th[:, hyp[:, 1]]) * 0.5)
    lr = fixed((om[:, hyp[:, 0]] + om[:, hyp[:, 1]]) * 0.5)
    ll = _segment_sum(r[:, None] * lr[row] + a[:, None] * la[row], col, n_cols)
    cnt = _segment_sum(np.stack([np.ones_like(r), r, a], 1), col, n_cols)
    return ll, cnt


def cluster(row, col, ref, alt, n_rows, n_cols, k, restarts=8, seed=0):
    """-> dict with the fields of vtx_clusters (NumPy arrays)"""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    r, a = np.asarray(ref, np.int64), np.asarray(alt, np.int64)
    o = np.lexsort((col, row))
    row, col, r, a = row[o], col[o], r[o], a[o]
    used = used_rows(row, r, a, n_rows)
    keep = used[row] & (r + a > 0)
    cells = (row[keep], col[keep], r[keep], a[keep])
    urows = np.flatnonzero(used)
    entries_used = tuple(x[used[row]] for x in (row, col, r, a))
    scores, iters, finals = [], [], []
    for s in range(restarts):
        la = np.zeros((n_rows, k), np.int64)
        lr = np.zeros((n_rows, k), np.int64)
        la[urows], lr[urows] = init_logs(seed, s, k, urows)
        prev = np.full((n_cols, k), -1, np.int64)
        for it in range(1, MAX_ITERS + 1):
            w, m = estep(cells, la, lr, n_cols)
            changed = bool((w != prev).any())
            prev = w
            if not changed or it == MAX_ITERS:
                break
            A, T = msums(entries_used, w, n_rows)
            la[urows], lr[urows] = row_logs(A[urows], T[urows])
        scores.append(int(m.sum()))
        iters.append(it)
        finals.append(w)
    best = max(range(restarts), key=lambda s: (scores[s], -s))
    w = finals[best]
    tot = w.sum(axis=0)
    perm = sorted(range(k), key=lambda j: (-int(tot[j]), j))
    A, T = msums((row, col, r, a), w[:, perm], n_rows)
    ll, cnt = score(cells, A, T, k, n_cols)
    return dict(k=k, n_hyp=k + k * (k - 1) // 2, best_restart=best, rows_used=int(used.sum()), ll=ll, counts=cnt,
                row_used=used.astype(np.uint8), alt_w=A, depth_w=T, restart_score=np.asarray(scores, np.int64),
                restart_iters=np.asarray(iters, np.uint32))


# ---- the CLI's two files --------------------------------------------------------------------------------------------------
def names(k):
    return [f"C{j}" for j in range(k)]


def clusters_text(barcodes, res) -> str:
    k = res["k"]
    return DO.text(names(k), barcodes, res["ll"].tolist(), res["counts"].tolist())


def variant_labels(vcf: str):
    out = []
    for ln in open(vcf):
        if ln.startswith("#") or not ln.strip():
            continue
        f = ln.split("\t")
        out.append(f"{f[0]}_{int(f[1]) - 1}")
    return out


def alleles_text(labels, res) -> str:
    k = res["k"]
    lines = ["\t".join(["variant", "used"] + [x for j in range(k) for x in (f"ref_C{j}", f"alt_C{j}")])]
    A, T = res["alt_w"].tolist(), res["depth_w"].tolist()
    for v, lab in enumerate(labels):
        f = [lab, str(int(res["row_used"][v]))]
        for j in range(k):
            f += [f"{(T[v][j] - A[v][j]) / W1:.4f}", f"{A[v][j] / W1:.4f}"]
        lines.append("\t".join(f))
    return "\n".join(lines) + "\n"


def calls(text: str):
    """-> [(barcode, variants, call, assignment)] of a clusters file"""
    out = []
    for ln in text.splitlines()[1:]:
        f = ln.split("\t")
        out.append((f[0], int(f[1]), f[4], f[5]))
    return out


def expected(vcf, bam, fasta, barcodes, k, restarts=8, seed=0, **kw):
    """-> (clusters text, alleles text, result) that the CLI's --out-clusters / --out-cluster-alleles should write"""
    keys, row, col, alt, ref = DO.coverage_counts(vcf, bam, fasta, barcodes, **kw)
    labels = variant_labels(vcf)
    res = cluster(row, col, ref, alt, len(labels), len(keys), k, restarts, seed)
    return clusters_text(keys, res), alleles_text(labels, res), res
