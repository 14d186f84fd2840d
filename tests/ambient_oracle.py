"""A restatement of `--ambient-rna` / vtx_donors_ambient (DESIGN.md §5h) in NumPy integers and float64 basic operations.

The model is §5f's (donor_oracle: GT parse, hypotheses, counts, file text) with every hypothesis's ALT fraction mixed with the
pool's: q_vs = (1 - rho) q_s + rho f_v.  The logs are cluster_oracle.ll_log, which equals the engine's bit for bit (NumPy
evaluates every +, *, / of a float64 array as one correctly rounded operation), and everything after them is int64."""
from __future__ import annotations

import numpy as np

import cluster_oracle as CO
import donor_oracle as DO

SCALE = DO.SCALE
THRESHOLD = DO.THRESHOLD
MAX_PERMILLE = 500
COARSE = list(range(0, MAX_PERMILLE + 1, 10))
FINE_REACH = 9


def fractions(eps: float):
    """§5f's q_s and 1 - q_s, in make_tables' expressions"""
    q = [eps, (eps + 0.5) / 2, 0.5, (1.5 - eps) / 2, 1 - eps]
    return np.array(q), np.array([1 - x for x in q])


def row_fraction(A, T):
    """f_v and 1 - f_v of the row sums, each its own quotient"""
    A, T = np.asarray(A, np.int64), np.asarray(T, np.int64)
    den = (T + 2).astype(np.float64)
    return (A + 1).astype(np.float64) / den, (T - A + 1).astype(np.float64) / den


def tables(m: int, A, T, eps: float):
    """-> La, Lr int64 [rows, 5] at rho = m / 1000"""
    q, oq = fractions(eps)
    f, of = row_fraction(A, T)
    rho, orho = m / 1000.0, (1000 - m) / 1000.0
    return CO.fixed(orho * q[None, :] + rho * f[:, None]), CO.fixed(orho * oq[None, :] + rho * of[:, None])


def prepare(row, col, ref, alt, n_rows, dosage):
    """-> dict: the entries sorted by (row, col), A / T per row, the kept entries (usable row, r + a > 0) and their index s
    per hypothesis"""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    r, a = np.asarray(ref, np.int64), np.asarray(alt, np.int64)
    o = np.lexsort((col, row))
    row, col, r, a = row[o], col[o], r[o], a[o]
    g = np.asarray(dosage, np.uint8).reshape(n_rows, -1)
    d = g.shape[1]
    usable = (g <= 2).all(axis=1)
    A = np.zeros(n_rows, np.int64)
    np.add.at(A, row, a)
    T = np.zeros(n_rows, np.int64)
    np.add.at(T, row, r + a)
    keep = usable[row] & (r + a > 0)
    hyp = np.asarray(DO.hypotheses(d))
    kr = row[keep]
    s = g[kr][:, hyp[:, 0]].astype(np.int64) + g[kr][:, hyp[:, 1]].astype(np.int64)      # [kept, H]
    touched, tix = np.unique(kr, return_inverse=True)
    return dict(d=d, n_rows=n_rows, usable=usable, A=A, T=T, row=kr, col=col[keep], r=r[keep], a=a[keep], s=s, touched=touched,
                tix=tix.reshape(-1))


def score(p, m: int, eps: float, n_cols: int):
    """-> ll int64 [n_cols, H], counts int64 [n_cols, 3] at rho = m / 1000"""
    la, lr = tables(m, p["A"][p["touched"]], p["T"][p["touched"]], eps)     # the rows some kept entry touches
    t, r, a = p["tix"], p["r"], p["a"]
    c5 = r[:, None] * lr[t] + a[:, None] * la[t]                              # [kept, 5]
    per = np.take_along_axis(c5, p["s"], axis=1)                               # [kept, H]
    ll = np.zeros((n_cols, p["s"].shape[1]), np.int64)
    np.add.at(ll, p["col"], per)
    cnt = np.zeros((n_cols, 3), np.int64)
    np.add.at(cnt, p["col"], np.stack([np.ones_like(r), r, a], 1))
    return ll, cnt


def calls(ll, cnt, d: int):
    """-> int [n_cols]: 0 singlet, 1 doublet, 2 unassigned (§5f's rule); and max_h LL [n_cols]"""
    sing = np.sort(ll[:, :d], axis=1)
    best, second = sing[:, -1], sing[:, -2]
    pair = ll[:, d:].max(axis=1)
    call = np.where(cnt[:, 0] == 0, 2, np.where(pair - best >= THRESHOLD, 1, np.where(best - second >= THRESHOLD, 0, 2)))
    return call, np.maximum(best, pair)


def evaluate(p, m, eps, n_cols):
    """-> (J, [singlet, doublet, unassigned]) at m"""
    ll, cnt = score(p, m, eps, n_cols)
    call, mx = calls(ll, cnt, p["d"])
    return int(mx[cnt[:, 0] > 0].sum()), [int((call == k).sum()) for k in range(3)]


def best_of(grid):
    """the largest J, ties the smallest m; grid = {m: (J, calls)}"""
    return max(grid, key=lambda m: (grid[m][0], -m))


def ambient(row, col, ref, alt, n_rows, n_cols, dosage, eps=0.01, rho=None):
    """-> dict with the fields of vtx_ambient (NumPy arrays); rho None estimates it, else the given m (thousandths)"""
    p = prepare(row, col, ref, alt, n_rows, dosage)
    grid = {}
    if rho is None:
        for m in COARSE:
            grid[m] = evaluate(p, m, eps, n_cols)
        mc = best_of(grid)
        for m in range(max(0, mc - FINE_REACH), min(MAX_PERMILLE, mc + FINE_REACH) + 1):
            if m not in grid:
                grid[m] = evaluate(p, m, eps, n_cols)
        chosen = best_of(grid)
    else:
        chosen = int(rho)
        grid[chosen] = evaluate(p, chosen, eps, n_cols)
    ll, cnt = score(p, chosen, eps, n_cols)
    ms = sorted(grid)
    d = p["d"]
    return dict(rho_permille=chosen, n_hyp=d + d * (d - 1) // 2, rows_usable=int(p["usable"].sum()), ll=ll, counts=cnt,
                grid_permille=np.asarray(ms, np.uint16), grid_objective=np.asarray([grid[m][0] for m in ms], np.int64),
                grid_calls=np.asarray([grid[m][1] for m in ms], np.int64).reshape(len(ms), 3),
                row_alt=p["A"], row_depth=p["T"])


# ---- the CLI's two files --------------------------------------------------------------------------------------------------
def ambient_text(res) -> str:
    lines = ["rho\tobjective\tsinglet\tdoublet\tunassigned\tchosen"]
    for m, j, c in zip(res["grid_permille"].tolist(), res["grid_objective"].tolist(), res["grid_calls"].tolist()):
        lines.append(f"{m / 1000:.3f}\t{j / SCALE:.6f}\t{c[0]}\t{c[1]}\t{c[2]}\t{int(m == res['rho_permille'])}")
    return "\n".join(lines) + "\n"


def parse_mode(mode: str):
    """--ambient-rna MODE -> None (estimate) or m"""
    return None if mode == "estimate" else int(round(float(mode) * 1000))


def expected(vcf, bam, fasta, barcodes, mode="estimate", donors=None, error_rate=0.01, **kw):
    """-> (donors text, ambient text, result) that the CLI's --out-donors / --out-ambient should write with --ambient-rna MODE"""
    samples, dosage = DO.read_genotypes(vcf)
    names, table = DO.select(samples, dosage, donors)
    keys, row, col, alt, ref = DO.coverage_counts(vcf, bam, fasta, barcodes, **kw)
    res = ambient(row, col, ref, alt, table.shape[0], len(keys), table, error_rate, parse_mode(mode))
    return DO.text(names, keys, res["ll"].tolist(), res["counts"].tolist()), ambient_text(res), res
