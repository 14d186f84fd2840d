"""A restatement of `--out-cluster-genotypes` / `--out-cluster-matches` / vtx_cluster_genotypes (DESIGN.md §5i) in NumPy
integers and float64 basic operations.

The genotype fractions are §5h's q_vs for s = 2g (ambient_oracle.tables, whose logs equal the engine's bit for bit), and
everything after them is integer arithmetic.  LL_vkg = floor((A La + R Lr) / 2^16) is exact here without 128-bit integers:
with A = Ah 2^16 + Al (and R likewise) it is Ah La + Rh Lr + floor((Al La + Rl Lr) / 2^16), and every term fits int64 while
depth_w <= 2^51; ll_int states the same value with Python ints.  The clusters come from cluster_oracle.cluster and the counts
from the C oracle (donor_oracle.coverage_counts)."""
from __future__ import annotations

import numpy as np

import ambient_oracle as AO
import cluster_oracle as CO
import donor_oracle as DO

SCALE = 1 << 24
L10 = 38630967                  # llrint(log(10) 2^24)
MAX_PL = (1 << 31) - 1
MAX_GQ = 99
MIN_GQ = 20
MIN_LLR = 5 * SCALE
MISSING = 0xFF
ERROR_RATE = 0.01               # the CLI's (§5f's default)


def logs(m: int, A, T, eps: float):
    """-> La, Lr int64 [rows, 3]: the logs of g = 0, 1, 2 (§5h's fractions s = 0, 2, 4) at rho = m / 1000"""
    la, lr = AO.tables(m, np.asarray(A, np.int64), np.asarray(T, np.int64), eps)
    return la[:, 0::2], lr[:, 0::2]


def gt_ll(A, T, la, lr):
    """floor((A La + (T - A) Lr) / 2^16), exact (broadcasting int64 arrays)"""
    A, T = np.asarray(A, np.int64), np.asarray(T, np.int64)
    R = T - A
    return (A >> 16) * la + (R >> 16) * lr + (((A & 0xFFFF) * la + (R & 0xFFFF) * lr) >> 16)


def ll_int(a: int, t: int, la: int, lr: int) -> int:
    """the same value in Python integers"""
    return (a * la + (t - a) * lr) >> 16


def lls(m: int, Aw, Tw, row_alt, row_depth, eps: float):
    """-> LL int64 [rows, K, 3] of the listed rows"""
    la, lr = logs(m, row_alt, row_depth, eps)
    return gt_ll(np.asarray(Aw)[:, :, None], np.asarray(Tw)[:, :, None], la[:, None, :], lr[:, None, :])


def phred(d):
    """floor((10 d + floor(L10 / 2)) / L10) saturated at 2^31 - 1, for int64 d >= 0 (it saturates for every d >= 2^54)"""
    d = np.asarray(d, np.int64)
    big = d >= (1 << 54)
    q = (np.where(big, 0, d) * 10 + L10 // 2) // L10
    return np.where(big, MAX_PL, np.minimum(q, MAX_PL)).astype(np.int64)


def phred_int(d: int) -> int:
    return min((10 * d + L10 // 2) // L10, MAX_PL)


def call(ll, T):
    """-> GT uint8 [rows, K] (MISSING where T = 0), PL int64 [rows, K, 3] (0 there)"""
    reached = np.asarray(T) > 0
    gt = np.where(reached, ll.argmax(axis=2), MISSING).astype(np.uint8)
    pl = np.where(reached[..., None], phred(ll.max(axis=2)[..., None] - ll), 0)
    return gt, pl


def gq(pl):
    return np.minimum(np.sort(pl, axis=-1)[..., 1], MAX_GQ)


def match(ll, gt, pl, T, g):
    """over compared rows: ll [n, K, 3], gt / T [n, K], pl [n, K, 3], g [n, S] -> M, discordant [K, S], rows, called [K]"""
    called = gq(pl) >= MIN_GQ
    K, S = ll.shape[1], g.shape[1]
    M = np.zeros((K, S), np.int64)
    agree = np.zeros((K, S), np.int64)
    for x in range(3):
        one = (g == x).astype(np.int64)
        M += ll[:, :, x].T @ one
        agree += (called & (gt == x)).astype(np.int64).T @ one
    return M, called.sum(axis=0)[:, None] - agree, (np.asarray(T) > 0).sum(axis=0), called.sum(axis=0)


def assign(M, disc, called: int):
    """one cluster's (best, second or None, llr or None, assigned) from its M [S], discordant [S]"""
    S = len(M)
    best = max(range(S), key=lambda s: (M[s], -s))
    if S == 1:
        return best, None, None, int(disc[best]) * 10 <= called
    second = max((s for s in range(S) if s != best), key=lambda s: (M[s], -s))
    llr = int(M[best]) - int(M[second])
    return best, second, llr, int(disc[best]) * 10 <= called and llr >= MIN_LLR


def genotypes(clusters: dict, row_alt, row_depth, dosage=None, eps: float = ERROR_RATE, rho=None) -> dict:
    """-> dict with the fields Engine.cluster_genotypes returns; rho None estimates it, else the given m"""
    Aw, Tw = np.asarray(clusters["alt_w"], np.int64), np.asarray(clusters["depth_w"], np.int64)
    K = Aw.shape[1]
    used = np.asarray(clusters["row_used"]) != 0
    touched = np.flatnonzero((Tw > 0).any(axis=1))
    At, Tt = Aw[touched], Tw[touched]
    ra, rd = np.asarray(row_alt, np.int64)[touched], np.asarray(row_depth, np.int64)[touched]
    fit = used[touched]

    def objective(m):
        return (int(lls(m, At[fit], Tt[fit], ra[fit], rd[fit], eps).max(axis=2).sum()),)
    grid = {}
    if rho is None:
        for m in AO.COARSE:
            grid[m] = objective(m)
        mc = AO.best_of(grid)
        for m in range(max(0, mc - AO.FINE_REACH), min(AO.MAX_PERMILLE, mc + AO.FINE_REACH) + 1):
            if m not in grid:
                grid[m] = objective(m)
        chosen = AO.best_of(grid)
    else:
        chosen = int(rho)
        grid[chosen] = objective(chosen)
    ll = lls(chosen, At, Tt, ra, rd, eps)
    gt, pl = call(ll, Tt)
    S = 0 if dosage is None else np.asarray(dosage).shape[1]
    out = dict(rho_permille=chosen, rho=chosen / 1000, rows_fit=int(fit.sum()), rows_compared=0,
               grid_permille=np.asarray(sorted(grid), np.uint16), grid_objective=np.asarray([grid[m][0] for m in sorted(grid)], np.int64),
               touched=touched.astype(np.uint64), gt=gt, pl=pl, ll=ll, match_ll=np.zeros((K, S), np.int64),
               match_discordant=np.zeros((K, S), np.int64), match_rows=np.zeros(K, np.int64), match_called=np.zeros(K, np.int64))
    if S:
        g = np.asarray(dosage, np.uint8)
        every = (g <= 2).all(axis=1)
        cmp = every[touched]
        out["rows_compared"] = int(every.sum())
        out["match_ll"], out["match_discordant"], out["match_rows"], out["match_called"] = match(ll[cmp], gt[cmp], pl[cmp], Tt[cmp],
                                                                                               g[touched][cmp])
    return out


# ---- the CLI's two files --------------------------------------------------------------------------------------------------
def records(vcf: str):
    """-> [(CHROM, POS, ID, REF, ALT)] as written"""
    out = []
    for ln in open(vcf):
        if ln.startswith("#") or not ln.strip():
            continue
        f = ln.rstrip("\n").split("\t")
        out.append(tuple(f[:5]))
    return out


def genotypes_text(recs, clusters, res) -> str:
    K = res["gt"].shape[1]
    lines = ["##fileformat=VCFv4.2", "##source=vartrix_b200", f"##vartrix_ambient_rna={res['rho_permille'] / 1000:.3f}",
             "##vartrix_ambient_rna_estimated=true",
             '##INFO=<ID=USED,Number=0,Type=Flag,Description="The cells were clustered and the ambient fraction fitted on this variant">',
             '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">',
             '##FORMAT=<ID=GQ,Number=1,Type=Integer,Description="Genotype quality: the second-smallest PL, at most 99">',
             '##FORMAT=<ID=PL,Number=G,Type=Integer,Description="Phred-scaled genotype likelihoods, with the pool\'s ambient RNA mixed in">',
             "\t".join(["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"] + CO.names(K))]
    q = gq(res["pl"])
    for i, v in enumerate(res["touched"].tolist()):
        f = list(recs[v]) + [".", ".", "USED" if clusters["row_used"][v] else ".", "GT:GQ:PL"]
        for j in range(K):
            g = int(res["gt"][i, j])
            p = res["pl"][i, j].tolist()
            f.append("./." if g == MISSING else f"{('0/0', '0/1', '1/1')[g]}:{int(q[i, j])}:{p[0]},{p[1]},{p[2]}")
        lines.append("\t".join(f))
    return "\n".join(lines) + "\n"


def matches_text(samples, res) -> str:
    S = len(samples)
    lines = ["\t".join(["cluster", "rows", "called", "best_sample", "discordant", "second_sample", "llr", "assignment"] +
                       [f"ll_{s}" for s in samples])]
    for j in range(res["match_ll"].shape[0]):
        M, disc = res["match_ll"][j].tolist(), res["match_discordant"][j].tolist()
        called = int(res["match_called"][j])
        best, second, llr, ok = assign(M, disc, called)
        lines.append("\t".join([f"C{j}", str(int(res["match_rows"][j])), str(called), samples[best], str(disc[best]),
                                "." if second is None else samples[second], "." if llr is None else f"{llr / SCALE:.6f}",
                                samples[best] if ok else "."] + [f"{x / SCALE:.6f}" for x in M]))
    return "\n".join(lines) + "\n"


def row_sums(row, ref, alt, n_rows):
    A = np.zeros(n_rows, np.int64)
    T = np.zeros(n_rows, np.int64)
    np.add.at(A, np.asarray(row, np.int64), np.asarray(alt, np.int64))
    np.add.at(T, np.asarray(row, np.int64), np.asarray(ref, np.int64) + np.asarray(alt, np.int64))
    return A, T


def expected(vcf, bam, fasta, barcodes, k, restarts=8, seed=0, **kw):
    """-> (genotypes text, matches text, result, clusters) that --out-cluster-genotypes / --out-cluster-matches should write"""
    samples, dosage = DO.read_genotypes(vcf)
    keys, row, col, alt, ref = DO.coverage_counts(vcf, bam, fasta, barcodes, **kw)
    recs = records(vcf)
    cl = CO.cluster(row, col, ref, alt, len(recs), len(keys), k, restarts, seed)
    A, T = row_sums(row, ref, alt, len(recs))
    res = genotypes(cl, A, T, dosage)
    return genotypes_text(recs, cl, res), matches_text(samples, res), res, cl
