"""A restatement of `--out-cluster-calls` / vtx_cluster_refine (DESIGN.md §5j) in NumPy integers and float64 basic operations.

Each round fits §5i's model (cluster_gt_oracle.genotypes) on the round's sums: §5g's final sums in round 0, then the hard sums
of the previous round's singlet labels (cluster_oracle.msums with W = 2^16 on the label's cluster).  The nine-entry tables are
§5h's five (ambient_oracle.tables), the three one-P fractions and f_v itself, each a correctly rounded float64 expression in the
engine's order, so the logs equal the engine's bit for bit; the scores are int64 sums and the calls §5f's rule."""
from __future__ import annotations

import numpy as np

import ambient_oracle as AO
import cluster_gt_oracle as GO
import cluster_oracle as CO
import donor_oracle as DO

P = 3                           # no called genotype: the pool's fraction
NONE = 0xFFFFFFFF               # VTX_NO_LABEL
MAX_ROUNDS = 8                  # the CLI's
W1 = CO.W1


def codes(gt, pl):
    """-> uint8 [rows, K]: GT where GQ >= 20, else P"""
    return np.where(GO.gq(pl) >= GO.MIN_GQ, gt, P).astype(np.uint8)


def entry_of(c1, c2):
    """the table entry of a hypothesis whose clusters have codes c1, c2 (arrays)"""
    c1, c2 = np.asarray(c1, np.int64), np.asarray(c2, np.int64)
    k1, k2 = c1 != P, c2 != P
    return np.where(k1 & k2, c1 + c2, np.where(k1, 5 + c1, np.where(k2, 5 + c2, 8)))


def logs9(m: int, A, T, eps: float):
    """-> La, Lr int64 [rows, 9] at rho = m / 1000: §5h's five, then one P with g = 0, 1, 2, then both P"""
    la5, lr5 = AO.tables(m, A, T, eps)
    q, oq = AO.fractions(eps)
    f, of = AO.row_fraction(A, T)
    rho, orho = m / 1000.0, (1000 - m) / 1000.0
    la1 = CO.fixed(orho * ((q[[0, 2, 4]][None, :] + f[:, None]) * 0.5) + rho * f[:, None])
    lr1 = CO.fixed(orho * ((oq[[0, 2, 4]][None, :] + of[:, None]) * 0.5) + rho * of[:, None])
    return (np.concatenate([la5, la1, CO.fixed(f)[:, None]], axis=1), np.concatenate([lr5, lr1, CO.fixed(of)[:, None]], axis=1))


def sorted_entries(row, col, ref, alt):
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    r, a = np.asarray(ref, np.int64), np.asarray(alt, np.int64)
    o = np.lexsort((col, row))
    return row[o], col[o], r[o], a[o]


def hard_sums(entries, label, k, n_rows):
    """-> A, T int64 [n_rows, k]: 2^16 sum a, 2^16 sum (r + a) over the entries of the cells labelled k"""
    lab = np.asarray(label, np.int64)
    w = np.zeros((lab.size, k), np.int64)
    hit = lab != NONE
    w[np.flatnonzero(hit), lab[hit]] = W1
    return CO.msums(entries, w, n_rows)


def score(entries, sidx, code, la, lr, k, n_cols):
    """-> ll int64 [n_cols, H], counts int64 [n_cols, 3] over the entries at scored rows (sidx >= 0) with r + a > 0"""
    row, col, r, a = entries
    s = sidx[row]
    keep = (s >= 0) & (r + a > 0)
    s, col, r, a = s[keep], col[keep], r[keep], a[keep]
    hyp = np.asarray(DO.hypotheses(k))
    c = code[s]                                                   # [kept, K]
    e = entry_of(c[:, hyp[:, 0]], c[:, hyp[:, 1]])                # [kept, H]
    c9 = r[:, None] * lr[s] + a[:, None] * la[s]                  # [kept, 9]
    ll = CO._segment_sum(np.take_along_axis(c9, e, axis=1), col, n_cols)
    cnt = CO._segment_sum(np.stack([np.ones_like(r), r, a], 1), col, n_cols)
    return ll, cnt


def labels(ll, cnt, k):
    """-> call [n_cols] (0 singlet, 1 doublet, 2 unassigned), label [n_cols]"""
    call, _ = AO.calls(ll, cnt, k)
    return call, np.where(call == 0, ll[:, :k].argmax(axis=1), NONE).astype(np.int64)


def refine(row, col, ref, alt, n_rows, n_cols, clusters: dict, eps: float = GO.ERROR_RATE, max_rounds: int = MAX_ROUNDS) -> dict:
    """-> dict with the fields Engine.cluster_refine returns, plus the labels of every round (round_labels)"""
    entries = sorted_entries(row, col, ref, alt)
    rowA, rowT = GO.row_sums(entries[0], entries[2], entries[3], n_rows)
    A, T = np.asarray(clusters["alt_w"], np.int64), np.asarray(clusters["depth_w"], np.int64)
    k = A.shape[1]
    used = clusters["row_used"]
    prev = np.full(n_cols, NONE, np.int64)
    rounds, round_labels, converged = [], [], False
    for r in range(max_rounds + 1):
        if r:
            A, T = hard_sums(entries, prev, k, n_rows)
        g = GO.genotypes(dict(alt_w=A, depth_w=T, row_used=used), rowA, rowT, None, eps)
        touched = g["touched"].astype(np.int64)
        code = codes(g["gt"], g["pl"])
        scored = (code != P).any(axis=1)
        sidx = np.full(n_rows, -1, np.int64)
        sidx[touched[scored]] = np.arange(int(scored.sum()))
        la, lr = logs9(g["rho_permille"], rowA[touched[scored]], rowT[touched[scored]], eps)
        ll, cnt = score(entries, sidx, code[scored], la, lr, k, n_cols)
        call, lab = labels(ll, cnt, k)
        changed = int((lab != prev).sum())
        rounds.append(dict(rho_permille=g["rho_permille"], rows_fit=g["rows_fit"], n_touched=touched.size, rows_scored=int(scored.sum()),
                           calls=[int((call == x).sum()) for x in range(3)], changed=changed))
        round_labels.append(lab)
        prev = lab
        if r and changed == 0:
            converged = True
            break
    fields = ("rho_permille", "rows_fit", "n_touched", "rows_scored", "changed")
    return dict(k=k, n_hyp=k + k * (k - 1) // 2, n_rounds=len(rounds), converged=converged, ll=ll, counts=cnt, label=lab,
                calls=np.asarray([x["calls"] for x in rounds], np.int64).reshape(-1, 3), touched=g["touched"], gt=g["gt"], pl=g["pl"],
                round_labels=round_labels, **{f: np.asarray([x[f] for x in rounds], np.int64) for f in fields})


# ---- the CLI's file ---------------------------------------------------------------------------------------------------------
def expected(vcf, bam, fasta, barcodes, k, restarts=8, seed=0, **kw):
    """-> (cluster calls text, result, clusters) that --out-cluster-calls should write"""
    keys, row, col, alt, ref = DO.coverage_counts(vcf, bam, fasta, barcodes, **kw)
    n_rows = len(CO.variant_labels(vcf))
    cl = CO.cluster(row, col, ref, alt, n_rows, len(keys), k, restarts, seed)
    res = refine(row, col, ref, alt, n_rows, len(keys), cl)
    return DO.text(CO.names(k), keys, res["ll"].tolist(), res["counts"].tolist()), res, cl
