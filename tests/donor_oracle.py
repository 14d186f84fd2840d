"""An independent restatement of `--out-donors` (DESIGN.md §5f): per-cell singlet / doublet log-likelihoods from the donors'
VCF genotypes and the cells' REF / ALT counts.

The genotypes come from this module's own parse of the VCF's GT columns.  The counts come from the existing CPU expectations
in coverage mode (baseq_oracle.run_files with scoring_method="coverage": the unchanged C oracle's triplets, val = ALT and
val2 = REF after the UMI or name-key collapse), so they are the counts the matrix is built from in every `-s` mode.  The model
is applied in Python integers; the ten log constants use math.log from the same libm as the CLI's log."""
from __future__ import annotations

import gzip
import math

import numpy as np

import baseq_oracle as B

MISSING = 0xFF
SCALE = 1 << 24
THRESHOLD = 5 * SCALE


def gt_dosage(gt: str) -> int:
    """ALT dosage of one GT value: diploid a/b or a|b over {0, 1} -> the number of 1s, haploid 0 -> 0, haploid 1 -> 2,
    anything else missing."""
    alleles = gt.replace("|", "/").split("/")
    if any(a not in ("0", "1") for a in alleles) or len(alleles) > 2:
        return MISSING
    ones = sum(a == "1" for a in alleles)
    return 2 * ones if len(alleles) == 1 else ones


def read_genotypes(vcf: str):
    """-> (sample names in header order, uint8[records, samples] dosage)"""
    with open(vcf, "rb") as fh:
        data = fh.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    samples, rows = [], []
    for raw in lines:
        ln = raw.decode()
        ln = ln[:-1] if ln.endswith("\r") else ln
        if ln.startswith("#CHROM"):
            samples = ln.split("\t")[9:]
            continue
        if not ln or ln.startswith("#"):
            continue
        f = ln.split("\t")
        cols = f[9:]
        if len(cols) != len(samples):
            raise ValueError(f"malformed VCF line: {len(cols)} sample columns, the header has {len(samples)}")
        keys = f[8].split(":") if len(f) > 8 else []
        gt = keys.index("GT") if "GT" in keys else None
        row = []
        for c in cols:
            sub = c.split(":")
            row.append(gt_dosage(sub[gt]) if gt is not None and gt < len(sub) else MISSING)
        rows.append(row)
    return samples, np.asarray(rows, np.uint8).reshape(len(rows), len(samples))


def hypotheses(d: int):
    """[(d1, d2)] in the model's order: singlets (h, h), then the doublets (0,1), (0,2), ..., (d-2, d-1)"""
    return [(h, h) for h in range(d)] + [(a, b) for a in range(d) for b in range(a + 1, d)]


def tables(eps: float):
    q = [eps, (eps + 0.5) / 2, 0.5, (1.5 - eps) / 2, 1 - eps]
    return [round(math.log(1 - x) * SCALE) for x in q], [round(math.log(x) * SCALE) for x in q]


def select(samples, dosage, donors=None):
    """-> (donor names, uint8[records, D]) for a --donors list (None: every sample)"""
    idx = list(range(len(samples))) if donors is None else [samples.index(n) for n in donors]
    return [samples[i] for i in idx], dosage[:, idx]


def likelihoods(table: np.ndarray, n_cols: int, row, col, alt, ref, eps: float):
    """-> (ll int[n_cols][H] as Python ints, counts [n_cols][3]) from the per-(row, col) counts"""
    d = table.shape[1]
    hyp = hypotheses(d)
    lr, la = tables(eps)
    ll = [[0] * len(hyp) for _ in range(n_cols)]
    cnt = [[0, 0, 0] for _ in range(n_cols)]
    for rw, c, a, r in zip(np.asarray(row).tolist(), np.asarray(col).tolist(), np.asarray(alt).tolist(), np.asarray(ref).tolist()):
        a, r = int(a), int(r)
        g = table[rw].tolist()
        if r + a == 0 or any(x == MISSING for x in g):
            continue
        for h, (d1, d2) in enumerate(hyp):
            s = g[d1] + g[d2]
            ll[c][h] += r * lr[s] + a * la[s]
        cnt[c][0] += 1; cnt[c][1] += r; cnt[c][2] += a
    return ll, cnt


def call(ll_c, n_variants: int, d: int) -> dict:
    sing = ll_c[:d]
    best = max(range(d), key=lambda h: (sing[h], -h))
    second = max((h for h in range(d) if h != best), key=lambda h: (sing[h], -h))
    pair = max(range(d, len(ll_c)), key=lambda h: (ll_c[h], -h))
    s_llr, d_llr = sing[best] - sing[second], ll_c[pair] - sing[best]
    kind = "unassigned" if n_variants == 0 else "doublet" if d_llr >= THRESHOLD else "singlet" if s_llr >= THRESHOLD else "unassigned"
    return dict(best=best, second=second, pair=pair, singlet_llr=s_llr, doublet_llr=d_llr, call=kind)


def text(names, barcodes, ll, cnt) -> str:
    d = len(names)
    hyp = hypotheses(d)
    pname = lambda h: f"{names[hyp[h][0]]}+{names[hyp[h][1]]}"
    out = ["\t".join(["barcode", "variants", "ref", "alt", "call", "assignment", "singlet_llr", "doublet_llr", "best_singlet",
                      "second_singlet", "best_doublet"] + [f"ll_{n}" for n in names])]
    for c, bc in enumerate(barcodes):
        k = call(ll[c], cnt[c][0], d)
        assignment = names[k["best"]] if k["call"] == "singlet" else pname(k["pair"]) if k["call"] == "doublet" else "."
        f = [bc.decode() if isinstance(bc, bytes) else bc, *map(str, cnt[c]), k["call"], assignment,
             f"{k['singlet_llr'] / SCALE:.6f}", f"{k['doublet_llr'] / SCALE:.6f}", names[k["best"]], names[k["second"]],
             pname(k["pair"])] + [f"{ll[c][h] / SCALE:.6f}" for h in range(d)]
        out.append("\t".join(f))
    return "\n".join(out) + "\n"


def coverage_counts(vcf, bam, fasta, barcodes, **kw):
    """-> (barcode keys, row, col, alt, ref) of the coverage-mode triplets the C oracle computes"""
    _, _, res, _, bcs = B.run_files(vcf, bam, fasta, barcodes, scoring_method="coverage", n_threads=4, **kw)
    return bcs.keys, res.row, res.col, np.asarray(res.val).astype(np.int64), np.asarray(res.val2).astype(np.int64)


def expected(vcf, bam, fasta, barcodes, donors=None, error_rate=0.01, **kw):
    """-> (file text, ll, counts, names) the CLI's --out-donors should write"""
    samples, dosage = read_genotypes(vcf)
    names, table = select(samples, dosage, donors)
    keys, row, col, alt, ref = coverage_counts(vcf, bam, fasta, barcodes, **kw)
    ll, cnt = likelihoods(table, len(keys), row, col, alt, ref, error_rate)
    return text(names, keys, ll, cnt), ll, cnt, names
