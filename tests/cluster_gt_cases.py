"""Seeded pools for `--out-cluster-genotypes` / `--out-cluster-matches`: ambient_cases' pools (six donors, ambient RNA at rate
rho) with the VCF rewritten for matching.

The rewritten VCF gives every record an ID (rs1, rs2, ...) and adds two sample columns that are not in the pool:
  decoy_hwe    Hardy-Weinberg genotypes at a random ALT frequency per locus
  decoy_half   D0's genotype at half the loci, Hardy-Weinberg draws at the others
A second VCF has the same records and columns without D5.  The records are the pool's, so the BAM's counts are unchanged."""
from __future__ import annotations

import os

import numpy as np

from ambient_cases import RHOS, write_pool as write_ambient_pool  # noqa: F401  (RHOS: the pools' ambient fractions)

DECOYS = ("decoy_hwe", "decoy_half")


def _rewrite(src: str, dst: str, rng, drop=()):
    head, body = [], []
    for ln in open(src):
        (head if ln.startswith("#") else body).append(ln.rstrip("\n"))
    n = len(body)
    freq = rng.uniform(0.1, 0.9, n)
    hwe = rng.binomial(2, freq)
    half = rng.random(n) < 0.5
    other = rng.binomial(2, freq)
    gt = ("0/0", "0/1", "1/1")
    cols = head[-1].split("\t")
    keep = [i for i, c in enumerate(cols) if c not in drop]
    with open(dst, "w") as f:
        f.write("\n".join(head[:-1]) + "\n")
        f.write("\t".join([cols[i] for i in keep] + list(DECOYS)) + "\n")
        for i, ln in enumerate(body):
            x = ln.split("\t")
            x[2] = f"rs{i + 1}"
            d0 = x[9]
            extra = [gt[hwe[i]], d0 if half[i] else gt[other[i]]]
            f.write("\t".join([x[j] for j in keep] + extra) + "\n")


def write_pool(out_dir: str, rho: float) -> dict:
    """-> ambient_cases' dict plus vcf_match (IDs and decoys) and vcf_no_d5 (the same without D5)"""
    p = write_ambient_pool(out_dir, rho)
    p["vcf_match"] = os.path.join(out_dir, "v_match.vcf")
    p["vcf_no_d5"] = os.path.join(out_dir, "v_no_d5.vcf")
    _rewrite(p["vcf"], p["vcf_match"], np.random.default_rng(99))
    _rewrite(p["vcf"], p["vcf_no_d5"], np.random.default_rng(99), drop=("D5",))
    return p
