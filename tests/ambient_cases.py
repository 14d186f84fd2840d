"""Seeded pooled data sets with ambient RNA for `--ambient-rna`, written with synth_files.BamWriter, and their truth.

Six donors (D0 .. D5), NL SNV loci 100 bases apart on chrA with Hardy-Weinberg genotypes (ALT frequency 0.1 .. 0.9), written
into the VCF as GT columns.  The cells:
  singlets   cells of one donor, 5 .. 300 molecules
  doublets   cells whose molecules come from two donors, 50/50, 50 .. 300 molecules
  empty      barcodes that are listed but have no read
Each molecule picks its locus, then its source: with probability rho it is ambient and takes a donor of a randomly drawn cell
of the pool, else a donor of its own cell.  It shows that donor's allele (ALT with probability g / 2), then one molecule in a
hundred is flipped.  As in donor_cases.py, every molecule carries a UB and is read 1 to 3 times, one in five is a mate pair
(one QNAME, two records over the site), and a few reads are at mapq 10, duplicates, secondary, or have the site base at
quality 5, so the record filters change the counts.
"""
from __future__ import annotations

import json
import os

import numpy as np

from donor_cases import HIGH, _barcode, _umi

SPACING = 100
NL = 600
N_DONORS = 6
SINGLET_DEPTHS = [5, 10, 20, 50, 100, 200, 300]
DOUBLET_DEPTHS = [50, 100, 200, 300]
N_SINGLET, N_DOUBLET, N_EMPTY = 300, 20, 4
RHOS = (0.0, 0.05, 0.15, 0.3)


def write_pool(out_dir: str, rho: float, seed: int = 4242) -> dict:
    """-> dict(vcf, bam, fasta, barcodes, truth, donors)"""
    from vartrix_b200.synth_files import BamWriter
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    A = b"ACGT"
    length = NL * SPACING + 300
    gen = rng.integers(0, 4, size=length, dtype=np.uint8)
    gs = bytes(A[x] for x in gen)
    pos = [150 + SPACING * i for i in range(NL)]
    alt = {p: A[(int(gen[p]) + 1) % 4] for p in pos}
    freq = rng.uniform(0.1, 0.9, NL)
    geno = np.stack([rng.binomial(2, freq) for _ in range(N_DONORS)], axis=1)        # [locus][donor]
    donors = [f"D{d}" for d in range(N_DONORS)]

    cells = []
    for k in range(N_SINGLET):
        cells.append(dict(kind="singlet", donors=[k % N_DONORS], depth=SINGLET_DEPTHS[(k // N_DONORS) % len(SINGLET_DEPTHS)]))
    for k in range(N_DOUBLET):
        a, b = sorted(rng.choice(N_DONORS, 2, replace=False).tolist())
        cells.append(dict(kind="doublet", donors=[a, b], depth=DOUBLET_DEPTHS[k % len(DOUBLET_DEPTHS)]))
    for k in range(N_EMPTY):
        cells.append(dict(kind="empty", donors=[], depth=0))
    seen = set()
    for c in cells:
        while True:
            bc = _barcode(rng)
            if bc not in seen:
                seen.add(bc); c["barcode"] = bc.decode(); break
    cells = [cells[i] for i in rng.permutation(len(cells))]
    pool = [c for c in cells if c["depth"]]

    recs = []
    n_name = [0]

    def add_read(li, is_alt, bc, umi, flag=0, name=None):
        p = pos[li]
        p0 = p - int(rng.integers(10, 60))
        seq = bytearray(gs[p0:p0 + 70])
        if is_alt:
            seq[p - p0] = alt[p]
        q = bytearray([HIGH] * 70)
        mapq, u = 60, rng.random()
        if u < 0.02: mapq = 10
        elif u < 0.03: flag |= 0x400
        elif u < 0.04: flag |= 0x100
        elif u < 0.05: q[p - p0] = 5
        if name is None:
            name = b"r%07d" % n_name[0]; n_name[0] += 1
        recs.append((p0, mapq, flag, bytes(seq), bytes(q), name, b"CBZ" + bc + b"\0" + b"UBZ" + umi + b"\0"))

    for c in cells:
        bc = c["barcode"].encode()
        for _ in range(c["depth"]):
            li = int(rng.integers(0, NL))
            src = pool[int(rng.integers(0, len(pool)))] if rng.random() < rho else c
            d = src["donors"][int(rng.integers(0, len(src["donors"])))]
            is_alt = rng.random() < geno[li, d] / 2
            if rng.random() < 0.01:
                is_alt = not is_alt
            umi = _umi(rng)
            if rng.random() < 0.2:
                name = b"m%07d" % n_name[0]; n_name[0] += 1
                add_read(li, is_alt, bc, umi, flag=0x43, name=name)
                add_read(li, is_alt, bc, umi, flag=0x83, name=name)
            else:
                for _ in range(int(rng.integers(1, 4))):
                    add_read(li, is_alt, bc, umi)

    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), bam=os.path.join(out_dir, "r.bam"),
                 barcodes=os.path.join(out_dir, "b.tsv"), truth=os.path.join(out_dir, "truth.json"))
    bw = BamWriter(paths["bam"], [("chrA", length)])
    for p0, mapq, flag, seq, qual, nm, aux in sorted(recs, key=lambda r: r[0]):
        bw.add(0, p0, mapq, flag, [("M", 70)], seq, nm, aux, qual=qual)
    bw.close()
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        f.write(b">chrA\n"); off = f.tell()
        for s0 in range(0, length, 60):
            f.write(gs[s0:s0 + 60] + b"\n")
        fai.write(f"chrA\t{length}\t{off}\t60\t61\n")
    with open(paths["vcf"], "w") as f:
        f.write(f"##fileformat=VCFv4.2\n##contig=<ID=chrA,length={length}>\n"
                '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">\n'
                "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(donors) + "\n")
        for i, p in enumerate(pos):
            gts = [("0/0", "0/1", "1/1")[int(g)] for g in geno[i]]
            f.write(f"chrA\t{p + 1}\t.\t{chr(gs[p])}\t{chr(alt[p])}\t.\tPASS\t.\tGT\t" + "\t".join(gts) + "\n")
    with open(paths["barcodes"], "w") as f:
        f.write("".join(c["barcode"] + "\n" for c in cells))
    with open(paths["truth"], "w") as f:
        json.dump({c["barcode"]: dict(kind=c["kind"], donors=[donors[d] for d in c["donors"]], molecules=c["depth"]) for c in cells}, f)
    paths["donors"] = donors
    return paths
