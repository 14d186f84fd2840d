"""A seeded pooled data set for `--out-donors`, written with synth_files.BamWriter, and its truth.

Six donors (D0 .. D5) and a seventh VCF sample (X) that is not one of the pool's donors; the header lists them as
D0 D1 D2 X D3 D4 D5.  NL SNV loci, 200 bases apart on chrA, with Hardy-Weinberg genotypes (ALT frequency 0.2 .. 0.8).
The cells:
  singlets   ~100 cells of one donor each
  doublets   ~15 cells whose molecules come from two donors, 50/50
  empty      barcodes that are listed but have no read
Every molecule carries a UB and is read 1 to 3 times (a multi-read UMI); one molecule in five is a mate pair (one QNAME,
two records over the site).  A molecule shows its donor's allele: ALT with probability g / 2, then one base in a hundred is
flipped.  A few reads are at mapq 10, duplicates, secondary, or have the site base at quality 5, so the record filters and the
base-quality floor of the runs that use them change the counts.
Cell depth spans 2 .. 300 molecules (doublets 16 .. 400), so the thin cells are the unassigned ones.

The first rows are the VCF's edge rows (each also has reads):
  row 0  D1 is ./.                      -> not usable
  row 1  D4 is a bare .                 -> not usable
  row 2  D2 is phased 1|0               -> dosage 1
  row 3  D0 is haploid 1, D5 haploid 0  -> dosage 2 and 0
  row 4  FORMAT DP:GT                   -> usable
  row 5  FORMAT DP (no GT)              -> not usable
  row 6  FORMAT DP:GT, D3's column "7"  -> not usable (too short to hold GT)
  row 7  multi-allelic A,C with D2 1/2  -> never scored
  row 8  every donor 0/1                -> usable, the same for every hypothesis
  row 9  X is ./. (X is not a donor)    -> usable with --donors
"""
from __future__ import annotations

import json
import os

import numpy as np

NAMES = ["D0", "D1", "D2", "X", "D3", "D4", "D5"]
DONORS = ["D0", "D1", "D2", "D3", "D4", "D5"]
NL = 300
SPACING = 200
L = NL * SPACING + 400
N_SINGLET, N_DOUBLET, N_EMPTY = 100, 15, 8
HIGH = 38


def _barcode(rng) -> bytes:
    return bytes(b"ACGT"[x] for x in rng.integers(0, 4, 16)) + b"-1"


def _umi(rng) -> bytes:
    return bytes(b"ACGT"[x] for x in rng.integers(0, 4, 10))


def _gt(g: int, rng) -> str:
    return ["0/0", "0/1" if rng.random() < 0.5 else "1/0", "1/1"][g]


def write_cases(out_dir: str, seed: int = 2024) -> dict:
    """-> dict(vcf, bam, fasta, barcodes, truth)"""
    from vartrix_b200.synth_files import BamWriter
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    A = b"ACGT"
    gen = rng.integers(0, 4, size=L, dtype=np.uint8)
    gs = bytes(A[x] for x in gen)
    pos = [200 + SPACING * i for i in range(NL)]
    alt = {p: A[(int(gen[p]) + 1) % 4] for p in pos}
    # genotypes of the seven samples (Hardy-Weinberg at a per-locus ALT frequency)
    freq = rng.uniform(0.2, 0.8, NL)
    geno = np.stack([rng.binomial(2, freq) for _ in NAMES], axis=1)       # [locus][sample]
    geno[8, :] = 1
    # what the reads see: the dosage the molecule's donor has (edge rows use the genotype written below)
    truth_g = geno.copy()
    truth_g[3, NAMES.index("D0")] = 2; truth_g[3, NAMES.index("D5")] = 0
    truth_g[2, NAMES.index("D2")] = 1

    # cells
    cells = []
    for k in range(N_SINGLET):
        cells.append(dict(kind="singlet", donors=[DONORS[k % 6]]))
    for k in range(N_DOUBLET):
        a, b = sorted(rng.choice(6, 2, replace=False).tolist())
        cells.append(dict(kind="doublet", donors=[DONORS[a], DONORS[b]]))
    for k in range(N_EMPTY):
        cells.append(dict(kind="empty", donors=[]))
    seen = set()
    for c in cells:
        while True:
            bc = _barcode(rng)
            if bc not in seen:
                seen.add(bc); c["barcode"] = bc.decode(); break
    order = rng.permutation(len(cells))
    cells = [cells[i] for i in order]

    recs = []           # (pos, mapq, flag, cigar, seq, qual, name, aux)
    n_name = [0]

    def add_read(locus_i, allele_alt, bc, umi, flag=0, name=None):
        p = pos[locus_i]
        p0 = p - int(rng.integers(10, 90))
        seq = bytearray(gs[p0:p0 + 100])
        if allele_alt:
            seq[p - p0] = alt[p]
        q = bytearray([HIGH] * 100)
        mapq, u = 60, rng.random()
        if u < 0.03: mapq = 10
        elif u < 0.05: flag |= 0x400
        elif u < 0.06: flag |= 0x100
        elif u < 0.08: q[p - p0] = 5
        if name is None:
            name = b"r%07d" % n_name[0]; n_name[0] += 1
        recs.append((p0, mapq, flag, [("M", 100)], bytes(seq), bytes(q), name, b"CBZ" + bc + b"\0" + b"UBZ" + umi + b"\0"))

    for c in cells:
        if c["kind"] == "empty":
            continue
        bc = c["barcode"].encode()
        depth = int(rng.choice([2, 4, 8, 16, 40, 100, 200, 300] if c["kind"] == "singlet" else [16, 100, 200, 300, 400]))
        for _ in range(depth):
            li = int(rng.integers(0, NL))
            donor = c["donors"][int(rng.integers(0, len(c["donors"])))]
            g = int(truth_g[li, NAMES.index(donor)])
            is_alt = rng.random() < g / 2
            if rng.random() < 0.01:
                is_alt = not is_alt
            umi = _umi(rng)
            if rng.random() < 0.2:          # a mate pair: one QNAME, two records over the site
                name = b"m%07d" % n_name[0]; n_name[0] += 1
                add_read(li, is_alt, bc, umi, flag=0x43, name=name)
                add_read(li, is_alt, bc, umi, flag=0x83, name=name)
            else:
                for _ in range(int(rng.integers(1, 4))):
                    add_read(li, is_alt, bc, umi)

    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), bam=os.path.join(out_dir, "r.bam"),
                 barcodes=os.path.join(out_dir, "b.tsv"), truth=os.path.join(out_dir, "truth.json"))
    bw = BamWriter(paths["bam"], [("chrA", L)])
    for p0, mapq, flag, cig, seq, qual, name, aux in sorted(recs, key=lambda r: r[0]):
        bw.add(0, p0, mapq, flag, cig, seq, name, aux, qual=qual)
    bw.close()
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        f.write(b">chrA\n"); off = f.tell()
        for s0 in range(0, L, 60):
            f.write(gs[s0:s0 + 60] + b"\n")
        fai.write(f"chrA\t{L}\t{off}\t60\t61\n")

    with open(paths["vcf"], "w") as f:
        f.write(f"##fileformat=VCFv4.2\n##contig=<ID=chrA,length={L}>\n"
                '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">\n'
                '##FORMAT=<ID=DP,Number=1,Type=Integer,Description="Depth">\n'
                "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(NAMES) + "\n")
        for i, p in enumerate(pos):
            ref_b, alt_s = chr(gs[p]), chr(alt[p])
            gts = [_gt(int(geno[i, s]), rng) for s in range(len(NAMES))]
            fmt, cols = "GT:DP", None
            if i == 0: gts[NAMES.index("D1")] = "./."
            if i == 1: gts[NAMES.index("D4")] = "."
            if i == 2: gts[NAMES.index("D2")] = "1|0"
            if i == 3: gts[NAMES.index("D0")] = "1"; gts[NAMES.index("D5")] = "0"
            if i == 4:
                fmt, cols = "DP:GT", [f"{int(rng.integers(5, 40))}:{g}" for g in gts]
            if i == 5:
                fmt, cols = "DP", [str(int(rng.integers(5, 40))) for _ in gts]
            if i == 6:
                fmt, cols = "DP:GT", [f"{int(rng.integers(5, 40))}:{g}" for g in gts]
                cols[NAMES.index("D3")] = "7"
            if i == 7:
                alt_s = alt_s + "," + chr(A[(int(gen[p]) + 2) % 4])
                gts[NAMES.index("D2")] = "1/2"
            if i == 9: gts[NAMES.index("X")] = "./."
            if cols is None:
                cols = [f"{g}:{int(rng.integers(5, 40))}" for g in gts]
            f.write(f"chrA\t{p + 1}\t.\t{ref_b}\t{alt_s}\t.\tPASS\t.\t{fmt}\t" + "\t".join(cols) + "\n")
    with open(paths["barcodes"], "w") as f:
        f.write("".join(c["barcode"] + "\n" for c in cells))
    with open(paths["truth"], "w") as f:
        json.dump({c["barcode"]: dict(kind=c["kind"], donors=c["donors"]) for c in cells}, f)
    return paths
