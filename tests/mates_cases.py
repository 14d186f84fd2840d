"""A small paired-end data set for `--collapse-mates`, written with synth_files.BamWriter.

Every case the flag has to get right sits at its own locus of chrA (SNVs; reads are 100M unless said otherwise):
  1000  concordant overlapping mates (ALT/ALT, REF/REF), discordant mates (ALT/REF -> UNKNOWN), unpaired reads; names that
        are prefixes of each other (r1 / r10 / r100), equal-length names that differ in the last byte, 254-byte names
  2000  a mate removed by --mapq 10, one removed by --no-duplicates, one that does not intersect the variant (50M 30N 50M);
        a supplementary and a secondary record of a template whose mates are there too
  3000 / 3010  templates whose reads serve both loci
  4000  mates with different CB tags, several "*" records in one cell, a template with a mate on chrB, reads without CB or
        with an unlisted one
  6000  a depth-3 000 locus (1 500 pairs in 5 cells, mostly concordant): the deep-locus slot kernel
"""
from __future__ import annotations

import os

import numpy as np

CELLS = [b"AAACCTGAGAAACCAT-1", b"AAACCTGAGAAACCGC-1", b"AAACCTGAGAAACCTA-1", b"AAACCTGAGAAACGAG-1",
         b"AAACCTGAGAAACGCC-1", b"AAACCTGAGAAAGTGG-1"]
UNLISTED = b"TTTTTTTTTTTTTTTT-1"
LOCI = [1000, 2000, 3000, 3010, 4000, 6000]
LONG = b"N" * 253


def write_paired(out_dir: str, seed: int = 17) -> dict:
    from vartrix_b200.synth_files import BamWriter
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    contigs = [("chrA", 9000), ("chrB", 3000)]
    genome = [rng.integers(0, 4, size=L, dtype=np.uint8) for _, L in contigs]
    acgt = np.frombuffer(b"ACGT", np.uint8)
    alt_of = {p: (int(genome[0][p]) + 1) % 4 for p in LOCI}
    recs = []           # (contig, pos, mapq, flag, cigar, seq, name, cb)

    def read(name, locus, allele, cb=0, flag=0x41, mapq=60, start=None, ci=0, cigar=None, also=()):
        """a 100-base read over `locus` carrying `allele` ("alt" / "ref") there and at every locus in `also`"""
        p0 = locus - int(rng.integers(5, 60)) if start is None else start
        g = genome[ci]
        if cigar is None:
            seq = g[p0:p0 + 100].copy()
        else:                                                  # M N M: the bases of both M blocks
            m1, n, m2 = cigar[0][1], cigar[1][1], cigar[2][1]
            seq = np.concatenate([g[p0:p0 + m1], g[p0 + m1 + n:p0 + m1 + n + m2]])
        if ci == 0:
            for lp in (locus, *also):
                if allele == "alt" and cigar is None and p0 <= lp < p0 + 100:
                    seq[lp - p0] = alt_of[lp]
        tag = None if cb is None else (UNLISTED if cb == -1 else CELLS[cb])
        recs.append((ci, p0, mapq, flag, cigar or [("M", 100)], acgt[seq].tobytes(), name, tag))

    def pair(name, locus, a1, a2, cb=0, cb2=None, **kw):
        read(name, locus, a1, cb, flag=0x43, **kw)
        read(name, locus, a2, cb if cb2 is None else cb2, flag=0x83, **kw)

    # 1000
    for k, (a1, a2) in enumerate([("alt", "alt"), ("ref", "ref"), ("alt", "ref"), ("ref", "alt"), ("alt", "alt"), ("ref", "ref")]):
        pair(b"frag_%04d" % k, 1000, a1, a2, cb=k % 3)
    pair(b"r1", 1000, "alt", "alt", cb=0); pair(b"r10", 1000, "alt", "ref", cb=0); pair(b"r100", 1000, "ref", "ref", cb=0)
    pair(b"tmplA1", 1000, "alt", "alt", cb=1); pair(b"tmplA2", 1000, "alt", "alt", cb=1); pair(b"tmplA3", 1000, "ref", "alt", cb=1)
    pair(LONG + b"a", 1000, "alt", "alt", cb=2); pair(LONG + b"b", 1000, "ref", "ref", cb=2); pair(LONG + b"c", 1000, "alt", "ref", cb=2)
    for k in range(5):
        read(b"single_%d" % k, 1000, "alt" if k % 2 else "ref", cb=k % 3, flag=0)
    # 2000: a mate the filters remove, supplementary / secondary records of one template
    pair(b"lowq", 2000, "alt", "ref", cb=0)
    recs[-1] = recs[-1][:2] + (3,) + recs[-1][3:]                                        # mate 2 at mapq 3
    pair(b"dup", 2000, "alt", "ref", cb=0)
    recs[-1] = recs[-1][:3] + (recs[-1][3] | 0x400,) + recs[-1][4:]                      # mate 2 a duplicate
    read(b"notuse", 2000, "alt", cb=1, flag=0x43)
    read(b"notuse", 2000, "ref", cb=1, flag=0x83, start=2000 - 60, cigar=[("M", 50), ("N", 30), ("M", 50)])
    pair(b"suppl", 2000, "alt", "alt", cb=2)
    read(b"suppl", 2000, "ref", cb=2, flag=0x843)
    pair(b"second", 2000, "ref", "ref", cb=2)
    read(b"second", 2000, "alt", cb=2, flag=0x143)
    for k in range(4):
        pair(b"plain2_%d" % k, 2000, "alt" if k < 2 else "ref", "alt" if k < 2 else "ref", cb=k % 3)
    # 3000 / 3010: reads that serve two loci
    for k in range(6):
        a = "alt" if k % 3 else "ref"
        pair(b"both_%d" % k, 3000, a, a if k != 4 else "ref", cb=k % 2, also=(3010,), start=3000 - int(rng.integers(10, 80)))
    pair(b"only3010", 3010, "alt", "alt", cb=0)
    # 4000: mates in different cells, "*" names, a mate on chrB, no CB / unlisted CB
    pair(b"twocells", 4000, "alt", "alt", cb=0, cb2=1)
    pair(b"twocells2", 4000, "ref", "alt", cb=2, cb2=3)
    for k, a in enumerate(["alt", "alt", "ref", "alt"]):
        read(b"*", 4000, a, cb=0, flag=0)
    read(b"*", 4000, "alt", cb=1, flag=0)
    read(b"farmate", 4000, "alt", cb=1, flag=0x41)
    read(b"farmate", 0, "ref", cb=1, flag=0x81, ci=1, start=500)
    pair(b"nocb", 4000, "alt", "alt", cb=None)
    pair(b"unlisted", 4000, "alt", "ref", cb=-1)
    pair(b"cb3", 4000, "alt", "alt", cb=3)
    # 6000: depth 3 000
    for k in range(1500):
        a1 = "alt" if rng.random() < 0.4 else "ref"
        a2 = a1 if rng.random() < 0.85 else ("ref" if a1 == "alt" else "alt")
        pair(b"deep_%05d" % k, 6000, a1, a2, cb=int(rng.integers(0, 5)))

    order = sorted(range(len(recs)), key=lambda i: (recs[i][0], recs[i][1]))
    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), bam=os.path.join(out_dir, "r.bam"),
                 barcodes=os.path.join(out_dir, "b.tsv"))
    bw = BamWriter(paths["bam"], contigs)
    for i in order:
        ci, p0, mapq, flag, cig, seq, name, cb = recs[i]
        bw.add(ci, p0, mapq, flag, cig, seq, name, b"" if cb is None else b"CBZ" + cb + b"\0")
    bw.close()
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        for (name, L), g in zip(contigs, genome):
            f.write(f">{name}\n".encode()); off = f.tell()
            seq = acgt[g]
            for s0 in range(0, L, 60):
                f.write(seq[s0:s0 + 60].tobytes() + b"\n")
            fai.write(f"{name}\t{L}\t{off}\t60\t61\n")
    with open(paths["vcf"], "w") as f:
        f.write("##fileformat=VCFv4.2\n" + "".join(f"##contig=<ID={n},length={L}>\n" for n, L in contigs))
        f.write("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for p in LOCI:
            f.write(f"chrA\t{p + 1}\t.\t{'ACGT'[genome[0][p]]}\t{'ACGT'[alt_of[p]]}\t.\t.\t.\n")
    with open(paths["barcodes"], "wb") as f:
        f.write(b"\n".join(CELLS) + b"\n")
    return paths
