"""A small data set for `--out-variant-stats`: every column of the table nonzero somewhere and every status present, written
with synth_files.BamWriter.

Every case sits at its own locus of chrA; reads are 100 bases at quality HIGH, carry a listed CB and a UB of their own unless
said otherwise.  The runs that use it add `--mapq 30 --primary-alignments --no-duplicates --min-base-quality 20`.
   500  SNV: no read at all (nothing fetched)
  1000  SNV: every read at mapq 10 (lost to --mapq 30)
  1500  SNV: secondary and supplementary records only (lost to --primary-alignments)
  2000  SNV: duplicates only (lost to --no-duplicates)
  2500  SNV: reads whose N skip covers the site: fetched, not useful (useful_alignment)
  3000  SNV: every read's site base at quality 5 (lost to --min-base-quality 20)
  3500  SNV: reads without a CB tag, one with a CB outside the list, one good read
  4000  SNV: reads without a UB tag (lost under --umi), one with
  4500  SNV: a read of random bases (both scores below MIN_SCORE: a None call), REF and ALT reads
  5000  multi-allelic record (ALT "A,C" style)
  5500  SNV whose ALT is "N", outside --valid-chars (invalid_alt)
  6000  REF of two bases with ALT "." (an empty ALT: the REF bases deleted), REF reads
  6500 / 6510  SNVs with reads over both loci
  7000  SNV: ties -- two reads of one cell with a third base at the site (UNKNOWN twice in that cell); one UMI whose four
        reads disagree (2 ALT, 2 REF: UNKNOWN after the collapse); mates (one QNAME, ALT and REF) in another cell
  8000  SNV: 1 025 pairs
  9500  SNV: 2 100 pairs (vtx_k_slots_big)
"""
from __future__ import annotations

import os

import numpy as np

HIGH = 38
CELLS = [b"AAACCTGAGAAACCAT-1", b"AAACCTGAGAAACCGC-1", b"AAACCTGAGAAACCTA-1", b"AAACCTGAGAAACGAG-1",
         b"AAACCTGAGAAACGCC-1", b"AAACCTGAGAAAGTGG-1"]
UNLISTED = b"TTTTTTTTTTTTTTTT-1"
SNVS = (500, 1000, 1500, 2000, 2500, 3000, 3500, 4000, 4500, 5500, 6500, 6510, 7000, 8000, 9500)
L = 12_000


def _umi(k: int) -> bytes:
    return bytes(b"ACGT"[(k >> (2 * i)) & 3] for i in range(10))


def write_cases(out_dir: str, seed: int = 31) -> dict:
    """-> dict(vcf, bam, fasta, barcodes)"""
    from vartrix_b200.synth_files import BamWriter
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    A = b"ACGT"
    g = rng.integers(0, 4, size=L, dtype=np.uint8)
    gs = bytes(A[x] for x in g)
    alt_base = {p: A[(int(g[p]) + 1) % 4] for p in SNVS}
    third_base = {p: A[(int(g[p]) + 2) % 4] for p in SNVS}
    recs = []           # (pos, mapq, flag, cigar, seq, qual, name, aux)
    n_umi = [0]

    def add(p0, cigar, seq, name, cb=0, flag=0, mapq=60, qual=None, ub=True, umi=None):
        aux = b""
        if cb is not None:
            aux += b"CBZ" + (CELLS[cb] if cb >= 0 else UNLISTED) + b"\0"
        if ub:
            if umi is None:
                umi = _umi(n_umi[0]); n_umi[0] += 1
            aux += b"UBZ" + umi + b"\0"
        recs.append((p0, mapq, flag, cigar, seq, bytes(qual) if qual is not None else bytes([HIGH] * len(seq)), name, aux))

    def read(name, locus, allele, start=None, also=(), **kw):
        """100M from `start`: the ALT (or a third) base at `locus` and every locus in `also`"""
        p0 = locus - int(rng.integers(10, 80)) if start is None else start
        seq = bytearray(gs[p0:p0 + 100])
        for lp in (locus, *also):
            if allele in ("alt", "third") and p0 <= lp < p0 + 100:
                seq[lp - p0] = (alt_base if allele == "alt" else third_base)[lp]
        add(p0, [("M", 100)], bytes(seq), name, **kw)

    # 1000 / 1500 / 2000: one record filter takes every read
    for k in range(3):
        read(b"lowmapq_%d" % k, 1000, "alt", cb=k, mapq=10)
    for k, fl in enumerate((0x100, 0x800, 0x100)):
        read(b"nonprim_%d" % k, 1500, "ref", cb=k, flag=fl)
    for k in range(2):
        read(b"dup_%d" % k, 2000, "alt", cb=k, flag=0x400)
    # 2500: an N skip over the site (positions 2495 .. 2514 skipped)
    for k in range(2):
        p0 = 2450
        add(p0, [("M", 45), ("N", 20), ("M", 55)], gs[p0:2495] + gs[2515:2570], b"skip_%d" % k, cb=k)
    # 3000: the site base is low
    for k in range(3):
        p0 = 3000 - int(rng.integers(10, 80))
        q = bytearray([HIGH] * 100); q[3000 - p0] = 5
        seq = bytearray(gs[p0:p0 + 100]); seq[3000 - p0] = alt_base[3000]
        add(p0, [("M", 100)], bytes(seq), b"lowbq_%d" % k, cb=k, qual=q)
    # 3500: no CB, an unlisted CB, one good read
    read(b"nocb_0", 3500, "alt", cb=None)
    read(b"nocb_1", 3500, "ref", cb=None)
    read(b"unlisted", 3500, "alt", cb=-1)
    read(b"cb_ok", 3500, "alt", cb=3)
    # 4000: no UB
    read(b"noub_0", 4000, "alt", cb=1, ub=False)
    read(b"noub_1", 4000, "ref", cb=2, ub=False)
    read(b"ub_ok", 4000, "ref", cb=2)
    # 4500: a read of random bases (None), REF and ALT reads
    p0 = 4450
    add(p0, [("M", 100)], bytes(A[x] for x in rng.integers(0, 4, 100)), b"random", cb=4)
    read(b"r4500_ref", 4500, "ref", cb=4)
    read(b"r4500_alt", 4500, "alt", cb=5)
    # 5000: multi-allelic; 5500: ALT "N" -- reads that would be fetched if the records were scored
    read(b"multi", 5000, "ref", cb=0)
    read(b"invalid", 5500, "ref", cb=0)
    # 6000: REF of two bases, ALT "." -- REF reads
    for k in range(2):
        read(b"emptyalt_%d" % k, 6000, "ref", cb=k)
    # 6500 / 6510: reads over both loci
    for k, allele in enumerate(("alt", "ref", "alt")):
        read(b"two_%d" % k, 6500, allele, start=6450 + k, also=(6510,), cb=k)
    # 7000: ties, a disagreeing UMI, mates
    read(b"tie_0", 7000, "third", cb=0)
    read(b"tie_1", 7000, "third", cb=0)
    for k, allele in enumerate(("alt", "alt", "ref", "ref")):
        read(b"umi_mix_%d" % k, 7000, allele, cb=1, umi=b"GATTACAGAT")
    read(b"mate", 7000, "alt", cb=2, flag=0x43, umi=b"CCCCAAAAGG")
    read(b"mate", 7000, "ref", cb=2, flag=0x83, umi=b"CCCCAAAAGG")
    # 8000 / 9500: deep loci, random cells and alleles (both / REF-only / ALT-only cells)
    for locus, depth in ((8000, 1025), (9500, 2100)):
        for k in range(depth):
            read(b"deep_%d_%05d" % (locus, k), locus, "alt" if rng.random() < 0.3 else "ref", cb=int(rng.integers(0, 6)),
                 umi=_umi(int(rng.integers(0, 400))))

    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), bam=os.path.join(out_dir, "r.bam"),
                 barcodes=os.path.join(out_dir, "b.tsv"))
    bw = BamWriter(paths["bam"], [("chrA", L)])
    for p0, mapq, flag, cig, seq, qual, name, aux in sorted(recs, key=lambda r: r[0]):
        bw.add(0, p0, mapq, flag, cig, seq, name, aux, qual=qual)
    bw.close()
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        f.write(b">chrA\n"); off = f.tell()
        for s0 in range(0, L, 60):
            f.write(gs[s0:s0 + 60] + b"\n")
        fai.write(f"chrA\t{L}\t{off}\t60\t61\n")
    rows = [(p, gs[p:p + 1].decode(), chr(alt_base[p])) for p in SNVS if p != 5500]
    rows += [(5000, gs[5000:5001].decode(), ",".join(chr(A[(int(g[5000]) + d) % 4]) for d in (1, 2))),
             (5500, gs[5500:5501].decode(), "N"), (6000, gs[6000:6002].decode(), ".")]
    with open(paths["vcf"], "w") as f:
        f.write(f"##fileformat=VCFv4.2\n##contig=<ID=chrA,length={L}>\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for p, ref, alt in sorted(rows):
            f.write(f"chrA\t{p + 1}\t.\t{ref}\t{alt}\t.\t.\t.\n")
    with open(paths["barcodes"], "wb") as f:
        f.write(b"\n".join(CELLS) + b"\n")
    return paths
