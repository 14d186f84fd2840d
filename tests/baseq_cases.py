"""A small data set for `--min-base-quality`, written with synth_files.BamWriter and explicit base qualities.

Every case sits at its own locus of chrA.  Reads are 100 bases; every base has quality HIGH unless said otherwise.  Each
record carries a hand-written list of the qualities of its judged bases at each locus it reaches (`judged`, keyed by
(QNAME, flag)); None = the record has no qualities.  The floor the cases are built around is Q = 20.
  1000  SNV: the site base at Q-1 / Q / Q+1
  1500  SNV: low bases only away from the site (either side of it)
  2000  SNV: the site base at 0 and at 93
  2500  SNV: a record without qualities (0xFF) with ALT at the site
  3000  MNP (3 bases): the first base aligned, the other two inside a low-quality soft clip (kept); one read whose aligned
        REF base is low
  3500  MNP (3 bases): one low base in the middle of the span
  4000  deletion REF=4 bases, ALT=anchor: a REF read with one low base inside the span; ALT reads (anchor + 3D) with a
        low base right after the deletion (kept) and with a low anchor; a read whose deletion spans the whole REF span
        with low bases on both sides (no judged base: kept)
  5000  insertion REF=1 base, ALT=+3 bases: ALT reads with a low inserted base, with a low anchor, with a low base right
        after the insertion (kept)
  5500  SNV: low inserted bases of an insertion ten bases away and of one anchored right before the site (not judged)
  6000  SNV: a 1-base N skip over the site (useful through the base at end, but nothing judged: kept)
  7000 / 7010  reads that serve both loci, one of them low at 7000 only
  7500  SNV: every read low at the site (an empty row)
  8000  SNV: depth 2 100 (the deep-locus slot kernel), a third of the reads low at the site
  9000  SNV: UB tags and mates -- one UMI of three reads (ALT, ALT, REF) whose REF read is low; mates (ALT, REF) whose REF
        mate is low; other UMIs and mates untouched; one UB outside vtx_pack_umi's alphabet (with --umi, --gpu-stage
        declines the shard and the host stager takes it)
"""
from __future__ import annotations

import os

import numpy as np

Q = 20
HIGH = 38
CELLS = [b"AAACCTGAGAAACCAT-1", b"AAACCTGAGAAACCGC-1", b"AAACCTGAGAAACCTA-1", b"AAACCTGAGAAACGAG-1",
         b"AAACCTGAGAAACGCC-1", b"AAACCTGAGAAAGTGG-1"]
# locus -> (REF length, kind)
LOCI = {1000: (1, "snv"), 1500: (1, "snv"), 2000: (1, "snv"), 2500: (1, "snv"), 3000: (3, "mnp"), 3500: (3, "mnp"),
        4000: (4, "del"), 5000: (1, "ins"), 5500: (1, "snv"), 6000: (1, "snv"), 7000: (1, "snv"), 7010: (1, "snv"),
        7500: (1, "snv"), 8000: (1, "snv"), 9000: (1, "snv")}
INS = b"TTT"
DEEP = 2100


def write_cases(out_dir: str, seed: int = 23) -> dict:
    """-> dict(vcf, bam, fasta, barcodes, judged={(qname, flag): {locus: [judged qualities] or None}})"""
    from vartrix_b200.synth_files import BamWriter
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    L = 10_000
    g = rng.integers(0, 4, size=L, dtype=np.uint8)
    A = b"ACGT"
    gs = bytes(A[x] for x in g)
    alt_base = {p: A[(int(g[p]) + 1) % 4] for p in LOCI}
    recs = []           # (pos, flag, cigar, seq, qual, name, aux)
    judged = {}

    def snv_read(name, locus, allele, start=None, low=(), cb=0, flag=0, aux=b"", also=(), qual=True):
        """100M from `start`: ALT base at `locus` (and at every locus in `also`) when allele == "alt"; `low` = {ref pos: q}"""
        p0 = locus - int(rng.integers(10, 80)) if start is None else start
        seq = bytearray(gs[p0:p0 + 100])
        if allele == "alt":
            for lp in (locus, *also):
                if p0 <= lp < p0 + 100:
                    seq[lp - p0] = alt_base[lp]
        q = bytearray([HIGH] * 100)
        for rp, v in dict(low).items():
            q[rp - p0] = v
        add(p0, flag, [("M", 100)], bytes(seq), bytes(q) if qual else None, name, cb, aux)
        return p0, q

    def add(p0, flag, cigar, seq, qual, name, cb, aux=b""):
        tag = b"CBZ" + CELLS[cb] + b"\0" if cb is not None else b""
        recs.append((p0, flag, cigar, seq, qual, name, tag + aux))

    def note(name, flag, locus, quals):
        judged.setdefault((name, flag), {})[locus] = quals

    # 1000: the site base at Q-1 / Q / Q+1, ALT each
    for k, v in enumerate((Q - 1, Q, Q + 1)):
        snv_read(b"site_q%d" % v, 1000, "alt", low={1000: v}, cb=k)
        note(b"site_q%d" % v, 0, 1000, [v])
    snv_read(b"site_ref", 1000, "ref", cb=0); note(b"site_ref", 0, 1000, [HIGH])
    # 1500: low bases right next to the site and further away
    snv_read(b"near_low", 1500, "alt", low={1499: 2, 1501: 2, 1480: 0}, cb=1); note(b"near_low", 0, 1500, [HIGH])
    # 2000: Q 0 and Q 93
    snv_read(b"q0", 2000, "alt", low={2000: 0}, cb=2); note(b"q0", 0, 2000, [0])
    snv_read(b"q93", 2000, "alt", low={2000: 93}, cb=2); note(b"q93", 0, 2000, [93])
    # 2500: no qualities
    snv_read(b"noqual", 2500, "alt", cb=3, qual=False); note(b"noqual", 0, 2500, None)
    snv_read(b"noqual_ref", 2500, "ref", cb=3); note(b"noqual_ref", 0, 2500, [HIGH])
    # 3000: MNP, its last two REF bases inside a low soft clip
    mnp_alt = {}
    for lp in (3000, 3500):
        mnp_alt[lp] = bytes(A[(int(g[lp + k]) + 1) % 4] for k in range(3))
    p0 = 3000 - 79                                    # 80M aligned [2921, 3001), 20S: the clip holds 3001..
    seq = bytearray(gs[p0:p0 + 100]); seq[79:82] = mnp_alt[3000]
    q = bytearray([HIGH] * 100); q[80:100] = bytes([3] * 20)
    add(p0, 0, [("M", 80), ("S", 20)], bytes(seq), bytes(q), b"mnp_clip", 0); note(b"mnp_clip", 0, 3000, [HIGH])
    seq = bytearray(gs[p0:p0 + 100]); q = bytearray([HIGH] * 100); q[79] = 5; q[80:100] = bytes([HIGH - 1] * 20)
    add(p0, 0, [("M", 80), ("S", 20)], bytes(seq), bytes(q), b"mnp_clip_low", 1); note(b"mnp_clip_low", 0, 3000, [5])
    # 3500: MNP, one low base in the middle
    for name, lowq, allele in ((b"mnp_mid_low", 7, "alt"), (b"mnp_ok", HIGH, "alt"), (b"mnp_ref", HIGH, "ref")):
        p0 = 3500 - int(rng.integers(10, 80))
        seq = bytearray(gs[p0:p0 + 100])
        if allele == "alt":
            seq[3500 - p0:3503 - p0] = mnp_alt[3500]
        q = bytearray([HIGH] * 100); q[3501 - p0] = lowq
        add(p0, 0, [("M", 100)], bytes(seq), bytes(q), name, 2)
        note(name, 0, 3500, [HIGH, lowq, HIGH])
    # 4000: deletion REF = g[4000:4004], ALT = g[4000]
    snv_read(b"del_ref_low", 4000, "ref", low={4002: 4}, cb=0); note(b"del_ref_low", 0, 4000, [HIGH, HIGH, 4, HIGH])
    snv_read(b"del_ref_ok", 4000, "ref", cb=0); note(b"del_ref_ok", 0, 4000, [HIGH] * 4)
    for name, qa, qafter in ((b"del_alt_after_low", HIGH, 1), (b"del_alt_anchor_low", 9, HIGH), (b"del_alt_ok", HIGH, HIGH)):
        p0 = 4000 - 60                                 # 61M (anchor at 4000) 3D 39M
        seq = gs[p0:4001] + gs[4004:4004 + 39]
        q = bytearray([HIGH] * 100); q[60] = qa; q[61] = qafter
        add(p0, 0, [("M", 61), ("D", 3), ("M", 39)], seq, bytes(q), name, 1)
        note(name, 0, 4000, [qa])
    p0 = 4000 - 50                                     # 50M 4D 50M: the deletion is the whole REF span
    q = bytearray([HIGH] * 100); q[49] = 2; q[50] = 2
    add(p0, 0, [("M", 50), ("D", 4), ("M", 50)], gs[p0:4000] + gs[4004:4054], bytes(q), b"del_whole", 1)
    note(b"del_whole", 0, 4000, [])
    # 5000: insertion after the REF base g[5000]
    for name, qa, qins, qafter in ((b"ins_mid_low", HIGH, (HIGH, 6, HIGH), HIGH), (b"ins_anchor_low", 8, (HIGH,) * 3, HIGH),
                                   (b"ins_after_low", HIGH, (HIGH,) * 3, 1), (b"ins_ok", HIGH, (HIGH,) * 3, HIGH)):
        p0 = 5000 - 40                                 # 41M (anchor at 5000) 3I 56M
        seq = gs[p0:5001] + INS + gs[5001:5001 + 56]
        q = bytearray([HIGH] * 100); q[40] = qa; q[41:44] = bytes(qins); q[44] = qafter
        add(p0, 0, [("M", 41), ("I", 3), ("M", 56)], seq, bytes(q), name, 2)
        note(name, 0, 5000, [qa, *qins])
    snv_read(b"ins_ref", 5000, "ref", cb=2); note(b"ins_ref", 0, 5000, [HIGH])
    # 5500: insertions that are not judged
    p0 = 5500 - 30                                     # 41M 3I 56M: the insertion after 5510
    seq = bytearray(gs[p0:p0 + 41] + b"GGG" + gs[p0 + 41:p0 + 97]); seq[30] = alt_base[5500]
    q = bytearray([HIGH] * 100); q[41:44] = bytes([2, 2, 2])
    add(p0, 0, [("M", 41), ("I", 3), ("M", 56)], bytes(seq), bytes(q), b"ins_far", 3); note(b"ins_far", 0, 5500, [HIGH])
    p0 = 5500 - 40                                     # 40M 2I 58M: anchored on 5499, right before the site
    seq = bytearray(gs[p0:5500] + b"CC" + gs[5500:5558]); seq[42] = alt_base[5500]
    q = bytearray([HIGH] * 100); q[40:42] = bytes([1, 1])
    add(p0, 0, [("M", 40), ("I", 2), ("M", 58)], bytes(seq), bytes(q), b"ins_before", 3); note(b"ins_before", 0, 5500, [HIGH])
    # 6000: a 1-base N over the site; the base after it (6001) is low
    p0 = 6000 - 50
    q = bytearray([HIGH] * 100); q[50] = 2
    add(p0, 0, [("M", 50), ("N", 1), ("M", 50)], gs[p0:6000] + gs[6001:6051], bytes(q), b"skip", 4); note(b"skip", 0, 6000, [])
    snv_read(b"skip_alt", 6000, "alt", cb=4); note(b"skip_alt", 0, 6000, [HIGH])
    # 7000 / 7010: reads serving both loci
    for k, (name, low) in enumerate(((b"two_low_first", {7000: 3}), (b"two_ok", {}), (b"two_low_second", {7010: 3}))):
        snv_read(name, 7000, "alt", start=6950 + k, low=low, cb=k, also=(7010,))
        note(name, 0, 7000, [low.get(7000, HIGH)]); note(name, 0, 7010, [low.get(7010, HIGH)])
    # 7500: all reads low at the site
    for k in range(3):
        snv_read(b"empty_%d" % k, 7500, "alt" if k else "ref", low={7500: 10 + k}, cb=k)
        note(b"empty_%d" % k, 0, 7500, [10 + k])
    # 8000: deep
    for k in range(DEEP):
        v = int(rng.integers(2, 20)) if rng.random() < 1 / 3 else int(rng.integers(20, 42))
        name = b"deep_%05d" % k
        snv_read(name, 8000, "alt" if rng.random() < 0.4 else "ref", low={8000: v}, cb=int(rng.integers(0, 5)))
        note(name, 0, 8000, [v])
    # 9000: UMIs and mates
    ub = lambda u: b"UBZ" + u + b"\0"
    for name, allele, umi, v, cb in ((b"u1_a", "alt", b"ACGTACGTAC", HIGH, 0), (b"u1_b", "alt", b"ACGTACGTAC", HIGH, 0),
                                     (b"u1_c", "ref", b"ACGTACGTAC", 4, 0), (b"u2_a", "ref", b"TTGTACGTAC", HIGH, 0),
                                     (b"u3_a", "alt", b"GGGTACGTAC", HIGH, 1), (b"u3_b", "ref", b"GGGTACGTAC", HIGH, 1)):
        snv_read(name, 9000, allele, low={9000: v}, cb=cb, aux=ub(umi)); note(name, 0, 9000, [v])
    # a UB that vtx_pack_umi cannot express: with --umi, --gpu-stage hands this locus's shard back to the host stager
    snv_read(b"u4_exotic", 9000, "alt", cb=1, aux=ub(b"ACGTQQ")); note(b"u4_exotic", 0, 9000, [HIGH])
    for name, (a1, v1), (a2, v2), cb in ((b"mate_low", ("alt", HIGH), ("ref", 3), 2), (b"mate_ok", ("alt", HIGH), ("ref", HIGH), 3),
                                         (b"mate_same", ("alt", HIGH), ("alt", HIGH), 3)):
        snv_read(name, 9000, a1, low={9000: v1}, cb=cb, flag=0x43, aux=ub(b"CCCCAAAAGG"))
        snv_read(name, 9000, a2, low={9000: v2}, cb=cb, flag=0x83, aux=ub(b"CCCCAAAAGG"))
        note(name, 0x43, 9000, [v1]); note(name, 0x83, 9000, [v2])

    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), bam=os.path.join(out_dir, "r.bam"),
                 barcodes=os.path.join(out_dir, "b.tsv"))
    bw = BamWriter(paths["bam"], [("chrA", L)])
    for p0, flag, cig, seq, qual, name, aux in sorted(recs, key=lambda r: r[0]):
        bw.add(0, p0, 60, flag, cig, seq, name, aux, qual=qual)
    bw.close()
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        f.write(b">chrA\n"); off = f.tell()
        for s0 in range(0, L, 60):
            f.write(gs[s0:s0 + 60] + b"\n")
        fai.write(f"chrA\t{L}\t{off}\t60\t61\n")
    with open(paths["vcf"], "w") as f:
        f.write(f"##fileformat=VCFv4.2\n##contig=<ID=chrA,length={L}>\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for p, (n, kind) in LOCI.items():
            ref = gs[p:p + n].decode()
            alt = {"snv": lambda: chr(alt_base[p]), "mnp": lambda: mnp_alt[p].decode(), "del": lambda: ref[0],
                   "ins": lambda: ref + INS.decode()}[kind]()
            f.write(f"chrA\t{p + 1}\t.\t{ref}\t{alt}\t.\t.\t.\n")
    with open(paths["barcodes"], "wb") as f:
        f.write(b"\n".join(CELLS) + b"\n")
    return dict(paths, judged=judged)
