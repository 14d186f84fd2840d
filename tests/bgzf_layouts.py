"""One BAM record stream, many BGZF layouts (test support).

`synth_files.BamWriter` -- like htslib -- flushes a BGZF member before a record that would not fit, so every record of every
test BAM lies inside one member.  Writers built on htsjdk fill members to a fixed size and cut records wherever that lands.
This module writes the same uncompressed BAM byte stream cut into members by a layout policy, and the BAI that goes with
that layout's virtual offsets (bins, chunks merged like `BamWriter._close_pending`, linear index filled like `BamWriter.close`):

  whole       members as BamWriter cuts them: byte-identical to BamWriter, the control
  fill        every member 65 280 output bytes, records cut wherever that lands
  cut_at      members cut inside records at chosen fields: block_size, the fixed part, QNAME, CIGAR, SEQ, QUAL, CB and UB values
  tiny        members of 1..40 output bytes: one record spans dozens of members
  empty       members with ISIZE 0 between data members; offsets on such a boundary name the empty member
  isize_voff  every index offset on a member boundary written as (k, ISIZE_k) instead of (k + 1, 0), and each bin's chunks
              listed last to first (the specification does not order them; htslib sorts them when it reads)
  codecs      members compressed at zlib levels 0 / 1 / 9, with Z_RLE, Z_HUFFMAN_ONLY, Z_FIXED, and by tests/deflate_craft.py
              (many small blocks, stored blocks of odd lengths)

`dataset()` writes the FASTA, VCF, barcodes and record list these layouts are filled with.
"""
from __future__ import annotations

import bisect
import os
import random
import struct
import zlib

import numpy as np

from vartrix_b200.synth_files import BamWriter, reg2bin

LAYOUTS = ("whole", "fill", "cut_at", "tiny", "empty", "isize_voff", "codecs")
CUT_FIELDS = ("block_size", "fixed", "qname", "cigar", "seq", "qual", "cb", "ub")
EOF_MEMBER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


class _RecordEncoder(BamWriter):
    """BamWriter.add's record encoding without a file: encode() returns the record bytes (block_size included)"""

    def __init__(self):
        self.block = bytearray()
        self._pending = None

    def _flush(self):
        pass

    def _voff(self):
        return 0

    def _close_pending(self, v_end):
        pass

    def encode(self, *a, **kw) -> bytes:
        self.block = bytearray(); self._pending = None
        self.add(*a, **kw)
        return bytes(self.block)


def header_bytes(refs) -> bytes:
    text = "@HD\tVN:1.6\tSO:coordinate\n" + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in refs)
    hdr = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, l in refs:
        hdr += struct.pack("<i", len(n) + 1) + n.encode() + b"\x00" + struct.pack("<i", l)
    return hdr


def field_offsets(rec: bytes) -> dict:
    """byte offset (inside the record, block_size included) of a point inside each field a cut_at layout splits"""
    l_name, n_cig = rec[12], struct.unpack_from("<H", rec, 16)[0]
    l_seq = struct.unpack_from("<i", rec, 20)[0]
    q = 36 + l_name; s = q + 4 * n_cig; ql = s + (l_seq + 1) // 2; aux = ql + l_seq
    out = dict(block_size=2, fixed=4 + 13, qname=36 + l_name // 2)
    if n_cig:
        out["cigar"] = q + 2 * n_cig - 1
    if l_seq > 1:
        out["seq"] = s + (l_seq + 1) // 4; out["qual"] = ql + l_seq // 2
    for tag in (b"CBZ", b"UBZ"):
        k = rec.find(tag, aux)
        if k >= 0 and rec.find(b"\0", k) - k > 5:
            out[tag[:2].decode().lower()] = k + 5
    return out


def _craft_payload(raw: bytes, rng):
    """raw bytes as a crafted DEFLATE stream: small fixed / dynamic blocks and stored blocks of odd lengths.  The dynamic
    blocks give every one of the 286 literal/length and 30 distance symbols a code, weighted so that unused and rare symbols
    get 15-bit codes (deep second-level tables; rare bytes of the block decode through them).
    -> (stream, number of symbols written with a 15-bit code)"""
    from deflate_craft import build, limited_lengths, lit
    blocks, p, n_long = [], 0, 0
    dist_lens = limited_lengths([1 << (29 - k) for k in range(30)], 15)          # 1, 2, ..., 15, 15, ... bits
    while p < len(raw):
        n = rng.choice([1, 3, 7, 31, 255, 999])
        kind = rng.choice(["stored", "fixed", "dynamic"])
        chunk = raw[p:p + n]
        if kind == "dynamic":
            freq = [1] * 286                     # every symbol gets a code; the block's last byte stays as rare as the unused ones
            for b in chunk[:-1]:
                freq[b] += 1 << 12
            lit_lens = limited_lengths(freq, 15)
            n_long += sum(1 for b in chunk if lit_lens[b] == 15)
            blocks.append((kind, lit(chunk), dict(lit_lens=lit_lens, dist_lens=dist_lens)))
        else:
            blocks.append(("stored", chunk) if kind == "stored" else (kind, lit(chunk)))
        p += n
    if not blocks:
        blocks = [("fixed", [])]
    s, out = build(blocks)
    assert out == raw
    return s, n_long


def _member(raw: bytes, codec):
    """-> (BGZF member, symbols written with a 15-bit code)"""
    n_long = 0
    if codec == "craft":
        comp, n_long = _craft_payload(raw, random.Random(len(raw)))
    else:
        level, strategy = codec
        co = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
        comp = co.compress(raw) + co.flush()
    assert len(comp) + 26 <= 65536
    return struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, len(comp) + 25) + comp + \
        struct.pack("<II", zlib.crc32(raw) & 0xFFFFFFFF, len(raw)), n_long


def _cuts(layout, hdr_len, recs, rec_start, total, rng):
    """member boundaries (stream offsets, ascending, 0 and total included; a repeated offset is an empty member) and the
    (record, field) pairs a cut lands in"""
    if layout == "whole":                                    # BamWriter: header alone, then flush before a record that does not fit
        cuts, cur = [0, hdr_len], hdr_len
        for r, s in zip(recs, rec_start):
            if s - cur + len(r) > 0xFF00 and s > cur:
                cuts.append(s); cur = s
        return cuts + [total], []
    if layout == "fill":
        return list(range(0, total, 0xFF00)) + [total], []
    if layout == "tiny":
        cuts, p = [0], 0
        while p < total:
            p = min(total, p + rng.randrange(1, 41)); cuts.append(p)
        return cuts, []
    split = []
    if layout == "cut_at":                                   # cycle through the fields, one record in three
        cuts, k = {0, total}, 0
        for i in range(0, len(recs), 3):
            fo = field_offsets(recs[i])
            f = CUT_FIELDS[k % len(CUT_FIELDS)]
            k += 1
            if f in fo:
                cuts.add(rec_start[i] + fo[f]); split.append((i, f))
        cuts = sorted(cuts)
        out = [cuts[0]]
        for c in cuts[1:]:                                   # members stay <= 0xFF00 output bytes
            while c - out[-1] > 0xFF00:
                out.append(out[-1] + 0xFF00)
            out.append(c)
        return out, split
    cuts, p = [0], 0
    while p < total:
        p = min(total, p + rng.randrange(1, 20000)); cuts.append(p)
    if layout == "empty":                                    # empty members: at boundaries, at record starts, one or two in a row
        extra = [c for c in cuts[1:-1] if rng.random() < 0.3] + [x for x in rec_start if rng.random() < 0.02]
        for x in extra:
            cuts += [x] * rng.choice([1, 1, 2])
        cuts = sorted(cuts)
    if layout == "isize_voff":                               # members that end right before a record: its offset is (k, ISIZE_k)
        cuts = sorted(set(cuts) | {x for x in rec_start if rng.random() < 0.1})
    return cuts, split


def write_layout(path: str, refs, recs, layout: str, seed: int = 1) -> dict:
    """recs: [(refid, pos, end, record bytes)] in file order -> writes path and path.bai; returns facts about the layout"""
    rng = random.Random(seed)
    hdr = header_bytes(refs)
    stream = bytearray(hdr)
    rec_start = []
    for r in recs:
        rec_start.append(len(stream)); stream += r[3]
    total = len(stream)
    cuts, split = _cuts(layout, len(hdr), [r[3] for r in recs], rec_start, total, rng)
    codecs = [(6, zlib.Z_DEFAULT_STRATEGY)]
    if layout == "codecs":
        codecs = [(0, 0), (1, 0), (9, 0), (6, zlib.Z_RLE), (6, zlib.Z_HUFFMAN_ONLY), (6, zlib.Z_FIXED), "craft"]
    mem_start, mem_len, coffs, long_codes = [], [], [], 0
    with open(path, "wb") as f:
        for k in range(len(cuts) - 1):
            a, b = cuts[k], cuts[k + 1]
            coffs.append(f.tell()); mem_start.append(a); mem_len.append(b - a)
            member, n = _member(bytes(stream[a:b]), codecs[k % len(codecs)])
            f.write(member); long_codes += n
        end_coff = f.tell()
        f.write(EOF_MEMBER)

    def voff(p):
        """virtual offset of stream position p"""
        if p >= total:
            return end_coff << 16
        h = bisect.bisect_right(mem_start, p) - 1            # the data member holding byte p (empty members at p come before it)
        if mem_start[h] == p:
            j = bisect.bisect_left(mem_start, p)
            if layout == "empty" and j < h:
                return coffs[j] << 16                        # the first of the empty members in front of it
            if layout == "isize_voff" and h > 0:
                return (coffs[h - 1] << 16) | mem_len[h - 1]
        return (coffs[h] << 16) | (p - mem_start[h])

    # BAI as BamWriter builds it
    index = [dict(bins={}, linear={}) for _ in refs]
    pend = None
    for i, (refid, pos, end, _) in enumerate(recs + [(-1, 0, 0, b"")]):
        v0 = voff(rec_start[i]) if i < len(recs) else voff(total)
        if pend is not None:
            prefid, ppos, pendpos, pv0 = pend
            ix = index[prefid]
            chunks = ix["bins"].setdefault(reg2bin(ppos, pendpos), [])
            if chunks and chunks[-1][1] == pv0:
                chunks[-1][1] = v0
            else:
                chunks.append([pv0, v0])
            for w in range(ppos >> 14, ((pendpos - 1) >> 14) + 1):
                if w not in ix["linear"] or pv0 < ix["linear"][w]:
                    ix["linear"][w] = pv0
            pend = None
        if refid >= 0 and i < len(recs):
            pend = (refid, pos, end, v0)
    with open(path + ".bai", "wb") as b:
        b.write(b"BAI\x01" + struct.pack("<i", len(refs)))
        for ix in index:
            b.write(struct.pack("<i", len(ix["bins"])))
            for bin_id, chunks in sorted(ix["bins"].items()):
                if layout == "isize_voff":
                    chunks = chunks[::-1]
                b.write(struct.pack("<Ii", bin_id, len(chunks)))
                for c0, c1 in chunks:
                    b.write(struct.pack("<QQ", c0, c1))
            n_intv = (max(ix["linear"]) + 1) if ix["linear"] else 0
            b.write(struct.pack("<i", n_intv))
            last = 0
            for w in range(n_intv):
                last = ix["linear"].get(w, last)
                b.write(struct.pack("<Q", last))
    # facts: records split across members (and at which field), empty members, offsets written as (k, ISIZE_k)
    rec_voff = [voff(x) for x in rec_start]
    len_of = dict(zip(coffs, mem_len))
    return dict(n_members=len(mem_len), n_records=len(recs), split=split, n_empty=sum(1 for n in mem_len if n == 0),
                crossing=sum(1 for x, r in zip(rec_start, recs) if bisect.bisect_right(mem_start, x) < bisect.bisect_left(mem_start, x + len(r[3]))),
                isize_offsets=sum(1 for v in rec_voff if (v & 0xFFFF) and (v & 0xFFFF) == len_of.get(v >> 16)),
                empty_offsets=sum(1 for v in rec_voff if len_of.get(v >> 16) == 0), rec_voff=rec_voff,
                index=index, coffs=coffs, mem_len=mem_len, long_codes=long_codes)


def shard_range(facts, tid, starts, ends):
    """The BGZF members (indices into the layout) that a device-staged shard of loci [starts, ends) on `tid` must carry: those
    starting between the smallest chunk start and the largest chunk end of the loci's index chunks, starts raised to the
    linear index and ends clipped at the first record of the first 16 kb bin behind each locus -- restated from the SAM
    specification's binning scheme, independently of the reader."""
    ix = facts["index"][tid]
    n_intv = (max(ix["linear"]) + 1) if ix["linear"] else 0
    lin, last = [], 0
    for w in range(n_intv):
        last = ix["linear"].get(w, last); lin.append(last)
    bins = ix["bins"]
    lo, hi = None, 0
    for beg, end in zip(starts, ends):
        min_off = lin[min(beg >> 14, len(lin) - 1)] if lin else 0
        later = [b for b in sorted(bins) if b >= 4681 + ((end - 1) >> 14) + 1 and bins[b]]
        clip = min(c[0] for c in bins[later[0]]) if later else (1 << 64) - 1
        e1 = end - 1
        want = [0] + [k for sh, base in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)) for k in range(base + (beg >> sh), base + (e1 >> sh) + 1)]
        for b in want:
            for c0, c1 in bins.get(b, []):
                if c1 > min_off and c0 < clip:
                    lo = max(c0, min_off) if lo is None else min(lo, max(c0, min_off)); hi = max(hi, min(c1, clip))
    if lo is None:
        return []
    return [k for k, c in enumerate(facts["coffs"]) if lo >> 16 <= c <= hi >> 16]


# ---------------------------------------------------------------------------------------------------------------------
# the record content
# ---------------------------------------------------------------------------------------------------------------------
_ACGT = np.frombuffer(b"ACGT", np.uint8)


def dataset(out_dir: str, seed: int = 3):
    """FASTA, VCF, barcodes and the record list -> dict(fasta, vcf, barcodes, refs, recs).  Two contigs; loci with reads
    of every kind the filters and the record walk care about (see the comments below); unplaced unmapped reads at the end."""
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    refs = [("chrA", 420_000), ("chrB", 60_000)]
    genome = [rng.integers(0, 4, size=L, dtype=np.uint8) for _, L in refs]
    paths = dict(fasta=os.path.join(out_dir, "g.fa"), vcf=os.path.join(out_dir, "v.vcf"), barcodes=os.path.join(out_dir, "b.tsv"))
    with open(paths["fasta"], "wb") as f, open(paths["fasta"] + ".fai", "w") as fai:
        for (name, L), g in zip(refs, genome):
            f.write(f">{name}\n".encode()); off = f.tell()
            seq = _ACGT[g]
            for s0 in range(0, L, 60):
                f.write(seq[s0:s0 + 60].tobytes() + b"\n")
            fai.write(f"{name}\t{L}\t{off}\t60\t61\n")
    cbs = ["".join("ACGT"[(i >> (2 * k)) & 3] for k in range(16)) + "-1" for i in range(40)]
    with open(paths["barcodes"], "w") as f:
        f.write("".join(c + "\n" for c in cbs[:32]))                       # 8 of them unlisted
    enc = _RecordEncoder()
    reads = []            # (refid, pos, mapq, flag, cigar, seq, long_aux)
    loci = []
    b_arrays = b"".join(b"X" + bytes([48 + k]) + b"B" + sub + struct.pack("<i", 3) + bytes(3 * sz)
                        for k, (sub, sz) in enumerate([(b"c", 1), (b"C", 1), (b"s", 2), (b"S", 2), (b"i", 4), (b"I", 4), (b"f", 4)]))

    def aux_for(i, long_aux=False):
        a = b""
        if i % 5 == 0:
            a += b_arrays                                                       # CB behind B arrays of every subtype
        if long_aux:
            a += b"ZZZ" + b"N" * 6000 + b"\0"                                   # longer than the walker's 4 KB window
        if i % 23 != 7:
            a += b"CBZ" + cbs[i % len(cbs)].encode() + b"\0"
        if i % 17 != 3:
            a += b"UBZ" + "".join("ACGT"[(i * 7 + k) % 4 if k % 3 else (i >> k) & 3] for k in range(10)).encode() + b"\0"
        return a

    def read(ci, start, cigar_ops, flag=0, mapq=60, long_aux=False, alt_at=None):
        qlen = sum(n for o, n in cigar_ops if o in "MIS=X")
        g = genome[ci]
        seq = g[start:start + qlen].copy() if start + qlen <= len(g) else rng.integers(0, 4, qlen, dtype=np.uint8)
        if alt_at is not None and 0 <= alt_at - start < qlen and rng.random() < 0.5:
            seq[alt_at - start] = (seq[alt_at - start] + 1) % 4
        reads.append((ci, start, mapq, flag, cigar_ops, _ACGT[seq].tobytes(), long_aux))

    # loci on chrA: every 1 700 bp from 2 000, plus a dense 16 kb window (thousands of records) around 200 000
    for ci, (name, L) in enumerate(refs):
        positions = list(range(2_000, L - 2_000, 1_700 if ci == 0 else 2_300))
        for p in positions:
            loci.append((ci, p))
            for k in range(int(rng.integers(6, 14))):
                s0 = p - int(rng.integers(0, 99))
                r = rng.random()
                if r < 0.05:
                    read(ci, s0, [("M", 100)], mapq=int(rng.integers(0, 30)), alt_at=p)            # low MAPQ
                elif r < 0.10:
                    read(ci, s0, [("M", 100)], flag=0x100, alt_at=p)                               # secondary
                elif r < 0.14:
                    read(ci, s0, [("M", 100)], flag=0x800, alt_at=p)                               # supplementary
                elif r < 0.18:
                    read(ci, s0, [("M", 100)], flag=0x400, alt_at=p)                               # duplicate
                elif r < 0.22 and p - s0 > 12 and s0 + 100 - p > 12:
                    a = p - s0 - 5
                    read(ci, s0, [("M", a), ("N", 400), ("M", 100 - a)])                           # skips the locus: not useful
                elif r < 0.25:
                    read(ci, s0, [("M", 100)], flag=0x4)                                           # unmapped, placed
                elif r < 0.28:
                    read(ci, p, [("I", 3), ("S", 40)])                                             # only I and S: end = pos + 1
                elif r < 0.31:
                    read(ci, p - 100, [("M", 100)])                                                # ends exactly at the locus start
                elif r < 0.34:
                    read(ci, p, [("M", 100)], alt_at=p)                                            # starts at end - 1 (SNV: end = p + 1)
                elif r < 0.36:
                    read(ci, s0, [("M", 50)] + [("M", 1), ("I", 1)] * 600 + [("M", 50)], alt_at=p)  # 1 202 CIGAR ops: > 4 KB
                elif r < 0.38:
                    read(ci, s0, [("M", 100)], alt_at=p, long_aux=True)                            # aux > 4 KB
                else:
                    read(ci, s0, [("M", 100)], alt_at=p)
        if ci == 0:
            for k in range(3000):                                                                   # one dense 16 kb window
                s0 = 196_608 + int(rng.integers(0, 16_000))
                read(ci, s0, [("M", 100)])
            for k in range(40):                                                                     # 150 kb spliced reads
                s0 = int(rng.integers(1_000, L - 160_000))
                read(ci, s0, [("M", 50), ("N", 150_000), ("M", 50)])
    reads.sort(key=lambda r: (r[0], r[1]))
    recs, adds = [], []
    for i, (ci, start, mapq, flag, cig, seq, long_aux) in enumerate(reads):
        qual = bytes(int(x) for x in rng.integers(2, 41, len(seq)))
        adds.append((ci, start, mapq, flag, cig, seq, f"q{i:06d}".encode(), aux_for(i, long_aux), qual))
        rec = enc.encode(*adds[-1])
        rlen = sum(n for o, n in cig if o in "MDN=X") if not (flag & 4) else 0
        recs.append((ci, start, start + (rlen if rlen > 0 else 1), rec))
    for i in range(25):                                                                             # unplaced unmapped reads
        adds.append((-1, -1, 0, 0x4, [], b"ACGTACGTAC", f"u{i}".encode(), aux_for(i)))
        recs.append((-1, -1, 0, enc.encode(*adds[-1])))
    with open(paths["vcf"], "w") as f:
        f.write("##fileformat=VCFv4.2\n" + "".join(f"##contig=<ID={n},length={L}>\n" for n, L in refs) + "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for ci, p in loci:
            refb = "ACGT"[genome[ci][p]]
            f.write(f"{refs[ci][0]}\t{p + 1}\t.\t{refb}\t{'ACGT'[(genome[ci][p] + 1) % 4]}\t.\t.\t.\n")
        for p in range(196_700, 212_000, 900):                                                      # loci inside the dense window
            f.write(f"chrA\t{p + 1}\t.\t{'ACGT'[genome[0][p]]}\t{'ACGT'[(genome[0][p] + 2) % 4]}\t.\t.\t.\n")
    # the VCF must be sorted for the device path to take every shard: rewrite it sorted
    lines = open(paths["vcf"]).read().splitlines()
    head = [ln for ln in lines if ln.startswith("#")]
    body = sorted((ln for ln in lines if not ln.startswith("#")), key=lambda ln: (ln.split("\t")[0], int(ln.split("\t")[1])))
    with open(paths["vcf"], "w") as f:
        f.write("\n".join(head + body) + "\n")
    paths.update(refs=refs, recs=recs, adds=adds, n_loci=len(body))
    return paths
