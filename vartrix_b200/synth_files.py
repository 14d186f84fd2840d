"""Synthetic datasets as real files: FASTA + .fai, VCF, coordinate-sorted BAM + .bai, barcodes.tsv --
the same inputs the reference binary consumes (SURVEY.md 7.5), so the CLI (csrc/host/main.cpp) and the
oracle pipeline can be run on identical files anywhere.  Pure Python + zlib (no htslib in this image).

Besides the BASELINE.json read model (reads covering the variant, ref/alt 50/50, 0.5 % errors) the
generator sprinkles in the cases the record filters and parsers must handle: soft clips, spliced (N)
reads that skip the locus, secondary / duplicate / low-mapq records, reads without CB or UB, unmapped
placed reads, multi-allelic and symbolic records, a deletion written with an empty ALT ("."), lower-case
FASTA stretches and a second contig.
"""
from __future__ import annotations

import os
import struct
import zlib

import numpy as np

_ASCII = np.frombuffer(b"ACGT", np.uint8)
_NIB = {65: 1, 67: 2, 71: 4, 84: 8, 78: 15}
_OPS = {"M": 0, "I": 1, "D": 2, "N": 3, "S": 4, "H": 5, "P": 6, "=": 7, "X": 8}


def reg2bin(beg: int, end: int) -> int:
    end -= 1
    if beg >> 14 == end >> 14: return ((1 << 15) - 1) // 7 + (beg >> 14)
    if beg >> 17 == end >> 17: return ((1 << 12) - 1) // 7 + (beg >> 17)
    if beg >> 20 == end >> 20: return ((1 << 9) - 1) // 7 + (beg >> 20)
    if beg >> 23 == end >> 23: return ((1 << 6) - 1) // 7 + (beg >> 23)
    if beg >> 26 == end >> 26: return ((1 << 3) - 1) // 7 + (beg >> 26)
    return 0


class BamWriter:
    """Minimal BGZF/BAM/BAI writer; every BGZF block holds whole records so virtual offsets are simple."""

    def __init__(self, path: str, refs):
        self.path, self.refs = path, refs
        self.f = open(path, "wb")
        self.block = bytearray()
        self.index = [dict(bins={}, linear={}) for _ in refs]
        self._pending = None
        text = "@HD\tVN:1.6\tSO:coordinate\n" + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in refs)
        hdr = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
        for n, l in refs:
            hdr += struct.pack("<i", len(n) + 1) + n.encode() + b"\x00" + struct.pack("<i", l)
        self.block += hdr
        self._flush()

    def _flush(self):
        if not self.block:
            return
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        comp = co.compress(bytes(self.block)) + co.flush()
        bsize = len(comp) + 25
        self.f.write(struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, bsize))
        self.f.write(comp)
        self.f.write(struct.pack("<II", zlib.crc32(bytes(self.block)) & 0xFFFFFFFF, len(self.block)))
        self.block = bytearray()

    def _voff(self):
        return (self.f.tell() << 16) | len(self.block)

    def add(self, refid, pos, mapq, flag, cigar, seq: bytes, qname: bytes, aux: bytes, qual: bytes | None = None):
        """cigar = [(op char, len)], seq = ASCII bases, qual = one Phred value (not +33) per base; None writes absent
        qualities (0xFF, as samtools does)."""
        l_seq = len(seq)
        if qual is not None and len(qual) != l_seq:
            raise ValueError(f"{len(qual)} qualities for {l_seq} bases")
        nib = bytearray((l_seq + 1) // 2)
        for i, c in enumerate(seq):
            v = _NIB.get(c, 15)
            nib[i >> 1] |= v << 4 if not (i & 1) else v
        cig = b"".join(struct.pack("<I", (n << 4) | _OPS[o]) for o, n in cigar)
        rlen = sum(n for o, n in cigar if o in "MDN=X") if not (flag & 4) else 0
        end = pos + (rlen if rlen > 0 else 1)
        body = struct.pack("<iiBBHHHiiii", refid, pos, len(qname) + 1, mapq, reg2bin(pos, end), len(cigar), flag, l_seq, -1, -1, 0)
        body += qname + b"\x00" + cig + bytes(nib) + (b"\xff" * l_seq if qual is None else bytes(qual)) + aux
        rec = struct.pack("<i", len(body)) + body
        if len(self.block) + len(rec) > 0xFF00:
            self._flush()
        v0 = self._voff()
        if self._pending is not None:          # close the previous record's chunk at this record's start
            self._close_pending(v0)
        self.block += rec
        if refid >= 0:
            self._pending = (refid, pos, end, v0)

    def _close_pending(self, v_end):
        refid, pos, end, v0 = self._pending
        ix = self.index[refid]
        chunks = ix["bins"].setdefault(reg2bin(pos, end), [])
        if chunks and chunks[-1][1] == v0:
            chunks[-1][1] = v_end
        else:
            chunks.append([v0, v_end])
        for w in range(pos >> 14, ((end - 1) >> 14) + 1):
            if w not in ix["linear"] or v0 < ix["linear"][w]:
                ix["linear"][w] = v0
        self._pending = None

    def close(self):
        self._flush()
        if self._pending is not None:
            self._close_pending(self.f.tell() << 16)
        self.f.write(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))   # BGZF EOF marker
        self.f.close()
        with open(self.path + ".bai", "wb") as b:
            b.write(b"BAI\x01" + struct.pack("<i", len(self.refs)))
            for ix in self.index:
                b.write(struct.pack("<i", len(ix["bins"])))
                for bin_id, chunks in sorted(ix["bins"].items()):
                    b.write(struct.pack("<Ii", bin_id, len(chunks)))
                    for c0, c1 in chunks:
                        b.write(struct.pack("<QQ", c0, c1))
                n_intv = (max(ix["linear"]) + 1) if ix["linear"] else 0
                b.write(struct.pack("<i", n_intv))
                last = 0
                for w in range(n_intv):            # htslib fills empty windows with the previous offset
                    last = ix["linear"].get(w, last)
                    b.write(struct.pack("<Q", last))


def _aux_z(tag: bytes, val: bytes) -> bytes:
    return tag + b"Z" + val + b"\x00"


def write_dataset(out_dir: str, n_loci: int = 200, n_barcodes: int = 50, depth: int = 30, read_len: int = 100, seed: int = 1,
                  kind: str = "mixed", umi: bool = True, edge_cases: bool = True, line_width: int = 60):
    """-> dict of paths.  kind: snv | indel | mixed."""
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    spacing = 700
    contigs = [("chr1", 1000 + spacing * (n_loci - n_loci // 4) + 1000), ("chr2", 1000 + spacing * (n_loci // 4) + 1000)]
    genome = [rng.integers(0, 4, size=L, dtype=np.uint8) for _, L in contigs]
    lower = [np.zeros(L, bool) for _, L in contigs]
    if edge_cases:
        for g in lower:                         # soft-masked stretches: the reference upper-cases windows (main.rs:952)
            for s in rng.integers(0, len(g) - 50, size=max(1, len(g) // 5000)):
                g[s:s + 40] = True
    paths = {k: os.path.join(out_dir, v) for k, v in dict(fasta="genome.fa", vcf="variants.vcf", bam="reads.bam",
                                                         barcodes="barcodes.tsv").items()}
    # FASTA + .fai
    with open(paths["fasta"], "wb") as fa, open(paths["fasta"] + ".fai", "w") as fai:
        for (name, L), g, lo in zip(contigs, genome, lower):
            fa.write(f">{name}\n".encode())
            off = fa.tell()
            seq = _ASCII[g].copy(); seq[lo] += 32
            for s in range(0, L, line_width):
                fa.write(seq[s:s + line_width].tobytes() + b"\n")
            fai.write(f"{name}\t{L}\t{off}\t{line_width}\t{line_width + 1}\n")
    # barcodes (a duplicate line and CRLF exercise load_barcodes)
    codes = rng.permutation(4 ** 8)[: n_barcodes + 8]
    def bc(v): return "".join("ACGT"[(int(v) >> (2 * k)) & 3] for k in range(8)) + "ACGTACGT-1"
    listed = [bc(v) for v in codes[:n_barcodes]]; unlisted = [bc(v) for v in codes[n_barcodes:]]
    with open(paths["barcodes"], "w", newline="") as f:
        for i, b in enumerate(listed):
            f.write(b + ("\r\n" if edge_cases and i == 1 else "\n"))
            if edge_cases and i == 2:
                f.write(listed[0] + "\n")
    # loci
    recs_vcf, reads = [], []
    for li in range(n_loci):
        ci = 0 if li < n_loci - n_loci // 4 else 1
        k = li if ci == 0 else li - (n_loci - n_loci // 4)
        pos = 800 + spacing * k + int(rng.integers(0, 100))
        g = genome[ci]
        t = kind if kind != "mixed" else ("snv", "ins", "del")[li % 3]
        if t == "indel": t = "ins" if rng.random() < 0.5 else "del"
        special = None
        if edge_cases and li % 37 == 5: special = "multi"
        elif edge_cases and li % 41 == 7: special = "symbolic"
        elif edge_cases and li % 43 == 9: special = "emptyalt"
        refb = "ACGT"[g[pos]]
        if t == "snv":
            ref, alt = refb, "ACGT"[(g[pos] + int(rng.integers(1, 4))) % 4]
        elif t == "ins":
            L = int(rng.integers(1, 31)); ref = refb; alt = refb + "".join("ACGT"[x] for x in rng.integers(0, 4, size=L))
        else:
            L = int(rng.integers(1, 31)); ref = "".join("ACGT"[x] for x in g[pos:pos + 1 + L]); alt = refb
        alt_field = alt
        if special == "multi": alt_field = alt + "," + alt + "A"
        if special == "symbolic": alt_field = "<DEL>"
        if special == "emptyalt": ref = "".join("ACGT"[x] for x in g[pos:pos + 3]); alt_field = "."; alt = ""
        recs_vcf.append((contigs[ci][0], pos + 1, ref, alt_field))
        # reads of this locus
        alt_codes = np.array(["ACGT".index(c) for c in alt], np.uint8) if alt else np.zeros(0, np.uint8)
        n_here = depth if not edge_cases else int(rng.integers(max(1, depth // 2), depth + depth // 2 + 1))
        n_pool = max(1, n_here // 3)
        pool = ["".join("ACGT"[x] for x in rng.integers(0, 4, size=10)) for _ in range(n_pool)]
        for _ in range(n_here):
            is_alt = rng.random() < 0.5
            start = pos - int(rng.integers(0, read_len))
            if is_alt:
                left = g[start:pos]
                mid = alt_codes
                need = read_len - len(left) - len(mid)
                if need < 0:
                    mid = mid[:read_len - len(left)]; need = 0
                right = g[pos + len(ref): pos + len(ref) + need]
                seq = np.concatenate([left, mid, right])
                d = len(alt) - len(ref)
                if d == 0: cigar = [("M", read_len)]
                elif d > 0:
                    a = len(left) + 1; ins = min(d, read_len - a)
                    cigar = [("M", a)] + ([("I", ins)] if ins > 0 else []) + ([("M", read_len - a - ins)] if read_len - a - ins > 0 else [])
                    if a >= read_len: cigar = [("M", read_len)]
                else:
                    a = len(left) + len(mid)
                    cigar = [("M", a), ("D", -d), ("M", read_len - a)] if 0 < a < read_len else [("M", read_len)]
            else:
                seq = g[start:start + read_len]; cigar = [("M", read_len)]
            seq = seq.copy()
            errs = rng.random(len(seq)) < 0.005
            seq[errs] = (seq[errs] + rng.integers(1, 4, size=int(errs.sum()))) % 4
            s_ascii = bytearray(_ASCII[seq].tobytes())
            flag, mapq, rpos = 0, 60, start
            cb = listed[int(rng.integers(0, n_barcodes))] if rng.random() > 0.08 else unlisted[int(rng.integers(0, len(unlisted)))]
            ub = pool[int(rng.integers(0, n_pool))]
            aux = b""
            if edge_cases:
                r = rng.random()
                if r < 0.03: flag |= 0x100
                elif r < 0.06: flag |= 0x400
                elif r < 0.09: mapq = int(rng.integers(0, 20))
                elif r < 0.11: flag |= 0x800
                elif r < 0.14 and len(cigar) == 1:          # soft clip the first bases
                    c = int(rng.integers(1, 20)); cigar = [("S", c), ("M", read_len - c)]; rpos = start + c
                elif r < 0.17 and len(cigar) == 1 and pos - start > 12 and start + read_len - pos > 12:
                    a = pos - start - 5                      # spliced read that skips the locus (not useful)
                    cigar = [("M", a), ("N", 400), ("M", read_len - a)]
                elif r < 0.18: s_ascii[int(rng.integers(0, len(s_ascii)))] = ord("N")
                elif r < 0.19: flag |= 0x4                   # unmapped but placed
                q = rng.random()
                if q < 0.03: cb = None
                elif q < 0.05: aux += b"CBi" + struct.pack("<i", 7)          # CB of the wrong type
                if rng.random() < 0.04: ub = None
                aux += b"NHC\x01" + b"xbBC" + struct.pack("<i", 3) + b"\x01\x02\x03"
            if cb is not None and b"CBi" not in aux: aux += _aux_z(b"CB", cb.encode())
            if ub is not None and umi: aux += _aux_z(b"UB", ub.encode())
            reads.append((ci, rpos, mapq, flag, cigar, bytes(s_ascii), aux))
    with open(paths["vcf"], "w") as f:
        f.write("##fileformat=VCFv4.2\n" + "".join(f"##contig=<ID={n},length={L}>\n" for n, L in contigs))
        f.write("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for c, p, r, a in recs_vcf:
            f.write(f"{c}\t{p}\t.\t{r}\t{a}\t.\t.\t.\n")
    reads.sort(key=lambda r: (r[0], r[1]))
    bw = BamWriter(paths["bam"], contigs)
    for i, (ci, rpos, mapq, flag, cigar, seq, aux) in enumerate(reads):
        bw.add(ci, rpos, mapq, flag, cigar, seq, f"r{i}".encode(), aux)
    bw.close()
    paths.update(n_loci=n_loci, n_barcodes=n_barcodes, n_reads=len(reads))
    return paths


# ---------------------------------------------------------------------------------------------------------------
# Bulk writer for the BASELINE-sized file sets (config 3: 100 k SNV loci x 50 reads): every record has the same
# length, so the BAM body, the BGZF blocks and the BAI are built with numpy instead of one Python call per read.
# ---------------------------------------------------------------------------------------------------------------
def _reg2bin_vec(beg, end):
    end = end - 1
    out = np.zeros(len(beg), np.int64)
    done = np.zeros(len(beg), bool)
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        hit = ~done & ((beg >> shift) == (end >> shift))
        out[hit] = base + (beg[hit] >> shift)
        done |= hit
    return out


def write_dataset_fast(out_dir: str, n_loci: int = 100_000, n_barcodes: int = 50_000, depth: int = 50, read_len: int = 150, seed: int = 2,
                       umi: bool = False, spacing: int = 1200, unlisted_frac: float = 0.05, err: float = 0.005, level: int = 1, line_width: int = 60,
                       quals: str = "missing"):
    """SNV loci `spacing` apart on one contig, `depth` reads of `read_len` bases per locus (start uniform over the
    positions that cover the variant, allele ref/alt 50/50, `err` substitution errors, CIGAR <read_len>M, mapq 60), cell tags
    16-mer + "-1" with `unlisted_frac` of the reads carrying an unlisted one; `quals` = "missing" (0xFF) or "binned" (four
    quality levels, i.i.d.: BGZF then compresses ~3.5x like a real BAM instead of ~10x).  -> dict of paths like write_dataset."""
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(seed)
    paths = {k: os.path.join(out_dir, v) for k, v in dict(fasta="genome.fa", vcf="variants.vcf", bam="reads.bam", barcodes="barcodes.tsv").items()}
    L = 2000 + spacing * n_loci
    genome = rng.integers(0, 4, size=L, dtype=np.uint8)
    with open(paths["fasta"], "wb") as fa, open(paths["fasta"] + ".fai", "w") as fai:
        fa.write(b">chr1\n")
        off = fa.tell()
        seq = _ASCII[genome]
        full = L // line_width * line_width
        body = np.empty((full // line_width, line_width + 1), np.uint8)
        body[:, :line_width] = seq[:full].reshape(-1, line_width); body[:, line_width] = 10
        fa.write(body.tobytes())
        if full < L:
            fa.write(seq[full:].tobytes() + b"\n")
        fai.write(f"chr1\t{L}\t{off}\t{line_width}\t{line_width + 1}\n")
    # barcodes: 16 random bases + "-1"; listed ones go to the file
    n_unl = max(16, n_barcodes // 20)
    vals = rng.permutation(np.unique(rng.integers(0, 2**32, size=int((n_barcodes + n_unl) * 1.3) + 64, dtype=np.uint64)))[: n_barcodes + n_unl]
    bases = ((vals[:, None] >> (np.arange(15, -1, -1, dtype=np.uint64) * 2)[None, :]) & 3).astype(np.uint8)
    tags = np.empty((len(vals), 18), np.uint8)
    tags[:, :16] = _ASCII[bases]; tags[:, 16] = ord("-"); tags[:, 17] = ord("1")
    with open(paths["barcodes"], "wb") as f:
        f.write(b"\n".join(bytes(t) for t in tags[:n_barcodes]) + b"\n")
    # variants
    pos = 1000 + spacing * np.arange(n_loci, dtype=np.int64) + rng.integers(0, 100, size=n_loci)
    refb = genome[pos]
    altb = (refb + rng.integers(1, 4, size=n_loci, dtype=np.uint8)) % 4
    with open(paths["vcf"], "w") as f:
        f.write(f"##fileformat=VCFv4.2\n##contig=<ID=chr1,length={L}>\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        f.write("".join(f"chr1\t{p + 1}\t.\t{'ACGT'[r]}\t{'ACGT'[a]}\t.\t.\t.\n" for p, r, a in zip(pos.tolist(), refb.tolist(), altb.tolist())))
    # BAM: fixed-length records
    name_len = 9                                         # "r" + 7 digits + NUL  (wraps above 10 M reads: names only need to exist)
    aux_len = 22 + (14 if umi else 0)
    nb = (read_len + 1) // 2
    body_len = 32 + name_len + 4 + nb + read_len + aux_len
    rec_len = 4 + body_len
    header_text = f"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:{L}\n"
    hdr = b"BAM\x01" + struct.pack("<i", len(header_text)) + header_text.encode() + struct.pack("<i", 1) + struct.pack("<i", 5) + b"chr1\x00" + struct.pack("<i", L)
    per_block = max(1, 0xFF00 // rec_len)
    f = open(paths["bam"], "wb")

    def put_block(raw: bytes) -> int:
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        comp = co.compress(raw) + co.flush()
        start = f.tell()
        f.write(struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, len(comp) + 25))
        f.write(comp)
        f.write(struct.pack("<II", zlib.crc32(raw) & 0xFFFFFFFF, len(raw)))
        return start

    put_block(hdr)
    rec_pos, rec_voff = [], []
    read_no = 0
    carry = np.zeros((0, rec_len), np.uint8); carry_pos = np.zeros(0, np.int64)
    chunk = 4096
    for lo in range(0, n_loci, chunk):
        hi = min(n_loci, lo + chunk); n = (hi - lo) * depth
        loc = np.repeat(np.arange(lo, hi), depth)
        start = pos[loc] - rng.integers(0, read_len, size=n)
        order = np.lexsort((start, loc)); loc, start = loc[order], start[order]
        idx = start[:, None] + np.arange(read_len, dtype=np.int64)[None, :]
        seq = genome[idx]
        is_alt = rng.random(n) < 0.5
        col = (pos[loc] - start)
        rows = np.nonzero(is_alt)[0]
        seq[rows, col[rows]] = altb[loc[rows]]
        n_err = int(rng.binomial(n * read_len, err))
        if n_err:
            ep = rng.integers(0, n * read_len, size=n_err)
            flat = seq.reshape(-1); flat[ep] = (flat[ep] + rng.integers(1, 4, size=n_err, dtype=np.uint8)) % 4
        nibv = np.array([1, 2, 4, 8], np.uint8)[seq]
        if read_len & 1:
            nibv = np.concatenate([nibv, np.zeros((n, 1), np.uint8)], axis=1)
        rec = np.zeros((n, rec_len), np.uint8)
        def put32(c, v): rec[:, c:c + 4] = np.ascontiguousarray(v, dtype="<i4").view(np.uint8).reshape(-1, 4)
        def put16(c, v): rec[:, c:c + 2] = np.ascontiguousarray(v, dtype="<u2").view(np.uint8).reshape(-1, 2)
        put32(0, np.full(n, body_len)); put32(4, np.zeros(n)); put32(8, start)
        rec[:, 12] = name_len; rec[:, 13] = 60
        put16(14, _reg2bin_vec(start, start + read_len)); put16(16, np.ones(n)); put16(18, np.zeros(n))
        put32(20, np.full(n, read_len)); put32(24, np.full(n, -1)); put32(28, np.full(n, -1)); put32(32, np.zeros(n))
        ids = (read_no + np.arange(n)) % 10_000_000
        rec[:, 36] = ord("r")
        for d in range(7):
            rec[:, 37 + d] = 48 + (ids // 10 ** (6 - d)) % 10
        c = 36 + name_len
        put32(c, np.full(n, (read_len << 4) | 0)); c += 4
        rec[:, c:c + nb] = (nibv[:, 0::2] << 4) | nibv[:, 1::2]; c += nb
        if quals == "binned":          # four-level binned qualities drawn independently: ~1 bit per base, harsher on DEFLATE than real runs
            rec[:, c:c + read_len] = np.array([2, 11, 25, 37], np.uint8)[rng.choice(4, size=(n, read_len), p=[0.02, 0.06, 0.12, 0.80])]
        else:                          # "missing": 0xFF as samtools writes absent qualities
            rec[:, c:c + read_len] = 0xFF
        c += read_len
        listed = rng.random(n) >= unlisted_frac
        cbi = np.where(listed, rng.integers(0, n_barcodes, size=n), n_barcodes + rng.integers(0, n_unl, size=n))
        rec[:, c] = ord("C"); rec[:, c + 1] = ord("B"); rec[:, c + 2] = ord("Z"); rec[:, c + 3:c + 21] = tags[cbi]; c += 22
        if umi:
            ub = _ASCII[rng.integers(0, 4, size=(hi - lo, max(1, depth // 3), 10), dtype=np.uint8)]
            pick = rng.integers(0, ub.shape[1], size=n)
            rec[:, c] = ord("U"); rec[:, c + 1] = ord("B"); rec[:, c + 2] = ord("Z"); rec[:, c + 3:c + 13] = ub[loc - lo, pick]
        read_no += n
        rec = np.concatenate([carry, rec]); spos = np.concatenate([carry_pos, start])
        n_full = len(rec) // per_block * per_block if hi < n_loci else len(rec)
        for b0 in range(0, n_full, per_block):
            blk = rec[b0:b0 + per_block]
            co = put_block(blk.tobytes())
            rec_pos.append(spos[b0:b0 + len(blk)])
            rec_voff.append((np.int64(co) << 16) + np.arange(len(blk), dtype=np.int64) * rec_len)
        carry, carry_pos = rec[n_full:], spos[n_full:]
    end_voff = np.int64(f.tell()) << 16
    f.write(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))
    f.close()
    rpos = np.concatenate(rec_pos); voff = np.concatenate(rec_voff)
    vend = np.concatenate([voff[1:], [end_voff]])
    bins = _reg2bin_vec(rpos, rpos + read_len)
    # chunks: maximal runs of consecutive records with the same bin
    run_start = np.nonzero(np.concatenate([[True], bins[1:] != bins[:-1]]))[0]
    run_end = np.concatenate([run_start[1:], [len(bins)]]) - 1
    run_bin, c0, c1 = bins[run_start], voff[run_start], vend[run_end]
    order = np.argsort(run_bin, kind="stable")
    with open(paths["bam"] + ".bai", "wb") as b:
        b.write(b"BAI\x01" + struct.pack("<i", 1))
        ub_, first = np.unique(run_bin[order], return_index=True)
        b.write(struct.pack("<i", len(ub_)))
        bounds = np.concatenate([first, [len(order)]])
        for k, bin_id in enumerate(ub_.tolist()):
            sel = order[bounds[k]:bounds[k + 1]]
            b.write(struct.pack("<Ii", bin_id, len(sel)))
            b.write(np.stack([c0[sel], c1[sel]], axis=1).astype("<u8").tobytes())
        # linear index: smallest record offset per 16 kb window the record overlaps
        w0, w1 = rpos >> 14, (rpos + read_len - 1) >> 14
        n_intv = int(w1.max()) + 1
        lin = np.full(n_intv, np.iinfo(np.int64).max, np.int64)
        np.minimum.at(lin, w0, voff); np.minimum.at(lin, w1, voff)
        last = 0
        out = np.zeros(n_intv, np.int64)
        filled = lin != np.iinfo(np.int64).max
        for w in range(n_intv):                      # htslib fills empty windows with the previous offset
            if filled[w]: last = lin[w]
            out[w] = last
        b.write(struct.pack("<i", n_intv)); b.write(out.astype("<u8").tobytes())
    paths.update(n_loci=n_loci, n_barcodes=n_barcodes, n_reads=int(n_loci) * depth)
    return paths
