"""CPU ORACLE (test infrastructure, NOT product code) -- file decode + orchestration.

Pure-Python restatement of the host side of vartrix src/main.rs (`_main`, 163-418):
barcode loading, VCF slurp, haplotype construction, BAM region fetch + the four record filters,
staging into the batch layout of ``vtx_oracle.h`` and hand-off to the C oracle
(``libvtx_oracle.so``) for CB lookup, Smith-Waterman and aggregation.  Only tests/,
``__graft_entry__.smoke()`` and bench.py's cpu_baseline may import this package.

External semantics restated from their published behaviour (sources not vendored in the reference):
  * htslib region iterator (rust-htslib 0.36 ``IndexedReader::fetch`` + ``records``, main.rs:822-829):
    every record on the contig with ``pos < end`` and ``bam_endpos > start`` in file order, where
    bam_endpos = pos + reference length of the CIGAR (pos + 1 for unmapped / empty CIGAR).
  * ``Record::aux`` (main.rs:742, 753): first aux field with that tag; only type ``Z`` is accepted.
  * sprs 0.7.1 ``write_matrix_market`` text layout (observed in every golden, SURVEY.md A.9).
"""
from __future__ import annotations

import ctypes
import gzip
import os
import struct
import subprocess
import zlib
from dataclasses import dataclass, field
from decimal import Decimal

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

MODE_CONSENSUS, MODE_COVERAGE, MODE_ALT_FRAC = 0, 1, 2
MODES = {"consensus": MODE_CONSENSUS, "coverage": MODE_COVERAGE, "alt_frac": MODE_ALT_FRAC}
NO_CB = 0xFFFFFFFF
NO_UMI = 0xFFFFFFFFFFFFFFFF


# --------------------------------------------------------------------------------------------
# ctypes binding of the C oracle
# --------------------------------------------------------------------------------------------
class CBatch(ctypes.Structure):
    _fields_ = [
        ("n_loci", ctypes.c_uint32), ("locus_row", ctypes.c_void_p),
        ("hap_bytes", ctypes.c_void_p), ("hap_bytes_len", ctypes.c_uint64),
        ("ref_off", ctypes.c_void_p), ("ref_len", ctypes.c_void_p),
        ("alt_off", ctypes.c_void_p), ("alt_len", ctypes.c_void_p),
        ("cand_start", ctypes.c_void_p),
        ("n_reads", ctypes.c_uint32), ("read_nib", ctypes.c_void_p), ("read_nib_len", ctypes.c_uint64),
        ("read_off", ctypes.c_void_p), ("read_len", ctypes.c_void_p),
        ("cb_bytes", ctypes.c_void_p), ("cb_bytes_len", ctypes.c_uint64),
        ("read_cb_off", ctypes.c_void_p), ("read_cb_len", ctypes.c_void_p),
        ("read_umi_key", ctypes.c_void_p),
        ("n_cand", ctypes.c_uint64), ("cand_read", ctypes.c_void_p),
    ]


class CMetrics(ctypes.Structure):
    _fields_ = [("num_not_cell_bc", ctypes.c_uint64), ("num_non_umi", ctypes.c_uint64),
                ("num_scored", ctypes.c_uint64)]


class CResult(ctypes.Structure):
    _fields_ = [("n", ctypes.c_uint64), ("row", ctypes.c_void_p), ("col", ctypes.c_void_p),
                ("ref_cnt", ctypes.c_void_p), ("alt_cnt", ctypes.c_void_p), ("unk_cnt", ctypes.c_void_p),
                ("val", ctypes.c_void_p), ("val2", ctypes.c_void_p), ("metrics", CMetrics)]


_LIB = None


def build_oracle() -> str:
    """Compile oracle/libvtx_oracle.so with the committed Makefile (idempotent)."""
    subprocess.run(["make", "-s", "-C", _HERE], check=True)
    return os.path.join(_HERE, "libvtx_oracle.so")


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libvtx_oracle.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "vtx_oracle.c")):
            build_oracle()
        L = ctypes.CDLL(path)
        L.vtxo_sw_full.restype = ctypes.c_int32
        L.vtxo_sw_full.argtypes = [ctypes.c_char_p, ctypes.c_int32, ctypes.c_char_p, ctypes.c_int32]
        L.vtxo_sw_fold.restype = ctypes.c_int32
        L.vtxo_sw_fold.argtypes = [ctypes.c_char_p, ctypes.c_int32, ctypes.c_char_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32]
        L.vtxo_sw_band_model.restype = ctypes.c_int32
        L.vtxo_sw_band_model.argtypes = [ctypes.c_char_p, ctypes.c_int32, ctypes.c_char_p, ctypes.c_int32,
                                         ctypes.c_int32, ctypes.c_int32]
        L.vtxo_evaluate_scores.restype = ctypes.c_int32
        L.vtxo_evaluate_scores.argtypes = [ctypes.c_int32, ctypes.c_int32]
        L.vtxo_useful_alignment.restype = ctypes.c_int32
        L.vtxo_useful_alignment.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_int64]
        L.vtxo_score_pairs.restype = ctypes.c_int32
        L.vtxo_score_pairs.argtypes = [ctypes.POINTER(CBatch), ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]
        L.vtxo_run_batch.restype = ctypes.c_int32
        L.vtxo_run_batch.argtypes = [ctypes.POINTER(CBatch), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32,
                                     ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                     ctypes.c_int32, ctypes.POINTER(CResult)]
        L.vtxo_free_result.restype = None
        L.vtxo_free_result.argtypes = [ctypes.POINTER(CResult)]
        _LIB = L
    return _LIB


# --------------------------------------------------------------------------------------------
# staged batch (numpy side)
# --------------------------------------------------------------------------------------------
@dataclass
class Batch:
    """Staged (read, ref-window, alt-window, CB-tag) batch; field meaning = vtxo_batch."""
    locus_row: np.ndarray
    hap_bytes: np.ndarray
    ref_off: np.ndarray
    ref_len: np.ndarray
    alt_off: np.ndarray
    alt_len: np.ndarray
    cand_start: np.ndarray
    read_nib: np.ndarray
    read_off: np.ndarray
    read_len: np.ndarray
    cb_bytes: np.ndarray
    read_cb_off: np.ndarray
    read_cb_len: np.ndarray
    read_umi_key: np.ndarray
    cand_read: np.ndarray
    n_rows: int = 0
    host_metrics: dict = field(default_factory=dict)

    FIELDS = ("locus_row", "hap_bytes", "ref_off", "ref_len", "alt_off", "alt_len", "cand_start",
              "read_nib", "read_off", "read_len", "cb_bytes", "read_cb_off", "read_cb_len",
              "read_umi_key", "cand_read")
    DTYPES = dict(locus_row=np.uint32, hap_bytes=np.uint8, ref_off=np.uint32, ref_len=np.uint32,
                  alt_off=np.uint32, alt_len=np.uint32, cand_start=np.uint64, read_nib=np.uint8,
                  read_off=np.uint64, read_len=np.uint32, cb_bytes=np.uint8, read_cb_off=np.uint32,
                  read_cb_len=np.uint16, read_umi_key=np.uint64, cand_read=np.uint32)

    def normalized(self) -> "Batch":
        kw = {f: np.ascontiguousarray(getattr(self, f), dtype=self.DTYPES[f]) for f in self.FIELDS}
        return Batch(n_rows=self.n_rows, host_metrics=dict(self.host_metrics), **kw)

    @property
    def n_loci(self): return int(len(self.locus_row))
    @property
    def n_reads(self): return int(len(self.read_len))
    @property
    def n_cand(self): return int(len(self.cand_read))

    def to_c(self) -> CBatch:
        c = CBatch()
        def p(a):
            return a.ctypes.data if a.size else None
        c.n_loci = self.n_loci; c.locus_row = p(self.locus_row)
        c.hap_bytes = p(self.hap_bytes); c.hap_bytes_len = self.hap_bytes.size
        c.ref_off = p(self.ref_off); c.ref_len = p(self.ref_len)
        c.alt_off = p(self.alt_off); c.alt_len = p(self.alt_len)
        c.cand_start = p(self.cand_start)
        c.n_reads = self.n_reads; c.read_nib = p(self.read_nib); c.read_nib_len = self.read_nib.size
        c.read_off = p(self.read_off); c.read_len = p(self.read_len)
        c.cb_bytes = p(self.cb_bytes); c.cb_bytes_len = self.cb_bytes.size
        c.read_cb_off = p(self.read_cb_off); c.read_cb_len = p(self.read_cb_len)
        c.read_umi_key = p(self.read_umi_key)
        c.n_cand = self.n_cand; c.cand_read = p(self.cand_read)
        return c

    def save(self, path: str):
        np.savez_compressed(path, n_rows=np.int64(self.n_rows), **{f: getattr(self, f) for f in self.FIELDS})

    @staticmethod
    def load(path: str) -> "Batch":
        z = np.load(path)
        return Batch(n_rows=int(z["n_rows"]), **{f: z[f] for f in Batch.FIELDS}).normalized()


@dataclass
class Barcodes:
    """load_barcodes (main.rs:697-718): first-seen order, duplicates keep the first index."""
    keys: list
    bytes_: np.ndarray = None
    off: np.ndarray = None

    def __post_init__(self):
        off = np.zeros(len(self.keys) + 1, dtype=np.uint32)
        if self.keys:
            off[1:] = np.cumsum([len(k) for k in self.keys])
        self.off = off
        self.bytes_ = np.frombuffer(b"".join(self.keys), dtype=np.uint8).copy() if self.keys else np.zeros(0, np.uint8)

    def __len__(self): return len(self.keys)


def load_barcodes(path: str) -> Barcodes:
    opener = gzip.open if path.endswith(".gz") else open     # by extension only, main.rs:727
    seen, keys = set(), []
    with opener(path, "rb") as fh:
        data = fh.read()
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    for ln in lines:                                         # BufRead::lines strips \n and \r\n
        if ln.endswith(b"\r"):
            ln = ln[:-1]
        if ln not in seen:
            seen.add(ln); keys.append(ln)
    if not keys:
        raise SystemExit("Loaded 0 barcodes. Is your barcode file gzipped or empty?")   # main.rs:712-715
    return Barcodes(keys)


@dataclass
class Result:
    row: np.ndarray
    col: np.ndarray
    ref_cnt: np.ndarray
    alt_cnt: np.ndarray
    unk_cnt: np.ndarray
    val: np.ndarray
    val2: np.ndarray
    metrics: dict


MIN_SCORE = 25                                               # main.rs:30


def run_batch(batch: Batch, barcodes: Barcodes, mode: int, use_umi: bool, n_threads: int = 1,
              band_model: bool = False, min_score: int = MIN_SCORE) -> Result:
    """min_score: evaluate_scores' MIN_SCORE (a pair is None when both scores are below it), like Engine(min_score=)."""
    L = lib()
    b = batch.normalized()
    cb = b.to_c()
    res = CResult()
    rc = L.vtxo_run_batch(ctypes.byref(cb), barcodes.bytes_.ctypes.data if barcodes.bytes_.size else None,
                          barcodes.off.ctypes.data, len(barcodes), mode, int(use_umi), n_threads,
                          int(band_model), int(min_score), ctypes.byref(res))
    if rc != 0:
        raise RuntimeError(f"vtxo_run_batch failed: {rc}")
    n = int(res.n)
    def arr(ptr, dt):
        if n == 0:
            return np.zeros(0, dt)
        return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(np.ctypeslib.as_ctypes_type(dt))), shape=(n,)).copy()
    out = Result(arr(res.row, np.uint32), arr(res.col, np.uint32), arr(res.ref_cnt, np.uint32),
                 arr(res.alt_cnt, np.uint32), arr(res.unk_cnt, np.uint32), arr(res.val, np.float64),
                 arr(res.val2, np.float64),
                 dict(num_not_cell_bc=int(res.metrics.num_not_cell_bc), num_non_umi=int(res.metrics.num_non_umi),
                      num_scored=int(res.metrics.num_scored)))
    L.vtxo_free_result(ctypes.byref(res))
    return out


def score_pairs(batch: Batch, pair_read: np.ndarray, pair_locus: np.ndarray, n_threads: int = 1):
    L = lib()
    b = batch.normalized(); cb = b.to_c()
    pr = np.ascontiguousarray(pair_read, np.uint32); pl = np.ascontiguousarray(pair_locus, np.uint32)
    rs = np.zeros(len(pr), np.int32); as_ = np.zeros(len(pr), np.int32)
    L.vtxo_score_pairs(ctypes.byref(cb), len(pr), pr.ctypes.data, pl.ctypes.data, n_threads,
                       rs.ctypes.data, as_.ctypes.data)
    return rs, as_


def sw_full(x: bytes, y: bytes) -> int:
    return lib().vtxo_sw_full(x, len(x), y, len(y))


def sw_fold(x: bytes, y: bytes, p: int, s: int) -> int:
    """The same score through the prefix / reversed-suffix / middle / junction decomposition (vtxo_sw_fold)."""
    return lib().vtxo_sw_fold(x, len(x), y, len(y), p, s)


def sw_band_model(x: bytes, y: bytes, k: int = 6, w: int = 20) -> int:
    return lib().vtxo_sw_band_model(x, len(x), y, len(y), k, w)


# --------------------------------------------------------------------------------------------
# Matrix Market text (sprs 0.7.1 write_matrix_market, main.rs:381-389)
# --------------------------------------------------------------------------------------------
def fmt_f64(v: float) -> str:
    """Rust `{}` for f64: shortest round-trip digits, never an exponent, `NaN`."""
    if v != v:
        return "NaN"
    if v in (float("inf"), float("-inf")):
        return "inf" if v > 0 else "-inf"
    if v == int(v) and abs(v) < 1e16:
        return str(int(v))
    return format(Decimal(repr(float(v))), "f")


def mtx_text(n_rows: int, n_cols: int, row, col, val) -> str:
    lines = ["%%MatrixMarket matrix coordinate real general", "% written by sprs", f"{n_rows} {n_cols} {len(row)}"]
    lines += [f"{int(r) + 1} {int(c) + 1} {fmt_f64(float(v))}" for r, c, v in zip(row, col, val)]
    return "\n".join(lines) + "\n"


def read_mtx(path: str):
    """-> (n_rows, n_cols, {(row0, col0): value}) ; the reference compares goldens as CSR sets (main.rs:1230-1232)."""
    with open(path) as fh:
        lines = [ln for ln in fh.read().split("\n") if ln and not ln.startswith("%")]
    nr, nc, nnz = (int(t) for t in lines[0].split())
    ent = {}
    for ln in lines[1:]:
        r, c, v = ln.split()
        key = (int(r) - 1, int(c) - 1)
        ent[key] = ent.get(key, 0.0) + float(v)          # to_csr sums duplicates
    assert len(lines) - 1 == nnz
    return nr, nc, ent


# --------------------------------------------------------------------------------------------
# FASTA (.fai) / VCF / BAM readers
# --------------------------------------------------------------------------------------------
class Fasta:
    def __init__(self, path: str):
        self.seqs, self.order = {}, []
        name, parts = None, []
        with open(path, "rb") as fh:
            for ln in fh:
                ln = ln.rstrip(b"\r\n")
                if ln.startswith(b">"):
                    if name is not None:
                        self.seqs[name] = b"".join(parts)
                    name = ln[1:].split()[0].decode(); parts = []; self.order.append(name)
                else:
                    parts.append(ln)
        if name is not None:
            self.seqs[name] = b"".join(parts)

    def length(self, chrom): return len(self.seqs[chrom])

    def fetch_upper(self, chrom, start, end):       # read_locus, main.rs:936-954
        return self.seqs[chrom][start:end].upper()


@dataclass
class VcfRec:
    chrom: str
    pos0: int            # rec.pos(), 0-based
    alleles: list        # [REF, ALT...] as bytes; ALT '.' -> 1 allele (main.rs:654-659)


def read_vcf(path: str):
    opener = gzip.open if path.endswith(".gz") else open
    recs = []
    with opener(path, "rb") as fh:
        for ln in fh:
            if ln.startswith(b"#") or not ln.strip():
                continue
            f = ln.rstrip(b"\r\n").split(b"\t")
            alleles = [f[3]] + ([] if f[4] == b"." else f[4].split(b","))
            recs.append(VcfRec(f[0].decode(), int(f[1]) - 1, alleles))
    return recs


class Bam:
    """Whole-file BAM decode (BGZF via zlib) into numpy columns + per-record byte views."""

    def __init__(self, path: str):
        raw = open(path, "rb").read()
        out, p = [], 0
        while p < len(raw):
            # BGZF block: gzip member with BC extra subfield holding BSIZE
            xlen = struct.unpack_from("<H", raw, p + 10)[0]
            bsize = None
            q = p + 12
            while q < p + 12 + xlen:
                si1, si2, slen = raw[q], raw[q + 1], struct.unpack_from("<H", raw, q + 2)[0]
                if si1 == 66 and si2 == 67:
                    bsize = struct.unpack_from("<H", raw, q + 4)[0]
                q += 4 + slen
            cdata = raw[p + 12 + xlen: p + bsize + 1 - 8]
            out.append(zlib.decompress(cdata, -15))
            p += bsize + 1
        data = b"".join(out)
        assert data[:4] == b"BAM\x01"
        l_text = struct.unpack_from("<i", data, 4)[0]
        p = 8 + l_text
        n_ref = struct.unpack_from("<i", data, p)[0]; p += 4
        self.ref_names, self.ref_lens = [], []
        for _ in range(n_ref):
            l_name = struct.unpack_from("<i", data, p)[0]; p += 4
            self.ref_names.append(data[p:p + l_name - 1].decode()); p += l_name
            self.ref_lens.append(struct.unpack_from("<i", data, p)[0]); p += 4
        self.data = data
        offs = []
        while p < len(data):
            bs = struct.unpack_from("<i", data, p)[0]
            offs.append(p + 4); p += 4 + bs
        self.rec_off = np.array(offs, dtype=np.int64)
        n = len(offs)
        self.refid = np.zeros(n, np.int32); self.pos = np.zeros(n, np.int64); self.endpos = np.zeros(n, np.int64)
        self.mapq = np.zeros(n, np.uint8); self.flag = np.zeros(n, np.uint16); self.l_seq = np.zeros(n, np.int32)
        self._cig = [None] * n; self._meta = [None] * n
        for i, o in enumerate(offs):
            refid, pos, l_rn, mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", data, o)
            self.refid[i] = refid; self.pos[i] = pos; self.mapq[i] = mapq; self.flag[i] = flag; self.l_seq[i] = l_seq
            co = o + 32 + l_rn
            cig = np.frombuffer(data, dtype="<u4", count=n_cig, offset=co)
            self._cig[i] = cig
            rlen = 0
            if not (flag & 4):
                for c in cig:
                    if (c & 0xF) in (0, 2, 3, 7, 8):
                        rlen += int(c >> 4)
            self.endpos[i] = pos + (rlen if rlen > 0 else 1)
            so = co + 4 * n_cig
            ao = so + (l_seq + 1) // 2 + l_seq
            bs = struct.unpack_from("<i", data, o - 4)[0]
            self._meta[i] = (so, ao, o + bs)

    def __len__(self): return len(self.rec_off)

    def cigar(self, i): return self._cig[i]

    def seq_nib(self, i) -> bytes:
        so, _, _ = self._meta[i]
        return self.data[so: so + (int(self.l_seq[i]) + 1) // 2]

    def aux_z(self, i, tag: bytes):
        """First aux field named `tag`; value bytes if its type is Z else None (main.rs:742-749)."""
        _, p, end = self._meta[i]
        d = self.data
        while p + 3 <= end:
            t, ty = d[p:p + 2], d[p + 2:p + 3]
            p += 3
            if ty == b"Z" or ty == b"H":
                q = d.index(b"\x00", p)
                if t == tag:
                    return d[p:q] if ty == b"Z" else None
                p = q + 1
            else:
                if ty in b"AcC": sz = 1
                elif ty in b"sS": sz = 2
                elif ty in b"iIf": sz = 4
                elif ty == b"B":
                    sub = d[p:p + 1]; cnt = struct.unpack_from("<i", d, p + 1)[0]
                    sz = 5 + cnt * {b"c": 1, b"C": 1, b"s": 2, b"S": 2, b"i": 4, b"I": 4, b"f": 4}[sub]
                else:
                    raise ValueError(f"bad aux type {ty!r}")
                if t == tag:
                    return None
                p += sz
        return None

    def fetch(self, chrom: str, start: int, end: int) -> np.ndarray:
        tid = self.ref_names.index(chrom)
        m = (self.refid == tid) & (self.pos < end) & (self.endpos > start)
        return np.nonzero(m)[0]


# --------------------------------------------------------------------------------------------
# orchestration: files -> staged batch (evaluate_rec / evaluate_alns up to the CB lookup)
# --------------------------------------------------------------------------------------------
def construct_haplotypes(fa: Fasta, chrom: str, start: int, end: int, alt: bytes, padding: int):
    """main.rs:958-994."""
    L = fa.length(chrom)
    alt_hap = fa.fetch_upper(chrom, max(start - padding, 0), start) + alt + fa.fetch_upper(chrom, end, min(end + padding, L))
    ref_hap = fa.fetch_upper(chrom, max(0, start - padding), min(end + padding, L))
    return ref_hap, alt_hap


def stage_from_files(vcf: str, bam: str, fasta: str, padding: int = 100, mapq: int = 0,
                     primary_only: bool = False, no_duplicates: bool = False, bam_tag: str = "CB",
                     valid_chars: str = "ATGCatgc", rec_lo: int = 0, rec_hi: int | None = None) -> Batch:
    L = lib()
    recs = read_vcf(vcf)
    fa = Fasta(fasta)
    bm = Bam(bam)
    valid = set(valid_chars.encode())
    met = dict(num_reads=0, num_low_mapq=0, num_non_primary=0, num_duplicates=0, num_not_useful=0,
               num_invalid_recs=0, num_multiallelic_recs=0)
    locus_row, ref_off, ref_len, alt_off, alt_len, cand_start = [], [], [], [], [], [0]
    haps = bytearray()
    read_index = {}                      # BAM record index -> staged read id
    read_nib = bytearray(); read_off, read_len = [], []
    cb_bytes = bytearray(); read_cb_off, read_cb_len, read_umi_key = [], [], []
    umi_intern = {}
    cand_read = []
    tag = bam_tag.encode()
    for i, rec in enumerate(recs):
        if i < rec_lo or (rec_hi is not None and i >= rec_hi):
            continue
        start = rec.pos0; end = start + len(rec.alleles[0])              # main.rs:619-623
        if len(rec.alleles) > 2:                                         # main.rs:646-653
            met["num_multiallelic_recs"] += 1; continue
        alt = rec.alleles[1] if len(rec.alleles) == 2 else b""          # main.rs:656-659
        ref_hap, alt_hap = construct_haplotypes(fa, rec.chrom, start, end, alt, padding)
        if any(c not in valid for c in alt_hap):                         # main.rs:675-684
            met["num_invalid_recs"] += 1; continue
        def put(h):
            while len(haps) % 16: haps.append(0)
            o = len(haps); haps.extend(h); return o
        locus_row.append(i)
        ref_off.append(put(ref_hap)); ref_len.append(len(ref_hap))
        alt_off.append(put(alt_hap)); alt_len.append(len(alt_hap))
        for ri in bm.fetch(rec.chrom, start, end):                       # main.rs:822-829
            ri = int(ri)
            met["num_reads"] += 1
            fl = int(bm.flag[ri])
            if int(bm.mapq[ri]) < mapq: met["num_low_mapq"] += 1; continue                        # 833
            if primary_only and (fl & 0x100 or fl & 0x800): met["num_non_primary"] += 1; continue  # 841
            if no_duplicates and (fl & 0x400): met["num_duplicates"] += 1; continue                # 849
            cig = np.ascontiguousarray(bm.cigar(ri), dtype=np.uint32)
            if not L.vtxo_useful_alignment(int(bm.pos[ri]), cig.ctypes.data if cig.size else None, len(cig), start, end):
                met["num_not_useful"] += 1; continue                                               # 857
            if ri not in read_index:
                read_index[ri] = len(read_len)
                while len(read_nib) % 16: read_nib.append(0)
                read_off.append(len(read_nib)); read_nib.extend(bm.seq_nib(ri)); read_len.append(int(bm.l_seq[ri]))
                cb = bm.aux_z(ri, tag)
                if cb is None:
                    read_cb_off.append(NO_CB); read_cb_len.append(0)
                else:
                    read_cb_off.append(len(cb_bytes)); read_cb_len.append(len(cb)); cb_bytes.extend(cb)
                ub = bm.aux_z(ri, b"UB")                                                           # main.rs:752-757
                read_umi_key.append(NO_UMI if ub is None else umi_intern.setdefault(ub, len(umi_intern)))
            cand_read.append(read_index[ri])
        cand_start.append(len(cand_read))
    while len(read_nib) % 16: read_nib.append(0)
    b = Batch(np.array(locus_row, np.uint32), np.frombuffer(bytes(haps), np.uint8).copy(),
              np.array(ref_off, np.uint32), np.array(ref_len, np.uint32), np.array(alt_off, np.uint32),
              np.array(alt_len, np.uint32), np.array(cand_start, np.uint64),
              np.frombuffer(bytes(read_nib), np.uint8).copy(), np.array(read_off, np.uint64),
              np.array(read_len, np.uint32), np.frombuffer(bytes(cb_bytes), np.uint8).copy(),
              np.array(read_cb_off, np.uint32), np.array(read_cb_len, np.uint16),
              np.array(read_umi_key, np.uint64), np.array(cand_read, np.uint32),
              n_rows=len(recs), host_metrics=met)
    return b.normalized()


def run_files(vcf, bam, fasta, cell_barcodes, scoring_method="consensus", umi=False, n_threads=1, **kw):
    """The reference's `_main` on the CPU oracle: -> (n_rows, n_cols, Result, Batch, Barcodes)."""
    bcs = load_barcodes(cell_barcodes)
    batch = stage_from_files(vcf, bam, fasta, **kw)
    res = run_batch(batch, bcs, MODES[scoring_method], umi, n_threads)
    return batch.n_rows, len(bcs), res, batch, bcs
