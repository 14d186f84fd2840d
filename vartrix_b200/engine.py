"""Python host mirror of the engine's C ABI (used by the tests and bench.py; a production host is
the C++ CLI in csrc/host or any FFI binding of include/vartrix_b200.h).

Names follow the reference (``vartrix src/main.rs``): a *locus* is one VCF record, a
*candidate* one BAM record fetched for a locus that passed the record filters (main.rs:833-865), a
*pair* a candidate whose cell barcode is in the barcode list (main.rs:867-877) -- the unit that
reaches the aligner (main.rs:896-930).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _capi

MODES = _capi.MODES
NO_CB, NO_UMI = _capi.NO_CB, _capi.NO_UMI


class VtxError(RuntimeError):
    pass


_FIELDS = ("locus_row", "hap_bytes", "ref_off", "ref_len", "alt_off", "alt_len", "cand_start", "read_nib",
           "read_off", "read_len", "cb_bytes", "read_cb_off", "read_cb_len", "read_umi_key", "cand_read")
_DTYPES = dict(locus_row=np.uint32, hap_bytes=np.uint8, ref_off=np.uint32, ref_len=np.uint32, alt_off=np.uint32,
               alt_len=np.uint32, cand_start=np.uint64, read_nib=np.uint8, read_off=np.uint64, read_len=np.uint32,
               cb_bytes=np.uint8, read_cb_off=np.uint32, read_cb_len=np.uint16, read_umi_key=np.uint64,
               cand_read=np.uint32)


@dataclass
class StagedBatch:
    """One shard of loci staged as the SoA `vtx_batch` of include/vartrix_b200.h (numpy, host)."""
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

    FIELDS = _FIELDS

    def __post_init__(self):
        for f in _FIELDS:
            setattr(self, f, np.ascontiguousarray(getattr(self, f), dtype=_DTYPES[f]))

    @classmethod
    def from_fields(cls, src, n_rows=None) -> "StagedBatch":
        """Build from any object/dict exposing the same field names (e.g. the oracle's Batch)."""
        get = (lambda k: src[k]) if isinstance(src, dict) else (lambda k: getattr(src, k))
        nr = n_rows if n_rows is not None else int(src["n_rows"] if isinstance(src, dict) else getattr(src, "n_rows", 0))
        return cls(n_rows=nr, **{f: get(f) for f in _FIELDS})

    @property
    def n_loci(self): return int(self.locus_row.size)
    @property
    def n_reads(self): return int(self.read_len.size)
    @property
    def n_cand(self): return int(self.cand_read.size)

    def nbytes(self) -> int:
        return int(sum(getattr(self, f).nbytes for f in _FIELDS))

    def to_c(self) -> _capi.Batch:
        b = _capi.Batch()
        p = lambda a: a.ctypes.data if a.size else None
        b.n_loci = self.n_loci; b.locus_row = p(self.locus_row)
        b.hap_bytes = p(self.hap_bytes); b.hap_bytes_len = self.hap_bytes.size
        b.ref_off = p(self.ref_off); b.ref_len = p(self.ref_len); b.alt_off = p(self.alt_off); b.alt_len = p(self.alt_len)
        b.cand_start = p(self.cand_start)
        b.n_reads = self.n_reads; b.read_nib = p(self.read_nib); b.read_nib_len = self.read_nib.size
        b.read_off = p(self.read_off); b.read_len = p(self.read_len)
        b.cb_bytes = p(self.cb_bytes); b.cb_bytes_len = self.cb_bytes.size
        b.read_cb_off = p(self.read_cb_off); b.read_cb_len = p(self.read_cb_len); b.read_umi_key = p(self.read_umi_key)
        b.n_cand = self.n_cand; b.cand_read = p(self.cand_read)
        return b

    def shard(self, lo: int, hi: int) -> "StagedBatch":
        """Loci [lo, hi) as a self-contained shard (reads, CB bytes and windows re-packed and re-indexed) --
        what a staging producer emits per chunk, and how loci are sharded across GPUs."""
        cs = self.cand_start
        c0, c1 = int(cs[lo]), int(cs[hi])
        used, inv = np.unique(self.cand_read[c0:c1], return_inverse=True)
        nu = len(used)
        # reads (16-byte aligned)
        rl = self.read_len[used]
        nb = (rl.astype(np.int64) + 1) // 2
        stride = (nb + 15) // 16 * 16
        new_off = np.zeros(nu, np.uint64)
        if nu:
            new_off[1:] = np.cumsum(stride)[:-1].astype(np.uint64)
        n_reads = self.n_reads
        st0 = int(self.read_off[1] - self.read_off[0]) if n_reads > 1 else 0
        uniform = (n_reads > 1 and st0 > 0 and self.read_nib.size == st0 * n_reads and
                   bool((np.diff(self.read_off.astype(np.int64)) == st0).all()) and bool((stride == st0).all()))
        if uniform:
            nib = self.read_nib.reshape(n_reads, st0)[used].reshape(-1)
        else:
            nib = np.zeros(int(stride.sum()) if nu else 0, np.uint8)
            for i, r in enumerate(used):
                o = int(self.read_off[r]); n = int(nb[i])
                nib[int(new_off[i]): int(new_off[i]) + n] = self.read_nib[o:o + n]
        # CB bytes
        cbo = self.read_cb_off[used]; cbl = self.read_cb_len[used].astype(np.int64)
        has = cbo != NO_CB
        new_cbo = np.full(nu, NO_CB, np.uint32)
        L0 = int(cbl[0]) if nu else 0
        if nu and L0 > 0 and bool(has.all()) and bool((cbl == L0).all()) and bool((cbo % L0 == 0).all()) and \
                self.cb_bytes.size % L0 == 0:
            cb = self.cb_bytes.reshape(-1, L0)[cbo // L0].reshape(-1)
            new_cbo = (np.arange(nu, dtype=np.uint32) * np.uint32(L0))
        else:
            tot = int(cbl[has].sum()) if nu else 0
            cb = np.zeros(tot, np.uint8); pos = 0
            for i in np.nonzero(has)[0]:
                n = int(cbl[i]); cb[pos:pos + n] = self.cb_bytes[int(cbo[i]): int(cbo[i]) + n]; new_cbo[i] = pos; pos += n
        # haplotype windows
        nl = hi - lo
        ro, ra = self.ref_off[lo:hi].astype(np.int64), self.alt_off[lo:hi].astype(np.int64)
        rln, aln = self.ref_len[lo:hi].astype(np.int64), self.alt_len[lo:hi].astype(np.int64)
        hs = int(ra[0] - ro[0]) if nl else 0
        if nl and hs > 0 and hs % 16 == 0 and bool((ra - ro == hs).all()) and bool((np.diff(ro) == 2 * hs).all()) and \
                bool((rln <= hs).all()) and bool((aln <= hs).all()) and int(ro[-1]) + 2 * hs <= self.hap_bytes.size:
            hap = self.hap_bytes[int(ro[0]): int(ro[-1]) + 2 * hs].copy()
            n_ro = (np.arange(nl, dtype=np.uint32) * np.uint32(2 * hs)); n_ra = n_ro + np.uint32(hs)
        else:
            pieces, n_ro, n_ra, pos = [], np.zeros(nl, np.uint32), np.zeros(nl, np.uint32), 0
            for i in range(nl):
                for off, ln, dst in ((ro[i], rln[i], n_ro), (ra[i], aln[i], n_ra)):
                    dst[i] = pos; w = np.zeros(int((ln + 15) // 16 * 16), np.uint8)
                    w[:int(ln)] = self.hap_bytes[int(off): int(off + ln)]; pieces.append(w); pos += w.size
            hap = np.concatenate(pieces) if pieces else np.zeros(0, np.uint8)
        return StagedBatch(
            locus_row=self.locus_row[lo:hi].copy(), hap_bytes=hap, ref_off=n_ro, ref_len=self.ref_len[lo:hi].copy(),
            alt_off=n_ra, alt_len=self.alt_len[lo:hi].copy(), cand_start=(cs[lo:hi + 1] - cs[lo]), read_nib=nib,
            read_off=new_off, read_len=rl, cb_bytes=cb, read_cb_off=new_cbo, read_cb_len=self.read_cb_len[used],
            read_umi_key=self.read_umi_key[used], cand_read=inv.astype(np.uint32), n_rows=self.n_rows)


_CB_CODE = np.full(256, 255, np.uint8)
for _i, _b in enumerate(b"ACGT"):
    _CB_CODE[_b] = _i


def pack_cb_keys(cb_bytes: np.ndarray, read_cb_off: np.ndarray, read_cb_len: np.ndarray):
    """vtx_pack_cb over all reads -> (keys u64 [n_reads], exotic tag bytes, exotic offsets u32 [n_exotic + 1]).
    Tags the code cannot express (anything but [ACGT]{1,24}(-N)?) are listed as exotic: key = CB_EXOTIC | index."""
    n = len(read_cb_off)
    keys = np.full(n, _capi.NO_CB_KEY, np.uint64)
    has = read_cb_off != NO_CB
    ex_bytes, ex_off = [], [0]
    lens = read_cb_len.astype(np.int64)
    done = np.zeros(n, bool)
    # fast path: tags of one common length, vectorised (synthetic shards and Cell Ranger BAMs: 16 bases + "-1")
    if has.any():
        L = int(np.bincount(lens[has]).argmax())
        sel = np.nonzero(has & (lens == L))[0]
        if L > 0 and len(sel):
            mat = cb_bytes[read_cb_off[sel].astype(np.int64)[:, None] + np.arange(L)[None, :]]
            code = _CB_CODE[mat]
            nb = np.where((code == 255).any(axis=1), (code == 255).argmax(axis=1), L)          # leading ACGT run
            ok = (nb >= 1) & (nb <= 24)
            suffix = np.zeros(len(sel), np.uint64)
            rest = L - nb
            # suffix forms: none, "-d", "-dd" (no leading zero)
            good = ok & (rest == 0)
            for d in (1, 2):
                cand = ok & (rest == d + 1)
                if not cand.any():
                    continue
                idx = np.nonzero(cand)[0]
                dash = mat[idx, nb[idx]] == ord("-")
                d1 = mat[idx, nb[idx] + 1].astype(np.int64) - 48
                val = d1.copy(); okd = dash & (d1 >= 1) & (d1 <= 9)
                if d == 2:
                    d2 = mat[idx, nb[idx] + 2].astype(np.int64) - 48
                    okd &= (d2 >= 0) & (d2 <= 9); val = d1 * 10 + d2
                suffix[idx[okd]] = val[okd].astype(np.uint64)
                good[idx[okd]] = True
            if good.any():
                g = np.nonzero(good)[0]
                k = np.zeros(len(g), np.uint64)
                cg, nbg = code[g].astype(np.uint64), nb[g]
                for j in range(min(L, 24)):
                    use = j < nbg
                    k = np.where(use, (k << np.uint64(2)) | (cg[:, j] & np.uint64(3)), k)
                keys[sel[g]] = (k << np.uint64(12)) | (nbg.astype(np.uint64) << np.uint64(7)) | suffix[g]
                done[sel[g]] = True
    L_ = _capi.load()
    for r in np.nonzero(has & ~done)[0]:
        o, ln = int(read_cb_off[r]), int(lens[r])
        raw = cb_bytes[o:o + ln].tobytes()
        k = int(L_.vtx_pack_cb(raw, ln))
        if k == _capi.NO_CB_KEY:
            k = _capi.CB_EXOTIC | (len(ex_off) - 1)
            ex_bytes.append(raw); ex_off.append(ex_off[-1] + ln)
        keys[r] = k
    exb = np.frombuffer(b"".join(ex_bytes), np.uint8).copy() if ex_bytes else np.zeros(0, np.uint8)
    return keys, exb, np.asarray(ex_off, np.uint32)


@dataclass
class SlimBatch:
    """The same shard in the slim staging layout `vtx_batch2` (include/vartrix_b200.h): reads packed back to back on
    4-byte boundaries, u16 lengths, one u64 code per cell tag, UMI keys only with --umi, no candidate list when every
    read serves exactly one locus."""
    locus_row: np.ndarray
    hap_bytes: np.ndarray
    ref_off: np.ndarray
    ref_len: np.ndarray
    alt_off: np.ndarray
    alt_len: np.ndarray
    cand_start: np.ndarray
    read_nib: np.ndarray
    read_len: np.ndarray            # u16
    read_cb_key: np.ndarray         # u64
    cb_bytes: np.ndarray            # exotic tags only
    cb_off: np.ndarray              # u32 [n_exotic + 1]
    read_umi_key: np.ndarray        # u64 or None
    cand_read: np.ndarray           # u32 or None (identity)
    n_rows: int = 0

    ARRAYS = ("locus_row", "hap_bytes", "ref_off", "ref_len", "alt_off", "alt_len", "cand_start", "read_nib", "read_len",
              "read_cb_key", "cb_bytes", "cb_off", "read_umi_key", "cand_read")

    @property
    def n_loci(self): return int(self.locus_row.size)
    @property
    def n_reads(self): return int(self.read_len.size)
    @property
    def n_cand(self): return int(self.cand_start[-1]) if self.cand_start.size else 0
    @property
    def n_exotic(self): return int(self.cb_off.size) - 1

    def nbytes(self) -> int:
        return int(sum(getattr(self, f).nbytes for f in self.ARRAYS if getattr(self, f) is not None))

    @staticmethod
    def units(read_len):
        return ((read_len.astype(np.int64) + 1) // 2 + 3) // 4

    @classmethod
    def from_staged(cls, sb: "StagedBatch", umi: bool) -> "SlimBatch":
        assert sb.n_reads == 0 or int(sb.read_len.max()) <= 0xFFFF, "reads longer than 65535 bases need the vtx_batch layout"
        units = cls.units(sb.read_len)
        nb = (sb.read_len.astype(np.int64) + 1) // 2
        n = sb.n_reads
        st0 = int(sb.read_off[1] - sb.read_off[0]) if n > 1 else 0
        uniform = (n > 1 and st0 > 0 and sb.read_nib.size >= st0 * n and bool((np.diff(sb.read_off.astype(np.int64)) == st0).all())
                   and bool((units == units[0]).all()) and int(sb.read_off[0]) == 0)
        if uniform:
            w = int(units[0]) * 4
            nib = np.ascontiguousarray(sb.read_nib[:st0 * n].reshape(n, st0)[:, :w]).copy() if w <= st0 else None
            if nib is not None and w > int(nb[0]):
                nib[:, int(nb[0]):] = 0
        if not uniform or nib is None:
            off = np.zeros(n + 1, np.int64); off[1:] = np.cumsum(units * 4)
            nib = np.zeros(int(off[-1]), np.uint8)
            for r in range(n):
                o = int(sb.read_off[r]); nib[off[r]: off[r] + nb[r]] = sb.read_nib[o:o + nb[r]]
        keys, exb, exo = pack_cb_keys(sb.cb_bytes, sb.read_cb_off, sb.read_cb_len)
        ident = sb.n_cand == n and bool((sb.cand_read == np.arange(n, dtype=np.uint32)).all())
        return cls(sb.locus_row, sb.hap_bytes, sb.ref_off, sb.ref_len, sb.alt_off, sb.alt_len, sb.cand_start,
                   nib.reshape(-1), sb.read_len.astype(np.uint16), keys, exb, exo,
                   np.ascontiguousarray(sb.read_umi_key) if umi else None, None if ident else sb.cand_read, n_rows=sb.n_rows)

    def shard(self, lo: int, hi: int) -> "SlimBatch":
        """Loci [lo, hi) as a self-contained slim shard."""
        cs = self.cand_start
        c0, c1 = int(cs[lo]), int(cs[hi])
        if self.cand_read is None:
            used = np.arange(c0, c1, dtype=np.int64); new_cand = None
        else:
            used, inv = np.unique(self.cand_read[c0:c1], return_inverse=True)
            new_cand = inv.astype(np.uint32)
        units = self.units(self.read_len)
        off = np.zeros(self.n_reads + 1, np.int64); off[1:] = np.cumsum(units * 4)
        if len(used) and int(used[-1]) - int(used[0]) + 1 == len(used):
            nib = self.read_nib[off[used[0]]: off[used[-1] + 1]].copy()          # a contiguous run of reads
        else:
            nib = np.concatenate([self.read_nib[off[r]: off[r + 1]] for r in used]) if len(used) else np.zeros(0, np.uint8)
        keys = self.read_cb_key[used].copy()
        exb, exo = np.zeros(0, np.uint8), np.zeros(1, np.uint32)
        ex = np.nonzero((keys != np.uint64(_capi.NO_CB_KEY)) & ((keys & np.uint64(_capi.CB_EXOTIC)) != 0))[0]
        if len(ex):
            pieces, offs = [], [0]
            for j, r in enumerate(ex):
                i = int(keys[r] & np.uint64(0xFFFFFFFF))
                pieces.append(self.cb_bytes[int(self.cb_off[i]): int(self.cb_off[i + 1])]); offs.append(offs[-1] + len(pieces[-1]))
                keys[r] = np.uint64(_capi.CB_EXOTIC | j)
            exb, exo = np.concatenate(pieces), np.asarray(offs, np.uint32)
        nl = hi - lo
        ro, ra = self.ref_off[lo:hi].astype(np.int64), self.alt_off[lo:hi].astype(np.int64)
        h0 = int(min(ro.min(), ra.min())) if nl else 0
        h1 = int(max((ro + self.ref_len[lo:hi]).max(), (ra + self.alt_len[lo:hi]).max())) if nl else 0
        h1 = (h1 + 15) // 16 * 16
        hap = self.hap_bytes[h0:h1].copy()           # windows of consecutive loci are stored consecutively
        return SlimBatch(self.locus_row[lo:hi].copy(), hap, (ro - h0).astype(np.uint32), self.ref_len[lo:hi].copy(),
                         (ra - h0).astype(np.uint32), self.alt_len[lo:hi].copy(), (cs[lo:hi + 1] - cs[lo]), nib, self.read_len[used].copy(),
                         keys, exb, exo, None if self.read_umi_key is None else self.read_umi_key[used].copy(), new_cand, n_rows=self.n_rows)

    def to_c(self, ptr=None) -> _capi.Batch2:
        """ptr: optional {field: address} of copies of the arrays elsewhere (pinned / device memory)."""
        b = _capi.Batch2()
        def p(f):
            a = getattr(self, f)
            if a is None or a.size == 0:
                return None
            return ptr[f] if ptr is not None else a.ctypes.data
        b.n_loci = self.n_loci; b.locus_row = p("locus_row")
        b.hap_bytes = p("hap_bytes"); b.hap_bytes_len = self.hap_bytes.size
        b.ref_off = p("ref_off"); b.ref_len = p("ref_len"); b.alt_off = p("alt_off"); b.alt_len = p("alt_len")
        b.cand_start = p("cand_start")
        b.n_reads = self.n_reads; b.read_nib = p("read_nib"); b.read_nib_len = self.read_nib.size
        b.read_off4 = None; b.read_len = p("read_len"); b.read_cb_key = p("read_cb_key")
        b.n_exotic_cb = self.n_exotic; b.cb_bytes = p("cb_bytes"); b.cb_off = p("cb_off") if self.n_exotic else None
        b.read_umi_key = p("read_umi_key")
        b.n_cand = self.n_cand; b.cand_read = p("cand_read")
        return b


@dataclass
class Barcodes:
    """De-duplicated barcode list in first-seen order (load_barcodes, main.rs:697-718)."""
    keys: list
    bytes_: np.ndarray = field(default=None)
    off: np.ndarray = field(default=None)

    def __post_init__(self):
        off = np.zeros(len(self.keys) + 1, np.uint32)
        if self.keys:
            off[1:] = np.cumsum([len(k) for k in self.keys])
        self.off = off
        self.bytes_ = (np.frombuffer(b"".join(self.keys), np.uint8).copy() if self.keys else np.zeros(0, np.uint8))

    def __len__(self): return len(self.keys)


@dataclass
class Triplets:
    """Finished (row, col, value) entries in TriMat insertion order (main.rs:320-348)."""
    row: np.ndarray
    col: np.ndarray
    ref_cnt: np.ndarray
    alt_cnt: np.ndarray
    unk_cnt: np.ndarray
    val: np.ndarray
    val2: np.ndarray
    metrics: dict


def _np_from(ptr, n, dt, copy=True):
    if n == 0 or not ptr:
        return np.zeros(0, dt)
    ct = np.ctypeslib.as_ctypes_type(dt)
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(n,))
    return a.copy() if copy else a


def _arr(ptr, count, dtype, shape):
    """a NumPy copy of `count` elements at a library-owned pointer (which the next call of the same kind reuses)"""
    if count == 0:
        return np.zeros(shape, dtype)
    return np.ctypeslib.as_array(ptr, shape=(count,)).astype(dtype, copy=True).reshape(shape)


def _entries(row, col, ref, alt):
    """the count entries (row, col, REF, ALT) as uint32 arrays, and their common length"""
    arrs = [np.ascontiguousarray(x, dtype=np.uint32) for x in (row, col, ref, alt)]
    n = len(arrs[0])
    if any(len(x) != n for x in arrs):
        raise ValueError("row, col, ref and alt must have the same length")
    return arrs, n


def _permille(rho_permille, estimate: bool) -> int:
    """rho_permille as the C ABI takes it: an integer m (thousandths), or with `estimate`, None as -1"""
    if estimate and rho_permille is None:
        return -1
    if isinstance(rho_permille, (bool, np.bool_)) or not isinstance(rho_permille, (int, np.integer)):
        raise TypeError(f"rho_permille must be {'None or ' if estimate else ''}an integer number of thousandths, not {rho_permille!r}")
    return int(rho_permille)


def _clusters_dict(out, restarts: int) -> dict:
    """NumPy copies of a vtx_clusters (library-owned memory that the next clustering call reuses)"""
    nc, nh, nr, kk = int(out.n_cols), int(out.n_hyp), int(out.n_rows), int(out.k)
    return dict(k=kk, n_hyp=nh, best_restart=int(out.best_restart), rows_used=int(out.rows_used),
                ll=_arr(out.ll, nc * nh, np.int64, (nc, nh)), counts=_arr(out.counts, nc * 3, np.uint64, (nc, 3)),
                row_used=_arr(out.row_used, nr, np.uint8, (nr,)), alt_w=_arr(out.alt_w, nr * kk, np.int64, (nr, kk)),
                depth_w=_arr(out.depth_w, nr * kk, np.int64, (nr, kk)),
                restart_score=_arr(out.restart_score, restarts, np.int64, (restarts,)),
                restart_iters=_arr(out.restart_iters, restarts, np.uint32, (restarts,)))


class Engine:
    """One engine context = one GPU (vtx_ctx).  Mirrors the role of the rayon pool + merge loop."""

    def __init__(self, scoring_method: str = "consensus", umi: bool = False, device: int = 0, stream: int = 0,
                 keep_scores: bool = False, min_score: int = 25, no_split: bool = False,
                 values_only: bool = False, no_fold: bool = False, band_k: int = 0, band_w: int = 0, band_mode: int = 0,
                 collapse_mates: bool = False, min_base_quality: int = 0, locus_stats: bool = False):
        """collapse_mates: count each template once per (locus, cell) -- the reads' keys are QNAME keys and go through the
        UMI collapse.  Host batches carry those keys in read_umi_key (the CLI's `--collapse-mates --dump-staged` writes
        them); submit_bam interns the names on the device.  Not combinable with umi=True.
        min_base_quality: submit_bam drops a (read, locus) pair when a base it has at the variant is below this quality
        (`--min-base-quality`, 0..93, 0 = off; bam_metrics()["num_low_base_quality"] counts them).  Host batches carry no
        qualities: the CLI's stager applies the floor to them before they are submitted.
        locus_stats: every submit also sums, per locus, why its row holds what it holds; locus_stats() returns them after
        finish() / finish_device() (vtx_set_locus_stats, include/vartrix_b200.h)."""
        if umi and collapse_mates:
            raise ValueError("collapse_mates replaces the UB keys: it cannot be combined with umi=True")
        if not isinstance(min_base_quality, (int, np.integer)) or not 0 <= min_base_quality <= 93:
            raise ValueError(f"min_base_quality must be an integer in 0..93, not {min_base_quality!r}")
        min_base_quality = int(min_base_quality)
        self._L = _capi.load()
        cfg = _capi.Config(device=device, mode=MODES[scoring_method], use_umi=int(bool(umi or collapse_mates)), match=1, mismatch=-5,
                           gap_open=-5, gap_extend=-1, min_score=min_score, stream=stream or None,
                           flags=(_capi.F_KEEP_SCORES if keep_scores else 0) | (_capi.F_NO_SPLIT if no_split else 0) |
                           (_capi.F_VALUES_ONLY if values_only else 0) | (_capi.F_NO_FOLD if no_fold else 0) |
                           (_capi.F_NAME_KEYS if collapse_mates else 0),
                           band_k=band_k, band_w=band_w, band_mode=band_mode)
        h = C.c_void_p()
        rc = self._L.vtx_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise VtxError(f"vtx_create failed ({rc}): {self._L.vtx_last_error(None).decode()}")
        self._h = h
        self.scoring_method, self.umi, self.device, self.collapse_mates = scoring_method, umi, device, collapse_mates
        self.min_base_quality = min_base_quality
        if min_base_quality:
            self._ck(self._L.vtx_set_min_base_quality(h, min_base_quality), "vtx_set_min_base_quality")
        if locus_stats:
            self._ck(self._L.vtx_set_locus_stats(h, 1), "vtx_set_locus_stats")
        self._keep = []     # host buffers that must outlive the asynchronous copies

    def close(self):
        if getattr(self, "_h", None):
            self._L.vtx_destroy(self._h)
            self._h = None

    def __enter__(self): return self
    def __exit__(self, *a): self.close()
    def __del__(self):
        try: self.close()
        except Exception: pass

    def _ck(self, rc, what):
        if rc != 0:
            raise VtxError(f"{what} failed ({rc}): {self._L.vtx_last_error(self._h).decode()}")

    def set_barcodes(self, bcs: Barcodes):
        self._ck(self._L.vtx_set_barcodes(self._h, bcs.bytes_.ctypes.data if bcs.bytes_.size else None,
                                          bcs.off.ctypes.data, len(bcs)), "vtx_set_barcodes")
        self.n_cols = len(bcs)

    def submit(self, batch: StagedBatch):
        cb = batch.to_c()
        self._keep.append(batch)
        self._ck(self._L.vtx_submit(self._h, C.byref(cb)), "vtx_submit")

    def submit2(self, slim: "SlimBatch"):
        """One shard in the slim staging layout (vtx_submit2)."""
        cb = slim.to_c()
        self._keep.append(slim)
        self._ck(self._L.vtx_submit2(self._h, C.byref(cb)), "vtx_submit2")

    def submit2_device(self, cbatch2: _capi.Batch2, max_read_len: int, max_hap_len: int):
        self._ck(self._L.vtx_submit2_device(self._h, C.byref(cbatch2), max_read_len, max_hap_len), "vtx_submit2_device")

    def submit_device(self, cbatch: _capi.Batch, max_read_len: int, max_hap_len: int):
        self._ck(self._L.vtx_submit_device_ex(self._h, C.byref(cbatch), max_read_len, max_hap_len), "vtx_submit_device_ex")

    def _triplets(self, res: _capi.Result, copy: bool = True) -> Triplets:
        """copy=False returns views of the library-owned pinned arrays (valid until the next engine call)."""
        n = int(res.n)
        m = res.metrics
        return Triplets(_np_from(res.row, n, np.uint32, copy), _np_from(res.col, n, np.uint32, copy),
                        _np_from(res.ref_cnt, n, np.uint32, copy), _np_from(res.alt_cnt, n, np.uint32, copy),
                        _np_from(res.unk_cnt, n, np.uint32, copy), _np_from(res.val, n, np.float64, copy),
                        _np_from(res.val2, n, np.float64, copy),
                        dict(num_not_cell_bc=int(m.num_not_cell_bc), num_non_umi=int(m.num_non_umi), num_scored=int(m.num_scored)))

    def finish(self, copy: bool = True) -> Triplets:
        res = _capi.Result()
        self._ck(self._L.vtx_finish(self._h, C.byref(res)), "vtx_finish")
        self._keep.clear()
        return self._triplets(res, copy)

    def finish_device(self) -> _capi.Result:
        res = _capi.Result()
        self._ck(self._L.vtx_finish_device(self._h, C.byref(res)), "vtx_finish_device")
        self._keep.clear()
        return res

    def sync(self):
        self._ck(self._L.vtx_sync(self._h), "vtx_sync")

    def wait_copies(self):
        """Wait until the host->device copies of every submit so far have landed (vtx_wait_copies): the host arrays of
        those submits may then be overwritten, though their kernels may still be running."""
        self._ck(self._L.vtx_wait_copies(self._h), "vtx_wait_copies")

    def timing(self) -> dict:
        t = _capi.Timing()
        self._ck(self._L.vtx_last_timing(self._h, C.byref(t)), "vtx_last_timing")
        return dict(h2d_ms=t.h2d_ms, prep_ms=t.prep_ms, sw_ms=t.sw_ms, post_ms=t.post_ms, n_pairs=int(t.n_pairs),
                    sw_launches=int(t.sw_launches), total_launches=int(t.total_launches))

    def tile_counts(self) -> list:
        """Warp tiles per SW kernel class of the last submit / score_pairs (classes: see vtx_last_tile_counts)."""
        out = (C.c_uint32 * 16)()
        n = self._L.vtx_last_tile_counts(self._h, out, 16)
        if n < 0:
            self._ck(n, "vtx_last_tile_counts")
        return [int(out[i]) for i in range(n)]

    def run(self, batch: StagedBatch) -> Triplets:
        self.submit(batch)
        return self.finish()

    def score_pairs(self, batch: StagedBatch, pair_read, pair_locus):
        pr = np.ascontiguousarray(pair_read, np.uint32); pl = np.ascontiguousarray(pair_locus, np.uint32)
        rs = np.zeros(len(pr), np.int16); as_ = np.zeros(len(pr), np.int16)
        cb = batch.to_c()
        self._ck(self._L.vtx_score_pairs(self._h, C.byref(cb), len(pr), pr.ctypes.data if len(pr) else None,
                                         pl.ctypes.data if len(pr) else None, rs.ctypes.data if len(pr) else None,
                                         as_.ctypes.data if len(pr) else None), "vtx_score_pairs")
        return rs, as_

    # ---- multi-GPU ------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        L = _capi.load()
        buf = (C.c_uint8 * 128)()
        rc = L.vtx_comm_unique_id(buf)
        if rc != 0:
            raise VtxError(f"vtx_comm_unique_id failed ({rc}): {L.vtx_last_error(None).decode()}")
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, n_ranks: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._ck(self._L.vtx_comm_init(self._h, buf, rank, n_ranks), "vtx_comm_init")

    def gather(self) -> _capi.Result:
        """Allgatherv of every rank's triplets (device-resident on return)."""
        res = _capi.Result()
        self._ck(self._L.vtx_gather(self._h, C.byref(res)), "vtx_gather")
        return res

    def gather_start(self, root: int = _capi.GATHER_ALL):
        """Asynchronous gather (root = rank that receives; GATHER_ALL = allgatherv); later submits overlap it."""
        self._ck(self._L.vtx_gather_start(self._h, root), "vtx_gather_start")

    def gather_wait(self) -> _capi.Result:
        res = _capi.Result()
        self._ck(self._L.vtx_gather_wait(self._h, C.byref(res)), "vtx_gather_wait")
        return res

    def bgzf_inflate(self, members, check_crc: bool = True):
        """members: list of (deflate payload bytes, isize, crc32) of BGZF members -> (list of inflated bytes, status array).
        Raises nothing on corrupt members: inspect the status array (0 = ok)."""
        n = len(members)
        blocks = (_capi.BgzfBlock * max(n, 1))()
        comp = bytearray(); out_len = 0
        for i, (payload, isize, crc) in enumerate(members):
            while len(comp) & 7:
                comp.append(0)
            blocks[i].in_off = len(comp); blocks[i].in_len = len(payload); blocks[i].out_len = isize
            blocks[i].out_off = out_len; blocks[i].crc32 = crc
            comp += payload; out_len += (isize + 7) & ~7
        comp += b"\0" * 16
        cbuf = (C.c_uint8 * len(comp)).from_buffer(comp)
        out = np.zeros(max(out_len, 1), np.uint8)
        status = np.full(max(n, 1), -1, np.int32)
        rc = self._L.vtx_bgzf_inflate(self._h, blocks, n, cbuf, len(comp) - 16, out.ctypes.data, out_len, status.ctypes.data, 1 if check_crc else 0)
        if rc not in (0, -1):
            self._ck(rc, "vtx_bgzf_inflate")
        res = [out[int(blocks[i].out_off): int(blocks[i].out_off) + int(blocks[i].out_len)].tobytes() for i in range(n)]
        return res, status[:n]

    def submit_bam(self, sh: dict, mapq: int = 0, primary_only: bool = False, no_duplicates: bool = False, bam_tag: bytes = b"CB") -> int:
        """vtx_submit_bam on the host's share of a device-staged shard: dict with tid, row, start, end, hap, ref_off, ref_len,
        alt_off, alt_len, members (structured array like vtx_bgzf_block), comp (payload bytes followed by 16 bytes of padding) and
        entry (u64) -- what `vartrix_b200 --gpu-stage --dump-staged` writes.  Returns the ABI code (0, or VTX_E_UNSUPPORTED / VTX_E_INVALID with the message in last_error())."""
        keep = {k: np.ascontiguousarray(sh[k], dt) for k, dt in (("row", np.uint32), ("start", np.int64), ("end", np.int64), ("hap", np.uint8),
                ("ref_off", np.uint32), ("ref_len", np.uint32), ("alt_off", np.uint32), ("alt_len", np.uint32), ("entry", np.uint64))}
        members = np.ascontiguousarray(sh["members"])
        comp = np.frombuffer(bytes(sh["comp"]), np.uint8)              # payloads + the 16 readable bytes behind them, as dumped
        P = lambda a: a.ctypes.data if a.size else None
        b = _capi.BamShard()
        b.n_loci = len(keep["row"]); b.locus_row = P(keep["row"]); b.locus_start = P(keep["start"]); b.locus_end = P(keep["end"])
        b.hap_bytes = P(keep["hap"]); b.hap_bytes_len = keep["hap"].size
        b.ref_off = P(keep["ref_off"]); b.ref_len = P(keep["ref_len"]); b.alt_off = P(keep["alt_off"]); b.alt_len = P(keep["alt_len"])
        b.tid = int(sh["tid"]); b.n_members = len(members); b.members = P(members); b.comp = comp.ctypes.data; b.comp_len = max(0, comp.size - 16)
        b.n_entry = len(keep["entry"]); b.entry_off = P(keep["entry"])
        b.mapq = mapq; b.primary_only = int(primary_only); b.no_duplicates = int(no_duplicates); b.bam_tag = bam_tag[:2]
        rc = self._L.vtx_submit_bam(self._h, C.byref(b))
        self._L.vtx_sync(self._h)                     # the arrays above may go away once this returns
        return rc

    def bam_metrics(self) -> dict:
        m = _capi.BamMetrics()
        self._ck(self._L.vtx_bam_metrics_get(self._h, C.byref(m)), "vtx_bam_metrics_get")
        low_bq = C.c_uint64()
        self._ck(self._L.vtx_bam_low_base_quality(self._h, C.byref(low_bq)), "vtx_bam_low_base_quality")
        return {**{k: int(getattr(m, k)) for k, _ in _capi.BamMetrics._fields_}, "num_low_base_quality": int(low_bq.value)}

    LOCUS_STATS_DTYPE = np.dtype([(f, np.uint32) for f in _capi.LOCUS_STATS_FIELDS])

    def locus_stats(self) -> np.ndarray:
        """One record per locus submitted before the last finish, in submit order (vtx_locus_stats_get): a NumPy structured
        array with the fields of vtx_locus_stats.  Needs Engine(..., locus_stats=True)."""
        p = C.POINTER(_capi.LocusStats)()
        n = C.c_uint64()
        self._ck(self._L.vtx_locus_stats_get(self._h, C.byref(p), C.byref(n)), "vtx_locus_stats_get")
        if n.value == 0:
            return np.zeros(0, self.LOCUS_STATS_DTYPE)
        raw = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint32)), shape=(int(n.value) * len(_capi.LOCUS_STATS_FIELDS),))
        return raw.copy().view(self.LOCUS_STATS_DTYPE)

    def set_donors(self, dosage: np.ndarray, error_rate: float = 0.01):
        """Donor genotypes for per-cell demultiplexing (vtx_set_donors, include/vartrix_b200.h): dosage is uint8[rows, D], the
        ALT dosage 0..2 of donor d at matrix row `row`, or _capi.GT_MISSING; 2 <= D <= 32, 1e-6 <= error_rate <= 0.25.  Before
        the first submit."""
        g = np.ascontiguousarray(dosage, dtype=np.uint8)
        if g.ndim != 2:
            raise ValueError(f"dosage must be a [rows, donors] array, not shape {g.shape}")
        self._ck(self._L.vtx_set_donors(self._h, g.shape[1], g.shape[0], g.ctypes.data if g.size else None, float(error_rate)),
                 "vtx_set_donors")

    def donor_ll(self):
        """-> (ll int64[cols, H] x 2^24 in vtx_set_donors' hypothesis order, counts uint64[cols, 3] = variants, ref, alt),
        summed over the submits before the last finish (vtx_donor_ll_get)."""
        ll, cnt = C.POINTER(C.c_int64)(), C.POINTER(C.c_uint64)()
        n_cols, n_hyp = C.c_uint32(), C.c_uint32()
        self._ck(self._L.vtx_donor_ll_get(self._h, C.byref(ll), C.byref(cnt), C.byref(n_cols), C.byref(n_hyp)), "vtx_donor_ll_get")
        nc, nh = int(n_cols.value), int(n_hyp.value)
        if nc == 0:
            return np.zeros((0, nh), np.int64), np.zeros((0, 3), np.uint64)
        return (np.ctypeslib.as_array(ll, shape=(nc * nh,)).reshape(nc, nh).copy(),
                np.ctypeslib.as_array(cnt, shape=(nc * 3,)).reshape(nc, 3).copy())

    def cluster_cells(self, row, col, ref, alt, n_rows: int, n_cols: int, k: int, restarts: int = 8, seed: int = 0) -> dict:
        """Genotype-free clustering of the cells (vtx_cluster_cells, include/vartrix_b200.h; DESIGN.md §5g): count entries
        (row, col, REF, ALT) strictly ascending by (row, col), e.g. a finished coverage result's row / col / ref_cnt / alt_cnt.
        -> dict of NumPy copies: ll int64[n_cols, H] (x 2^24), counts uint64[n_cols, 3], row_used uint8[n_rows],
        alt_w / depth_w int64[n_rows, k] (x 2^16), restart_score int64[restarts], restart_iters uint32[restarts], and the
        scalars k, n_hyp, best_restart, rows_used."""
        arrs, n = _entries(row, col, ref, alt)
        out = _capi.Clusters()
        p = _capi.ClusterParams(int(k), int(restarts), int(seed) & 0xFFFFFFFFFFFFFFFF)
        ptr = [x.ctypes.data if n else None for x in arrs]
        self._ck(self._L.vtx_cluster_cells(self._h, n, *ptr, int(n_rows), int(n_cols), C.byref(p), C.byref(out)), "vtx_cluster_cells")
        return _clusters_dict(out, int(restarts))

    def cluster_cells_pinned(self, row, col, ref, alt, n_rows: int, n_cols: int, k: int, dosage, rho_permille: int = 0,
                             error_rate: float = 0.01, restarts: int = 8, seed: int = 0) -> dict:
        """Clustering with the first J clusters pinned to known genotypes (vtx_cluster_cells_pinned, include/vartrix_b200.h;
        DESIGN.md §5k): count entries as cluster_cells takes them, dosage uint8[n_rows, J] (0, 1, 2 or GT_MISSING) of the J
        genotyped samples, 1 <= J <= k - 1, and the ambient fraction rho_permille / 1000 (an integer m in 0..500).  -> the dict
        cluster_cells returns; clusters 0 .. J - 1 are the samples in dosage's column order, J .. k - 1 the free clusters."""
        arrs, n = _entries(row, col, ref, alt)
        g = np.ascontiguousarray(dosage, dtype=np.uint8)
        if g.ndim != 2 or g.shape[0] != int(n_rows):
            raise ValueError(f"dosage must be a [n_rows, samples] array, not shape {g.shape}")
        m = _permille(rho_permille, estimate=False)
        out = _capi.Clusters()
        p = _capi.ClusterPinnedParams(int(k), int(restarts), int(seed) & 0xFFFFFFFFFFFFFFFF, g.shape[1], float(error_rate), m)
        ptr = [x.ctypes.data if n else None for x in arrs]
        self._ck(self._L.vtx_cluster_cells_pinned(self._h, n, *ptr, int(n_rows), int(n_cols), g.ctypes.data, C.byref(p), C.byref(out)),
                 "vtx_cluster_cells_pinned")
        return _clusters_dict(out, int(restarts))

    def donors_ambient(self, row, col, ref, alt, n_rows: int, n_cols: int, dosage, error_rate: float = 0.01, rho_permille=None,
                       grid_batch: int = 0) -> dict:
        """Donor assignment against ambient RNA (vtx_donors_ambient, include/vartrix_b200.h; DESIGN.md §5h): count entries as
        cluster_cells takes them and dosage uint8[n_rows, D] as set_donors takes it.  rho_permille=None estimates the ambient
        fraction; an integer m in 0..500 fixes it at m / 1000 (anything else, e.g. the fraction 0.15, raises).  -> dict of NumPy copies: ll int64[n_cols, H] (x 2^24), counts
        uint64[n_cols, 3], grid_permille uint16[E], grid_objective int64[E], grid_calls uint64[E, 3] (ascending m),
        row_alt / row_depth uint64[n_rows], and the scalars rho_permille, rho (= rho_permille / 1000), n_hyp, rows_usable."""
        arrs, n = _entries(row, col, ref, alt)
        g = np.ascontiguousarray(dosage, dtype=np.uint8)
        if g.ndim != 2 or g.shape[0] != int(n_rows):
            raise ValueError(f"dosage must be a [n_rows, donors] array, not shape {g.shape}")
        m = _permille(rho_permille, estimate=True)
        out = _capi.Ambient()
        p = _capi.AmbientParams(g.shape[1], float(error_rate), m, int(grid_batch))
        ptr = [x.ctypes.data if n else None for x in arrs]
        self._ck(self._L.vtx_donors_ambient(self._h, n, *ptr, int(n_rows), int(n_cols), g.ctypes.data if g.size else None,
                                            C.byref(p), C.byref(out)), "vtx_donors_ambient")
        nc, nh, nr, ne = int(out.n_cols), int(out.n_hyp), int(out.n_rows), int(out.n_evaluated)
        return dict(rho_permille=int(out.rho_permille), rho=int(out.rho_permille) / 1000, n_hyp=nh, rows_usable=int(out.rows_usable),
                    ll=_arr(out.ll, nc * nh, np.int64, (nc, nh)), counts=_arr(out.counts, nc * 3, np.uint64, (nc, 3)),
                    grid_permille=_arr(out.grid_permille, ne, np.uint16, (ne,)), grid_objective=_arr(out.grid_objective, ne, np.int64, (ne,)),
                    grid_calls=_arr(out.grid_calls, ne * 3, np.uint64, (ne, 3)), row_alt=_arr(out.row_alt, nr, np.uint64, (nr,)),
                    row_depth=_arr(out.row_depth, nr, np.uint64, (nr,)))

    def cluster_genotypes(self, clusters: dict, row_alt, row_depth, dosage=None, error_rate: float = 0.01, rho_permille=None) -> dict:
        """Genotypes of the clusters against ambient RNA and their match to genotyped samples (vtx_cluster_genotypes,
        include/vartrix_b200.h; DESIGN.md §5i): `clusters` is the dict cluster_cells returns, row_alt / row_depth the pool's
        ALT and REF + ALT sums per row (uint64[n_rows], as donors_ambient returns them), dosage None or uint8[n_rows, S] as
        set_donors takes it.  rho_permille=None estimates the ambient fraction; an integer m in 0..500 fixes it at m / 1000.
        -> dict of NumPy copies: grid_permille uint16[E], grid_objective int64[E] (ascending m), touched uint64[n_touched],
        gt uint8[n_touched, k] (GT_MISSING where no molecule reached the cluster), pl uint32[n_touched, k, 3], match_ll
        int64[k, S] (x 2^24), match_discordant uint64[k, S], match_rows / match_called uint64[k], and the scalars rho_permille,
        rho, rows_fit, rows_compared."""
        A = np.ascontiguousarray(clusters["alt_w"], dtype=np.int64)
        T = np.ascontiguousarray(clusters["depth_w"], dtype=np.int64)
        used = np.ascontiguousarray(clusters["row_used"], dtype=np.uint8)
        if A.ndim != 2 or A.shape != T.shape or used.shape != (A.shape[0],):
            raise ValueError("clusters must hold alt_w / depth_w [n_rows, k] and row_used [n_rows]")
        n_rows, k = A.shape
        ra = np.ascontiguousarray(row_alt, dtype=np.uint64)
        rd = np.ascontiguousarray(row_depth, dtype=np.uint64)
        if ra.shape != (n_rows,) or rd.shape != (n_rows,):
            raise ValueError(f"row_alt and row_depth must have {n_rows} entries")
        g = None
        if dosage is not None:
            g = np.ascontiguousarray(dosage, dtype=np.uint8)
            if g.ndim != 2 or g.shape[0] != n_rows:
                raise ValueError(f"dosage must be a [n_rows, samples] array, not shape {g.shape}")
        s = 0 if g is None else g.shape[1]
        m = _permille(rho_permille, estimate=True)
        out = _capi.ClusterGt()
        p = _capi.ClusterGtParams(k, float(error_rate), m, s)
        ptr = [x.ctypes.data if n_rows else None for x in (A, T, used, ra, rd)]
        self._ck(self._L.vtx_cluster_genotypes(self._h, n_rows, *ptr, g.ctypes.data if g is not None and g.size else None,
                                               C.byref(p), C.byref(out)), "vtx_cluster_genotypes")
        ne, nt = int(out.n_evaluated), int(out.n_touched)
        return dict(rho_permille=int(out.rho_permille), rho=int(out.rho_permille) / 1000, rows_fit=int(out.rows_fit),
                    rows_compared=int(out.rows_compared), grid_permille=_arr(out.grid_permille, ne, np.uint16, (ne,)),
                    grid_objective=_arr(out.grid_objective, ne, np.int64, (ne,)), touched=_arr(out.touched, nt, np.uint64, (nt,)),
                    gt=_arr(out.gt, nt * k, np.uint8, (nt, k)), pl=_arr(out.pl, nt * k * 3, np.uint32, (nt, k, 3)),
                    match_ll=_arr(out.match_ll, k * s, np.int64, (k, s)), match_discordant=_arr(out.match_discordant, k * s, np.uint64, (k, s)),
                    match_rows=_arr(out.match_rows, k, np.uint64, (k,)), match_called=_arr(out.match_called, k, np.uint64, (k,)))

    def cluster_refine(self, row, col, ref, alt, n_rows: int, n_cols: int, clusters: dict, error_rate: float = 0.01,
                       max_rounds: int = 8) -> dict:
        """The cells called against their clusters' fitted genotypes and ambient RNA, with the clusters refit from their singlets
        (vtx_cluster_refine, include/vartrix_b200.h; DESIGN.md §5j): count entries as cluster_cells takes them, and the dict
        cluster_cells returned for them.  -> dict of NumPy copies: ll int64[n_cols, H] (x 2^24) and counts uint64[n_cols, 3] of the
        last round, label uint32[n_cols] (NO_LABEL unless singlet), rho_permille / rows_fit / n_touched / rows_scored / changed
        int64[rounds] and calls int64[rounds, 3] per round, the last round's touched uint64[n_touched], gt uint8[n_touched, k] and
        pl uint32[n_touched, k, 3], and the scalars k, n_hyp, n_rounds, converged."""
        arrs, n = _entries(row, col, ref, alt)
        A = np.ascontiguousarray(clusters["alt_w"], dtype=np.int64)
        T = np.ascontiguousarray(clusters["depth_w"], dtype=np.int64)
        used = np.ascontiguousarray(clusters["row_used"], dtype=np.uint8)
        if A.ndim != 2 or A.shape != T.shape or A.shape[0] != int(n_rows) or used.shape != (int(n_rows),):
            raise ValueError("clusters must hold alt_w / depth_w [n_rows, k] and row_used [n_rows]")
        k = A.shape[1]
        out = _capi.ClusterCalls()
        p = _capi.ClusterCallsParams(k, float(error_rate), int(max_rounds))
        ptr = [x.ctypes.data if n else None for x in arrs] + [x.ctypes.data if int(n_rows) else None for x in (A, T, used)]
        self._ck(self._L.vtx_cluster_refine(self._h, n, *ptr[:4], int(n_rows), int(n_cols), *ptr[4:], C.byref(p), C.byref(out)),
                 "vtx_cluster_refine")
        nc, nh, nt, nr = int(out.n_cols), int(out.n_hyp), int(out.n_touched), int(out.n_rounds)
        rounds = [out.rounds[i] for i in range(nr)]
        return dict(k=k, n_hyp=nh, n_rounds=nr, converged=bool(out.converged),
                    ll=_arr(out.ll, nc * nh, np.int64, (nc, nh)), counts=_arr(out.counts, nc * 3, np.uint64, (nc, 3)),
                    label=_arr(out.label, nc, np.uint32, (nc,)),
                    rho_permille=np.array([x.rho_permille for x in rounds], np.int64),
                    rows_fit=np.array([x.rows_fit for x in rounds], np.int64), n_touched=np.array([x.n_touched for x in rounds], np.int64),
                    rows_scored=np.array([x.rows_scored for x in rounds], np.int64),
                    calls=np.array([list(x.calls) for x in rounds], np.int64).reshape(nr, 3),
                    changed=np.array([x.changed for x in rounds], np.int64),
                    touched=_arr(out.touched, nt, np.uint64, (nt,)), gt=_arr(out.gt, nt * k, np.uint8, (nt, k)),
                    pl=_arr(out.pl, nt * k * 3, np.uint32, (nt, k, 3)))

    def last_error(self) -> str:
        return (self._L.vtx_last_error(self._h) or b"").decode()

    def fetch(self, dev_res: _capi.Result, copy: bool = True) -> Triplets:
        out = _capi.Result()
        self._ck(self._L.vtx_fetch(self._h, C.byref(dev_res), C.byref(out)), "vtx_fetch")
        return self._triplets(out, copy)


def pack_cb(s: bytes) -> int:
    return int(_capi.load().vtx_pack_cb(s, len(s)))


def pack_umi(s: bytes) -> int:
    return int(_capi.load().vtx_pack_umi(s, len(s)))


def shard_bounds(cand_start: np.ndarray, n_shards: int, first_frac: float = 0.0, growth: float = 0.0):
    """Contiguous locus ranges balanced by candidate count (SURVEY.md 8e): -> list of (lo, hi).
    first_frac > 0 makes the first shard that small a fraction of the candidates (a staging producer primes the
    copy/compute pipeline with a small shard so the kernels start early) and balances the rest.
    growth > 1 (with first_frac > 0) sizes the shards geometrically instead -- first_frac, first_frac * growth, ... --
    so that the host->device copy of every shard hides behind the kernels of the one before it (copy time per
    candidate is ~0.7x kernel time, so growth <= 1.4); shards stop growing at 1/n_shards of the total and the number
    of shards follows from that."""
    n_loci = len(cand_start) - 1
    total = int(cand_start[-1])
    targets = []
    if first_frac > 0 and growth > 1.0 and n_shards > 1:
        acc, f, cap = 0.0, first_frac, 1.0 / n_shards
        while acc + f < 1.0 - 1e-9:
            acc += f
            targets.append(int(total * acc))
            f = min(f * growth, cap)
    else:
        for s in range(1, n_shards):
            if first_frac > 0 and n_shards > 1:
                targets.append(int(total * (first_frac + (1.0 - first_frac) * (s - 1) / (n_shards - 1))))
            else:
                targets.append(total * s // n_shards)
    cuts = [0] + [int(np.searchsorted(cand_start, t, side="left")) for t in targets] + [n_loci]
    cuts = [min(max(c, 0), n_loci) for c in cuts]
    for i in range(1, len(cuts)):
        cuts[i] = max(cuts[i], cuts[i - 1])
    return [(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
