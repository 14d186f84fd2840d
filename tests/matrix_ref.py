"""Matrix assembly restated in NumPy (test infrastructure, a third implementation next to the kernels and the C oracle).

What the reference does between the alignments and the matrix (vartrix src/main.rs):
  * get_cell_barcode (737-750): the CB tag looked up in the barcode map, a dict of byte strings.
  * the record loop (867-894): no listed barcode -> num_not_cell_bc; else with --umi and no UB -> num_non_umi;
    every other candidate is scored (num_scored) and pushed, then sorted by cell (932).
  * evaluate_scores (1019-1030), parse_scores (1041-1109): per cell, or per (cell, UMI) with the f64 0.75 rule,
    convert_to_counts, and the mode value of consensus_scoring / alt_frac / coverage (1111-1164).
Written from the reference, not from the kernels: the UMI rule uses the f64 fractions exactly as parse_scores does,
and every count is int64, so nothing here can overflow.  Input scores are one (ref, alt) pair per candidate."""
from types import SimpleNamespace

import numpy as np

NO_CB = 0xFFFFFFFF
NO_UMI = 0xFFFFFFFFFFFFFFFF
MIN_SCORE = 25
CONSENSUS_THRESHOLD = 0.75
NONE, REF, ALT, UNKNOWN = 0, 1, 2, 3          # evaluate_scores: None, REF_VALUE, ALT_VALUE, UNKNOWN_VALUE
MODES = {"consensus": 0, "coverage": 1, "alt_frac": 2}


def evaluate_scores(ref_score, alt_score, min_score=MIN_SCORE):
    """main.rs:1019-1030 over arrays of scores"""
    ref_score, alt_score = np.asarray(ref_score, np.int64), np.asarray(alt_score, np.int64)
    call = np.full(ref_score.shape, UNKNOWN, np.int8)
    call[ref_score > alt_score] = REF
    call[alt_score > ref_score] = ALT
    call[(ref_score < min_score) & (alt_score < min_score)] = NONE
    return call


def barcode_index(barcodes):
    """load_barcodes (main.rs:697-718): tag bytes -> column id; a repeated barcode keeps its first index"""
    index = {}
    for k in barcodes:
        index.setdefault(bytes(k), len(index))
    return index


def _cell_of_read(batch, barcodes):
    """get_cell_barcode for every read: column id, or -1 when the tag is missing or not listed"""
    index = barcodes if isinstance(barcodes, dict) else barcode_index(barcodes)
    off = np.asarray(batch.read_cb_off, np.int64)
    ln = np.asarray(batch.read_cb_len, np.int64)
    col = np.full(off.size, -1, np.int64)
    has = off != NO_CB
    raw = np.asarray(batch.cb_bytes, np.uint8).tobytes()
    tags, inv = np.unique(np.stack([off[has], ln[has]], 1), axis=0, return_inverse=True)
    looked = np.array([index.get(raw[o:o + n], -1) for o, n in tags], np.int64)
    col[has] = looked[inv.reshape(-1)] if tags.size else col[has]
    return col


def _runs(*keys):
    """start of every run of equal key tuples in arrays already sorted by them"""
    n = keys[0].size
    new = np.ones(n, bool)
    if n:
        new[1:] = False
        for k in keys:
            new[1:] |= k[1:] != k[:-1]
    return np.nonzero(new)[0]


def _count(call, starts):
    """convert_to_counts over runs: (ref, alt, unknown) per run, int64"""
    if starts.size == 0:
        z = np.zeros(0, np.int64)
        return z, z, z
    return tuple(np.add.reduceat((call == v).astype(np.int64), starts) for v in (REF, ALT, UNKNOWN))


def assemble(batch, barcodes, mode, umi, ref_score, alt_score, min_score=MIN_SCORE):
    """-> namespace(row, col, ref_cnt, alt_cnt, unk_cnt, val, val2, metrics) in row-major order.
    batch: any object with the staged-batch fields; barcodes: the barcode list, or its barcode_index();
    ref_score / alt_score: one score per candidate."""
    mode = MODES.get(mode, mode)
    cand_start = np.asarray(batch.cand_start, np.int64)
    n_loci = cand_start.size - 1
    cand_read = np.asarray(batch.cand_read, np.int64)
    locus = np.repeat(np.arange(n_loci, dtype=np.int64), np.diff(cand_start))
    col = _cell_of_read(batch, barcodes)[cand_read]
    read_umi = np.asarray(batch.read_umi_key, np.uint64)[cand_read]
    no_cb = col < 0
    no_umi = ~no_cb & (read_umi == np.uint64(NO_UMI)) if umi else np.zeros(col.size, bool)
    keep = ~no_cb & ~no_umi
    metrics = dict(num_not_cell_bc=int(no_cb.sum()), num_non_umi=int(no_umi.sum()), num_scored=int(keep.sum()))

    locus, col = locus[keep], col[keep]
    # a dummy UMI without --umi (main.rs:890-891): then one group per cell
    umik = read_umi[keep] if umi else np.ones(int(keep.sum()), np.uint64)
    call = evaluate_scores(np.asarray(ref_score)[keep], np.asarray(alt_score)[keep], min_score)

    order = np.lexsort((umik, col, locus))
    locus, col, umik, call = locus[order], col[order], umik[order], call[order]
    cells = _runs(locus, col)                      # group_by cell_index, per locus
    if not umi:
        r, a, u = _count(call, cells)
    else:
        groups = _runs(locus, col, umik)
        gr, ga, gu = _count(call, groups)
        t = ga + gr + gu
        seen = t > 0                               # a UMI whose every read is None never enters parsed_scores
        with np.errstate(invalid="ignore", divide="ignore"):
            ref_frac = gr.astype(np.float64) / (ga.astype(np.float64) + gr.astype(np.float64) + gu.astype(np.float64))
            alt_frac = ga.astype(np.float64) / (ga.astype(np.float64) + gr.astype(np.float64) + gu.astype(np.float64))
        collapsed = np.where((ref_frac < CONSENSUS_THRESHOLD) & (alt_frac < CONSENSUS_THRESHOLD), UNKNOWN,
                             np.where(alt_frac >= CONSENSUS_THRESHOLD, ALT, REF))
        assert ((collapsed != REF) | (ref_frac >= CONSENSUS_THRESHOLD) | ~seen).all()
        cell_of_group = np.searchsorted(cells, groups, side="right") - 1
        r, a, u = (np.bincount(cell_of_group[seen & (collapsed == v)], minlength=cells.size).astype(np.int64)
                   for v in (REF, ALT, UNKNOWN))
    c_locus, c_col = locus[cells], col[cells]
    val2 = np.zeros(cells.size, np.float64)
    if mode == 0:                                  # consensus_scoring: cells with neither REF nor ALT are left out
        present = (r > 0) | (a > 0)
        val = np.where((r > 0) & (a > 0), 3.0, np.where(a > 0, 2.0, 1.0))
    elif mode == 2:                                # alt_frac: f64 division, 0 / 0 is NaN
        present = np.ones(cells.size, bool)
        with np.errstate(invalid="ignore"):
            val = a.astype(np.float64) / (r.astype(np.float64) + a.astype(np.float64) + u.astype(np.float64))
    else:                                          # coverage: alt count, ref count
        present = np.ones(cells.size, bool)
        val, val2 = a.astype(np.float64), r.astype(np.float64)
    row = np.asarray(batch.locus_row, np.uint32)[c_locus]
    return SimpleNamespace(row=row[present], col=c_col[present].astype(np.uint32), ref_cnt=r[present],
                           alt_cnt=a[present], unk_cnt=u[present], val=val[present], val2=val2[present],
                           locus=c_locus[present], metrics=metrics)
