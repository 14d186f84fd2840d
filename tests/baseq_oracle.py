"""The CPU oracle with `--min-base-quality`: a (read, locus) pair is dropped when one of its judged bases is below the floor.

`oracle.pipeline` stages the reads exactly as the reference does and is not changed.  This module replays its fetch and
the four record filters (mates_oracle.fetched_records), judges every surviving (record, locus) pair with its own Python
restatement of the rule below, drops the pairs that fail, restages the batch as the host stager would (a read is staged at
its first kept pair) and runs the same C oracle.

Judged bases of a record at the locus [start, end) = [pos, pos + len(REF)), walking the CIGAR from the record's pos:
  M / = / X  the bases aligned to a reference position inside [start, end)
  I          every inserted base, when the reference base right before the insertion lies inside [start, end)
  S H D N P  none
Query positions at or beyond l_seq judge nothing.  A pair without judged bases is kept, and so is a record without
qualities (first quality byte 0xFF)."""
from __future__ import annotations

import numpy as np

from oracle import pipeline as P
import mates_oracle as M

MAX_Q = 93
_CONSUMES_REF = {0: True, 1: False, 2: True, 3: True, 4: False, 5: False, 6: False, 7: True, 8: True}
_CONSUMES_QUERY = {0: True, 1: True, 2: False, 3: False, 4: True, 5: False, 6: False, 7: True, 8: True}


def qualities(bm: "P.Bam", ri: int):
    """The record's quality bytes, or None when they are absent (0xFF)."""
    l_seq = int(bm.l_seq[ri])
    so, _, _ = bm._meta[ri]
    q0 = so + (l_seq + 1) // 2
    q = bm.data[q0:q0 + l_seq]
    if l_seq > 0 and q[0] == 0xFF:
        return None
    return q


def judged_positions(bm: "P.Bam", ri: int, start: int, end: int) -> list:
    """Query positions of the judged bases of record `ri` at the locus [start, end)."""
    ops = [(int(c) & 0xF, int(c) >> 4) for c in bm.cigar(ri)]
    l_seq = int(bm.l_seq[ri])
    ref, query, out = int(bm.pos[ri]), 0, []
    for op, n in ops:
        if op in (0, 7, 8):
            out += [query + k for k in range(n) if start <= ref + k < end]
        elif op == 1 and start <= ref - 1 < end:
            out += [query + k for k in range(n)]
        ref += n if _CONSUMES_REF.get(op, False) else 0
        query += n if _CONSUMES_QUERY.get(op, False) else 0
    return [q for q in out if q < l_seq]


def judged_quals(bm: "P.Bam", ri: int, start: int, end: int):
    """Qualities of the judged bases, in query order; None when the record carries no qualities."""
    q = qualities(bm, ri)
    if q is None:
        return None
    return [int(q[k]) for k in judged_positions(bm, ri, start, end)]


def keeps(bm: "P.Bam", ri: int, start: int, end: int, min_q: int) -> bool:
    if min_q == 0:
        return True
    jq = judged_quals(bm, ri, start, end)
    return jq is None or all(q >= min_q for q in jq)


def check_floor(min_q) -> int:
    if not isinstance(min_q, (int, np.integer)) or isinstance(min_q, bool) or not 0 <= min_q <= MAX_Q:
        raise ValueError(f"--min-base-quality must be an integer from 0 to {MAX_Q}, not {min_q!r}")
    return int(min_q)


def kept_pairs(batch: "P.Batch", vcf: str, bam, min_q: int, **kw):
    """-> (keep mask per candidate of `batch`, BAM record per candidate, the decoded Bam)"""
    recs, bm = M.fetched_records(batch, vcf, bam, **kw)
    vrecs = P.read_vcf(vcf)
    locus = np.repeat(np.arange(batch.n_loci), np.diff(batch.cand_start.astype(np.int64)))
    keep = np.ones(len(recs), bool)
    for c, (ri, l) in enumerate(zip(recs.tolist(), locus.tolist())):
        v = vrecs[int(batch.locus_row[l])]
        keep[c] = keeps(bm, ri, v.pos0, v.pos0 + len(v.alleles[0]), min_q)
    return keep, recs, bm


def restage(batch: "P.Batch", keep: np.ndarray) -> "P.Batch":
    """`batch` without the candidates where keep is False; reads renumbered by their first kept candidate, their bases and
    tags re-packed as the stager packs them."""
    cand_read = batch.cand_read[keep]
    locus = np.repeat(np.arange(batch.n_loci), np.diff(batch.cand_start.astype(np.int64)))[keep]
    cand_start = np.zeros(batch.n_loci + 1, np.uint64)
    cand_start[1:] = np.cumsum(np.bincount(locus, minlength=batch.n_loci))
    new_id, order = {}, []
    for r in cand_read.tolist():
        if r not in new_id:
            new_id[r] = len(order); order.append(r)
    nib, cb = bytearray(), bytearray()
    read_off, read_len, cb_off, cb_len = [], [], [], []
    for r in order:
        while len(nib) % 16: nib.append(0)
        o, n = int(batch.read_off[r]), int(batch.read_len[r])
        read_off.append(len(nib)); read_len.append(n); nib += bytes(batch.read_nib[o:o + (n + 1) // 2])
        co, cn = int(batch.read_cb_off[r]), int(batch.read_cb_len[r])
        if co == P.NO_CB:
            cb_off.append(P.NO_CB); cb_len.append(0)
        else:
            cb_off.append(len(cb)); cb_len.append(cn); cb += bytes(batch.cb_bytes[co:co + cn])
    while len(nib) % 16: nib.append(0)
    umi = batch.read_umi_key[np.asarray(order, np.int64)] if order else np.zeros(0, np.uint64)
    out = P.Batch(batch.locus_row, batch.hap_bytes, batch.ref_off, batch.ref_len, batch.alt_off, batch.alt_len, cand_start,
                  np.frombuffer(bytes(nib), np.uint8).copy(), np.asarray(read_off, np.uint64), np.asarray(read_len, np.uint32),
                  np.frombuffer(bytes(cb), np.uint8).copy(), np.asarray(cb_off, np.uint32), np.asarray(cb_len, np.uint16), umi,
                  np.asarray([new_id[r] for r in cand_read.tolist()], np.uint32), n_rows=batch.n_rows,
                  host_metrics=dict(batch.host_metrics))
    return out.normalized()


def stage_from_files(vcf: str, bam: str, fasta: str, min_base_quality: int = 0, collapse_mates: bool = False, **kw) -> "P.Batch":
    """mates_oracle.stage_from_files, then the base-quality floor; host_metrics gains num_low_base_quality."""
    min_q = check_floor(min_base_quality)
    batch = M.stage_from_files(vcf, bam, fasta, collapse_mates=collapse_mates, **kw)
    if min_q == 0:
        batch.host_metrics["num_low_base_quality"] = 0
        return batch
    keep, _, _ = kept_pairs(batch, vcf, bam, min_q, **kw)
    out = restage(batch, keep)
    out.host_metrics["num_low_base_quality"] = int((~keep).sum())
    return out


def run_files(vcf, bam, fasta, cell_barcodes, scoring_method="consensus", umi=False, collapse_mates=False, min_base_quality=0,
              n_threads=1, **kw):
    """-> (n_rows, n_cols, Result, Batch, Barcodes), like oracle.pipeline.run_files."""
    if umi and collapse_mates:
        raise ValueError("--collapse-mates cannot be combined with --umi")
    bcs = P.load_barcodes(cell_barcodes)
    batch = stage_from_files(vcf, bam, fasta, min_base_quality=min_base_quality, collapse_mates=collapse_mates, **kw)
    res = P.run_batch(batch, bcs, P.MODES[scoring_method], umi or collapse_mates, n_threads)
    return batch.n_rows, len(bcs), res, batch, bcs


def metric_lines(batch: "P.Batch", res: "P.Result", min_base_quality: int) -> list:
    """The CLI's metric log lines (without the "[INFO] " prefix), in its order."""
    m = batch.host_metrics
    lines = [f"Number of alignments evaluated: {m['num_reads']}",
             f"Number of alignments skipped due to low mapping quality: {m['num_low_mapq']}",
             f"Number of alignments skipped due to not being primary: {m['num_non_primary']}",
             f"Number of alignments skipped due to being duplicates: {m['num_duplicates']}",
             f"Number of alignments skipped due to not being associated with a cell barcode: {res.metrics['num_not_cell_bc']}",
             f"Number of alignments skipped due to not intersecting variant: {m['num_not_useful']}"]
    if min_base_quality:
        lines.append(f"Number of alignments skipped due to low base quality at the variant: {m['num_low_base_quality']}")
    lines += [f"Number of alignments skipped due to not having a UMI: {res.metrics['num_non_umi']}",
              f"Number of VCF records skipped due to having invalid characters in the alternative haplotype: {m['num_invalid_recs']}",
              f"Number of VCF records skipped due to being multi-allelic: {m['num_multiallelic_recs']}",
              f"Number of (read, locus) pairs scored on the GPU: {res.metrics['num_scored']}"]
    return lines


def expected(vcf, bam, fasta, cell_barcodes, scoring_method, n_threads=4, **kw):
    """-> (out-matrix text, ref-matrix text or None, metric lines) exactly as the CLI writes and logs them."""
    n_rows, n_cols, res, batch, _ = run_files(vcf, bam, fasta, cell_barcodes, scoring_method, n_threads=n_threads, **kw)
    out = P.mtx_text(n_rows, n_cols, res.row, res.col, res.val)
    ref = P.mtx_text(n_rows, n_cols, res.row, res.col, res.val2) if scoring_method == "coverage" else None
    return out, ref, metric_lines(batch, res, kw.get("min_base_quality", 0))
