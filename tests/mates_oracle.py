"""The CPU oracle with `--collapse-mates`: reads keyed by QNAME and collapsed by the UMI rule (main.rs:1047-1082).

`oracle.pipeline` stages the reads exactly as the reference does; this module only replaces each staged read's UB key with
a key of its record's QNAME (the read-name bytes without the NUL; "*" = no name, a key of its own) and runs the same C
oracle, which already collapses by key.  Without collapse_mates everything is delegated unchanged."""
from __future__ import annotations

import numpy as np

from oracle import pipeline as P


def qname(bm: "P.Bam", i: int) -> bytes:
    o = int(bm.rec_off[i])
    l_rn = bm.data[o + 8]
    return bytes(bm.data[o + 32: o + 32 + max(l_rn - 1, 0)])


def fetched_records(batch: "P.Batch", vcf: str, bam, mapq: int = 0, primary_only: bool = False, no_duplicates: bool = False,
                    **_ignored):
    """BAM record index of every candidate of `batch` (locus-major, file order): the fetch and the four record filters of
    main.rs:822-865 replayed over the staged loci.  -> (records int64 [n_cand], the decoded Bam)."""
    recs = P.read_vcf(vcf)
    bm = bam if isinstance(bam, P.Bam) else P.Bam(bam)
    L = P.lib()
    out = []
    for row in batch.locus_row.tolist():
        rec = recs[row]
        start = rec.pos0; end = start + len(rec.alleles[0])
        for ri in bm.fetch(rec.chrom, start, end).tolist():
            fl = int(bm.flag[ri])
            if int(bm.mapq[ri]) < mapq: continue
            if primary_only and (fl & 0x900): continue
            if no_duplicates and (fl & 0x400): continue
            cig = np.ascontiguousarray(bm.cigar(ri), dtype=np.uint32)
            if not L.vtxo_useful_alignment(int(bm.pos[ri]), cig.ctypes.data if cig.size else None, len(cig), start, end):
                continue
            out.append(ri)
    out = np.asarray(out, np.int64)
    assert len(out) == batch.n_cand
    return out, bm


def name_keys(names) -> np.ndarray:
    """One key per name, equal exactly for equal names; every b"*" gets a key of its own."""
    keys, seen = np.zeros(len(names), np.uint64), {}
    for i, n in enumerate(names):
        keys[i] = i if n == b"*" else seen.setdefault(n, i)
    return keys


def stage_from_files(vcf: str, bam: str, fasta: str, collapse_mates: bool = False, **kw) -> "P.Batch":
    batch = P.stage_from_files(vcf, bam, fasta, **kw)
    if not collapse_mates:
        return batch
    recs, bm = fetched_records(batch, vcf, bam, **kw)
    rec_of_read = np.full(batch.n_reads, -1, np.int64)
    rec_of_read[batch.cand_read] = recs
    assert (rec_of_read >= 0).all()
    for c, r in enumerate(batch.cand_read.tolist()):            # one staged read per record
        assert rec_of_read[r] == recs[c]
    batch.read_umi_key = name_keys([qname(bm, int(ri)) for ri in rec_of_read])
    return batch.normalized()


def run_files(vcf, bam, fasta, cell_barcodes, scoring_method="consensus", umi=False, collapse_mates=False, n_threads=1, **kw):
    """oracle.pipeline.run_files with `collapse_mates`: -> (n_rows, n_cols, Result, Batch, Barcodes)."""
    if umi and collapse_mates:
        raise ValueError("--collapse-mates cannot be combined with --umi")
    bcs = P.load_barcodes(cell_barcodes)
    batch = stage_from_files(vcf, bam, fasta, collapse_mates=collapse_mates, **kw)
    res = P.run_batch(batch, bcs, P.MODES[scoring_method], umi or collapse_mates, n_threads)
    return batch.n_rows, len(bcs), res, batch, bcs


def mtx_texts(vcf, bam, fasta, cell_barcodes, scoring_method, **kw):
    """-> (out-matrix text, ref-matrix text or None) exactly as the CLI writes them."""
    n_rows, n_cols, res, _, _ = run_files(vcf, bam, fasta, cell_barcodes, scoring_method, **kw)
    out = P.mtx_text(n_rows, n_cols, res.row, res.col, res.val)
    ref = P.mtx_text(n_rows, n_cols, res.row, res.col, res.val2) if scoring_method == "coverage" else None
    return out, ref
