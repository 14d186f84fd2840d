"""The CPU restatement of `--out-variant-stats`: one line per VCF record saying why its matrix row holds what it holds.

Independent of the engine's reduction: the fetch, the four record filters and the base-quality floor are replayed per locus
here (the oracle's stager only keeps run-wide counters); the CB / UB gate is applied per candidate of the oracle's staged
batch (tests/baseq_oracle.py, which also carries --collapse-mates' name keys); the pairs are scored with the unchanged C
oracle's `score_pairs` and called with MIN_SCORE (evaluate_scores, main.rs:1019-1030); the reads of one (locus, cell, key)
are collapsed with the 4a >= 3t rule (main.rs:1058-1082).  `expected_text` is the TSV exactly as the CLI writes it."""
from __future__ import annotations

from collections import defaultdict

import numpy as np

from oracle import pipeline as P
import baseq_oracle as B

COLUMNS = ("fetched", "low_mapq", "non_primary", "duplicate", "not_useful", "low_base_quality", "no_cell_barcode", "no_umi",
           "scored", "reads_ref", "reads_alt", "reads_unknown", "reads_none", "calls_ref", "calls_alt", "calls_unknown",
           "cells", "cells_ref_only", "cells_alt_only", "cells_both", "cells_multi_unknown")
HEADER = "\t".join(("variant", "chrom", "pos", "ref", "alt", "status") + COLUMNS) + "\n"
FILTERS = COLUMNS[:6]


def call(rs: int, as_: int, min_score: int = P.MIN_SCORE) -> str:
    if rs < min_score and as_ < min_score:
        return "none"
    return "ref" if rs > as_ else "alt" if as_ > rs else "unknown"


def locus_filters(bm: "P.Bam", rec, mapq=0, primary_only=False, no_duplicates=False, min_base_quality=0) -> dict:
    """fetch + the four filters + the floor for one locus, each record counted once at the first filter that drops it."""
    L = P.lib()
    start, end = rec.pos0, rec.pos0 + len(rec.alleles[0])
    n = dict.fromkeys(FILTERS, 0)
    for ri in bm.fetch(rec.chrom, start, end).tolist():
        n["fetched"] += 1
        fl = int(bm.flag[ri])
        if int(bm.mapq[ri]) < mapq: n["low_mapq"] += 1; continue
        if primary_only and (fl & 0x900): n["non_primary"] += 1; continue
        if no_duplicates and (fl & 0x400): n["duplicate"] += 1; continue
        cig = np.ascontiguousarray(bm.cigar(ri), dtype=np.uint32)
        if not L.vtxo_useful_alignment(int(bm.pos[ri]), cig.ctypes.data if cig.size else None, len(cig), start, end):
            n["not_useful"] += 1; continue
        if not B.keeps(bm, ri, start, end, min_base_quality): n["low_base_quality"] += 1; continue
    return n


def stats(vcf, bam, fasta, cell_barcodes, umi=False, collapse_mates=False, min_base_quality=0, mapq=0, primary_only=False,
          no_duplicates=False, **kw) -> list:
    """-> one (status, {column: count}) per VCF record, in row order."""
    recs = P.read_vcf(vcf)
    bm = P.Bam(bam)
    bcs = P.load_barcodes(cell_barcodes)
    col_of = {k: i for i, k in enumerate(bcs.keys)}
    flt = dict(mapq=mapq, primary_only=primary_only, no_duplicates=no_duplicates)
    batch = B.stage_from_files(vcf, bam, fasta, min_base_quality=min_base_quality, collapse_mates=collapse_mates, **flt, **kw)
    keyed = umi or collapse_mates
    out = [("multiallelic" if len(r.alleles) > 2 else "invalid_alt", dict.fromkeys(COLUMNS, 0)) for r in recs]
    # the CB / UB gate per candidate (main.rs:867-894)
    pair_read, pair_locus, pair_col, pair_key = [], [], [], []
    gate = np.zeros((batch.n_loci, 2), np.int64)
    for l in range(batch.n_loci):
        for c in range(int(batch.cand_start[l]), int(batch.cand_start[l + 1])):
            r = int(batch.cand_read[c])
            o, n = int(batch.read_cb_off[r]), int(batch.read_cb_len[r])
            col = -1 if o == P.NO_CB else col_of.get(bytes(batch.cb_bytes[o:o + n]), -1)
            if col < 0:
                gate[l, 0] += 1
            elif keyed and int(batch.read_umi_key[r]) == P.NO_UMI:
                gate[l, 1] += 1
            else:
                pair_read.append(r); pair_locus.append(l); pair_col.append(col); pair_key.append(int(batch.read_umi_key[r]))
    rs, as_ = P.score_pairs(batch, np.asarray(pair_read, np.uint32), np.asarray(pair_locus, np.uint32), n_threads=4) \
        if pair_read else (np.zeros(0, np.int32), np.zeros(0, np.int32))
    calls_of = defaultdict(list)                 # locus -> [(col, key, call)]
    for l, col, key, a, b in zip(pair_locus, pair_col, pair_key, rs.tolist(), as_.tolist()):
        calls_of[l].append((col, key, call(a, b)))
    for l, row in enumerate(batch.locus_row.tolist()):
        n = dict.fromkeys(COLUMNS, 0)
        n.update(locus_filters(bm, recs[row], min_base_quality=min_base_quality, **flt))
        n["no_cell_barcode"], n["no_umi"] = int(gate[l, 0]), int(gate[l, 1])
        pairs = calls_of.get(l, [])
        n["scored"] = len(pairs)
        for _, _, c in pairs:
            n[f"reads_{c}"] += 1
        cells = defaultdict(list)
        for col, key, c in pairs:
            cells[col].append((key, c))
        for col, items in cells.items():
            cnt = dict(ref=0, alt=0, unknown=0)
            if keyed:
                by_key = defaultdict(list)
                for key, c in items:
                    by_key[key].append(c)
                for cs in by_key.values():
                    r_, a_, u_ = cs.count("ref"), cs.count("alt"), cs.count("unknown")
                    t = r_ + a_ + u_
                    if t == 0:
                        continue
                    cnt["alt" if 4 * a_ >= 3 * t else "ref" if 4 * r_ >= 3 * t else "unknown"] += 1
            else:
                for _, c in items:
                    if c != "none":
                        cnt[c] += 1
            for k, v in cnt.items():
                n[f"calls_{k}"] += v
            n["cells"] += 1
            n["cells_ref_only"] += cnt["ref"] > 0 and cnt["alt"] == 0
            n["cells_alt_only"] += cnt["alt"] > 0 and cnt["ref"] == 0
            n["cells_both"] += cnt["ref"] > 0 and cnt["alt"] > 0
            n["cells_multi_unknown"] += cnt["unknown"] > 1
        out[row] = ("scored", {k: int(v) for k, v in n.items()})
    return out


def text(vcf, table) -> str:
    lines = [HEADER]
    for rec, (status, n) in zip(P.read_vcf(vcf), table):
        alt = b",".join(rec.alleles[1:]) if len(rec.alleles) > 1 else b"."
        lines.append("\t".join([f"{rec.chrom}_{rec.pos0}", rec.chrom, str(rec.pos0 + 1), rec.alleles[0].decode(), alt.decode(), status] +
                               [str(n[c]) for c in COLUMNS]) + "\n")
    return "".join(lines)


def expected_text(vcf, bam, fasta, cell_barcodes, **kw) -> str:
    return text(vcf, stats(vcf, bam, fasta, cell_barcodes, **kw))


def parse(tsv: str) -> list:
    """The written file -> [(variant, status, {column: count})] in row order."""
    lines = tsv.splitlines()
    assert lines[0] + "\n" == HEADER, lines[0]
    out = []
    for ln in lines[1:]:
        f = ln.split("\t")
        out.append((f[0], f[5], {c: int(v) for c, v in zip(COLUMNS, f[6:])}))
    return out


def check_invariants(tsv: str, keyed: bool, metric_lines: list = None, mtx: dict = None, n_rows: int = None):
    """The per-row invariants of the file itself.  metric_lines: the CLI's "Number of ..." lines (column sums);
    mtx: {"mode": ..., "out": text, "ref": text or None} to check the rows against the written matrices."""
    rows = parse(tsv)
    if n_rows is not None:
        assert len(rows) == n_rows
    for variant, status, n in rows:
        assert n["fetched"] == sum(n[c] for c in ("low_mapq", "non_primary", "duplicate", "not_useful", "low_base_quality",
                                                   "no_cell_barcode", "no_umi", "scored")), variant
        assert n["scored"] == n["reads_ref"] + n["reads_alt"] + n["reads_unknown"] + n["reads_none"], variant
        if not keyed:
            assert (n["calls_ref"], n["calls_alt"], n["calls_unknown"]) == (n["reads_ref"], n["reads_alt"], n["reads_unknown"]), variant
        else:
            assert n["calls_ref"] + n["calls_alt"] + n["calls_unknown"] <= n["scored"] - n["reads_none"], variant
        assert n["cells_ref_only"] + n["cells_alt_only"] + n["cells_both"] <= n["cells"] <= n["scored"], variant
        if status != "scored":
            assert all(v == 0 for v in n.values()), variant
    if metric_lines is not None:
        total = {c: sum(n[c] for _, _, n in rows) for c in COLUMNS}
        want = {"Number of alignments evaluated": "fetched",
                "Number of alignments skipped due to low mapping quality": "low_mapq",
                "Number of alignments skipped due to not being primary": "non_primary",
                "Number of alignments skipped due to being duplicates": "duplicate",
                "Number of alignments skipped due to not being associated with a cell barcode": "no_cell_barcode",
                "Number of alignments skipped due to not intersecting variant": "not_useful",
                "Number of alignments skipped due to low base quality at the variant": "low_base_quality",
                "Number of alignments skipped due to not having a UMI": "no_umi",
                "Number of (read, locus) pairs scored on the GPU": "scored"}
        seen = set()
        for ln in metric_lines:
            name, _, v = ln.rpartition(": ")
            if name in want:
                assert total[want[name]] == int(v), ln
                seen.add(want[name])
            elif name.startswith("Number of VCF records skipped due to having invalid"):
                assert sum(s == "invalid_alt" for _, s, _ in rows) == int(v), ln
            elif name.startswith("Number of VCF records skipped due to being multi-allelic"):
                assert sum(s == "multiallelic" for _, s, _ in rows) == int(v), ln
        if "low_base_quality" not in seen:
            assert total["low_base_quality"] == 0
    if mtx is not None:
        out = _mtx_rows(mtx["out"])
        if mtx["mode"] == "coverage":
            ref = _mtx_rows(mtx["ref"])
            for k, (_, _, n) in enumerate(rows):
                assert len(out.get(k, [])) == n["cells"], k
                assert sum(out.get(k, [])) == n["calls_alt"] and sum(ref.get(k, [])) == n["calls_ref"], k
        elif mtx["mode"] == "consensus":
            for k, (_, _, n) in enumerate(rows):
                vals = out.get(k, [])
                assert (vals.count(1.0), vals.count(2.0), vals.count(3.0)) == (n["cells_ref_only"], n["cells_alt_only"], n["cells_both"]), k
                assert len(vals) == n["cells_ref_only"] + n["cells_alt_only"] + n["cells_both"], k
    return rows


def _mtx_rows(txt: str) -> dict:
    rows = defaultdict(list)
    for ln in txt.splitlines()[3:]:
        r, _, v = ln.split()
        rows[int(r) - 1].append(float(v))
    return rows
