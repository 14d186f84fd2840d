"""GPU: `--out-variant-stats` end to end.  The CLI on the reference's DNA and RNA fixtures, on the statistics cases file
(tests/variant_stats_cases.py: a locus emptied by each record filter, nothing fetched, no CB, no UB, a None read, ties, a
disagreeing UMI, mates, multi-allelic / invalid-ALT / empty-ALT records, loci of 1 025 and 2 100 pairs) and on the base-quality
cases file (tests/baseq_cases.py: a UB the device cannot key, a locus emptied by the floor), through host
staging, --gpu-inflate and --gpu-stage, in the three modes, plain / --umi / --collapse-mates, with and without the record
filters and the floor, against the restatement (tests/variant_stats_oracle.py) byte for byte -- and, in the same runs, the
matrices and metric lines against the existing expectations, with the file's invariants checked against the written files.
Also: the host fallback of --gpu-stage, vtx_submit_bam against host-staged shards, the deep-locus ladder through the engine,
the flag off, several GPUs."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import baseq_oracle as B
import variant_stats_oracle as V
from test_host_staging_cpu import _read_vtxd

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR
FIXTURES = {
    "dna": (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv"),
    "rna": (f"{T}/test.vcf", f"{T}/test.bam", f"{T}/test.fa", f"{T}/barcodes.tsv"),
}
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
FILTER_ARGS = ["--mapq", "30", "--primary-alignments", "--no-duplicates", "--min-base-quality", "20"]
FILTER_KW = dict(mapq=30, primary_only=True, no_duplicates=True, min_base_quality=20)


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    import baseq_cases
    p = baseq_cases.write_cases(str(tmp_path_factory.mktemp("vstats")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@pytest.fixture(scope="module")
def vcases(tmp_path_factory):
    import variant_stats_cases
    p = variant_stats_cases.write_cases(str(tmp_path_factory.mktemp("vcases")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected_stats(files, keys, filtered):
    return V.expected_text(*files, **KEYS[keys][1], **(FILTER_KW if filtered else {}))


@functools.lru_cache(maxsize=None)
def _expected_outputs(files, mode, keys, filtered):
    return B.expected(*files, mode, **KEYS[keys][1], **(FILTER_KW if filtered else {}))


def _run(tmp_path, files, mode, *extra, tag="r", stats=True):
    """-> (out text, ref text or None, metric log lines, stats text or None, stderr)"""
    out, ref, st = str(tmp_path / f"{tag}.mtx"), str(tmp_path / f"{tag}_ref.mtx"), str(tmp_path / f"{tag}.tsv")
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", *(["--out-variant-stats", st] if stats else []), *extra],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln[len("[INFO] "):] for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return open(out).read(), (open(ref).read() if mode == "coverage" else None), lines, (open(st).read() if stats else None), r.stderr


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("which", ["dna", "rna", "cases", "vcases"])
def test_cli_matches_oracle(tmp_path, cases, vcases, which, path, keys, filtered):
    files = {"cases": cases, "vcases": vcases}.get(which) or FIXTURES[which]
    if which == "cases" and keys == "umi" and path == "stage":
        pytest.skip("a declined shard: test_gpu_stage_host_fallback")
    want = _expected_stats(files, keys, filtered)
    for mode in ("consensus", "coverage", "alt_frac"):
        out, ref, lines, tsv, _ = _run(tmp_path, files, mode, "--threads", "3", "--shard-loci", "4", *PATHS[path], *KEYS[keys][0],
                                       *(FILTER_ARGS if filtered else []), tag=mode)
        exp_out, exp_ref, exp_lines = _expected_outputs(files, mode, keys, filtered)
        if not filtered:        # the floor's own metric line is logged only with the flag
            exp_lines = [ln for ln in exp_lines if "low base quality" not in ln]
        assert (out, ref, lines) == (exp_out, exp_ref, exp_lines), mode
        assert tsv == want, mode
        V.check_invariants(tsv, keys != "plain", metric_lines=lines, mtx=dict(mode=mode, out=out, ref=ref))


def test_gpu_stage_host_fallback(tmp_path, cases):
    """With --umi, the shard holding a UB outside vtx_pack_umi's alphabet is declined by the device and staged on the host: its
    filter counters come from the host stager, every other shard's from locus_cands -- the same file."""
    *_, tsv, err = _run(tmp_path, cases, "coverage", "--threads", "2", "--shard-loci", "1", "--gpu-stage", "--umi", *FILTER_ARGS)
    assert "1 shard(s) staged on the host after the device declined them" in err
    assert tsv == _expected_stats(cases, "umi", True)


def test_flag_off_changes_nothing(tmp_path, vcases):
    """Without the flag: the same outputs and metric lines, no file, and one kernel launch fewer per shard than with it (the
    per-locus reduction; test_engine_launches_nothing_extra_when_off pins the count per submit)."""
    import re
    for path in ("host", "stage"):
        a = _run(tmp_path, vcases, "coverage", "--threads", "1", "--shard-loci", "3", *PATHS[path], tag=f"{path}_a", stats=False)
        b = _run(tmp_path, vcases, "coverage", "--threads", "1", "--shard-loci", "3", *PATHS[path], tag=f"{path}_b")
        assert a[:3] == b[:3]
        assert not os.path.exists(tmp_path / f"{path}_a.tsv")
        shards = int(re.search(r"GPU\(s\), (\d+) shards", a[4]).group(1))
        la, lb = (int(re.search(r"pairs, (\d+) launches\)", x[4]).group(1)) for x in (a, b))
        assert shards > 3 and lb == la + shards, (la, lb, shards)


def _barcodes(path):
    import vartrix_b200 as vb
    return vb.Barcodes(list(dict.fromkeys(ln.strip().encode() for ln in open(path) if ln.strip())))


def test_engine_launches_nothing_extra_when_off():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(64, 40, depth=25, seed=7, umi=True)
    counts = {}
    for on in (False, True):
        with vb.Engine("coverage", umi=True, locus_stats=on) as e:
            e.set_barcodes(bcs)
            e.submit(sb)
            counts[on] = (e.finish(), e.timing()["total_launches"])
            if on:
                st = e.locus_stats()
    assert counts[True][1] == counts[False][1] + 1
    for f in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt", "unk_cnt"):
        assert np.array_equal(getattr(counts[True][0], f), getattr(counts[False][0], f), equal_nan=True)
    assert len(st) == sb.n_loci and np.array_equal(st["row"], sb.locus_row)


def test_set_locus_stats_after_submit_is_refused():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        e.set_barcodes(bcs)
        assert e._L.vtx_locus_stats_get(e._h, C.byref(C.POINTER(vb._capi.LocusStats)()), C.byref(C.c_uint64())) == -5
        e.submit(sb)
        assert e._L.vtx_set_locus_stats(e._h, 1) == -5 and "before the first submit" in e.last_error()
        e.finish()


@pytest.mark.parametrize("which,shard,umi", [("dna", "7", False), ("rna", "3", True), ("cases", "1", False), ("cases", "1000", False),
                                             ("vcases", "2", False), ("vcases", "1000", True)])
def test_submit_bam_equals_host_staged(tmp_path, cases, vcases, which, shard, umi):
    """vtx_submit_bam's entries = the host-staged vtx_submit entries (whose filter counters are 0) + the restatement's
    per-locus filter counters, for the same shards."""
    import vartrix_b200 as vb
    from vartrix_b200.staged_io import read_dump
    files = {"cases": cases, "vcases": vcases}.get(which) or FIXTURES[which]
    base = [CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "--shard-loci", shard, "--threads", "2", *FILTER_ARGS]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host) and all(d is not None for d in dev)
    bcs = _barcodes(files[3])
    with vb.Engine("coverage", umi=umi, locus_stats=True) as e_host, \
            vb.Engine("coverage", umi=umi, min_base_quality=20, locus_stats=True) as e_dev:
        e_host.set_barcodes(bcs); e_dev.set_barcodes(bcs)
        for d, (hb, _) in zip(dev, host):
            e_host.submit(hb)
            assert e_dev.submit_bam(d, mapq=30, primary_only=True, no_duplicates=True) == 0, e_dev.last_error()
        e_host.finish(); e_dev.finish()
        sh, sd = e_host.locus_stats(), e_dev.locus_stats()
    assert len(sh) == len(sd) > 0 and np.array_equal(sh["row"], sd["row"])
    table = V.stats(*files, umi=umi, **FILTER_KW)
    for i, row in enumerate(sd["row"].tolist()):
        _, n = table[row]
        for f in V.COLUMNS:
            want = n[f]
            assert sd[f][i] == want, (row, f)
            assert sh[f][i] == (0 if f in V.FILTERS else want), (row, f)


def test_deep_loci_ladder():
    """The slot_cases ladder (depths up to 100 000 pairs, runs of 1-pair loci) in coverage mode: every locus's entry against
    NumPy over the finished triplets and the shard's candidates."""
    import slot_cases as S
    import vartrix_b200 as vb
    shard = S.ladder()
    sb = vb.StagedBatch.from_fields(S.fields(shard))
    bcs = vb.Barcodes(S.barcodes())
    for umi in (False, True):
        with vb.Engine("coverage", umi=umi, locus_stats=True) as e:
            e.set_barcodes(bcs)
            e.submit(sb)
            got = e.finish()
            st = e.locus_stats()
        assert len(st) == sb.n_loci and np.array_equal(st["row"], sb.locus_row)
        depth = np.diff(sb.cand_start.astype(np.int64))
        assert (depth > 100_000 - 1).any() and ((depth > 2048) & (depth < 2100)).any()
        lo = np.searchsorted(got.row, sb.locus_row, side="left")
        hi = np.searchsorted(got.row, sb.locus_row, side="right")
        for i in range(sb.n_loci):
            r, a, u = (got.ref_cnt[lo[i]:hi[i]].astype(np.int64), got.alt_cnt[lo[i]:hi[i]].astype(np.int64), got.unk_cnt[lo[i]:hi[i]].astype(np.int64))
            want = dict(calls_ref=r.sum(), calls_alt=a.sum(), calls_unknown=u.sum(), cells=hi[i] - lo[i],
                        cells_ref_only=((r > 0) & (a == 0)).sum(), cells_alt_only=((a > 0) & (r == 0)).sum(),
                        cells_both=((r > 0) & (a > 0)).sum(), cells_multi_unknown=(u > 1).sum())
            for f, v in want.items():
                assert int(st[f][i]) == int(v), (umi, i, int(depth[i]), f)
            assert st["no_cell_barcode"][i] + st["no_umi"][i] + st["scored"][i] == depth[i], (umi, i)
            assert st["scored"][i] == st["reads_ref"][i] + st["reads_alt"][i] + st["reads_unknown"][i] + st["reads_none"][i]
            if not umi:
                assert (st["reads_ref"][i], st["reads_alt"][i], st["reads_unknown"][i]) == (want["calls_ref"], want["calls_alt"], want["calls_unknown"])
        assert int(st["scored"].sum()) == got.metrics["num_scored"] and int(st["no_cell_barcode"].sum()) == got.metrics["num_not_cell_bc"]


def test_two_gpus_equal_one(tmp_path, vcases):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, vcases, "coverage", "--threads", "2", "--shard-loci", "1", *PATHS[path], *FILTER_ARGS, tag=f"one_{path}")
        two = _run(tmp_path, vcases, "coverage", "--threads", "2", "--shard-loci", "1", "--devices", "0,1", *PATHS[path], *FILTER_ARGS,
                   tag=f"two_{path}")
        assert one[:4] == two[:4]
        assert one[3] == _expected_stats(vcases, "plain", True)
