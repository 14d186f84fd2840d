"""GPU: `--collapse-mates` end to end.  The CLI on the reference's DNA and RNA fixtures and on a paired-end file built for the
flag (tests/mates_cases.py), through host staging, --gpu-inflate and --gpu-stage (device QNAME interning), against the oracle
with the same flag -- byte-identical Matrix Market text; vtx_submit_bam with VTX_F_NAME_KEYS against the host-staged shards,
up to one shard of more than a million used records; repeat runs; several GPUs."""
import functools
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import mates_oracle as M
from test_host_staging_cpu import _read_vtxd

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR
FIXTURES = {
    "dna": (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv"),
    "rna": (f"{T}/test.vcf", f"{T}/test.bam", f"{T}/test.fa", f"{T}/barcodes.tsv"),
}
PATHS = {"host": [], "inflate": ["--gpu-inflate", "--shard-loci", "9"], "stage": ["--gpu-stage", "--shard-loci", "9"]}
RNA_GOLDEN = {"consensus": ("test_consensus.mtx", None), "alt_frac": ("test_frac.mtx", None),
              "coverage": ("test_coverage.mtx", "test_coverage_ref.mtx")}


@functools.lru_cache(maxsize=None)
def _expected(files, mode, extra_kw=()):
    return M.mtx_texts(*files, mode, collapse_mates=True, n_threads=4, **dict(extra_kw))


def _run(tmp_path, files, mode, *extra, tag="r"):
    out, ref = str(tmp_path / f"{tag}.mtx"), str(tmp_path / f"{tag}_ref.mtx")
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--collapse-mates", "--log-level", "info", *extra], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "staged on the host after the device declined" not in r.stderr
    assert "not having a UMI: 0" in r.stderr
    return open(out).read(), (open(ref).read() if mode == "coverage" else None)


@pytest.mark.parametrize("threads", ["1", "3"])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", ["consensus", "coverage", "alt_frac"])
@pytest.mark.parametrize("pre", ["dna", "rna"])
def test_reference_fixtures(tmp_path, pre, mode, path, threads):
    files = FIXTURES[pre]
    got = _run(tmp_path, files, mode, "--threads", threads, *PATHS[path])
    assert got == _expected(files, mode)
    if pre == "rna":          # unpaired: one record per name, so the non-UMI goldens of the reference come out
        from test_gpu_ref_cli import read_mtx
        gold_out, gold_ref = RNA_GOLDEN[mode]
        assert read_mtx(str(tmp_path / "r.mtx")) == read_mtx(f"{T}/{gold_out}")
        if gold_ref:
            assert read_mtx(str(tmp_path / "r_ref.mtx")) == read_mtx(f"{T}/{gold_ref}")


@pytest.fixture(scope="module")
def paired(tmp_path_factory):
    import mates_cases
    p = mates_cases.write_paired(str(tmp_path_factory.mktemp("paired")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@pytest.mark.parametrize("filters", [False, True])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", ["consensus", "coverage", "alt_frac"])
def test_paired_file(tmp_path, paired, mode, path, filters):
    extra = ["--mapq", "10", "--no-duplicates", "--primary-alignments"] if filters else []
    kw = (("mapq", 10), ("no_duplicates", True), ("primary_only", True)) if filters else ()
    got = _run(tmp_path, paired, mode, "--threads", "3", "--shard-loci", "2", *PATHS[path][:1], *extra)
    assert got == _expected(paired, mode, kw)
    assert got[0].count("\n") > 20


def test_paired_file_collapses_something(paired):
    """the flag changes this file's matrices (else the test above would prove little)"""
    from oracle import pipeline as P
    n_rows, n_cols, res, _, _ = P.run_files(*paired, "coverage")
    assert P.mtx_text(n_rows, n_cols, res.row, res.col, res.val) != _expected(paired, "coverage")[0]


def test_repeat_runs_are_identical(tmp_path, paired):
    a = _run(tmp_path, paired, "coverage", "--threads", "3", "--gpu-stage", "--shard-loci", "1", tag="a")
    b = _run(tmp_path, paired, "coverage", "--threads", "3", "--gpu-stage", "--shard-loci", "1", tag="b")
    assert a == b


def test_two_gpus_equal_one(tmp_path, paired):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, paired, "coverage", "--threads", "2", "--shard-loci", "1", *PATHS[path][:1], tag=f"one_{path}")
        two = _run(tmp_path, paired, "coverage", "--threads", "2", "--shard-loci", "1", "--devices", "0,1", *PATHS[path][:1], tag=f"two_{path}")
        assert one == two


# ---- vtx_submit_bam with VTX_F_NAME_KEYS --------------------------------------------------------------------------------
def _dumps(tmp_path, files, shard, extra=()):
    from vartrix_b200.staged_io import read_dump
    base = [CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "--shard-loci", shard, "--threads", "2",
            "--collapse-mates", *extra]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host) and all(d is not None for d in dev)
    return dev, host


def _barcodes(path):
    import vartrix_b200 as vb
    return vb.Barcodes(list(dict.fromkeys(ln.strip().encode() for ln in open(path) if ln.strip())))


def _submit_bam_vs_host(dev, host, bcs, mode, **kw):
    import vartrix_b200 as vb
    with vb.Engine(mode, collapse_mates=True) as e_host, vb.Engine(mode, collapse_mates=True) as e_dev:
        e_host.set_barcodes(bcs); e_dev.set_barcodes(bcs)
        for d, (hb, _) in zip(dev, host):
            e_host.submit(hb)
            assert e_dev.submit_bam(d, **kw) == 0, e_dev.last_error()
        rh, rd = e_host.finish(), e_dev.finish()
    for f in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt", "unk_cnt"):
        assert np.array_equal(getattr(rh, f), getattr(rd, f), equal_nan=True), f
    assert rh.metrics == rd.metrics and rh.metrics["num_non_umi"] == 0 and rh.metrics["num_scored"] > 0
    return rh


@pytest.mark.parametrize("which,shard,mode", [("dna", "7", "coverage"), ("dna", "1000", "consensus"), ("paired", "1", "alt_frac"),
                                              ("paired", "1000", "coverage")])
def test_submit_bam_name_keys_equal_host_staged(tmp_path, paired, which, shard, mode):
    files = FIXTURES["dna"] if which == "dna" else paired
    dev, host = _dumps(tmp_path, files, shard)
    _submit_bam_vs_host(dev, host, _barcodes(files[3]), mode)


def test_submit_bam_needs_use_umi_for_name_keys():
    import ctypes as C
    from vartrix_b200 import _capi
    L = _capi.load()
    cfg = _capi.Config(device=0, mode=1, use_umi=0, match=1, mismatch=-5, gap_open=-5, gap_extend=-1, min_score=25,
                       flags=_capi.F_NAME_KEYS)
    h = C.c_void_p()
    assert L.vtx_create(C.byref(cfg), C.byref(h)) == -1 and b"use_umi" in L.vtx_last_error(None)


def test_submit_bam_name_keys_on_a_million_records(tmp_path):
    """one shard with more than a million used records (unique names): the device table at scale; the collapsed matrix then
    equals the one without any keys"""
    import vartrix_b200 as vb
    from vartrix_b200 import synth_files
    p = synth_files.write_dataset_fast(str(tmp_path / "big"), n_loci=11_000, n_barcodes=2_000, depth=100, read_len=100, spacing=400, seed=4)
    files = (p["vcf"], p["bam"], p["fasta"], p["barcodes"])
    dev, host = _dumps(tmp_path, files, "1000000")
    assert len(dev) == 1 and host[0][0].n_reads >= 1_000_000
    rh = _submit_bam_vs_host(dev, host, _barcodes(files[3]), "coverage")
    with vb.Engine("coverage") as e:
        e.set_barcodes(_barcodes(files[3]))
        e.submit(host[0][0])
        plain = e.finish()
    for f in ("row", "col", "val", "val2"):
        assert np.array_equal(getattr(rh, f), getattr(plain, f)), f
