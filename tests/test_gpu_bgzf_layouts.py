"""GPU: the CLI on one record stream written in many BGZF layouts (tests/bgzf_layouts.py) -- records split across members at every
field, members of a few bytes, empty members, (k, ISIZE_k) index offsets, members from other compressors -- through host staging,
--gpu-inflate and --gpu-stage, in all three modes, with and without --umi.  The matrices, label files and metric lines must be
byte-identical to the oracle (which inflates the whole file with zlib and fetches without the index), the device path must take
every shard, and vtx_submit_bam on the dumped device shards must equal the host-staged shards, filter counters included."""
import os
import subprocess

import numpy as np
import pytest

from bgzf_layouts import LAYOUTS, dataset, write_layout
from conftest import ROOT
from test_host_staging_cpu import _read_vtxd

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
SHARD = "9"          # small shards: their compressed ranges begin and end inside split records
FILTERS = ["--mapq", "30", "--primary-alignments", "--no-duplicates"]
FILTER_KW = dict(mapq=30, primary_only=True, no_duplicates=True)
COUNTERS = ("num_reads", "num_low_mapq", "num_non_primary", "num_duplicates", "num_not_useful")
# (mode, --umi, record filters on)
MODES = [(m, u, False) for m in ("consensus", "coverage", "alt_frac") for u in (False, True)] + [("coverage", True, True), ("alt_frac", False, True)]


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_layouts")
    ds = dataset(str(d))
    ds["bams"] = {}
    for lay in LAYOUTS:
        path = str(d / f"{lay}.bam")
        write_layout(path, ds["refs"], ds["recs"], lay, seed=LAYOUTS.index(lay) + 1)
        ds["bams"][lay] = path
    return ds


@pytest.fixture(scope="module")
def expected(oracle, data):
    """the oracle's outputs per (mode, umi, filters): they do not depend on the layout"""
    out = {}
    for mode, umi, filtered in MODES:
        n_rows, n_cols, res, batch, bcs = oracle.run_files(data["vcf"], data["bams"]["whole"], data["fasta"], data["barcodes"], mode, umi, n_threads=8,
                                                           **(FILTER_KW if filtered else {}))
        if filtered:
            assert all(batch.host_metrics[c] > 0 for c in COUNTERS), batch.host_metrics
        out[(mode, umi, filtered)] = dict(
            out=oracle.mtx_text(n_rows, n_cols, res.row, res.col, res.val),
            ref=oracle.mtx_text(n_rows, n_cols, res.row, res.col, res.val2) if mode == "coverage" else None,
            metrics=[f"Number of alignments evaluated: {batch.host_metrics['num_reads']}",
                     f"not being associated with a cell barcode: {res.metrics['num_not_cell_bc']}",
                     f"not having a UMI: {res.metrics['num_non_umi']}"],
            n=len(res.row))
    return out


@pytest.mark.parametrize("path", ["host", "gpu_inflate", "gpu_stage"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_cli_byte_identical_to_oracle(data, expected, tmp_path, layout, path):
    extra = {"host": [], "gpu_inflate": ["--gpu-inflate"], "gpu_stage": ["--gpu-stage"]}[path]
    for mode, umi, filtered in MODES:
        d = tmp_path / f"{mode}_{int(umi)}_{int(filtered)}"; d.mkdir()
        cmd = [CLI, "-v", data["vcf"], "-b", data["bams"][layout], "-f", data["fasta"], "-c", data["barcodes"], "-o", str(d / "out.mtx"),
               "--ref-matrix", str(d / "ref.mtx"), "-s", mode, "--log-level", "info", "--shard-loci", SHARD, "--threads", "3", *extra]
        cmd += (["--umi"] if umi else []) + (FILTERS if filtered else [])
        r = subprocess.run(cmd, cwd=str(d), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        e = expected[(mode, umi, filtered)]
        assert open(d / "out.mtx").read() == e["out"], (mode, umi, filtered)
        if e["ref"] is not None:
            assert open(d / "ref.mtx").read() == e["ref"], (mode, umi, filtered)
        for line in e["metrics"]:
            assert line in r.stderr, (mode, umi, filtered, line)
        assert "declined them" not in r.stderr                      # the device path took every shard
        assert e["n"] > 100


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_submit_bam_equals_host_staged_shards(data, tmp_path, layout, filtered):
    import vartrix_b200 as vb
    from vartrix_b200.staged_io import read_dump
    base = [CLI, "-v", data["vcf"], "-b", data["bams"][layout], "-f", data["fasta"], "-c", data["barcodes"], "--shard-loci", SHARD,
            "--threads", "2", "--umi", *(FILTERS if filtered else [])]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host) and all(d is not None for d in dev)
    b = vb.Barcodes([ln.strip().encode() for ln in open(data["barcodes"]) if ln.strip()])
    with vb.Engine("coverage", umi=True) as e_host, vb.Engine("coverage", umi=True) as e_dev:
        e_host.set_barcodes(b); e_dev.set_barcodes(b)
        for d, (hb, _) in zip(dev, host):
            e_host.submit(hb)
            assert e_dev.submit_bam(d, **(FILTER_KW if filtered else {})) == 0, e_dev.last_error()
        rh, rd = e_host.finish(), e_dev.finish()
        for f in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt", "unk_cnt"):
            assert np.array_equal(getattr(rh, f), getattr(rd, f), equal_nan=True), f
        assert rh.metrics == rd.metrics and rh.metrics["num_scored"] > 0
        bm = e_dev.bam_metrics()
    for k in COUNTERS:
        assert bm[k] == sum(int(m[k]) for _, m in host), k
    assert bm["num_reads"] > 2000 and bm["num_not_useful"] > 0
    if filtered:
        assert all(bm[k] > 0 for k in COUNTERS), bm                 # every filter rejects records, on both sides
