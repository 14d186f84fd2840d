"""GPU: `--min-base-quality` end to end.  The CLI on the reference's DNA and RNA fixtures and on the cases file
(tests/baseq_cases.py), through host staging, --gpu-inflate and --gpu-stage (the floor in the device's locus_cands), in the
three scoring modes, plain, with --umi and with --collapse-mates, against the oracle extension (tests/baseq_oracle.py) --
byte-identical Matrix Market text and metric log lines; vtx_submit_bam against the host-staged shards; the host fallback of
--gpu-stage; repeat runs; a floor of 0; several GPUs."""
import functools
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import baseq_oracle as B
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
FLOOR = {"dna": 26, "rna": 26, "cases": 20}        # the fixtures' binned qualities are 2 / 11 / 25 / 37


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    import baseq_cases
    p = baseq_cases.write_cases(str(tmp_path_factory.mktemp("baseq")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, mode, q, keys):
    return B.expected(*files, mode, min_base_quality=q, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r"):
    """-> (out text, ref text or None, metric log lines, stderr)"""
    out, ref = str(tmp_path / f"{tag}.mtx"), str(tmp_path / f"{tag}_ref.mtx")
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", *extra], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln[len("[INFO] "):] for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return open(out).read(), (open(ref).read() if mode == "coverage" else None), lines, r.stderr


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", ["consensus", "coverage", "alt_frac"])
@pytest.mark.parametrize("which", ["dna", "rna", "cases"])
def test_cli_matches_oracle(tmp_path, cases, which, mode, path, keys):
    files = FIXTURES.get(which, cases)
    q = FLOOR[which]
    out, ref, lines, _ = _run(tmp_path, files, mode, "--threads", "3", "--shard-loci", "4", "--min-base-quality", str(q),
                              *PATHS[path], *KEYS[keys][0])
    assert (out, ref, lines) == _expected(files, mode, q, keys)
    assert any(ln.startswith("Number of alignments skipped due to low base quality at the variant: ") and not ln.endswith(": 0")
               for ln in lines)


def test_the_floor_changes_the_matrices(cases):
    """(else the test above would prove little; on the RNA fixture at 26 only the REF coverage matrix changes)"""
    for which in ("dna", "rna", "cases"):
        files = FIXTURES.get(which, cases)
        assert _expected(files, "coverage", FLOOR[which], "plain")[:2] != _expected(files, "coverage", 0, "plain")[:2], which


@pytest.mark.parametrize("path", list(PATHS))
def test_floor_zero_and_no_flag_are_identical(tmp_path, cases, path):
    """Without the flag, or at 0, the outputs and the metric lines are the plain oracle's, and the new line is not logged."""
    for which in ("dna", "cases"):
        files = FIXTURES.get(which, cases)
        a = _run(tmp_path, files, "coverage", "--threads", "2", *PATHS[path], tag=f"{which}_a")
        b = _run(tmp_path, files, "coverage", "--threads", "2", "--min-base-quality", "0", *PATHS[path], tag=f"{which}_b")
        assert a[:3] == b[:3] == _expected(files, "coverage", 0, "plain")
        assert "low base quality" not in a[3] + b[3]


def test_gpu_stage_host_fallback(tmp_path, cases):
    """With --umi, a shard holding a UB that vtx_pack_umi cannot express is declined by the device and staged on the host:
    the floor and its counter come from the host stager there and from the device everywhere else."""
    out, ref, lines, err = _run(tmp_path, cases, "coverage", "--threads", "2", "--shard-loci", "1", "--gpu-stage", "--umi",
                                "--min-base-quality", "20")
    assert "1 shard(s) staged on the host after the device declined them" in err
    assert (out, ref, lines) == _expected(cases, "coverage", 20, "umi")


def test_repeat_runs_are_identical(tmp_path, cases):
    a = _run(tmp_path, cases, "coverage", "--threads", "3", "--gpu-stage", "--shard-loci", "1", "--min-base-quality", "20", tag="a")
    b = _run(tmp_path, cases, "coverage", "--threads", "3", "--gpu-stage", "--shard-loci", "1", "--min-base-quality", "20", tag="b")
    assert a[:3] == b[:3]


def test_two_gpus_equal_one(tmp_path, cases):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, cases, "coverage", "--threads", "2", "--shard-loci", "1", *PATHS[path], "--min-base-quality", "20", tag=f"one_{path}")
        two = _run(tmp_path, cases, "coverage", "--threads", "2", "--shard-loci", "1", "--devices", "0,1", *PATHS[path],
                   "--min-base-quality", "20", tag=f"two_{path}")
        assert one[:3] == two[:3]


# ---- vtx_submit_bam with a floor ------------------------------------------------------------------------------------------
def _barcodes(path):
    import vartrix_b200 as vb
    return vb.Barcodes(list(dict.fromkeys(ln.strip().encode() for ln in open(path) if ln.strip())))


@pytest.mark.parametrize("which,shard,mode,q", [("dna", "7", "coverage", 26), ("dna", "1000", "consensus", 38), ("rna", "3", "alt_frac", 26),
                                                ("cases", "1", "coverage", 20), ("cases", "1000", "consensus", 25)])
def test_submit_bam_equals_host_staged(tmp_path, cases, which, shard, mode, q):
    """Engine(min_base_quality=q).submit_bam on the host's share of every device-staged shard against the same shards staged on
    the host with the floor: same matrix, same counters (num_low_base_quality against the oracle)."""
    import vartrix_b200 as vb
    from vartrix_b200.staged_io import read_dump
    files = FIXTURES.get(which, cases)
    base = [CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "--shard-loci", shard, "--threads", "2",
            "--min-base-quality", str(q)]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host) and all(d is not None for d in dev)
    bcs = _barcodes(files[3])
    with vb.Engine(mode) as e_host, vb.Engine(mode, min_base_quality=q) as e_dev:
        e_host.set_barcodes(bcs); e_dev.set_barcodes(bcs)
        for d, (hb, _) in zip(dev, host):
            e_host.submit(hb)
            assert e_dev.submit_bam(d) == 0, e_dev.last_error()
        rh, rd = e_host.finish(), e_dev.finish()
        bm = e_dev.bam_metrics()
    for f in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt", "unk_cnt"):
        assert np.array_equal(getattr(rh, f), getattr(rd, f), equal_nan=True), f
    assert rh.metrics == rd.metrics and rh.metrics["num_scored"] > 0
    for k in ("num_reads", "num_low_mapq", "num_non_primary", "num_duplicates", "num_not_useful"):
        assert bm[k] == sum(int(m[k]) for _, m in host), k
    want = B.stage_from_files(*files[:3], min_base_quality=q).host_metrics["num_low_base_quality"]
    assert bm["num_low_base_quality"] == want > 0


def test_set_min_base_quality_refuses_above_93():
    import ctypes as C
    import vartrix_b200 as vb
    with vb.Engine("coverage") as e:
        assert e._L.vtx_set_min_base_quality(e._h, 94) == -1 and "93" in e.last_error()
        assert e._L.vtx_set_min_base_quality(e._h, 93) == 0
        n = C.c_uint64(7)
        assert e._L.vtx_bam_low_base_quality(e._h, C.byref(n)) == 0 and n.value == 0
        assert e.bam_metrics()["num_low_base_quality"] == 0
