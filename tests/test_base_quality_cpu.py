"""`--min-base-quality` without a GPU: the oracle's judged-base restatement against the hand-written expectations of the cases
file (tests/baseq_cases.py), the host stager (`--dump-staged`, host inflate and the `--gpu-inflate` bulk path) against the
oracle, the shared decision body run serially (tests/baseq_shim.cpp) against the restatement, and the refusals."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import baseq_oracle as B
from test_host_staging_cpu import _same_staging

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR
FIXTURES = {
    "dna": (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv"),
    "rna": (f"{T}/test.vcf", f"{T}/test.bam", f"{T}/test.fa", f"{T}/barcodes.tsv"),
}
FLOORS = [1, 12, 25, 26, 37, 38]          # around the fixtures' binned qualities 2 / 11 / 25 / 37


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    import baseq_cases
    return baseq_cases.write_cases(str(tmp_path_factory.mktemp("baseq")))


def _files(which, cases):
    return FIXTURES[which] if which in FIXTURES else (cases["vcf"], cases["bam"], cases["fasta"], cases["barcodes"])


def _pairs(files):
    """every fetched (record, locus) pair of the file: -> (decoded Bam, records, starts, ends)"""
    from oracle import pipeline as P
    bm = P.Bam(files[1])
    recs, starts, ends = [], [], []
    for v in P.read_vcf(files[0]):
        s, e = v.pos0, v.pos0 + len(v.alleles[0])
        for ri in bm.fetch(v.chrom, s, e).tolist():
            recs.append(ri); starts.append(s); ends.append(e)
    return bm, np.asarray(recs, np.int64), np.asarray(starts, np.int64), np.asarray(ends, np.int64)


def test_restatement_matches_hand_written_cases(cases):
    """Every fetched pair of the cases file: the oracle's judged qualities are the ones written down beside the read."""
    from oracle import pipeline as P
    import mates_oracle as M
    bm, recs, starts, ends = _pairs(_files("cases", cases))
    assert len(recs) > 2100
    for ri, s, e in zip(recs.tolist(), starts.tolist(), ends.tolist()):
        want = cases["judged"][(M.qname(bm, ri), int(bm.flag[ri]))][s]
        assert B.judged_quals(bm, ri, s, e) == want, (M.qname(bm, ri), s)
    # the floors the cases are built around
    keep = lambda name, locus, q: B.keeps(bm, next(r for r in recs.tolist() if M.qname(bm, r) == name), locus,
                                         locus + {3000: 3, 3500: 3, 4000: 4}.get(locus, 1), q)
    assert [keep(b"site_q%d" % v, 1000, 20) for v in (19, 20, 21)] == [False, True, True]
    assert keep(b"q0", 2000, 1) is False and keep(b"q93", 2000, 93) is True and keep(b"noqual", 2500, 93) is True
    assert keep(b"del_whole", 4000, 93) is True and keep(b"del_ref_low", 4000, 5) is False and keep(b"del_alt_after_low", 4000, 20) is True
    assert keep(b"ins_mid_low", 5000, 20) is False and keep(b"ins_anchor_low", 5000, 20) is False and keep(b"ins_after_low", 5000, 20) is True
    assert keep(b"ins_far", 5500, 20) is True and keep(b"ins_before", 5500, 20) is True and keep(b"skip", 6000, 93) is True
    assert keep(b"mnp_clip", 3000, 20) is True and keep(b"mnp_clip_low", 3000, 20) is False and keep(b"mnp_mid_low", 3500, 20) is False
    assert keep(b"two_low_first", 7000, 20) is False and keep(b"two_low_first", 7010, 20) is True
    assert keep(b"near_low", 1500, 20) is True


def test_oracle_floor_zero_is_the_plain_oracle():
    from oracle import pipeline as P
    a, b = B.stage_from_files(*FIXTURES["dna"][:3]), P.stage_from_files(*FIXTURES["dna"][:3])
    for f in P.Batch.FIELDS:
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.host_metrics == dict(b.host_metrics, num_low_base_quality=0)


def _dump_file(tmp_path, files, *extra, tag="d"):
    out = tmp_path / f"{tag}.staged"
    subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "--dump-staged", str(out), *extra],
                   check=True, cwd=str(tmp_path))
    return out


def _dump(tmp_path, files, *extra, tag="d"):
    from vartrix_b200.staged_io import read_dump
    return read_dump(str(_dump_file(tmp_path, files, *extra, tag=tag)))[2]


@pytest.mark.parametrize("q", FLOORS)
@pytest.mark.parametrize("path", ["host", "inflate"])
@pytest.mark.parametrize("which", ["dna", "rna", "cases"])
def test_dump_staged_matches_oracle(tmp_path, cases, which, path, q):
    """The staged candidate lists, reads and counters of every shard equal the oracle's restaged batch."""
    files = _files(which, cases)
    n = 5
    extra = ["--gpu-inflate"] if path == "inflate" else []
    shards = _dump(tmp_path, files, "--shard-loci", str(n), "--threads", "3", "--min-base-quality", str(q), *extra)
    dropped = 0
    for k, (sb, met) in enumerate(shards):
        ob = B.stage_from_files(*files[:3], min_base_quality=q, rec_lo=n * k, rec_hi=n * k + n)
        _same_staging(sb, ob)
        assert met == {m: ob.host_metrics[m] for m in met}
        dropped += ob.host_metrics["num_low_base_quality"]
    if which == "cases" or q >= 26:
        assert dropped > 0


def test_dump_staged_with_umi_and_mates(tmp_path, cases):
    files = _files("cases", cases)
    for extra, kw in ((["--umi"], {}), (["--collapse-mates"], dict(collapse_mates=True))):
        shards = _dump(tmp_path, files, "--shard-loci", "4", "--threads", "2", "--min-base-quality", "20", *extra, tag=extra[0][2:])
        for k, (sb, met) in enumerate(shards):
            _same_staging(sb, B.stage_from_files(*files[:3], min_base_quality=20, rec_lo=4 * k, rec_hi=4 * k + 4, **kw))


@pytest.mark.parametrize("extra", [[], ["--gpu-inflate"], ["--gpu-stage"], ["--umi", "--threads", "2", "--shard-loci", "3"]])
def test_floor_zero_dump_is_byte_identical(tmp_path, cases, extra):
    for which in ("dna", "cases"):
        files = _files(which, cases)
        a = _dump_file(tmp_path, files, *extra, tag=f"{which}_plain")
        b = _dump_file(tmp_path, files, *extra, "--min-base-quality", "0", tag=f"{which}_zero")
        assert open(a, "rb").read() == open(b, "rb").read()


# ---- the shared decision body on the CPU ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bq_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bqshim") / "libbaseq_shim.so")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, "-o", so, os.path.join(ROOT, "tests", "baseq_shim.cpp")], check=True)
    return ctypes.CDLL(so)


@pytest.mark.parametrize("which", ["dna", "rna", "cases"])
def test_shared_body_equals_restatement(bq_shim, cases, which):
    """base_quality_ok -- the body locus_cands and the host stager call -- on every fetched (record, locus) pair of the file, at
    every floor from 0 to 93, against the Python restatement."""
    bm, recs, starts, ends = _pairs(_files(which, cases))
    data = np.frombuffer(bm.data, np.uint8)
    offs = np.ascontiguousarray(bm.rec_off[recs], np.uint64)
    jq = [B.judged_quals(bm, ri, s, e) for ri, s, e in zip(recs.tolist(), starts.tolist(), ends.tolist())]
    lowest = np.array([99 if j is None else min(j, default=99) for j in jq])
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    n_diff = 0
    for q in range(0, 94):
        keep = np.zeros(len(recs), np.uint8)
        assert bq_shim.vtx_test_base_quality(P(data), ctypes.c_uint64(len(recs)), P(offs), P(starts), P(ends), ctypes.c_uint32(q), P(keep)) == 0
        want = (lowest >= q) | (q == 0)
        assert np.array_equal(keep.astype(bool), want), (q, np.nonzero(keep.astype(bool) != want)[0][:5])
        n_diff += int((~want).sum())
    assert n_diff > 0


# ---- refusals --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", ["-1", "94", "abc", "", "2.5", "20x"])
def test_cli_refuses_bad_floors(tmp_path, value):
    f = FIXTURES["dna"]
    r = subprocess.run([CLI, "-v", f[0], "-b", f[1], "-f", f[2], "-c", f[3], "-o", str(tmp_path / "o.mtx"), "--min-base-quality", value],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 1 and "--min-base-quality" in r.stderr and "0 to 93" in r.stderr
    assert os.listdir(tmp_path) == []


def test_help_lists_the_flag():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert "--min-base-quality" in r.stdout


def test_engine_and_oracle_refuse_bad_floors():
    import vartrix_b200 as vb
    for bad in (-1, 94, 2.5, "20"):
        with pytest.raises(ValueError):
            vb.Engine("coverage", min_base_quality=bad)
        with pytest.raises(ValueError):
            B.stage_from_files(*FIXTURES["dna"][:3], min_base_quality=bad)
