"""GPU: `--out-cluster-genotypes` / `--out-cluster-matches` end to end and the engine's post-pass (vtx_cluster_genotypes).

The CLI on a seeded pool with 15 % ambient RNA and two decoy sample columns (tests/cluster_gt_cases.py) through host staging,
--gpu-inflate and --gpu-stage, plain / --umi / --collapse-mates, in the three modes, at default shards and at --shard-loci 4
--threads 3: both files equal the restatement (tests/cluster_gt_oracle.py) byte for byte, and the matrices, metric lines and
the clusters / alleles files equal a run without the flags.  Engine level: K = 2, 17, 32 and S = 0, 1, 33, 1024, fixed and
estimated, twice in a row; a seam ladder of fitted and compared rows and sample chunks; a sparse touch of a 5 M-row table; every
refusal's code."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import cluster_gt_cases as GC
import cluster_gt_oracle as O
import cluster_oracle as CO

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
SHARDS = {"default": [], "small": ["--shard-loci", "4", "--threads", "3"]}
MODES = ("consensus", "coverage", "alt_frac")


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = GC.write_pool(str(tmp_path_factory.mktemp("cgpool")), 0.15)
    return (p["vcf_match"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys):
    return O.expected(*files, 6, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r", gt=False):
    """-> (out text, ref text or None, metric lines, clusters text, alleles text, genotypes text, matches text, stderr)"""
    out, ref, cl, al, g, m = (str(tmp_path / f"{tag}{s}") for s in (".mtx", "_ref.mtx", "_cl.tsv", "_al.tsv", "_gt.vcf", "_m.tsv"))
    opt = ["--out-cluster-genotypes", g, "--out-cluster-matches", m] if gt else []
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", "--out-clusters", cl, "--clusters", "6", "--out-cluster-alleles", al, *opt, *extra],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of") or ln.startswith("[INFO] Clusters:")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(cl).read(), open(al).read(),
            open(g).read() if gt else None, open(m).read() if gt else None, r.stderr)


def _check_info(stderr, res, n_rows):
    m = re.search(r"Cluster genotypes: ambient RNA (\S+) \(estimated, (\d+) fractions evaluated\); rows fit: (\d+); touched rows: (\d+) of "
                  r"(\d+); genotypes called at GQ >= 20: (\d+); assignments: (\S+)", stderr)
    assert m, stderr
    g = m.groups()
    assert g[0] == f"{res['rho_permille'] / 1000:.3f}" and int(g[1]) == len(res["grid_permille"])
    assert (int(g[2]), int(g[3]), int(g[4])) == (res["rows_fit"], res["touched"].size, n_rows)
    assert int(g[5]) == int((O.gq(res["pl"]) >= O.MIN_GQ).sum())
    assert g[6].count("=") == res["gt"].shape[1]


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cli_matches_restatement(tmp_path, pool, path, keys):
    want_g, want_m, res, _ = _expected(pool, keys)
    for shard, sargs in SHARDS.items():
        common = [*sargs, *PATHS[path], *KEYS[keys][0]]
        for mode in MODES:
            base = _run(tmp_path, pool, mode, *common, tag=f"off_{shard}_{mode}")
            assert "Cluster genotypes" not in base[7]
            got = _run(tmp_path, pool, mode, *common, tag=f"on_{shard}_{mode}", gt=True)
            assert got[5] == want_g and got[6] == want_m, (shard, mode)
            assert got[:5] == base[:5], (shard, mode)
            _check_info(got[7], res, len(O.records(pool[0])))


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], tag=f"one_{path}", gt=True)
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], tag=f"two_{path}", gt=True)
        assert one[:7] == two[:7]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _synthetic(n_rows, k, s, seed, reach=0.7):
    """clusters dict (alt_w / depth_w x 2^16 of 0-40 molecules, a quarter of the (row, cluster) pairs empty, rows no cluster
    reaches), row sums, and dosage [n_rows, s] (None for s = 0) with missing values"""
    rng = np.random.default_rng(seed)
    T = rng.integers(0, 40 << 16, (n_rows, k))
    T[rng.random((n_rows, k)) < 0.25] = 0
    T[rng.random(n_rows) > reach] = 0
    A = (T * rng.beta(0.7, 0.7, (n_rows, k))).astype(np.int64)
    used = (rng.random(n_rows) < 0.6).astype(np.uint8)
    rd = rng.integers(0, 5000, n_rows).astype(np.uint64)
    ra = (rd * rng.random(n_rows)).astype(np.uint64)
    g = None
    if s:
        g = rng.integers(0, 3, (n_rows, s)).astype(np.uint8)
        g[rng.random((n_rows, s)) < 0.3 / s] = 0xFF
    return dict(alt_w=A, depth_w=T.astype(np.int64), row_used=used), ra, rd, g


def _same(got, want):
    for f in ("rho_permille", "rows_fit", "rows_compared"):
        assert got[f] == want[f], f
    for f in ("grid_permille", "grid_objective", "touched", "gt", "pl", "match_ll", "match_discordant", "match_rows", "match_called"):
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


@pytest.mark.parametrize("rho", [None, 0, 230, 500])
@pytest.mark.parametrize("s", [0, 1, 33, 1024])
@pytest.mark.parametrize("k", [2, 17, 32])
def test_engine_equals_restatement(k, s, rho):
    import vartrix_b200 as vb
    n_rows = 3000 if s < 1024 else 1200
    cl, ra, rd, g = _synthetic(n_rows, k, s, seed=k * 7 + s)
    eps = {2: 1e-6, 17: 0.01, 32: 0.25}[k]
    want = O.genotypes(cl, ra, rd, g, eps, rho)
    with vb.Engine("coverage") as e:
        got = e.cluster_genotypes(cl, ra, rd, g, eps, rho)
        again = e.cluster_genotypes(cl, ra, rd, g, eps, rho)
    _same(got, want)
    _same(again, got)
    assert got["rho"] == got["rho_permille"] / 1000
    if rho is not None:
        assert got["grid_permille"].tolist() == [rho]
    if s:
        assert got["match_called"].sum() > 0 and got["rows_compared"] > 0


def test_seam_ladder_equals_numpy():
    """fitted and compared rows 1, 31, 32, 33 and 2 049 (the match's 32-row tiles); S = 63, 64, 65, 129 (its 64-sample CTA
    columns) at K = 32 (8 pairs per thread) and K = 5"""
    import vartrix_b200 as vb
    with vb.Engine("coverage") as e:
        for n in (1, 31, 32, 33, 2049):
            for k, s in ((32, 63), (32, 64), (5, 65), (32, 129)):
                cl, ra, rd, g = _synthetic(n, k, s, seed=n + s, reach=1.0)
                cl["row_used"][:] = 1
                cl["depth_w"][:, 0] = np.maximum(cl["depth_w"][:, 0], 1 << 16)      # every row reached, fitted and compared
                g[g == 0xFF] = 1
                _same(e.cluster_genotypes(cl, ra, rd, g, 0.01, None), O.genotypes(cl, ra, rd, g, 0.01, None))


def test_sparse_touch_of_a_large_table():
    """a 5 M-row table of which 3 000 rows are reached, some of them at rows a sample has no genotype"""
    import vartrix_b200 as vb
    rng = np.random.default_rng(11)
    n_rows, k, s = 5_000_000, 4, 16
    rows = np.sort(rng.choice(n_rows, 3000, replace=False))
    small, ra_s, rd_s, g_s = _synthetic(3000, k, s, seed=5, reach=1.0)
    cl = dict(alt_w=np.zeros((n_rows, k), np.int64), depth_w=np.zeros((n_rows, k), np.int64), row_used=np.zeros(n_rows, np.uint8))
    for f in cl:
        cl[f][rows] = small[f]
    ra, rd = np.zeros(n_rows, np.uint64), np.zeros(n_rows, np.uint64)
    ra[rows], rd[rows] = ra_s, rd_s
    g = rng.integers(0, 3, (n_rows, s)).astype(np.uint8)
    g[rows] = g_s
    want = O.genotypes(cl, ra, rd, g, 0.01, None)
    with vb.Engine("coverage") as e:
        got = e.cluster_genotypes(cl, ra, rd, g, 0.01, None)
    _same(got, want)
    assert 0 < got["touched"].size <= 3000 and got["rows_compared"] > n_rows - 3000


def test_refusals_return_their_codes():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    cl, ra, rd, g = _synthetic(50, 3, 4, seed=1)
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        L, h = e._L, e._h
        out = _capi.ClusterGt()

        def call(A=cl["alt_w"], T=cl["depth_w"], used=cl["row_used"], ra=ra, rd=rd, dosage=g, k=3, s=4, eps=0.01, rho=-1, n_rows=50):
            p = _capi.ClusterGtParams(k, eps, rho, s)
            return L.vtx_cluster_genotypes(h, n_rows, A.ctypes.data, T.ctypes.data, used.ctypes.data, ra.ctypes.data, rd.ctypes.data,
                                           None if dosage is None else dosage.ctypes.data, C.byref(p), C.byref(out))
        assert call() == 0 and call(dosage=None, s=0) == 0
        for kw in (dict(k=1), dict(k=33), dict(s=1025), dict(dosage=None), dict(eps=0.0), dict(eps=0.3), dict(eps=float("nan")),
                   dict(rho=-2), dict(rho=501)):
            assert call(**kw) == -1, kw
        assert call(rho=500) == 0 and call(rho=0) == 0
        bad = cl["alt_w"].copy(); bad[3, 1] = -1
        assert call(A=bad) == -1 and "alt_w" in e.last_error()
        bad = cl["alt_w"].copy(); bad[3, 1] = cl["depth_w"][3, 1] + 1
        assert call(A=bad) == -1
        deep = cl["depth_w"].copy(); deep[4, 0] = (1 << 51) + 1
        assert call(T=deep) == -1 and "2^51" in e.last_error()
        deep = np.zeros_like(cl["depth_w"]); deep[:2, 0] = 1 << 51           # each at the bound, their sum above it
        z = np.zeros_like(cl["alt_w"])
        assert call(A=z, T=deep) == -1 and "sums" in e.last_error()
        deep[1, 0] = 0
        assert call(A=z, T=deep) == 0
        bad = ra.copy(); bad[5] = rd[5] + 1
        assert call(ra=bad) == -1 and "row_alt" in e.last_error()
        big = rd.copy(); big[6] = (1 << 53) - 2
        assert call(rd=big) == -1
        big[6] = (1 << 53) - 3
        assert call(rd=big) == 0
        bad = g.copy(); bad[7, 1] = 3
        assert call(dosage=bad) == -1 and "dosage" in e.last_error()
        with pytest.raises(TypeError):                          # the Python call takes thousandths, not a fraction
            e.cluster_genotypes(cl, ra, rd, g, 0.01, 0.15)
        e.set_barcodes(bcs)
        e.submit(sb)
        assert call() == -5
        e.finish()
        assert call() == 0
