"""GPU: `--out-cluster-calls` end to end and the engine's post-pass (vtx_cluster_refine).

The CLI on a seeded pool with 15 % ambient RNA (tests/cluster_gt_cases.py) through host staging, --gpu-inflate and --gpu-stage,
plain / --umi / --collapse-mates, in the three modes, at default shards and at --shard-loci 4 --threads 3: the file equals the
restatement (tests/cluster_refine_oracle.py) byte for byte, and the matrices, metric lines and the clusters, alleles, genotypes
and matches files equal a run without the flag.  Engine level: K = 2, 17, 32 at max_rounds 0, 1 and 8, twice in a row; round 0's
fit against vtx_cluster_genotypes; a seam ladder of scored rows, cells and entries; rows where every code is P; a cluster that
no cell is labelled with; a sparse touch of a 5 M-row table; every refusal's code."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import cluster_gt_cases as GC
import cluster_gt_oracle as GO
import cluster_refine_cases as RC
import cluster_refine_oracle as O

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
SHARDS = {"default": [], "small": ["--shard-loci", "4", "--threads", "3"]}
MODES = ("consensus", "coverage", "alt_frac")
FIELDS = ("ll", "counts", "label", "rho_permille", "rows_fit", "n_touched", "rows_scored", "calls", "changed", "touched", "gt", "pl")


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = GC.write_pool(str(tmp_path_factory.mktemp("crpool")), 0.15)
    return (p["vcf_match"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys):
    return O.expected(*files, 6, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r", calls=False):
    """-> (out, ref or None, metric lines, clusters, alleles, genotypes, matches, calls or None, stderr)"""
    names = ("o.mtx", "ref.mtx", "cl.tsv", "al.tsv", "gt.vcf", "m.tsv", "calls.tsv")
    out, ref, cl, al, g, m, cc = (str(tmp_path / f"{tag}_{s}") for s in names)
    opt = ["--out-cluster-calls", cc] if calls else []
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", "--out-clusters", cl, "--clusters", "6", "--out-cluster-alleles", al,
                        "--out-cluster-genotypes", g, "--out-cluster-matches", m, *opt, *extra], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of") or ln.startswith("[INFO] Clusters:")
             or ln.startswith("[INFO] Cluster genotypes:")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(cl).read(), open(al).read(), open(g).read(),
            open(m).read(), open(cc).read() if calls else None, r.stderr)


def _check_info(stderr, genotypes_vcf, res, n_rows):
    m = re.search(r"Cluster calls: ambient RNA per round (\S+); rounds: (\d+) \((converged|hit the cap)\); scored rows: (\d+) of (\d+); "
                  r"cells: (\d+) singlet, (\d+) doublet, (\d+) unassigned", stderr)
    assert m, stderr
    g = m.groups()
    assert g[0] == ",".join(f"{x / 1000:.3f}" for x in res["rho_permille"].tolist())
    assert int(g[1]) == res["n_rounds"] and (g[2] == "converged") == res["converged"]
    assert (int(g[3]), int(g[4])) == (res["rows_scored"][-1], n_rows)
    assert [int(x) for x in g[5:]] == res["calls"][-1].tolist()
    assert f"##vartrix_ambient_rna={g[0].split(',')[0]}\n" in genotypes_vcf        # round 0 is --out-cluster-genotypes' fit


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cli_matches_restatement(tmp_path, pool, path, keys):
    want, res, _ = _expected(pool, keys)
    for shard, sargs in SHARDS.items():
        common = [*sargs, *PATHS[path], *KEYS[keys][0]]
        for mode in MODES:
            base = _run(tmp_path, pool, mode, *common, tag=f"off_{shard}_{mode}")
            assert "Cluster calls" not in base[8]
            got = _run(tmp_path, pool, mode, *common, tag=f"on_{shard}_{mode}", calls=True)
            assert got[7] == want, (shard, mode)
            assert got[:7] == base[:7], (shard, mode)
            _check_info(got[8], got[5], res, len(GO.records(pool[0])))


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], tag=f"one_{path}", calls=True)
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], tag=f"two_{path}", calls=True)
        assert one[:8] == two[:8]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _same(got, want):
    for f in ("k", "n_hyp", "n_rounds", "converged"):
        assert got[f] == want[f], f
    for f in FIELDS:
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


def _both(entries, n_rows, n_cols, cl, eps=0.01, max_rounds=8):
    import vartrix_b200 as vb
    want = O.refine(*entries, n_rows, n_cols, cl, eps, max_rounds)
    with vb.Engine("coverage") as e:
        got = e.cluster_refine(*entries, n_rows, n_cols, cl, eps, max_rounds)
    _same(got, want)
    return got, want


@pytest.mark.parametrize("k", [2, 17, 32])
def test_engine_equals_restatement(k):
    import vartrix_b200 as vb
    n_rows, n_cols = 800, {2: 600, 17: 600, 32: 300}[k]
    entries, cl, _ = RC.pool(n_rows, n_cols, k, seed=k)
    eps = {2: 1e-6, 17: 0.01, 32: 0.25}[k]
    with vb.Engine("coverage") as e:
        for max_rounds in (0, 1, 8):
            want = O.refine(*entries, n_rows, n_cols, cl, eps, max_rounds)
            got = e.cluster_refine(*entries, n_rows, n_cols, cl, eps, max_rounds)
            again = e.cluster_refine(*entries, n_rows, n_cols, cl, eps, max_rounds)
            _same(got, want)
            _same(again, got)
            assert got["n_rounds"] <= max_rounds + 1 and got["calls"].sum(axis=1).tolist() == [n_cols] * got["n_rounds"]
            if max_rounds == 1 and k == 17:          # the loop stops at the cap with labels still moving
                assert got["n_rounds"] == 2 and not got["converged"] and got["changed"][-1] > 0


def test_round0_fit_is_cluster_genotypes():
    import vartrix_b200 as vb
    entries, cl, _ = RC.pool(700, 400, 5, seed=3)
    ra, rd = GO.row_sums(entries[0], entries[2], entries[3], 700)
    with vb.Engine("coverage") as e:
        r0 = e.cluster_refine(*entries, 700, 400, cl, 0.01, 0)
        cg = e.cluster_genotypes(cl, ra.astype(np.uint64), rd.astype(np.uint64))
    assert r0["n_rounds"] == 1 and not r0["converged"] and r0["rho_permille"][0] == cg["rho_permille"]
    for f in ("touched", "gt", "pl"):
        assert np.array_equal(r0[f], cg[f]), f


def _deep_clusters(n_rows, k, seed, depth=400):
    """clusters whose every (row, cluster) is called: depth molecules at the dosage's fraction"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, k))
    T = np.full((n_rows, k), depth << 16, np.int64)
    A = (T * np.array([0.0, 0.5, 1.0])[g]).astype(np.int64)
    return dict(alt_w=A, depth_w=T, row_used=np.ones(n_rows, np.uint8))


def test_seam_ladder_equals_numpy():
    """one cell over 1, 31, 32, 33 and 2 049 scored rows (the warp's 32-entry loads); one row over 100 000 cells; 3 000
    one-entry cells"""
    rng = np.random.default_rng(21)
    for n in (1, 31, 32, 33, 2049):
        cl = _deep_clusters(n, 3, seed=n)
        entries = (np.arange(n), np.zeros(n, np.int64), rng.integers(0, 4, n), rng.integers(1, 4, n))
        got, _ = _both(entries, n, 1, cl, max_rounds=0)
        assert got["rows_scored"][0] == n and got["counts"][0, 0] == n
    n_cols = 100_000
    entries = (np.zeros(n_cols, np.int64), np.arange(n_cols), rng.integers(0, 5, n_cols), rng.integers(0, 5, n_cols))
    _both(entries, 1, n_cols, _deep_clusters(1, 4, seed=1, depth=100_000))
    n_rows, n_cols = 500, 3000
    row = rng.integers(0, n_rows, n_cols)
    o = np.lexsort((np.arange(n_cols), row))
    entries = (row[o], np.arange(n_cols)[o], rng.integers(0, 6, n_cols)[o], rng.integers(0, 6, n_cols)[o])
    _both(entries, n_rows, n_cols, _deep_clusters(n_rows, 6, seed=2))


def test_rows_where_every_code_is_p():
    """half the rows have one molecule per cluster (GQ < 20 everywhere: not scored); a cell with entries only there has no
    scored row and is unassigned"""
    entries, cl, _ = RC.pool(600, 300, 4, seed=8)
    shallow = np.arange(600) % 2 == 1
    cl["depth_w"][shallow] = 1 << 16
    cl["alt_w"][shallow] = 0
    row, col, ref, alt = entries
    keep = (col != 0) | shallow[row]                         # cell 0 keeps only its entries at shallow rows
    got, want = _both(tuple(x[keep] for x in entries), 600, 300, cl, max_rounds=0)
    assert got["rows_scored"][0] < got["n_touched"][0] and got["counts"][0, 0] == 0 and got["label"][0] == O.NONE


def test_clusters_without_singlets():
    """a third cluster with cluster 0's sums: donor 0's cells tie between the two, so no cell is labelled 0 or 2 after round
    0, both clusters have T = 0 and codes P everywhere from round 1 on, and both stay"""
    entries, cl, _ = RC.pool(600, 400, 2, seed=9)
    for f in ("alt_w", "depth_w"):
        cl[f] = np.concatenate([cl[f], cl[f][:, :1]], axis=1)
    got, want = _both(entries, 600, 400, cl)
    assert not np.isin(want["round_labels"][0], [0, 2]).any() and (want["round_labels"][0] == 1).any()
    assert got["n_rounds"] >= 2 and (got["gt"][:, [0, 2]] == GO.MISSING).all() and got["ll"].shape == (400, 6)


def test_sparse_touch_of_a_large_table():
    """a 5 M-row table of which 1 500 rows hold entries"""
    n_rows, k = 5_000_000, 4
    small, cls, _ = RC.pool(1500, 300, k, seed=12)
    rows = np.sort(np.random.default_rng(12).choice(n_rows, 1500, replace=False))
    entries = (rows[small[0]], *small[1:])
    cl = dict(alt_w=np.zeros((n_rows, k), np.int64), depth_w=np.zeros((n_rows, k), np.int64), row_used=np.zeros(n_rows, np.uint8))
    for f in cl:
        cl[f][rows] = cls[f]
    got, _ = _both(entries, n_rows, 300, cl)
    assert 0 < got["touched"].size <= 1500


def test_refusals_return_their_codes():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    entries, cl, _ = RC.pool(60, 40, 3, seed=1)
    ent = [np.ascontiguousarray(x, np.uint32) for x in entries]
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        L, h = e._L, e._h
        out = _capi.ClusterCalls()

        def call(ent=ent, A=cl["alt_w"], T=cl["depth_w"], used=cl["row_used"], k=3, eps=0.01, rounds=8, n_rows=60, n_cols=40):
            p = _capi.ClusterCallsParams(k, eps, rounds)
            return L.vtx_cluster_refine(h, len(ent[0]), *(x.ctypes.data for x in ent), n_rows, n_cols, A.ctypes.data, T.ctypes.data,
                                        used.ctypes.data, C.byref(p), C.byref(out))
        assert call() == 0 and call(rounds=0) == 0 and call(rounds=32) == 0
        for kw in (dict(k=1), dict(k=33), dict(eps=0.0), dict(eps=0.3), dict(eps=float("nan")), dict(rounds=33)):
            assert call(**kw) == -1, kw
        bad = [x.copy() for x in ent]; bad[0][-1] = 60
        assert call(ent=bad) == -1 and "row" in e.last_error()
        i = int(np.flatnonzero(ent[0][1:] == ent[0][:-1])[0])                # two entries of one row
        bad = [x.copy() for x in ent]; bad[1][i + 1] = bad[1][i]
        assert call(ent=bad) == -1 and "ascending" in e.last_error()
        bad = cl["alt_w"].copy(); bad[3, 1] = -1
        assert call(A=bad) == -1 and "alt_w" in e.last_error()
        deep = cl["depth_w"].copy(); deep[4, 0] = (1 << 51) + 1
        assert call(T=deep) == -1 and "2^51" in e.last_error()
        deep = np.zeros_like(cl["depth_w"]); deep[:2, 0] = 1 << 51
        assert call(A=np.zeros_like(cl["alt_w"]), T=deep) == -1 and "sums" in e.last_error()
        big = [np.arange(9, dtype=np.uint32), np.zeros(9, np.uint32), np.full(9, 0xFFFFFFFF, np.uint32), np.zeros(9, np.uint32)]
        assert call(ent=big) == -1 and "2^35" in e.last_error()          # 9 (2^32 - 1) molecules: over 2^35 in all, not per row
        big = [x[:8] for x in big]
        assert call(ent=big) == 0
        e.set_barcodes(bcs)
        e.submit(sb)
        assert call() == -5
        e.finish()
        assert call() == 0
