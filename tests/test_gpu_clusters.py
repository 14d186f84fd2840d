"""GPU: `--out-clusters` end to end and the engine's clustering (vtx_cluster_cells).

The CLI on the seeded pool (tests/cluster_cases.py) through host staging, --gpu-inflate and --gpu-stage, plain / --umi /
--collapse-mates, in the three modes, at default shards and at --shard-loci 4 --threads 3, against the restatement
(tests/cluster_oracle.py) byte for byte; in the same runs the matrices and metric lines equal a run without the flag.  Engine
level: K = 2, 17, 32 at R = 1 and 8 against the restatement, repeat calls, a seam ladder, and every refusal's code."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import cluster_cases as CC
import cluster_oracle as O

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
SHARDS = {"default": [], "small": ["--shard-loci", "4", "--threads", "3"]}


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = CC.write_pool(str(tmp_path_factory.mktemp("clpool")), "k6")
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys, k, restarts, seed):
    return O.expected(*files, k, restarts, seed, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r", clusters=None):
    """-> (out text, ref text or None, metric lines, clusters text, alleles text, stderr)"""
    out, ref, cl, al = (str(tmp_path / f"{tag}{s}") for s in (".mtx", "_ref.mtx", "_cl.tsv", "_al.tsv"))
    opt = ["--out-clusters", cl, "--clusters", str(clusters), "--out-cluster-alleles", al] if clusters else []
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", *opt, *extra], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(cl).read() if clusters else None,
            open(al).read() if clusters else None, r.stderr)


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cli_matches_restatement(tmp_path, pool, path, keys):
    want_cl, want_al, res = _expected(pool, keys, 6, 8, 0)
    for shard, sargs in SHARDS.items():
        common = [*sargs, *PATHS[path], *KEYS[keys][0]]
        for mode in ("consensus", "coverage", "alt_frac"):
            base = _run(tmp_path, pool, mode, *common, tag=f"off_{shard}_{mode}")
            got = _run(tmp_path, pool, mode, *common, tag=f"on_{shard}_{mode}", clusters=6)
            assert got[3] == want_cl, (shard, mode)
            assert got[4] == want_al, (shard, mode)
            assert got[:3] == base[:3], (shard, mode)
            assert "Clusters:" not in base[5]
            calls = [c[2] for c in O.calls(got[3])]
            m = re.search(r"Clusters: 6, restarts 8, seed 0; best restart (\d+) after (\d+) iterations; rows used: (\d+) of (\d+); "
                          r"cells: (\d+) singlet, (\d+) doublet, (\d+) unassigned", got[5])
            assert m, got[5]
            assert [int(x) for x in m.groups()] == [res["best_restart"], int(res["restart_iters"][res["best_restart"]]), res["rows_used"],
                                                    len(res["row_used"]), calls.count("singlet"), calls.count("doublet"),
                                                    calls.count("unassigned")]


def test_seed_and_restarts_reach_the_cli(tmp_path, pool):
    want_cl, want_al, _ = _expected(pool, "plain", 6, 3, 12345678901234567890)
    got = _run(tmp_path, pool, "coverage", "--cluster-restarts", "3", "--cluster-seed", "12345678901234567890", clusters=6)
    assert got[3] == want_cl and got[4] == want_al


def test_donor_singlets_map_onto_clusters(tmp_path, pool):
    """with --out-donors in the same run: the cells both files call singlet pair donors and clusters one to one"""
    dn = str(tmp_path / "d.tsv")
    got = _run(tmp_path, pool, "coverage", "--umi", "--out-donors", dn, clusters=6)
    donors = {ln.split("\t")[0]: ln.split("\t") for ln in open(dn).read().splitlines()[1:]}
    pairs = set()
    n_donor_singlets = 0
    for bc, _, call, assignment in O.calls(got[3]):
        d = donors[bc]
        if d[4] != "singlet":
            continue
        n_donor_singlets += 1
        if call == "singlet":
            pairs.add((d[5], assignment))
    assert len(pairs) == 6 and len({p[0] for p in pairs}) == 6 and len({p[1] for p in pairs}) == 6, pairs
    assert n_donor_singlets > 300


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], tag=f"one_{path}", clusters=6)
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], tag=f"two_{path}",
                   clusters=6)
        assert one[:5] == two[:5]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _synthetic(n_rows, n_cols, per_cell, k_true, seed):
    """cells of k_true groups, each with per_cell random rows; -> row, col, ref, alt sorted by (row, col)"""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.02, 0.98, (n_rows, k_true))
    group = rng.integers(0, k_true, n_cols)
    rows, cols = [], []
    for c in range(n_cols):
        rr = np.unique(rng.integers(0, n_rows, per_cell))
        rows.append(rr); cols.append(np.full(rr.size, c))
    row, col = np.concatenate(rows), np.concatenate(cols)
    depth = rng.integers(0, 6, row.size)
    alt = rng.binomial(depth, p[row, group[col]])
    ref = depth - alt
    o = np.lexsort((col, row))
    return row[o].astype(np.uint32), col[o].astype(np.uint32), ref[o].astype(np.uint32), alt[o].astype(np.uint32)


def _same(got, want):
    for f in ("k", "n_hyp", "best_restart", "rows_used"):
        assert got[f] == want[f], f
    for f in ("ll", "counts", "row_used", "alt_w", "depth_w", "restart_score", "restart_iters"):
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


@pytest.mark.parametrize("restarts", [1, 8])
@pytest.mark.parametrize("k", [2, 17, 32])
def test_engine_equals_restatement(k, restarts):
    import vartrix_b200 as vb
    n_rows, n_cols = (1500, 2000) if k < 32 else (700, 900)
    row, col, ref, alt = _synthetic(n_rows, n_cols, 25, min(k, 8), seed=k * 10 + restarts)
    # rows without entries after the last, and a row with REF and ALT in only three cells: not used, but in the allele sums
    last = np.arange(3, dtype=np.uint32)
    row, col = np.concatenate([row, np.full(3, n_rows + 5, np.uint32)]), np.concatenate([col, last])
    ref, alt = np.concatenate([ref, last + 1]), np.concatenate([alt, last + 2])
    n_rows += 40
    want = O.cluster(row, col, ref, alt, n_rows, n_cols, k, restarts, seed=k)
    with vb.Engine("coverage") as e:
        got = e.cluster_cells(row, col, ref, alt, n_rows, n_cols, k, restarts, seed=k)
        again = e.cluster_cells(row, col, ref, alt, n_rows, n_cols, k, restarts, seed=k)
    _same(got, want)
    _same(again, got)
    assert 0 < want["rows_used"] <= n_rows - 40 and want["row_used"][n_rows - 35] == 0 and want["depth_w"][n_rows - 35].sum() > 0


def test_seam_ladder_equals_numpy():
    """cells 0..4 over the first 1, 31, 32, 33 and 2 049 rows; row 2 049 over 100 000 cells; 3 000 one-entry cells"""
    import vartrix_b200 as vb
    rng = np.random.default_rng(5)
    n_rows, n_cols = 2100, 104_000
    ent = {}
    for c, reach in enumerate((1, 31, 32, 33, 2049)):
        for v in range(reach):
            ent[(v, c)] = (int(rng.integers(0, 4)), int(rng.integers(0, 4)))
    for c in range(5, 13):                  # background cells that make every row used
        for v in range(n_rows):
            ent[(v, c)] = (int(rng.integers(1, 5)), int(rng.integers(1, 5)))
    for c in range(13, 100_013):
        ent[(2049, c)] = (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
    for c in range(100_013, 103_013):
        ent[(int(rng.integers(0, n_rows)), c)] = (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
    keys = sorted(ent)
    row = np.array([k[0] for k in keys], np.uint32)
    col = np.array([k[1] for k in keys], np.uint32)
    ref = np.array([ent[k][0] for k in keys], np.uint32)
    alt = np.array([ent[k][1] for k in keys], np.uint32)
    want = O.cluster(row, col, ref, alt, n_rows, n_cols, 4, 2, seed=3)
    with vb.Engine("coverage") as e:
        got = e.cluster_cells(row, col, ref, alt, n_rows, n_cols, 4, 2, seed=3)
    _same(got, want)
    assert got["counts"][4, 0] > 1500 and got["counts"][103_500, 0] == 0


def test_refusals_return_their_codes():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    row, col, ref, alt = _synthetic(50, 60, 10, 2, seed=1)
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        L, h = e._L, e._h
        out = _capi.Clusters()

        def call(row, col, ref, alt, n_rows=50, n_cols=60, k=3, r=2, seed=0):
            p = _capi.ClusterParams(k, r, seed)
            return L.vtx_cluster_cells(h, len(row), row.ctypes.data, col.ctypes.data, ref.ctypes.data, alt.ctypes.data, n_rows, n_cols,
                                       C.byref(p), C.byref(out))
        assert call(row, col, ref, alt) == 0
        for kw in (dict(k=1), dict(k=33), dict(r=0), dict(r=65)):
            assert call(row, col, ref, alt, **kw) == -1, kw
        assert call(row, col, ref, alt, n_rows=int(row.max())) == -1 and "row" in e.last_error()
        assert call(row, col, ref, alt, n_cols=int(col.max())) == -1 and "col" in e.last_error()
        swapped = row.copy(); swapped[[3, 40]] = swapped[[40, 3]]
        assert call(swapped, col, ref, alt) == -1
        dup = col.copy(); dup[1] = dup[0]; rdup = row.copy(); rdup[1] = rdup[0]
        assert call(rdup, dup, ref, alt) == -1
        big = np.full(40, 0xFFFFFFFF, np.uint32)
        assert call(np.zeros(40, np.uint32), np.arange(40, dtype=np.uint32), big, big, n_cols=40) == -1 and "molecules" in e.last_error()
        assert call(row, col, ref, alt, n_rows=0xFFFFFFFF, k=32, r=64) == -3
        e.set_barcodes(bcs)
        e.submit(sb)
        assert call(row, col, ref, alt) == -5
        e.finish()
        assert call(row, col, ref, alt) == 0
