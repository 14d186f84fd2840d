"""GPU: `--known-donors` end to end and the engine's pinned clustering (vtx_cluster_cells_pinned).

The CLI on a seeded pool with 15 % ambient RNA (tests/cluster_gt_cases.py), D0, D2 and D4 pinned at K = 6 with rho given as
0.15, through host staging, --gpu-inflate and --gpu-stage, plain / --umi / --collapse-mates, in the three modes, at default
shards and at --shard-loci 4 --threads 3: the clusters and alleles files equal the restatement (tests/cluster_pinned_oracle.py)
byte for byte, and the matrices and metric lines equal a run without the flag.  Engine level: K = 2, 17, 32 with J = 1 and
K - 1, R = 1 and 8, m = 0 and 150, twice in a row; a seam ladder; a sample missing at every row; every refusal's code."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import ambient_oracle as AO
import cluster_gt_cases as GC
import cluster_oracle as CO
import cluster_pinned_oracle as O

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
SHARDS = {"default": [], "small": ["--shard-loci", "4", "--threads", "3"]}
MODES = ("consensus", "coverage", "alt_frac")
KNOWN = ("D0", "D2", "D4")
FIELDS = ("ll", "counts", "row_used", "alt_w", "depth_w", "restart_score", "restart_iters")


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = GC.write_pool(str(tmp_path_factory.mktemp("cppool")), 0.15)
    return (p["vcf_match"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys):
    return O.expected(*files, 6, KNOWN, 150, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r", known=True):
    """-> (out, ref or None, metric lines, clusters, alleles, stderr)"""
    out, ref, cl, al = (str(tmp_path / f"{tag}_{s}") for s in ("o.mtx", "ref.mtx", "cl.tsv", "al.tsv"))
    opt = ["--known-donors", ",".join(KNOWN), "--ambient-rna", "0.15"] if known else []
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", "--out-clusters", cl, "--clusters", "6", "--out-cluster-alleles", al, *opt, *extra],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(cl).read(), open(al).read(), r.stderr)


def _check_info(stderr, res, n_rows):
    m = re.search(r"Clusters with known donors: 6, known D0,D2,D4, ambient RNA 0\.150 \(given\), restarts 8, seed 0; best restart (\d+) "
                  r"after (\d+) iterations; rows used: (\d+) of (\d+); cells: (\d+) singlet, (\d+) doublet, (\d+) unassigned", stderr)
    assert m, stderr
    g = [int(x) for x in m.groups()]
    assert g[:4] == [res["best_restart"], int(res["restart_iters"][res["best_restart"]]), res["rows_used"], n_rows]
    assert sum(g[4:]) == res["counts"].shape[0]
    assert "[INFO] Clusters: " not in stderr


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cli_matches_restatement(tmp_path, pool, path, keys):
    want_cl, want_al, res = _expected(pool, keys)
    for shard, sargs in SHARDS.items():
        common = [*sargs, *PATHS[path], *KEYS[keys][0]]
        for mode in MODES:
            base = _run(tmp_path, pool, mode, *common, tag=f"off_{shard}_{mode}", known=False)
            assert "known donors" not in base[5]
            got = _run(tmp_path, pool, mode, *common, tag=f"on_{shard}_{mode}")
            assert got[3] == want_cl, (shard, mode)
            assert got[4] == want_al, (shard, mode)
            assert got[:3] == base[:3], (shard, mode)
            _check_info(got[5], res, len(res["row_used"]))


def test_ambient_fraction_also_applies_to_out_donors(tmp_path, pool):
    """--out-donors in the same run is scored at the given fraction, as --ambient-rna 0.15 alone would score it"""
    dn = str(tmp_path / "d.tsv")
    got = _run(tmp_path, pool, "coverage", "--umi", "--out-donors", dn, "--donors", "D0,D1,D2,D3,D4,D5")
    want_dn, _, _ = AO.expected(*pool, mode="0.15", donors=[f"D{d}" for d in range(6)], umi=True)
    assert open(dn).read() == want_dn
    assert got[3] == _expected(pool, "umi")[0]


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], tag=f"one_{path}")
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], tag=f"two_{path}")
        assert one[:5] == two[:5]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _synthetic(n_rows, n_cols, per_cell, k_true, seed, rho=0.15):
    """cells of k_true donors with dosages g [n_rows, k_true] (one in ten missing), ALT at the donor's fraction mixed with rho of
    the pool's; -> (row, col, ref, alt) sorted by (row, col), g"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, k_true))
    q = np.array([0.01, 0.5, 0.99])[g]
    p = (1 - rho) * q + rho * q.mean(axis=1, keepdims=True)
    donor = rng.integers(0, k_true, n_cols)
    rows, cols = [], []
    for c in range(n_cols):
        rr = np.unique(rng.integers(0, n_rows, per_cell))
        rows.append(rr); cols.append(np.full(rr.size, c))
    row, col = np.concatenate(rows), np.concatenate(cols)
    depth = rng.integers(0, 6, row.size)
    alt = rng.binomial(depth, p[row, donor[col]])
    ref = depth - alt
    o = np.lexsort((col, row))
    gd = g.astype(np.uint8)
    gd[rng.random(gd.shape) < 0.1] = O.MISSING
    return (row[o].astype(np.uint32), col[o].astype(np.uint32), ref[o].astype(np.uint32), alt[o].astype(np.uint32)), gd


def _same(got, want):
    for f in ("k", "n_hyp", "best_restart", "rows_used"):
        assert got[f] == want[f], f
    for f in FIELDS:
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


@pytest.mark.parametrize("restarts", [1, 8])
@pytest.mark.parametrize("k", [2, 17, 32])
def test_engine_equals_restatement(k, restarts):
    import vartrix_b200 as vb
    n_rows, n_cols = (800, 1000) if k < 32 else (500, 600)
    entries, g = _synthetic(n_rows, n_cols, 25, min(k, 8), seed=k * 10 + restarts)
    # rows without entries after the last: pinned, never used
    n_rows += 20
    g = np.concatenate([np.tile(g, (1, (k + g.shape[1] - 1) // g.shape[1]))[:, :k - 1], np.ones((20, k - 1), np.uint8)])
    with vb.Engine("coverage") as e:
        for J in (1, k - 1):
            for m in (0, 150):
                eps = 0.25 if m else 1e-6
                want = O.cluster_pinned(*entries, n_rows, n_cols, k, g[:, :J], m, eps, restarts, seed=k)
                got = e.cluster_cells_pinned(*entries, n_rows, n_cols, k, g[:, :J], m, eps, restarts, seed=k)
                again = e.cluster_cells_pinned(*entries, n_rows, n_cols, k, g[:, :J], m, eps, restarts, seed=k)
                _same(got, want)
                _same(again, got)
        # the unpinned call on the same context is unchanged by the pinned ones
        _same(e.cluster_cells(*entries, n_rows, n_cols, k, restarts, seed=k), CO.cluster(*entries, n_rows, n_cols, k, restarts, seed=k))


def test_seam_ladder_equals_numpy():
    """cells 0..4 over the first 1, 31, 32, 33 and 2 049 rows; row 2 049 over 100 000 cells; 3 000 one-entry cells; sample 1
    missing at every row"""
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
    entries = (np.array([x[0] for x in keys], np.uint32), np.array([x[1] for x in keys], np.uint32),
               np.array([ent[x][0] for x in keys], np.uint32), np.array([ent[x][1] for x in keys], np.uint32))
    g = np.stack([rng.integers(0, 3, n_rows), np.full(n_rows, O.MISSING)], axis=1).astype(np.uint8)
    want = O.cluster_pinned(*entries, n_rows, n_cols, 4, g, 150, 0.01, 2, seed=3)
    with vb.Engine("coverage") as e:
        got = e.cluster_cells_pinned(*entries, n_rows, n_cols, 4, g, 150, 0.01, 2, seed=3)
    _same(got, want)
    assert got["counts"][4, 0] > 1500 and got["counts"][103_500, 0] == 0


def test_refusals_return_their_codes():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    (row, col, ref, alt), g = _synthetic(50, 60, 10, 3, seed=1)
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        L, h = e._L, e._h
        out = _capi.Clusters()

        def call(row=row, col=col, ref=ref, alt=alt, dos=g, n_rows=50, n_cols=60, k=4, r=2, J=None, eps=0.01, m=100, null=False):
            d = np.ascontiguousarray(dos)
            p = _capi.ClusterPinnedParams(k, r, 0, d.shape[1] if J is None else J, eps, m)
            return L.vtx_cluster_cells_pinned(h, len(row), row.ctypes.data, col.ctypes.data, ref.ctypes.data, alt.ctypes.data, n_rows,
                                              n_cols, None if null else d.ctypes.data, C.byref(p), C.byref(out))
        assert call() == 0 and call(m=0) == 0 and call(m=500) == 0 and call(eps=1e-6) == 0 and call(eps=0.25) == 0
        assert call(dos=g[:, :1]) == 0
        for kw in (dict(k=1), dict(k=33), dict(r=0), dict(r=65), dict(k=3), dict(J=0), dict(eps=0.0), dict(eps=0.3),
                   dict(eps=float("nan")), dict(m=-1), dict(m=501), dict(null=True)):
            assert call(**kw) == -1, kw
        bad = g.copy(); bad[7, 1] = 3
        assert call(dos=bad) == -1 and "dosage 3" in e.last_error()
        assert call(n_rows=int(row.max())) == -1 and "row" in e.last_error()
        big = np.full(40, 0xFFFFFFFF, np.uint32)
        assert call(np.zeros(40, np.uint32), np.arange(40, dtype=np.uint32), big, big, n_cols=40) == -1 and "molecules" in e.last_error()
        assert call(n_rows=0xFFFFFFFF, k=32, r=64) == -3             # refused before the dosage of 2^32 - 1 rows is read
        e.set_barcodes(bcs)
        e.submit(sb)
        assert call() == -5
        e.finish()
        assert call() == 0
