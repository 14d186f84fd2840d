"""GPU: `--ambient-rna` end to end and the engine's post-pass (vtx_donors_ambient).

The CLI on a seeded pool with 15 % ambient RNA (tests/ambient_cases.py) through host staging, --gpu-inflate and --gpu-stage,
plain / --umi / --collapse-mates, in the three modes, at default shards and at --shard-loci 4 --threads 3: the donor and
ambient files equal the restatement (tests/ambient_oracle.py) byte for byte in both modes, and the matrices and metric lines
equal a run without the flag; `--ambient-rna 0` writes the per-submit §5f file.  Engine level: D = 2, 17, 32 fixed and
estimated against the restatement, repeat calls, a seam ladder, the pass size, a sparse touch of a 5 M-row table, and every
refusal's code."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import ambient_cases as AC
import ambient_oracle as O

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
SHARDS = {"default": [], "small": ["--shard-loci", "4", "--threads", "3"]}
MODES = ("consensus", "coverage", "alt_frac")


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = AC.write_pool(str(tmp_path_factory.mktemp("ampool")), 0.15)
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys, mode):
    return O.expected(*files, mode, **KEYS[keys][1])


def _run(tmp_path, files, mode, *extra, tag="r", ambient=None):
    """-> (out text, ref text or None, metric lines, donors text, ambient text or None, stderr)"""
    out, ref, dn, am = (str(tmp_path / f"{tag}{s}") for s in (".mtx", "_ref.mtx", "_dn.tsv", "_am.tsv"))
    opt = ["--ambient-rna", ambient, "--out-ambient", am] if ambient else []
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", "--out-donors", dn, *opt, *extra], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(dn).read(),
            open(am).read() if ambient else None, r.stderr)


def _check_info(stderr, res, given):
    m = re.search(r"Ambient RNA: rho (\S+) \((\w+)\); fractions evaluated: (\d+); doublets: (?:(\d+) at rho 0\.000, )?(\d+) at rho (\S+)", stderr)
    assert m, stderr
    g = m.groups()
    i = res["grid_permille"].tolist().index(res["rho_permille"])
    assert g[0] == g[5] == f"{res['rho_permille'] / 1000:.3f}" and g[1] == ("given" if given else "estimated")
    assert int(g[2]) == len(res["grid_permille"]) and int(g[4]) == res["grid_calls"][i][1]
    if 0 in res["grid_permille"].tolist():
        assert int(g[3]) == res["grid_calls"][0][1]
    else:
        assert g[3] is None


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cli_matches_restatement(tmp_path, pool, path, keys):
    want_dn, want_am, res = _expected(pool, keys, "estimate")
    fix_dn, fix_am, fres = _expected(pool, keys, "0.15")
    assert res["rho_permille"] > 100
    for shard, sargs in SHARDS.items():
        common = [*sargs, *PATHS[path], *KEYS[keys][0]]
        for i, mode in enumerate(MODES):
            base = _run(tmp_path, pool, mode, *common, tag=f"off_{shard}_{mode}")
            assert "Ambient RNA" not in base[5]
            got = _run(tmp_path, pool, mode, *common, tag=f"est_{shard}_{mode}", ambient="estimate")
            assert got[3] == want_dn and got[4] == want_am, (shard, mode)
            assert got[:3] == base[:3], (shard, mode)
            _check_info(got[5], res, False)
            if i == (0 if shard == "default" else 1):             # fixed mode, and rho = 0 against the per-submit path
                fix = _run(tmp_path, pool, mode, *common, tag=f"fix_{shard}_{mode}", ambient="0.15")
                assert fix[3] == fix_dn and fix[4] == fix_am and fix[:3] == base[:3], (shard, mode)
                _check_info(fix[5], fres, True)
                zero = _run(tmp_path, pool, mode, *common, tag=f"zero_{shard}_{mode}", ambient="0")
                assert zero[3] == base[3] and zero[:3] == base[:3], (shard, mode)


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], tag=f"one_{path}", ambient="estimate")
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], tag=f"two_{path}",
                   ambient="estimate")
        assert one[:5] == two[:5]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _synthetic(n_rows, n_cols, per_cell, d, rho, seed, missing=0.02):
    """cells of single donors (one in ten a doublet) with per_cell random rows and ambient molecules at rate rho;
    -> row, col, ref, alt sorted by (row, col), dosage [n_rows, d]"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    g[rng.random((n_rows, d)) < missing] = 0xFF
    d1 = rng.integers(0, d, n_cols)
    d2 = np.where(rng.random(n_cols) < 0.1, rng.integers(0, d, n_cols), d1)
    pool = np.where(g <= 2, g, 1).mean(axis=1) / 2
    rows, cols = [], []
    for c in range(n_cols):
        rr = np.unique(rng.integers(0, n_rows, per_cell))
        rows.append(rr); cols.append(np.full(rr.size, c))
    row, col = np.concatenate(rows), np.concatenate(cols)
    gd = np.where(g <= 2, g, 1) / 2
    p = (1 - rho) * 0.5 * (gd[row, d1[col]] + gd[row, d2[col]]) + rho * pool[row]
    depth = rng.integers(0, 6, row.size)
    alt = rng.binomial(depth, np.clip(p * 0.98 + 0.01, 0, 1))
    ref = depth - alt
    o = np.lexsort((col, row))
    return row[o].astype(np.uint32), col[o].astype(np.uint32), ref[o].astype(np.uint32), alt[o].astype(np.uint32), g


def _same(got, want):
    for f in ("rho_permille", "n_hyp", "rows_usable"):
        assert got[f] == want[f], f
    for f in ("ll", "counts", "grid_permille", "grid_objective", "grid_calls", "row_alt", "row_depth"):
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


@pytest.mark.parametrize("rho", [None, 0, 230, 500])
@pytest.mark.parametrize("d", [2, 17, 32])
def test_engine_equals_restatement(d, rho):
    import vartrix_b200 as vb
    n_rows, n_cols = (1500, 2000) if d < 32 else (700, 900)
    row, col, ref, alt, g = _synthetic(n_rows, n_cols, 25, d, 0.2, seed=d)
    # rows without entries after the last, cells without entries after the last
    g = np.concatenate([g, np.zeros((40, d), np.uint8)])
    n_rows += 40; n_cols += 7
    eps = {2: 1e-6, 17: 0.01, 32: 0.25}[d]
    want = O.ambient(row, col, ref, alt, n_rows, n_cols, g, eps, rho)
    with vb.Engine("coverage") as e:
        got = e.donors_ambient(row, col, ref, alt, n_rows, n_cols, g, eps, rho)
        again = e.donors_ambient(row, col, ref, alt, n_rows, n_cols, g, eps, rho)
    _same(got, want)
    _same(again, got)
    m, j = want["grid_permille"].tolist(), want["grid_objective"].tolist()
    if rho is None:                         # 60 fractions when the coarse winner is 0 or 500 (the fine pass is clipped), else 69
        mc = max((x for x in m if x % 10 == 0), key=lambda x: (j[m.index(x)], -x))
        assert len(m) == (60 if mc in (0, 500) else 69)
    else:
        assert m == [rho]
    assert got["rho"] == got["rho_permille"] / 1000


def _entries(ent):
    keys = sorted(ent)
    return (np.array([k[0] for k in keys], np.uint32), np.array([k[1] for k in keys], np.uint32),
            np.array([ent[k][0] for k in keys], np.uint32), np.array([ent[k][1] for k in keys], np.uint32))


def test_seam_ladder_equals_numpy():
    """cells 0..4 over the first 1, 31, 32, 33 and 2 049 rows; row 2 049 over 100 000 cells; 3 000 one-entry cells; the pass
    size 1, 7 and as memory allows"""
    import vartrix_b200 as vb
    rng = np.random.default_rng(7)
    n_rows, n_cols, d = 2100, 103_100, 5
    ent = {}
    for c, reach in enumerate((1, 31, 32, 33, 2049)):
        for v in range(reach):
            ent[(v, c)] = (int(rng.integers(0, 4)), int(rng.integers(0, 4)))
    for c in range(13, 100_013):
        ent[(2049, c)] = (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
    for c in range(100_013, 103_013):
        ent[(int(rng.integers(0, n_rows)), c)] = (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
    row, col, ref, alt = _entries(ent)
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    g[2049] = [0, 1, 2, 1, 0]
    want = O.ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, None)
    with vb.Engine("coverage") as e:
        for batch in (1, 7, 0):
            _same(e.donors_ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, None, grid_batch=batch), want)
        got = e.donors_ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, 321, grid_batch=7)
    _same(got, O.ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, 321))
    assert got["counts"][4, 0] > 1500 and got["counts"][103_050, 0] == 0


def test_sparse_touch_of_a_large_table():
    """a 5 M-row dosage table of which 3 000 rows have entries, some of them at rows no donor genotyped"""
    import vartrix_b200 as vb
    rng = np.random.default_rng(11)
    n_rows, n_cols, d = 5_000_000, 400, 8
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    g[rng.random(n_rows) < 0.1, 3] = 0xFF
    rows = np.sort(rng.choice(n_rows, 3000, replace=False))
    ent = {}
    for v in rows.tolist():
        for c in rng.choice(n_cols, 12, replace=False).tolist():
            ent[(v, c)] = (int(rng.integers(0, 4)), int(rng.integers(0, 4)))
    row, col, ref, alt = _entries(ent)
    want = O.ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, None)
    with vb.Engine("coverage") as e:
        got = e.donors_ambient(row, col, ref, alt, n_rows, n_cols, g, 0.01, None)
    _same(got, want)
    assert got["rows_usable"] == int((g <= 2).all(axis=1).sum()) < n_rows


def test_refusals_return_their_codes():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    row, col, ref, alt, g = _synthetic(50, 60, 10, 3, 0.1, seed=1, missing=0.0)
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    with vb.Engine("coverage") as e:
        L, h = e._L, e._h
        out = _capi.Ambient()

        def call(row, col, ref, alt, n_rows=50, n_cols=60, dosage=g, d=3, eps=0.01, rho=-1):
            p = _capi.AmbientParams(d, eps, rho, 0)
            return L.vtx_donors_ambient(h, len(row), row.ctypes.data, col.ctypes.data, ref.ctypes.data, alt.ctypes.data, n_rows, n_cols,
                                        dosage.ctypes.data, C.byref(p), C.byref(out))
        assert call(row, col, ref, alt) == 0
        for kw in (dict(d=1), dict(d=33), dict(eps=0.0), dict(eps=0.3), dict(eps=float("nan")), dict(rho=-2), dict(rho=501)):
            assert call(row, col, ref, alt, **kw) == -1, kw
        assert call(row, col, ref, alt, rho=500) == 0 and call(row, col, ref, alt, rho=0) == 0
        assert call(row, col, ref, alt, n_rows=int(row.max())) == -1 and "row" in e.last_error()
        assert call(row, col, ref, alt, n_cols=int(col.max())) == -1 and "col" in e.last_error()
        swapped = row.copy(); swapped[[3, 40]] = swapped[[40, 3]]
        assert call(swapped, col, ref, alt) == -1
        dup = col.copy(); dup[1] = dup[0]; rdup = row.copy(); rdup[1] = rdup[0]
        assert call(rdup, dup, ref, alt) == -1
        bad = g.copy(); bad[7, 1] = 3
        assert call(row, col, ref, alt, dosage=bad) == -1 and "dosage" in e.last_error()
        # one row of 2^20 + 1 entries: 2^53 - 2 molecules (T + 2 reaches 2^53) is refused, one fewer is scored
        n = (1 << 20) + 1
        rr, aa = np.full(n, 0xFFFFFFFF, np.uint32), np.full(n, 0xFFFFFFFF, np.uint32)
        rr[-1] = aa[-1] = (1 << 20) - 1
        assert int(rr.astype(np.uint64).sum()) + int(aa.astype(np.uint64).sum()) == (1 << 53) - 2
        z, cc, gz = np.zeros(n, np.uint32), np.arange(n, dtype=np.uint32), np.zeros((1, 3), np.uint8)
        assert call(z, cc, rr, aa, n_rows=1, n_cols=n, dosage=gz) == -1 and "molecules" in e.last_error()
        rr[-1] -= 1
        assert call(z, cc, rr, aa, n_rows=1, n_cols=n, dosage=gz, rho=7) == 0
        # 2^32 - 1 rows and cells at 32 donors need terabytes: refused before the (here 1-byte) dosage table is read
        huge = np.zeros(1, np.uint8)
        assert call(row, col, ref, alt, n_rows=0xFFFFFFFF, n_cols=0xFFFFFFFF, dosage=huge, d=32) == -3 and "MB" in e.last_error()
        with pytest.raises(TypeError):                          # the Python call takes thousandths, not a fraction
            e.donors_ambient(row, col, ref, alt, 50, 60, g, 0.01, 0.15)
        e.set_barcodes(bcs)
        e.submit(sb)
        assert call(row, col, ref, alt) == -5
        e.finish()
        assert call(row, col, ref, alt) == 0
