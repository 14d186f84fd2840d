"""`--ambient-rna` without a GPU: the engine's table and scoring bodies (tests/ambient_shim.cpp) equal the NumPy restatement
(tests/ambient_oracle.py) bit for bit, the model at rho = 0 has §5f's constants, the restatement recovers the seeded pools'
ambient fraction (tests/ambient_cases.py) and fixes the false doublets of the contaminated ones, and the CLI refuses bad
options before any GPU work."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import ambient_cases as AC
import ambient_oracle as O
import donor_oracle as DO

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("amshim") / "libambient_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "ambient_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


EPS = (1e-6, 0.25)
MS = (0, 1, 499, 500)


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eps", EPS + (0.01,))
@pytest.mark.parametrize("m", MS + (137,))
def test_tables_equal_restatement(shim, eps, m):
    rng = np.random.default_rng(m)
    T = np.concatenate([[0, 0, 1, 1, 7, (1 << 53) - 3, (1 << 53) - 3, 1 << 40], rng.integers(0, 1 << 30, 500)]).astype(np.uint64)
    A = np.concatenate([[0, 0, 0, 1, 3, 0, (1 << 53) - 3, 1 << 39], [rng.integers(0, t + 1) for t in T[8:]]]).astype(np.uint64)
    tab = np.zeros((T.size, 5, 2), np.int32)
    shim.vtx_test_am_tables(ctypes.c_double(eps), ctypes.c_uint32(m), ctypes.c_uint32(T.size), _p(A), _p(T), _p(tab))
    la, lr = O.tables(m, A.astype(np.int64), T.astype(np.int64), eps)
    assert np.array_equal(tab[:, :, 0], la) and np.array_equal(tab[:, :, 1], lr)


def _matrix(rng, n_rows, n_cols, density, d):
    m = rng.random((n_rows, n_cols)) < density
    row, col = np.nonzero(m)
    r = rng.integers(0, 30, row.size)
    a = rng.integers(0, 30, row.size)
    r[rng.random(row.size) < 0.3] = 0
    a[rng.random(row.size) < 0.3] = 0
    big = rng.random(row.size) < 0.01
    r[big] = rng.integers(0, 1 << 20, big.sum())
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    g[rng.random((n_rows, d)) < 0.01] = DO.MISSING
    return row.astype(np.int64), col.astype(np.int64), r.astype(np.int64), a.astype(np.int64), g


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("d", [2, 17, 32])
def test_score_equals_restatement(shim, d, eps):
    """every cell's log-likelihoods, counts and call at m = 0, 1, 499, 500, with empty cells, unusable rows and r + a = 0"""
    rng = np.random.default_rng(d)
    n_rows, n_cols = 80, 75
    row, col, r, a, g = _matrix(rng, n_rows, n_cols - 5, 0.1, d)          # the last five cells have no entry
    p = O.prepare(row, col, r, a, n_rows, g)
    assert 0 < p["usable"].sum() < n_rows
    touched = np.unique(p["row"])
    tix = np.zeros(n_rows, np.uint32)
    tix[touched] = np.arange(touched.size)
    dos = np.ascontiguousarray(g[touched])
    o = np.argsort(p["col"], kind="stable")
    start = np.concatenate([[0], np.cumsum(np.bincount(p["col"], minlength=n_cols))]).astype(np.uint32)
    c_row, c_r, c_a = (np.ascontiguousarray(x[o], np.uint32) for x in (p["row"], p["r"], p["a"]))
    H = d + d * (d - 1) // 2
    for m in MS:
        la, lr = O.tables(m, p["A"][touched], p["T"][touched], eps)
        tab = np.ascontiguousarray(np.stack([la, lr], 2).astype(np.int32))
        ll, cnt, call = np.zeros((n_cols, H), np.int64), np.zeros((n_cols, 3), np.uint64), np.zeros(n_cols, np.uint32)
        shim.vtx_test_am_score(ctypes.c_uint32(n_cols), ctypes.c_uint32(d), _p(start), _p(c_row), _p(c_r), _p(c_a), _p(tix), _p(dos), _p(tab),
                               _p(ll), _p(cnt), _p(call))
        wll, wcnt = O.score(p, m, eps, n_cols)
        assert np.array_equal(ll, wll) and np.array_equal(cnt.astype(np.int64), wcnt), m
        wcall, _ = O.calls(wll, wcnt, d)
        assert np.array_equal(call, wcall), m
        assert (wcnt[:, 0] == 0).any()


@pytest.mark.parametrize("eps", [0.01, 0.02, 1e-6, 0.25])
def test_rho_zero_constants_equal_donor_tables(shim, eps):
    """at m = 0 the ten ll_log constants are make_tables' libm constants: --ambient-rna 0 writes §5f's file"""
    la, lr = O.tables(0, np.array([0, 5, 1 << 40]), np.array([0, 9, 1 << 41]), eps)
    wlr, wla = DO.tables(eps)
    clr, cla = np.zeros(5, np.int64), np.zeros(5, np.int64)
    shim.vtx_test_donor_tables(ctypes.c_double(eps), _p(clr), _p(cla))
    for v in range(3):
        assert la[v].tolist() == wla == cla.tolist() and lr[v].tolist() == wlr == clr.tolist()


# ---- the restatement on the pools ------------------------------------------------------------------------------------------
# The pools read every molecule 1 to 3 times, so the model's counts are molecules: the calls after the UMI collapse (--umi).
@pytest.fixture(scope="module")
def pools(tmp_path_factory):
    out = {}
    for rho in AC.RHOS:
        p = AC.write_pool(str(tmp_path_factory.mktemp(f"am_{rho}")), rho)
        samples, dosage = DO.read_genotypes(p["vcf"])
        keys, row, col, alt, ref = DO.coverage_counts(p["vcf"], p["bam"], p["fasta"], p["barcodes"], umi=True)
        out[rho] = dict(p, truth=json.load(open(p["truth"])), keys=keys, counts=(row, col, ref, alt), dosage=dosage)
    return out


def _files(p):
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


def _run(p, rho):
    res = O.ambient(*p["counts"], p["dosage"].shape[0], len(p["keys"]), p["dosage"], 0.01, rho)
    text = DO.text(p["donors"], p["keys"], res["ll"].tolist(), res["counts"].tolist())
    return res, [ln.split("\t") for ln in text.splitlines()[1:]]


ESTIMATES = {0.0: 1, 0.05: 54, 0.15: 149, 0.3: 289}          # m of the estimate on each pool


@pytest.mark.parametrize("rho", AC.RHOS)
def test_restatement_recovers_rho(pools, rho):
    res, rows = _run(pools[rho], None)
    assert res["rho_permille"] == ESTIMATES[rho]
    assert abs(res["rho_permille"] / 1000 - rho) <= 0.015
    m, j = res["grid_permille"].tolist(), res["grid_objective"].tolist()
    coarse = [x for x in m if x % 10 == 0]
    assert coarse == list(range(0, 501, 10)) and m == sorted(m)
    mc = max(coarse, key=lambda x: (j[m.index(x)], -x))
    assert [x for x in m if x % 10] == [x for x in range(max(0, mc - 9), min(500, mc + 9) + 1) if x % 10]
    assert j[m.index(res["rho_permille"])] == max(j) and j.index(max(j)) == m.index(res["rho_permille"])
    assert (res["grid_calls"].sum(axis=1) == len(rows)).all()


# singlets the rho = 0 model calls `doublet` on the contaminated pools
FALSE_DOUBLETS_AT_ZERO = {0.15: 11, 0.3: 87}


@pytest.mark.parametrize("rho", [0.15, 0.3])
def test_estimate_fixes_false_doublets(pools, rho):
    p = pools[rho]
    truth = p["truth"]
    _, at_zero = _run(p, 0)
    _, at_est = _run(p, None)
    false0 = sum(r[4] == "doublet" for r in at_zero if truth[r[0]]["kind"] == "singlet")
    assert false0 == FALSE_DOUBLETS_AT_ZERO[rho] > 0
    for r in at_est:
        t = truth[r[0]]
        if t["kind"] == "empty":
            assert r[1:6] == ["0", "0", "0", "unassigned", "."]
        if t["kind"] == "singlet" and t["molecules"] >= 100:
            assert r[4] == "singlet" and r[5] == t["donors"][0], (r[:6], t)
    assert sum(r[4] == "doublet" for r in at_est if truth[r[0]]["kind"] == "singlet") == 0


def test_read_counts_overstate_the_evidence(pools):
    """Without a UMI collapse the 1-3 reads of a molecule count as independent observations: on the rho = 0.3 pool the
    estimate is about the same, but two singlets of 100 molecules (about 200 reads each) are called `doublet`."""
    p = pools[0.3]
    keys, row, col, alt, ref = DO.coverage_counts(*_files(p))
    res, rows = _run(dict(p, keys=keys, counts=(row, col, ref, alt)), None)
    assert res["rho_permille"] == 294
    deep = [r[0] for r in rows if p["truth"][r[0]]["kind"] == "singlet" and p["truth"][r[0]]["molecules"] >= 100 and r[4] == "doublet"]
    assert len(deep) == 2 and all(p["truth"][bc]["molecules"] == 100 for bc in deep)


# ---- refusals: all of them before any GPU work (this machine may have none) ----------------------------------------------
def _cli(tmp_path, files, *extra):
    return subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", str(tmp_path / "o.mtx"), *extra],
                          cwd=str(tmp_path), capture_output=True, text=True)


def _refused(r, tmp_path, *words, keep=()):
    assert r.returncode == 1, r.stdout + r.stderr
    for w in words:
        assert w in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(keep)


@pytest.mark.parametrize("mode", ["0.5001", "0.501", "0.6", "1", "-0.1", "x", "", "0.", ".5", "estimated", "0.1234", "1e-2", "0,1",
                                  " 0.1", "0.1 ", "+0.1", "0000.1"])
def test_bad_modes_are_refused(tmp_path, pools, mode):
    _refused(_cli(tmp_path, _files(pools[0.0]), "--out-donors", str(tmp_path / "d.tsv"), "--ambient-rna", mode), tmp_path, "--ambient-rna",
             "'" + mode + "'")


@pytest.mark.parametrize("extra,words", [
    (["--ambient-rna", "estimate"], ["--ambient-rna", "--out-donors"]),
    (["--ambient-rna", "0.1", "--out-ambient", "a.tsv"], ["--ambient-rna", "--out-donors"]),
    (["--out-donors", "d.tsv", "--out-ambient", "a.tsv"], ["--out-ambient", "--ambient-rna"]),
    (["--out-ambient", "a.tsv"], ["--out-ambient", "--ambient-rna"]),
])
def test_orphan_options_are_refused(tmp_path, pools, extra, words):
    _refused(_cli(tmp_path, _files(pools[0.0]), *extra), tmp_path, *words)


def test_refused_with_dump_staged(tmp_path, pools):
    _refused(_cli(tmp_path, _files(pools[0.0]), "--out-donors", str(tmp_path / "d.tsv"), "--ambient-rna", "estimate", "--dump-staged",
                  str(tmp_path / "s")), tmp_path, "--ambient-rna", "--dump-staged")


@pytest.mark.parametrize("which", ["d.tsv", "a.tsv"])
def test_existing_output_path_is_refused(tmp_path, pools, which):
    (tmp_path / which).write_text("keep me\n")
    r = _cli(tmp_path, _files(pools[0.0]), "--out-donors", str(tmp_path / "d.tsv"), "--ambient-rna", "0.2", "--out-ambient",
             str(tmp_path / "a.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / which).read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == [which]


def test_help_and_readme_list_the_flags():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    readme = open(os.path.join(ROOT, "README.md")).read()
    for flag in ("--ambient-rna", "--out-ambient"):
        assert flag in r.stdout and flag in readme
