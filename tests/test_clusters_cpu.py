"""`--out-clusters` without a GPU: the engine's log / exp routines and its E-, M- and scoring bodies (tests/cluster_shim.cpp)
equal the NumPy restatement (tests/cluster_oracle.py) bit for bit, the restatement recovers the seeded pools' donors
(tests/cluster_cases.py), and the CLI refuses bad clustering options before any GPU work."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import cluster_cases as CC
import cluster_oracle as O

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
KEYS = {"plain": {}, "umi": dict(umi=True), "mates": dict(collapse_mates=True)}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("clshim") / "libcluster_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cluster_shim.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.vtx_test_splitmix64.restype = ctypes.c_uint64
    return lib


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


# ---- ll_log / ll_exp ------------------------------------------------------------------------------------------------------
def test_ll_log_equals_restatement_and_libm(shim):
    x = np.concatenate([np.linspace(2.0 ** -40, 1.0, 400_001), np.geomspace(2.0 ** -45, 1.0, 200_001),
                        np.nextafter(np.geomspace(2.0 ** -40, 1.0, 1001), 0.0), [1.0, 0.5, np.sqrt(0.5), 2.0 ** -37]])
    y = np.zeros_like(x)
    shim.vtx_test_ll_log(ctypes.c_uint64(x.size), _p(x), _p(y))
    assert np.array_equal(y, O.ll_log(x))
    assert np.abs(y - np.log(x)).max() <= 2.0 ** -40
    assert y[-4] == 0.0


def test_ll_exp_equals_restatement_and_libm(shim):
    x = np.concatenate([np.linspace(-40.0, 0.0, 800_001), -np.geomspace(1e-300, 40.0, 100_001), [0.0, -0.0, -40.0, -40.000001, -1e9]])
    y = np.zeros_like(x)
    shim.vtx_test_ll_exp(ctypes.c_uint64(x.size), _p(x), _p(y))
    assert np.array_equal(y, O.ll_exp(x))
    inside = x >= -40.0
    assert np.abs(y[inside] - np.exp(x[inside])).max() <= 2.0 ** -40
    assert y[-5] == 1.0 and y[-4] == 1.0 and y[-3] > 0.0 and y[-2] == 0.0 and y[-1] == 0.0


def test_splitmix64(shim):
    for v in (0, 1, 12345, 1 << 63, (1 << 64) - 1):
        assert shim.vtx_test_splitmix64(ctypes.c_uint64(v)) == O.splitmix64(v) == int(O.splitmix64_np(np.array([v], np.uint64))[0])
    assert O.splitmix64(0) == 0xE220A8397B1DCDAF          # the published first output of splitmix64 seeded with 0


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------
def _matrix(rng, n_rows, n_cols, density):
    m = rng.random((n_rows, n_cols)) < density
    row, col = np.nonzero(m)
    r = rng.integers(0, 40, row.size)
    a = rng.integers(0, 40, row.size)
    r[rng.random(row.size) < 0.3] = 0
    a[rng.random(row.size) < 0.3] = 0
    big = rng.random(row.size) < 0.01
    r[big] = rng.integers(0, 1 << 20, big.sum())
    return row.astype(np.int64), col.astype(np.int64), r.astype(np.int64), a.astype(np.int64)


def _by_cell(row, col, r, a, n_cols):
    o = np.argsort(col, kind="stable")
    start = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=n_cols))]).astype(np.uint32)
    return start, *(np.ascontiguousarray(x[o], np.uint32) for x in (row, r, a))


@pytest.mark.parametrize("k", [2, 17, 32])
def test_bodies_equal_restatement(shim, k):
    """init, E-step, M-step and scoring of every cell / row against the restatement, with empty cells and rows"""
    rng = np.random.default_rng(k)
    n_rows, n_cols = 70, 90
    row, col, r, a = _matrix(rng, n_rows, n_cols, 0.08)
    used = O.used_rows(row, r, a, n_rows)
    assert 0 < used.sum() < n_rows
    keep = used[row] & (r + a > 0)
    cells = (row[keep], col[keep], r[keep], a[keep])
    start, c_row, c_r, c_a = _by_cell(*cells, n_cols)
    urows = np.flatnonzero(used).astype(np.uint32)
    for s in (0, 5):
        la, lr = np.zeros((n_rows, k), np.int32), np.zeros((n_rows, k), np.int32)
        shim.vtx_test_cl_init(ctypes.c_uint64(99), ctypes.c_uint32(s), ctypes.c_uint32(k), ctypes.c_uint32(urows.size), _p(urows), _p(la), _p(lr))
        wla, wlr = O.init_logs(99, s, k, urows)
        assert np.array_equal(la[urows], wla) and np.array_equal(lr[urows], wlr)
        w, m = np.zeros((n_cols, k), np.uint32), np.zeros(n_cols, np.int64)
        shim.vtx_test_cl_estep(ctypes.c_uint32(n_cols), ctypes.c_uint32(k), _p(start), _p(c_row), _p(c_r), _p(c_a), _p(la), _p(lr), _p(w), _p(m))
        ww, wm = O.estep(cells, la.astype(np.int64), lr.astype(np.int64), n_cols)
        assert np.array_equal(w, ww) and np.array_equal(m, wm)
        # M-step over every row (the final pass) with a permuted cluster order
        perm = rng.permutation(k).astype(np.uint32)
        rs = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n_rows))]).astype(np.uint32)
        A, T = np.zeros((n_rows, k), np.int64), np.zeros((n_rows, k), np.int64)
        mla, mlr = np.zeros((n_rows, k), np.int32), np.zeros((n_rows, k), np.int32)
        cc, rr, aa = (np.ascontiguousarray(x, np.uint32) for x in (col, r, a))
        shim.vtx_test_cl_mstep(ctypes.c_uint32(n_rows), _p(rs), _p(cc), _p(rr), _p(aa), _p(w), ctypes.c_uint32(k), _p(perm), _p(A), _p(T), _p(mla), _p(mlr))
        wA, wT = O.msums((row, col, r, a), ww[:, perm], n_rows)
        assert np.array_equal(A, wA) and np.array_equal(T, wT)
        xla, xlr = O.row_logs(wA, wT)
        assert np.array_equal(mla, xla) and np.array_equal(mlr, xlr)
        H = k + k * (k - 1) // 2
        ll, cnt = np.zeros((n_cols, H), np.int64), np.zeros((n_cols, 3), np.uint64)
        shim.vtx_test_cl_score(ctypes.c_uint32(n_cols), ctypes.c_uint32(k), _p(start), _p(c_row), _p(c_r), _p(c_a), _p(A), _p(T), _p(ll), _p(cnt))
        wll, wcnt = O.score(cells, wA, wT, k, n_cols)
        assert np.array_equal(ll, wll) and np.array_equal(cnt.astype(np.int64), wcnt)


def test_theta_extremes_stay_exact():
    """theta's integers are exact in double up to the row limit, and its logs fit in int32"""
    A = np.array([0, 0, (1 << 52) - 1], np.int64)
    T = np.array([0, (1 << 53) - (1 << 17), (1 << 53) - (1 << 17)], np.int64)
    la, lr = O.row_logs(A, T)
    assert la[0] == lr[0] == O.fixed(np.array([0.5]))[0]
    assert (la >= -(1 << 31)).all() and (lr >= -(1 << 31)).all()


# ---- the restatement on the pools ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pools(tmp_path_factory):
    return {n: CC.write_pool(str(tmp_path_factory.mktemp(f"cl_{n}")), n) for n in CC.POOLS}


def _files(p):
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


# the doublets of 300 molecules the restatement calls `doublet` (of 10 in k6, 2 in k2), per key mode
DOUBLETS_AT_300 = {("k6", "plain"): 10, ("k6", "umi"): 6, ("k6", "mates"): 8, ("k2", "plain"): 1, ("k2", "umi"): 0, ("k2", "mates"): 1}
# one D1 singlet of exactly 50 molecules in k6 is the only deep singlet the restatement does not place in its donor's cluster
MISSES_AT_50 = {"k6": 1, "k2": 0}


@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("pool", list(CC.POOLS))
def test_restatement_recovers_the_donors(pools, pool, keys):
    p = pools[pool]
    k = len(p["donors"])
    text, alleles, res = O.expected(*_files(p), k, **KEYS[keys])
    truth = json.load(open(p["truth"]))
    calls = O.calls(text)
    assert [c[0] for c in calls] == open(p["barcodes"]).read().split()
    match = CC.match_clusters(calls, truth, k)
    assert sorted(match.values()) == sorted(p["donors"])
    misses = 0
    for bc, variants, call, assignment in calls:
        t = truth[bc]
        if t["kind"] == "empty":
            assert (variants, call, assignment) == (0, "unassigned", ".")
        if t["kind"] != "singlet" or t["molecules"] < 50:
            continue
        assert call != "doublet", (bc, t)
        if t["molecules"] >= 100:
            assert call == "singlet" and match[assignment] == t["donors"][0], (bc, t, call, assignment)
        misses += not (call == "singlet" and match[assignment] == t["donors"][0])
    assert misses == MISSES_AT_50[pool]
    dbl = sum(call == "doublet" for bc, _, call, _ in calls if truth[bc]["kind"] == "doublet" and truth[bc]["molecules"] == 300)
    assert dbl == DOUBLETS_AT_300[(pool, keys)]
    # the allele file: one line per record, the used flag and the sums
    lines = alleles.splitlines()
    assert len(lines) == 1 + len(O.variant_labels(p["vcf"])) and lines[0].split("\t")[:4] == ["variant", "used", "ref_C0", "alt_C0"]
    assert sum(int(ln.split("\t")[1]) for ln in lines[1:]) == res["rows_used"] > 0
    # every restart ran, and at least one converged before the cap
    assert (res["restart_iters"] >= 1).all() and (res["restart_iters"] < O.MAX_ITERS).any()


def test_best_restart_is_not_always_the_first(pools):
    """restarts matter: on k6 with the default seed the winner is restart 6, and seeds give other winners"""
    p = pools["k6"]
    keys, row, col, alt, ref = O.DO.coverage_counts(*_files(p))
    res = O.cluster(row, col, ref, alt, len(O.variant_labels(p["vcf"])), len(keys), 6, 8, 0)
    assert res["best_restart"] == 6
    assert len(set(res["restart_score"].tolist())) > 1


# ---- refusals: all of them before any GPU work (this machine may have none) ----------------------------------------------
def _cli(tmp_path, files, *extra):
    return subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", str(tmp_path / "o.mtx"), *extra],
                          cwd=str(tmp_path), capture_output=True, text=True)


def _refused(r, tmp_path, *words, keep=()):
    assert r.returncode == 1, r.stdout + r.stderr
    for w in words:
        assert w in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(keep)


@pytest.mark.parametrize("extra,words", [
    (["--clusters", "1"], ["--clusters", "2 to 32", "'1'"]),
    (["--clusters", "33"], ["--clusters", "'33'"]),
    (["--clusters", "x"], ["--clusters"]),
    (["--clusters", "-4"], ["--clusters"]),
    (["--clusters", "4", "--cluster-restarts", "0"], ["--cluster-restarts", "1 to 64"]),
    (["--clusters", "4", "--cluster-restarts", "65"], ["--cluster-restarts"]),
    (["--clusters", "4", "--cluster-seed", "-1"], ["--cluster-seed"]),
    (["--clusters", "4", "--cluster-seed", "18446744073709551616"], ["--cluster-seed"]),
    (["--clusters", "4", "--cluster-seed", "1x"], ["--cluster-seed"]),
])
def test_bad_values_are_refused(tmp_path, pools, extra, words):
    _refused(_cli(tmp_path, _files(pools["k2"]), "--out-clusters", str(tmp_path / "c.tsv"), *extra), tmp_path, *words)


@pytest.mark.parametrize("extra", [
    ["--out-clusters", "c.tsv"],
    ["--clusters", "3"],
    ["--cluster-restarts", "4"],
    ["--cluster-seed", "5"],
    ["--out-cluster-alleles", "a.tsv"],
    ["--clusters", "3", "--out-cluster-alleles", "a.tsv"],
])
def test_orphan_options_are_refused(tmp_path, pools, extra):
    _refused(_cli(tmp_path, _files(pools["k2"]), *extra), tmp_path, "--out-clusters")


def test_refused_with_dump_staged(tmp_path, pools):
    _refused(_cli(tmp_path, _files(pools["k2"]), "--out-clusters", str(tmp_path / "c.tsv"), "--clusters", "2", "--dump-staged",
                  str(tmp_path / "s")), tmp_path, "--out-clusters", "--dump-staged")


@pytest.mark.parametrize("which", ["c.tsv", "a.tsv"])
def test_existing_output_path_is_refused(tmp_path, pools, which):
    (tmp_path / which).write_text("keep me\n")
    r = _cli(tmp_path, _files(pools["k2"]), "--out-clusters", str(tmp_path / "c.tsv"), "--clusters", "2", "--out-cluster-alleles",
             str(tmp_path / "a.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / which).read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == [which]


def test_help_and_readme_list_the_flags():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    readme = open(os.path.join(ROOT, "README.md")).read()
    for flag in ("--out-clusters", "--clusters", "--cluster-restarts", "--cluster-seed", "--out-cluster-alleles"):
        assert flag in r.stdout and flag in readme
