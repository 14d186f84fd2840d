"""`--known-donors` without a GPU: the engine's pinned-log and scoring bodies (tests/cluster_pinned_shim.cpp) equal the
restatement (tests/cluster_pinned_oracle.py) bit for bit; the restatement with no pinned sample is cluster_oracle.cluster; on
the seeded ambient pools (C oracle counts -> the restatement) the calls are pinned, with the quality they reach; and the CLI
refuses bad options before any GPU work."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from conftest import ROOT
import ambient_cases as AC
import cluster_gt_cases as GC
import cluster_oracle as CO
import cluster_pinned_oracle as O
import donor_oracle as DO

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
EPS = (1e-6, 0.25)
MS = (0, 1, 499, 500)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cpshim") / "libcluster_pinned_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cluster_pinned_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _u32(*xs):
    return [np.ascontiguousarray(x, np.uint32) for x in xs]


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------
def _row_sums(rng, n):
    """A_v <= T_v with the extremes: empty rows, T_v + 2 = 2^53 - 1 with A_v at 0 and at T_v"""
    rd = np.concatenate([[0, (1 << 53) - 3, (1 << 53) - 3, 1], rng.integers(0, 1 << 30, n - 4)]).astype(np.uint64)
    ra = np.concatenate([[0, 0, (1 << 53) - 3, 1], [rng.integers(0, int(t) + 1) for t in rd[4:]]]).astype(np.uint64)
    return ra, rd


def _dosage(rng, n_rows, J):
    g = rng.integers(0, 3, (n_rows, J)).astype(np.uint8)
    g[rng.random((n_rows, J)) < 0.2] = O.MISSING
    g[5] = O.MISSING                                          # a row where no pinned sample has a dosage
    return g


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("k,J", [(2, 1), (17, 1), (17, 16), (32, 1), (32, 31)])
def test_bodies_equal_restatement(shim, k, J, eps):
    rng = np.random.default_rng(k * 100 + J)
    n_rows, n_cols = 200, 40
    ra, rd = _row_sums(rng, n_rows)
    g = _dosage(rng, n_rows, J)
    # A, T of every cluster (x 2^16) for the free (row, cluster) pairs of the scoring
    T = rng.integers(0, 1 << 40, (n_rows, k)).astype(np.int64)
    A = (T * rng.random((n_rows, k))).astype(np.int64)
    m_ent = 1500
    col = np.sort(rng.integers(0, n_cols, m_ent))
    row, r, a = rng.integers(0, n_rows, m_ent), rng.integers(0, 50, m_ent), rng.integers(0, 50, m_ent)
    start = np.searchsorted(col, np.arange(n_cols + 1)).astype(np.uint32)
    has = g != O.MISSING
    for m in MS:
        la, lr = np.full((n_rows, J), 7, np.int32), np.full((n_rows, J), 7, np.int32)
        shim.vtx_test_cp_logs(ctypes.c_double(eps), ctypes.c_uint32(m), ctypes.c_uint32(n_rows), ctypes.c_uint32(J), _p(g), _p(ra), _p(rd),
                              _p(la), _p(lr))
        wla, wlr = O.pinned_logs(g, m, ra.astype(np.int64), rd.astype(np.int64), eps)
        assert np.array_equal(la[has], wla[has]) and np.array_equal(lr[has], wlr[has]), m
        assert (la[~has] == 7).all() and (lr[~has] == 7).all()
        # the logs are those of the fractions the scoring mixes
        th, om = O.pinned_theta(g, m, ra.astype(np.int64), rd.astype(np.int64), eps)
        assert np.array_equal(CO.fixed(th)[has], wla[has]) and np.array_equal(CO.fixed(om)[has], wlr[has])
        H = k + k * (k - 1) // 2
        ll, cnt = np.zeros((n_cols, H), np.int64), np.zeros((n_cols, 3), np.uint64)
        rw, rr, aa = _u32(row, r, a)
        shim.vtx_test_cp_score(ctypes.c_uint32(n_cols), ctypes.c_uint32(k), ctypes.c_uint32(J), ctypes.c_double(eps), ctypes.c_uint32(m),
                               _p(start), _p(rw), _p(rr), _p(aa), _p(g), _p(ra), _p(rd), _p(A), _p(T), _p(ll), _p(cnt))
        wll, wcnt = O.score((row, col, r, a), A, T, k, n_cols, g, m, ra.astype(np.int64), rd.astype(np.int64), eps)
        assert np.array_equal(ll, wll) and np.array_equal(cnt.astype(np.int64), wcnt), m


def _matrix(rng, n_rows, n_cols, density):
    mask = rng.random((n_rows, n_cols)) < density
    row, col = np.nonzero(mask)
    r, a = rng.integers(0, 30, row.size), rng.integers(0, 30, row.size)
    r[rng.random(row.size) < 0.3] = 0
    a[rng.random(row.size) < 0.3] = 0
    return row, col, r, a


def _same(got, want):
    for f in ("k", "n_hyp", "best_restart", "rows_used"):
        assert got[f] == want[f], f
    for f in ("ll", "counts", "row_used", "alt_w", "depth_w", "restart_score", "restart_iters"):
        assert np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64)), f


@pytest.mark.parametrize("k", [2, 5])
def test_no_pinned_sample_is_cluster_oracle(k):
    rng = np.random.default_rng(40 + k)
    n_rows, n_cols = 120, 150
    row, col, r, a = _matrix(rng, n_rows, n_cols, 0.1)
    got = O.cluster_pinned(row, col, r, a, n_rows, n_cols, k, np.zeros((n_rows, 0), np.uint8), 150, 0.25, 4, 9)
    _same(got, CO.cluster(row, col, r, a, n_rows, n_cols, k, 4, 9))


def test_sample_missing_at_every_row_is_a_free_cluster():
    """a pinned sample without any dosage: the EM is §5g's; only the relabelling keeps cluster 0 first"""
    rng = np.random.default_rng(3)
    n_rows, n_cols, k = 150, 200, 4
    row, col, r, a = _matrix(rng, n_rows, n_cols, 0.1)
    got = O.cluster_pinned(row, col, r, a, n_rows, n_cols, k, np.full((n_rows, 1), O.MISSING, np.uint8), 200)
    want = CO.cluster(row, col, r, a, n_rows, n_cols, k)
    for f in ("best_restart", "rows_used", "restart_score", "restart_iters"):
        assert np.array_equal(got[f], want[f]), f
    # the same clusters in another order: match the columns of alt_w / depth_w
    cols = [next(j for j in range(k) if np.array_equal(got["depth_w"][:, i], want["depth_w"][:, j])) for i in range(k)]
    assert sorted(cols) == list(range(k)) and np.array_equal(got["alt_w"], want["alt_w"][:, cols])
    assert np.array_equal(got["ll"][:, :k], want["ll"][:, cols])


# ---- the restatement on the pools -----------------------------------------------------------------------------------------
# The pools read every molecule 1 to 3 times, so the model's counts are molecules: the calls after the UMI collapse (--umi).
PINNED = ("D0", "D2", "D4")
DECOY = ("decoy_hwe", "D0")


@pytest.fixture(scope="module")
def pools(tmp_path_factory):
    out = {}
    for rho in GC.RHOS:
        p = GC.write_pool(str(tmp_path_factory.mktemp(f"cp_{rho}")), rho)
        keys, row, col, alt, ref = DO.coverage_counts(p["vcf_match"], p["bam"], p["fasta"], p["barcodes"], umi=True)
        keys = [k.decode() if isinstance(k, bytes) else k for k in keys]
        samples, dosage = DO.read_genotypes(p["vcf_match"])
        n_rows = dosage.shape[0]
        m = int(round(rho * 1000))

        def run(known, k, mm, e=(row, col, ref, alt), keys=keys, samples=samples, dosage=dosage):
            res = O.cluster_pinned(*e, len(dosage), len(keys), k, DO.select(samples, dosage, list(known))[1], mm)
            return O.clusters_text(keys, res, known)
        out[rho] = dict(p, keys=keys, truth=json.load(open(p["truth"])), m=m, run=run,
                        free=CO.clusters_text(keys, CO.cluster(row, col, ref, alt, n_rows, len(keys), 6)),
                        pinned=run(PINNED, 6, m), decoy=run(DECOY, 7, m))
    return out


def _quality(text, truth, known):
    """-> (deep singlets on their donor's cluster, singlets called singlet on another donor's cluster, true doublets called
    doublet, deep singlets called doublet).  A pinned cluster must carry its donor's name; the free clusters are matched to the
    other donors by the Hungarian algorithm on the singlet calls.  Deep: >= 100 molecules."""
    calls = CO.calls(text)
    donors = [f"D{d}" for d in range(AC.N_DONORS)]
    other = [d for d in donors if d not in known]
    free = sorted({a for _, _, c, a in calls if c == "singlet" and a not in known})
    n = np.zeros((len(free), len(other)))
    for bc, _, c, a in calls:
        t = truth[bc]
        if c == "singlet" and a in free and t["kind"] == "singlet" and t["donors"][0] in other:
            n[free.index(a), other.index(t["donors"][0])] += 1
    match = {x: x for x in known}
    match.update({free[i]: other[j] for i, j in zip(*linear_sum_assignment(-n))})
    deep = wrong = dbl = deep_dbl = 0
    for bc, _, c, a in calls:
        t = truth[bc]
        if t["kind"] == "singlet":
            wrong += c == "singlet" and match.get(a) != t["donors"][0]
            if t["molecules"] >= 100:
                deep += c == "singlet" and match.get(a) == t["donors"][0]
                deep_dbl += c == "doublet"
        dbl += t["kind"] == "doublet" and c == "doublet"
    return deep, wrong, dbl, deep_dbl


N_DEEP = 126            # singlets of >= 100 molecules in every pool
# (§5g at K = 6, D0 / D2 / D4 pinned at K = 6 with rho given as the truth, decoy_hwe + D0 pinned at K = 7 with rho the truth)
QUALITY = {0.0: ((126, 0, 0, 0), (126, 0, 12, 0), (126, 0, 8, 0)),
           0.05: ((126, 0, 1, 0), (126, 0, 8, 0), (126, 0, 5, 0)),
           0.15: ((126, 0, 1, 0), (126, 0, 5, 0), (126, 0, 4, 0)),
           0.3: ((53, 84, 0, 0), (125, 0, 3, 0), (109, 16, 1, 1))}


@pytest.mark.parametrize("rho", GC.RHOS)
def test_quality_on_the_pools(pools, rho):
    p = pools[rho]
    free, pinned, decoy = (_quality(p[f], p["truth"], kn) for f, kn in (("free", ()), ("pinned", PINNED), ("decoy", DECOY)))
    assert (free, pinned, decoy) == QUALITY[rho]
    # the bars: every deep singlet on its donor's cluster (at most one miss at 0.3), no singlet on another donor's cluster, at
    # least as many true doublets as §5g
    assert pinned[0] >= N_DEEP - (rho == 0.3) and pinned[1] == 0 and pinned[2] >= free[2]
    # the decoy sample is not in the pool: no cell is called singlet on its cluster
    assert not any(c == "singlet" and a == "decoy_hwe" for _, _, c, a in CO.calls(p["decoy"]))
    # the pinned clusters carry their samples' names, the free ones C0 ..
    assert CO.calls(p["pinned"]) and p["pinned"].split("\n")[0].endswith("\tll_D0\tll_D2\tll_D4\tll_C0\tll_C1\tll_C2")


def test_rho_given_as_zero_calls_deep_singlets_doublet(pools):
    """at 15 % ambient RNA, pinned clusters that expect no ambient RNA call 11 deep singlets doublet: the model needs rho"""
    p = pools[0.15]
    assert _quality(p["run"](PINNED, 6, 0), p["truth"], PINNED) == (115, 1, 6, 11)


# ---- the CLI's files ------------------------------------------------------------------------------------------------------
def test_alleles_text_names_the_clusters(pools):
    res = dict(k=3, alt_w=np.array([[1 << 16, 0, 3 << 15]]), depth_w=np.array([[2 << 16, 0, 1 << 17]]), row_used=np.array([1], np.uint8))
    text = O.alleles_text(["chrA_10"], res, ["S1"])
    assert text == "variant\tused\tref_S1\talt_S1\tref_C0\talt_C0\tref_C1\talt_C1\nchrA_10\t1\t1.0000\t1.0000\t0.0000\t0.0000\t0.5000\t1.5000\n"
    assert text.split("\n", 1)[1] == CO.alleles_text(["chrA_10"], res).split("\n", 1)[1]


# ---- refusals: all of them before any GPU work (this machine may have none) ----------------------------------------------
def _cli(tmp_path, p, *extra):
    return subprocess.run([CLI, "-v", p["vcf_match"], "-b", p["bam"], "-f", p["fasta"], "-c", p["barcodes"], "-o", str(tmp_path / "o.mtx"),
                           *extra], cwd=str(tmp_path), capture_output=True, text=True)


def _refused(r, tmp_path, *words, keep=()):
    assert r.returncode == 1, r.stdout + r.stderr
    for w in words:
        assert w in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(keep)


CL = ["--out-clusters", "c.tsv", "--clusters", "4"]


@pytest.mark.parametrize("extra,words", [
    (["--known-donors", "D0"], ["--known-donors", "--out-clusters"]),
    ([*CL, "--known-donors", "D0,D9"], ["--known-donors", "'D9'", "not a sample"]),
    ([*CL, "--known-donors", "D0,D1,D0"], ["--known-donors", "'D0'", "twice"]),
    ([*CL, "--known-donors", "D0,,D1"], ["--known-donors", "empty"]),
    ([*CL, "--known-donors", ""], ["--known-donors", "at least one"]),
    ([*CL, "--known-donors", "D0,D1,D2,D3"], ["--known-donors", "4 samples", "1 to 3"]),
    (["--out-clusters", "c.tsv", "--clusters", "3", "--known-donors", "C1"], ["--known-donors", "'C1'", "free cluster"]),
    ([*CL, "--known-donors", "D0", "--ambient-rna", "estimate"], ["--known-donors", "--ambient-rna estimate"]),
    ([*CL, "--known-donors", "D0", "--ambient-rna", "0.1", "--out-ambient", "a.tsv"], ["--out-ambient", "--out-donors"]),
    ([*CL, "--known-donors", "D0", "--out-cluster-genotypes", "g.vcf"], ["--known-donors", "--out-cluster-genotypes"]),
    ([*CL, "--known-donors", "D0", "--out-cluster-matches", "m.tsv"], ["--known-donors", "--out-cluster-matches"]),
    ([*CL, "--known-donors", "D0", "--out-cluster-calls", "x.tsv"], ["--known-donors", "--out-cluster-calls"]),
    ([*CL, "--known-donors", "D0", "--dump-staged", "s"], ["--known-donors", "--dump-staged"]),
    ([*CL, "--known-donors", "D0", "--ambient-rna", "0.6"], ["--ambient-rna"]),
])
def test_bad_options_are_refused(tmp_path, pools, extra, words):
    _refused(_cli(tmp_path, pools[0.0], *extra), tmp_path, *words)


def test_ambient_rna_without_donors_or_known_donors_is_refused(tmp_path, pools):
    _refused(_cli(tmp_path, pools[0.0], *CL, "--ambient-rna", "0.1"), tmp_path, "--ambient-rna", "--out-donors", "--known-donors")


@pytest.mark.parametrize("which", ["c.tsv", "a.tsv"])
def test_existing_output_path_is_refused(tmp_path, pools, which):
    (tmp_path / which).write_text("keep me\n")
    r = _cli(tmp_path, pools[0.0], "--out-clusters", str(tmp_path / "c.tsv"), "--clusters", "4", "--known-donors", "D0",
             "--out-cluster-alleles", str(tmp_path / "a.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / which).read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == [which]


def test_help_and_readme_list_the_flag():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    readme = open(os.path.join(ROOT, "README.md")).read()
    assert "--known-donors" in r.stdout and "--known-donors" in readme
    assert "--ambient-rna MODE      With --out-donors or --known-donors" in r.stdout
