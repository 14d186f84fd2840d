"""`--out-cluster-calls` without a GPU: the engine's code, nine-entry log and score bodies (tests/cluster_refine_shim.cpp) equal
the restatement (tests/cluster_refine_oracle.py) bit for bit; on the seeded ambient pools the whole chain (C oracle counts ->
cluster_oracle.cluster -> the restatement) is pinned round by round, with the quality it reaches; and the CLI refuses bad
options before any GPU work."""
import ctypes
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

from conftest import ROOT
import ambient_oracle as AO
import cluster_cases as CC
import cluster_gt_cases as GC
import cluster_gt_oracle as GO
import cluster_oracle as CO
import cluster_refine_oracle as O
import donor_oracle as DO

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
EPS = (1e-6, 0.25)
MS = (0, 1, 499, 500)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("crshim") / "libcluster_refine_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cluster_refine_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _u32(*xs):
    return [np.ascontiguousarray(x, np.uint32) for x in xs]


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------
def _row_sums(rng, n):
    rd = np.concatenate([[0, (1 << 53) - 3, (1 << 53) - 3, 1], rng.integers(0, 1 << 30, n - 4)]).astype(np.uint64)
    ra = np.concatenate([[0, 0, (1 << 53) - 3, 1], [rng.integers(0, int(t) + 1) for t in rd[4:]]]).astype(np.uint64)
    return ra, rd


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("k", [2, 17, 32])
def test_bodies_equal_restatement(shim, k, eps):
    rng = np.random.default_rng(k)
    n_rows, n_cols = 300, 40
    ra, rd = _row_sums(rng, n_rows)
    # codes from GT / PL with GQ on both sides of 20, and rows with every code P
    gt = rng.integers(0, 3, (n_rows, k)).astype(np.uint8)
    pl = rng.integers(0, 45, (n_rows, k, 3)).astype(np.uint32)
    pl[np.arange(n_rows)[:, None], np.arange(k)[None, :], gt] = 0
    pl[::7] = 0
    code = np.zeros((n_rows, k), np.uint8)
    shim.vtx_test_cr_codes(ctypes.c_uint32(n_rows), ctypes.c_uint32(k), _p(gt), _p(pl), _p(code))
    assert np.array_equal(code, O.codes(gt, pl.astype(np.int64)))
    assert (code == O.P).any() and (code != O.P).any() and (code[::7] == O.P).all()
    # cells over every row; rows 3, 5, 8, ... are not scored
    sidx = np.where(np.arange(n_rows) % 3 == 2, -1, 0)
    sidx[sidx == 0] = np.arange(int((sidx == 0).sum()))
    scode = code[sidx >= 0]
    m_ent = 2000
    col = np.sort(rng.integers(0, n_cols, m_ent))
    row, r, a = rng.integers(0, n_rows, m_ent), rng.integers(0, 50, m_ent), rng.integers(0, 50, m_ent)
    start = np.searchsorted(col, np.arange(n_cols + 1)).astype(np.uint32)
    for m in MS:
        tab = np.zeros((n_rows, 9, 2), np.int32)
        shim.vtx_test_cr_logs9(ctypes.c_double(eps), ctypes.c_uint32(m), ctypes.c_uint32(n_rows), _p(ra), _p(rd), _p(tab))
        la, lr = O.logs9(m, ra.astype(np.int64), rd.astype(np.int64), eps)
        assert np.array_equal(tab[:, :, 0], la) and np.array_equal(tab[:, :, 1], lr), m
        la5, lr5 = AO.tables(m, ra.astype(np.int64), rd.astype(np.int64), eps)       # both called: §5h's row_logs
        assert np.array_equal(la[:, :5], la5) and np.array_equal(lr[:, :5], lr5)
        stab = np.ascontiguousarray(tab[sidx >= 0])
        H = k + k * (k - 1) // 2
        ll, cnt = np.zeros((n_cols, H), np.int64), np.zeros((n_cols, 3), np.uint64)
        rw, rr, aa, sx = _u32(row, r, a, np.where(sidx >= 0, sidx, 0xFFFFFFFF))
        shim.vtx_test_cr_score(ctypes.c_uint32(n_cols), ctypes.c_uint32(k), _p(start), _p(rw), _p(rr), _p(aa), _p(sx),
                               _p(np.ascontiguousarray(scode)), _p(stab), _p(ll), _p(cnt))
        wll, wcnt = O.score((row, col, r, a), sidx, scode, la[sidx >= 0], lr[sidx >= 0], k, n_cols)
        assert np.array_equal(ll, wll) and np.array_equal(cnt.astype(np.int64), wcnt), m


def test_entry_of_covers_the_nine_entries():
    c = np.arange(4)
    e = O.entry_of(c[:, None], c[None, :])
    assert e.tolist() == [[0, 1, 2, 5], [1, 2, 3, 6], [2, 3, 4, 7], [5, 6, 7, 8]]


# ---- the whole chain on the pools -----------------------------------------------------------------------------------------
# The pools read every molecule 1 to 3 times, so the model's counts are molecules: the calls after the UMI collapse (--umi).
@pytest.fixture(scope="module")
def pools(tmp_path_factory):
    out = {}
    for rho in GC.RHOS:
        p = GC.write_pool(str(tmp_path_factory.mktemp(f"cr_{rho}")), rho)
        keys, row, col, alt, ref = DO.coverage_counts(p["vcf"], p["bam"], p["fasta"], p["barcodes"], umi=True)
        keys = [k.decode() if isinstance(k, bytes) else k for k in keys]
        n_rows = len(CO.variant_labels(p["vcf"]))
        cl = CO.cluster(row, col, ref, alt, n_rows, len(keys), 6)
        res = O.refine(row, col, ref, alt, n_rows, len(keys), cl)
        out[rho] = dict(p, keys=keys, counts=(row, col, ref, alt), n_rows=n_rows, cl=cl, res=res, truth=json.load(open(p["truth"])))
    return out


def test_round0_is_the_cluster_genotypes_fit(pools):
    p = pools[0.15]
    row, col, ref, alt = p["counts"]
    r0 = O.refine(row, col, ref, alt, p["n_rows"], len(p["keys"]), p["cl"], max_rounds=0)
    g = GO.genotypes(p["cl"], *GO.row_sums(row, ref, alt, p["n_rows"]))
    assert r0["n_rounds"] == 1 and not r0["converged"] and r0["rho_permille"].tolist() == [g["rho_permille"]] == [212]
    for f in ("touched", "gt", "pl"):
        assert np.array_equal(r0[f], g[f]), f
    assert r0["round_labels"][0].tolist() == p["res"]["round_labels"][0].tolist()


# (rho per round, scored rows per round, [singlet, doublet, unassigned] per round, changed labels per round, converged)
ROUNDS = {
    0.0: ([79, 78, 74, 75, 74, 75, 74, 75, 74], [597, 594, 595, 594, 595, 594, 595, 594, 595],
          [[195, 0, 129], [189, 0, 135], [191, 0, 133], [189, 0, 135], [191, 0, 133], [189, 0, 135], [191, 0, 133], [189, 0, 135],
           [191, 0, 133]], [195, 6, 2, 2, 2, 2, 2, 2, 2], False),
    0.05: ([121, 99, 99, 95, 96, 95], [579, 569, 567, 569, 568, 568],
           [[172, 2, 150], [165, 3, 156], [166, 3, 155], [166, 3, 155], [167, 3, 154], [167, 3, 154]], [172, 7, 3, 2, 1, 0], True),
    0.15: ([212, 209, 196, 176, 142, 92, 163, 173, 31], [459, 369, 308, 271, 232, 208, 110, 58, 126],
           [[139, 0, 185], [110, 0, 214], [90, 0, 234], [72, 0, 252], [50, 0, 274], [30, 0, 294], [25, 0, 299], [19, 0, 305],
            [17, 0, 307]], [139, 29, 20, 18, 24, 22, 5, 6, 2], False),
    0.3: ([480, 0], [30, 0], [[0, 0, 324], [0, 0, 324]], [0, 0], True),
}


@pytest.mark.parametrize("rho", GC.RHOS)
def test_chain_is_pinned_round_by_round(pools, rho):
    res = pools[rho]["res"]
    ms, scored, calls, changed, converged = ROUNDS[rho]
    assert res["rho_permille"].tolist() == ms and res["rows_scored"].tolist() == scored
    assert res["calls"].tolist() == calls and res["changed"].tolist() == changed
    assert res["converged"] == converged and res["n_rounds"] == len(ms) <= O.MAX_ROUNDS + 1
    prev = np.full(len(pools[rho]["keys"]), O.NONE)
    for r, lab in enumerate(res["round_labels"]):             # the labels: singlets only, and `changed` counts their moves
        assert int((lab != O.NONE).sum()) == calls[r][0] and int((lab != prev).sum()) == changed[r]
        prev = lab
    assert zlib.crc32(np.asarray(res["label"], np.uint32).tobytes()) == LABEL_CRC[rho]


LABEL_CRC = {0.0: 3550546206, 0.05: 342693381, 0.15: 3289576245, 0.3: 3081013225}      # crc32 of the final labels (uint32)


def _quality(text, truth):
    """(deep singlets not on their donor's cluster, true doublets called doublet, singlets of >= 50 molecules called doublet)"""
    calls = CO.calls(text)
    match = CC.match_clusters(calls, truth, 6)
    deep = sum(1 for bc, _, call, a in calls if truth[bc]["kind"] == "singlet" and truth[bc]["molecules"] >= 100
               and not (call == "singlet" and match[a] == truth[bc]["donors"][0]))
    dbl = sum(call == "doublet" for bc, _, call, _ in calls if truth[bc]["kind"] == "doublet")
    s50 = sum(call == "doublet" for bc, _, call, _ in calls if truth[bc]["kind"] == "singlet" and truth[bc]["molecules"] >= 50)
    return deep, dbl, s50


# What the model reaches on the pools (DESIGN.md §5j, "What it does on the seeded pools").  The bars it was expected to meet:
# final rho within 0.03 of the truth up to 0.15, every singlet of >= 100 molecules on its donor's cluster, no fewer true
# doublets and no more deep singlets called doublet than §5g.  It meets the last everywhere and misses the others: the labelled
# set shrinks round by round (ROUNDS), because an unlabelled cell's molecules leave the next round's sums.
FINAL_RHO = {0.0: 74, 0.05: 95, 0.15: 31, 0.3: 0}
QUALITY = {0.0: ((0, 0, 0), (0, 0, 0)), 0.05: ((0, 1, 0), (1, 3, 0)), 0.15: ((0, 1, 0), (110, 0, 0)), 0.3: ((73, 0, 0), (126, 0, 0))}


@pytest.mark.parametrize("rho", GC.RHOS)
def test_quality_on_the_pools(pools, rho):
    p = pools[rho]
    res = p["res"]
    assert res["rho_permille"][-1] == FINAL_RHO[rho]
    g = CO.clusters_text(p["keys"], p["cl"])
    f = DO.text(CO.names(6), p["keys"], res["ll"].tolist(), res["counts"].tolist())
    q5g, q5j = _quality(g, p["truth"]), _quality(f, p["truth"])
    assert (q5g, q5j) == QUALITY[rho]
    assert q5j[2] <= q5g[2]                                   # no more deep singlets called doublet than §5g


# ---- refusals: all of them before any GPU work (this machine may have none) ----------------------------------------------
def _cli(tmp_path, p, *extra):
    return subprocess.run([CLI, "-v", p["vcf"], "-b", p["bam"], "-f", p["fasta"], "-c", p["barcodes"], "-o", str(tmp_path / "o.mtx"),
                           *extra], cwd=str(tmp_path), capture_output=True, text=True)


def _refused(r, tmp_path, *words, keep=()):
    assert r.returncode == 1, r.stdout + r.stderr
    for w in words:
        assert w in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(keep)


def test_flag_needs_out_clusters(tmp_path, pools):
    _refused(_cli(tmp_path, pools[0.0], "--out-cluster-calls", "x.tsv"), tmp_path, "--out-cluster-calls", "--out-clusters")


def test_refused_with_dump_staged(tmp_path, pools):
    _refused(_cli(tmp_path, pools[0.0], "--out-clusters", "c.tsv", "--clusters", "6", "--out-cluster-calls", "x.tsv", "--dump-staged", "s"),
             tmp_path, "--out-cluster-calls", "--dump-staged")


def test_existing_output_path_is_refused(tmp_path, pools):
    (tmp_path / "x.tsv").write_text("keep me\n")
    r = _cli(tmp_path, pools[0.0], "--out-clusters", str(tmp_path / "c.tsv"), "--clusters", "6", "--out-cluster-calls", str(tmp_path / "x.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / "x.tsv").read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == ["x.tsv"]


def test_help_and_readme_list_the_flag():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert "--out-cluster-calls" in r.stdout and "--out-cluster-calls" in open(os.path.join(ROOT, "README.md")).read()
