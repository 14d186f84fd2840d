"""`--out-cluster-genotypes` / `--out-cluster-matches` without a GPU: the engine's fit, call and match bodies
(tests/cluster_gt_shim.cpp) equal the restatement (tests/cluster_gt_oracle.py) bit for bit, the whole chain on the seeded
ambient pools (C oracle counts -> cluster_oracle.cluster -> the restatement) recovers rho, the donors' genotypes and the
cluster-to-donor match, and the CLI refuses bad options before any GPU work."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import ambient_oracle as AO
import cluster_gt_cases as GC
import cluster_gt_oracle as O
import cluster_oracle as CO
import donor_oracle as DO

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
EPS = (1e-6, 0.25)
MS = (0, 1, 499, 500)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cgshim") / "libcluster_gt_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cluster_gt_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------
def _rows(rng, n, k):
    """alt_w / depth_w [n, k] with zeros, 2^51, alt = 0 and alt = depth, and row sums with their extremes"""
    T = rng.integers(0, 1 << 40, (n, k))
    T[rng.random((n, k)) < 0.2] = 0
    T[0, :] = 0
    T[1, :] = 1 << 51
    T[2, 0] = 1 << 51
    A = (T * rng.random((n, k))).astype(np.int64)
    A[1, 0] = 0
    A[1, -1] = T[1, -1]
    A[3] = T[3]
    rd = np.concatenate([[0, (1 << 53) - 3, (1 << 53) - 3, 1], rng.integers(0, 1 << 30, n - 4)]).astype(np.uint64)
    ra = np.concatenate([[0, 0, (1 << 53) - 3, 1], [rng.integers(0, int(t) + 1) for t in rd[4:]]]).astype(np.uint64)
    return A.astype(np.int64), T.astype(np.int64), ra, rd


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("k", [2, 17, 32])
def test_fit_and_call_equal_restatement(shim, k, eps):
    rng = np.random.default_rng(k)
    n = 300
    A, T, ra, rd = _rows(rng, n, k)
    for m in MS:
        L = np.zeros((n, 6), np.int32)
        shim.vtx_test_cg_logs(ctypes.c_double(eps), ctypes.c_uint32(m), ctypes.c_uint32(n), _p(ra), _p(rd), _p(L))
        la, lr = O.logs(m, ra.astype(np.int64), rd.astype(np.int64), eps)
        assert np.array_equal(L[:, 0::2], la) and np.array_equal(L[:, 1::2], lr), m
        wla, wlr = AO.tables(m, ra.astype(np.int64), rd.astype(np.int64), eps)          # §5h's s = 0, 2, 4
        assert np.array_equal(la, wla[:, [0, 2, 4]]) and np.array_equal(lr, wlr[:, [0, 2, 4]])
        ll, mx = np.zeros((n, k, 3), np.int64), np.zeros((n, k), np.int64)
        shim.vtx_test_cg_fit(ctypes.c_uint32(n), ctypes.c_uint32(k), _p(L), _p(A), _p(T), _p(ll), _p(mx))
        want = O.lls(m, A, T, ra, rd, eps)
        assert np.array_equal(ll, want) and np.array_equal(mx, want.max(axis=2)), m
        for i in (0, 1, 2, 3, 17):                                # the split product equals the Python-int one
            for j in range(k):
                for g in range(3):
                    assert int(want[i, j, g]) == O.ll_int(int(A[i, j]), int(T[i, j]), int(la[i, g]), int(lr[i, g]))
        gt, pl, gq = np.zeros((n, k), np.uint8), np.zeros((n, k, 3), np.uint32), np.zeros((n, k), np.uint32)
        shim.vtx_test_cg_call(ctypes.c_uint32(n), ctypes.c_uint32(k), _p(ll), _p(T), _p(gt), _p(pl), _p(gq))
        wgt, wpl = O.call(want, T)
        assert np.array_equal(gt, wgt) and np.array_equal(pl.astype(np.int64), wpl) and np.array_equal(gq.astype(np.int64), O.gq(wpl)), m
        assert (gt[0] == O.MISSING).all() and (pl[0] == 0).all()
        assert (pl.max(axis=2) == O.MAX_PL).any()                 # the 2^51 rows saturate


def test_phred_equals_the_128_bit_expression(shim):
    sat = -(-(O.MAX_PL * O.L10 - O.L10 // 2) // 10)               # the smallest d whose quotient reaches 2^31 - 1
    d = [0, 1, O.L10 // 20, O.L10 // 20 + 1, O.L10 // 10, O.L10, sat - 1, sat, sat + 1, (1 << 54) - 1, 1 << 54, (1 << 63) - 1]
    d += np.random.default_rng(3).integers(0, 1 << 62, 2000).tolist()
    x = np.asarray(d, np.int64)
    out = np.zeros(x.size, np.uint32)
    shim.vtx_test_cg_phred(ctypes.c_uint32(x.size), _p(x), _p(out))
    want = [O.phred_int(v) for v in d]
    assert out.tolist() == want == O.phred(x).tolist()
    assert want[6] == O.MAX_PL - 1 and want[7] == O.MAX_PL


@pytest.mark.parametrize("s", [1, 2, 33])
@pytest.mark.parametrize("k", [2, 17, 32])
def test_match_equals_restatement(shim, k, s):
    rng = np.random.default_rng(100 * k + s)
    n = 400
    A, T, ra, rd = _rows(rng, n, k)
    A, T = A >> 20, T >> 20                                       # depths where GQ lands on both sides of 20
    ll = O.lls(250, A, T, ra, rd, 0.01)
    gt, pl = O.call(ll, T)
    g = rng.integers(0, 3, (n, s)).astype(np.uint8)
    M, disc, pl32 = np.zeros((k, s), np.int64), np.zeros((k, s), np.uint64), pl.astype(np.uint32)
    shim.vtx_test_cg_match(ctypes.c_uint32(n), ctypes.c_uint32(k), ctypes.c_uint32(s), _p(ll), _p(gt), _p(pl32), _p(g), _p(M), _p(disc))
    wM, wd, wrows, wcalled = O.match(ll, gt, pl, T, g)
    assert np.array_equal(M, wM) and np.array_equal(disc.astype(np.int64), wd)
    called = np.ascontiguousarray(wcalled, np.uint64)
    assert 0 < called.sum() < (T > 0).sum()
    # the assignment rule, with ties and the llr threshold at its seam
    M[0, :] = 7
    if s > 1:
        M[1, 1] = M[1, 0] + O.MIN_LLR
        M[1, 2:] = M[1, 0]
    out, llr = np.zeros((k, 4), np.uint32), np.zeros(k, np.int64)
    disc = np.ascontiguousarray(disc)
    shim.vtx_test_cg_assign(ctypes.c_uint32(k), ctypes.c_uint32(s), _p(M), _p(disc), _p(called), _p(out), _p(llr))
    for j in range(k):
        best, second, l, ok = O.assign(M[j].tolist(), disc[j].tolist(), int(called[j]))
        assert (out[j, 0], out[j, 2]) == (best, int(ok)), j
        assert s == 1 and (out[j, 1], llr[j]) == (best, 0) or (out[j, 1], llr[j]) == (second, l), j
    assert out[0, 0] == 0 and (s == 1 or out[0, 1] == 1)
    if s > 1:
        assert out[1, 0] == 1 and llr[1] == O.MIN_LLR


def _plurality(calls, truth):
    """-> {cluster: the donor most of its singlet calls come from}.  Equal to cluster_cases.match_clusters' Hungarian matching
    on the pools up to rho = 0.15; at 0.3 the EM's clusters are mixtures and two of them are mostly D0's cells."""
    from collections import Counter
    n = Counter((a, truth[bc]["donors"][0]) for bc, _, call, a in calls if call == "singlet" and truth[bc]["kind"] == "singlet")
    return {c: max((x for x in n if x[0] == c), key=lambda x: (n[x], x[1]))[1] for c in {a for a, _ in n}}


# ---- the whole chain on the pools -----------------------------------------------------------------------------------------
# The pools read every molecule 1 to 3 times, so the model's counts are molecules: the calls after the UMI collapse (--umi).
@pytest.fixture(scope="module")
def pools(tmp_path_factory):
    out = {}
    for rho in GC.RHOS:
        p = GC.write_pool(str(tmp_path_factory.mktemp(f"cg_{rho}")), rho)
        keys, row, col, alt, ref = DO.coverage_counts(p["vcf"], p["bam"], p["fasta"], p["barcodes"], umi=True)
        recs = O.records(p["vcf_match"])
        cl = CO.cluster(row, col, ref, alt, len(recs), len(keys), len(p["donors"]))
        A, T = O.row_sums(row, ref, alt, len(recs))
        truth = json.load(open(p["truth"]))
        match = _plurality(CO.calls(CO.clusters_text(keys, cl)), truth)
        keys = [k.decode() if isinstance(k, bytes) else k for k in keys]
        out[rho] = dict(p, keys=keys, cl=cl, A=A, T=T, recs=recs, truth=truth, match=match, counts=(keys, row, col, alt, ref))
    return out


def _fit(p, vcf="vcf_match", rho=None):
    samples, dosage = DO.read_genotypes(p[vcf])
    return samples, O.genotypes(p["cl"], p["A"], p["T"], dosage, O.ERROR_RATE, rho)


def _miscalls(p, res):
    """(rows with GQ >= 20 where GT is not the matched donor's true dosage, all such rows)"""
    _, truth = DO.read_genotypes(p["vcf"])
    g = truth[res["touched"].astype(np.int64)]
    called = O.gq(res["pl"]) >= O.MIN_GQ
    donor = [int(p["match"][f"C{j}"][1:]) for j in range(res["gt"].shape[1])]
    wrong = called & (res["gt"] != g[:, donor])
    return int(wrong.sum()), int(called.sum())


# m of the estimate on each pool.  It lies above the truth: the EM's cluster sums carry the doublets' molecules (and the soft
# weights of shallow cells), a mix of donors that the model can only read as ambient RNA (DESIGN.md §5i);
# test_singlet_sums_recover_rho shows the estimate within 0.03 once the sums hold the true singlets only.
ESTIMATES = {0.0: 79, 0.05: 121, 0.15: 212, 0.3: 480}
MISCALLS = {0.0: (4, 1853), 0.05: (6, 1548), 0.15: (2, 818), 0.3: (0, 30)}      # (wrong, called at GQ >= 20) at the estimate
MISCALLS_AT_ZERO = (646, 1997)                         # the rho = 0.3 pool fitted at rho = 0
SINGLET_ESTIMATES = {0.0: 10, 0.05: 54, 0.15: 171, 0.3: 295}


@pytest.mark.parametrize("rho", GC.RHOS)
def test_chain_recovers_genotypes(pools, rho):
    p = pools[rho]
    _, res = _fit(p)
    assert res["rho_permille"] == ESTIMATES[rho] > 1000 * rho
    m, j = res["grid_permille"].tolist(), res["grid_objective"].tolist()
    assert [x for x in m if x % 10 == 0] == AO.COARSE and j[m.index(res["rho_permille"])] == max(j)
    wrong, called = _miscalls(p, res)
    assert (wrong, called) == MISCALLS[rho]
    assert wrong <= 0.01 * called
    if rho < 0.3:                                      # at 0.3 the biased estimate leaves 30 of 3 600 genotypes at GQ >= 20
        assert called > 0.2 * res["gt"].size
    assert res["rows_fit"] == int(p["cl"]["row_used"].sum()) > 0


@pytest.mark.parametrize("rho", GC.RHOS)
def test_singlet_sums_recover_rho(pools, rho):
    """the estimator itself: cluster sums of the true singlets, each in its own donor's cluster, at weight 2^16"""
    p = pools[rho]
    keys, row, col, alt, ref = p["counts"]
    donor = np.array([int(p["truth"][k]["donors"][0][1:]) if p["truth"][k]["kind"] == "singlet" else -1 for k in keys])
    d = donor[np.asarray(col, np.int64)]
    keep = d >= 0
    n_rows = len(p["recs"])
    A = np.zeros((n_rows, 6), np.int64)
    T = np.zeros((n_rows, 6), np.int64)
    np.add.at(A, (np.asarray(row, np.int64)[keep], d[keep]), np.asarray(alt, np.int64)[keep] << 16)
    np.add.at(T, (np.asarray(row, np.int64)[keep], d[keep]), (np.asarray(alt, np.int64) + np.asarray(ref, np.int64))[keep] << 16)
    res = O.genotypes(dict(alt_w=A, depth_w=T, row_used=p["cl"]["row_used"]), p["A"], p["T"])
    assert res["rho_permille"] == SINGLET_ESTIMATES[rho]
    assert abs(res["rho_permille"] / 1000 - rho) <= 0.03


def test_fit_at_zero_miscalls_more(pools):
    p = pools[0.3]
    _, at_zero = _fit(p, rho=0)
    _, est = _fit(p)
    assert _miscalls(p, at_zero) == MISCALLS_AT_ZERO
    assert MISCALLS_AT_ZERO[0] > _miscalls(p, est)[0]


@pytest.mark.parametrize("rho", GC.RHOS)
def test_clusters_match_their_donors(pools, rho):
    p = pools[rho]
    samples, res = _fit(p)
    text = O.matches_text(samples, res).splitlines()
    assert text[0].split("\t")[:8] == ["cluster", "rows", "called", "best_sample", "discordant", "second_sample", "llr", "assignment"]
    for j, ln in enumerate(text[1:]):
        f = ln.split("\t")
        assert f[0] == f"C{j}" and f[3] == p["match"][f"C{j}"] and f[7] == f[3], ln
        assert float(f[6]) >= 5 and f[3] not in GC.DECOYS, ln
    # without D5's column, D5's cluster is unassigned and the others keep their donors
    samples5, res5 = _fit(p, "vcf_no_d5")
    for j, ln in enumerate(O.matches_text(samples5, res5).splitlines()[1:]):
        f = ln.split("\t")
        want = "." if p["match"][f"C{j}"] == "D5" else p["match"][f"C{j}"]
        assert f[7] == want, ln


def test_genotype_file_is_vcf_and_lists_the_reached_rows(pools):
    p = pools[0.15]
    _, res = _fit(p)
    text = O.genotypes_text(p["recs"], p["cl"], res)
    lines = text.splitlines()
    assert lines[0] == "##fileformat=VCFv4.2" and all(ln.startswith("##") for ln in lines[:8])
    head = lines[8].split("\t")
    assert head == ["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"] + [f"C{j}" for j in range(6)]
    alleles = CO.alleles_text(CO.variant_labels(p["vcf"]), p["cl"]).splitlines()[1:]
    reached = [i for i, ln in enumerate(alleles) if any(float(x) > 0 for x in ln.split("\t")[2:])]
    body = [ln.split("\t") for ln in lines[9:]]
    assert [int(f[1]) for f in body] == [int(p["recs"][v][1]) for v in reached] and len(body) == res["touched"].size
    for f in body:
        assert len(f) == 15 and f[2].startswith("rs") and f[5:7] == [".", "."] and f[7] in ("USED", ".") and f[8] == "GT:GQ:PL"
        for x in f[9:]:
            if x != "./.":
                gt, gq, pl = x.split(":")
                pls = [int(v) for v in pl.split(",")]
                assert gt in ("0/0", "0/1", "1/1") and pls[("0/0", "0/1", "1/1").index(gt)] == 0 and 0 <= int(gq) <= 99


# ---- refusals: all of them before any GPU work (this machine may have none) ----------------------------------------------
def _cli(tmp_path, p, *extra, vcf=None):
    return subprocess.run([CLI, "-v", vcf or p["vcf_match"], "-b", p["bam"], "-f", p["fasta"], "-c", p["barcodes"], "-o",
                           str(tmp_path / "o.mtx"), *extra], cwd=str(tmp_path), capture_output=True, text=True)


def _refused(r, tmp_path, *words, keep=()):
    assert r.returncode == 1, r.stdout + r.stderr
    for w in words:
        assert w in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(keep)


@pytest.mark.parametrize("flag", ["--out-cluster-genotypes", "--out-cluster-matches"])
def test_flags_need_out_clusters(tmp_path, pools, flag):
    _refused(_cli(tmp_path, pools[0.0], flag, "x.txt"), tmp_path, flag, "--out-clusters")


@pytest.mark.parametrize("flag", ["--out-cluster-genotypes", "--out-cluster-matches"])
def test_refused_with_dump_staged(tmp_path, pools, flag):
    _refused(_cli(tmp_path, pools[0.0], "--out-clusters", "c.tsv", "--clusters", "6", flag, "x.txt", "--dump-staged", "s"), tmp_path,
             flag, "--dump-staged")


@pytest.mark.parametrize("which", ["g.vcf", "m.tsv"])
def test_existing_output_path_is_refused(tmp_path, pools, which):
    (tmp_path / which).write_text("keep me\n")
    r = _cli(tmp_path, pools[0.0], "--out-clusters", str(tmp_path / "c.tsv"), "--clusters", "6", "--out-cluster-genotypes",
             str(tmp_path / "g.vcf"), "--out-cluster-matches", str(tmp_path / "m.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / which).read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == [which]


@pytest.mark.parametrize("n_samples", [0, 1025])
def test_sample_columns_are_checked(tmp_path, pools, n_samples):
    p = pools[0.0]
    src = tmp_path.parent / f"v_{n_samples}.vcf"
    with open(src, "w") as f:
        for ln in open(p["vcf"]):
            x = ln.rstrip("\n").split("\t")
            if ln.startswith("##"):
                f.write(ln)
            elif ln.startswith("#"):
                f.write("\t".join(x[:8] + (["FORMAT"] + [f"S{i}" for i in range(n_samples)] if n_samples else [])) + "\n")
            else:
                f.write("\t".join(x[:8] + (["GT"] + ["0/1"] * n_samples if n_samples else [])) + "\n")
    r = _cli(tmp_path, p, "--out-clusters", "c.tsv", "--clusters", "6", "--out-cluster-matches", "m.tsv", vcf=str(src))
    _refused(r, tmp_path, "--out-cluster-matches", "1 to 1024 sample columns", f"not {n_samples}")


def test_help_and_readme_list_the_flags():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    readme = open(os.path.join(ROOT, "README.md")).read()
    for flag in ("--out-cluster-genotypes", "--out-cluster-matches"):
        assert flag in r.stdout and flag in readme
