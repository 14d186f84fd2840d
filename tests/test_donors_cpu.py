"""`--out-donors` without a GPU: the restatement (tests/donor_oracle.py) recovers the pooled cases' truth
(tests/donor_cases.py), its invariants hold, the engine's per-slot bodies (tests/donor_shim.cpp) equal NumPy, the CLI's GT
parser (tests/gt_shim.cpp) equals the restatement's, and the CLI refuses bad donor options before any GPU work."""
import ctypes
import functools
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import donor_cases as DC
import donor_oracle as O

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
KEYS = {"plain": {}, "umi": dict(umi=True), "mates": dict(collapse_mates=True)}
FILTER_KW = dict(mapq=30, primary_only=True, no_duplicates=True, min_base_quality=20)
# With the committed seed, every singlet with at least N_SINGLET usable REF + ALT counts and every doublet with at least
# N_DOUBLET is called right in every key mode, with and without the filters (about half the singlets and two thirds of the
# doublets lie above them); thinner cells may be unassigned or wrong.
N_SINGLET, N_DOUBLET = 40, 100


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    return DC.write_cases(str(tmp_path_factory.mktemp("donors")))


def _files(p):
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@functools.lru_cache(maxsize=None)
def _expected(files, keys, filtered):
    return O.expected(*files, donors=DC.DONORS, **KEYS[keys], **(FILTER_KW if filtered else {}))


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("keys", list(KEYS))
def test_restatement_recovers_truth(pool, keys, filtered):
    text, *_ = _expected(_files(pool), keys, filtered)
    truth = json.load(open(pool["truth"]))
    lines = text.splitlines()
    assert lines[0].split("\t")[-6:] == [f"ll_{n}" for n in DC.DONORS]
    called = {"singlet": 0, "doublet": 0}
    seen = set()
    for ln in lines[1:]:
        f = ln.split("\t")
        t = truth[f[0]]
        seen.add(f[0])
        usable = int(f[2]) + int(f[3])
        if t["kind"] == "empty":
            assert f[1:6] == ["0", "0", "0", "unassigned", "."], ln
        elif t["kind"] == "singlet" and usable >= N_SINGLET:
            assert (f[4], f[5]) == ("singlet", t["donors"][0]), ln
            called["singlet"] += 1
        elif t["kind"] == "doublet" and usable >= N_DOUBLET:
            assert (f[4], f[5]) == ("doublet", "+".join(t["donors"])), ln
            called["doublet"] += 1
    assert seen == set(truth)
    assert called["singlet"] >= 40 and called["doublet"] >= 5, called


@pytest.mark.parametrize("keys", list(KEYS))
def test_invariants(pool, keys):
    files = _files(pool)
    text, ll, cnt, names = _expected(files, keys, False)
    samples, dosage = O.read_genotypes(files[0])
    usable = np.all(O.select(samples, dosage, DC.DONORS)[1] != O.MISSING, axis=1)
    keys_, row, col, alt, ref = O.coverage_counts(*files, **KEYS[keys])
    m = usable[row] & (alt + ref > 0)
    want_ref = np.bincount(col[m], weights=ref[m], minlength=len(keys_)).astype(np.int64)
    want_alt = np.bincount(col[m], weights=alt[m], minlength=len(keys_)).astype(np.int64)
    want_var = np.bincount(col[m], minlength=len(keys_))
    lines = text.splitlines()[1:]
    assert len(lines) == len(keys_)
    for c, ln in enumerate(lines):
        f = ln.split("\t")
        assert (int(f[1]), int(f[2]), int(f[3])) == (want_var[c], want_ref[c], want_alt[c]), ln
        if cnt[c][0] == 0:
            assert all(v == 0 for v in ll[c]) and f[4] == "unassigned" and f[5] == "."
    # the edge rows: 0, 1, 5, 6 and 7 (multi-allelic, D2 is 1/2, never scored) are not usable, 2, 3, 4, 8, 9 are
    assert [bool(usable[r]) for r in range(10)] == [False, False, True, True, True, False, False, False, True, True]
    assert not (row == 7).any() and (row == 8).any()


# ---- the engine's per-slot bodies against NumPy -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dshim") / "libdonor_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "donor_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


@pytest.mark.parametrize("eps", [1e-6, 0.01, 0.25])
def test_tables_equal_python(shim, eps):
    lr, la = np.zeros(5, np.int64), np.zeros(5, np.int64)
    shim.vtx_test_donor_tables(ctypes.c_double(eps), _p(lr), _p(la))
    assert (lr.tolist(), la.tolist()) == O.tables(eps)


@pytest.mark.parametrize("d", [2, 17, 32])
def test_hypothesis_order(shim, d):
    h = d + d * (d - 1) // 2
    d1, d2 = np.zeros(h, np.uint32), np.zeros(h, np.uint32)
    shim.vtx_test_hyp_donors(ctypes.c_uint32(d), _p(d1), _p(d2))
    assert list(zip(d1.tolist(), d2.tolist())) == O.hypotheses(d)


@pytest.mark.parametrize("eps", [1e-6, 0.25])
@pytest.mark.parametrize("d", [2, 17, 32])
def test_slot_bodies_equal_numpy(shim, d, eps):
    """H = 3, 153, 528 hypotheses (across the 32-lane multiples), counts up to 2^20, missing dosages, rows outside the table,
    unlisted columns and zero-count slots."""
    rng = np.random.default_rng(d * 7 + int(eps * 1e6))
    n_rows, n_loci, n_cols, n_slots = 60, 50, 40, 3000
    dosage = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    dosage[rng.random((n_rows, d)) < 0.01] = O.MISSING
    usable = np.all(dosage != O.MISSING, axis=1).astype(np.uint8)
    locus_row = rng.integers(0, n_rows + 3, n_loci).astype(np.uint32)        # a few loci beyond the table
    cslot_locus = rng.integers(0, n_loci, n_slots).astype(np.uint32)
    cslot_col = rng.integers(0, n_cols, n_slots).astype(np.uint32)
    cslot_col[rng.random(n_slots) < 0.05] = 0xFFFFFFFF
    ccnt = np.zeros((n_slots, 4), np.uint32)
    ccnt[:, :3] = rng.integers(0, 1 << 20, (n_slots, 3))
    ccnt[rng.random(n_slots) < 0.5, :2] //= 1 << 18                          # small counts too
    ccnt[rng.random(n_slots) < 0.05, :2] = 0
    H = d + d * (d - 1) // 2
    ll, cnt = np.zeros((n_cols, H), np.int64), np.zeros((n_cols, 3), np.uint64)
    n = shim.vtx_test_donor_ll(ctypes.c_uint32(n_slots), _p(cslot_col), _p(cslot_locus), _p(locus_row), _p(ccnt), _p(dosage), _p(usable),
                               ctypes.c_uint64(n_rows), ctypes.c_uint32(n_cols), ctypes.c_uint32(d), ctypes.c_double(eps), _p(ll), _p(cnt))
    # NumPy: every qualifying slot's contribution, per hypothesis
    row = locus_row[cslot_locus].astype(np.int64)
    r, a = ccnt[:, 0].astype(np.int64), ccnt[:, 1].astype(np.int64)
    ok = (cslot_col < n_cols) & (row < n_rows)
    ok[ok] &= usable[row[ok]] == 1
    ok &= r + a > 0
    assert n == ok.sum()
    lr, la = (np.asarray(t, np.int64) for t in O.tables(eps))
    hyp = np.asarray(O.hypotheses(d))
    g = dosage[row[ok]].astype(np.int64)
    s = g[:, hyp[:, 0]] + g[:, hyp[:, 1]]                                   # [slot][H]
    contrib = r[ok, None] * lr[s] + a[ok, None] * la[s]
    want = np.zeros((n_cols, H), np.int64)
    np.add.at(want, cslot_col[ok].astype(np.int64), contrib)
    assert np.array_equal(ll, want)
    want_cnt = np.zeros((n_cols, 3), np.int64)
    np.add.at(want_cnt, cslot_col[ok].astype(np.int64), np.stack([np.ones(ok.sum(), np.int64), r[ok], a[ok]], 1))
    assert np.array_equal(cnt.astype(np.int64), want_cnt)


# ---- the CLI's GT parser against the restatement's -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def gt_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gtshim") / "libgt_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "gt_shim.cpp"), "-lz"], check=True)
    return ctypes.CDLL(so)


def _cli_genotypes(gt_shim, vcf, out):
    rc = gt_shim.vtx_test_read_genotypes(vcf.encode(), out.encode())
    text = open(out).read()
    if rc:
        return rc, text
    lines = text.split("\n")[:-1]
    samples = lines[0].split("\t") if lines[0] else []
    return 0, (samples, np.asarray([[int(x) for x in ln.split(",")] if ln else [] for ln in lines[1:]], np.uint8).reshape(len(lines) - 1, len(samples)))


def test_gt_parser_equals_python(gt_shim, pool, tmp_path):
    rc, (samples, dosage) = _cli_genotypes(gt_shim, pool["vcf"], str(tmp_path / "g.txt"))
    ps, pd = O.read_genotypes(pool["vcf"])
    assert rc == 0 and samples == ps == DC.NAMES and np.array_equal(dosage, pd)
    # the edge rows as the docstring of donor_cases states them
    i = {n: k for k, n in enumerate(DC.NAMES)}
    assert dosage[0, i["D1"]] == dosage[1, i["D4"]] == dosage[6, i["D3"]] == dosage[7, i["D2"]] == dosage[9, i["X"]] == O.MISSING
    assert dosage[2, i["D2"]] == 1 and dosage[3, i["D0"]] == 2 and dosage[3, i["D5"]] == 0
    assert (dosage[5] == O.MISSING).all() and (dosage[8] == 1).all() and (dosage[4] != O.MISSING).all()


def test_gt_parser_edge_values(gt_shim, tmp_path):
    """Every GT form the model names, in one VCF, both parsers."""
    gts = ["0/0", "0/1", "1/0", "1/1", "0|1", "1|1", "0", "1", ".", "./.", ".|.", "0/.", "1/2", "2/2", "0/1/1", "", "01", "0//1", "a/b"]
    vcf = tmp_path / "e.vcf"
    names = [f"S{k}" for k in range(len(gts))]
    vcf.write_text("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(names) + "\n"
                   "c\t1\t.\tA\tC\t.\t.\t.\tGT\t" + "\t".join(gts) + "\n"
                   "c\t2\t.\tA\tC\t.\t.\t.\tGQ:DP:GT\t" + "\t".join(f"9:3:{g}" for g in gts) + "\n"
                   "c\t3\t.\tA\tC\t.\t.\t.\tGQ:GT:DP\t" + "\t".join(["9"] * len(gts)) + "\n")
    rc, (samples, dosage) = _cli_genotypes(gt_shim, str(vcf), str(tmp_path / "g.txt"))
    ps, pd = O.read_genotypes(str(vcf))
    assert rc == 0 and samples == ps and np.array_equal(dosage, pd)
    M = O.MISSING
    assert dosage[0].tolist() == dosage[1].tolist() == [0, 1, 1, 2, 1, 2, 0, 2] + [M] * 11
    assert (dosage[2] == M).all()


def test_gt_parser_refuses_a_short_record(gt_shim, tmp_path):
    vcf = tmp_path / "m.vcf"
    vcf.write_text("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tA\tB\nc\t1\t.\tA\tC\t.\t.\t.\tGT\t0/1\n")
    rc, text = _cli_genotypes(gt_shim, str(vcf), str(tmp_path / "g.txt"))
    assert rc == 1 and "malformed VCF line" in text
    with pytest.raises(ValueError, match="malformed VCF line"):
        O.read_genotypes(str(vcf))


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
    (["--donors", "D0,D1,Z9"], ["'Z9' is not a sample column"]),
    (["--donors", "D0,D1,D0"], ["'D0' is listed twice"]),
    (["--donors", "D3"], ["2 to 32 donors, not 1"]),
    (["--donor-error-rate", "0.3"], ["--donor-error-rate", "0.3"]),
    (["--donor-error-rate", "1e-7"], ["--donor-error-rate"]),
    (["--donor-error-rate", "x"], ["--donor-error-rate"]),
])
def test_bad_donor_options_are_refused(tmp_path, pool, extra, words):
    _refused(_cli(tmp_path, _files(pool), "--out-donors", str(tmp_path / "d.tsv"), *extra), tmp_path, *words)


def test_too_few_and_too_many_samples_are_refused(tmp_path, pool):
    T = REF_TEST_DIR          # the reference's DNA fixture has one sample column
    dna = (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv")
    _refused(_cli(tmp_path, dna, "--out-donors", str(tmp_path / "d.tsv")), tmp_path, "2 to 32 donors, not 1", "--donors")
    many = tmp_path / "many"
    many.mkdir()
    vcf = many / "v.vcf"
    vcf.write_text("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(f"S{k}" for k in range(33)) + "\n")
    _refused(_cli(many, (str(vcf), *_files(pool)[1:]), "--out-donors", str(many / "d.tsv")), many, "2 to 32 donors, not 33",
             keep=["v.vcf"])


def test_options_without_out_donors_are_refused(tmp_path, pool):
    _refused(_cli(tmp_path, _files(pool), "--donors", "D0,D1"), tmp_path, "--out-donors")
    _refused(_cli(tmp_path, _files(pool), "--donor-error-rate", "0.02"), tmp_path, "--out-donors")


def test_refused_with_dump_staged(tmp_path, pool):
    _refused(_cli(tmp_path, _files(pool), "--out-donors", str(tmp_path / "d.tsv"), "--dump-staged", str(tmp_path / "s")), tmp_path,
             "--out-donors", "--dump-staged")


def test_existing_output_path_is_refused(tmp_path, pool):
    (tmp_path / "d.tsv").write_text("keep me\n")
    r = _cli(tmp_path, _files(pool), "--out-donors", str(tmp_path / "d.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / "d.tsv").read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == ["d.tsv"]


def test_help_and_readme_list_the_flags():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    readme = open(os.path.join(ROOT, "README.md")).read()
    for flag in ("--out-donors", "--donors", "--donor-error-rate"):
        assert flag in r.stdout and flag in readme
