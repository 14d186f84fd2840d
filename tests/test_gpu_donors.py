"""GPU: `--out-donors` end to end and the engine's donor reduction (vtx_set_donors / vtx_donor_ll_get).

The CLI on the pooled cases file (tests/donor_cases.py) and on the reference's DNA fixture with its sample column replaced by
three seeded genotype columns, through host staging, --gpu-inflate and --gpu-stage, plain / --umi / --collapse-mates, with and
without the record filters and the floor, in the three modes, against the restatement (tests/donor_oracle.py) byte for byte;
in the same runs the matrices and metric lines equal a run without the flag.  Engine level: submits accumulate and the next
finish resets, the call-order and argument refusals, a row beyond the table, and a depth ladder against NumPy."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import donor_cases as DC
import donor_oracle as O

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
PATHS = {"host": [], "inflate": ["--gpu-inflate"], "stage": ["--gpu-stage"]}
KEYS = {"plain": ([], {}), "umi": (["--umi"], dict(umi=True)), "mates": (["--collapse-mates"], dict(collapse_mates=True))}
FILTER_ARGS = ["--mapq", "30", "--primary-alignments", "--no-duplicates", "--min-base-quality", "20"]
FILTER_KW = dict(mapq=30, primary_only=True, no_duplicates=True, min_base_quality=20)
POOL_DONORS = ["D5", "D0", "D3", "D1", "D4", "D2"]          # a subset (not X) in another order than the header's


@pytest.fixture(scope="module")
def pool(tmp_path_factory):
    p = DC.write_cases(str(tmp_path_factory.mktemp("pool")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@pytest.fixture(scope="module")
def dna3(tmp_path_factory):
    """the reference's DNA fixture, its one sample column replaced by three seeded GT columns"""
    T = REF_TEST_DIR
    rng = np.random.default_rng(77)
    out = []
    for ln in open(f"{T}/test_dna.vcf"):
        ln = ln.rstrip("\n")
        if ln.startswith("#CHROM"):
            ln = "\t".join(ln.split("\t")[:9] + ["S1", "S2", "S3"])
        elif not ln.startswith("#") and ln:
            f = ln.split("\t")
            gts = [("0/0", "0/1", "1/1")[int(g)] for g in rng.integers(0, 3, 3)]
            if rng.random() < 0.1:
                gts[int(rng.integers(0, 3))] = "./."
            ln = "\t".join(f[:8] + ["GT"] + gts)
        out.append(ln)
    vcf = str(tmp_path_factory.mktemp("dna3") / "v.vcf")
    open(vcf, "w").write("\n".join(out) + "\n")
    return (vcf, f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv")


@functools.lru_cache(maxsize=None)
def _expected(files, keys, filtered, donors, rate):
    return O.expected(*files, donors=list(donors) if donors else None, error_rate=rate, **KEYS[keys][1],
                      **(FILTER_KW if filtered else {}))[0]


def _run(tmp_path, files, mode, *extra, tag="r", donors_file=True):
    """-> (out text, ref text or None, metric lines, donors text or None, stderr)"""
    out, ref, dn = str(tmp_path / f"{tag}.mtx"), str(tmp_path / f"{tag}_ref.mtx"), str(tmp_path / f"{tag}.tsv")
    r = subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "-o", out, "--ref-matrix", ref, "-s", mode,
                        "--log-level", "info", *(["--out-donors", dn] if donors_file else []), *extra],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[INFO] Number of")]
    return (open(out).read(), open(ref).read() if mode == "coverage" else None, lines, open(dn).read() if donors_file else None,
            r.stderr)


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("which", ["pool", "dna3"])
def test_cli_matches_restatement(tmp_path, pool, dna3, which, path, keys, filtered):
    files = pool if which == "pool" else dna3
    donors, rate = (tuple(POOL_DONORS), 0.02) if which == "pool" else (None, 0.01)
    opts = (["--donors", ",".join(donors), "--donor-error-rate", str(rate)] if donors else [])
    common = ["--threads", "3", "--shard-loci", "4", *PATHS[path], *KEYS[keys][0], *(FILTER_ARGS if filtered else [])]
    want = _expected(files, keys, filtered, donors, rate)
    base = _run(tmp_path, files, "coverage", *common, tag="off", donors_file=False)
    for mode in ("consensus", "coverage", "alt_frac"):
        out, ref, lines, tsv, err = _run(tmp_path, files, mode, *common, *opts, tag=mode)
        assert tsv == want, mode
        assert lines == base[2], mode
        if mode == "coverage":
            assert (out, ref) == base[:2]
        calls = [ln.split("\t")[4] for ln in tsv.splitlines()[1:]]
        m = re.search(r"Donors: (\d+) .*cells: (\d+) singlet, (\d+) doublet, (\d+) unassigned", err)
        assert m and [int(x) for x in m.groups()] == [len(donors or (1, 2, 3)), calls.count("singlet"), calls.count("doublet"),
                                                      calls.count("unassigned")]
    assert "Donors:" not in base[4]


def test_flag_off_changes_nothing(tmp_path, pool):
    for path in ("host", "stage"):
        a = _run(tmp_path, pool, "coverage", "--threads", "1", "--shard-loci", "50", *PATHS[path], tag=f"{path}_a", donors_file=False)
        b = _run(tmp_path, pool, "coverage", "--threads", "1", "--shard-loci", "50", *PATHS[path], "--donors", "D0,D1", tag=f"{path}_b")
        assert a[:3] == b[:3]
        assert not os.path.exists(tmp_path / f"{path}_a.tsv")


def test_two_gpus_equal_one(tmp_path, pool):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path in ("host", "stage"):
        one = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", *PATHS[path], *FILTER_ARGS, tag=f"one_{path}")
        two = _run(tmp_path, pool, "coverage", "--threads", "2", "--shard-loci", "7", "--devices", "0,1", *PATHS[path], *FILTER_ARGS,
                   tag=f"two_{path}")
        assert one[:4] == two[:4]


# ---- engine level --------------------------------------------------------------------------------------------------------
def _numpy_ll(trip, dosage, eps, n_cols):
    """the model on finished coverage triplets (ref_cnt / alt_cnt per (row, col)), in NumPy int64"""
    d = dosage.shape[1]
    hyp = np.asarray(O.hypotheses(d))
    lr, la = (np.asarray(t, np.int64) for t in O.tables(eps))
    row, col = trip.row.astype(np.int64), trip.col.astype(np.int64)
    r, a = trip.ref_cnt.astype(np.int64), trip.alt_cnt.astype(np.int64)
    ok = np.all(dosage[row] != O.MISSING, axis=1) & (r + a > 0)
    ll = np.zeros((n_cols, hyp.shape[0]), np.int64)
    cnt = np.zeros((n_cols, 3), np.int64)
    idx = np.flatnonzero(ok)
    for k in range(0, idx.size, 8192):
        i = idx[k:k + 8192]
        g = dosage[row[i]].astype(np.int64)
        s = g[:, hyp[:, 0]] + g[:, hyp[:, 1]]
        np.add.at(ll, col[i], r[i, None] * lr[s] + a[i, None] * la[s])
    np.add.at(cnt, col[ok], np.stack([np.ones(ok.sum(), np.int64), r[ok], a[ok]], 1))
    return ll, cnt


def _dosage(rng, n_rows, d, missing=0.02):
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    g[rng.random((n_rows, d)) < missing] = O.MISSING
    return g


def test_submits_accumulate_and_finish_resets():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(96, 60, depth=30, seed=5, umi=True)
    g = _dosage(np.random.default_rng(1), sb.n_rows, 5)
    with vb.Engine("coverage", umi=True) as e:
        e.set_barcodes(bcs)
        e.set_donors(g, 0.03)
        whole = e.run(sb)
        ll1, cnt1 = e.donor_ll()
        for lo, hi in ((0, 30), (30, 31), (31, 96)):
            e.submit(sb.shard(lo, hi))
        e.finish()
        ll3, cnt3 = e.donor_ll()
        e.finish()                      # nothing submitted since: zeros
        ll0, cnt0 = e.donor_ll()
    want_ll, want_cnt = _numpy_ll(whole, g, 0.03, len(bcs))
    assert cnt1[:, 0].sum() > 100 and np.array_equal(ll1, want_ll) and np.array_equal(cnt1.astype(np.int64), want_cnt)
    assert np.array_equal(ll3, ll1) and np.array_equal(cnt3, cnt1)
    assert not ll0.any() and not cnt0.any() and ll0.shape == ll1.shape


def test_call_order_and_arguments_are_checked():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(8, 10, depth=5, seed=3)
    g = np.zeros((sb.n_rows, 3), np.uint8)
    with vb.Engine("coverage") as e:
        e.set_barcodes(bcs)
        L, h = e._L, e._h
        P = lambda a: a.ctypes.data
        assert L.vtx_set_donors(h, 1, sb.n_rows, P(g), 0.01) == -1
        assert L.vtx_set_donors(h, 33, sb.n_rows, P(np.zeros((sb.n_rows, 33), np.uint8)), 0.01) == -1
        assert L.vtx_set_donors(h, 3, sb.n_rows, P(g), 0.26) == -1
        assert L.vtx_set_donors(h, 3, sb.n_rows, P(g), 1e-7) == -1
        bad = g.copy(); bad[0, 1] = 3
        assert L.vtx_set_donors(h, 3, sb.n_rows, P(bad), 0.01) == -1
        args = [C.byref(C.POINTER(C.c_int64)()), C.byref(C.POINTER(C.c_uint64)()), C.byref(C.c_uint32()), C.byref(C.c_uint32())]
        assert L.vtx_donor_ll_get(h, *args) == -5                   # no donors set
        e.submit(sb)
        assert L.vtx_set_donors(h, 3, sb.n_rows, P(g), 0.01) == -5 and "before the first submit" in e.last_error()
        e.finish()
    with vb.Engine("coverage") as e:
        e.set_barcodes(bcs)
        e.set_donors(g, 0.25)
        e.submit(sb)
        assert e._L.vtx_donor_ll_get(e._h, *args) == -5             # before the finish
        e.finish()
        assert e.donor_ll()[0].shape == (len(bcs), 6)


def test_row_beyond_the_table_fails_the_finish():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(16, 20, depth=10, seed=9)
    g = np.ones((int(sb.locus_row.max()), 2), np.uint8)            # the last locus's row is outside
    with vb.Engine("coverage") as e:
        e.set_barcodes(bcs)
        e.set_donors(g, 0.01)
        e.submit(sb)
        with pytest.raises(vb.VtxError, match="outside the donor dosage table"):
            e.finish()
        # the loci inside the table were still counted, and the next result set is clean
        e.submit(sb.shard(0, 4))
        got = e.finish()
        ll, cnt = e.donor_ll()
    want_ll, want_cnt = _numpy_ll(got, g, 0.01, len(bcs))
    assert np.array_equal(ll, want_ll) and np.array_equal(cnt.astype(np.int64), want_cnt)


def _ladder_shard(n_barcodes=120_000, seed=8):
    """one shard of 95 000 one-or-two-pair loci: cells 0..5 have a slot in the first 1, 31, 32, 33, 2 049 and 95 000 loci,
    and every locus has one more pair of a random other column of 120 000 (tens of thousands of one-slot cells)"""
    import slot_cases as S
    rng = np.random.default_rng(seed)
    n_loci = 95_000
    reach = np.array([1, 31, 32, 33, 2049, 95_000])
    tmpl, cb, depth = [], [], []
    for l in range(n_loci):
        cells = [c for c in range(6) if l < reach[c]] + [int(rng.integers(6, n_barcodes))]
        depth.append(len(cells)); cb += cells
        tmpl += rng.choice(4, len(cells), p=(0.4, 0.4, 0.15, 0.05)).tolist()
    n = len(cb)
    return S.Shard("donor_ladder", np.zeros(n_loci, np.int8), np.concatenate([[0], np.cumsum(depth)]).astype(np.int64),
                   np.asarray(tmpl, np.int8), np.asarray(cb, np.int64), np.full(n, S.UMI_POOL[0], np.uint64), n_barcodes=n_barcodes)


@pytest.mark.parametrize("d", [2, 17, 32])
def test_depth_ladder_equals_numpy(d):
    import slot_cases as S
    import vartrix_b200 as vb
    shard = _ladder_shard()
    sb = vb.StagedBatch.from_fields(S.fields(shard))
    bcs = vb.Barcodes(S.barcodes(shard.n_barcodes))
    g = _dosage(np.random.default_rng(d), shard.n_loci, d, missing=0.002)
    with vb.Engine("coverage") as e:
        e.set_barcodes(bcs)
        e.set_donors(g, 1e-6 if d == 17 else 0.01)
        e.submit(sb)
        got = e.finish()
        ll, cnt = e.donor_ll()
    want_ll, want_cnt = _numpy_ll(got, g, 1e-6 if d == 17 else 0.01, len(bcs))
    # a slot qualifies only with a REF or ALT molecule at a usable row: about three in four of the ladder's slots do
    assert cnt[5, 0] > 60_000 and cnt[4, 0] > 1_200 and 0 < cnt[3, 0] <= 33 and (cnt[6:, 0] == 1).sum() > 10_000
    assert np.array_equal(cnt.astype(np.int64), want_cnt)
    assert np.array_equal(ll, want_ll)


def test_launches_only_with_donors():
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(64, 40, depth=25, seed=7, umi=True)
    counts = {}
    for on in (False, True):
        with vb.Engine("coverage", umi=True) as e:
            e.set_barcodes(bcs)
            if on:
                e.set_donors(np.zeros((sb.n_rows, 4), np.uint8))
            e.submit(sb)
            counts[on] = (e.finish(), e.timing()["total_launches"])
    assert counts[True][1] == counts[False][1] + 6          # count, the three scan kernels, scatter, the per-column warps
    for f in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt", "unk_cnt"):
        assert np.array_equal(getattr(counts[True][0], f), getattr(counts[False][0], f), equal_nan=True)
