"""CPU suite: the split of vtx_sw_fold.cuh with a shared extension (prefix | shared extension | allele columns | shared
extension | suffix), restated in tests/fold_shared_cases.py, against the full-matrix oracle, and how x is chosen."""
import numpy as np
import pytest

import fold_shared_cases as fs


@pytest.mark.parametrize("pad, kind, alen, x", [
    (96, "snv", 1, 0), (97, "snv", 1, 1), (100, "snv", 1, 4), (100, "del_anchor", 3, 4), (100, "ins_bare", 5, 4),
    (101, "ins_anchor", 1, 5), (109, "snv", 1, 11),      # 27 allele columns: the 1280-byte table holds 11 shared ones
    (106, "mnp", 12, 7), (100, "mnp", 32, 0),            # 32 allele columns: 7 of 10; 40 (kFoldMaxMid): none
])
def test_shared_columns_rule(pad, kind, alen, x):
    rng = np.random.default_rng(pad * 100 + alen)
    ref, alt = fs.window(rng, pad, kind, alen)
    got = fs.shared_columns(ref, alt)
    assert got == x
    mid = max(len(ref), len(alt)) - 192
    assert 100 * got + 32 * (mid - 2 * got) <= 1280 and min(len(ref), len(alt)) - 192 - 2 * got >= 1


def test_alleles_that_share_nothing_extend_nothing():
    left, right = b"A" * 96, b"C" * 96
    assert fs.shared_columns(left + b"G" + right, left + b"T" + right) == 0
    assert fs.shared_columns(left + b"GTT" + right, left + b"TTG" + right) == 0   # both sides differ
    assert fs.shared_columns(left + b"GTTA" + right, left + b"GAT" + right) == 0  # the left side shares, the right not


@pytest.mark.parametrize("pad", [96, 97, 100, 104, 109])
@pytest.mark.parametrize("kind", fs.KINDS)
def test_split_with_shared_extension_equals_full_matrix(oracle, pad, kind):
    rng = np.random.default_rng(pad * 10 + fs.KINDS.index(kind))
    checked = 0
    for it in range(6):
        ref, alt = fs.window(rng, pad, kind, int(rng.integers(1, 7)))
        x = fs.shared_columns(ref, alt)
        rd = fs.reads(rng, ref, alt, x, 52, rng.integers(1, 153, 48).tolist() + [1, 2, max(1, x - 1), 152])
        got_r, got_a = fs.split_scores(rd, ref, alt, x)
        exp_r = [oracle.sw_full(r, ref) for r in rd]
        exp_a = [oracle.sw_full(r, alt) for r in rd]
        assert np.array_equal(got_r, exp_r) and np.array_equal(got_a, exp_a), (pad, kind, it, x)
        # every smaller x is a valid split too (x = 0 is the kernel without extension)
        for y in {0, 1, x // 2} - {x}:
            if y <= x:
                yr, ya = fs.split_scores(rd, ref, alt, y)
                assert np.array_equal(yr, exp_r) and np.array_equal(ya, exp_a), (pad, kind, it, y)
        checked += len(rd)
    assert checked == 6 * 52


def test_gaps_across_both_seams_are_witnessed(oracle):
    """Reads whose best alignment has a gap across a seam: scoring each side of the seam on its own (no carry) loses
    score, so these reads need the boundary handed over"""
    rng = np.random.default_rng(5)
    found = {"fwd": 0, "rev": 0}
    for _ in range(40):
        ref, alt = fs.window(rng, 100, "snv")
        x = fs.shared_columns(ref, alt)
        assert x == 4
        for side, seam in (("fwd", 96 + x), ("rev", len(ref) - 96 - x)):
            g = int(rng.integers(2, 6))
            a = int(rng.integers(1, g))
            rd = ref[seam - 40:seam - a] + ref[seam - a + g:seam + 40]       # a deletion of g bases across the seam
            full = oracle.sw_full(rd, ref)
            cut = max(oracle.sw_full(rd, ref[:seam]), oracle.sw_full(rd, ref[seam:]))
            if full > cut:
                found[side] += 1
            got_r, _ = fs.split_scores([rd], ref, alt, x)
            assert got_r[0] == full
    assert found["fwd"] >= 10 and found["rev"] >= 10, found
