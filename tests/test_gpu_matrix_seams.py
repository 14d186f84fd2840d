"""The matrix-assembly kernels at their seams (-m gpu): vtx_k_slots (pair keys staged in chunks of 1024, a grid capped
at 65 535 x 8 CTAs), vtx_k_slots_big (loci deeper than 2048 pairs: hash set, bitonic sort over P = 2^k >= D cells,
one CTA per SM walking the deep loci), vtx_k_umi_collapse (the 0.75 rule), vtx_k_finalize and vtx_k_emit.

Shards come from tests/slot_cases.py: reads are copies of eight templates whose calls are known, so the expected
matrix is tests/matrix_ref.py fed the template scores, for shards of up to 4.2 M pairs.  Each case runs in the three
modes with and without --umi and must match bit for bit (triplets, NaN, metrics); shards small enough also go
through the oracle.  A failure names the case, mode, locus, depth and distinct cells."""
import functools
import re
from fractions import Fraction

import numpy as np
import pytest

import matrix_ref
import slot_cases as S
from conftest import assert_same_triplets, to_oracle_batch

pytestmark = pytest.mark.gpu

MODES = ("consensus", "coverage", "alt_frac")
CASES = ("ladder", "umi_grid", "modes", "crowd", "many_loci", "counters")
ORACLE_MAX_PAIRS = 200_000
FOLD_CLASS = 7


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def template_scores(oracle):
    f, pr, pl = S.template_batch()
    n_rows = f.pop("n_rows")
    return oracle.score_pairs(oracle.Batch(**f, n_rows=n_rows), pr, pl)


@functools.lru_cache(maxsize=None)
def _shard(case, n_sm):
    return {"ladder": S.ladder, "umi_grid": S.umi_grid, "modes": S.modes, "crowd": lambda: S.crowd(n_sm),
            "many_loci": S.many_loci, "counters": S.counters}[case]()


@functools.lru_cache(maxsize=None)
def _barcodes():
    import vartrix_b200 as vb
    return vb.Barcodes(S.barcodes())


@functools.lru_cache(maxsize=None)
def _barcode_index():
    return matrix_ref.barcode_index(_barcodes().keys)


@functools.lru_cache(maxsize=None)
def _staged(case, n_sm):
    import vartrix_b200 as vb
    return vb.StagedBatch.from_fields(S.fields(_shard(case, n_sm)))


def _run(vb, mode, umi, submit, trace=False):
    """-> (triplets, tile counts of the last submit, kernel names when traced); submit(eng) submits the shards"""
    import contextlib

    import torch
    from torch.profiler import ProfilerActivity, profile
    prof_cm = profile(activities=[ProfilerActivity.CUDA]) if trace else contextlib.nullcontext()
    with vb.Engine(mode, umi=umi) as eng, prof_cm as prof:
        eng.set_barcodes(_barcodes())
        submit(eng)
        got = eng.finish()
        tiles = eng.tile_counts()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()} if trace else set()
    return got, tiles, names


def _where(got, exp, shard):
    """the first entry where got and exp differ, as (locus, depth, distinct cells, got, expected)"""
    n = min(len(got.row), len(exp.row))
    bad = np.zeros(n, bool)
    for f in ("row", "col", "ref_cnt", "alt_cnt", "unk_cnt"):
        bad |= np.asarray(getattr(got, f))[:n] != np.asarray(getattr(exp, f))[:n]
    for f in ("val", "val2"):
        a, b = np.asarray(getattr(got, f))[:n], np.asarray(getattr(exp, f))[:n]
        bad |= ~((a == b) | (np.isnan(a) & np.isnan(b)))
    i = int(np.argmax(bad)) if bad.any() else n
    src = exp if i < len(exp.row) else got
    if i >= len(src.row):
        return f"{len(got.row)} entries, expected {len(exp.row)}"
    l = int(src.row[i])
    f = S.locus_facts(shard, l)
    pick = lambda t: {k: np.asarray(getattr(t, k))[i].item() for k in ("row", "col", "ref_cnt", "alt_cnt", "unk_cnt", "val")
                      } if i < len(t.row) else None
    return f"locus {l} (depth {f['d']}, D {f['D']}, P {f['P']}): got {pick(got)}, expected {pick(exp)}"


def _compare(got, exp, shard, what):
    try:
        assert_same_triplets(got, exp)
    except AssertionError as e:
        raise AssertionError(f"{what}: {_where(got, exp, shard)}") from e
    assert got.metrics == exp.metrics, (what, got.metrics, exp.metrics)


def _expected(shard, sb, mode, umi, template_scores):
    rs, as_ = S.expected_scores(shard, *template_scores)
    return matrix_ref.assemble(sb, _barcode_index(), mode, umi, rs, as_)


def _expected_tiles(shard, umi):
    """warp tiles of class 0 (short windows) and of the folded kernel (production windows): 4 pairs per tile"""
    kept = (shard.cb >= 0) & ((shard.umi != np.uint64(S.NO_UMI)) | (not umi))
    per = np.bincount(np.repeat(np.arange(shard.n_loci), shard.depth()), weights=kept, minlength=shard.n_loci)
    tiles = (per.astype(np.int64) + 3) // 4
    return int(tiles[shard.fam == S.SHORT].sum()), int(tiles[shard.fam == S.PROD].sum())


@pytest.mark.parametrize("umi", [False, True], ids=["no_umi", "umi"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES)
def test_assembly_matches_reference(vb, oracle, n_sm, template_scores, case, mode, umi):
    shard, sb = _shard(case, n_sm), _staged(case, n_sm)
    what = f"{case} {mode} {'umi' if umi else 'no umi'}"
    got, tiles, names = _run(vb, mode, umi, lambda eng: eng.submit(sb), trace=(mode == "coverage"))
    exp = _expected(shard, sb, mode, umi, template_scores)
    _compare(got, exp, shard, what)
    # routing: the window families reach their kernels, deep loci reach vtx_k_slots_big
    assert (tiles[0], tiles[FOLD_CLASS]) == _expected_tiles(shard, umi) and sum(tiles) == tiles[0] + tiles[FOLD_CLASS], \
        (what, tiles)
    if mode == "coverage" and shard.depth().max() > S.SMALL_MAX:
        assert any(re.search(r"\bvtx_k_slots_big\b", n) for n in names), (what, sorted(names))
    if shard.n_pairs <= ORACLE_MAX_PAIRS:
        ref = oracle.run_batch(to_oracle_batch(oracle, sb), oracle.Barcodes(_barcodes().keys), oracle.MODES[mode], umi,
                               n_threads=16)
        _compare(got, ref, shard, what + " (oracle)")
    if case == "ladder" and mode == "alt_frac" and not umi:
        # the cell with 100 000 reads: the quotient is correctly rounded
        one = [l for l in np.nonzero(shard.depth() == 100_000)[0] if S.locus_facts(shard, l)["D"] == 1]
        i = int(np.nonzero(got.row == one[0])[0][0])
        s, e = int(shard.cand_start[one[0]]), int(shard.cand_start[one[0] + 1])
        t = int(got.ref_cnt[i]) + int(got.alt_cnt[i]) + int(got.unk_cnt[i])
        assert t == int((shard.tmpl[s:e] != S.T_NONE).sum())
        assert got.val[i] == float(Fraction(int(got.alt_cnt[i]), t))
    if case == "counters" and not umi:
        assert (int(got.alt_cnt[0]), int(got.unk_cnt[0]), int(got.ref_cnt[0])) == ((1 << 21) + 1, (1 << 21) + 1, 3)


def _many_submits(vb, shard):
    """each deep locus in a submit of its own with an empty submit after it; runs of shallow loci together"""
    deep = shard.depth() > S.SMALL_MAX
    parts, run = [], []
    for l in range(shard.n_loci):
        if deep[l]:
            if run:
                parts.append(run); run = []
            parts += [[l], []]
        else:
            run.append(l)
    if run:
        parts.append(run)
    return [vb.StagedBatch.from_fields(S.fields(shard, p)) for p in parts]


@pytest.mark.parametrize("umi", [False, True], ids=["no_umi", "umi"])
def test_ladder_in_every_layout(vb, n_sm, template_scores, umi):
    """the depth ladder through vtx_submit, vtx_submit2 (slim), vtx_submit2_device (resident) and many submits"""
    from test_gpu_slim import _resident
    shard, sb = _shard("ladder", n_sm), _staged("ladder", n_sm)
    mode = "coverage"
    exp = _expected(shard, sb, mode, umi, template_scores)
    base, _t, _n = _run(vb, mode, umi, lambda eng: eng.submit(sb))
    _compare(base, exp, shard, f"ladder submit umi={umi}")
    sl = vb.SlimBatch.from_staged(sb, umi)
    slim, _t, _n = _run(vb, mode, umi, lambda eng: eng.submit2(sl))
    _compare(slim, exp, shard, f"ladder submit2 umi={umi}")
    res = _resident(sl, sb.cand_start, _barcodes(), mode, umi, 1)
    _compare(res, exp, shard, f"ladder submit2_device umi={umi}")
    parts = _many_submits(vb, shard)
    assert sum(p.n_loci == 0 for p in parts) == int((shard.depth() > S.SMALL_MAX).sum())

    def submit_all(eng):
        for p in parts:
            eng.submit(p)
    many, _t, _n = _run(vb, mode, umi, submit_all)
    _compare(many, exp, shard, f"ladder in {len(parts)} submits umi={umi}")
