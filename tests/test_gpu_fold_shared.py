"""Per-locus tables shared by the warps of a vtx_k_sw_fold CTA (-m gpu).

The warps of a CTA take consecutive tiles and share one merged profile and allele table per locus in a ring of slots
(vartrix_b200/csrc/vtx_fold_ring.cuh).  These shards stress the ring: 1-tile loci that wrap it constantly, one locus
with tens of thousands of tiles that spans many runs of every CTA, neighbouring windows that always differ (SNV and
indel alleles of 1-40 columns), runs of loci with no fold tiles in between, and tile totals of 1, fewer than one CTA's
warps, and not a multiple of the run length.  Every pair must run in the folded kernel and match the oracle bit for
bit.

The launcher runs 20 warps sharing 9 slots for shards with at least 6 candidates per locus and 13 warps with a table
each below that.  The ring-wrap and neighbours shards run under both shapes: padded with one deep fold locus (its reads repeated)
to force the deep shape, or with loci without reads to force the shallow one.  The kernel that ran is read from a
torch.profiler trace of the call."""
import re

import numpy as np
import pytest

import seam_cases
import test_gpu_sw_scale as scale
from conftest import to_oracle_batch

pytestmark = pytest.mark.gpu

FOLD_CLASS = 7
M_RANGE = (40, 152)
DEEP_DEPTH = 6                                   # candidates per locus from which the deep shape runs
SHAPES = {"deep": ("20", "9", "true"), "shallow": ("13", "13", "false")}   # warps, slots, shared


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pool(vb, oracle, n_templates, max_reads, seed):
    """fold windows with 1..max_reads reads each, scored once by the oracle"""
    refs, alts, reads, count = scale._pool("fold", n_templates, M_RANGE, max_reads, seed)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    pr = np.arange(len(reads), dtype=np.uint32)
    pl = np.repeat(np.arange(n_templates), count).astype(np.uint32)
    rs, as_ = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=16)
    start = np.concatenate([[0], np.cumsum(count)[:-1]])
    return (sb, count, start), rs, as_


def _run(vb, sb, pr, pl, exp_r, exp_a, only_fold=True):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with vb.Engine("coverage") as eng, profile(activities=[ProfilerActivity.CUDA]) as prof:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
        torch.cuda.synchronize()
    shapes = {m.groups() for e in prof.events() if (m := re.search(r"vtx_k_sw_fold<(\d+), (\d+), (true|false)>", e.name))}
    assert tiles[FOLD_CLASS] > 0, tiles
    if only_fold:
        assert sum(tiles) == tiles[FOLD_CLASS], tiles
    bad = np.nonzero((rs.astype(np.int32) != exp_r) | (as_.astype(np.int32) != exp_a))[0]
    assert bad.size == 0, (f"{bad.size} of {len(pr)} pairs differ", bad[:5], pl[bad[:5]])
    expect = "deep" if len(pr) >= DEEP_DEPTH * len(sb.ref_len) else "shallow"
    assert shapes == {SHAPES[expect]}, (shapes, expect)
    return tiles, expect


def _shaped(pool, seq, shape, rng):
    """the loci of `seq` (templates of `pool`) padded so that the launcher runs `shape`: one more locus whose reads are
    repeated until the shard has DEEP_DEPTH candidates per locus, or loci without reads until it has fewer"""
    n = len(seq)
    pad = rng.integers(0, len(pool[1]), n + 1)
    sb, pr, pl = scale._big_call([pool], np.zeros(2 * n + 1, np.int64), np.concatenate([seq, pad]))
    if shape == "deep":
        keep = pl <= n
        pr, pl = pr[keep], pl[keep]
        deep = pr[pl == n]
        extra = np.resize(deep, max(DEEP_DEPTH * (2 * n + 1) - len(pr) + deep.size, deep.size))
        pr = np.concatenate([pr[pl < n], extra]).astype(np.uint32)
        pl = np.concatenate([pl[pl < n], np.full(extra.size, n)]).astype(np.uint32)
    else:
        keep = pl < n
        pr, pl = pr[keep], pl[keep]
        assert len(pr) < DEEP_DEPTH * (2 * n + 1)
    return sb, pr, pl


@pytest.mark.parametrize("shape", ["deep", "shallow"])
def test_one_tile_loci_wrap_the_ring(vb, oracle, shape):
    """100 000 loci of 1-4 reads: every tile starts a new locus, so in the deep shape (20 warps sharing 9 slots) every
    booking takes a slot and warps wait on a full ring; the shallow shape rebuilds every warp's table at every tile.
    Consecutive windows always differ"""
    pool, prs, pas = _pool(vb, oracle, 3000, 4, 101)
    rng = np.random.default_rng(1)
    seq = scale._order(rng, 3000, 100_000)
    sb, pr, pl = _shaped(pool, seq, shape, rng)
    tiles, ran = _run(vb, sb, pr, pl, prs[pr], pas[pr])
    assert ran == shape
    assert tiles[FOLD_CLASS] >= len(seq)


@pytest.mark.parametrize("shape", ["deep", "shallow"])
def test_neighbours_differ_at_every_depth(vb, oracle, shape):
    """loci of 1-9 reads (1-3 tiles) in shuffled order: SNV- and indel-like windows with 1-40 allele columns, mid_ref
    and mid_alt mostly different, so a slot reused without rebuilding both tables gives wrong scores"""
    pool, prs, pas = _pool(vb, oracle, 3000, 9, 102)
    sbp = pool[0]
    mids = np.stack([sbp.ref_len.astype(int) - 192, sbp.alt_len.astype(int) - 192], 1)
    assert mids.min() == 1 and mids.max() == 40 and (mids[:, 0] != mids[:, 1]).mean() > 0.3
    rng = np.random.default_rng(2)
    seq = scale._order(rng, 3000, 60_000)
    sb, pr, pl = _shaped(pool, seq, shape, rng)
    _tiles, ran = _run(vb, sb, pr, pl, prs[pr], pas[pr])
    assert ran == shape


def test_zero_fold_tile_loci_between(vb, oracle):
    """runs of 0-5 loci of the two-phase kernel (no fold tiles) between 1-2-tile fold loci"""
    pool, prs, pas = _pool(vb, oracle, 2000, 8, 103)
    opool, ors, oas = scale._scored_pool(vb, oracle, "split0", 400, 104)
    rng = np.random.default_rng(3)
    n = 40_000
    seq_t = scale._order(rng, 2000, n)
    runs = rng.integers(0, 6, n)
    seq_pool = np.repeat(np.stack([np.zeros(n, np.int64), np.ones(n, np.int64)], 1).reshape(-1),
                         np.stack([np.ones(n, np.int64), runs], 1).reshape(-1))
    tmpl = np.zeros(len(seq_pool), np.int64)
    tmpl[seq_pool == 0] = seq_t
    tmpl[seq_pool == 1] = scale._order(rng, 400, int(runs.sum()))
    sb, pr, pl = scale._big_call([pool, opool], seq_pool, tmpl)
    er, ea = np.concatenate([prs, ors]), np.concatenate([pas, oas])
    tiles, _ = _run(vb, sb, pr, pl, er[pr], ea[pr], only_fold=False)
    assert sum(tiles) > tiles[FOLD_CLASS]


def test_one_locus_of_tens_of_thousands_of_tiles(vb, oracle):
    """one locus of 40 000 tiles between shallow loci: it spans many runs of every CTA, so its table is found again
    or rebuilt at every run boundary while other warps still read it"""
    rng = np.random.default_rng(4)
    refs, alts, reads = [], [], []
    owner = []
    for loc in range(7):
        ref, alt = seam_cases._fold_window(rng)
        refs.append(ref); alts.append(alt)
        k = 600 if loc == 3 else int(rng.integers(1, 10))
        for _ in range(k):
            m = int(rng.integers(*M_RANGE))
            src = ref if rng.random() < 0.5 else alt
            s = int(rng.integers(0, len(src) - m // 2))
            reads.append((seam_cases._edit(rng, src[s:s + m], 0.02) + seam_cases._rand(rng, m))[:m])
            owner.append(loc)
    owner = np.array(owner, np.uint32)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    rs, as_ = oracle.score_pairs(to_oracle_batch(oracle, sb), np.arange(len(reads), dtype=np.uint32), owner, n_threads=16)
    # the deep locus's pairs reuse its 600 reads in a random order
    deep = np.nonzero(owner == 3)[0]
    pr = np.concatenate([np.nonzero(owner == loc)[0] if loc != 3 else rng.choice(deep, 160_000) for loc in range(7)])
    pr = pr.astype(np.uint32)
    pl = owner[pr]
    tiles, _ = _run(vb, sb, pr, pl, rs[pr], as_[pr])
    assert tiles[FOLD_CLASS] >= 40_000


@pytest.mark.parametrize("kind", ["one_tile", "under_one_cta", "ragged_runs"])
def test_tile_totals(vb, oracle, n_sm, kind):
    """1 tile; 7 tiles (fewer than the warps of one CTA, so most warps find no tile); n_sm * 16 * 3 + 5 tiles, so the
    run length is 3 and the last run is short"""
    pool, prs, pas = _pool(vb, oracle, 400, 4, 105)
    n = {"one_tile": 1, "under_one_cta": 7, "ragged_runs": n_sm * 16 * 3 + 5}[kind]
    seq = scale._order(np.random.default_rng(5), 400, n) if n > 1 else np.array([0])
    sb, pr, pl = scale._big_call([pool], np.zeros(len(seq), np.int64), seq)
    tiles, _ = _run(vb, sb, pr, pl, prs[pr], pas[pr])
    assert tiles[FOLD_CLASS] == n
