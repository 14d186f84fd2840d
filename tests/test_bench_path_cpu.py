"""CPU: the helpers tests/test_gpu_bench_path.py relies on restate bench.py exactly -- the dump's seeded sample of
entries, and e2e shard schedules that hand every locus over once."""
import types

import numpy as np
import pytest

import bench
from bench_path import bench_args, dump_sample, e2e_bounds, value_submits, with_empty_submits


def _fake_triplets(n, values_only, rng):
    empty = np.zeros(0, np.uint32)
    cnt = (lambda: empty) if values_only else (lambda: rng.integers(0, 9, n).astype(np.uint32))
    val2 = rng.random(n)
    val2[rng.random(n) < 0.1] = np.nan
    return types.SimpleNamespace(row=np.arange(n, dtype=np.uint32), col=rng.integers(0, 50_000, n).astype(np.uint32),
                                 ref_cnt=cnt(), alt_cnt=cnt(), unk_cnt=cnt(), val=rng.random(n),
                                 val2=np.zeros(0) if values_only else val2,
                                 metrics=dict(num_not_cell_bc=3, num_non_umi=0, num_scored=n))


@pytest.mark.parametrize("dump_bytes,n,values_only", [
    (1 << 16, 100, False),          # below the cap: everything, in order
    (1 << 16, 5_000, False),        # above it: the seeded sample of the 7 arrays' cap
    (1 << 16, 5_000, True),         # values only: 3 arrays, a larger cap
    (None, 3_000_000, True),        # bench.py's own 64 MB cap (2.8 M entries of 3 arrays)
])
def test_dump_sample_matches_dump_outputs(tmp_path, monkeypatch, dump_bytes, n, values_only):
    if dump_bytes is not None:
        monkeypatch.setattr(bench, "DUMP_BYTES", dump_bytes)
    trip = _fake_triplets(n, values_only, np.random.default_rng(n))
    info = bench.dump_outputs(str(tmp_path), trip)
    names = [a for a in info["arrays"] if a != "metrics"]
    assert names == sorted(["row", "col", "val"] if values_only else ["row", "col", "ref_cnt", "alt_cnt", "unk_cnt", "val", "val2"])
    keep = dump_sample(n, len(names))
    assert info["n_triplets"] == n and info["n_dumped"] == len(keep)
    assert (len(keep) < n) == (n > (bench.DUMP_BYTES - 4096) // (8 * len(names)))
    for name in names:
        got = np.load(tmp_path / f"{name}.npy")
        assert np.array_equal(got, getattr(trip, name)[keep].astype(np.float64), equal_nan=True), name
    assert list(np.load(tmp_path / "metrics.npy")) == [3, 0, n]


def _cand_start(n_loci, seed):
    depth = np.random.default_rng(seed).poisson(50, n_loci)
    cs = np.zeros(n_loci + 1, np.uint64)
    cs[1:] = np.cumsum(depth)
    return cs


@pytest.mark.parametrize("growth", [None, 1.4, 1.1, 0.0])
@pytest.mark.parametrize("n_loci", [100_000, 15_000, 1_500])
def test_e2e_schedule_covers_every_locus_once(growth, n_loci):
    args = bench_args()
    g = args.growth if growth is None else growth
    cs = _cand_start(n_loci, n_loci)
    n_cand = int(cs[-1])
    b = e2e_bounds(args, cs, g)
    assert b[0][0] == 0 and b[-1][1] == n_loci
    assert all(hi > lo for lo, hi in b) and all(b[i][1] == b[i + 1][0] for i in range(len(b) - 1))
    sizes = [int(cs[hi] - cs[lo]) for lo, hi in b]
    # the priming shard is the larger of --first-chunk and --min-shard (or everything), and no shard passes 1/--chunks of
    # the step by more than one locus
    first = max(args.first_chunk, min(1.0, args.min_shard / n_cand))
    assert abs(sizes[0] - first * n_cand) <= 200 or len(b) == 1
    if g > 1.0 and len(b) > 1:
        assert max(sizes) <= n_cand / args.chunks + 200
        assert all(b2 <= g * b1 + 200 for b1, b2 in zip(sizes, sizes[1:-1]))
    else:
        assert len(b) <= args.chunks


def test_value_submits_follow_bench():
    args = bench_args()
    assert value_submits(args, 5_000_000) == 1 and value_submits(args, 9_000_000) == 4
    assert value_submits(bench_args("--submits", "7"), 5_000_000) == 7


@pytest.mark.parametrize("n_submits", [1, 2, 4095, 4096, 4097, 5000])
def test_seam_splits_cover_every_locus_once(n_submits):
    cs = _cand_start(10_000, 5)
    b = with_empty_submits(cs, n_submits)
    assert len(b) == n_submits
    assert b[0][0] == 0 and b[-1][1] == 10_000
    assert all(b[i][1] == b[i + 1][0] for i in range(len(b) - 1))
    n_empty = sum(hi == lo for lo, hi in b)
    if n_submits >= 5:
        assert b[0] == (0, 0) and b[-1] == (10_000, 10_000) and n_empty >= 4
