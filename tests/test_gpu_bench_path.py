"""GPU: the calls bench.py times, against the C oracle entry by entry -- row, col, val and val2 with NaN, the three counts
whenever the engine returns them, and the three metrics.

- bench.py itself, both staging layouts: the triplets it dumps from its last timed `value` step.
- `value` restated: shards resident in HBM (vtx_submit2_device / vtx_submit_device_ex) submitted 1, 4 or 7 at a time,
  8 steps on one context driven from a caller's stream, values-only results on and off.
- `e2e` restated: pinned slim shards growing from bench.py's priming shard (vtx_submit2, vtx_finish without a copy), then
  re-staged at another growth on the same context, then a resident step on it, as bench.py runs `value` and `e2e` on one
  engine.
- The streamed vtx_finish on both sides of the 4 096 submits per finish whose triplets it copies out early, with empty
  submits among them.
- vtx_wait_copies as the CLI's staging lanes use it before reusing a pinned arena, and with every pinned buffer
  overwritten before the finish.
- A config-5 shard above 8 M candidates, where bench.py streams `value` in 4 submits.

Workloads come from bench.workload_config and shard schedules from bench.py's own arguments, so the tests follow its
defaults.  Each oracle runs once per module on every host core (about 1 min for config 3, a few for the config-5
shard)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from bench_path import bench_workload, c_batch, dump_sample, e2e_bounds, place, value_submits, with_empty_submits
from conftest import ROOT, to_oracle_batch

pytestmark = pytest.mark.gpu

COUNTS = ("ref_cnt", "alt_cnt", "unk_cnt")


class Workload:
    """One of bench.py's workloads, staged in both layouts, with the oracle's triplets."""

    def __init__(self, oracle, *argv):
        import vartrix_b200 as vb
        self.args, self.cfg = bench_workload(*argv)
        self.sb, self.bcs, self.info = vb.synth.make_shard(**self.cfg)
        self.mode, self.umi = self.cfg["scoring_method"], bool(self.cfg.get("umi"))
        self.slim = vb.SlimBatch.from_staged(self.sb, self.umi)
        self.max_read, self.max_hap = int(self.info["read_len"]), int(self.info["max_hap_len"])
        self.exp = oracle.run_batch(to_oracle_batch(oracle, self.sb), oracle.Barcodes(self.bcs.keys), oracle.MODES[self.mode],
                                    self.umi, n_threads=len(os.sched_getaffinity(0)))
        assert self.exp.metrics["num_scored"] == self.info["n_pairs"]
        self._shards = {}

    def shards(self, layout, bounds):
        """Host shards of `layout` ("slim" or "v1") for the locus ranges `bounds` (the whole batch for one range)."""
        key = (layout, tuple(bounds))
        if key not in self._shards:
            staged = self.slim if layout == "slim" else self.sb
            if len(bounds) == 1:
                self._shards[key] = [staged]
            else:
                # shard() reads the whole batch's read table, so thousands of small shards are cut from blocks of loci
                block, blocks, out = max(256, staged.n_loci // 64), {}, []
                for lo, hi in bounds:
                    b = lo - lo % block
                    e = min(staged.n_loci, max(hi, b + block))
                    if (b, e) not in blocks:
                        blocks[(b, e)] = staged.shard(b, e)
                    out.append(blocks[(b, e)].shard(lo - b, hi - b))
                self._shards[key] = out
        return self._shards[key]

    def engine(self, **kw):
        import vartrix_b200 as vb
        eng = vb.Engine(self.mode, umi=self.umi, **kw)
        eng.set_barcodes(self.bcs)
        return eng


@pytest.fixture(scope="module")
def config3(oracle):
    return Workload(oracle, "--workload", "config3")


@pytest.fixture(scope="module")
def config2(oracle):
    return Workload(oracle, "--workload", "config2")


@pytest.fixture(scope="module")
def config5(oracle):
    return Workload(oracle, "--workload", "config5_shard", "--loci", "15000")


def check(got, w, values_only, what):
    """got equals the oracle's triplets of workload w, in order; with values_only the counts (and val2 outside coverage
    mode) must stay on the device."""
    exp = w.exp
    assert len(got.row) == len(exp.row), (what, len(got.row), len(exp.row))
    for f in ("row", "col"):
        assert np.array_equal(getattr(got, f), getattr(exp, f)), (what, f)
    assert np.array_equal(got.val, exp.val, equal_nan=True), (what, "val")
    device_only = (COUNTS + (("val2",) if w.mode != "coverage" else ())) if values_only else ()
    for f in device_only:
        assert getattr(got, f).size == 0, (what, f, "returned by a values-only engine")
    for f in COUNTS:
        if f not in device_only:
            assert np.array_equal(getattr(got, f), getattr(exp, f)), (what, f)
    if "val2" not in device_only:
        assert np.array_equal(got.val2, exp.val2, equal_nan=True), (what, "val2")
    assert got.metrics == exp.metrics, what


def resident_parts(w, layout, n_sub, keep):
    import vartrix_b200 as vb
    fields = vb.SlimBatch.ARRAYS if layout == "slim" else vb.StagedBatch.FIELDS
    bounds = [(lo, hi) for lo, hi in vb.shard_bounds(w.sb.cand_start, n_sub) if hi > lo]
    return [c_batch(p, place(p, fields, "cuda", keep)) for p in w.shards(layout, bounds)]


def resident_step(eng, w, layout, parts):
    for cb in parts:
        (eng.submit2_device if layout == "slim" else eng.submit_device)(cb, w.max_read, w.max_hap)
    return eng.fetch(eng.finish_device())


# ------------------------------------------------------------------------------------------------
# 1. bench.py itself
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["slim", "v1"])
def test_bench_dump_equals_oracle(config3, layout, tmp_path):
    out = tmp_path / "dump"
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    cmd = py + [os.path.join(ROOT, "bench.py"), "--gpus", "1", "--workload", "config3", "--warmup", "3", "--steps", "2",
                "--no-cpu-baseline", "--layout", layout, "--dump-outputs", str(out)]
    p = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stderr[-4000:]
    line = json.loads(p.stdout.strip().splitlines()[-1])
    dumped = line["dump_outputs"]
    exp = config3.exp
    assert dumped["n_triplets"] == len(exp.row)
    names = [a for a in dumped["arrays"] if a != "metrics"]
    assert names == ["col", "row", "val"]          # bench.py's engine is values-only, and config 3 is consensus mode
    keep = dump_sample(len(exp.row), len(names))
    assert dumped["n_dumped"] == len(keep)
    for name in names:
        got = np.load(out / f"{name}.npy")
        assert np.array_equal(got, getattr(exp, name)[keep].astype(np.float64), equal_nan=True), name
    m = exp.metrics
    assert list(np.load(out / "metrics.npy")) == [m["num_not_cell_bc"], m["num_non_umi"], m["num_scored"]]


# ------------------------------------------------------------------------------------------------
# 2. `value`: resident shards, repeated steps on one context
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("values_only", [True, False])
@pytest.mark.parametrize("n_sub", [1, 4, 7])
@pytest.mark.parametrize("layout", ["slim", "v1"])
def test_resident_steps(config3, layout, n_sub, values_only):
    import torch
    w = config3
    keep = []
    parts = resident_parts(w, layout, n_sub, keep)
    assert len(parts) == n_sub
    stream = torch.cuda.Stream()
    with w.engine(stream=stream.cuda_stream, values_only=values_only) as eng:
        for step in range(8):
            check(resident_step(eng, w, layout, parts), w, values_only, f"step {step}")
            assert eng.tile_counts()[7] > 0            # the folded kernel took the work
            assert eng.timing()["n_pairs"] == w.info["n_pairs"]


# ------------------------------------------------------------------------------------------------
# 3. `e2e`: pinned shards growing from the priming shard, re-staged, then a resident step on the same context
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("growth,restage", [(None, 1.4), (1.4, 1.1), (1.1, 0.0), (0.0, None)])
def test_e2e_steps(config3, growth, restage):
    import torch
    import vartrix_b200 as vb
    w = config3
    g0 = w.args.growth if growth is None else growth
    g1 = w.args.growth if restage is None else restage

    def stage(g, keep):
        parts = w.shards("slim", e2e_bounds(w.args, w.sb.cand_start, g))
        return [c_batch(p, place(p, vb.SlimBatch.ARRAYS, "pinned", keep)) for p in parts]

    def step(hparts, what):
        for cb in hparts:
            eng._ck(eng._L.vtx_submit2(eng._h, C.byref(cb)), "vtx_submit2")
        got = eng.finish(copy=False)          # views of the engine's pinned arrays, valid until the next engine call
        try:
            check(got, w, True, what)
        except AssertionError as e:           # a report that kept `got` would read the arrays after the engine is closed
            raise AssertionError(str(e)) from None

    stream = torch.cuda.Stream()
    with w.engine(stream=stream.cuda_stream, values_only=True) as eng:
        keep = []
        hparts = stage(g0, keep)
        assert len(hparts) >= 3
        for s in range(5):                    # 3 warm-up steps and 2 timed ones
            step(hparts, f"growth {g0}, step {s}")
        keep2 = []
        hparts = stage(g1, keep2)
        for s in range(2):
            step(hparts, f"re-staged at growth {g1}, step {s}")
        dkeep = []
        check(resident_step(eng, w, "slim", resident_parts(w, "slim", 1, dkeep)), w, True, "resident step after e2e")


# ------------------------------------------------------------------------------------------------
# 4. the streamed finish on both sides of kMaxCum = 4 096 submits
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_submits", [1, 2, 4095, 4096, 4097, 5000])
def test_streamed_finish_seam(config2, n_submits):
    w = config2
    bounds = with_empty_submits(w.sb.cand_start, n_submits)
    shards = w.shards("slim", bounds) if n_submits > 1 else [w.slim]
    assert len(shards) == n_submits
    for values_only in (False, True):
        with w.engine(values_only=values_only) as eng:
            for s in shards:
                eng.submit2(s)
            check(eng.finish(), w, values_only, f"{n_submits} submits, values_only={values_only}")
            assert eng.timing()["n_pairs"] == w.exp.metrics["num_scored"]


# ------------------------------------------------------------------------------------------------
# 5. vtx_wait_copies before pinned staging memory is reused
# ------------------------------------------------------------------------------------------------
def test_wait_copies_before_pinned_arenas_are_reused(config3):
    """Shards of >= 100 MB go round-robin through 3 pinned arenas, as the CLI's staging lanes use them: before an arena
    takes its next shard, wait_copies.  After each step's last submit and wait_copies, every arena is overwritten with
    0xFF before the finish: the copies must have landed by then.  Two steps, the arenas rotating on across them."""
    import torch
    import vartrix_b200 as vb
    w = config3
    n_parts = min(6, w.slim.nbytes() // (100 << 20))
    assert n_parts >= 4                       # at least one arena is reused within a step
    parts = w.shards("slim", vb.shard_bounds(w.sb.cand_start, n_parts))
    assert min(p.nbytes() for p in parts) >= 100 << 20

    def aligned(n):
        return (n + 255) // 256 * 256

    size = max(sum(aligned(getattr(p, f).nbytes) for f in vb.SlimBatch.ARRAYS if getattr(p, f) is not None) for p in parts)
    arenas = [torch.empty(size, dtype=torch.uint8).pin_memory() for _ in range(3)]
    mem = [a.numpy() for a in arenas]

    def stage(part, k):
        """part copied into arena k -> a SlimBatch whose arrays are views of the arena"""
        off, arrays = 0, {}
        for f in vb.SlimBatch.ARRAYS:
            a = getattr(part, f)
            if a is None:
                arrays[f] = None
                continue
            dst = mem[k][off: off + a.nbytes].view(a.dtype)
            dst[:] = a.reshape(-1)
            arrays[f] = dst
            off += aligned(a.nbytes)
        return vb.SlimBatch(**arrays, n_rows=part.n_rows)

    k = 0
    with w.engine() as eng:
        for step in range(2):
            used = []
            for part in parts:
                if k >= 3:
                    eng.wait_copies()         # the arena's previous shard must have reached the device
                eng.submit2(stage(part, k % 3))
                used.append(k % 3)
                k += 1
            eng.wait_copies()
            for a in dict.fromkeys(reversed(used)):       # the arena copied last first
                mem[a].fill(0xFF)
            check(eng.finish(), w, False, f"step {step}")


# ------------------------------------------------------------------------------------------------
# 6. above 8 M candidates: `value` in 4 streamed submits
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("values_only", [True, False])
def test_resident_above_8m_candidates(config5, values_only):
    import torch
    w = config5
    n_sub = value_submits(w.args, w.info["n_cand"])
    assert w.info["n_cand"] > 8_000_000 and n_sub == 4
    keep = []
    parts = resident_parts(w, "slim", n_sub, keep)
    stream = torch.cuda.Stream()
    with w.engine(stream=stream.cuda_stream, values_only=values_only) as eng:
        for step in range(2):
            check(resident_step(eng, w, "slim", parts), w, values_only, f"step {step}")
    frac = w.exp.val[~np.isnan(w.exp.val)]
    assert ((frac > 0) & (frac < 1)).any()            # alt_frac: genuinely fractional entries
