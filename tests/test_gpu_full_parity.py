"""Full-size bit-exactness: complete BASELINE.json-shaped shards (configs 2, 3 and 4) and a depth-600 alt_frac shard of
the config-5 shape, the CUDA path through the C ABI against the CPU oracle, entry by entry (row, col, the three counts
and both f64 values incl. NaN), plus the metric counters.  The oracle runs on every host core (~1 min for config 3)."""
import os

import numpy as np
import pytest

from conftest import assert_same_triplets, to_oracle_batch

pytestmark = pytest.mark.gpu


def _run(oracle, cfg, n_submits, engine_flags=({},)):
    """the oracle once; the engine once per entry of engine_flags (Engine keyword arguments)"""
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(**cfg)
    umi = bool(cfg.get("umi"))
    exp = oracle.run_batch(to_oracle_batch(oracle, sb), oracle.Barcodes(bcs.keys), oracle.MODES[cfg["scoring_method"]], umi,
                           n_threads=len(os.sched_getaffinity(0)))
    for kw in engine_flags:
        with vb.Engine(cfg["scoring_method"], umi=umi, **kw) as eng:
            eng.set_barcodes(bcs)
            for lo, hi in vb.shard_bounds(sb.cand_start, n_submits):
                eng.submit(sb.shard(lo, hi))
            got = eng.finish()
        assert_same_triplets(got, exp)
        assert got.metrics == exp.metrics, kw
        assert got.metrics["num_scored"] == info["n_pairs"], kw
    return got, info


@pytest.mark.parametrize("name,n_submits", [("config2", 3), ("config4", 4), ("config3", 5)])
def test_full_config_bit_exact(oracle, name, n_submits):
    import vartrix_b200 as vb
    # config 2 also through the two-phase kernels alone (no_fold) and the single-phase classes alone (no_split): the
    # whole pipeline (slots, counts) at full size through those kernels (chunked tiles: tests/test_gpu_sw_scale.py)
    flags = ({}, dict(no_fold=True), dict(no_split=True)) if name == "config2" else ({},)
    got, info = _run(oracle, dict(vb.synth.CONFIGS[name]), n_submits, flags)
    assert len(got.row) > 0.8 * info["n_pairs"]          # ~1 read per cell at these barcode counts


def test_config5_depth600_alt_frac_bit_exact(oracle):
    """BASELINE config 5: 600 reads per locus x 100k barcodes, alt_frac (main.rs:1131-1145) -- fractional values,
    several reads per cell, every present cell emitted."""
    import vartrix_b200 as vb
    cfg = dict(vb.synth.CONFIGS["config5_shard"]); cfg["n_loci"] = 1500
    got, info = _run(oracle, cfg, 3)
    assert info["depth"] == 600 and got.metrics["num_scored"] > 800_000
    frac = got.val[~np.isnan(got.val)]
    assert ((frac > 0) & (frac < 1)).any()                # genuinely fractional entries exist
