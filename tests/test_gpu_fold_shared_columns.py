"""The shared extension of vtx_k_sw_fold (-m gpu): columns that ref and alt still share after the main pass are scored
once for both haplotypes (tests/fold_shared_cases.py restates the split).

VCF-like windows with --padding 96 / 97 / 100 / 109 / 120 around SNVs, MNPs (up to kFoldMaxMid allele columns) and
insertions and deletions with and without an anchor base, so x runs from 0 through 1 and 4 to the table's capacity;
reads of 1-152 bases (some shorter than x) with gaps and substitutions at both seams.  Shards of depth 8 and 3 run the
20-warp shared-table shape and the 13-warp one.  Pair scores and the whole path's triplets must match the oracle bit
for bit.  Windows padded by 120 have too many allele columns for the folded kernel and keep going elsewhere."""
import numpy as np
import pytest

import fold_shared_cases as fs
import seam_cases
from conftest import assert_same_triplets, to_oracle_batch

pytestmark = pytest.mark.gpu

FOLD_CLASS = 7
DEEP_DEPTH = 6                                   # candidates per locus from which the 20-warp shape runs
PADS = (96, 97, 100, 109, 120)


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


def _loci(pad, depth, seed):
    rng = np.random.default_rng(seed)
    loci, xs = [], []
    lengths = np.arange(1, 153)
    for l in range(96):
        kind = fs.KINDS[l % len(fs.KINDS)]
        room = fs.MAX_MID - 2 * (pad - 96)                               # MNP bases that still fit the folded kernel
        if kind == "mnp" and room >= 1:
            alen = room if l % 12 == 5 else int(rng.integers(1, room + 1))
        else:
            alen = int(rng.integers(1, 8))
        ref, alt = fs.window(rng, pad, kind, alen)
        x = fs.shared_columns(ref, alt) if max(len(ref), len(alt)) - 192 <= fs.MAX_MID else None
        lens = np.roll(lengths, -(l * depth) % 152)[:depth]
        if x:
            lens[0] = int(rng.integers(1, x + 1))                        # a read shorter than the extension
        loc = seam_cases.Locus(ref, alt)
        loc.reads = fs.reads(rng, ref, alt, x or 0, depth, lens)
        loc.cases = [None] * depth
        loci.append(loc); xs.append(x)
    return loci, xs


@pytest.mark.parametrize("depth", [8, 3], ids=["deep", "shallow"])
@pytest.mark.parametrize("pad", PADS)
def test_shared_extension_bit_exact(vb, oracle, pad, depth):
    loci, xs = _loci(pad, depth, 7000 + pad * 10 + depth)
    fold = [x is not None for x in xs]
    if pad == 96:
        assert set(xs) == {0}
    elif pad == 97:
        assert 1 in xs
    elif pad == 100:
        assert 4 in xs and 0 in xs                                       # 0: MNPs at kFoldMaxMid
    elif pad == 109:
        assert 11 in xs                                                  # the table's capacity
    else:
        assert not any(fold)
    refs, alts, reads, pr, pl, _ = seam_cases.pairs(loci)
    lens = {len(r) for r in reads}
    assert {1, 152} <= lens and len(lens) >= 140
    assert (len(pr) >= DEEP_DEPTH * len(loci)) == (depth >= DEEP_DEPTH)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    ors, oas = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=8)
    with vb.Engine("coverage") as eng:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
    assert (tiles[FOLD_CLASS] > 0) == any(fold), tiles
    bad = np.nonzero((rs.astype(np.int32) != ors) | (as_.astype(np.int32) != oas))[0]
    msgs = [f"pair {p}: locus {pl[p]} (x {xs[pl[p]]}, ref {len(refs[pl[p]])} alt {len(alts[pl[p]])}), read {len(reads[p])} "
            f"bases: gpu ({rs[p]}, {as_[p]}) oracle ({ors[p]}, {oas[p]})" for p in bad[:8]]
    assert bad.size == 0, f"{bad.size} of {len(pr)} pairs differ\n" + "\n".join(msgs)


@pytest.mark.parametrize("pad", [97, 100, 109])
def test_shared_extension_triplets(vb, oracle, pad):
    loci, _ = _loci(pad, 8, 9000 + pad)
    sb = seam_cases.whole_path_batch(vb, loci)
    ob = to_oracle_batch(oracle, sb)
    for mode in ("consensus", "coverage", "alt_frac"):
        with vb.Engine(mode) as eng:
            eng.set_barcodes(vb.Barcodes(seam_cases.BARCODES))
            got = eng.run(sb)
            tiles = eng.tile_counts()
        exp = oracle.run_batch(ob, oracle.Barcodes(seam_cases.BARCODES), oracle.MODES[mode], False, n_threads=8)
        assert tiles[FOLD_CLASS] > 0, tiles
        assert_same_triplets(got, exp)
        assert got.metrics == exp.metrics
