"""GPU seam suite (-m gpu): the planted-seam cases of tests/seam_cases.py, scored by the kernel family they are routed
to and compared bit for bit with the oracle.  Every case's optimal alignment crosses a named seam of that kernel (a lane,
pass, phase, row-block or fold seam) in a way that a dropped carry would change, so a kernel that loses a carry fails
here with the kernel, the seam, the witness and the pair named."""
import numpy as np
import pytest

import seam_cases
from conftest import assert_same_triplets, to_oracle_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


def _check(vb, oracle, fam_name, kernel, engine_kw, cls, ppw, loci, what):
    refs, alts, reads, pr, pl, cases = seam_cases.pairs(loci)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    ors, oas = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=8)
    with vb.Engine("coverage", **engine_kw) as eng:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
    assert tiles[cls] > 0 and sum(tiles) == tiles[cls], (fam_name, kernel, "tiles went elsewhere", tiles)
    bad = np.nonzero((rs.astype(np.int32) != ors) | (as_.astype(np.int32) != oas))[0]
    msgs = [f"{kernel}: seam '{cases[p].seam}' ({cases[p].style}), witness {cases[p].witness}, pair {p} "
            f"(locus {pl[p]}, tile slot {int(p - np.searchsorted(pl, pl[p])) % ppw}, read {len(reads[p])} bases): "
            f"gpu ({rs[p]}, {as_[p]}) oracle ({ors[p]}, {oas[p]})" for p in bad[:8]]
    assert bad.size == 0, f"{what}: {bad.size} of {len(pr)} pairs differ\n" + "\n".join(msgs)


@pytest.mark.parametrize("name", list(seam_cases.FAMILIES))
def test_planted_seams_bit_exact(vb, oracle, name):
    fam = seam_cases.FAMILIES[name]
    _check(vb, oracle, name, fam.kernel, fam.engine, fam.cls, fam.ppw, seam_cases.build(name), name)


def _generic_loci(names=tuple(seam_cases.FAMILIES)):
    """the planted loci of these families with an 'N' after both windows: exotic, so vtx_k_sw_generic scores them"""
    return [seam_cases.Locus(loc.ref + b"N", loc.alt + b"N", loc.reads, loc.cases)
            for name in names for loc in seam_cases.build(name)]


def test_planted_seams_generic_control(vb, oracle):
    """The same planted cases through vtx_k_sw_generic; it has no seams, so it must agree with the oracle on all of them."""
    _check(vb, oracle, "generic", "vtx_k_sw_generic", {}, 4, 16, _generic_loci(), "generic control")


# ------------------------------------------------------------------------------------------------
# vtx_config.min_score is a run-time field that every kernel's epilogue (call_and_scatter) reads
# ------------------------------------------------------------------------------------------------
MIN_SCORES = [-1, 0, 1, 24, 26, 60, 10 ** 6]


@pytest.mark.parametrize("name", list(seam_cases.FAMILIES) + ["generic"])
def test_min_score_through_every_kernel(vb, oracle, name):
    if name == "generic":                           # vtx_k_sw_generic: planted loci of a single-phase and the folded family
        engine, cls = {}, 4
        loci = _generic_loci(("class0", "fold"))[::4]
    else:
        fam = seam_cases.FAMILIES[name]
        engine, cls = fam.engine, fam.cls
        loci = seam_cases.build(name)[:12]
    sb = seam_cases.whole_path_batch(vb, loci)
    ob = to_oracle_batch(oracle, sb)
    obc = oracle.Barcodes(seam_cases.BARCODES)
    bcs = vb.Barcodes(seam_cases.BARCODES)
    n_listed = int(sum(1 for i in range(sb.n_reads) if i % 6 < 5))
    n_allN = int(sum((sb.cand_start[1:].astype(np.int64) - 1) % 6 < 5))       # the last read of every locus, if listed
    for s in MIN_SCORES:
        for mode in ("consensus", "coverage", "alt_frac"):
            with vb.Engine(mode, min_score=s, **engine) as eng:
                eng.set_barcodes(bcs)
                got = eng.run(sb)
                tiles = eng.tile_counts()
            exp = oracle.run_batch(ob, obc, oracle.MODES[mode], False, n_threads=4, min_score=s)
            assert tiles[cls] > 0 and sum(tiles) == tiles[cls], (name, s, tiles)
            assert_same_triplets(got, exp)
            assert got.metrics == exp.metrics and got.metrics["num_scored"] == n_listed, (name, s, mode)
            if mode == "consensus":                 # cells with UNKNOWN calls only emit no entry in this mode
                continue
            calls = int(got.ref_cnt.sum() + got.alt_cnt.sum() + got.unk_cnt.sum())
            if s <= 0:                              # every pair gets a call; a read of all N (a tie) is UNKNOWN
                assert calls == n_listed and int(got.unk_cnt.sum()) >= n_allN, (name, s, mode)
            if s == 10 ** 6:                        # nothing is called
                assert calls == 0, (name, s, mode)
