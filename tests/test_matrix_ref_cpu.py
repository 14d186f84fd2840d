"""CPU: tests/matrix_ref.py (the NumPy restatement of matrix assembly) against the C oracle, bit for bit, and the seam
shards of tests/slot_cases.py checked for the seams they are built to cross.  The GPU suite
(test_gpu_matrix_seams.py) compares the kernels with matrix_ref on shards too large for the oracle, so matrix_ref is
pinned here on every input the oracle can take."""
import numpy as np
import pytest

import matrix_ref
import slot_cases as S
from conftest import assert_same_triplets

MODES = ("consensus", "coverage", "alt_frac")


def _check(oracle, batch, keys, mode, umi, min_score=25, threads=4):
    """matrix_ref fed the oracle's scores of every candidate == oracle.run_batch"""
    b = batch.normalized()
    loc = np.repeat(np.arange(b.n_loci), np.diff(b.cand_start.astype(np.int64))).astype(np.uint32)
    rs, as_ = oracle.score_pairs(b, b.cand_read, loc, n_threads=threads)
    got = matrix_ref.assemble(b, keys, mode, umi, rs, as_, min_score)
    exp = oracle.run_batch(b, oracle.Barcodes(list(dict.fromkeys(keys))), oracle.MODES[mode], umi, n_threads=threads,
                           min_score=min_score)
    assert_same_triplets(got, exp)
    assert got.metrics == exp.metrics
    return got


def test_golden_batches_every_mode_and_barcode_list(oracle, goldens, golden_batches):
    for name, batch in golden_batches.items():
        for bl, keys in goldens["barcodes"].items():
            for mode in MODES:
                for umi in (False, True):
                    _check(oracle, batch, [k.encode() for k in keys], mode, umi)
    # and each golden case as the reference's tests run it
    n = 0
    for case in goldens["cases"]:
        n += len(_check(oracle, golden_batches[case["batch"]], [k.encode() for k in goldens["barcodes"][case["barcodes"]]],
                        case["scoring_method"], case["umi"]).row)
    assert n > 0


@pytest.mark.parametrize("umi", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_synthetic_shards(oracle, mode, umi):
    import vartrix_b200 as vb
    sb, bcs, _info = vb.synth.make_shard(150, 60, depth=20, seed=31, kind="indel" if umi else "snv", umi=True,
                                         read_len=60, padding=40)
    from conftest import to_oracle_batch
    got = _check(oracle, to_oracle_batch(oracle, sb), bcs.keys, mode, umi)
    assert got.metrics["num_not_cell_bc"] > 0


def _irregular(oracle, rng):
    """shared reads, repeated candidates, missing tags and UMIs, tiny and repeated barcode lists, calls near 25"""
    n_loci = int(rng.integers(1, 8))
    n_reads = int(rng.integers(1, 40))
    tags = [b"AAAC-1", b"AAAG-1", b"CCCC-1", b"GGTT-1", b"TTTT-2", b"A"]
    keys = [tags[i] for i in rng.integers(0, len(tags), int(rng.integers(1, 6)))]      # may repeat: first index wins
    refs, alts, reads = [], [], []
    for _ in range(n_loci):
        ref = bytes(rng.choice(list(b"ACGT"), int(rng.integers(30, 60))).astype(np.uint8))
        v = int(rng.integers(0, len(ref)))
        alt = ref[:v] + bytes(rng.choice(list(b"ACGT"), int(rng.integers(0, 3))).astype(np.uint8)) + ref[v + 1:]
        refs.append(ref); alts.append(alt)
    for _ in range(n_reads):
        src = refs[int(rng.integers(0, n_loci))] if rng.random() < 0.5 else alts[int(rng.integers(0, n_loci))]
        m = int(rng.integers(10, 40))
        s = int(rng.integers(0, max(1, len(src) - m)))
        rd = bytearray(src[s:s + m] or b"A")
        for _ in range(int(rng.integers(0, 3))):
            rd[int(rng.integers(0, len(rd)))] = b"ACGT"[int(rng.integers(0, 4))]
        reads.append(bytes(rd))
    import seam_cases

    class _VB:                                  # seam_cases.staged_batch builds through vb.StagedBatch(**fields)
        StagedBatch = staticmethod(lambda **f: f)
    f = seam_cases.staged_batch(_VB, refs, alts, reads)
    depth = rng.integers(0, 12, n_loci)
    f["cand_start"] = np.concatenate([[0], np.cumsum(depth)]).astype(np.uint64)
    f["cand_read"] = rng.integers(0, n_reads, int(depth.sum())).astype(np.uint32)      # shared and repeated reads
    pool = tags + [b"NNNN-1"]
    pick = rng.integers(0, len(pool), n_reads)
    offs = np.concatenate([[0], np.cumsum([len(t) for t in pool])])
    f["cb_bytes"] = np.frombuffer(b"".join(pool), np.uint8).copy()
    f["read_cb_off"] = np.where(rng.random(n_reads) < 0.1, 0xFFFFFFFF, offs[pick]).astype(np.uint32)
    f["read_cb_len"] = np.array([len(pool[i]) for i in pick], np.uint16)
    umis = np.array([0, 1, 2, 1 << 40, 0xFFFFFFFFFFFFFFFF], np.uint64)
    f["read_umi_key"] = umis[rng.integers(0, len(umis), n_reads)]
    for k in ("ref_off", "ref_len", "alt_off", "alt_len", "read_off", "read_len", "read_cb_off", "read_cb_len"):
        f[k] = np.asarray(f[k])
    f["locus_row"] = np.arange(n_loci, dtype=np.uint32)
    n_rows = f.pop("n_rows")
    return oracle.Batch(**f, n_rows=n_rows), keys


def test_random_irregular_shards(oracle):
    rng = np.random.default_rng(77)
    for i in range(300):
        batch, keys = _irregular(oracle, rng)
        _check(oracle, batch, keys, MODES[i % 3], bool(i & 4), min_score=(0, 25, 26)[(i // 3) % 3], threads=1)


@pytest.fixture(scope="module")
def template_scores(oracle):
    f, pr, pl = S.template_batch()
    n_rows = f.pop("n_rows")
    return oracle.score_pairs(oracle.Batch(**f, n_rows=n_rows), pr, pl)


def test_templates_make_the_calls_they_are_named_for(template_scores):
    rs, as_ = template_scores
    calls = matrix_ref.evaluate_scores(rs, as_).reshape(2, 4)
    want = [matrix_ref.REF, matrix_ref.ALT, matrix_ref.UNKNOWN, matrix_ref.NONE]
    assert (calls == want).all(), (rs, as_)
    assert (rs.reshape(2, 4)[:, 2] == 30).all() and (rs.reshape(2, 4)[:, 3] == 20).all()


def _oracle_batch(oracle, shard):
    f = S.fields(shard)
    n_rows = f.pop("n_rows")
    return oracle.Batch(**f, n_rows=n_rows)


@pytest.mark.parametrize("case", ["ladder", "umi_grid", "modes"])
def test_seam_shards_at_reduced_depth(oracle, template_scores, case):
    """matrix_ref fed the template scores == the oracle scoring every read (the GPU suite's expectation, pinned)"""
    shard = {"ladder": lambda: S.ladder(depths=(1, 127, 128, 129, 1023, 1024, 1025, 1152, 2047, 2048, 2049)),
             "umi_grid": S.umi_grid, "modes": S.modes}[case]()
    batch = _oracle_batch(oracle, shard)
    keys = S.barcodes(shard.n_barcodes)
    bcs = oracle.Barcodes(keys)
    for mode in MODES:
        for umi in (False, True):
            rs, as_ = S.expected_scores(shard, *template_scores)
            got = matrix_ref.assemble(batch, keys, mode, umi, rs, as_)
            exp = oracle.run_batch(batch, bcs, oracle.MODES[mode], umi, n_threads=8)
            assert_same_triplets(got, exp)
            assert got.metrics == exp.metrics, (case, mode, umi)


def test_umi_rule_grid_is_complete(template_scores):
    g = S.umi_groups()
    assert all((r, a, u, nn) in set(g) for r in range(9) for a in range(9 - r) for u in range(9 - r - a) for nn in (0, 2)
               if r + a + u or nn)
    assert {(0, 0, 0, k) for k in (1, 2, 3)} <= set(g)
    for k in range(1, 51):
        for top in (3 * k, 3 * k - 1):
            assert any(a == top and r + a + u == 4 * k for r, a, u, _ in g)
            assert any(r == top and r + a + u == 4 * k for r, a, u, _ in g)
    shard = S.umi_grid()
    d = shard.depth()
    assert d[:-1].max() <= S.SMALL_MAX and d[-1] > S.SMALL_MAX
    # each copy of the grid mixes collapsed calls of several groups in a cell
    rs, as_ = S.expected_scores(shard, *template_scores)
    for lo, hi in ((0, shard.n_loci - 1), (shard.n_loci - 1, shard.n_loci)):
        s, e = int(shard.cand_start[lo]), int(shard.cand_start[hi])
        cells = np.unique(shard.cb[s:e])
        assert 20 <= cells.size < len(g) / 10
    # keys that differ only in the high or only in the low half, bit 61, VTX_UMI_KEY_MAX
    keys = set(int(k) for k in S.UMI_POOL)
    assert S.UMI_KEY_MAX in keys and any(k >> 61 & 1 and k != S.UMI_KEY_MAX for k in keys)
    assert any((a ^ b) >> 32 and not (a ^ b) & 0xFFFFFFFF for a in keys for b in keys)
    assert any((a ^ b) and not (a ^ b) >> 32 for a in keys for b in keys)


def test_ladder_reaches_every_seam():
    shard = S.ladder()
    facts = [S.locus_facts(shard, l, umi=True) for l in range(shard.n_loci)]
    depths = {f["d"] for f in facts}
    assert depths == set(S.LADDER)
    assert {f["P"] for f in facts} >= {1024, 2048, 4096, 131072}
    for d in S.LADDER:
        Ds = {f["D"] for f in facts if f["d"] == d}
        assert Ds == set(S.ladder_pairs(d)), d
    mid = [f for f in facts if S.SLOT_CHUNK < f["d"] <= S.SMALL_MAX]
    assert any(f["first_and_repeat_in_chunk1"] for f in mid)
    assert any(f["chunk0_repeats_only_in_chunk1"] for f in mid)
    assert any(f["twin_1023_1024"] for f in mid)
    deep = [f for f in facts if f["d"] > S.SMALL_MAX]
    # hash-table wrap-around: with two distinct keys in the last bucket, linear probing wraps to bucket 0
    assert all(f["cell_wraps"] >= min(f["D"], 2) for f in deep)
    assert all(f["umi_wraps"] >= 2 for f in deep)
    # columns above 16 bits, descending against file order
    assert shard.cb.max() >= 1 << 16 and shard.n_barcodes > 1 << 17
    for l in range(shard.n_loci):
        s, e = int(shard.cand_start[l]), int(shard.cand_start[l + 1])
        cb = shard.cb[s:e]
        _, first = np.unique(cb, return_index=True)
        first_cols = cb[np.sort(first)]
        assert (np.diff(first_cols) < 0).all(), l
    assert np.isin(S.UMI_POOL, shard.umi).all()
    assert (shard.depth() == 100_000).any() and shard.n_pairs > 1_000_000


def test_crowd_many_loci_counters_modes():
    crowd = S.crowd(132)
    d = crowd.depth()
    deep = d > S.SMALL_MAX
    assert deep.sum() == 2 * 132 + 1 and d[deep].max() <= 2100 and deep[0] and deep[-1]
    runs = np.diff(np.nonzero(np.diff(np.concatenate([[0], deep.astype(int), [0]])))[0])[::2]
    assert runs.max() > 1 and (~deep).sum() > 0
    many = S.many_loci()
    assert many.n_loci > 65_535 * 8 and many.depth().min() == 1 and many.depth().max() == 3
    cnt = S.counters()
    assert cnt.n_loci == 1 and np.unique(cnt.cb).size == 1 and np.unique(cnt.umi).size == 1
    assert (cnt.tmpl == S.T_ALT).sum() == (1 << 21) + 1 == (cnt.tmpl == S.T_TIE).sum() and (cnt.tmpl == S.T_REF).sum() == 3
    modes = S.modes()
    assert (modes.cb == S.UNLISTED).any() and (modes.cb == S.NO_TAG).any() and (modes.umi == S.NO_UMI).any()


def test_mode_value_cells(oracle, template_scores):
    """the modes shard has cells with only None reads (coverage 0/0, alt_frac NaN, no consensus entry), cells with only
    UNKNOWN calls and cells of every consensus value"""
    shard = S.modes()
    batch = _oracle_batch(oracle, shard)
    rs, as_ = S.expected_scores(shard, *template_scores)
    keys = S.barcodes(shard.n_barcodes)
    for umi in (False, True):
        cov = matrix_ref.assemble(batch, keys, "coverage", umi, rs, as_)
        frac = matrix_ref.assemble(batch, keys, "alt_frac", umi, rs, as_)
        cons = matrix_ref.assemble(batch, keys, "consensus", umi, rs, as_)
        none = (cov.ref_cnt + cov.alt_cnt + cov.unk_cnt) == 0
        assert none.sum() >= 20 and np.isnan(frac.val[none]).all()
        assert ((cov.unk_cnt > 0) & (cov.ref_cnt == 0) & (cov.alt_cnt == 0)).sum() >= 20
        assert {1.0, 2.0, 3.0} <= set(cons.val.tolist()) and len(cons.row) < len(cov.row)
