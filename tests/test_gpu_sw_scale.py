"""Chunked work stealing at production tile counts (-m gpu).

The tiled Smith-Waterman kernels take tile_chunk = max(1, min(8, n_tiles / (warps * 16))) consecutive tiles per atomic
and walk them across locus boundaries, reusing the per-locus profile / allele tables while the locus stays the same.
Small test batches only ever run tile_chunk = 1.  Here one score_pairs call holds at least 8 * 16 * 64 * n_SM tiles of
the kernel under test (64 warps per SM is the hardware maximum, so tile_chunk = 8 at any occupancy), built by repeating
a pool of distinct template loci in a shuffled order: consecutive loci are always different windows, read counts vary
(chunks start inside loci, last tiles are partial), and one variant puts loci of other kernels in between (runs of
zero-tile loci in the class's tile_start).  The oracle scores the pool once; every pair is checked bit for bit."""
import numpy as np
import pytest

import seam_cases
from conftest import to_oracle_batch

pytestmark = pytest.mark.gpu

# family -> (Engine flags, tile class, pairs per tile, read lengths, family whose loci go in between)
FAMILIES = {
    "class0": (dict(no_split=True), 0, 4, (40, 151), "class2"),
    "class1": (dict(no_split=True), 1, 4, (40, 200), "class0"),
    "class2": (dict(no_split=True), 2, 4, (40, 256), "class3"),
    "class3": (dict(no_split=True), 3, 4, (40, 256), "class1"),
    "multi": (dict(), 3, 4, (40, 256), "split0"),
    "split0": (dict(no_fold=True), 5, 8, (40, 256), "class3"),
    "split1": (dict(no_fold=True), 6, 8, (40, 256), "split0"),
    "fold": (dict(), 7, 4, (40, 152), "split1"),
}


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


def _pool(name, n_templates, m_range, max_reads, seed):
    """n_templates distinct loci of the family's window shape, each with 1..max_reads reads (substrings of ref or alt
    with substitutions and short indels, some random)"""
    rng = np.random.default_rng(seed)
    window = seam_cases.FAMILIES[name].window
    refs, alts, reads, count = [], [], [], []
    for _ in range(n_templates):
        ref, alt = window(rng)
        refs.append(ref); alts.append(alt)
        k = int(rng.integers(1, max_reads + 1))
        count.append(k)
        for _ in range(k):
            m = int(rng.integers(m_range[0], m_range[1] + 1))
            src = ref if rng.random() < 0.5 else alt
            if rng.random() < 0.15:
                reads.append(seam_cases._rand(rng, m))
                continue
            s = int(rng.integers(-10, max(1, len(src) - m // 2)))
            seq = (seam_cases._rand(rng, max(0, -s)) + src[max(0, s):max(0, s) + m])
            seq = seam_cases._edit(rng, seq, 0.02)
            reads.append((seq + seam_cases._rand(rng, m))[:m])
    return refs, alts, reads, np.array(count, np.int64)


def _order(rng, n_templates, n_loci):
    """n_loci template ids, shuffled rounds of the whole pool, never the same template twice in a row"""
    rounds = -(-n_loci // n_templates)
    seq = np.concatenate([rng.permutation(n_templates) for _ in range(rounds)])[:n_loci]
    for i in np.nonzero(seq[1:] == seq[:-1])[0] + 1:
        j = i + 1 if i + 1 < len(seq) else i - 2
        seq[i], seq[j] = seq[j], seq[i]
    assert not (seq[1:] == seq[:-1]).any()
    return seq


def _big_call(pools, seq_pool, seq_tmpl):
    """one batch whose locus l is template seq_tmpl[l] of pool seq_pool[l]: windows and reads are shared by offset"""
    hap, ref_off, ref_len, alt_off, alt_len, nib, read_off, read_len, rbase = [], [], [], [], [], [], [], [], []
    hpos, npos, nreads = 0, 0, 0
    for sb, _count, _start in pools:
        ref_off.append(sb.ref_off.astype(np.int64) + hpos); alt_off.append(sb.alt_off.astype(np.int64) + hpos)
        ref_len.append(sb.ref_len); alt_len.append(sb.alt_len)
        read_off.append(sb.read_off.astype(np.int64) + npos); read_len.append(sb.read_len)
        hap.append(sb.hap_bytes); nib.append(sb.read_nib)
        rbase.append(nreads)
        hpos += sb.hap_bytes.size; npos += sb.read_nib.size; nreads += sb.n_reads
    L = len(seq_tmpl)
    # per-locus fields gathered through a flat index into the concatenated pools
    tbase = np.cumsum([0] + [len(c) for _sb, c, _s in pools])[:-1]
    flat = tbase[seq_pool] + seq_tmpl
    cat = lambda xs: np.concatenate(xs)
    cnt_all = cat([c for _sb, c, _s in pools]); start_all = cat([s + rbase[p] for p, (_sb, _c, s) in enumerate(pools)])
    cnt = cnt_all[flat]
    first = np.repeat(start_all[flat], cnt)
    within = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    pair_read = (first + within).astype(np.uint32)
    pair_locus = np.repeat(np.arange(L), cnt).astype(np.uint32)
    import vartrix_b200 as vb
    sb = vb.StagedBatch(
        locus_row=np.arange(L), hap_bytes=cat(hap), ref_off=cat(ref_off)[flat], ref_len=cat(ref_len)[flat],
        alt_off=cat(alt_off)[flat], alt_len=cat(alt_len)[flat], cand_start=np.zeros(L + 1, np.uint64),
        read_nib=cat(nib), read_off=cat(read_off), read_len=cat(read_len), cb_bytes=np.zeros(0, np.uint8),
        read_cb_off=np.full(nreads, 0xFFFFFFFF), read_cb_len=np.zeros(nreads),
        read_umi_key=np.full(nreads, 0xFFFFFFFFFFFFFFFF, np.uint64), cand_read=np.zeros(0, np.uint32), n_rows=L)
    return sb, pair_read, pair_locus


def _scored_pool(vb, oracle, name, n_templates, seed):
    kw, cls, ppw, m_range, _other = FAMILIES[name]
    refs, alts, reads, count = _pool(name, n_templates, m_range, 2 * ppw + 1, seed)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    start = np.concatenate([[0], np.cumsum(count)[:-1]])
    pr = np.arange(len(reads), dtype=np.uint32); pl = np.repeat(np.arange(n_templates), count).astype(np.uint32)
    rs, as_ = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=16)
    return (sb, count, start), rs, as_


@pytest.mark.parametrize("interleaved", [False, True], ids=["alone", "interleaved"])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_chunked_tiles_bit_exact(vb, oracle, name, interleaved):
    import torch
    kw, cls, ppw, _m, other = FAMILIES[name]
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    need = 8 * 16 * 64 * n_sm                      # tiles for tile_chunk = 8 at any occupancy
    rng = np.random.default_rng(sum(map(ord, name)) + interleaved)
    pool, prs, pas = _scored_pool(vb, oracle, name, 3000, sum(map(ord, name)))
    pools, exp_r, exp_a = [pool], [prs], [pas]
    tiles_per = -(-pool[1] // ppw)
    n_target = int(1.05 * need / tiles_per.mean()) + 1
    seq_tmpl = _order(rng, len(pool[1]), n_target)
    seq_pool = np.zeros(n_target, np.int64)
    if interleaved:
        # loci of another kernel in runs of 0-3 between the target loci
        opool, ors_, oas_ = _scored_pool(vb, oracle, other, 600, sum(map(ord, other)) + 1)
        pools.append(opool); exp_r.append(ors_); exp_a.append(oas_)
        runs = rng.integers(0, 4, n_target)
        seq_pool = np.repeat(np.stack([np.zeros(n_target, np.int64), np.ones(n_target, np.int64)], 1).reshape(-1),
                             np.stack([np.ones(n_target, np.int64), runs], 1).reshape(-1))
        ot = _order(rng, len(opool[1]), int(runs.sum()))
        tmpl = np.zeros(len(seq_pool), np.int64)
        tmpl[seq_pool == 0] = seq_tmpl; tmpl[seq_pool == 1] = ot
        seq_tmpl = tmpl
    sb, pr, pl = _big_call(pools, seq_pool, seq_tmpl)
    with vb.Engine("coverage", **kw) as eng:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
    assert tiles[cls] >= need, (name, tiles, need)
    if not interleaved:
        assert sum(tiles) == tiles[cls], tiles
    else:
        assert sum(tiles) > tiles[cls], tiles
    er, ea = np.concatenate(exp_r), np.concatenate(exp_a)
    bad = np.nonzero((rs.astype(np.int32) != er[pr]) | (as_.astype(np.int32) != ea[pr]))[0]
    assert bad.size == 0, (name, interleaved, f"{bad.size} of {len(pr)} pairs differ", bad[:5], pl[bad[:5]])
