"""CPU tests of the Smith-Waterman reference (tests/sw_ref.py) and of the planted-seam generator (tests/seam_cases.py):
sw_ref agrees with the oracle, its ablations mean what they say, and every kernel family's cases witness every seam
the GPU seam suite relies on."""
from collections import defaultdict

import numpy as np
import pytest

import seam_cases
import sw_ref


def _mutated(rng, src: bytes, alpha: bytes) -> bytes:
    s = bytearray(src)
    for _ in range(int(rng.integers(0, 6))):
        if not s:
            break
        k = int(rng.integers(0, len(s))); op = int(rng.integers(0, 3))
        if op == 0:
            s[k] = alpha[int(rng.integers(0, len(alpha)))]
        elif op == 1:
            del s[k:k + int(rng.integers(1, 7))]
        else:
            s[k:k] = bytes(rng.choice(np.frombuffer(alpha, np.uint8), int(rng.integers(1, 7))).tolist())
    return bytes(s)


def _random_pairs(seed, n_pairs):
    """random, mutated (substitutions and 1-6 base indels) and low-complexity pairs; reads decoded from BAM nibbles
    (N and IUPAC codes included), haplotypes with IUPAC bytes and lower case sometimes"""
    rng = np.random.default_rng(seed)
    reads, haps = [], []
    for i in range(n_pairs):
        alpha = (b"ACGT", b"AC", b"A", b"ACGTN", b"ACGTacgtRYN=")[i % 5]
        n = int(rng.integers(0, 260)); m = int(rng.integers(0, 200))
        hap = bytes(rng.choice(np.frombuffer(alpha, np.uint8), n).tolist())
        if n and rng.random() < 0.7:
            s = int(rng.integers(0, n))
            read = _mutated(rng, hap[s:s + m].upper(), b"ACGT")
        else:
            read = bytes(sw_ref.decode(rng.choice([1, 2, 4, 8, 15, 0, 3, 5], m)).tolist())
        reads.append(read); haps.append(hap)
    return reads, haps


def test_sw_ref_matches_oracle(oracle):
    reads, haps = _random_pairs(5, 3000)
    got = np.concatenate([sw_ref.score(reads[i:i + 500], haps[i:i + 500]) for i in range(0, len(reads), 500)])
    exp = np.array([oracle.sw_full(r, h) for r, h in zip(reads, haps)])
    bad = np.nonzero(got != exp)[0]
    assert bad.size == 0, [(int(i), reads[i], haps[i], int(got[i]), int(exp[i])) for i in bad[:3]]
    assert exp.max() > 100 and (exp == 0).any()


def test_sw_ref_ablations(oracle):
    """cut = the better of the two halves (columns or rows); gap never raises a score and only differs when a gap
    crosses; max_cols restricts the maximum only."""
    reads, haps = _random_pairs(6, 120)
    for r, h in zip(reads, haps):
        if len(h) < 4 or len(r) < 4:
            continue
        full = oracle.sw_full(r, h)
        c, q = len(h) // 2, len(r) // 2
        assert sw_ref.score_pair(r, h, col_cut=[c]) == max(oracle.sw_full(r, h[:c]), oracle.sw_full(r, h[c:]))
        assert sw_ref.score_pair(r, h, row_cut=[q]) == max(oracle.sw_full(r[:q], h), oracle.sw_full(r[q:], h))
        assert sw_ref.score_pair(r, h, col_gap=[c]) <= full and sw_ref.score_pair(r, h, row_gap=[q]) <= full
        assert sw_ref.score_pair(r, h, max_cols=(0, len(h))) == full
    # a 3-base deletion across column 40: gap at 40 costs a reopened gap (-5), a gap elsewhere costs nothing
    hap = bytes(np.random.default_rng(1).choice(np.frombuffer(b"ACGT", np.uint8), 80).tolist())
    read = hap[10:39] + hap[42:70]
    full = oracle.sw_full(read, hap)
    assert full == 29 + 28 - 8
    assert sw_ref.score_pair(read, hap, col_gap=[40]) == full - 5
    assert sw_ref.score_pair(read, hap, col_gap=[20, 60]) == full
    # a 3-base insertion across read row 30
    read = hap[10:38] + b"TTT" + hap[38:70]
    full = oracle.sw_full(read, hap)
    assert sw_ref.score_pair(read, hap, row_gap=[30]) < full and sw_ref.score_pair(read, hap, row_gap=[10]) == full


@pytest.mark.parametrize("name", list(seam_cases.FAMILIES))
def test_seam_generator_covers_every_seam(oracle, name):
    fam = seam_cases.FAMILIES[name]
    loci = seam_cases.build(name)
    refs, alts, reads, pr, pl, cases = seam_cases.pairs(loci)
    # coverage: every (seam, kind), every (kind, halves)
    need, need_halves = seam_cases.required(name)
    # the seam table itself: every lane hand-off of the single-phase classes, both row blocks with F and the diagonal
    C = dict(class0=26, class1=29, class2=32, class3=40).get(name)
    if C:
        assert {s for s, _k in need} == {f"lane {k * C}" for k in range(1, 8)}
    if name == "rowblock":
        assert need == {(f"row block {b} lane {g}", k) for b in (1024, 2048) for g in range(8) for k in ("gap", "cut")}
    got, got_halves = set(), set()
    for c in cases:
        for kind, h in c.witness.items():
            got.add((c.seam, kind)); got_halves.add((kind, h))
    assert not need - got, sorted(need - got)
    assert not need_halves - got_halves, sorted(need_halves - got_halves)
    # witness cases on every pair slot of a tile, ragged read lengths inside a tile
    slots, ragged = set(), False
    for loc in loci:
        for i, c in enumerate(loc.cases):
            if c.witness:
                slots.add(i % fam.ppw)
        for t in range(0, len(loc.reads), fam.ppw):
            ragged |= len({len(r) for r in loc.reads[t:t + fam.ppw]}) > 1
    assert slots == set(range(fam.ppw)) and ragged
    lens = np.array([len(r) for r in reads])
    assert lens.min() >= 1 and lens.max() <= (fam.m_hi if fam.m_lo < 1024 else 6000)
    if fam.m_lo > 1024:
        assert lens.min() > 1024
    if name.startswith("split"):
        assert lens.max() <= 256 and any(len(loc.reads) % 2 for loc in loci)      # read B of a phase-1 unit absent
        assert all(loc.ref[:96] == loc.alt[:96] for loc in loci)
    if name == "fold":
        assert lens.max() <= 152
        assert all(loc.ref[:96] == loc.alt[:96] and loc.ref[-96:] == loc.alt[-96:] and 193 <= len(loc.ref) <= 232
                   and 193 <= len(loc.alt) <= 232 for loc in loci)
        assert any(len(loc.reads[t:t + 4]) == 4 and all(149 <= len(r) <= 152 for r in loc.reads[t:t + 4])
                   for loc in loci for t in range(0, len(loc.reads), 4))
    # sw_ref agrees with the oracle on every case, and every recorded witness holds under sw_ref
    true_r = sw_ref.score(reads, [refs[l] for l in pl])
    true_a = sw_ref.score(reads, [alts[l] for l in pl])
    assert np.array_equal(true_r, [oracle.sw_full(r, refs[l]) for r, l in zip(reads, pl)])
    assert np.array_equal(true_a, [oracle.sw_full(r, alts[l]) for r, l in zip(reads, pl)])
    seams = {s.name: s for s in fam.seams}
    groups = defaultdict(list)                 # one sw_ref call per distinct ablation
    for p, c in enumerate(cases):
        for kind, h in c.witness.items():
            for half, hap, t in (("ref", refs[pl[p]], true_r[p]), ("alt", alts[pl[p]], true_a[p])):
                if h in (half, "both"):
                    kw = seam_cases._ablations(seams[c.seam], len(hap))[kind]
                    groups[repr(sorted(kw.items()))].append((kw, reads[p], hap, t, (c.seam, kind, half, p)))
    assert groups
    for items in groups.values():
        abl = sw_ref.score([x[1] for x in items], [x[2] for x in items], **items[0][0])
        same = [x[4] for x, a in zip(items, abl) if a == x[3]]
        assert not same, same[:5]
