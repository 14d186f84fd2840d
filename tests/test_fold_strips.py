"""The folded kernel's allele columns score each read in eight 19-row strips, one per lane, that advance over the columns
together; the vertical gap F reaches a strip through an exclusive max-scan over the strips above it.  A seam case of
tests/seam_cases.py ("allele rows 19k") crosses one strip boundary with a 2-6 base insertion, so it only sees the strip
directly above.  Here every read carries a 21-45 base insertion at an allele column that starts just above row 19 k and
runs across rows 19 k and 19 (k + 1) (and 19 (k + 2) when long enough): the gap reaches a strip from two or more strips up.

A best alignment through an insertion of L bases needs L + 6 matched bases on either side of it (the gap costs 5 + L),
so in reads of at most 152 bases such a gap can only start just above rows 38, 57, 76 or 95.

Each case keeps its witness: the haplotype halves whose score changes under the ablation "F not carried across
strips" (tests/sw_ref.py row "gap" seams at every strip boundary in the allele columns).  A kernel that drops F at a
strip boundary gets that half wrong.  CPU: every start row and every halves pattern is witnessed, and sw_ref agrees
with the oracle.  GPU: vtx_k_sw_fold takes every tile and agrees with the oracle bit for bit."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import pytest

import seam_cases
import sw_ref
from conftest import to_oracle_batch

STRIP, ROWS = 19, 152              # the folded kernel's allele columns: 8 lanes x 19 read rows
STARTS = (38, 57, 76, 95)
HALVES = ("ref", "alt", "both")
FOLD_CLASS = 7                     # tile class of vtx_k_sw_fold in vtx_last_tile_counts


@dataclass
class StripCase:
    seam: str
    style: str
    witness: dict                  # {"strips": "ref" / "alt" / "both"}
    read: bytes
    first: int                     # read row of the first inserted base
    length: int                    # inserted bases


def strip_ablation(n: int) -> dict:
    """sw_ref.score arguments: F stopped at every strip boundary inside the allele columns [96, n - 96)"""
    return dict(row_gap=[(r, 96, n - 96) for r in range(STRIP, ROWS, STRIP)])


def _plant(rng, T: bytes, r: int, m: int):
    """a read of m bases whose insertion after an allele column starts just above row r and reaches row r + 19"""
    n = len(T)
    if n - 192 < 2:
        return None
    p = int(rng.integers(97, n - 96))                 # inserted after hap column p - 1
    q = r - int(rng.integers(1, 5))
    L_lo = r + STRIP + 1 - q                          # the last inserted row is at least r + 19
    L_hi = min(45, q - 6, (m - q - 6) // 2)           # room for L + 6 matched bases on either side
    if L_hi < L_lo:
        return None
    L = int(rng.integers(L_lo, L_hi + 1))
    L1 = min(q, L + 6 + int(rng.integers(0, 10)))
    L2 = min(n - p, m - q - L, L + 6 + int(rng.integers(0, 10)))
    if L2 < L + 6:
        return None
    read = seam_cases._rand(rng, q - L1) + T[p - L1:p] + seam_cases._rand(rng, L) + T[p:p + L2]
    return read + seam_cases._rand(rng, m - len(read)), q, L


def witness(read: bytes, ref: bytes, alt: bytes):
    true = sw_ref.score([read, read], [ref, alt])
    abl = [sw_ref.score_pair(read, ref, **strip_ablation(len(ref))), sw_ref.score_pair(read, alt, **strip_ablation(len(alt)))]
    hit = [h for h, t, a in zip(("ref", "alt"), true, abl) if t != a]
    return ("both" if len(hit) == 2 else hit[0]) if hit else None


@functools.lru_cache(maxsize=None)
def build(seed: int = 0) -> tuple:
    """loci of folded-kernel windows whose reads all carry a witnessed multi-strip insertion"""
    rng = np.random.default_rng(seed + 1900)
    need_start = {r: 2 for r in STARTS}
    need_half = {h: 1 for h in HALVES}
    loci = []
    for _it in range(3000):
        if len(loci) >= 12 and not any(need_start.values()) and not any(need_half.values()):
            break
        ref, alt = seam_cases._fold_window(rng)
        loc = seam_cases.Locus(ref, alt)
        long_reads = rng.random() < 0.25              # a tile of 149-152-base reads fills every strip
        for _slot in range(8 if long_reads else int(rng.integers(1, 10))):
            for _try in range(8):
                open_starts = [r for r in STARTS if need_start[r]] or list(STARTS)
                r = open_starts[int(rng.integers(0, len(open_starts)))]
                src = alt if need_half["alt"] or rng.random() < 0.4 else ref
                m = int(rng.integers(149, 153)) if long_reads else int(rng.integers(110, 153))
                got = _plant(rng, src, r, m)
                if got is None:
                    continue
                read, q, L = got
                h = witness(read, ref, alt)
                if h:
                    break
            else:
                continue
            loc.reads.append(read)
            loc.cases.append(StripCase(f"allele strips {r}", "long_ins", {"strips": h}, read, q, L))
            need_start[r] = max(0, need_start[r] - 1)
            need_half[h] = 0
        if loc.reads:
            loci.append(loc)
    return tuple(loci)


def test_strip_cases_are_witnessed(oracle):
    loci = build()
    refs, alts, reads, pr, pl, cases = seam_cases.pairs(loci)
    assert {c.seam for c in cases} == {f"allele strips {r}" for r in STARTS}
    assert {c.witness["strips"] for c in cases} == set(HALVES)
    for c in cases:                                   # the gap covers rows just above 19 k, 19 k and 19 (k + 1)
        k = int(c.seam.split()[-1])
        assert c.first < k and c.first + c.length - 1 >= k + STRIP and 21 <= c.length <= 45, c
    lens = np.array([len(r) for r in reads])
    assert lens.max() <= ROWS and any(len(loc.reads[t:t + 4]) == 4 and all(len(r) >= 149 for r in loc.reads[t:t + 4])
                                      for loc in loci for t in range(0, len(loc.reads), 4))
    assert all(loc.ref[:96] == loc.alt[:96] and loc.ref[-96:] == loc.alt[-96:] for loc in loci)
    true_r = sw_ref.score(reads, [refs[l] for l in pl])
    true_a = sw_ref.score(reads, [alts[l] for l in pl])
    assert np.array_equal(true_r, [oracle.sw_full(r, refs[l]) for r, l in zip(reads, pl)])
    assert np.array_equal(true_a, [oracle.sw_full(r, alts[l]) for r, l in zip(reads, pl)])
    for p, c in enumerate(cases):                     # the recorded witness holds
        for half, hap, t in (("ref", refs[pl[p]], true_r[p]), ("alt", alts[pl[p]], true_a[p])):
            if c.witness["strips"] in (half, "both"):
                assert sw_ref.score_pair(reads[p], hap, **strip_ablation(len(hap))) != t, (p, c)


@pytest.mark.gpu
def test_gpu_fold_strips_bit_exact(oracle):
    import vartrix_b200 as vb
    refs, alts, reads, pr, pl, cases = seam_cases.pairs(build())
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    ors, oas = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=8)
    with vb.Engine("coverage") as eng:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
    assert tiles[FOLD_CLASS] > 0 and sum(tiles) == tiles[FOLD_CLASS], tiles
    bad = np.nonzero((rs.astype(np.int32) != ors) | (as_.astype(np.int32) != oas))[0]
    msgs = [f"{cases[p].seam}: {cases[p].length}-base insertion from row {cases[p].first}, witness {cases[p].witness}, "
            f"pair {p} (read {len(reads[p])} bases): gpu ({rs[p]}, {as_[p]}) oracle ({ors[p]}, {oas[p]})" for p in bad[:8]]
    assert bad.size == 0, f"{bad.size} of {len(pr)} pairs differ\n" + "\n".join(msgs)
