"""The merged profile of vtx_k_sw_fold (-m gpu).

The folded kernel's main pass looks up one 25-row table per locus: row 5 a + b, column c holds
{s(a, hap[c]), s(b, hap[n - 1 - c])}, where a is the code of read row i and b the code of read row m - 1 - i
(A, C, G, T -> 0..3, N and every IUPAC base -> 4).  Here reads are built so that every one of the 25 (a, b) pairs
meets every lane's 12-column block of the table in both halves; the reads are substrings of the window with bases
overwritten, so a row lines up with a known column of the forward and of the reversed DP.  Every pair is scored by the
folded kernel and compared bit for bit with the oracle."""
import numpy as np
import pytest

import seam_cases
from conftest import to_oracle_batch

pytestmark = pytest.mark.gpu

FOLD_CLASS = 7
P, LANE_COLS = 96, 12
ACGT = b"ACGT"
IUPAC = b"NRYKMSWBDHV="
CODE = {**{c: i for i, c in enumerate(ACGT)}, **{c: 4 for c in IUPAC}}


@pytest.fixture(scope="module")
def vb():
    import vartrix_b200
    return vartrix_b200


def _rand(rng, n):
    return np.frombuffer(ACGT, np.uint8)[rng.integers(0, 4, n)].tobytes()


def _window(rng, mid_ref, mid_alt):
    """a folded window: two common 96-base flanks (a few lower-case bytes, which match no read base), then alleles"""
    left, right = bytearray(_rand(rng, P)), bytearray(_rand(rng, P))
    for fl in (left, right):
        for j in rng.integers(0, P, 3):
            fl[j] = fl[j] | 0x20
    return bytes(left) + _rand(rng, mid_ref) + bytes(right), bytes(left) + _rand(rng, mid_alt) + bytes(right)


def _base(rng, code):
    return ACGT[code] if code < 4 else IUPAC[int(rng.integers(0, len(IUPAC)))]


def _read(rng, ref, kind, k):
    """(read, start): a substring of the ref window starting at `start`, with rows overwritten by `kind`"""
    n = len(ref)
    if kind == "allN":
        m = int(rng.integers(1, 153))
        return b"N" * m, int(rng.integers(0, n - m + 1))
    if kind == "ragged":                                       # the extremes, then any length
        m = (1, 152, 2, 151)[k] if k < 4 else int(rng.integers(1, 153))
    else:
        m = int(rng.integers(100, 153))
    s = int(rng.integers(0, n - m + 1))
    r = bytearray(ref[s:s + m].upper())
    if kind == "palindrome":                                   # read[i] == read[m - 1 - i]: pair rows (a, a) only
        for i in range(m // 2):
            r[m - 1 - i] = r[i]
    elif kind in ("pairs", "ragged"):                          # planted (a, b) pairs at rows i and m - 1 - i
        for i in rng.choice(m, max(1, m // 6), replace=False):
            a, b = int(rng.integers(0, 5)), int(rng.integers(0, 5))
            r[i] = _base(rng, a)
            r[m - 1 - i] = _base(rng, b) if m - 1 - i != i else r[i]
    elif kind in ("n_fwd", "n_rev", "n_both"):                 # N / IUPAC at row i, at row m - 1 - i, or at both
        for i in rng.choice(m, max(1, m // 8), replace=False):
            if kind != "n_rev":
                r[i] = _base(rng, 4)
            if kind != "n_fwd":
                r[m - 1 - i] = _base(rng, 4)
    return bytes(r), s


KINDS = ("pairs", "ragged", "palindrome", "n_fwd", "n_rev", "n_both", "allN")


def _batch(vb, rng, n_loci, reads_per_locus, mids):
    refs, alts, reads, pl, seen = [], [], [], [], np.zeros((25, 2, P // LANE_COLS), bool)
    for loc in range(n_loci):
        ref, alt = _window(rng, *mids[loc % len(mids)])
        refs.append(ref); alts.append(alt)
        n = len(ref)
        for k in range(reads_per_locus):
            rd, s = _read(rng, ref, KINDS[(loc + k) % len(KINDS)], loc // len(KINDS))
            m = len(rd)
            for i in range(m):                                 # row i meets column s + i forward, n - s - m + i reversed
                p = 5 * CODE[rd[i]] + CODE[rd[m - 1 - i]]
                for half, c in enumerate((s + i, n - s - m + i)):
                    if 0 <= c < P:
                        seen[p, half, c // LANE_COLS] = True
            reads.append(rd); pl.append(loc)
    sb = seam_cases.staged_batch(vb, refs, alts, reads)
    return sb, np.arange(len(reads), dtype=np.uint32), np.array(pl, np.uint32), reads, seen


@pytest.mark.parametrize("mids", [[(9, 9)], [(1, 1), (9, 9), (40, 40), (9, 1), (3, 40)]], ids=["snv", "mixed"])
def test_every_pair_row_bit_exact(vb, oracle, mids):
    rng = np.random.default_rng(20261015 + len(mids))
    sb, pr, pl, reads, seen = _batch(vb, rng, n_loci=240, reads_per_locus=14, mids=mids)
    assert seen.all(), f"pair rows x lane blocks not covered: {np.argwhere(~seen)[:8].tolist()}"
    lens = np.array([len(r) for r in reads])
    assert (lens % 2 == 0).any() and (lens % 2 == 1).any() and lens.min() == 1 and lens.max() == 152
    ors, oas = oracle.score_pairs(to_oracle_batch(oracle, sb), pr, pl, n_threads=8)
    with vb.Engine("coverage") as eng:
        rs, as_ = eng.score_pairs(sb, pr, pl)
        tiles = eng.tile_counts()
    assert tiles[FOLD_CLASS] > 0 and sum(tiles) == tiles[FOLD_CLASS], tiles
    bad = np.nonzero((rs.astype(np.int32) != ors) | (as_.astype(np.int32) != oas))[0]
    msgs = [f"pair {p} (locus {pl[p]}, read {reads[p]!r}): gpu ({rs[p]}, {as_[p]}) oracle ({ors[p]}, {oas[p]})"
            for p in bad[:6]]
    assert bad.size == 0, f"{bad.size} of {len(pr)} pairs differ\n" + "\n".join(msgs)
