"""GPU: the BGZF inflate kernel (vtx_bgzf_inflate, csrc/vtx_inflate.cuh) on hand-written DEFLATE streams (tests/deflate_craft.py)
that put batch, input-window and table seams where zlib's compressor rarely does, on a call of ~20 000 members spread over every
warp at non-contiguous output offsets, and on the trailer CRC flipped at each of its 32 bits.  zlib is the reference: a stream
it decodes comes out byte-identical with status 0; a stream it refuses gets a nonzero status, and its neighbours are unaffected."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from deflate_craft import build, corpus, lit, match, too_long

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import vartrix_b200 as vb
    with vb.Engine("coverage") as e:
        yield e


def _inflate_at(eng, members, out_offs, out_size, check_crc=True):
    """vtx_bgzf_inflate with explicit output offsets: members = [(payload, isize, crc)]"""
    from vartrix_b200 import _capi
    n = len(members)
    blocks = (_capi.BgzfBlock * max(n, 1))()
    comp = bytearray()
    for i, (payload, isize, crc) in enumerate(members):
        while len(comp) & 7:
            comp.append(0)
        blocks[i].in_off = len(comp); blocks[i].in_len = len(payload); blocks[i].out_len = isize
        blocks[i].out_off = out_offs[i]; blocks[i].crc32 = crc
        comp += payload
    comp += b"\0" * 16
    cbuf = (C.c_uint8 * len(comp)).from_buffer(comp)
    out = np.full(max(out_size, 1), 0xEE, np.uint8)
    status = np.full(max(n, 1), -1, np.int32)
    rc = eng._L.vtx_bgzf_inflate(eng._h, blocks, n, cbuf, len(comp) - 16, out.ctypes.data, out_size, status.ctypes.data, int(check_crc))
    assert rc == 0, eng._L.vtx_last_error(eng._h)
    return out, status[:n]


@pytest.mark.parametrize("check_crc", [True, False])
def test_crafted_corpus_matches_zlib(eng, check_crc):
    cases = corpus()
    members, want = [], []
    for name, s, out, _ in cases:
        if out is None:
            members.append((s, 4096, 0)); want.append(None)
        else:
            members.append((s, len(out), zlib.crc32(out) & 0xFFFFFFFF)); want.append(out)
    got, status = eng.bgzf_inflate(members, check_crc=check_crc)
    for (name, _, _, _), g, st, w in zip(cases, got, status, want):
        if w is None:
            assert st != 0, name
        else:
            assert st == 0 and g == w, (name, int(st))
    # the flawed streams again, and every valid one announced one byte short (output longer than ISIZE), each between two
    # valid neighbours in one call
    flawed = [m for m, w in zip(members, want) if w is None] + [(s, n, 0) for _, s, n in too_long(cases)]
    trio, expect = [], []
    valid = [(m, w) for m, w in zip(members, want) if w is not None]
    for k, m in enumerate(flawed):
        a, b = valid[(3 * k) % len(valid)], valid[(3 * k + 1) % len(valid)]
        trio += [a[0], m, b[0]]; expect += [a[1], None, b[1]]
    got, status = eng.bgzf_inflate(trio, check_crc=check_crc)
    for g, st, w in zip(got, status, expect):
        assert (st != 0) if w is None else (st == 0 and g == w)


def test_twenty_thousand_members_over_every_warp(eng):
    """one call, ~20 000 members: empty, 1-byte and 65 536-byte outputs among zlib and crafted ones, at output offsets with
    gaps between them (the gap bytes must stay untouched)"""
    rng = random.Random(5); nrng = np.random.default_rng(5)
    crafted = [(s, o) for _, s, o, _ in corpus(seed=11) if o is not None]
    members, raws = [], []
    for i in range(20_000):
        k = i % 20
        if k in (0, 7):
            raw = b""
        elif k in (1, 8, 15):
            raw = bytes([rng.randrange(256)])
        elif k == 3:
            raw = bytes(nrng.integers(0, 4, 65536, dtype=np.uint8) + 65)
        elif k in (5, 12):
            s, raw = crafted[rng.randrange(len(crafted))]
            members.append((s, len(raw), zlib.crc32(raw) & 0xFFFFFFFF)); raws.append(raw)
            continue
        else:
            raw = bytes(nrng.integers(0, 256, rng.randrange(2, 3000), dtype=np.uint8))
        co = zlib.compressobj(rng.choice([0, 1, 6, 9]), zlib.DEFLATED, -15)
        members.append((co.compress(raw) + co.flush(), len(raw), zlib.crc32(raw) & 0xFFFFFFFF)); raws.append(raw)
    offs, pos = [], 0
    for r in raws:
        pos += rng.choice([0, 3, 16, 100])
        offs.append(pos); pos += len(r)
    # vtx_bgzf_inflate copies its whole device output range back, gaps included: paint that range with 0xEE first (a call of
    # the same size reuses the engine's output buffer), so that a byte the kernel writes outside its members shows up
    paint, lens = [], [min(65536, pos + 64 - o) for o in range(0, pos + 64, 65536)]
    for n in lens:
        raw = b"\xEE" * n
        paint.append((zlib.compress(raw, 1)[2:-4], n, zlib.crc32(raw) & 0xFFFFFFFF))
    out, status = _inflate_at(eng, paint, list(range(0, pos + 64, 65536)), pos + 64)
    assert (status == 0).all() and (out == 0xEE).all()
    out, status = _inflate_at(eng, members, offs, pos + 64)
    assert (status == 0).all(), np.nonzero(status)[0][:5]
    mask = np.ones(pos + 64, bool)
    for o, r in zip(offs, raws):
        assert out[o:o + len(r)].tobytes() == r
        mask[o:o + len(r)] = False
    assert (out[mask] == 0xEE).all()                                       # nothing written between or behind members
    assert sum(1 for r in raws if len(r) == 65536) >= 1000 and sum(1 for r in raws if not r) >= 2000


def test_trailer_crc_flipped_at_every_bit(eng):
    """output lengths 0..64, 65 535 and 65 536: the right CRC gives status 0, each of the 32 single-bit flips status 7, and the
    members around a flipped one decode intact"""
    nrng = np.random.default_rng(9)
    members, raws, expect = [], [], []
    for n in list(range(65)) + [65535, 65536]:
        raw = bytes(nrng.integers(0, 256, n, dtype=np.uint8))
        comp = zlib.compress(raw, 6)[2:-4]
        crc = zlib.crc32(raw) & 0xFFFFFFFF
        for bit in [None] + list(range(32)):
            members.append((comp, n, crc if bit is None else crc ^ (1 << bit))); raws.append(raw); expect.append(0 if bit is None else 7)
    got, status = eng.bgzf_inflate(members)
    assert [int(s) for s in status] == expect
    for g, r, e in zip(got, raws, expect):
        if e == 0:
            assert g == r
    got, status = eng.bgzf_inflate(members, check_crc=False)
    assert (status == 0).all() and got == raws


def test_long_match_runs_across_batches(eng):
    """62 matches in a row after a stored block, so that two whole batches hold nothing but matches, with distances below and
    above the copy stride and lengths that are not a multiple of the distance"""
    pre = bytes(random.Random(1).randrange(256) for _ in range(600))
    toks = []
    for k in range(62):
        toks += match(3 + (k * 41) % 256, [1, 2, 3, 30, 31, 32, 33, 64, 255, 597][k % 10])
    s, out = build([("stored", pre), ("dynamic", toks)])
    assert zlib.decompress(s, -15) == out
    got, status = eng.bgzf_inflate([(s, len(out), zlib.crc32(out) & 0xFFFFFFFF)] * 64)
    assert (status == 0).all() and all(g == out for g in got)
    s2, out2 = build([("fixed", lit(b"abc") + [t for k in range(40) for t in match(31 + k, 1 + k % 33)])])
    got, status = eng.bgzf_inflate([(s2, len(out2), zlib.crc32(out2) & 0xFFFFFFFF)])
    assert status[0] == 0 and got[0] == out2
