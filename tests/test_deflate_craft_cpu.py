"""CPU suite: the project's two DEFLATE decoders on hand-written streams (tests/deflate_craft.py) that zlib's compressor never
writes -- batch, input-window and table seams of the device decoder, and streams with one flaw each.  zlib is the reference:
what it decodes, both decoders decode to the same bytes; what it refuses, both refuse.  The same corpus then runs under
AddressSanitizer, and on the GPU through the kernel (test_gpu_inflate_seams.py)."""
import os
import struct
import subprocess

import pytest

from conftest import ROOT
from deflate_craft import corpus, too_long
from test_inflate_cpu import inflater  # noqa: F401  (fixture: host decoder and the device decoder's bit-stream half)


@pytest.fixture(scope="module")
def cases():
    return corpus()


def test_corpus_reaches_every_seam(cases):
    by = {n: (s, o, f) for n, s, o, f in cases}
    starts = [f["header_at"] for _, _, _, f in cases if "header_at" in f]
    assert set(starts) == set(range(960, 1089)) | set(range(1984, 2113))
    for n, s, o, f in cases:
        if "header_at" in f:                       # the stored lead-in ends where the dynamic header is meant to start
            assert 5 + struct.unpack_from("<H", s, 1)[0] == f["header_at"]
            assert (s[f["header_at"]] >> 1) & 3 == 2          # BTYPE of the next block: dynamic
    assert any(f.get("match_batch31") for _, _, _, f in cases)                         # a batch of 31 matches
    assert by["codes15_both_alphabets"][2]["long_codes"]
    assert sum(1 for _, _, o, _ in cases if o is None) >= 12
    assert len(by["fixed_blocks_2000"][1]) == 2000 and len(by["stored65535_align0"][1]) == 65535
    for n in (0, 1, 2, 3, 4, 255, 256, 257, 65535):       # the stored payload at every input offset mod 4
        for a in range(4):
            s, o, _ = by[f"stored{n}_align{a}"]
            at = [p for p in range(5, min(24, len(s) + 1)) if struct.unpack_from("<HH", s, p - 4) == (n, n ^ 0xFFFF) and s[p:p + n] == o[:n]]
            assert at and at[-1] % 4 == a, (n, a)
    assert all(len(o) <= 65536 for _, _, o, _ in cases if o is not None)          # every stream fits one BGZF member


def test_crafted_streams_decode_like_zlib(inflater, cases):
    for name, s, out, _ in cases:
        ok, got = inflater(s, len(out) if out is not None else 4096)
        if out is None:
            assert not ok, name
        else:
            assert ok and got == out, name


def test_output_longer_than_isize_is_refused(inflater, cases):
    for name, s, n in too_long(cases):
        assert not inflater(s, n)[0], name


def test_crafted_streams_under_address_sanitizer(tmp_path, cases):
    exe = str(tmp_path / "inflate_asan")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-I", cuda_inc,
                        "-o", exe, os.path.join(ROOT, "tests", "inflate_asan_main.cpp")], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer runtime for g++ here: " + r.stderr[-200:])
    blob = bytearray()
    for _, s, out, _ in cases:
        blob += struct.pack("<III", len(s), len(out) if out is not None else 4096, int(out is not None)) + s + (out or b"")
    for _, s, n in too_long(cases)[::7]:
        blob += struct.pack("<III", len(s), n, 0) + s
    (tmp_path / "corpus.bin").write_bytes(bytes(blob))
    r = subprocess.run([exe, str(tmp_path / "corpus.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "disagreements 0" in r.stdout
