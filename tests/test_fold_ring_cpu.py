"""The tile hand-out and per-locus slot ring of the folded kernel, rehearsed on the CPU.

vtx_k_sw_fold's warps share per-locus tables through vartrix_b200/csrc/vtx_fold_ring.cuh.  fold_ring_rehearsal.cpp
runs the same take / book / publish / wait / release functions with std::thread workers in place of warps: ring sizes
1..13, one to three "CTAs" on one cursor, 1..20 workers each, over all-1-tile shards, one huge locus, mixed depths
with tile-less loci, and tiny sparse shards.  It is built under ThreadSanitizer, which also reports any read of a slot
that the ring does not order after the slot's build."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rehearsal(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fold_ring") / "fold_ring_rehearsal")
    subprocess.run(["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-pthread", "-o", exe,
                    os.path.join(ROOT, "tests", "fold_ring_rehearsal.cpp")], check=True)
    return exe


@pytest.mark.parametrize("mode", ["ones", "huge", "mixed", "sparse"])
@pytest.mark.parametrize("seed", [1, 2])
def test_every_tile_once_and_only_its_own_tables(rehearsal, mode, seed):
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66")
    r = subprocess.run([rehearsal, mode, str(seed)], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-4000:]
    assert r.stdout.startswith("ok 65 runs"), r.stdout
