"""CPU suite: the tile-class rule (vartrix_b200/csrc/vtx_tile_class.cuh), built with g++ (tests/tile_class_shim.cpp).

vtx_k_locus_prep gives each locus the class `tile_class` returns, and run_sw launches the kernels of the classes in the
batch's launch mask.  A class that gets tiles but is left out of the mask is never launched: its pairs drop out of the
matrix without an error.  So the class is checked against the decision tree of DESIGN.md section 4, the host-batch mask
against the classes of the batch's loci, and the device-batch mask against the launch rule it keeps."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

NO_SPLIT, NO_FOLD = 2, 8                     # VTX_F_NO_SPLIT, VTX_F_NO_FOLD
FLAGS = [0, NO_SPLIT, NO_FOLD, NO_SPLIT | NO_FOLD]
GENERIC, SPLIT0, FOLD = 4, 5, 7
FAST_MAX_N = (208, 232, 256, 320)            # widest window of single-phase classes 0..3
SPLIT_MAX_N = (204, 232)                     # ... of two-phase classes 5, 6
WIDTHS = [1, 96, 192, 193, 204, 205, 208, 209, 232, 233, 256, 257, 320, 321, 1000]
LONGEST = [0, 152, 153, 256, 257, 1024]
BATCH_READS = [100, 152, 153, 256, 257, 1024]


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("tcshim") / "libtile_class_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "tile_class_shim.cpp")], check=True)
    lib = ctypes.CDLL(so)
    u32, p = ctypes.c_uint32, ctypes.c_void_p
    lib.vtx_test_tile_class.argtypes = [ctypes.c_int] * 3 + [u32] * 5
    lib.vtx_test_device_mask.argtypes = [u32] * 3
    lib.vtx_test_device_mask.restype = u32
    lib.vtx_test_host_mask.argtypes = [p, u32, p, p, p, p, u32, u32]
    lib.vtx_test_host_mask.restype = u32
    return lib


def allow(flags, max_read, max_hap):
    """(split, multi, fold): the kernel families a batch may use"""
    return (max_read <= 256 and not flags & NO_SPLIT, max_read <= 256 and max_hap > 320, not flags & (NO_SPLIT | NO_FOLD))


def design_class(exotic, prefix, fold, width, longest, flags, max_read, max_hap):
    """DESIGN.md section 4, in its own order: the narrowest single-phase class that holds the window (the multi-pass class
    beyond 320 columns, else the generic kernel); a common prefix moves it to a two-phase class; fold-shaped windows
    whose reads all fit go to the folded kernel; exotic bytes override everything."""
    split_ok, multi_ok, fold_ok = allow(flags, max_read, max_hap)
    cls = next((c for c, n in enumerate(FAST_MAX_N) if width <= n), 3 if multi_ok else GENERIC)
    if prefix and split_ok:
        cls = next((SPLIT0 + c for c, n in enumerate(SPLIT_MAX_N) if width <= n), cls)
    if fold and fold_ok and longest <= 152:
        cls = FOLD
    return GENERIC if exotic else cls


def test_tile_class_matches_design_tree(shim):
    batches = [(256, 320), (256, 321), (257, 321), (152, 1000)]
    n = 0
    for (ex, pre, fo), w, L, f, (mr, mh) in itertools.product(itertools.product((0, 1), repeat=3), WIDTHS, LONGEST, FLAGS, batches):
        want = design_class(ex, pre, fo, w, L, f, mr, mh)
        assert shim.vtx_test_tile_class(ex, pre, fo, w, L, f, mr, mh) == want, (ex, pre, fo, w, L, f, mr, mh)
        n += 1
    assert n == 8 * len(WIDTHS) * len(LONGEST) * len(FLAGS) * len(batches)


def parent_device_rule(flags, max_read, max_hap):
    """The launch rule for batches whose loci the host does not see: a single-phase or two-phase class whose narrowest
    window is wider than max_hap has no tiles; the folded kernel runs whenever it is allowed, the generic one always."""
    split_ok, _, fold_ok = allow(flags, max_read, max_hap)
    mask = 1 << GENERIC
    for c in range(4):
        if c == 0 or max_hap > FAST_MAX_N[c - 1]:
            mask |= 1 << c
    for c in range(2):
        if split_ok and (c == 0 or max_hap > SPLIT_MAX_N[c - 1]):
            mask |= 1 << (SPLIT0 + c)
    return mask | (1 << FOLD if fold_ok else 0)


def test_device_mask_keeps_launch_rule(shim):
    for f, mr, mh in itertools.product(FLAGS, [1] + BATCH_READS, WIDTHS):
        assert shim.vtx_test_device_mask(f, mr, mh) == parent_device_rule(f, mr, mh), (f, mr, mh)


def _window_pairs(rng):
    """(ref, alt) windows of every shape: fold-shaped (flanks of 96+ columns on both sides), common prefix only, nothing
    common, and windows too short to share a prefix; widths on both sides of every class limit."""
    base = lambda n: rng.choice(np.frombuffer(b"ACGT", np.uint8), n)
    out = []
    for w in WIDTHS + [97, 200, 231, 300, 400]:
        for kind in ("fold", "prefix", "none"):
            r = base(w)
            a = r.copy()
            if kind == "fold":
                mid = a[96:96 + min(w - 192, 40)]                # the allele columns (none: the windows are equal)
                mid[:] = np.where(mid == ord("A"), ord("C"), ord("A"))
                if rng.random() < 0.5 and w > 193:              # an indel: the alt window one column shorter
                    a = np.delete(a, 96)
            elif kind == "prefix":
                a[-1] = ord("A") if a[-1] != ord("A") else ord("C")
            else:
                a[0] = ord("A") if a[0] != ord("A") else ord("C")
            out.append((r, a))
    return out


def _shape(r, a):
    nr, na = len(r), len(a)
    prefix = nr >= 96 and na >= 96 and bytes(r[:96]) == bytes(a[:96])
    fold = prefix and min(nr, na) > 192 and max(nr, na) <= 232 and bytes(r[-96:]) == bytes(a[-96:])
    return prefix, fold, max(nr, na)


def _host_mask(shim, pairs, flags, max_read):
    pool, offs = bytearray(), []
    for r, a in pairs:
        for h in (r, a):
            offs.append(len(pool))
            pool += bytes(h) + b"\0" * (-len(h) % 16)
    o = np.asarray(offs, np.uint32)
    lens = np.asarray([len(h) for pa in pairs for h in pa], np.uint32)
    ro, ao, rl, al = (np.ascontiguousarray(x) for x in (o[0::2], o[1::2], lens[0::2], lens[1::2]))
    buf = np.frombuffer(bytes(pool) or b"\0", np.uint8)
    ptr = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    return shim.vtx_test_host_mask(ptr(buf), len(pairs), ptr(ro), ptr(rl), ptr(ao), ptr(al), flags, max_read)


def _tight(shim, pairs, flags, max_read):
    """{generic} and the class of every locus, with its longest read anywhere from 0 to the batch's longest read"""
    max_hap = max(max(len(r), len(a)) for r, a in pairs)
    mask = 1 << GENERIC
    for r, a in pairs:
        prefix, fold, w = _shape(r, a)
        for L in (0, max_read):
            mask |= 1 << shim.vtx_test_tile_class(0, prefix, fold, w, L, flags, max_read, max_hap)
    return mask


def test_host_mask_single_shapes(shim):
    pairs = _window_pairs(np.random.default_rng(1))
    shapes = {_shape(r, a)[:2] for r, a in pairs}
    assert shapes == {(True, True), (True, False), (False, False)}
    for (r, a), f, mr in itertools.product(pairs, FLAGS, BATCH_READS):
        assert _host_mask(shim, [(r, a)], f, mr) == _tight(shim, [(r, a)], f, mr), (len(r), len(a), _shape(r, a), f, mr)


def test_host_mask_shape_sets(shim):
    rng = np.random.default_rng(2)
    pairs = _window_pairs(rng)
    for _ in range(400):
        pick = [pairs[i] for i in rng.choice(len(pairs), int(rng.integers(1, 8)), replace=False)]
        f, mr = FLAGS[rng.integers(len(FLAGS))], BATCH_READS[rng.integers(len(BATCH_READS))]
        assert _host_mask(shim, pick, f, mr) == _tight(shim, pick, f, mr)
