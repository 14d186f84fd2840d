import json
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
# the reference's own regression inputs and golden matrices (vartrix's test/ directory, committed verbatim as test data)
REF_TEST_DIR = os.path.join(GOLDEN, "ref_inputs")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    # the engine library, the CLI and the oracle are built in-tree; build them if a fresh checkout has none
    import subprocess
    need = [os.path.join(ROOT, "vartrix_b200", "lib", "libvartrix_b200.so"), os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200"),
            os.path.join(ROOT, "oracle", "libvtx_oracle.so")]
    if not all(os.path.exists(p) for p in need):
        subprocess.run(["make", "-s", "-C", ROOT, "all"], check=True)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


HAS_GPU = _has_gpu()


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import pipeline
    pipeline.lib()          # builds libvtx_oracle.so on first use
    return pipeline


@pytest.fixture(scope="session")
def goldens():
    with open(os.path.join(GOLDEN, "goldens.json")) as fh:
        return json.load(fh)


@pytest.fixture(scope="session")
def golden_batches(oracle):
    return {n: oracle.Batch.load(os.path.join(GOLDEN, n)) for n in ("rna_batch.npz", "dna_batch.npz")}


def triplet_dict(row, col, val):
    d = {}
    for r, c, v in zip(row, col, val):
        d[(int(r), int(c))] = d.get((int(r), int(c)), 0.0) + float(v)
    return d


def same_entries(a: dict, b: dict) -> bool:
    if a.keys() != b.keys():
        return False
    return all((math.isnan(a[k]) and math.isnan(b[k])) or a[k] == b[k] for k in a)


def golden_dict(g):
    return {(int(r), int(c)): float(v) for r, c, v in g["entries"]}


def assert_same_triplets(got, exp):
    """Bit-exact comparison of two triplet sets incl. order (row-major) -- got/exp expose row,col,val,val2,*_cnt."""
    for f in ("row", "col", "ref_cnt", "alt_cnt", "unk_cnt"):
        a, b = np.asarray(getattr(got, f)), np.asarray(getattr(exp, f))
        assert a.shape == b.shape, (f, a.shape, b.shape)
        assert np.array_equal(a, b), f
    for f in ("val", "val2"):
        a, b = np.asarray(getattr(got, f)), np.asarray(getattr(exp, f))
        assert np.array_equal(a, b, equal_nan=True), f


def to_oracle_batch(oracle, sb):
    return oracle.Batch(**{f: getattr(sb, f) for f in oracle.Batch.FIELDS}, n_rows=sb.n_rows).normalized()


def to_staged(ob):
    import vartrix_b200 as vb
    return vb.StagedBatch.from_fields(ob)
