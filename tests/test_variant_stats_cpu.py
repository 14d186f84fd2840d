"""`--out-variant-stats` without a GPU: the oracle's restatement (tests/variant_stats_oracle.py) against the unchanged C oracle
-- its column sums are the metric lines, its rows agree with the matrices --, the engine's per-locus reduction body run
serially (tests/locus_stats_shim.cpp) against a NumPy sum at the slot kernels' depth seams, and the CLI's refusals."""
import ctypes
import functools
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import baseq_oracle as B
import variant_stats_oracle as V

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR
FIXTURES = {
    "dna": (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv"),
    "rna": (f"{T}/test.vcf", f"{T}/test.bam", f"{T}/test.fa", f"{T}/barcodes.tsv"),
}
KEYS = {"plain": {}, "umi": dict(umi=True), "mates": dict(collapse_mates=True)}
FILTERED = dict(mapq=30, primary_only=True, no_duplicates=True)


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    import baseq_cases
    p = baseq_cases.write_cases(str(tmp_path_factory.mktemp("vstats")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


@pytest.fixture(scope="module")
def vcases(tmp_path_factory):
    import variant_stats_cases
    p = variant_stats_cases.write_cases(str(tmp_path_factory.mktemp("vcases")))
    return (p["vcf"], p["bam"], p["fasta"], p["barcodes"])


def _files(which, cases, vcases=None):
    return {"cases": cases, "vcases": vcases}.get(which) or FIXTURES[which]


@functools.lru_cache(maxsize=None)
def _table(files, keys, filtered):
    kw = dict(KEYS[keys], **(FILTERED if filtered else {}), min_base_quality=20 if filtered else 0)
    return V.text(files[0], V.stats(*files, **kw)), kw


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("keys", list(KEYS))
@pytest.mark.parametrize("which", ["dna", "rna", "cases", "vcases"])
def test_restatement_agrees_with_the_c_oracle(cases, vcases, which, keys, filtered):
    """Column sums = the C oracle's metric lines; coverage rows = its coverage / ref matrices; consensus rows = its 1 / 2 / 3."""
    files = _files(which, cases, vcases)
    tsv, kw = _table(files, keys, filtered)
    keyed = keys != "plain"
    for mode in ("coverage", "consensus"):
        out, ref, lines = B.expected(*files, mode, **kw)
        V.check_invariants(tsv, keyed, metric_lines=lines, mtx=dict(mode=mode, out=out, ref=ref))


def test_the_cases_file_makes_every_column_nonzero(vcases):
    """tests/variant_stats_cases.py, over the runs above: every column is nonzero in some row and every status occurs (else
    some of the checks would prove little); each record filter empties a locus of its own, so a swapped counter shows."""
    seen, statuses = set(), set()
    for keys in KEYS:
        for filtered in (False, True):
            for _, status, n in V.parse(_table(vcases, keys, filtered)[0]):
                seen |= {c for c, v in n.items() if v}
                statuses.add(status)
    assert seen == set(V.COLUMNS), set(V.COLUMNS) - seen
    assert statuses == {"scored", "multiallelic", "invalid_alt"}
    rows = {v: n for v, _, n in V.parse(_table(vcases, "umi", True)[0])}
    for variant, col in (("chrA_1000", "low_mapq"), ("chrA_1500", "non_primary"), ("chrA_2000", "duplicate"),
                         ("chrA_2500", "not_useful"), ("chrA_3000", "low_base_quality")):
        assert rows[variant]["fetched"] == rows[variant][col] > 0, (variant, col)
    assert rows["chrA_500"]["fetched"] == 0


# ---- locus_cands' per-locus filter counters on the CPU --------------------------------------------------------------------
@pytest.fixture(scope="module")
def filt_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lfshim") / "liblocus_filters_shim.so")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, "-o", so,
                    os.path.join(ROOT, "tests", "locus_filters_shim.cpp")], check=True)
    return ctypes.CDLL(so)


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("shard", ["2", "1000"])
@pytest.mark.parametrize("which", ["dna", "vcases"])
def test_device_filter_counters_per_locus(tmp_path, filt_shim, cases, vcases, which, shard, filtered):
    """locus_cands (pass 0, with the per-locus store) run serially over the shards --gpu-stage hands to vtx_submit_bam: each
    locus's fetched / low_mapq / non_primary / duplicate / not_useful / low_base_quality equal the restatement's, in that order."""
    import zlib
    from oracle import pipeline as P
    from test_host_staging_cpu import _read_vtxd
    files = _files(which, cases, vcases)
    flt = dict(FILTERED, min_base_quality=20) if filtered else {}
    args = ["--mapq", "30", "--primary-alignments", "--no-duplicates", "--min-base-quality", "20"] if filtered else []
    subprocess.run([CLI, "-v", files[0], "-b", files[1], "-f", files[2], "-c", files[3], "--shard-loci", shard, "--threads", "2",
                    *args, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    recs, bm = P.read_vcf(files[0]), P.Bam(files[1])
    n_checked, nonzero = 0, np.zeros(6, np.int64)
    for d in _read_vtxd(str(tmp_path / "dev.staged")):
        assert d is not None
        nl = len(d["row"])
        stream = b"".join(zlib.decompress(d["comp"][int(m["in_off"]): int(m["in_off"]) + int(m["in_len"])], -15) for m in d["members"])
        sbuf = np.frombuffer(stream + b"\0" * 8, np.uint8)
        entry = np.ascontiguousarray(d["entry"], np.uint64)
        ls, le = np.ascontiguousarray(d["start"], np.int64), np.ascontiguousarray(d["end"], np.int64)
        lfilt = np.full((max(nl, 1), 6), 0xDEADBEEF, np.uint32)
        Pt = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        assert filt_shim.vtx_test_locus_filters(Pt(sbuf), ctypes.c_uint64(len(stream)), ctypes.c_int32(int(d["tid"])),
                                                ctypes.c_uint32(flt.get("mapq", 0)), int(bool(flt)), int(bool(flt)),
                                                ctypes.c_uint32(flt.get("min_base_quality", 0)), ctypes.c_uint32(len(entry)), Pt(entry),
                                                ctypes.c_uint32(nl), Pt(ls), Pt(le), Pt(lfilt)) == 0
        for l, row in enumerate(d["row"].tolist()):
            want = V.locus_filters(bm, recs[row], **flt)
            assert lfilt[l].tolist() == [want[c] for c in V.FILTERS], (row, lfilt[l].tolist(), want)
            nonzero += lfilt[l] > 0
            n_checked += 1
    assert n_checked > 0
    if which == "vcases" and filtered:
        assert (nonzero > 0).all(), nonzero          # every counter, each emptying a locus of its own


# ---- the engine's reduction body on the CPU -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lsshim") / "liblocus_stats_shim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "locus_stats_shim.cpp")], check=True)
    return ctypes.CDLL(so)


NO_CELL = 0xFFFFFFFF


def _shard(depths, use_umi, with_filters, seed):
    """A shard shaped like the engine's buffers after vtx_k_umi_collapse: candidates per locus, the gate's outcome per read, and
    locus-contiguous cell / UMI slots with counts (unused slots zero, unused cells NO_CELL)."""
    rng = np.random.default_rng(seed)
    nl = len(depths)
    cand_start = np.zeros(nl + 1, np.uint64); cand_start[1:] = np.cumsum(depths)
    nc = int(cand_start[-1])
    read_col = rng.integers(-1, 40, nc).astype(np.int32)
    read_col[rng.random(nc) < 0.1] = -1
    umi = rng.integers(0, 50, nc).astype(np.uint64)
    umi[rng.random(nc) < 0.05] = np.uint64(0xFFFFFFFFFFFFFFFF)
    cand_read = rng.permutation(nc).astype(np.uint32)
    ok = (read_col[cand_read] >= 0) & ((umi[cand_read] != np.uint64(0xFFFFFFFFFFFFFFFF)) if use_umi else True)
    per = np.array([int(ok[int(cand_start[l]):int(cand_start[l + 1])].sum()) for l in range(nl)], np.int64)
    pair_start = np.zeros(nl + 1, np.uint32); pair_start[1:] = np.cumsum(per)
    npairs = int(pair_start[-1])
    ccnt = np.zeros((max(npairs, 1), 4), np.uint32)
    ucnt = np.zeros((max(npairs, 1), 4), np.uint32)
    cslot = np.full(max(npairs, 1), NO_CELL, np.uint32)
    for l in range(nl):
        ps, d = int(pair_start[l]), int(per[l])
        if d == 0:
            continue
        n_cells = int(rng.integers(1, min(d, 40) + 1))
        cslot[ps:ps + n_cells] = np.sort(rng.choice(40, n_cells, replace=False))
        # every pair calls once (or None); without use_umi those are the cell counts
        calls = rng.integers(0, 4, d)              # 0 ref, 1 alt, 2 unknown, 3 none
        slot = ps + rng.integers(0, d if use_umi else n_cells, d)        # UMI slots: any of the locus's d; cell slots: its cells
        tgt = ucnt if use_umi else ccnt
        for s_, c in zip(slot.tolist(), calls.tolist()):
            if c < 3:
                tgt[s_, c] += 1
        if use_umi:
            ccnt[ps:ps + n_cells, :3] = rng.integers(0, 3, (n_cells, 3))
    filters = rng.integers(0, 1000, (nl, 6)).astype(np.uint32) if with_filters else None
    return dict(cand_start=cand_start, cand_read=cand_read, read_col=read_col, read_umi=umi if use_umi else None,
                pair_start=pair_start if npairs else None, ucnt=ucnt if use_umi else None, ccnt=ccnt, cslot_col=cslot,
                locus_row=(np.arange(nl, dtype=np.uint32) * 3 + 7), filters=filters)


def _numpy_stats(s):
    nl = len(s["locus_row"])
    out = np.zeros((nl, 22), np.uint32)
    for l in range(nl):
        c0, c1 = int(s["cand_start"][l]), int(s["cand_start"][l + 1])
        r = s["cand_read"][c0:c1]
        col = s["read_col"][r]
        no_cb = int((col < 0).sum())
        no_umi = int(((col >= 0) & (s["read_umi"][r] == np.uint64(0xFFFFFFFFFFFFFFFF))).sum()) if s["read_umi"] is not None else 0
        ps = s["pair_start"]
        q0, q1 = (int(ps[l]), int(ps[l + 1])) if ps is not None else (0, 0)
        reads = (s["ucnt"] if s["ucnt"] is not None else s["ccnt"])[q0:q1, :3].sum(axis=0, dtype=np.int64)
        valid = s["cslot_col"][q0:q1] != NO_CELL
        cc = s["ccnt"][q0:q1][valid].astype(np.int64)
        calls = cc[:, :3].sum(axis=0)
        scored = q1 - q0
        filt = s["filters"][l] if s["filters"] is not None else np.zeros(6, np.uint32)
        out[l] = [s["locus_row"][l], *filt, no_cb, no_umi, scored, *reads, scored - reads.sum(), *calls, int(valid.sum()),
                  int(((cc[:, 0] > 0) & (cc[:, 1] == 0)).sum()), int(((cc[:, 1] > 0) & (cc[:, 0] == 0)).sum()),
                  int(((cc[:, 0] > 0) & (cc[:, 1] > 0)).sum()), int((cc[:, 2] > 1).sum())]
    return out


@pytest.mark.parametrize("use_umi", [False, True])
@pytest.mark.parametrize("depths", [[1023, 1024, 2049], [100000], [1] * 300 + [0, 5, 0], [0, 0]])
def test_reduction_body_equals_numpy(shim, depths, use_umi):
    s = _shard(depths, use_umi, with_filters=len(depths) != 1, seed=len(depths) + use_umi)
    P = lambda a: a.ctypes.data if a is not None else None
    out = np.zeros((len(depths), 22), np.uint32)
    assert shim.vtx_test_locus_stats(ctypes.c_uint32(len(depths)), *[ctypes.c_void_p(P(s[k])) for k in (
        "cand_start", "cand_read", "read_col", "read_umi", "pair_start", "ucnt", "ccnt", "cslot_col", "locus_row", "filters")],
        ctypes.c_void_p(out.ctypes.data)) == 22
    want = _numpy_stats(s)
    assert np.array_equal(out, want), np.nonzero(out != want)


def test_struct_layout_matches_the_kernel_record():
    import vartrix_b200 as vb
    from vartrix_b200 import _capi
    assert ctypes.sizeof(_capi.LocusStats) == 22 * 4 == vb.Engine.LOCUS_STATS_DTYPE.itemsize
    assert _capi.LOCUS_STATS_FIELDS[1:] == V.COLUMNS


# ---- refusals ------------------------------------------------------------------------------------------------------------
def _cli(tmp_path, *extra):
    f = FIXTURES["dna"]
    return subprocess.run([CLI, "-v", f[0], "-b", f[1], "-f", f[2], "-c", f[3], "-o", str(tmp_path / "o.mtx"), *extra],
                          cwd=str(tmp_path), capture_output=True, text=True)


def test_refused_with_dump_staged(tmp_path):
    r = _cli(tmp_path, "--dump-staged", str(tmp_path / "d.staged"), "--out-variant-stats", str(tmp_path / "s.tsv"))
    assert r.returncode == 1 and "--out-variant-stats" in r.stderr and "--dump-staged" in r.stderr
    assert os.listdir(tmp_path) == []


def test_existing_output_path_is_refused(tmp_path):
    (tmp_path / "s.tsv").write_text("keep me\n")
    r = _cli(tmp_path, "--out-variant-stats", str(tmp_path / "s.tsv"))
    assert r.returncode == 1 and "Output path already exists" in r.stderr
    assert (tmp_path / "s.tsv").read_text() == "keep me\n" and sorted(os.listdir(tmp_path)) == ["s.tsv"]


def test_help_lists_the_flag():
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert "--out-variant-stats" in r.stdout
    readme = open(os.path.join(ROOT, "README.md")).read()
    assert "--out-variant-stats" in readme
