"""`--collapse-mates` without a GPU: the oracle's semantics on the reference's paired-end DNA fixture, the host stager's QNAME
keys (`--dump-staged`), the device interning pass run serially on the CPU (tests/name_key_shim.cpp), and the refusals."""
import ctypes
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT
import mates_oracle as M
from test_host_staging_cpu import _labels, _read_vtxd, _same_staging

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR
DNA = (f"{T}/test_dna.vcf", f"{T}/test_dna.bam", f"{T}/test_dna.fa", f"{T}/dna_barcodes.tsv")


@pytest.fixture(scope="module")
def paired(tmp_path_factory):
    import mates_cases
    return mates_cases.write_paired(str(tmp_path_factory.mktemp("paired")))


def _cand_table(oracle, batch, bcs, vcf, bam):
    """per candidate: locus index, column (-1: no listed cell), QNAME"""
    recs, bm = M.fetched_records(batch, vcf, bam)
    index = {k: i for i, k in enumerate(bcs.keys)}
    col_of_read = np.array([-1 if o == oracle.NO_CB else index.get(bytes(batch.cb_bytes[o:o + n]), -1)
                            for o, n in zip(batch.read_cb_off.tolist(), batch.read_cb_len.tolist())], np.int64)
    locus = np.repeat(np.arange(batch.n_loci), np.diff(batch.cand_start.astype(np.int64)))
    names = [M.qname(bm, int(r)) for r in recs]
    return locus, col_of_read[batch.cand_read], names


def test_oracle_collapses_only_cells_that_hold_one_template_twice(oracle):
    """Against the golden coverage matrices (the reference's counts): the collapsed matrices differ exactly where a
    (locus, cell) holds two records of one template, and every such cell's counts are recomputed here from the fetched
    records: calls from the oracle's scores, grouped by QNAME, the 0.75 rule in integers (4a >= 3t)."""
    n_rows, n_cols, res, batch, bcs = M.run_files(*DNA, "coverage", collapse_mates=True)
    alt_gold, ref_gold = oracle.read_mtx(f"{T}/test_dna.mtx")[2], oracle.read_mtx(f"{T}/test_dna_ref.mtx")[2]
    got = {(int(r), int(c)): (int(a), int(f), int(u)) for r, c, a, f, u in zip(res.row, res.col, res.alt_cnt, res.ref_cnt, res.unk_cnt)}
    locus, col, names = _cand_table(oracle, batch, bcs, DNA[0], DNA[1])
    ref_s, alt_s = oracle.score_pairs(batch, batch.cand_read, locus)
    L = oracle.lib()
    calls = np.array([L.vtxo_evaluate_scores(int(r), int(a)) for r, a in zip(ref_s, alt_s)])     # 0 None, 1 REF, 2 ALT, -1 UNKNOWN
    groups = {}
    for c in range(len(names)):
        if col[c] >= 0:
            groups.setdefault((int(batch.locus_row[locus[c]]), int(col[c])), []).append(c)
    twice = set()
    for key, cs in groups.items():
        nm = [names[c] for c in cs if names[c] != b"*"]
        if len(nm) != len(set(nm)):
            twice.add(key)
    changed = {k for k in set(alt_gold) | set(ref_gold) | set(got)
               if (alt_gold.get(k, 0.0), ref_gold.get(k, 0.0)) != (float(got.get(k, (0, 0, 0))[0]), float(got.get(k, (0, 0, 0))[1]))}
    assert changed and changed <= twice, changed - twice
    assert alt_gold[(3, 1325)] == 4 and got[(3, 1325)][0] == 2
    for key in twice:
        frags = {}
        for c in groups[key]:
            if calls[c] != 0:                                     # None calls are dropped
                frags.setdefault(names[c] if names[c] != b"*" else ("*", c), []).append(int(calls[c]))
        a = r = u = 0
        for fc in frags.values():
            t, na, nr = len(fc), fc.count(2), fc.count(1)
            if 4 * na >= 3 * t: a += 1
            elif 4 * nr >= 3 * t: r += 1
            else: u += 1
        assert got.get(key, (0, 0, 0)) == (a, r, u), key
    # without the flag the oracle still reproduces the goldens, and the flag drops no read
    _, _, res0, _, _ = M.run_files(*DNA, "coverage")
    assert {(int(r), int(c)): float(v) for r, c, v in zip(res0.row, res0.col, res0.val)} == alt_gold
    assert res.metrics == dict(res0.metrics, num_non_umi=0) and res.metrics["num_non_umi"] == 0


def test_oracle_default_is_the_plain_oracle(oracle):
    a, b = M.stage_from_files(*DNA[:3]), oracle.stage_from_files(*DNA[:3])
    for f in oracle.Batch.FIELDS:
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


@pytest.mark.parametrize("shard,threads,extra", [("1000000", "1", []), ("7", "3", []), ("5", "2", ["--gpu-inflate"]),
                                                 ("3", "2", ["--mapq", "30", "--primary-alignments", "--no-duplicates"])])
def test_dump_staged_carries_name_keys(oracle, tmp_path, shard, threads, extra):
    """--dump-staged --collapse-mates on the DNA fixture: inside each shard (and so inside each locus) two reads have equal
    keys exactly when their QNAMEs are equal; everything else is staged as without the flag."""
    from vartrix_b200.staged_io import read_dump
    kw = dict(mapq=30, primary_only=True, no_duplicates=True) if "--mapq" in extra else {}
    out = tmp_path / "d.staged"
    subprocess.run([CLI, "-v", DNA[0], "-b", DNA[1], "-f", DNA[2], "-c", DNA[3], "--dump-staged", str(out), "--shard-loci", shard,
                    "--threads", threads, "--collapse-mates", *extra], check=True, cwd=str(tmp_path))
    _, _, shards = read_dump(str(out))
    n = int(shard)
    n_twice = 0
    for k, (sb, met) in enumerate(shards):
        ob = M.stage_from_files(*DNA[:3], collapse_mates=True, rec_lo=n * k, rec_hi=n * k + n, **kw)
        _same_staging(sb, ob)
        assert met == {m: ob.host_metrics[m] for m in met}
        assert (sb.read_umi_key != np.uint64(oracle.NO_UMI)).all()
        recs, bm = M.fetched_records(ob, DNA[0], DNA[1], **kw)
        for l in range(sb.n_loci):                       # per locus, straight from the decoded names
            c0, c1 = int(sb.cand_start[l]), int(sb.cand_start[l + 1])
            nm = [M.qname(bm, int(r)) for r in recs[c0:c1]]
            assert np.array_equal(_labels(sb.read_umi_key[sb.cand_read[c0:c1]]), _labels(M.name_keys(nm))), (k, l)
            n_twice += len(nm) - len(set(nm))
    assert n_twice > 0 or "--mapq" in extra


def test_dump_staged_on_paired_file(oracle, paired, tmp_path):
    from vartrix_b200.staged_io import read_dump
    out = tmp_path / "p.staged"
    subprocess.run([CLI, "-v", paired["vcf"], "-b", paired["bam"], "-f", paired["fasta"], "-c", paired["barcodes"], "--dump-staged", str(out),
                    "--shard-loci", "2", "--threads", "2", "--collapse-mates"], check=True, cwd=str(tmp_path))
    _, _, shards = read_dump(str(out))
    for k, (sb, _) in enumerate(shards):
        _same_staging(sb, M.stage_from_files(paired["vcf"], paired["bam"], paired["fasta"], collapse_mates=True, rec_lo=2 * k, rec_hi=2 * k + 2))


# ---- the device interning pass on the CPU ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def name_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nameshim") / "libname_key_shim.so")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, "-o", so, os.path.join(ROOT, "tests", "name_key_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def _records(stream: bytes, p: int, end: int):
    """offsets of the records of `stream` from p to end, and their QNAMEs"""
    offs, names = [], []
    while p < end:
        bs = struct.unpack_from("<I", stream, p)[0]
        l_rn = stream[p + 12]
        offs.append(p); names.append(bytes(stream[p + 36: p + 36 + l_rn - 1]))
        p += 4 + bs
    return np.asarray(offs, np.uint64), names


def _check_partition(lib, stream: bytes, offs, names, seed):
    """the constant hash probes O(n^2) slots: it runs on the first 3 000 records"""
    rng = np.random.default_rng(seed)
    used0 = (rng.random(len(offs)) < 0.85).astype(np.uint32)
    sbuf = np.frombuffer(stream, np.uint8)
    for const_hash in (0, 1):
        n = min(len(offs), 3000) if const_hash else len(offs)
        used = np.ascontiguousarray(used0[:n])
        want = _labels(M.name_keys([nm for nm, u in zip(names[:n], used) if u]))
        for order in (np.arange(n), np.arange(n)[::-1], rng.permutation(n)):
            order = np.ascontiguousarray(order, np.uint32)
            keys = np.zeros(n, np.uint64)
            P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
            assert lib.vtx_test_name_keys(P(sbuf), ctypes.c_uint64(len(stream)), ctypes.c_uint32(n), P(offs), P(used), P(order),
                                          const_hash, P(keys)) == 0
            assert (keys[used == 0] == np.uint64(0xFFFFFFFFFFFFFFFF)).all()
            k = keys[used == 1]
            assert (k < np.uint64(n)).all()
            assert np.array_equal(_labels(k), want), (const_hash, order[:5])


@pytest.mark.parametrize("shard", ["7", "1000"])
def test_device_name_keys_on_the_shards_the_cli_hands_over(tmp_path, name_shim, shard):
    """The records of every `--gpu-stage --dump-staged --collapse-mates` shard: the interning body gives equal keys exactly to
    equal names, with the kernel's hash and with every name in one probe chain, whichever record claims its slot first."""
    out = tmp_path / "dev.staged"
    subprocess.run([CLI, "-v", DNA[0], "-b", DNA[1], "-f", DNA[2], "-c", DNA[3], "--dump-staged", str(out), "--shard-loci", shard,
                    "--threads", "2", "--gpu-stage", "--collapse-mates"], check=True, cwd=str(tmp_path))
    n_dup = 0
    for k, d in enumerate(_read_vtxd(str(out))):
        stream = b"".join(zlib.decompress(d["comp"][int(m["in_off"]): int(m["in_off"]) + int(m["in_len"])], -15) for m in d["members"])
        if not len(d["entry"]):
            continue
        offs, names = _records(stream, int(d["entry"][0]), int(d["entry"][-1]))
        _check_partition(name_shim, stream + b"\0" * 8, offs, names, k)
        n_dup += len(names) - len(set(names))
    assert n_dup > 0


def test_device_name_keys_on_awkward_names(tmp_path, name_shim, paired):
    """prefixes (r1 / r10 / r100), equal lengths that differ in the last byte, 254-byte names, several "*" records"""
    from oracle import pipeline as P
    import mates_cases
    bm = P.Bam(paired["bam"])
    names = [M.qname(bm, i) for i in range(len(bm))]
    for want in (b"r1", b"r10", b"r100", b"tmplA1", b"tmplA2", mates_cases.LONG + b"a", mates_cases.LONG + b"b"):
        assert want in names
    assert sum(len(nm) == 254 for nm in names) >= 6 and names.count(b"*") >= 5
    _check_partition(name_shim, bm.data + b"\0" * 8, np.asarray(bm.rec_off - 4, np.uint64), names, 1)


def test_cli_refuses_umi_with_collapse_mates(tmp_path):
    out = tmp_path / "o.mtx"
    r = subprocess.run([CLI, "-v", DNA[0], "-b", DNA[1], "-f", DNA[2], "-c", DNA[3], "-o", str(out), "--umi", "--collapse-mates"],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 1 and "--collapse-mates" in r.stderr and "--umi" in r.stderr
    assert os.listdir(tmp_path) == []
    r = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert "--collapse-mates" in r.stdout


def test_engine_and_oracle_refuse_umi_with_collapse_mates():
    import vartrix_b200 as vb
    with pytest.raises(ValueError):
        vb.Engine("coverage", umi=True, collapse_mates=True)
    with pytest.raises(ValueError):
        M.run_files(*DNA, "coverage", umi=True, collapse_mates=True)
