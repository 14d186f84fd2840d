"""The C++ staging host (csrc/host: BGZF/BAM/BAI, .fai FASTA, VCF, filters) against the oracle's independent
pure-Python decode, on the reference's own fixtures (committed under tests/golden/ref_inputs)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_TEST_DIR, ROOT

CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
needs_ref = pytest.mark.skipif(not os.path.isdir(REF_TEST_DIR), reason="tests/golden/ref_inputs missing")


def _labels(keys):
    """equal key <=> equal label, labels numbered by first appearance"""
    _, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(np.argsort(first))
    return order[inv]


def _same_staging(sb, ob):
    for f in ("locus_row", "ref_len", "alt_len", "cand_start", "read_len", "read_cb_len", "cand_read", "ref_off",
              "alt_off", "read_off", "cb_bytes", "read_cb_off"):
        assert np.array_equal(getattr(sb, f), getattr(ob, f)), f
    for f in ("hap_bytes", "read_nib"):          # pools may differ by trailing 16-byte padding only
        a, b = getattr(sb, f), getattr(ob, f)
        n = min(len(a), len(b))
        assert np.array_equal(a[:n], b[:n]) and not a[n:].any() and not b[n:].any() and abs(len(a) - len(b)) < 16, f
    none = np.uint64(0xFFFFFFFFFFFFFFFF)
    assert np.array_equal(sb.read_umi_key == none, ob.read_umi_key == none)
    assert np.array_equal(_labels(sb.read_umi_key), _labels(ob.read_umi_key))       # same UB equivalence classes


def _dump(tmp_path, pre, bcs, *extra):
    out = tmp_path / f"{pre}.staged"
    cmd = [CLI, "-v", f"{REF_TEST_DIR}/{pre}.vcf", "-b", f"{REF_TEST_DIR}/{pre}.bam", "-f", f"{REF_TEST_DIR}/{pre}.fa",
           "-c", f"{REF_TEST_DIR}/{bcs}", "--dump-staged", str(out), *extra]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    return read_dump(str(out))


@needs_ref
@pytest.mark.parametrize("pre,bcs", [("test", "barcodes.tsv"), ("test_dna", "dna_barcodes.tsv")])
def test_cpp_staging_equals_oracle_decode(oracle, tmp_path, pre, bcs):
    n_rows, n_cols, shards = _dump(tmp_path, pre, bcs, "--shard-loci", "1000000", "--threads", "2")
    assert len(shards) == 1
    sb, met = shards[0]
    ob = oracle.stage_from_files(f"{REF_TEST_DIR}/{pre}.vcf", f"{REF_TEST_DIR}/{pre}.bam", f"{REF_TEST_DIR}/{pre}.fa")
    _same_staging(sb, ob)
    assert met == {k: ob.host_metrics[k] for k in met}
    assert n_rows == ob.n_rows and n_cols == len(oracle.load_barcodes(f"{REF_TEST_DIR}/{bcs}"))


@needs_ref
def test_cpp_staging_in_shards_and_with_filters(oracle, tmp_path):
    kw = dict(mapq=30, primary_only=True, no_duplicates=True, padding=60)
    n_rows, _, shards = _dump(tmp_path, "test_dna", "dna_barcodes.tsv", "--shard-loci", "7", "--threads", "3", "--mapq", "30",
                              "--primary-alignments", "--no-duplicates", "--padding", "60")
    assert len(shards) == (46 + 6) // 7
    for k, (sb, met) in enumerate(shards):
        ob = oracle.stage_from_files(f"{REF_TEST_DIR}/test_dna.vcf", f"{REF_TEST_DIR}/test_dna.bam", f"{REF_TEST_DIR}/test_dna.fa",
                                     rec_lo=7 * k, rec_hi=7 * k + 7, **kw)
        _same_staging(sb, ob)
        assert met == {m: ob.host_metrics[m] for m in met}, k


@needs_ref
def test_cli_refuses_to_overwrite_and_missing_inputs(tmp_path):
    (tmp_path / "out_matrix.mtx").write_text("x")
    base = [CLI, "-v", f"{REF_TEST_DIR}/test.vcf", "-b", f"{REF_TEST_DIR}/test.bam", "-f", f"{REF_TEST_DIR}/test.fa",
            "-c", f"{REF_TEST_DIR}/barcodes.tsv"]
    r = subprocess.run(base, cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 1 and "Output path already exists" in r.stderr            # main.rs:475-480
    r = subprocess.run([*base[:2], "/nonexistent.vcf", *base[3:]], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 1 and "does not exist" in r.stderr                        # main.rs:501-506


# ---- synthetic files (no reference needed: also runs on the GPU box) ------------------------------------
@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from vartrix_b200 import synth_files
    d = tmp_path_factory.mktemp("synth_files")
    return synth_files.write_dataset(str(d), n_loci=150, n_barcodes=40, depth=24, read_len=100, seed=5)


@pytest.mark.parametrize("extra,kw", [
    ([], {}),
    (["--mapq", "20", "--primary-alignments", "--no-duplicates", "--padding", "80", "--valid-chars", "ATGC"],
     dict(mapq=20, primary_only=True, no_duplicates=True, padding=80, valid_chars="ATGC")),
])
def test_cpp_staging_equals_oracle_on_synthetic_files(oracle, dataset, tmp_path, extra, kw):
    out = tmp_path / "d.staged"
    subprocess.run([CLI, "-v", dataset["vcf"], "-b", dataset["bam"], "-f", dataset["fasta"], "-c", dataset["barcodes"],
                    "--dump-staged", str(out), "--shard-loci", "1000000", "--threads", "2", *extra], check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    n_rows, n_cols, shards = read_dump(str(out))
    sb, met = shards[0]
    ob = oracle.stage_from_files(dataset["vcf"], dataset["bam"], dataset["fasta"], **kw)
    _same_staging(sb, ob)
    assert met == {k: ob.host_metrics[k] for k in met}
    assert n_rows == 150 and n_cols == 40                      # duplicate barcode line dropped (main.rs:706-709)
    assert met["num_multiallelic_recs"] > 0 and met["num_invalid_recs"] > 0 and met["num_not_useful"] > 0
    assert sb.n_cand > 1000 and (sb.read_cb_off == 0xFFFFFFFF).any()


@pytest.mark.parametrize("order", ["reversed", "shuffled_with_repeats"])
def test_cpp_staging_does_not_depend_on_vcf_order(oracle, dataset, tmp_path, order):
    """The BAM reader resumes a region scan where the previous region's scan found its first overlapping record, which
    is only valid for regions that do not move backwards: unsorted and repeated records must take the index path."""
    lines = open(dataset["vcf"]).read().splitlines()
    head = [ln for ln in lines if ln.startswith("#")]; body = [ln for ln in lines if not ln.startswith("#")]
    rng = np.random.default_rng(3)
    if order == "reversed":
        body = body[::-1]
    else:
        body = [body[i] for i in rng.permutation(len(body))] + body[:20] + body[40:20:-1]
    vcf = tmp_path / "perm.vcf"
    vcf.write_text("\n".join(head + body) + "\n")
    out = tmp_path / "perm.staged"
    subprocess.run([CLI, "-v", str(vcf), "-b", dataset["bam"], "-f", dataset["fasta"], "-c", dataset["barcodes"],
                    "--dump-staged", str(out), "--shard-loci", "37", "--threads", "3"], check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    _, _, shards = read_dump(str(out))
    for k, (sb, met) in enumerate(shards):
        ob = oracle.stage_from_files(str(vcf), dataset["bam"], dataset["fasta"], rec_lo=37 * k, rec_hi=37 * k + 37)
        _same_staging(sb, ob)
        assert met == {m: ob.host_metrics[m] for m in met}, k


def test_cpp_staging_with_dense_overlapping_loci(oracle, dataset, tmp_path):
    """Loci a few bases apart share most of their reads: the resumed scan must start at the first record that overlapped
    the previous locus, not after it."""
    lines = open(dataset["vcf"]).read().splitlines()
    head = [ln for ln in lines if ln.startswith("#")]; body = [ln for ln in lines if not ln.startswith("#")]
    dense = []
    for ln in body[:60]:
        f = ln.split("\t")
        dense.append(ln)
        if len(f[3]) == 1 and len(f[4]) == 1:
            for d in (1, 2, 30, 95):
                g = list(f); g[1] = str(int(f[1]) + d); g[3] = "A"; g[4] = "C"
                dense.append("\t".join(g))
    vcf = tmp_path / "dense.vcf"
    vcf.write_text("\n".join(head + dense) + "\n")
    out = tmp_path / "dense.staged"
    subprocess.run([CLI, "-v", str(vcf), "-b", dataset["bam"], "-f", dataset["fasta"], "-c", dataset["barcodes"],
                    "--dump-staged", str(out), "--shard-loci", "1000000", "--threads", "1"], check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    _, _, shards = read_dump(str(out))
    sb, met = shards[0]
    ob = oracle.stage_from_files(str(vcf), dataset["bam"], dataset["fasta"])
    _same_staging(sb, ob)
    assert met == {m: ob.host_metrics[m] for m in met}
    assert sb.n_cand > 1.5 * len(sb.read_len)        # reads are shared between neighbouring loci


def _spliced_dataset(tmp_path):
    from vartrix_b200.synth_files import BamWriter
    rng = np.random.default_rng(11)
    contigs = [("chrA", 400_000), ("chrB", 120_000)]
    genome = [rng.integers(0, 4, size=L, dtype=np.uint8) for _, L in contigs]
    acgt = np.frombuffer(b"ACGT", np.uint8)
    fa = tmp_path / "g.fa"
    with open(fa, "wb") as f, open(str(fa) + ".fai", "w") as fai:
        for (name, L), g in zip(contigs, genome):
            f.write(f">{name}\n".encode()); off = f.tell()
            seq = acgt[g]
            for s0 in range(0, L, 70):
                f.write(seq[s0:s0 + 70].tobytes() + b"\n")
            fai.write(f"{name}\t{L}\t{off}\t70\t71\n")
    reads = []
    for ci, (_, L) in enumerate(contigs):
        for _ in range(2500 if ci == 0 else 600):                      # short reads
            p0 = int(rng.integers(0, L - 120))
            reads.append((ci, p0, [("M", 100)], acgt[genome[ci][p0:p0 + 100]].tobytes()))
        for _ in range(160 if ci == 0 else 30):                        # spliced: 50M <1..150 kb>N 50M
            gap = int(rng.choice([900, 5000, 17000, 70000, 150000]))
            p0 = int(rng.integers(0, max(1, L - gap - 120)))
            if p0 + gap + 100 >= L:
                continue
            seq = np.concatenate([genome[ci][p0:p0 + 50], genome[ci][p0 + 50 + gap:p0 + 100 + gap]])
            reads.append((ci, p0, [("M", 50), ("N", gap), ("M", 50)], acgt[seq].tobytes()))
    reads.sort(key=lambda r: (r[0], r[1]))
    bam = tmp_path / "r.bam"
    bw = BamWriter(str(bam), contigs)
    for i, (ci, p0, cig, seq) in enumerate(reads):
        bw.add(ci, p0, 60, 0, cig, seq, f"q{i}".encode(), b"CBZ" + b"ACGTACGTACGTACGT-1\0" + b"UBZ" + b"ACGTACGTAC\0")
    bw.close()
    vcf = tmp_path / "v.vcf"
    with open(vcf, "w") as f:
        f.write("##fileformat=VCFv4.2\n" + "".join(f"##contig=<ID={n},length={L}>\n" for n, L in contigs))
        f.write("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for ci, (name, L) in enumerate(contigs):
            for p0 in np.sort(rng.integers(200, L - 200, size=220 if ci == 0 else 60)):
                ref = "ACGT"[genome[ci][p0]]
                f.write(f"{name}\t{p0 + 1}\t.\t{ref}\t{'ACGT'[(genome[ci][p0] + 1) % 4]}\t.\t.\t.\n")
    bcs = tmp_path / "b.tsv"; bcs.write_text("ACGTACGTACGTACGT-1\n")
    return vcf, bam, fa, bcs


def test_cpp_staging_with_long_spliced_records_across_index_bins(oracle, tmp_path):
    """Spliced records of up to 150 kb live in high-level BAI bins, far ahead (in file order) of the short reads around the
    loci they cover: the region iterator (chunk merging, linear-index lower bound, resumed scans) must still hand out
    exactly the records htslib would, in file order."""
    vcf, bam, fa, bcs = _spliced_dataset(tmp_path)
    for threads, shard in ((1, 1000000), (3, 41)):
        out = tmp_path / f"s{threads}.staged"
        subprocess.run([CLI, "-v", str(vcf), "-b", str(bam), "-f", str(fa), "-c", str(bcs), "--dump-staged", str(out),
                        "--shard-loci", str(shard), "--threads", str(threads)], check=True, cwd=str(tmp_path))
        from vartrix_b200.staged_io import read_dump
        _, _, shards = read_dump(str(out))
        for k, (sb, met) in enumerate(shards):
            ob = oracle.stage_from_files(str(vcf), str(bam), str(fa), rec_lo=shard * k, rec_hi=min(280, shard * k + shard))
            _same_staging(sb, ob)
            assert met == {m: ob.host_metrics[m] for m in met}, (threads, k)
        assert sum(int(m["num_not_useful"]) for _, m in shards) > 0        # spliced records that skip their locus


@pytest.mark.parametrize("shard", ["7", "1000000"])
def test_bulk_inflate_path_stages_the_same_shards(tmp_path, shard):
    """--gpu-inflate reads one compressed range per shard, walks the BGZF member headers and serves the records out of one
    bulk buffer (inflated by the device in the product; by the host decoder under --dump-staged): same staging, byte for byte."""
    outs = []
    for extra in ([], ["--gpu-inflate"]):
        out = tmp_path / f"d{len(outs)}.staged"
        subprocess.run([CLI, "-v", f"{REF_TEST_DIR}/test_dna.vcf", "-b", f"{REF_TEST_DIR}/test_dna.bam", "-f", f"{REF_TEST_DIR}/test_dna.fa",
                        "-c", f"{REF_TEST_DIR}/dna_barcodes.tsv", "--dump-staged", str(out), "--shard-loci", shard, "--threads", "2", *extra],
                       check=True, cwd=str(tmp_path))
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] and len(outs[0]) > 100_000


def test_bulk_inflate_path_reports_corruption(tmp_path):
    import shutil
    raw = bytearray(open(f"{REF_TEST_DIR}/test.bam", "rb").read())
    bsize0 = int.from_bytes(raw[16:18], "little") + 1
    for k in range(bsize0 + 40, bsize0 + 440):
        raw[k] ^= 0x5A
    bam = tmp_path / "bad.bam"
    bam.write_bytes(bytes(raw)); shutil.copy(f"{REF_TEST_DIR}/test.bam.bai", str(bam) + ".bai")
    r = subprocess.run([CLI, "-v", f"{REF_TEST_DIR}/test.vcf", "-b", str(bam), "-f", f"{REF_TEST_DIR}/test.fa", "-c", f"{REF_TEST_DIR}/barcodes.tsv",
                        "--dump-staged", str(tmp_path / "d.staged"), "--gpu-inflate"], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode != 0 and "inflate" in (r.stdout + r.stderr)


def _read_vtxd(path):
    """shards dumped by `--gpu-stage --dump-staged`: the host's share of device staging"""
    import struct
    data = open(path, "rb").read()
    p, out = 16, []
    def take():
        nonlocal p
        (nb,) = struct.unpack_from("<Q", data, p); p += 8
        b = data[p:p + nb]; p += nb
        return b
    while p < len(data):
        if data[p:p + 4] == b"VTXS":            # a shard the device path declined (several contigs): staged on the host
            p += 4
            for _ in range(15): take()
            p += 56
            out.append(None)
            continue
        assert data[p:p + 4] == b"VTXD"; p += 4
        tid = struct.unpack("<q", take())[0]
        row = np.frombuffer(take(), np.uint32); start = np.frombuffer(take(), np.int64); end = np.frombuffer(take(), np.int64)
        members = np.frombuffer(take(), np.dtype([("in_off", "<u8"), ("in_len", "<u4"), ("out_len", "<u4"), ("out_off", "<u8"), ("crc", "<u4"), ("pad", "<u4")]))
        comp = take(); entry = np.frombuffer(take(), np.uint64)
        hap = np.frombuffer(take(), np.uint8); ref_off = np.frombuffer(take(), np.uint32); ref_len = np.frombuffer(take(), np.uint32)
        alt_off = np.frombuffer(take(), np.uint32); alt_len = np.frombuffer(take(), np.uint32)
        out.append(dict(tid=tid, row=row, start=start, end=end, members=members, comp=comp, entry=entry, hap=hap, ref_off=ref_off, ref_len=ref_len,
                        alt_off=alt_off, alt_len=alt_len))
    return out


@pytest.mark.parametrize("pre,bcs,shard", [("test_dna", "dna_barcodes.tsv", "7"), ("test_dna", "dna_barcodes.tsv", "1000"), ("test", "barcodes.tsv", "1")])
def test_device_staging_host_share(tmp_path, pre, bcs, shard):
    """--gpu-stage: the host hands the device a member table, the compressed bytes and the record boundaries the index knows.
    Emulated here: the members inflate (zlib) to one stream with matching CRCs; walking the BAM records from the first entry
    hits every later entry exactly and ends on the last one; the records that overlap the loci are as many as the host stager
    fetches (its num_reads), i.e. the range is complete."""
    import struct, zlib
    base = [CLI, "-v", f"{REF_TEST_DIR}/{pre}.vcf", "-b", f"{REF_TEST_DIR}/{pre}.bam", "-f", f"{REF_TEST_DIR}/{pre}.fa", "-c", f"{REF_TEST_DIR}/{bcs}",
            "--shard-loci", shard, "--threads", "2"]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host)
    for d, (hb, hmet) in zip(dev, host):
        assert d is not None and np.array_equal(d["row"], hb.locus_row)
        stream = bytearray()
        for m in d["members"]:
            raw = zlib.decompress(d["comp"][int(m["in_off"]): int(m["in_off"]) + int(m["in_len"])], -15)
            assert len(raw) == m["out_len"] and int(m["out_off"]) == len(stream) and (zlib.crc32(raw) & 0xFFFFFFFF) == m["crc"] and m["in_off"] % 4 == 0
            stream += raw
        entry = [int(x) for x in d["entry"]]
        fetched = 0
        if entry:
            assert entry == sorted(set(entry)) and entry[-1] <= len(stream)
            p, hit, recs = entry[0], set(), []
            while p < entry[-1]:
                if p in entry: hit.add(p)
                bs = struct.unpack_from("<I", stream, p)[0]
                refid, pos, l_name, mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", stream, p + 4)
                cig = struct.unpack_from(f"<{n_cig}I", stream, p + 36 + l_name)
                rlen = 0 if flag & 4 else sum(c >> 4 for c in cig if (c & 15) in (0, 2, 3, 7, 8))
                recs.append((refid, pos, pos + (rlen if rlen > 0 else 1)))
                p += 4 + bs
            assert p == entry[-1] and hit == set(entry[:-1])
            for s0, e0 in zip(d["start"], d["end"]):
                fetched += sum(1 for (t, a, b) in recs if t == d["tid"] and a < e0 and b > s0)
        assert fetched == hmet["num_reads"]


@pytest.fixture(scope="module")
def stage_dev(tmp_path_factory):
    import ctypes
    so = str(tmp_path_factory.mktemp("stageshim") / "libstage_dev_shim.so")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, "-o", so, os.path.join(ROOT, "tests", "stage_dev_shim.cpp")], check=True)
    return ctypes.CDLL(so)


def test_shared_useful_alignment_equals_oracle_case_by_case(oracle, stage_dev):
    """Both stagers call one useful_alignment (csrc/vtx_record.cuh), so the host-versus-device comparisons cannot tell it
    from the reference.  The oracle's vtxo_useful_alignment can: the CIGAR table of test_oracle_cpu's
    test_useful_alignment_cigar_rules, plus an interior H (after an M, and in the leading section after a P), a leading N and
    an =/X block, at every locus near the read."""
    import ctypes
    code = {"M": 0, "I": 1, "D": 2, "N": 3, "S": 4, "H": 5, "P": 6, "=": 7, "X": 8}
    ua = oracle.lib().vtxo_useful_alignment
    mine = stage_dev.vtx_test_useful_alignment
    mine.restype = ctypes.c_int
    mine.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_int64]
    cigars = [[(50, "M")], [(10, "M"), (100, "N"), (10, "M")], [(10, "M"), (5, "D"), (10, "M")], [(5, "S"), (10, "M")],
              [(5, "D"), (10, "M")],
              [(10, "M"), (5, "H"), (10, "M")], [(2, "P"), (5, "H"), (10, "M")], [(5, "N"), (10, "M")], [(10, "="), (2, "X"), (10, "=")]]
    n_true = 0
    for ops in cigars:
        a = np.array([(n << 4) | code[o] for n, o in ops], np.uint32)
        for start in range(90, 240):
            for end in (start + 1, start + 3):
                want = ua(100, a.ctypes.data, len(a), start, end)
                assert mine(100, a.ctypes.data, len(a), start, end) == want, (ops, start, end)
                n_true += want
    assert n_true > 0


def _run_stage_dev(lib, stream, d, mapq, primary, nodup, umi, tag):
    import ctypes

    class StageOut(ctypes.Structure):
        _fields_ = [("n_rec", ctypes.c_uint32), ("err", ctypes.c_uint32), ("max_span", ctypes.c_uint32), ("max_read", ctypes.c_uint32),
                    ("n_cand", ctypes.c_uint64), ("metrics", ctypes.c_uint64 * 5)]
    nl = len(d["row"])
    rec_cap, cand_cap = len(stream) // 36 + 16, 1 << 22
    out = StageOut()
    sbuf = np.frombuffer(bytes(stream) + b"\0" * 8, np.uint8)
    entry = np.ascontiguousarray(d["entry"], np.uint64)
    ls, le = np.ascontiguousarray(d["start"], np.int64), np.ascontiguousarray(d["end"], np.int64)
    cand_first = np.zeros(nl + 1, np.uint32); cand_rec = np.zeros(cand_cap, np.uint32)
    read_off = np.zeros(rec_cap, np.uint64); read_len = np.zeros(rec_cap, np.uint32); cb_off = np.zeros(rec_cap, np.uint32)
    cb_len = np.zeros(rec_cap, np.uint16); umi_k = np.zeros(rec_cap, np.uint64); used = np.zeros(rec_cap, np.uint32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = lib.vtx_test_stage_dev(P(sbuf), ctypes.c_uint64(len(stream)), ctypes.c_int32(int(d["tid"])), ctypes.c_uint32(mapq), primary, nodup, umi,
                                tag.encode(), ctypes.c_uint32(len(entry)), P(entry), ctypes.c_uint32(nl), P(ls), P(le), ctypes.c_uint32(rec_cap),
                                ctypes.c_uint64(cand_cap), ctypes.byref(out), P(cand_first), P(cand_rec), P(read_off), P(read_len), P(cb_off),
                                P(cb_len), P(umi_k), P(used))
    assert rc == 0, (rc, out.err)
    return out, cand_first, cand_rec, read_off, read_len, cb_off, cb_len, umi_k, used


@pytest.mark.parametrize("pre,bcs,shard,extra", [
    ("test_dna", "dna_barcodes.tsv", "7", []), ("test_dna", "dna_barcodes.tsv", "1000", ["--mapq", "30", "--primary-alignments"]),
    ("test", "barcodes.tsv", "1", ["--umi"]), ("test", "barcodes.tsv", "1", ["--umi", "--no-duplicates", "--mapq", "4"]),
    ("test_dna", "dna_barcodes.tsv", "5", ["--bam-tag", "CB", "--mapq", "1"])])
def test_device_staging_logic_matches_host_stager(tmp_path, stage_dev, pre, bcs, shard, extra):
    """The bodies of the staging kernels (csrc/vtx_stage.cuh), run serially on the CPU over the shard the CLI hands to
    vtx_submit_bam, produce per locus exactly the candidates the host stager produces: same reads (bases, length), same cell tag
    bytes, same UMI keys, in the same order, and the same five filter counters (main.rs:831-865)."""
    _check_device_logic(tmp_path, stage_dev, f"{REF_TEST_DIR}/{pre}.vcf", f"{REF_TEST_DIR}/{pre}.bam", f"{REF_TEST_DIR}/{pre}.fa",
                        f"{REF_TEST_DIR}/{bcs}", shard, extra)


@pytest.mark.parametrize("shard,extra", [("40", []), ("13", ["--mapq", "20", "--primary-alignments", "--no-duplicates", "--padding", "80", "--umi"]),
                                         ("1000", ["--shard-bytes", "30000"])])          # shards cut by the compressed bytes of BAM they span
def test_device_staging_logic_on_synthetic_files(tmp_path, stage_dev, dataset, shard, extra):
    """... on files with multi-allelic / invalid records, reads without a cell tag, duplicates, secondary alignments"""
    n = _check_device_logic(tmp_path, stage_dev, dataset["vcf"], dataset["bam"], dataset["fasta"], dataset["barcodes"], shard, extra)
    assert n > 1000


@pytest.mark.parametrize("shard", ["41", "1000000"])
def test_device_staging_logic_with_long_spliced_records(tmp_path, stage_dev, shard):
    """... and with 150 kb spliced records in high-level index bins: the compressed range of a shard starts far ahead of its
    loci, and the per-locus window search (longest reference span) must still find them"""
    vcf, bam, fa, bcs = _spliced_dataset(tmp_path)
    n = _check_device_logic(tmp_path, stage_dev, str(vcf), str(bam), str(fa), str(bcs), shard, ["--umi"])
    assert n > 100


def _check_device_logic(tmp_path, stage_dev, vcf, bam, fa, bcs, shard, extra):
    import zlib
    from vartrix_b200.staged_io import read_dump
    base = [CLI, "-v", vcf, "-b", bam, "-f", fa, "-c", bcs, "--shard-loci", shard, "--threads", "2", *extra]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    subprocess.run([*base, "--dump-staged", str(tmp_path / "host.staged"), "--cut-at-contigs"], check=True, cwd=str(tmp_path))     # same shard boundaries
    _, _, host = read_dump(str(tmp_path / "host.staged"))
    dev = _read_vtxd(str(tmp_path / "dev.staged"))
    assert len(dev) == len(host) and all(d is not None for d in dev)          # sorted VCF: the device takes every shard
    mapq = int(extra[extra.index("--mapq") + 1]) if "--mapq" in extra else 0
    umi = 1 if "--umi" in extra else 0
    n_checked = 0
    for d, (hb, hmet) in zip(dev, host):
        if d is None:
            continue
        assert np.array_equal(d["row"], hb.locus_row)
        stream = b"".join(zlib.decompress(d["comp"][int(m["in_off"]): int(m["in_off"]) + int(m["in_len"])], -15) for m in d["members"])
        out, cand_first, cand_rec, read_off, read_len, cb_off, cb_len, umi_k, used = _run_stage_dev(
            stage_dev, stream, d, mapq, int("--primary-alignments" in extra), int("--no-duplicates" in extra), umi, "CB")
        assert [out.metrics[i] for i in range(5)] == [hmet[k] for k in ("num_reads", "num_low_mapq", "num_non_primary", "num_duplicates", "num_not_useful")]
        assert out.n_cand == len(hb.cand_read) and np.array_equal(cand_first.astype(np.uint64), hb.cand_start)
        assert out.max_read == (int(hb.read_len[hb.cand_read].max()) if len(hb.cand_read) else 0)
        sb = np.frombuffer(stream, np.uint8)
        for c in range(int(out.n_cand)):
            r, hr = int(cand_rec[c]), int(hb.cand_read[c])
            assert used[r] == 1 and read_len[r] == hb.read_len[hr]
            nb = (int(read_len[r]) + 1) // 2
            assert np.array_equal(sb[int(read_off[r]): int(read_off[r]) + nb], hb.read_nib[int(hb.read_off[hr]): int(hb.read_off[hr]) + nb])
            h_has_cb = hb.read_cb_off[hr] != 0xFFFFFFFF
            assert (cb_off[r] != 0xFFFFFFFF) == h_has_cb
            if h_has_cb:
                assert cb_len[r] == hb.read_cb_len[hr]
                assert bytes(sb[int(cb_off[r]): int(cb_off[r]) + int(cb_len[r])]) == bytes(hb.cb_bytes[int(hb.read_cb_off[hr]): int(hb.read_cb_off[hr]) + int(hb.read_cb_len[hr])])
            if umi:
                assert umi_k[r] == hb.read_umi_key[hr]
            n_checked += 1
        # records that serve several loci are one read on both sides
        assert len(set(cand_rec[:int(out.n_cand)].tolist())) == len(set(hb.cand_read.tolist()))
    assert n_checked > 0
    return n_checked


@pytest.fixture(scope="module")
def stage_fuzz(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("stagefuzz") / "stage_dev_fuzz")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.isdir(cuda_inc):
        pytest.skip("CUDA headers not found")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-I", cuda_inc, "-o", exe,
                        os.path.join(ROOT, "tests", "stage_dev_fuzz.cpp"), "-lz"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer runtime for g++ here: " + r.stderr[-200:])
    return exe


@pytest.mark.parametrize("pre,bcs,shard,extra,seed", [("test", "barcodes.tsv", "1", ["--umi"], 1), ("test_dna", "dna_barcodes.tsv", "7", [], 2)])
def test_device_staging_logic_is_memory_safe_on_damaged_input(tmp_path, stage_fuzz, pre, bcs, shard, extra, seed):
    """tests/stage_dev_fuzz.cpp under AddressSanitizer + UBSan: the staging kernels' bodies over shards whose inflated stream has
    random bytes overwritten (aimed at record heads half of the time), and the device DEFLATE decoder's bit-stream half over
    members with flipped bits: nothing is read or written outside the buffers the engine allocates, every symbol stays inside
    the member's output, and the decoder terminates."""
    dump = str(tmp_path / "dev.staged")
    subprocess.run([CLI, "-v", f"{REF_TEST_DIR}/{pre}.vcf", "-b", f"{REF_TEST_DIR}/{pre}.bam", "-f", f"{REF_TEST_DIR}/{pre}.fa", "-c", f"{REF_TEST_DIR}/{bcs}",
                    "--shard-loci", shard, "--threads", "2", "--gpu-stage", "--dump-staged", dump, *extra], check=True, cwd=str(tmp_path))
    r = subprocess.run([stage_fuzz, dump, "120", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr[-2000:]
    assert "refused" in r.stdout
