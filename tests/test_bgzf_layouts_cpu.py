"""CPU suite: the BAM front end on one record stream written in many BGZF layouts (tests/bgzf_layouts.py) -- records cut across
members at every field, members of a few bytes, empty members, index offsets of the form (k, ISIZE_k), members from other
compressors.  The oracle (oracle/pipeline.Bam: the whole file inflated with zlib, records fetched by brute force without the
index) does not depend on the layout; the host stager (plain and --gpu-inflate), the --gpu-stage host share and the staging
kernels' bodies must not either."""
import os
import subprocess

import pytest

from bgzf_layouts import CUT_FIELDS, LAYOUTS, dataset, shard_range, write_layout
from test_host_staging_cpu import CLI, _check_device_logic, _read_vtxd, _same_staging, stage_dev  # noqa: F401

SHARD = "9"          # small shards: their compressed ranges begin and end inside split records
FILTERS = ["--mapq", "30", "--primary-alignments", "--no-duplicates"]
COUNTERS = ("num_reads", "num_low_mapq", "num_non_primary", "num_duplicates", "num_not_useful")


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return dataset(str(tmp_path_factory.mktemp("layouts")))


@pytest.fixture(scope="module")
def layout_bams(data, tmp_path_factory):
    d = tmp_path_factory.mktemp("layout_bams")
    out = {}
    for lay in LAYOUTS:
        path = str(d / f"{lay}.bam")
        out[lay] = (path, write_layout(path, data["refs"], data["recs"], lay, seed=LAYOUTS.index(lay) + 1))
    return out


def test_whole_layout_is_byte_identical_to_bamwriter(data, layout_bams, tmp_path):
    from vartrix_b200.synth_files import BamWriter
    bw = BamWriter(str(tmp_path / "bw.bam"), data["refs"])
    for args in data["adds"]:
        bw.add(*args)
    bw.close()
    path, _ = layout_bams["whole"]
    assert open(path, "rb").read() == open(tmp_path / "bw.bam", "rb").read()
    assert open(path + ".bai", "rb").read() == open(str(tmp_path / "bw.bam") + ".bai", "rb").read()


def test_every_layout_reaches_its_seams(layout_bams):
    facts = {lay: f for lay, (_, f) in layout_bams.items()}
    assert facts["whole"]["crossing"] == 0
    for lay in ("fill", "cut_at", "tiny", "empty", "isize_voff", "codecs"):
        assert facts[lay]["crossing"] >= (facts[lay]["n_members"] - 2 if lay == "fill" else 50), lay
    assert {f for _, f in facts["cut_at"]["split"]} == set(CUT_FIELDS)          # every field has a record cut inside it
    assert facts["tiny"]["n_members"] > 10 * facts["tiny"]["n_records"]
    assert facts["empty"]["n_empty"] > 20 and facts["empty"]["empty_offsets"] > 0
    assert facts["isize_voff"]["isize_offsets"] > 20
    assert facts["codecs"]["long_codes"] > 100                 # hand-written members decode symbols through 15-bit codes


def test_oracle_reads_the_same_records_from_every_layout(oracle, layout_bams):
    ref = oracle.Bam(layout_bams["whole"][0])
    for lay, (path, _) in layout_bams.items():
        assert oracle.Bam(path).data == ref.data, lay


def _dump(tmp_path, data, bam, tag, *extra):
    out = tmp_path / f"{tag}.staged"
    subprocess.run([CLI, "-v", data["vcf"], "-b", bam, "-f", data["fasta"], "-c", data["barcodes"], "--dump-staged", str(out),
                    "--shard-loci", SHARD, "--threads", "3", "--umi", *extra], check=True, cwd=str(tmp_path))
    from vartrix_b200.staged_io import read_dump
    return read_dump(str(out))


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_host_staging_equals_oracle(oracle, data, layout_bams, tmp_path, layout, filtered):
    bam = layout_bams[layout][0]
    kw = dict(mapq=30, primary_only=True, no_duplicates=True) if filtered else {}
    shards = {}
    for tag, extra in (("plain", []), ("gpu_inflate", ["--gpu-inflate"])):
        _, _, shards[tag] = _dump(tmp_path, data, bam, tag, *extra, *(FILTERS if filtered else []))
        n = int(SHARD)
        for k, (sb, met) in enumerate(shards[tag]):
            ob = oracle.stage_from_files(data["vcf"], bam, data["fasta"], rec_lo=n * k, rec_hi=n * k + n, **kw)
            _same_staging(sb, ob)
            assert met == {m: ob.host_metrics[m] for m in met}, (tag, k)
    total = {c: sum(int(m[c]) for _, m in shards["plain"]) for c in COUNTERS}
    assert total["num_reads"] > 2000 and total["num_not_useful"] > 0
    if filtered:
        assert all(v > 0 for v in total.values()), total            # every filter rejects records in this file
    else:
        assert total["num_low_mapq"] == total["num_non_primary"] == total["num_duplicates"] == 0


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_device_staging_host_share_and_kernel_bodies(tmp_path, stage_dev, data, layout_bams, layout, filtered):
    """--gpu-stage: the members of every shard inflate to one stream whose entry points are record boundaries, and the staging
    kernels' bodies, run on the CPU over that stream, produce the host stager's candidates and counters"""
    import struct
    import zlib
    bam, facts = layout_bams[layout]
    base = [CLI, "-v", data["vcf"], "-b", bam, "-f", data["fasta"], "-c", data["barcodes"], "--shard-loci", SHARD, "--threads", "2"]
    subprocess.run([*base, "--dump-staged", str(tmp_path / "dev0.staged"), "--gpu-stage"], check=True, cwd=str(tmp_path))
    dev = _read_vtxd(str(tmp_path / "dev0.staged"))
    assert dev and all(d is not None for d in dev)
    for d in dev:
        # exactly the members the index names for these loci: no member of the range missing, none beyond it
        want = shard_range(facts, int(d["tid"]), [int(x) for x in d["start"]], [int(x) for x in d["end"]])
        assert [int(m["out_len"]) for m in d["members"]] == [facts["mem_len"][k] for k in want]
        stream = b"".join(zlib.decompress(d["comp"][int(m["in_off"]): int(m["in_off"]) + int(m["in_len"])], -15) for m in d["members"])
        entry = [int(x) for x in d["entry"]]
        if not entry:
            continue
        p, hit = entry[0], set()
        while p < entry[-1]:
            hit.add(p)
            p += 4 + struct.unpack_from("<I", stream, p)[0]
        assert p == entry[-1] and set(entry[:-1]) <= hit
    # the kernels' bodies with the record filters on compare their five counters with the host stager's, shard by shard
    n = _check_device_logic(tmp_path, stage_dev, data["vcf"], bam, data["fasta"], data["barcodes"], SHARD, ["--umi", *(FILTERS if filtered else [])])
    assert n > 1000


@pytest.mark.parametrize("layout", LAYOUTS)
def test_device_staging_under_address_sanitizer(tmp_path, data, layout_bams, layout):
    from conftest import ROOT
    exe = str(tmp_path / "stage_dev_fuzz")
    cuda_inc = "/usr/local/cuda/include"
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-I", cuda_inc, "-o", exe,
                        os.path.join(ROOT, "tests", "stage_dev_fuzz.cpp"), "-lz"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer runtime for g++ here: " + r.stderr[-200:])
    dump = str(tmp_path / "dev.staged")
    subprocess.run([CLI, "-v", data["vcf"], "-b", layout_bams[layout][0], "-f", data["fasta"], "-c", data["barcodes"], "--shard-loci", SHARD,
                    "--threads", "2", "--gpu-stage", "--umi", "--dump-staged", dump], check=True, cwd=str(tmp_path))
    r = subprocess.run([exe, dump, "20", "4"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr[-2000:]
