"""The reference's own regression suite (vartrix src/main.rs:1207-1466) through the product CLI on the GPU:
the seven argv of `mod tests`, the reference's input files (tests/golden/ref_inputs = vartrix's test/ directory verbatim)
and its twelve golden comparisons, compared the way the reference compares them -- as CSR matrices, i.e. as
(row, col) -> value sets (main.rs:1230-1232).  BASELINE.json configs[0] is `test_coverage_matrices`."""
import gzip
import os
import subprocess

import pytest

from conftest import REF_TEST_DIR, ROOT

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
T = REF_TEST_DIR


def read_mtx(path):
    """-> (n_rows, n_cols, {(row, col): value}) like sprs::io::read_matrix_market + to_csr (duplicates summed)."""
    with open(path) as fh:
        lines = [ln for ln in fh.read().split("\n") if ln and not ln.startswith("%")]
    nr, nc, nnz = (int(x) for x in lines[0].split())
    ent = {}
    for ln in lines[1:]:
        r, c, v = ln.split()
        ent[(int(r), int(c))] = ent.get((int(r), int(c)), 0.0) + float(v)
    assert len(lines) - 1 == nnz
    return nr, nc, ent


RNA = ["-v", f"{T}/test.vcf", "-b", f"{T}/test.bam", "-f", f"{T}/test.fa"]
DNA = ["-v", f"{T}/test_dna.vcf", "-b", f"{T}/test_dna.bam", "-f", f"{T}/test_dna.fa", "-c", f"{T}/dna_barcodes.tsv"]
# (test name in main.rs, argv after the output flags, golden for -o, golden for --ref-matrix)
CASES = [
    ("test_consensus_matrix", RNA + ["-c", f"{T}/barcodes.tsv"], "test_consensus.mtx", None),
    ("test_frac_matrix", RNA + ["-c", f"{T}/barcodes.tsv", "-s", "alt_frac"], "test_frac.mtx", None),
    ("test_coverage_matrices", RNA + ["-c", f"{T}/barcodes.tsv", "-s", "coverage"], "test_coverage.mtx", "test_coverage_ref.mtx"),
    ("test_coverage_matrices_umi", RNA + ["-c", f"{T}/barcodes.tsv", "--umi", "-s", "coverage"], "test_coverage_umi.mtx", "test_coverage_ref_umi.mtx"),
    ("test_coverage_matrices_umi_gzipped_bcs", RNA + ["-c", f"{T}/barcodes.tsv.gz", "--umi", "-s", "coverage"], "test_coverage_umi.mtx", "test_coverage_ref_umi.mtx"),
    ("test_coverage_matrices_umi_dna", DNA + ["--umi", "-s", "coverage"], "test_dna_umi.mtx", "test_dna_ref_umi.mtx"),
    ("test_coverage_matrices_dna", DNA + ["-s", "coverage"], "test_dna.mtx", "test_dna_ref.mtx"),
]


@pytest.mark.parametrize("name,argv,gold_out,gold_ref", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("threads", [1, 3])
def test_reference_regression_case(tmp_path, name, argv, gold_out, gold_ref, threads):
    out, ref, bco = str(tmp_path / "result.mtx"), str(tmp_path / "result_ref.mtx"), str(tmp_path / "bcs.tsv")
    cmd = [CLI, *argv, "-o", out, "--threads", str(threads)]
    if gold_ref:
        cmd += ["--ref-matrix", ref]
    if "gzipped" in name:
        cmd += ["--out-barcodes", bco]
    r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert read_mtx(out) == read_mtx(f"{T}/{gold_out}")
    if gold_ref:
        assert read_mtx(ref) == read_mtx(f"{T}/{gold_ref}")
    if "gzipped" in name:                                   # main.rs:1377-1389: barcode file round trip
        want = gzip.open(f"{T}/barcodes.tsv.gz", "rt").read().split()
        assert open(bco).read().split() == want


@pytest.mark.parametrize("name,argv,gold_out,gold_ref", [CASES[2], CASES[6]], ids=[CASES[2][0], CASES[6][0]])
def test_reference_regression_case_with_device_inflate(tmp_path, name, argv, gold_out, gold_ref):
    """The same goldens with --gpu-inflate: every BGZF member the loci need is inflated (and CRC-checked) on the GPU."""
    out, ref = str(tmp_path / "result.mtx"), str(tmp_path / "result_ref.mtx")
    r = subprocess.run([CLI, *argv, "-o", out, "--ref-matrix", ref, "--threads", "2", "--shard-loci", "9", "--gpu-inflate", "--log-level", "info"],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert read_mtx(out) == read_mtx(f"{T}/{gold_out}") and read_mtx(ref) == read_mtx(f"{T}/{gold_ref}")
    assert "BGZF blocks" in r.stderr


@pytest.mark.parametrize("name,argv,gold_out,gold_ref", [CASES[2], CASES[3], CASES[5], CASES[6]], ids=[CASES[i][0] for i in (2, 3, 5, 6)])
def test_reference_regression_case_with_device_staging(tmp_path, name, argv, gold_out, gold_ref):
    """The same goldens with --gpu-stage: the host reads compressed ranges and the index; the BAM is decoded on the GPU."""
    out, ref = str(tmp_path / "result.mtx"), str(tmp_path / "result_ref.mtx")
    r = subprocess.run([CLI, *argv, "-o", out, "--ref-matrix", ref, "--threads", "2", "--shard-loci", "9", "--gpu-stage", "--log-level", "info"],
                       cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert read_mtx(out) == read_mtx(f"{T}/{gold_out}") and read_mtx(ref) == read_mtx(f"{T}/{gold_ref}")
    assert "staged on the host after the device declined" not in r.stderr
