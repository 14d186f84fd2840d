"""Cost of `--out-cluster-genotypes` / `--out-cluster-matches`: vtx_cluster_genotypes on synthetic cluster sums, timed with a
host clock around the synchronous call.

  100 000 rows (90 % reached, 60 % used), K = 8 and 32, estimated (69 fractions, or 60 at the grid's ends) and fixed, matched
  against S = 8 and 256 samples; the eight alternate inside each round.
  5 000 000 rows of which ~200 000 are reached (a donor VCF against a pool), K = 8, S = 32, estimated.
  The CLI's wall clock on the seeded 15 % ambient pool (tests/cluster_gt_cases.py) with --out-clusters, with and without the
  two flags, alternated.

    python tools/cluster_gt_cost.py --rounds 2 > out.json

The card's name and power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def synthetic(n_rows, k, s, reached, seed):
    """clusters dict, row sums, dosage [n_rows, s]: a reached row holds 0-30 molecules per cluster"""
    rng = np.random.default_rng(seed)
    hit = rng.random(n_rows) < reached
    T = np.zeros((n_rows, k), np.int64)
    T[hit] = rng.integers(0, 30, (int(hit.sum()), k)) << 16
    A = (T * rng.random((n_rows, k))).astype(np.int64)
    used = (hit & (rng.random(n_rows) < 0.67)).astype(np.uint8)
    rd = (T.sum(axis=1) >> 16).astype(np.uint64)
    ra = (A.sum(axis=1) >> 16).astype(np.uint64)
    g = rng.integers(0, 3, (n_rows, s)).astype(np.uint8)
    return dict(alt_w=A, depth_w=T, row_used=used), ra, rd, g


def timed(e, case, rho):
    cl, ra, rd, g = case
    t0 = time.perf_counter()
    res = e.cluster_genotypes(cl, ra, rd, g, 0.01, rho)
    return (time.perf_counter() - t0) * 1e3, res


def cli_runs(rounds):
    import cluster_gt_cases as GC
    d = tempfile.mkdtemp()
    p = GC.write_pool(d, 0.15)
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    runs = []
    for rnd in range(rounds + 1):                   # round 0 warms the page cache and the driver
        for flags in (False, True):
            tag = f"{rnd}_{int(flags)}"
            extra = ["--out-cluster-genotypes", f"{d}/g{tag}.vcf", "--out-cluster-matches", f"{d}/m{tag}.tsv"] if flags else []
            t0 = time.perf_counter()
            r = subprocess.run([cli, "-v", p["vcf_match"], "-b", p["bam"], "-f", p["fasta"], "-c", p["barcodes"], "-o", f"{d}/o{tag}.mtx",
                                "--umi", "--out-clusters", f"{d}/c{tag}.tsv", "--clusters", "6", *extra], capture_output=True, text=True)
            assert r.returncode == 0, r.stdout + r.stderr
            if rnd:
                runs.append(dict(round=rnd, flags=flags, s=round(time.perf_counter() - t0, 3)))
                print(json.dumps(runs[-1]), file=sys.stderr)
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", type=int, default=100_000)
    a = ap.parse_args()
    import vartrix_b200 as vb
    import cluster_gt_oracle as O
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown"
    cases = {(k, s): synthetic(a.rows, k, s, 0.9, seed=k + s) for k in (8, 32) for s in (8, 256)}
    out = dict(card=card, rows=a.rows, runs=[])
    with vb.Engine("coverage") as e:
        for c in cases.values():                    # warm-up: module load, allocations
            timed(e, c, 100)
        for rnd in range(a.rounds):
            for (k, s), c in cases.items():
                for rho in (None, 150):
                    ms, res = timed(e, c, rho)
                    out["runs"].append(dict(round=rnd, k=k, s=s, mode="estimate" if rho is None else "fixed", ms=round(ms, 1),
                                            evaluated=len(res["grid_permille"]), touched=int(res["touched"].size),
                                            compared=res["rows_compared"], rho_permille=res["rho_permille"]))
                    print(json.dumps(out["runs"][-1]), file=sys.stderr)
        big = synthetic(5_000_000, 8, 32, 0.04, seed=3)
        timed(e, big, 100)
        for rnd in range(a.rounds):
            ms, res = timed(e, big, None)
            out["runs"].append(dict(round=rnd, k=8, s=32, rows=5_000_000, mode="estimate", ms=round(ms, 1), evaluated=len(res["grid_permille"]),
                                    touched=int(res["touched"].size), compared=res["rows_compared"], rho_permille=res["rho_permille"]))
            print(json.dumps(out["runs"][-1]), file=sys.stderr)
        # the engine equals the restatement on one of the timed cases
        cl, ra, rd, g = cases[(8, 256)]
        _, got = timed(e, cases[(8, 256)], None)
    t0 = time.perf_counter()
    want = O.genotypes(cl, ra, rd, g, 0.01, None)
    out["restatement"] = dict(rows=a.rows, k=8, s=256, s_cpu=round(time.perf_counter() - t0, 2),
                              engine_equal=bool(all(np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64))
                                                    for f in ("grid_objective", "gt", "pl", "match_ll", "match_discordant"))))
    out["cli"] = cli_runs(a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
