"""Cost of `--out-cluster-calls`: vtx_cluster_refine on a synthetic pool, timed with a host clock around the synchronous call.

  10 000 cells x 100 000 rows x ~19.8 M entries (§5g / §5h's cost shape), K = 8 and 32 donors, each cell a singlet of one
  donor (5 % doublets) with 1-3 molecules per entry; the clusters dict holds each donor's hard sums over 60 % of its singlets.
  The CLI cap of 8 rounds after round 0.  Two rounds, the two K alternating inside each.
  The NumPy restatement's CPU time on 1 000 cells x 10 000 rows at K = 8, with the engine's result compared to it.
  The CLI's wall clock on the seeded 15 % ambient pool (tests/cluster_gt_cases.py) with --out-clusters, with and without the
  flag, alternated.

    python tools/cluster_refine_cost.py --rounds 2 > out.json

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


def synthetic(n_rows, n_cols, per_cell, k, seed):
    """-> (row, col, ref, alt) sorted by (row, col), clusters dict"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, k)).astype(np.int8)
    donor = rng.integers(0, k, n_cols)
    other = (donor + 1 + rng.integers(0, k - 1, n_cols)) % k
    dbl = rng.random(n_cols) < 0.05
    col = np.repeat(np.arange(n_cols, dtype=np.int64), per_cell)
    row = rng.integers(0, n_rows, col.size)
    key = np.unique(row * n_cols + col)                      # sorted by (row, col), one entry per pair
    row, col = key // n_cols, key % n_cols
    q = np.array([0.01, 0.5, 0.99])
    qq = q[g[row, donor[col]]]
    qq = np.where(dbl[col], (qq + q[g[row, other[col]]]) / 2, qq)
    depth = rng.integers(1, 4, row.size)
    alt = rng.binomial(depth, 0.9 * qq + 0.05)
    ref = depth - alt
    lab = np.where(~dbl & (rng.random(n_cols) < 0.6), donor, -1)
    hit = lab[col] >= 0
    idx = row[hit] * k + lab[col[hit]]
    A = np.bincount(idx, weights=alt[hit].astype(np.float64), minlength=n_rows * k).astype(np.int64).reshape(n_rows, k) << 16
    T = np.bincount(idx, weights=depth[hit].astype(np.float64), minlength=n_rows * k).astype(np.int64).reshape(n_rows, k) << 16
    with_r = np.bincount(row[ref > 0], minlength=n_rows)
    with_a = np.bincount(row[alt > 0], minlength=n_rows)
    used = ((with_r >= 4) & (with_a >= 4)).astype(np.uint8)
    return (row.astype(np.uint32), col.astype(np.uint32), ref.astype(np.uint32), alt.astype(np.uint32)), dict(alt_w=A, depth_w=T, row_used=used)


def cli_runs(rounds):
    import cluster_gt_cases as GC
    d = tempfile.mkdtemp()
    p = GC.write_pool(d, 0.15)
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    runs = []
    for rnd in range(rounds + 1):                   # round 0 warms the page cache and the driver
        for flag in (False, True):
            tag = f"{rnd}_{int(flag)}"
            extra = ["--out-cluster-calls", f"{d}/x{tag}.tsv"] if flag else []
            t0 = time.perf_counter()
            r = subprocess.run([cli, "-v", p["vcf"], "-b", p["bam"], "-f", p["fasta"], "-c", p["barcodes"], "-o", f"{d}/o{tag}.mtx",
                                "--umi", "--out-clusters", f"{d}/c{tag}.tsv", "--clusters", "6", *extra], capture_output=True, text=True)
            assert r.returncode == 0, r.stdout + r.stderr
            if rnd:
                runs.append(dict(round=rnd, flag=flag, s=round(time.perf_counter() - t0, 3)))
                print(json.dumps(runs[-1]), file=sys.stderr)
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    import vartrix_b200 as vb
    import cluster_refine_oracle as O
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown"
    n_rows, n_cols = 100_000, 10_000
    cases = {k: synthetic(n_rows, n_cols, 2000, k, seed=k) for k in (8, 32)}
    out = dict(card=card, rows=n_rows, cells=n_cols, entries={k: int(c[0][0].size) for k, c in cases.items()}, runs=[])
    with vb.Engine("coverage") as e:
        for k, (ent, cl) in cases.items():          # warm-up: module load, allocations
            e.cluster_refine(*ent, n_rows, n_cols, cl, 0.01, 0)
        for rnd in range(a.rounds):
            for k, (ent, cl) in cases.items():
                t0 = time.perf_counter()
                res = e.cluster_refine(*ent, n_rows, n_cols, cl, 0.01, 8)
                ms = (time.perf_counter() - t0) * 1e3
                out["runs"].append(dict(round=rnd, k=k, ms=round(ms, 1), rounds=res["n_rounds"], ms_per_round=round(ms / res["n_rounds"], 1),
                                        converged=res["converged"], rho_permille=res["rho_permille"].tolist(),
                                        rows_scored=res["rows_scored"].tolist(), calls=res["calls"][-1].tolist()))
                print(json.dumps(out["runs"][-1]), file=sys.stderr)
        ent, cl = synthetic(10_000, 1_000, 200, 8, seed=5)
        got = e.cluster_refine(*ent, 10_000, 1_000, cl, 0.01, 8)
    t0 = time.perf_counter()
    want = O.refine(*ent, 10_000, 1_000, cl, 0.01, 8)
    out["restatement"] = dict(rows=10_000, cells=1_000, entries=int(ent[0].size), k=8, rounds=want["n_rounds"],
                              s_cpu=round(time.perf_counter() - t0, 2),
                              engine_equal=bool(all(np.array_equal(np.asarray(got[f]).astype(np.int64), np.asarray(want[f]).astype(np.int64))
                                                    for f in ("ll", "counts", "label", "rho_permille", "calls", "gt", "pl"))))
    out["cli"] = cli_runs(a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
