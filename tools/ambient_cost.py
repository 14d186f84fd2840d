"""Cost of `--ambient-rna`: vtx_donors_ambient on a synthetic pool matrix (10 000 cells x 100 000 rows, 2 000 rows per cell:
~20 M entries, 15 % ambient molecules), timed with a host clock around the synchronous call, at D = 8 and D = 32, in the
estimate mode (69 fractions, or 60 when the winner is below 0.010) and the fixed mode (one); the four alternate inside each
round.  Each record gives the call's time, the fractions evaluated and the time per fraction.  Then the NumPy restatement
(tests/ambient_oracle.py) on a smaller matrix, on the CPU, for scale, and whether the engine equals it there.

    python tools/ambient_cost.py --rounds 2 > out.json

The card's name and power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def synthetic(n_rows, n_cols, per_cell, d, rho, seed):
    """-> (row, col, ref, alt) sorted by (row, col), dosage [n_rows, d]; cells of one donor, one in ten a doublet"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, d)).astype(np.uint8)
    d1 = rng.integers(0, d, n_cols)
    d2 = np.where(rng.random(n_cols) < 0.1, rng.integers(0, d, n_cols), d1)
    pool = g.mean(axis=1) / 2
    rows = np.sort(rng.integers(0, n_rows, (n_cols, per_cell)), axis=1)
    keep = np.ones_like(rows, bool)
    keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
    col = np.broadcast_to(np.arange(n_cols)[:, None], rows.shape)[keep]
    row = rows[keep]
    p = (1 - rho) * (g[row, d1[col]] + g[row, d2[col]]) / 4 + rho * pool[row]
    depth = rng.integers(1, 4, row.size)
    alt = rng.binomial(depth, p * 0.98 + 0.01)
    o = np.lexsort((col, row))
    return (row[o].astype(np.uint32), col[o].astype(np.uint32), (depth - alt)[o].astype(np.uint32), alt[o].astype(np.uint32)), g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--cells", type=int, default=10_000)
    ap.add_argument("--per-cell", type=int, default=2_000)
    ap.add_argument("--oracle-rows", type=int, default=10_000)
    ap.add_argument("--oracle-cells", type=int, default=1_000)
    ap.add_argument("--oracle-per-cell", type=int, default=200)
    a = ap.parse_args()
    import vartrix_b200 as vb
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown"
    mats = {d: synthetic(a.rows, a.cells, a.per_cell, d, 0.15, seed=d) for d in (8, 32)}
    out = dict(card=card, rows=a.rows, cells=a.cells, entries=int(mats[8][0][0].size), runs=[])
    with vb.Engine("coverage") as e:
        for d in (8, 32):                                          # warm-up: module load, allocations
            e.donors_ambient(*mats[d][0], a.rows, a.cells, mats[d][1], 0.01, 100)
        for rnd in range(a.rounds):
            for d in (8, 32):
                for rho in (None, 150):
                    t0 = time.perf_counter()
                    res = e.donors_ambient(*mats[d][0], a.rows, a.cells, mats[d][1], 0.01, rho)
                    ms = (time.perf_counter() - t0) * 1e3
                    ne = len(res["grid_permille"])
                    out["runs"].append(dict(round=rnd, d=d, mode="estimate" if rho is None else "fixed", ms=round(ms, 1), evaluated=ne,
                                            ms_per_fraction=round(ms / (ne + (rho is None)), 2), rho_permille=res["rho_permille"]))
                    print(json.dumps(out["runs"][-1]), file=sys.stderr)
    import ambient_oracle as O
    s, g = synthetic(a.oracle_rows, a.oracle_cells, a.oracle_per_cell, 8, 0.15, seed=2)
    t0 = time.perf_counter()
    res = O.ambient(*s, a.oracle_rows, a.oracle_cells, g, 0.01, None)
    out["restatement"] = dict(rows=a.oracle_rows, cells=a.oracle_cells, entries=int(s[0].size), d=8, s=round(time.perf_counter() - t0, 2),
                              rho_permille=res["rho_permille"])
    with vb.Engine("coverage") as e:
        t0 = time.perf_counter()
        got = e.donors_ambient(*s, a.oracle_rows, a.oracle_cells, g, 0.01, None)
        out["restatement"]["engine_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["restatement"]["engine_equal"] = bool(np.array_equal(got["ll"], res["ll"]) and
                                              np.array_equal(got["grid_objective"], res["grid_objective"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
