"""Cost of `--out-clusters`: vtx_cluster_cells on a synthetic pool matrix (10 000 cells x 100 000 rows, 2 000 rows per cell:
~20 M entries, 8 true groups), timed with a host clock around the synchronous call, at K = 8 and K = 32 with R = 8; the two K
alternate inside each round.  Each record gives the iterations of every restart and ms per iteration (the restarts run in the
same launches, so an iteration is one E-step and one M-step over the restarts still active).  Then the NumPy restatement
(tests/cluster_oracle.py) on a smaller matrix, on the CPU, for scale.

    python tools/cluster_cost.py --rounds 2 > out.json

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


def synthetic(n_rows, n_cols, per_cell, groups, seed):
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.02, 0.98, (n_rows, groups))
    group = rng.integers(0, groups, n_cols)
    rows = np.sort(rng.integers(0, n_rows, (n_cols, per_cell)), axis=1)
    keep = np.ones_like(rows, bool)
    keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
    col = np.broadcast_to(np.arange(n_cols)[:, None], rows.shape)[keep]
    row = rows[keep]
    depth = rng.integers(1, 4, row.size)
    alt = rng.binomial(depth, p[row, group[col]])
    o = np.lexsort((col, row))
    return (row[o].astype(np.uint32), col[o].astype(np.uint32), (depth - alt)[o].astype(np.uint32), alt[o].astype(np.uint32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--cells", type=int, default=10_000)
    ap.add_argument("--per-cell", type=int, default=2_000)
    ap.add_argument("--restarts", type=int, default=8)
    ap.add_argument("--oracle-rows", type=int, default=10_000)
    ap.add_argument("--oracle-cells", type=int, default=1_000)
    ap.add_argument("--oracle-per-cell", type=int, default=200)
    a = ap.parse_args()
    import vartrix_b200 as vb
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown"
    m = synthetic(a.rows, a.cells, a.per_cell, 8, seed=1)
    out = dict(card=card, rows=a.rows, cells=a.cells, entries=int(m[0].size), restarts=a.restarts, runs=[])
    with vb.Engine("coverage") as e:
        e.cluster_cells(*m, a.rows, a.cells, 8, a.restarts, seed=99)          # warm-up: module load, allocations
        for rnd in range(a.rounds):
            for k in (8, 32):
                t0 = time.perf_counter()
                res = e.cluster_cells(*m, a.rows, a.cells, k, a.restarts, seed=rnd)
                ms = (time.perf_counter() - t0) * 1e3
                its = res["restart_iters"].tolist()
                out["runs"].append(dict(round=rnd, k=k, ms=round(ms, 1), iters=its, ms_per_iter=round(ms / max(its), 2),
                                        best_restart=res["best_restart"], rows_used=res["rows_used"]))
                print(json.dumps(out["runs"][-1]), file=sys.stderr)
    import cluster_oracle as O
    s = synthetic(a.oracle_rows, a.oracle_cells, a.oracle_per_cell, 8, seed=2)
    t0 = time.perf_counter()
    res = O.cluster(*s, a.oracle_rows, a.oracle_cells, 8, a.restarts, seed=0)
    out["restatement"] = dict(rows=a.oracle_rows, cells=a.oracle_cells, entries=int(s[0].size), k=8, restarts=a.restarts,
                              s=round(time.perf_counter() - t0, 2), iters=res["restart_iters"].tolist())
    with vb.Engine("coverage") as e:
        t0 = time.perf_counter()
        got = e.cluster_cells(*s, a.oracle_rows, a.oracle_cells, 8, a.restarts, seed=0)
        out["restatement"]["engine_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["restatement"]["engine_equal"] = bool(np.array_equal(got["ll"], res["ll"]) and np.array_equal(got["alt_w"], res["alt_w"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
