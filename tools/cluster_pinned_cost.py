"""Cost of `--known-donors`: vtx_cluster_cells_pinned against vtx_cluster_cells on the same synthetic pool matrix (10 000 cells
x 100 000 rows, 2 000 rows per cell: ~20 M entries, 16 donors with dosages 0 / 1 / 2 and 10 % ambient RNA), timed with a host
clock around the synchronous call.  K = 8 with the first 4 donors pinned and K = 32 with the first 16 pinned, R = 8, rho given
as 0.1; in each round the four calls alternate (K = 8 unpinned, pinned, K = 32 unpinned, pinned).  Each record gives the
iterations of every restart and ms per iteration of the longest restart (the restarts run in the same launches).

    python tools/cluster_pinned_cost.py --rounds 2 > out.json

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


def synthetic(n_rows, n_cols, per_cell, donors, seed, rho=0.1):
    """-> (row, col, ref, alt) sorted by (row, col), dosage uint8 [n_rows, donors]"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 3, (n_rows, donors))
    q = np.array([0.01, 0.5, 0.99])[g]
    p = (1 - rho) * q + rho * q.mean(axis=1, keepdims=True)
    donor = rng.integers(0, donors, n_cols)
    rows = np.sort(rng.integers(0, n_rows, (n_cols, per_cell)), axis=1)
    keep = np.ones_like(rows, bool)
    keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
    col = np.broadcast_to(np.arange(n_cols)[:, None], rows.shape)[keep]
    row = rows[keep]
    depth = rng.integers(1, 4, row.size)
    alt = rng.binomial(depth, p[row, donor[col]])
    o = np.lexsort((col, row))
    ent = (row[o].astype(np.uint32), col[o].astype(np.uint32), (depth - alt)[o].astype(np.uint32), alt[o].astype(np.uint32))
    return ent, g.astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--cells", type=int, default=10_000)
    ap.add_argument("--per-cell", type=int, default=2_000)
    ap.add_argument("--restarts", type=int, default=8)
    a = ap.parse_args()
    import vartrix_b200 as vb
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown"
    ent, g = synthetic(a.rows, a.cells, a.per_cell, 16, seed=1)
    out = dict(card=card, rows=a.rows, cells=a.cells, entries=int(ent[0].size), restarts=a.restarts, rho_permille=100, runs=[])
    cases = ((8, 4), (32, 16))
    with vb.Engine("coverage") as e:
        for k, J in cases:                          # warm-up: module load, allocations
            e.cluster_cells(*ent, a.rows, a.cells, k, a.restarts, seed=99)
            e.cluster_cells_pinned(*ent, a.rows, a.cells, k, g[:, :J], 100, 0.01, a.restarts, seed=99)
        for rnd in range(a.rounds):
            for k, J in cases:
                for pinned in (False, True):
                    t0 = time.perf_counter()
                    if pinned:
                        res = e.cluster_cells_pinned(*ent, a.rows, a.cells, k, g[:, :J], 100, 0.01, a.restarts, seed=rnd)
                    else:
                        res = e.cluster_cells(*ent, a.rows, a.cells, k, a.restarts, seed=rnd)
                    ms = (time.perf_counter() - t0) * 1e3
                    iters = res["restart_iters"].tolist()
                    ll = res["ll"]
                    calls = np.where(ll[:, k:].max(axis=1) - ll[:, :k].max(axis=1) >= 5 << 24, "d", "s")
                    out["runs"].append(dict(round=rnd, k=k, pinned=J if pinned else 0, ms=round(ms, 1), iters=iters,
                                            ms_per_iter=round(ms / max(iters), 2), rows_used=res["rows_used"],
                                            best_restart=res["best_restart"], doublet_over_singlet_5nats=int((calls == "d").sum())))
                    print(json.dumps(out["runs"][-1]), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
