"""Cost of `--out-donors`: (1) inside the engine: one config-3-shaped synthetic shard (95 000 loci, 50 000 barcodes, depth 50:
~4.75 M candidates, resident on the device), submitted with and without vtx_set_donors at D = 2, 8 and 32; vtx_last_timing's
post_ms (UMI collapse, the donor kernels, finalize, emit), sw_ms and launch count, the with / without runs alternated inside
each round; (2) through the whole CLI (files -> .mtx [+ .tsv]): a 5 M-read synthetic set with and without the flag, under host
staging and under --gpu-stage, alternated the same way.

    python tools/donor_cost.py --rounds 2 > out.json

The card's name and power limit are read in the same call."""
import argparse
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def engine_runs(a):
    import vartrix_b200 as vb
    sb, bcs, _ = vb.synth.make_shard(a.engine_loci, a.barcodes, depth=a.depth, seed=5, umi=True)
    rng = np.random.default_rng(3)
    out = []
    for rnd in range(a.rounds):
        for d in (2, 8, 32):
            for on in (False, True):
                with vb.Engine("coverage", umi=True) as e:
                    e.set_barcodes(bcs)
                    if on:
                        e.set_donors(rng.integers(0, 3, (sb.n_rows, d)).astype(np.uint8), 0.01)
                    e.submit(sb); e.finish()                  # warm-up: allocations, module load
                    e.submit(sb); e.finish()
                    t = e.timing()
                    slots = int(e.donor_ll()[1][:, 0].sum()) if on else 0
                out.append(dict(round=rnd, donors=d if on else 0, candidates=sb.n_cand, pairs=t["n_pairs"], post_ms=round(t["post_ms"], 4),
                                sw_ms=round(t["sw_ms"], 3), prep_ms=round(t["prep_ms"], 3), launches=t["total_launches"], donor_slots=slots))
                print(json.dumps(out[-1]), file=sys.stderr)
    return out


def cli_runs(a):
    from vartrix_b200 import synth_files
    d = tempfile.mkdtemp(prefix="vtx_donor_cost_")
    ds = synth_files.write_dataset_fast(d, n_loci=a.loci, n_barcodes=a.barcodes, depth=a.depth, read_len=150, seed=2)
    # the synthetic VCF has no sample columns: append eight seeded GT columns
    rng = np.random.default_rng(4)
    lines = open(ds["vcf"]).read().split("\n")
    with open(ds["vcf"], "w") as f:
        for ln in lines:
            if not ln:
                continue
            if ln.startswith("#CHROM"):
                ln = "\t".join(ln.split("\t")[:8] + ["FORMAT"] + [f"S{k}" for k in range(8)])
            elif not ln.startswith("#"):
                ln = "\t".join(ln.split("\t")[:8] + ["GT"] + [("0/0", "0/1", "1/1")[g] for g in rng.integers(0, 3, 8)])
            f.write(ln + "\n")
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    tsv = os.path.join(d, "donors.tsv")
    variants = [("host", ["--threads", str(a.host_threads)], []), ("host", ["--threads", str(a.host_threads)], ["--out-donors", tsv]),
                ("gpu-stage", ["--gpu-stage", "--threads", "4"], []), ("gpu-stage", ["--gpu-stage", "--threads", "4"], ["--out-donors", tsv])]
    runs = []
    for rnd in range(a.rounds):
        for stage, args, flag in variants:
            out = os.path.join(d, "o.mtx")
            for p in (out, os.path.join(d, "ref_matrix.mtx"), tsv):
                if os.path.exists(p):
                    os.remove(p)
            cmd = [cli, "-v", ds["vcf"], "-b", ds["bam"], "-f", ds["fasta"], "-c", ds["barcodes"], "-o", out, "-s", "consensus",
                   "--log-level", "info", *args, *flag]
            t0 = time.time()
            p = subprocess.run(cmd, capture_output=True, text=True, cwd=d)
            wall = time.time() - t0
            grab = lambda pat, f=float: (lambda m: f(m.group(1)) if m else None)(re.search(pat, p.stderr))
            runs.append(dict(round=rnd, stage=stage, flag="--out-donors" if flag else "-", rc=p.returncode, wall_s=round(wall, 3),
                             pairs_scored=grab(r"pairs scored on the GPU: (\d+)", int), post_ms=grab(r"post ([0-9.]+) \("),
                             sw_ms=grab(r"Smith-Waterman ([0-9.]+),"), launches=grab(r"pairs, (\d+) launches", int),
                             mtx_sha1=hashlib.sha1(open(out, "rb").read()).hexdigest()[:12] if os.path.exists(out) else None,
                             donor_line=(re.search(r"Donors: .*", p.stderr) or [None])[0] if flag else None,
                             **({"stderr_tail": p.stderr[-600:]} if p.returncode else {})))
            print(json.dumps(runs[-1]), file=sys.stderr)
    shutil.rmtree(d, ignore_errors=True)
    return runs, ds.get("n_reads")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loci", type=int, default=100_000)
    ap.add_argument("--engine-loci", type=int, default=95_000)
    ap.add_argument("--depth", type=int, default=50)
    ap.add_argument("--barcodes", type=int, default=50_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--host-threads", type=int, default=16)
    ap.add_argument("--skip-cli", action="store_true")
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except FileNotFoundError:
        card = "no nvidia-smi"
    eng = engine_runs(a)
    runs, n_reads = ([], None) if a.skip_cli else cli_runs(a)
    print(json.dumps(dict(what="--out-donors cost: the engine's post phase and whole CLI runs", card=card, engine_loci=a.engine_loci,
                          depth=a.depth, barcodes=a.barcodes, engine_runs=eng, loci=a.loci, reads_in_bam=n_reads, cli_runs=runs), indent=1))


if __name__ == "__main__":
    main()
