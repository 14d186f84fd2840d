"""Cost of `--out-variant-stats`: (1) through the whole CLI (files -> .mtx + .tsv): a 5 M-read synthetic set with and without
the flag, under host staging and under --gpu-stage, the four variants alternated inside each round; (2) inside the engine:
one synthetic shard submitted with and without vtx_set_locus_stats, vtx_last_timing's post_ms (UMI collapse, the per-locus
reduction, finalize, emit) and launch count, alternated the same way.

    python tools/variant_stats_cost.py --rounds 2 > out.json

CLI: wall clock of the whole process (CUDA context start included).  The card's name and power limit are read in the same call."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def engine_runs(a, rounds):
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(a.engine_loci, 50_000, depth=a.depth, seed=5, umi=True)
    out = []
    for rnd in range(rounds):
        for umi in (False, True):
            for on in (False, True):
                with vb.Engine("consensus", umi=umi, locus_stats=on) as e:
                    e.set_barcodes(bcs)
                    e.submit(sb); e.finish()                  # warm-up: allocations, module load
                    e.submit(sb); e.finish()
                    t = e.timing()
                    n = len(e.locus_stats()) if on else 0
                out.append(dict(round=rnd, umi=umi, locus_stats=on, candidates=sb.n_cand, pairs=t["n_pairs"], post_ms=round(t["post_ms"], 4),
                                sw_ms=round(t["sw_ms"], 3), launches=t["total_launches"], entries=n))
                print(json.dumps(out[-1]), file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loci", type=int, default=100_000)
    ap.add_argument("--engine-loci", type=int, default=95_000)
    ap.add_argument("--depth", type=int, default=50)
    ap.add_argument("--barcodes", type=int, default=50_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--host-threads", type=int, default=16)
    a = ap.parse_args()
    from vartrix_b200 import synth_files
    d = tempfile.mkdtemp(prefix="vtx_vs_cost_")
    ds = synth_files.write_dataset_fast(d, n_loci=a.loci, n_barcodes=a.barcodes, depth=a.depth, read_len=150, seed=2)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except FileNotFoundError:
        card = "no nvidia-smi"
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    stats = os.path.join(d, "stats.tsv")
    variants = [("host", ["--threads", str(a.host_threads)], []), ("host", ["--threads", str(a.host_threads)], ["--out-variant-stats", stats]),
                ("gpu-stage", ["--gpu-stage", "--threads", "4"], []), ("gpu-stage", ["--gpu-stage", "--threads", "4"], ["--out-variant-stats", stats])]
    runs = []
    for rnd in range(a.rounds):
        for stage, args, flag in variants:
            out = os.path.join(d, "o.mtx")
            for p in (out, os.path.join(d, "ref_matrix.mtx"), stats):
                if os.path.exists(p):
                    os.remove(p)
            cmd = [cli, "-v", ds["vcf"], "-b", ds["bam"], "-f", ds["fasta"], "-c", ds["barcodes"], "-o", out, "-s", "consensus",
                   "--log-level", "info", *args, *flag]
            t0 = time.time()
            p = subprocess.run(cmd, capture_output=True, text=True, cwd=d)
            wall = time.time() - t0
            grab = lambda pat, f=float: (lambda m: f(m.group(1)) if m else None)(re.search(pat, p.stderr))
            runs.append(dict(round=rnd, stage=stage, flag="--out-variant-stats" if flag else "-", rc=p.returncode, wall_s=round(wall, 3),
                             pairs_scored=grab(r"pairs scored on the GPU: (\d+)", int), post_ms=grab(r"post ([0-9.]+) \("),
                             launches=grab(r"pairs, (\d+) launches", int),
                             mtx_sha1=hashlib.sha1(open(out, "rb").read()).hexdigest()[:12] if os.path.exists(out) else None,
                             stats_sha1=hashlib.sha1(open(stats, "rb").read()).hexdigest()[:12] if flag and os.path.exists(stats) else None,
                             **({"stderr_tail": p.stderr[-600:]} if p.returncode else {})))
            print(json.dumps(runs[-1]), file=sys.stderr)
    shutil.rmtree(d, ignore_errors=True)
    eng = engine_runs(a, a.rounds)
    print(json.dumps(dict(what="--out-variant-stats cost: whole CLI runs and the engine's post phase", card=card, loci=a.loci, depth=a.depth,
                          barcodes=a.barcodes, reads_in_bam=ds.get("n_reads"), cli_runs=runs, engine_loci=a.engine_loci, engine_runs=eng), indent=1))


if __name__ == "__main__":
    main()
