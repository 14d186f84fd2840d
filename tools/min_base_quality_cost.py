"""Cost of `--min-base-quality` through the whole CLI (files -> .mtx): a 5 M-read synthetic set with binned qualities, with and
without the flag, under host staging and under --gpu-stage, the four variants alternated inside each round.

    python tools/min_base_quality_cost.py --rounds 2 > out.json

Wall clock of the whole process (CUDA context start included).  The card's name and power limit are read in the same call."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loci", type=int, default=100_000)
    ap.add_argument("--depth", type=int, default=50)
    ap.add_argument("--barcodes", type=int, default=50_000)
    ap.add_argument("--floor", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--host-threads", type=int, default=16)
    a = ap.parse_args()
    from vartrix_b200 import synth_files
    d = tempfile.mkdtemp(prefix="vtx_bq_cost_")
    ds = synth_files.write_dataset_fast(d, n_loci=a.loci, n_barcodes=a.barcodes, depth=a.depth, read_len=150, seed=2, quals="binned")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except FileNotFoundError:
        card = "no nvidia-smi"
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    variants = [("host", ["--threads", str(a.host_threads)], []), ("host", ["--threads", str(a.host_threads)], ["--min-base-quality", str(a.floor)]),
                ("gpu-stage", ["--gpu-stage", "--threads", "4"], []), ("gpu-stage", ["--gpu-stage", "--threads", "4"], ["--min-base-quality", str(a.floor)])]
    runs = []
    for rnd in range(a.rounds):
        for stage, args, flag in variants:
            out = os.path.join(d, "o.mtx")
            for p in (out, os.path.join(d, "ref_matrix.mtx")):
                if os.path.exists(p):
                    os.remove(p)
            cmd = [cli, "-v", ds["vcf"], "-b", ds["bam"], "-f", ds["fasta"], "-c", ds["barcodes"], "-o", out, "-s", "consensus",
                   "--log-level", "info", *args, *flag]
            t0 = time.time()
            p = subprocess.run(cmd, capture_output=True, text=True, cwd=d)
            wall = time.time() - t0
            grab = lambda pat: (lambda m: int(m.group(1)) if m else None)(re.search(pat, p.stderr))
            runs.append(dict(round=rnd, stage=stage, flag=" ".join(flag) or "-", rc=p.returncode, wall_s=round(wall, 3),
                             reads=grab(r"alignments evaluated: (\d+)"), low_base_quality=grab(r"low base quality at the variant: (\d+)"),
                             pairs_scored=grab(r"pairs scored on the GPU: (\d+)"),
                             mtx_sha1=hashlib.sha1(open(out, "rb").read()).hexdigest()[:12] if os.path.exists(out) else None,
                             **({"stderr_tail": p.stderr[-600:]} if p.returncode else {})))
            print(json.dumps(runs[-1]), file=sys.stderr)
    print(json.dumps(dict(what="--min-base-quality cost, whole CLI runs", card=card, loci=a.loci, depth=a.depth, barcodes=a.barcodes,
                          quals="binned", reads_in_bam=ds.get("n_reads"), floor=a.floor, runs=runs), indent=1))
    shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
