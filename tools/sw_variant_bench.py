"""Kernel-tuning aid: time the device-resident hot path with alternative builds of the library (VTX_LIB).
    python tools/sw_variant_bench.py --loci 30000 [--depth 50] build/variants/lib_*.so
One shard is generated once; every build runs in its own process on the same data."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(npz, steps):
    import torch
    import vartrix_b200 as vb
    z = np.load(npz, allow_pickle=True)
    sb = vb.StagedBatch(n_rows=int(z["n_rows"]), **{f: z[f] for f in vb.StagedBatch.FIELDS})
    bcs = vb.Barcodes([bytes(k) for k in z["keys"]])
    stream = torch.cuda.Stream()
    eng = vb.Engine(str(z["mode"]), umi=bool(z["umi"]), stream=stream.cuda_stream, no_split=bool(os.environ.get("VTX_NO_SPLIT")), no_fold=bool(os.environ.get("VTX_NO_FOLD")))
    eng.set_barcodes(bcs)
    dev = {}
    db = sb.to_c()
    for f in vb.StagedBatch.FIELDS:
        a = getattr(sb, f)
        t = torch.from_numpy(a.view(np.uint8).reshape(-1) if a.dtype.itemsize > 1 else a.reshape(-1)).cuda()
        dev[f] = t
        setattr(db, f, t.data_ptr() if t.numel() else None)
    mr, mh = int(sb.read_len.max()), int(max(sb.ref_len.max(), sb.alt_len.max()))
    for _ in range(3):
        eng.submit_device(db, mr, mh); eng.finish_device()
    sw, tot = [], []
    for _ in range(steps):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        eng.submit_device(db, mr, mh); r = eng.finish_device()
        tot.append((time.perf_counter() - t0) * 1e3)
        sw.append(eng.timing()["sw_ms"])
    n = int(r.metrics.num_scored)
    print(json.dumps(dict(lib=os.environ.get("VTX_LIB", "default"), no_split=bool(os.environ.get("VTX_NO_SPLIT")), no_fold=bool(os.environ.get("VTX_NO_FOLD")), pairs=n, sw_ms=float(np.median(sw)), step_ms=float(np.median(tot)),
                          mpairs_s_kernel=n / np.median(sw) / 1e3, checksum=int(r.n))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--loci", type=int, default=30000)
    ap.add_argument("--kind", default="snv")
    ap.add_argument("--depth", type=int, default=50, help="reads per locus (4: one fold tile per locus)")
    ap.add_argument("--umi", action="store_true")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--child", default="")
    a = ap.parse_args()
    if a.child:
        return child(a.child, a.steps)
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(a.loci, 5000, depth=a.depth, seed=1, kind=a.kind, umi=a.umi)
    npz = "/tmp/vtx_variant_shard.npz"
    np.savez(npz, n_rows=sb.n_rows, keys=np.array([np.frombuffer(k, np.uint8) for k in bcs.keys]), mode="coverage", umi=a.umi,
             **{f: getattr(sb, f) for f in vb.StagedBatch.FIELDS})
    for lib in (a.libs or [""]):
        env = dict(os.environ)
        if lib:
            env["VTX_LIB"] = os.path.abspath(lib)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--child", npz, "--steps", str(a.steps)], env=env, check=False)


if __name__ == "__main__":
    main()
