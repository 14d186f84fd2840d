"""2-GPU test of the engine's own NCCL allgatherv (vtx_comm_init / vtx_gather / vtx_fetch).  Needs >= 2 CUDA
devices (run on a machine with two GPUs); skipped elsewhere.  The host-side protocol is covered on CPU by
tests/test_dist_gloo.py."""
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch
    import torch.distributed as dist
    import vartrix_b200 as vb
    from vartrix_b200 import dist as vdist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    base = dict(n_loci=300, n_barcodes=80, depth=40, seed=2, kind="indel", umi=True)
    cfg = vdist.rank_workload(base, rank)
    sb, bcs, info = vb.synth.make_shard(**cfg)
    with vb.Engine("coverage", umi=True, device=rank) as eng:
        eng.set_barcodes(bcs)
        uid = vdist.broadcast_bytes(vb.Engine.comm_unique_id() if rank == 0 else None, 128, device="cuda")
        eng.comm_init(uid, rank, world)
        eng.submit(sb)
        eng.finish_device()
        full = eng.fetch(eng.gather())
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), row=full.row, col=full.col, val=full.val, val2=full.val2,
                 ref=full.ref_cnt, alt=full.alt_cnt, scored=full.metrics["num_scored"])
        # the asynchronous, rooted form: two steps in flight, the gather of step 1 overlaps the kernels of step 2, and only
        # rank 1 (the "writer") receives; the slim layout feeds the second pass
        sl = vb.SlimBatch.from_staged(sb, True)
        eng.submit2(sl); eng.finish_device(); eng.gather_start(1)
        eng.submit2(sl); eng.finish_device()
        r1 = eng.gather_wait()
        got1 = eng.fetch(r1) if rank == 1 else None
        n1, scored1 = int(r1.n), int(r1.metrics.num_scored)
        eng.gather_start(1)
        r2 = eng.gather_wait()
        got2 = eng.fetch(r2) if rank == 1 else None
        assert int(r2.n) == n1 == len(full.row) and scored1 == full.metrics["num_scored"]
        if rank == 1:
            for g in (got1, got2):
                assert np.array_equal(g.row, full.row) and np.array_equal(g.col, full.col) and np.array_equal(g.val, full.val)
                assert np.array_equal(g.val2, full.val2) and np.array_equal(g.alt_cnt, full.alt_cnt)
        else:
            assert not r1.row and not r2.val            # non-root ranks get the totals only
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two CUDA devices")
def test_two_gpu_gather_matches_oracle(tmp_path, oracle):
    import torch.multiprocessing as mp
    import vartrix_b200 as vb
    from vartrix_b200 import dist as vdist
    from conftest import to_oracle_batch
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    exp = {k: [] for k in ("row", "col", "val", "val2", "ref_cnt", "alt_cnt")}
    scored = 0
    for rank in range(2):
        sb, bcs, _ = vb.synth.make_shard(**vdist.rank_workload(dict(n_loci=300, n_barcodes=80, depth=40, seed=2, kind="indel", umi=True), rank))
        r = oracle.run_batch(to_oracle_batch(oracle, sb), oracle.Barcodes(bcs.keys), oracle.MODE_COVERAGE, True, n_threads=8)
        for k in exp: exp[k].append(getattr(r, k))
        scored += r.metrics["num_scored"]
    for rank in range(2):
        got = np.load(tmp_path / f"rank{rank}.npz")
        assert np.array_equal(got["row"], np.concatenate(exp["row"])) and np.array_equal(got["col"], np.concatenate(exp["col"]))
        assert np.array_equal(got["val"], np.concatenate(exp["val"])) and np.array_equal(got["val2"], np.concatenate(exp["val2"]))
        assert np.array_equal(got["ref"], np.concatenate(exp["ref_cnt"])) and int(got["scored"]) == scored


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two CUDA devices")
def test_cli_shards_loci_over_two_gpus(tmp_path):
    """`--devices 0,1`: contiguous locus ranges per GPU, one rooted NCCL gather, outputs byte-identical to one GPU."""
    import subprocess
    from vartrix_b200 import synth_files
    ds = synth_files.write_dataset(str(tmp_path / "files"), n_loci=600, n_barcodes=80, depth=25, read_len=100, seed=13)
    cli = os.path.join(ROOT, "vartrix_b200", "bin", "vartrix_b200")
    outs = {}
    for name, dev in (("one", ["--device", "0"]), ("two", ["--devices", "0,1"]), ("two_rev", ["--devices", "1,0"]),
                      ("two_dev_staged", ["--devices", "0,1", "--gpu-stage"])):          # each GPU decodes the BAM ranges of its own loci
        d = tmp_path / name; d.mkdir()
        cmd = [cli, "-v", ds["vcf"], "-b", ds["bam"], "-f", ds["fasta"], "-c", ds["barcodes"], "-o", str(d / "out.mtx"), "--ref-matrix", str(d / "ref.mtx"),
               "-s", "coverage", "--umi", "--threads", "4", "--shard-loci", "37", "--log-level", "info", *dev]
        r = subprocess.run(cmd, cwd=str(d), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        outs[name] = (open(d / "out.mtx").read(), open(d / "ref.mtx").read(),
                      [ln for ln in r.stderr.splitlines() if "Number of" in ln])
    assert outs["one"][0].count("\n") > 1000
    assert outs["two"] == outs["one"] and outs["two_rev"] == outs["one"] and outs["two_dev_staged"] == outs["one"]
