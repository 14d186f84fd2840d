"""The pieces of bench.py's timed path that the tests restate: its workload, its dump sample, its e2e shard schedule and
how it places a shard in pinned or device memory.  Everything here reads bench.py's own defaults and constants, so the
tests follow bench.py when they change."""
import numpy as np

import bench


def bench_args(*argv):
    """bench.py's parsed arguments for `argv` (its defaults for everything not given)."""
    return bench.parse_args(list(argv))


def bench_workload(*argv):
    """-> (args, cfg): the arguments and the synth config bench.py runs for `argv` on rank 0."""
    args = bench_args(*argv)
    return args, bench.workload_config(args, 0)


def dump_sample(n, n_arrays):
    """Indices of the triplets bench.dump_outputs keeps of n triplets in n_arrays arrays (all of them below its cap)."""
    cap = (bench.DUMP_BYTES - 4096) // (8 * max(n_arrays, 1))
    if n > cap:
        return np.sort(np.random.default_rng(0).choice(n, cap, replace=False))
    return np.arange(n)


def e2e_bounds(args, cand_start, growth):
    """The non-empty locus ranges of bench.py's e2e shards at `growth` (stage_e2e_shards)."""
    import vartrix_b200 as vb
    n_cand = int(cand_start[-1])
    first = max(args.first_chunk, min(1.0, args.min_shard / max(n_cand, 1)))
    return [(lo, hi) for lo, hi in vb.shard_bounds(cand_start, max(1, args.chunks), first_frac=first, growth=growth) if hi > lo]


def value_submits(args, n_cand):
    """Device-resident submits per `value` step (bench.py: --submits, else 4 above 8 M candidates)."""
    return args.submits or (4 if n_cand > 8_000_000 else 1)


def with_empty_submits(cand_start, n_submits):
    """n_submits contiguous locus ranges covering every locus once; from 5 submits on, four of them are empty (the first,
    two adjacent ones in the middle and the last)."""
    import vartrix_b200 as vb
    n_empty = 4 if n_submits >= 5 else 0
    full = vb.shard_bounds(cand_start, n_submits - n_empty)
    if not n_empty:
        return full
    n_loci = len(cand_start) - 1
    out = [(0, 0)] + full
    mid = len(out) // 2
    at = out[mid][0]
    out[mid:mid] = [(at, at), (at, at)]
    return out + [(n_loci, n_loci)]


def place(batch, fields, where, keep):
    """bench.py's place(): the arrays of `batch` copied to pinned host memory ("pinned") or to the device ("cuda") with
    torch; -> {field: address}.  The tensors are appended to `keep` (they must outlive the submits)."""
    import torch
    ptr = {}
    for f in fields:
        a = getattr(batch, f)
        if a is None or a.size == 0:
            continue
        t = torch.from_numpy(a.view(np.uint8).reshape(-1) if a.dtype.itemsize > 1 else a.reshape(-1))
        t = t.pin_memory() if where == "pinned" else t.cuda()
        keep.append(t)
        ptr[f] = t.data_ptr()
    return ptr


def c_batch(batch, ptr):
    """The C struct of a SlimBatch (vtx_batch2) or StagedBatch (vtx_batch) whose arrays live at ptr's addresses."""
    import vartrix_b200 as vb
    if isinstance(batch, vb.SlimBatch):
        return batch.to_c(ptr)
    cb = batch.to_c()
    for f in vb.StagedBatch.FIELDS:
        setattr(cb, f, ptr.get(f))
    return cb
