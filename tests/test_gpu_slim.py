"""GPU: the slim staging layout (vtx_submit2) gives bit-identical triplets and metrics to the vtx_batch layout and to the
oracle -- cell tags as codes and as exotic byte strings, reads without tags / UMIs, reads shared between loci
(explicit cand_read), dense read pools with ragged lengths, empty shards, and the device-side bounds check."""
import ctypes as C

import numpy as np
import pytest

from conftest import assert_same_triplets, to_oracle_batch

pytestmark = pytest.mark.gpu


def _both(oracle, sb, bcs, mode, umi, n_parts=1):
    import vartrix_b200 as vb
    exp = oracle.run_batch(to_oracle_batch(oracle, sb), oracle.Barcodes(bcs.keys), oracle.MODES[mode], umi, n_threads=4)
    sl = vb.SlimBatch.from_staged(sb, umi)
    with vb.Engine(mode, umi=umi) as eng:
        eng.set_barcodes(bcs)
        for lo, hi in vb.shard_bounds(sb.cand_start, n_parts):
            eng.submit2(sl.shard(lo, hi) if n_parts > 1 else sl)
        got = eng.finish()
    assert_same_triplets(got, exp)
    assert got.metrics == exp.metrics
    return sl, got


@pytest.mark.parametrize("mode,kind,umi,parts", [("consensus", "snv", False, 1), ("coverage", "indel", True, 3), ("alt_frac", "snv", True, 2),
                                                  ("coverage", "snv", False, 4)])
def test_slim_equals_oracle(oracle, mode, kind, umi, parts):
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(400, 120, depth=30, seed=21, kind=kind, umi=umi)
    _both(oracle, sb, bcs, mode, umi, parts)


def test_slim_exotic_tags_missing_tags_shared_reads_ragged_lengths(oracle):
    import vartrix_b200 as vb
    rng = np.random.default_rng(8)
    sb, bcs, info = vb.synth.make_shard(120, 40, depth=16, seed=4, kind="indel", umi=True, read_len=101)
    # barcode list with exotic members (lower case, N, too long, odd suffix) next to ordinary ones
    exotic = [b"acgtacgtacgtacgt-1", b"ACGTNCGTACGTACGT-1", b"A" * 30, b"ACGT-001", b"ACGT_1", b"TTTT"]
    keys = list(bcs.keys) + exotic
    bcs2 = vb.Barcodes(keys)
    n = sb.n_reads
    tags = [bytes(sb.cb_bytes[int(o): int(o) + 18]) for o in sb.read_cb_off]
    for r in rng.choice(n, 300, replace=False):
        tags[r] = exotic[int(rng.integers(0, len(exotic)))] if rng.random() < 0.7 else b"GGGGNNNN-1"     # listed / unlisted exotic
    off = np.zeros(n, np.uint32); ln = np.zeros(n, np.uint16); pos = 0
    for r, t in enumerate(tags):
        off[r] = pos; ln[r] = len(t); pos += len(t)
    none = rng.choice(n, 60, replace=False)
    off[none] = 0xFFFFFFFF; ln[none] = 0
    umi = sb.read_umi_key.copy(); umi[rng.choice(n, 80, replace=False)] = np.uint64(0xFFFFFFFFFFFFFFFF)
    # ragged read lengths (dense pool offsets come from a device scan) and reads shared by neighbouring loci
    rl = sb.read_len.copy(); rl[rng.choice(n, 500, replace=False)] = rng.integers(1, 101, 500).astype(np.uint32)
    cand = sb.cand_read.copy()
    d = 16
    for l in range(1, sb.n_loci, 3):
        cand[l * d: l * d + 4] = cand[(l - 1) * d: (l - 1) * d + 4]       # four reads of the previous locus are candidates here too
    sb2 = vb.StagedBatch(sb.locus_row, sb.hap_bytes, sb.ref_off, sb.ref_len, sb.alt_off, sb.alt_len, sb.cand_start, sb.read_nib, sb.read_off,
                         rl, np.frombuffer(b"".join(tags), np.uint8), off, ln, umi, cand, n_rows=sb.n_rows)
    for mode, use_umi, parts in (("coverage", True, 1), ("consensus", False, 3)):
        sl, got = _both(oracle, sb2, bcs2, mode, use_umi, parts)
        assert sl.n_exotic > 100 and sl.cand_read is not None
        assert got.metrics["num_not_cell_bc"] > 60
        # the same shards resident on the device (vtx_submit2_device): the host must not read their arrays
        res = _resident(sl, sb2.cand_start, bcs2, mode, use_umi, parts)
        assert_same_triplets(res, got)
        assert res.metrics == got.metrics


def _resident(sl, cand_start, bcs, mode, umi, n_parts):
    """Every shard copied to the device with torch and submitted through vtx_submit2_device."""
    import torch
    import vartrix_b200 as vb
    max_read = int(sl.read_len.max())
    max_hap = int(max(sl.ref_len.max(), sl.alt_len.max()))
    keep = []
    with vb.Engine(mode, umi=umi) as eng:
        eng.set_barcodes(bcs)
        for lo, hi in vb.shard_bounds(cand_start, n_parts):
            part = sl.shard(lo, hi) if n_parts > 1 else sl
            ptr = {}
            for f in vb.SlimBatch.ARRAYS:
                a = getattr(part, f)
                if a is None or a.size == 0:
                    continue
                t = torch.from_numpy(a.view(np.uint8).reshape(-1) if a.dtype.itemsize > 1 else a.reshape(-1)).cuda()
                keep.append(t)
                ptr[f] = t.data_ptr()
            eng.submit2_device(part.to_c(ptr), max_read, max_hap)
        return eng.finish()


def test_slim_empty_shards(oracle):
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(30, 10, depth=5, seed=2)
    sl = vb.SlimBatch.from_staged(sb, False)
    with vb.Engine("coverage") as eng:
        eng.set_barcodes(bcs)
        eng.submit2(sl.shard(0, 0)); eng.submit2(sl.shard(0, 12)); eng.submit2(sl.shard(12, 12)); eng.submit2(sl.shard(12, 30))
        got = eng.finish()
    exp = oracle.run_batch(to_oracle_batch(oracle, sb), oracle.Barcodes(bcs.keys), oracle.MODE_COVERAGE, False, n_threads=2)
    assert_same_triplets(got, exp)


def test_slim_rejects_malformed(oracle):
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(20, 10, depth=5, seed=2)
    sl = vb.SlimBatch.from_staged(sb, False)
    with vb.Engine("coverage") as eng:
        eng.set_barcodes(bcs)
        bad = vb.SlimBatch.from_staged(sb, False); bad.read_nib = bad.read_nib[:-40]
        with pytest.raises(vb.VtxError, match="dense read pool"):
            eng.submit2(bad)
        bad = vb.SlimBatch.from_staged(sb, False); bad.read_cb_key = bad.read_cb_key.copy(); bad.read_cb_key[3] = np.uint64(0x8000000000000005)
        with pytest.raises(vb.VtxError, match="CB outside"):
            eng.submit2(bad)
        bad = vb.SlimBatch.from_staged(sb, False); bad.read_cb_key = bad.read_cb_key.copy(); bad.read_cb_key[3] = np.uint64(1 << 61)
        with pytest.raises(vb.VtxError, match="vtx_pack_cb"):
            eng.submit2(bad)
        eng.submit2(sl)                     # the ctx is still usable
        assert eng.finish().metrics["num_scored"] == info["n_pairs"]
    with vb.Engine("coverage", umi=True) as eng:
        eng.set_barcodes(bcs)
        with pytest.raises(vb.VtxError, match="read arrays missing"):
            eng.submit2(sl)                 # --umi needs the UMI keys


def test_device_batch_that_breaks_its_promised_bounds_is_reported(oracle):
    """vtx_submit_device_ex sizes buffers from the caller's bounds; loci that exceed them are skipped on the device and the
    next finish says so (it used to be undefined behaviour)."""
    import torch
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(50, 10, depth=8, seed=3, read_len=150)
    with vb.Engine("coverage") as eng:
        eng.set_barcodes(bcs)
        dev = {}
        db = sb.to_c()
        for f in vb.StagedBatch.FIELDS:
            a = getattr(sb, f)
            t = torch.from_numpy(a.view(np.uint8).reshape(-1) if a.dtype.itemsize > 1 else a.reshape(-1)).cuda()
            dev[f] = t; setattr(db, f, t.data_ptr() if t.numel() else None)
        eng.submit_device(db, 100, 320)                       # reads are 150 bases: the promise is broken
        with pytest.raises(vb.VtxError, match="exceeded the bounds"):
            eng.finish()
        eng.submit_device(db, 150, 208)
        got = eng.finish()
        assert got.metrics["num_scored"] == info["n_pairs"] and len(got.row) > 0
