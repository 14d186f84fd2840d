"""GPU: a context frees everything it allocated.  Three rounds of create -> every kind of work -> destroy leave the
device's free memory where the first round left it."""
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _one_life(sb, bcs, members, raws):
    import vartrix_b200 as vb
    with vb.Engine("coverage", umi=True) as eng:
        eng.set_barcodes(bcs)
        eng.submit(sb)
        eng.submit2(vb.SlimBatch.from_staged(sb, True))
        got = eng.finish()
        assert len(got.row) > 0
        rs, _ = eng.score_pairs(sb, sb.cand_read[:50], np.zeros(50, np.uint32))
        assert len(rs) == 50
        out, status = eng.bgzf_inflate(members)
        assert (status == 0).all() and out == raws
        fetched = eng.fetch(eng.gather())           # one rank: the gather hands back the local result
        assert np.array_equal(fetched.row, got.row) and np.array_equal(fetched.val, got.val)


def test_context_memory_is_returned():
    import torch
    import vartrix_b200 as vb
    sb, bcs, info = vb.synth.make_shard(200, 60, depth=20, seed=5, kind="indel", umi=True)
    raws = [bytes(np.random.default_rng(i).integers(0, 4, 20000, dtype=np.uint8) + 65) for i in range(8)]
    members = [(zlib.compress(r, 6)[2:-4], len(r), zlib.crc32(r) & 0xFFFFFFFF) for r in raws]
    torch.cuda.init()
    free = []
    for _ in range(3):
        _one_life(sb, bcs, members, raws)
        torch.cuda.synchronize()
        free.append(torch.cuda.mem_get_info()[0])
    assert abs(free[2] - free[0]) <= 1 << 20, free
