// test shim: the --min-base-quality decision body (vtx::stage::base_quality_ok, vartrix_b200/csrc/vtx_base_quality.cuh),
// reached through vtx_stage.cuh as locus_cands reaches it on the device, run serially on the CPU over (record, locus) pairs.
#include "../vartrix_b200/csrc/vtx_stage.cuh"

// rec_off[i]: offset in `data` of pair i's record without its block_size field; the pair's locus is [start[i], end[i]).
extern "C" int vtx_test_base_quality(const uint8_t* data, uint64_t n, const uint64_t* rec_off, const int64_t* start, const int64_t* end,
                                     uint32_t min_q, uint8_t* keep)
{
    for (uint64_t i = 0; i < n; ++i) keep[i] = vtx::stage::base_quality_ok(data + rec_off[i], start[i], end[i], min_q) ? 1 : 0;
    return 0;
}
