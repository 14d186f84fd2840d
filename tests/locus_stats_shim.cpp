// test shim: the per-locus body of the locus-statistics kernel (vartrix_b200/csrc/vtx_locus_stats.cuh, __host__ __device__)
// run serially on the CPU over every locus of a shard, for tests/test_variant_stats_cpu.py.
#include "../vartrix_b200/csrc/vtx_locus_stats.cuh"

extern "C" int vtx_test_locus_stats(uint32_t n_loci, const uint64_t* cand_start, const uint32_t* cand_read, const int32_t* read_col,
                                    const uint64_t* read_umi, const uint32_t* pair_start, const uint32_t* ucnt, const uint32_t* ccnt,
                                    const uint32_t* cslot_col, const uint32_t* locus_row, const uint32_t* filters, uint32_t* out)
{
    const vtx::lstats::Inputs in{ cand_start, cand_read, read_col, read_umi, pair_start, ucnt, ccnt, cslot_col, locus_row, filters };
    for (uint32_t l = 0; l < n_loci; ++l) vtx::lstats::locus_serial(in, l, out + size_t(l) * vtx::lstats::kFields);
    return vtx::lstats::kFields;
}
