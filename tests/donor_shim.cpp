// test shim: the per-slot bodies of the donor kernels (vartrix_b200/csrc/vtx_donors.cuh, __host__ __device__) run serially on
// the CPU over every cell slot of a shard, for tests/test_donors_cpu.py.
#include "../vartrix_b200/csrc/vtx_donors.cuh"

extern "C" void vtx_test_donor_tables(double e, int64_t* lr, int64_t* la)
{
    const vtx::donors::Tables t = vtx::donors::make_tables(e);
    for (int s = 0; s < 5; ++s) { lr[s] = t.lr[s]; la[s] = t.la[s]; }
}

extern "C" void vtx_test_hyp_donors(uint32_t n_donors, uint32_t* d1, uint32_t* d2)
{
    for (uint32_t h = 0; h < vtx::donors::n_hyp(n_donors); ++h) vtx::donors::hyp_donors(h, n_donors, d1 + h, d2 + h);
}

// ll [n_cols][H] and cnt [n_cols][3] are added to; returns the number of qualifying slots
extern "C" uint64_t vtx_test_donor_ll(uint32_t n_slots, const uint32_t* cslot_col, const uint32_t* cslot_locus, const uint32_t* locus_row,
                                      const uint32_t* ccnt, const uint8_t* dosage, const uint8_t* usable, uint64_t n_rows, uint32_t n_cols,
                                      uint32_t n_donors, double e, int64_t* ll, uint64_t* cnt)
{
    using namespace vtx::donors;
    const uint32_t H = n_hyp(n_donors);
    const Inputs in{ cslot_col, cslot_locus, locus_row, ccnt, dosage, usable, n_rows, n_cols, n_donors, H, make_tables(e) };
    uint64_t n = 0;
    for (uint32_t q = 0; q < n_slots; ++q) {
        if (qualifying_row(in, q) < 0) continue;
        add_slot(in, q, ll + size_t(cslot_col[q]) * H, cnt + size_t(cslot_col[q]) * 3);
        ++n;
    }
    return n;
}
