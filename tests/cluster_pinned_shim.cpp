// test shim: the per-item bodies of the pinned clustering (vartrix_b200/csrc/vtx_cluster_pinned.cuh, __host__ __device__) run
// serially on the CPU, for tests/test_cluster_pinned_cpu.py.
#include "../vartrix_b200/csrc/vtx_cluster_pinned.cuh"

using namespace vtx;
using namespace vtx::cluster_pinned;

// la / lr [n_rows][J] of every (row, sample) with a dosage in dos [n_rows][J] (the others are left as they are)
extern "C" void vtx_test_cp_logs(double eps, uint32_t m, uint32_t n_rows, uint32_t J, const uint8_t* dos, const uint64_t* row_alt,
                                 const uint64_t* row_depth, int32_t* la, int32_t* lr)
{
    const ambient::Fractions fr = ambient::fractions(eps);
    for (size_t i = 0; i < size_t(n_rows) * J; ++i)
        if (dos[i] != kMissing) pinned_logs(fr, m, row_alt[i / J], row_depth[i / J], dos[i], la + i, lr + i);
}

// every cell's final scoring: ll [n_cols][H], cnt [n_cols][3]
extern "C" void vtx_test_cp_score(uint32_t n_cols, uint32_t K, uint32_t J, double eps, uint32_t m, const uint32_t* start, const uint32_t* row,
                                  const uint32_t* r, const uint32_t* a, const uint8_t* dos, const uint64_t* row_alt, const uint64_t* row_depth,
                                  const int64_t* A, const int64_t* T, int64_t* ll, uint64_t* cnt)
{
    const clusters::CellEntries ce{ start, row, r, a };
    Pins p{};
    p.J = J; p.m = m; p.fr = ambient::fractions(eps); p.dos = dos;
    p.rowA = reinterpret_cast<const unsigned long long*>(row_alt);
    p.rowT = reinterpret_cast<const unsigned long long*>(row_depth);
    const uint32_t H = donors::n_hyp(K);
    for (uint32_t c = 0; c < n_cols; ++c) score_cell(ce, c, K, p, A, T, ll + size_t(c) * H, cnt + size_t(c) * 3);
}
