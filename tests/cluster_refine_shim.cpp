// test shim: the per-item bodies of the cluster-refine kernels (vartrix_b200/csrc/vtx_cluster_refine.cuh, __host__ __device__)
// run serially on the CPU, for tests/test_cluster_refine_cpu.py.
#include "../vartrix_b200/csrc/vtx_cluster_refine.cuh"

using namespace vtx::cluster_refine;

// code [n][K] of gt [n][K] and pl [n][K][3]
extern "C" void vtx_test_cr_codes(uint32_t n, uint32_t K, const uint8_t* gt, const uint32_t* pl, uint8_t* code)
{
    for (size_t i = 0; i < size_t(n) * K; ++i) code[i] = code_of(gt[i], pl + i * 3);
}

// the nine-entry tables of every listed row at m: tab [n][9][2] (La, Lr)
extern "C" void vtx_test_cr_logs9(double eps, uint32_t m, uint32_t n, const uint64_t* A, const uint64_t* T, int32_t* tab)
{
    const vtx::ambient::Fractions fr = vtx::ambient::fractions(eps);
    for (uint32_t i = 0; i < n; ++i) row_logs9(fr, m, A[i], T[i], tab + size_t(i) * kEntries * 2);
}

// every cell against the scored rows: ll [n_cols][H], cnt [n_cols][3]
extern "C" void vtx_test_cr_score(uint32_t n_cols, uint32_t K, const uint32_t* start, const uint32_t* row, const uint32_t* r,
                                  const uint32_t* a, const uint32_t* sidx, const uint8_t* code, const int32_t* tab, int64_t* ll,
                                  uint64_t* cnt)
{
    const vtx::clusters::CellEntries ce{ start, row, r, a };
    const uint32_t H = vtx::donors::n_hyp(K);
    for (uint32_t c = 0; c < n_cols; ++c) score_cell(ce, c, K, sidx, code, tab, ll + size_t(c) * H, cnt + size_t(c) * 3);
}
