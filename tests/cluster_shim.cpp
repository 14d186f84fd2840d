// test shim: the per-item bodies of the clustering kernels (vartrix_b200/csrc/vtx_clusters.cuh, __host__ __device__) run
// serially on the CPU, for tests/test_clusters_cpu.py.
#include "../vartrix_b200/csrc/vtx_clusters.cuh"

using namespace vtx::clusters;

extern "C" void vtx_test_ll_log(uint64_t n, const double* x, double* y) { for (uint64_t i = 0; i < n; ++i) y[i] = ll_log(x[i]); }
extern "C" void vtx_test_ll_exp(uint64_t n, const double* x, double* y) { for (uint64_t i = 0; i < n; ++i) y[i] = ll_exp(x[i]); }
extern "C" uint64_t vtx_test_splitmix64(uint64_t x) { return splitmix64(x); }

// la / lr [n_rows][K] of restart s at the listed rows
extern "C" void vtx_test_cl_init(uint64_t seed, uint32_t s, uint32_t K, uint32_t n_used, const uint32_t* used_rows, int32_t* la, int32_t* lr)
{
    for (uint32_t i = 0; i < n_used; ++i)
        for (uint32_t k = 0; k < K; ++k) init_logs(seed, s, k, used_rows[i], la + size_t(used_rows[i]) * K + k, lr + size_t(used_rows[i]) * K + k);
}

// every cell's E-step: w [n_cols][K], m [n_cols]
extern "C" void vtx_test_cl_estep(uint32_t n_cols, uint32_t K, const uint32_t* start, const uint32_t* row, const uint32_t* r,
                                  const uint32_t* a, const int32_t* la, const int32_t* lr, uint32_t* w, int64_t* m)
{
    const CellEntries ce{ start, row, r, a };
    for (uint32_t c = 0; c < n_cols; ++c) m[c] = estep_cell(ce, c, K, la, lr, w + size_t(c) * K);
}

// every row's M-step sums (map: output column j sums EM cluster map[j]) and the tables of those sums
extern "C" void vtx_test_cl_mstep(uint32_t n_rows, const uint32_t* row_start, const uint32_t* col, const uint32_t* r, const uint32_t* a,
                                  const uint32_t* w, uint32_t K, const uint32_t* map, int64_t* A, int64_t* T, int32_t* la, int32_t* lr)
{
    for (uint32_t v = 0; v < n_rows; ++v) {
        mstep_row(col, r, a, row_start[v], row_start[v + 1], w, K, map, A + size_t(v) * K, T + size_t(v) * K);
        for (uint32_t j = 0; j < K; ++j) row_logs(A[size_t(v) * K + j], T[size_t(v) * K + j], la + size_t(v) * K + j, lr + size_t(v) * K + j);
    }
}

// every cell's final scoring: ll [n_cols][H], cnt [n_cols][3]
extern "C" void vtx_test_cl_score(uint32_t n_cols, uint32_t K, const uint32_t* start, const uint32_t* row, const uint32_t* r,
                                  const uint32_t* a, const int64_t* A, const int64_t* T, int64_t* ll, uint64_t* cnt)
{
    const CellEntries ce{ start, row, r, a };
    const uint32_t H = vtx::donors::n_hyp(K);
    for (uint32_t c = 0; c < n_cols; ++c) score_cell(ce, c, K, A, T, ll + size_t(c) * H, cnt + size_t(c) * 3);
}
