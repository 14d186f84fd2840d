// test shim: the per-item bodies of the cluster-genotype kernels (vartrix_b200/csrc/vtx_cluster_gt.cuh, __host__ __device__)
// run serially on the CPU, for tests/test_cluster_genotypes_cpu.py.
#include "../vartrix_b200/csrc/vtx_cluster_gt.cuh"

using namespace vtx::cluster_gt;

// the six logs of every listed row at m: out [n][6]
extern "C" void vtx_test_cg_logs(double eps, uint32_t m, uint32_t n, const uint64_t* A, const uint64_t* T, int32_t* out)
{
    const vtx::ambient::Fractions fr = vtx::ambient::fractions(eps);
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = 0; j < 6; ++j) out[size_t(i) * 6 + j] = gt_log(fr, m, A[i], T[i], j);
}

// fit_row of every (row, cluster): ll [n][K][3], mx [n][K]
extern "C" void vtx_test_cg_fit(uint32_t n, uint32_t K, const int32_t* L, const int64_t* Aw, const int64_t* Tw, int64_t* ll, int64_t* mx)
{
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t k = 0; k < K; ++k) {
            const size_t o = size_t(i) * K + k;
            mx[o] = fit_row(L + size_t(i) * 6, Aw[o], Tw[o], ll + o * 3);
        }
}

// call_row and gq_of of every (row, cluster): gt [n][K], pl [n][K][3], gq [n][K]
extern "C" void vtx_test_cg_call(uint32_t n, uint32_t K, const int64_t* ll, const int64_t* Tw, uint8_t* gt, uint32_t* pl, uint32_t* gq)
{
    for (size_t o = 0; o < size_t(n) * K; ++o) {
        call_row(ll + o * 3, Tw[o] > 0, gt + o, pl + o * 3);
        gq[o] = gq_of(pl + o * 3);
    }
}

// match_row over n compared rows: g [n][S]; M, disc [K][S]
extern "C" void vtx_test_cg_match(uint32_t n, uint32_t K, uint32_t S, const int64_t* ll, const uint8_t* gt, const uint32_t* pl,
                                  const uint8_t* g, int64_t* M, uint64_t* disc)
{
    for (uint32_t k = 0; k < K; ++k)
        for (uint32_t s = 0; s < S; ++s) {
            int64_t m = 0;
            uint32_t d = 0;
            for (uint32_t i = 0; i < n; ++i) {
                const size_t o = size_t(i) * K + k;
                match_row(ll + o * 3, gt[o], gq_of(pl + o * 3) >= kMinGq, g[size_t(i) * S + s], &m, &d);
            }
            M[size_t(k) * S + s] = m;
            disc[size_t(k) * S + s] = d;
        }
}

extern "C" void vtx_test_cg_phred(uint32_t n, const int64_t* d, uint32_t* out) { for (uint32_t i = 0; i < n; ++i) out[i] = phred(d[i]); }

// the assignment of every cluster: out [K][4] = best, second, assigned, and llr [K]
extern "C" void vtx_test_cg_assign(uint32_t K, uint32_t S, const int64_t* M, const uint64_t* disc, const uint64_t* called, uint32_t* out,
                                   int64_t* llr)
{
    for (uint32_t k = 0; k < K; ++k) {
        const Assignment a = assign(M + size_t(k) * S, disc + size_t(k) * S, called[k], S);
        out[k * 4] = a.best; out[k * 4 + 1] = a.second; out[k * 4 + 2] = a.assigned; out[k * 4 + 3] = 0;
        llr[k] = a.llr;
    }
}
