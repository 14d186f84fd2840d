// test shim: the per-item bodies of the ambient-RNA kernels (vartrix_b200/csrc/vtx_ambient.cuh, __host__ __device__) run
// serially on the CPU, for tests/test_ambient_cpu.py.
#include "../vartrix_b200/csrc/vtx_ambient.cuh"

using namespace vtx::ambient;

// the tables of every listed row at m: tab [n][5][2] (La, Lr)
extern "C" void vtx_test_am_tables(double eps, uint32_t m, uint32_t n, const uint64_t* A, const uint64_t* T, int32_t* tab)
{
    const Fractions fr = fractions(eps);
    for (uint32_t i = 0; i < n; ++i) row_logs(fr, m, A[i], T[i], tab + size_t(i) * 10);
}

// every cell's scoring against one table set: ll [n_cols][H], cnt [n_cols][3], call [n_cols] (§5f's rule)
extern "C" void vtx_test_am_score(uint32_t n_cols, uint32_t D, const uint32_t* start, const uint32_t* row, const uint32_t* r,
                                  const uint32_t* a, const uint32_t* tix, const uint8_t* dos, const int32_t* tab, int64_t* ll,
                                  uint64_t* cnt, uint32_t* call)
{
    const vtx::clusters::CellEntries ce{ start, row, r, a };
    const uint32_t H = vtx::donors::n_hyp(D);
    for (uint32_t c = 0; c < n_cols; ++c) {
        int64_t* L = ll + size_t(c) * H;
        score_cell(ce, c, D, tix, dos, tab, L, cnt + size_t(c) * 3);
        uint32_t best = 0, second = 1, pair = D;
        for (uint32_t h = 1; h < D; ++h) if (L[h] > L[best]) best = h;
        second = best == 0 ? 1 : 0;
        for (uint32_t h = second + 1; h < D; ++h) if (h != best && L[h] > L[second]) second = h;
        for (uint32_t h = D + 1; h < H; ++h) if (L[h] > L[pair]) pair = h;
        call[c] = vtx::donors::call_of(cnt[size_t(c) * 3], L[best], L[second], L[pair]);
    }
}

// vtx_set_donors' ten constants (libm log) for the comparison at m = 0
extern "C" void vtx_test_donor_tables(double eps, int64_t* lr, int64_t* la)
{
    const vtx::donors::Tables t = vtx::donors::make_tables(eps);
    for (int s = 0; s < 5; ++s) { lr[s] = t.lr[s]; la[s] = t.la[s]; }
}
