// test shim: the per-record body of the device QNAME interning pass (vtx_k_name_key, vartrix_b200/csrc/vtx_stage.cuh) run
// serially on the CPU over records of an inflated BAM stream, with the kernel's hash or with a constant one that puts every
// name into one probe chain.
#include <cstring>
#include <vector>
#include "../vartrix_b200/csrc/vtx_stage.cuh"

struct ConstHash {
    __host__ __device__ uint32_t operator()(const uint8_t*, uint32_t) const { return 7u; }
};

// rec_off[i]: offset of record i's block_size field in `stream`; read_umi[i] = the key of record i (VTX_NO_UMI if !used[i]).
// The records run in the given order (a permutation of 0..n_rec-1): on the device any of them may claim its slot first.
extern "C" int vtx_test_name_keys(const uint8_t* stream, uint64_t stream_len, uint32_t n_rec, const uint64_t* rec_off, const uint32_t* used,
                                  const uint32_t* order, int const_hash, uint64_t* read_umi)
{
    using namespace vtx::stage;
    Params P{};
    P.s = stream; P.s_len = stream_len;
    uint32_t size = 1;
    while (size < 2 * n_rec) size <<= 1;
    std::vector<uint32_t> tab(size, kEmptySlot);
    for (uint32_t k = 0; k < n_rec; ++k) {
        const uint32_t i = order[k];
        if (const_hash) name_key(P, i, rec_off, used, tab.data(), size - 1, read_umi, ConstHash{});
        else name_key(P, i, rec_off, used, tab.data(), size - 1, read_umi, NameHash{});
    }
    return 0;
}
