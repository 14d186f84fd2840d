// test shim: the tile-class rule (vartrix_b200/csrc/vtx_tile_class.cuh) on the CPU -- the class vtx_k_locus_prep gives a
// locus, and the kernels run_sw launches for a device batch and for a host batch.
#include "../vartrix_b200/csrc/vtx_tile_class.cuh"

using namespace vtx;

extern "C" int vtx_test_tile_class(int exotic, int prefix, int fold, uint32_t width, uint32_t longest_read, uint32_t flags,
                                   uint32_t max_read, uint32_t max_hap)
{
    const LocusShape s{ exotic != 0, prefix != 0, fold != 0, width };
    return tile_class(s, allowed_kernels(flags, max_read, max_hap), longest_read);
}

extern "C" uint32_t vtx_test_device_mask(uint32_t flags, uint32_t max_read, uint32_t max_hap)
{
    return device_class_mask(allowed_kernels(flags, max_read, max_hap), max_hap);
}

// A host batch as vtx_submit sees it: windows in `hap`, the shape key of every locus, the widest window as max_hap.
extern "C" uint32_t vtx_test_host_mask(const uint8_t* hap, uint32_t n_loci, const uint32_t* ref_off, const uint32_t* ref_len,
                                       const uint32_t* alt_off, const uint32_t* alt_len, uint32_t flags, uint32_t max_read)
{
    uint64_t seen = 0;
    uint32_t max_hap = 0;
    for (uint32_t l = 0; l < n_loci; ++l) {
        seen |= uint64_t(1) << shape_key(window_shape(hap + ref_off[l], ref_len[l], hap + alt_off[l], alt_len[l]));
        max_hap = std::max(max_hap, std::max(ref_len[l], alt_len[l]));
    }
    return host_class_mask(seen, allowed_kernels(flags, max_read, max_hap), max_read);
}
