// test shim: locus_cands' per-locus record-filter counters (vartrix_b200/csrc/vtx_stage.cuh, pass 0 with `lfilt`, the store
// vtx_set_locus_stats adds) run serially on the CPU after the record walk and parse, as vtx_submit_bam runs them.
#include <vector>
#include "../vartrix_b200/csrc/vtx_stage.cuh"

extern "C" int vtx_test_locus_filters(const uint8_t* stream, uint64_t stream_len, int32_t tid, uint32_t mapq, int primary_only,
                                      int no_duplicates, uint32_t min_base_quality, uint32_t n_entry, const uint64_t* entry,
                                      uint32_t n_loci, const int64_t* l_start, const int64_t* l_end, uint32_t* lfilt /* [n_loci][6] */)
{
    using namespace vtx::stage;
    Params P{};
    P.s = stream; P.s_len = stream_len; P.tid = tid; P.mapq_min = mapq; P.primary_only = primary_only; P.no_duplicates = no_duplicates;
    P.tag0 = 'C'; P.tag1 = 'B'; P.min_base_quality = min_base_quality;
    const uint32_t n_seg = n_entry ? n_entry - 1 : 0;
    std::vector<uint32_t> seg_count(n_seg + 1, 0), seg_first(n_seg + 2, 0);
    uint32_t err = 0, max_span = 0, max_read = 0;
    DirectFetch F{ stream };
    for (uint32_t k = 0; k < n_seg; ++k) walk_segment(P, k, entry, 0, seg_count.data(), nullptr, nullptr, &err, F);
    for (uint32_t k = 0; k < n_seg; ++k) seg_first[k + 1] = seg_first[k] + seg_count[k];
    if (err & (kErrWalk | kErrRecord)) return 1;
    const uint32_t n_rec = seg_first[n_seg];
    std::vector<uint64_t> rec_off(n_rec + 1);
    std::vector<int32_t> rec_tid(n_rec + 1), rec_pos(n_rec + 1), rec_end(n_rec + 1);
    std::vector<uint32_t> rec_fm(n_rec + 1), cand_count(n_loci + 1, 0);
    for (uint32_t k = 0; k < n_seg; ++k) walk_segment(P, k, entry, 1, nullptr, seg_first.data(), rec_off.data(), &err, F);
    for (uint32_t i = 0; i < n_rec; ++i) parse_record(P, i, rec_off.data(), rec_tid.data(), rec_pos.data(), rec_end.data(), rec_fm.data(), &max_span);
    LocusMetrics met{};
    for (uint32_t l = 0; l < n_loci; ++l)
        locus_cands(P, l, l_start, l_end, n_rec, rec_off.data(), rec_tid.data(), rec_pos.data(), rec_end.data(), rec_fm.data(), &max_span,
                    &max_read, 0, cand_count.data(), nullptr, nullptr, nullptr, &met, lfilt);
    return 0;
}
