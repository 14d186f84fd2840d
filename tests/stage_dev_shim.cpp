// test shim: the per-item bodies of the DEVICE staging kernels (vartrix_b200/csrc/vtx_stage.cuh: record walk, record parse,
// per-locus fetch + filters, read / tag extraction -- all __host__ __device__) run serially on the CPU, with plain exclusive
// scans where the engine runs its scan kernels.  Same call order as vtx_submit_bam (csrc/vtx_api.cu).
#include <cstring>
#include <vector>
#include "../vartrix_b200/csrc/vtx_stage.cuh"

struct StageOut {                     // arrays sized by the caller: n_rec_cap records, n_cand_cap candidates
    uint32_t n_rec, err, max_span, max_read;
    uint64_t n_cand;
    unsigned long long metrics[5];
};

extern "C" int vtx_test_stage_dev(const uint8_t* stream, uint64_t stream_len, int32_t tid, uint32_t mapq, int primary_only, int no_duplicates,
                                  int want_umi, const char* tag, uint32_t n_entry, const uint64_t* entry, uint32_t n_loci,
                                  const int64_t* l_start, const int64_t* l_end, uint32_t rec_cap, uint64_t cand_cap, StageOut* out,
                                  uint32_t* cand_first /* n_loci + 1 */, uint32_t* cand_rec, uint64_t* read_off, uint32_t* read_len,
                                  uint32_t* read_cb_off, uint16_t* read_cb_len, uint64_t* read_umi, uint32_t* used)
{
    using namespace vtx::stage;
    Params P{};
    P.s = stream; P.s_len = stream_len; P.tid = tid; P.mapq_min = mapq; P.primary_only = primary_only; P.no_duplicates = no_duplicates;
    P.want_umi = want_umi; P.tag0 = uint8_t(tag[0]); P.tag1 = uint8_t(tag[1]);
    memset(out, 0, sizeof(*out));
    const uint32_t n_seg = n_entry ? n_entry - 1 : 0;
    std::vector<uint32_t> seg_count(n_seg + 1, 0), seg_first(n_seg + 2, 0);
    DirectFetch F{ stream };
    for (uint32_t k = 0; k < n_seg; ++k) walk_segment(P, k, entry, 0, seg_count.data(), nullptr, nullptr, &out->err, F);
    for (uint32_t k = 0; k < n_seg; ++k) seg_first[k + 1] = seg_first[k] + seg_count[k];
    if (out->err & (kErrWalk | kErrRecord)) return 1;
    const uint32_t n_rec = seg_first[n_seg];
    out->n_rec = n_rec;
    if (n_rec > rec_cap) return 2;
    std::vector<uint64_t> rec_off(n_rec + 1);
    std::vector<int32_t> rec_tid(n_rec + 1), rec_pos(n_rec + 1), rec_end(n_rec + 1);
    std::vector<uint32_t> rec_fm(n_rec + 1);
    for (uint32_t k = 0; k < n_seg; ++k) walk_segment(P, k, entry, 1, nullptr, seg_first.data(), rec_off.data(), &out->err, F);
    for (uint32_t i = 0; i < n_rec; ++i) parse_record(P, i, rec_off.data(), rec_tid.data(), rec_pos.data(), rec_end.data(), rec_fm.data(), &out->max_span);
    memset(used, 0, size_t(n_rec) * 4);
    std::vector<uint32_t> cand_count(n_loci + 1, 0);
    LocusMetrics met{};
    for (uint32_t l = 0; l < n_loci; ++l)
        locus_cands(P, l, l_start, l_end, n_rec, rec_off.data(), rec_tid.data(), rec_pos.data(), rec_end.data(), rec_fm.data(), &out->max_span,
                    &out->max_read, 0, cand_count.data(), nullptr, nullptr, nullptr, &met);
    cand_first[0] = 0;
    for (uint32_t l = 0; l < n_loci; ++l) cand_first[l + 1] = cand_first[l] + cand_count[l];
    out->n_cand = cand_first[n_loci];
    if (out->n_cand > cand_cap) return 3;
    LocusMetrics scratch{};
    for (uint32_t l = 0; l < n_loci; ++l)
        locus_cands(P, l, l_start, l_end, n_rec, rec_off.data(), rec_tid.data(), rec_pos.data(), rec_end.data(), rec_fm.data(), &out->max_span,
                    &out->max_read, 1, nullptr, cand_first, cand_rec, used, &scratch);
    for (uint32_t i = 0; i < n_rec; ++i) read_emit(P, i, rec_off.data(), used, read_off, read_len, read_cb_off, read_cb_len, read_umi, &out->err);
    out->metrics[0] = met.num_reads; out->metrics[1] = met.num_low_mapq; out->metrics[2] = met.num_non_primary;
    out->metrics[3] = met.num_duplicates; out->metrics[4] = met.num_not_useful;
    return 0;
}

// the shared useful_alignment (vartrix_b200/csrc/vtx_record.cuh) on a minimal record at `pos`: the 32-byte header, a 1-byte
// name and the CIGAR, as the oracle's vtxo_useful_alignment takes them
extern "C" int vtx_test_useful_alignment(int64_t pos, const uint32_t* cigar, int32_t n_cigar, int64_t start, int64_t end)
{
    std::vector<uint8_t> b(33 + 4 * size_t(n_cigar), 0);
    const uint32_t p = uint32_t(int32_t(pos)), nc = uint32_t(n_cigar);
    memcpy(&b[4], &p, 4);                // little-endian host, as the BAM layout
    b[8] = 1;                            // l_read_name: the NUL
    b[12] = uint8_t(nc); b[13] = uint8_t(nc >> 8);
    if (n_cigar) memcpy(&b[33], cigar, 4 * size_t(n_cigar));
    return vtx::stage::useful_alignment(b.data(), start, end) ? 1 : 0;
}
