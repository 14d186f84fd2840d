// vtx_api.cu -- C ABI of the engine (include/vartrix_b200.h): context, device memory, stream
// orchestration of the kernels in vtx_pipeline.cuh / vtx_sw.cuh.  CUDA only -- there is no CPU path.
#include "../../include/vartrix_b200.h"
#include "vtx_pipeline.cuh"
#include "vtx_sw.cuh"
#include "vtx_sw_band.cuh"
#include "vtx_inflate.cuh"
#include "vtx_stage.cuh"
#include "vtx_locus_stats.cuh"
#include "vtx_donors.cuh"
#include "vtx_clusters.cuh"
#include "vtx_ambient.cuh"
#include "vtx_cluster_gt.cuh"
#include "vtx_cluster_refine.cuh"
#include "vtx_cluster_pinned.cuh"

#include <nvtx3/nvToolsExt.h>     // header-only; ranges cost nothing unless a profiler (nsys / ncu --nvtx) is attached

#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

using namespace vtx;

namespace {

thread_local std::string g_create_error;

// NVTX range around a host-side phase of the API (submit: copies / validation / kernel enqueue; finish; gather)
struct Nvtx {
    explicit Nvtx(const char* name) { nvtxRangePushA(name); }
    ~Nvtx() { nvtxRangePop(); }
};
constexpr int kBandK = 6, kBandW = 20;       // K, W of banded::Aligner::new (main.rs:33-34, 899)

// device memory owned by the context: freed with it, grown by ensure()
struct DBuf {
    void* p = nullptr;
    size_t cap = 0;
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    ~DBuf() { release(); }
    cudaError_t release()
    {
        const cudaError_t e = p ? cudaFree(p) : cudaSuccess;
        p = nullptr; cap = 0;
        return e;
    }
    void swap(DBuf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
};

// pinned host memory owned by the context
struct HostBuf {
    void* p = nullptr;
    HostBuf() = default;
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { release(); }
    void release() { if (p) cudaFreeHost(p); p = nullptr; }
    cudaError_t alloc(size_t bytes, unsigned flags = cudaHostAllocDefault)
    {
        release();
        const cudaError_t e = cudaHostAlloc(&p, bytes, flags);
        if (e != cudaSuccess) p = nullptr;
        return e;
    }
    template <typename T> T* as() const { return static_cast<T*>(p); }
};

// The seven triplet arrays of a result, in vtx_result order: row, col, ref_cnt, alt_cnt, unk_cnt, val, val2.
constexpr int kResArrays = 7;
constexpr size_t kResEsz[kResArrays] = { 4, 4, 4, 4, 4, 8, 8 };

struct HostResults {    // pinned host copies of the result arrays, room for `cap` triplets
    HostBuf a[kResArrays];
    size_t cap = 0;
};

enum { EV_START = 0, EV_H2D, EV_C0, EV_PREP, EV_SW, EV_POST, EV_COUNT };

constexpr size_t kMaxCum = 4096;   // submits per finish that can stream their triplets out early

struct TimeRec {   // CUDA events of one submit
    cudaEvent_t ev[EV_COUNT] = {};
    bool had_h2d = false;
    uint64_t sw_launches = 0, launches = 0;
};

// device copies of one staged shard; two slots so that the copy of shard k+1 overlaps the kernels of shard k
struct InSlot {
    DBuf locus_row, hap, ref_off, ref_len, alt_off, alt_len, cand_start, read_nib, read_off, read_len, cb_bytes,
        read_cb_off, read_cb_len, read_umi, cand_read;
    DBuf read_off4, read_len16, read_cb_key, cb_off_ex;     // slim layout (vtx_batch2)
    cudaEvent_t copy_done = nullptr, free_ev = nullptr;
    bool used = false;
};

// device buffers of one shard staged on the device (vtx_submit_bam); two slots: shard k+1 is inflated and scanned while the
// Smith-Waterman kernels of shard k still read shard k's stream
struct StageSlot {
    DBuf comp, desc, status, stream, entry, seg_count, seg_first, rec_off, rec_tid, rec_pos, rec_end, rec_fm, l_start, l_end,
        locus_row, hap, ref_off, ref_len, alt_off, alt_len, cand_count, cand_first, cand_rec, used, read_off, read_len,
        read_cb_off, read_cb_len, read_umi, cand_start, scalars, name_tab, lfilt;
    cudaEvent_t staged = nullptr, free_ev = nullptr;
    bool used_once = false;
};

}  // namespace

struct vtx_ctx {
    vtx_config cfg{};
    int device = 0;
    int n_sm = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;

    // barcode table
    DBuf bc_slot, bc_bytes, bc_off;
    DBuf bck_key, bck_idx;            // the barcodes that have a vtx_pack_cb code, keyed by it
    uint32_t bck_cap = 0;
    DBuf x_read_off, x_read_len, x_units, x_off4;      // slim layout expanded to the internal read arrays
    DBuf band_scratch;                                  // VTX_BAND_MODEL work buffers, one slice per resident warp
    DBuf inf_comp, inf_out, inf_desc, inf_status;       // vtx_bgzf_inflate
    bool inflate_attr_set = false;
    StageSlot sslot[2];                                 // vtx_submit_bam
    uint64_t n_bam_submits = 0;
    cudaStream_t stage_stream = nullptr;
    DBuf bam_metrics;                                   // stage::LocusMetrics, cumulative
    uint32_t min_base_quality = 0;                      // vtx_set_min_base_quality: for every later vtx_submit_bam
    DBuf stage_sums;                                    // block sums of the scans on the staging stream
    // vtx_set_locus_stats: one vtx_locus_stats per locus submitted since the last finish (device), copied out by the finish
    bool locus_stats = false, submitted = false;
    DBuf lstats;
    size_t lstats_cap = 0;                              // entries
    uint64_t stats_n = 0, stats_last_n = 0;             // entries of the running / the last finished result set
    HostBuf h_lstats;
    size_t h_lstats_cap = 0;
    // vtx_set_donors: the dosage table and, per column, H int64 log-likelihoods + 3 counters (then one u64 of rows outside the
    // table), summed over the submits since the last finish; the finish copies them to h_donor
    bool donors = false;
    uint32_t n_donors = 0, donor_cols = 0, donor_last_cols = 0;
    uint64_t donor_rows = 0;
    donors::Tables donor_tab{};
    DBuf donor_dosage, donor_usable, donor_acc, donor_count, donor_start, donor_list;
    HostBuf h_donor;
    size_t h_donor_cap = 0;                             // bytes
    bool donor_valid = false;                           // h_donor holds the last finished result set
    // vtx_cluster_cells: device work buffers and the host outputs of the last call
    DBuf cl_row, cl_col, cl_r, cl_a, cl_used, cl_used_rows, cl_row_start, cl_cell_count, cl_cell_start, cl_c_row, cl_c_r, cl_c_a,
        cl_la, cl_lr, cl_w, cl_flags, cl_A, cl_T, cl_ll, cl_cnt;
    std::vector<int64_t> h_cl_ll, h_cl_A, h_cl_T, h_cl_score;
    std::vector<uint64_t> h_cl_cnt;
    std::vector<uint8_t> h_cl_used;
    std::vector<uint32_t> h_cl_iters;
    // vtx_donors_ambient: device work buffers (the entries and their by-cell index live in the cl_* buffers above) and the
    // host outputs of the last call
    DBuf am_sums, am_tix, am_touched, am_dos, am_tab, am_grid;
    std::vector<int64_t> h_am_ll, h_am_obj;
    std::vector<uint64_t> h_am_cnt, h_am_calls, h_am_alt, h_am_depth;
    std::vector<uint16_t> h_am_m;
    // vtx_cluster_genotypes: device work buffers and the host outputs of the last call
    DBuf cg_AT, cg_rows, cg_fit, cg_ll, cg_gt, cg_pl, cg_cmp, cg_dos, cg_acc;
    std::vector<int64_t> h_cg_obj, h_cg_M;
    std::vector<uint64_t> h_cg_touched, h_cg_acc;
    std::vector<uint16_t> h_cg_m;
    std::vector<uint8_t> h_cg_gt;
    std::vector<uint32_t> h_cg_pl;
    // vtx_cluster_refine: device work buffers (the entries, their indexes, sums, weights and cell outputs live in the cl_* buffers,
    // the row sums in am_sums, the compacted fit in the cg_* buffers) and the host outputs of the last call
    DBuf cr_rowflags, cr_code, cr_sflag, cr_scode, cr_tab, cr_label, cr_scal;
    std::vector<int64_t> h_cr_ll;
    std::vector<uint64_t> h_cr_cnt, h_cr_touched;
    std::vector<uint32_t> h_cr_label, h_cr_pl;
    std::vector<uint8_t> h_cr_gt;
    std::vector<vtx_cluster_calls_round> h_cr_rounds;
    // vtx_cluster_cells_pinned: the pinned samples' dosage (everything else is vtx_cluster_cells', the row sums in am_sums)
    DBuf cp_dos;
    HostBuf h_stage;                                 // scalars read back between the staging phases
    uint32_t bc_cap = 0, n_barcodes = 0;
    bool have_barcodes = false;

    // staged inputs (device copies for vtx_submit): double-buffered, filled on a separate copy stream
    InSlot slot[2];
    uint64_t n_submits = 0;
    cudaStream_t copy_stream = nullptr;
    // work buffers
    DBuf read_col, keep, pidx, scan_sums, pair_read, pair_col, pair_umi, pair_locus, pair_start, tcount, tstart,
        pair_first, pair_cslot, pair_uslot, cslot_col, cslot_locus, uslot_cslot, ccnt, ucnt, keep2, oidx, tile_counters,
        scratch, pair_scores, d_metrics, d_res_n, big_list, slot_scratch;
    // results (device) + host mirrors
    DBuf res[kResArrays];
    size_t res_cap = 0;        // entries
    size_t res_ub = 0;         // upper bound of entries currently held
    bool finished = true;      // true: next submit starts a fresh result set
    HostResults h_res;
    HostBuf h_scalars;         // res_n (u64) + 3 metrics (u64)
    uint64_t last_n = 0;
    vtx_metrics last_metrics{};

    cudaStream_t fetch_stream = nullptr;                 // device->host copies of finished triplets
    HostBuf h_cum;                                       // host-mapped running triplet count after each submit
    unsigned long long* d_cum = nullptr;                 // device alias of h_cum
    std::vector<TimeRec> trecs;     // one per submit since the last finish (events are reused)
    size_t trec_used = 0;
    bool timing_valid = false;
    uint32_t last_tiles_nl = 0;       // loci of the most recent run_sw (vtx_last_tile_counts)
    bool last_tiles_valid = false;
    uint64_t t_pairs = 0;

    // multi-GPU (vtx_comm_init / vtx_gather_start)
    void* comm = nullptr;
    int rank = 0, n_ranks = 1;
    HostResults g_host;
    DBuf g_dev[kResArrays];
    DBuf g_counts;
    cudaStream_t comm_stream = nullptr;          // the gather runs here so that later submits overlap it
    cudaEvent_t ev_counts = nullptr, ev_gather = nullptr, ev_results = nullptr;
    HostBuf h_counts;                            // [n_ranks + 1][4]
    bool gather_pending = false;                 // started, not yet waited for
    bool gather_guard = false;                   // ev_gather must be awaited (on the device) before r_* are overwritten
    vtx_result g_out{};
};

namespace {

int set_err(vtx_ctx* c, int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    if (c) c->err = buf; else g_create_error = buf;
    return code;
}

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return set_err(ctx, VTX_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

int ensure(vtx_ctx* ctx, DBuf& b, size_t bytes)
{
    if (bytes <= b.cap) return VTX_OK;
    if (b.p) {
        CK(cudaStreamSynchronize(ctx->stream));
        if (ctx->copy_stream) CK(cudaStreamSynchronize(ctx->copy_stream));
        CK(b.release());
    }
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) { b.p = nullptr; return set_err(ctx, VTX_E_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); }
    b.cap = want;
    return VTX_OK;
}

#define ENS(buf, bytes) do { int rc_ = ensure(ctx, buf, (bytes)); if (rc_) return rc_; } while (0)

template <typename T> T* P(DBuf& b) { return static_cast<T*>(b.p); }

TimeRec* new_trec(vtx_ctx* ctx)
{
    if (ctx->finished) ctx->trec_used = 0;
    if (ctx->trec_used == ctx->trecs.size()) {
        TimeRec r;
        for (auto& e : r.ev) if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
        ctx->trecs.push_back(r);
    }
    TimeRec* r = &ctx->trecs[ctx->trec_used++];
    r->had_h2d = false; r->sw_launches = 0; r->launches = 0;
    return r;
}

inline unsigned blocks_for(uint64_t n, unsigned threads) { return unsigned((n + threads - 1) / threads); }

// the grid of a grid-stride kernel over `work` threads: at most per_sm CTAs per SM, at least one
inline unsigned grid_for(const vtx_ctx* ctx, uint64_t work, unsigned threads, unsigned per_sm = 16)
{
    return std::max(1u, std::min(blocks_for(work, threads), unsigned(ctx->n_sm) * per_sm));
}

// launch(std::integral_constant<int, KH>{}) for a warp-per-cell kernel over H hypotheses, lane l owning hypotheses l + 32j,
// j < KH: the smallest of the instantiations KH = 1, 2, 5, 9, 17 with 32 KH >= H
template <typename Launch> void by_kh(uint32_t H, Launch launch)
{
    if (H <= 32) launch(std::integral_constant<int, 1>{});
    else if (H <= 64) launch(std::integral_constant<int, 2>{});
    else if (H <= 160) launch(std::integral_constant<int, 5>{});
    else if (H <= 288) launch(std::integral_constant<int, 9>{});
    else launch(std::integral_constant<int, 17>{});
}

// exclusive scan on stream `st` with block sums in `sums`: out has n + 1 entries
int scan_u32(vtx_ctx* ctx, cudaStream_t st, DBuf& sums, const uint32_t* in, uint64_t n, uint32_t* out, uint64_t* launches)
{
    const unsigned nb = std::max(1u, blocks_for(n, kScanTile));
    ENS(sums, size_t(nb) * 4);
    vtx_k_scan_tiles<<<nb, kScanThreads, 0, st>>>(in, n, out, P<uint32_t>(sums));
    vtx_k_scan_sums<<<1, kScanThreads, 0, st>>>(P<uint32_t>(sums), nb, out + n);
    vtx_k_scan_add<<<nb, kScanThreads, 0, st>>>(out, n, P<uint32_t>(sums));
    if (launches) *launches += 3;
    CK(cudaGetLastError());
    return VTX_OK;
}

// one warp per BGZF member; the decoder's tables and input windows need the opt-in shared-memory size
int launch_inflate(vtx_ctx* ctx, cudaStream_t st, const void* desc, uint32_t n, const void* comp, void* out, void* status,
                   uint32_t* cursor, int check_crc)
{
    using namespace inflate;
    if (!ctx->inflate_attr_set) {
        CK(cudaFuncSetAttribute(vtx_k_bgzf_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, int(inflate_smem_bytes())));
        ctx->inflate_attr_set = true;
    }
    const unsigned ctas = unsigned(std::min<uint64_t>((n + kInflateWarps - 1) / kInflateWarps, uint64_t(ctx->n_sm) * 6));
    vtx_k_bgzf_inflate<<<ctas, kInflateWarps * 32, inflate_smem_bytes(), st>>>(static_cast<const BlockDesc*>(desc), n,
        static_cast<const uint8_t*>(comp), static_cast<uint8_t*>(out), static_cast<int32_t*>(status), cursor, check_crc);
    CK(cudaGetLastError());
    return VTX_OK;
}

// the result arrays that travel to the host: VTX_F_VALUES_ONLY keeps the three counts (and val2 outside coverage mode) on the device
uint32_t want_mask(const vtx_ctx* ctx)
{
    const bool values_only = (ctx->cfg.flags & VTX_F_VALUES_ONLY) != 0;
    return values_only ? (ctx->cfg.mode == VTX_MODE_COVERAGE ? 0x63u : 0x23u) : 0x7Fu;
}

template <typename Buf> std::array<const void*, kResArrays> ptrs(const Buf (&b)[kResArrays])
{
    std::array<const void*, kResArrays> a;
    for (int i = 0; i < kResArrays; ++i) a[i] = b[i].p;
    return a;
}

// points `out` at the arrays of `a` that `want` selects (NULL for the others)
void point_result(vtx_result* out, const std::array<const void*, kResArrays>& a, uint32_t want, uint64_t n, const vtx_metrics& m)
{
    auto u32 = [&](int i) { return (want >> i & 1) ? static_cast<const uint32_t*>(a[i]) : nullptr; };
    auto f64 = [&](int i) { return (want >> i & 1) ? static_cast<const double*>(a[i]) : nullptr; };
    out->n = n;
    out->row = u32(0); out->col = u32(1); out->ref_cnt = u32(2); out->alt_cnt = u32(3); out->unk_cnt = u32(4);
    out->val = f64(5); out->val2 = f64(6);
    out->metrics = m;
}

// pinned host result arrays with room for `n` triplets (only the wanted arrays are allocated)
int ensure_host(vtx_ctx* ctx, HostResults& h, size_t n)
{
    if (n <= h.cap) return VTX_OK;
    const size_t ncap = n + n / 4 + 1024;
    const uint32_t want = want_mask(ctx);
    for (int i = 0; i < kResArrays; ++i) {
        h.a[i].release();
        if (!(want >> i & 1)) continue;
        const cudaError_t e = h.a[i].alloc(ncap * kResEsz[i]);
        if (e != cudaSuccess) { h.cap = 0; return set_err(ctx, VTX_E_NOMEM, "pinned result alloc failed: %s", cudaGetErrorString(e)); }
    }
    h.cap = ncap;
    return VTX_OK;
}

// device->host copy of entries [from, to) of the wanted result arrays
int copy_results(vtx_ctx* ctx, HostResults& h, const std::array<const void*, kResArrays>& src, size_t from, size_t to, cudaStream_t st)
{
    const uint32_t want = want_mask(ctx);
    for (int i = 0; i < kResArrays; ++i)
        if ((want >> i & 1) && src[i])
            CK(cudaMemcpyAsync(h.a[i].as<uint8_t>() + from * kResEsz[i], static_cast<const uint8_t*>(src[i]) + from * kResEsz[i],
                               (to - from) * kResEsz[i], cudaMemcpyDeviceToHost, st));
    return VTX_OK;
}

struct DevBatch {   // device pointers
    uint32_t n_loci = 0; uint32_t n_reads = 0; uint64_t n_cand = 0;
    const uint32_t* locus_row; const uint8_t* hap; const uint32_t *ref_off, *ref_len, *alt_off, *alt_len;
    const uint64_t* cand_start; const uint8_t* read_nib; const uint64_t* read_off; const uint32_t* read_len;
    const uint8_t* cb_bytes; const uint32_t* read_cb_off; const uint16_t* read_cb_len; const uint64_t* read_umi;
    const uint32_t* cand_read;       // nullptr: candidate c is read c
    // slim layout: cell tags as codes (then cb_bytes / cb_off_ex hold the exotic tags only)
    const uint64_t* read_cb_key = nullptr; const uint32_t* cb_off_ex = nullptr;
    bool have_shapes = false;        // host batches: `shapes` holds the shape keys of the loci (scan_host_batch)
    uint64_t shapes = 0;
    uint32_t max_read_len = 0, max_hap_len = 0;
    uint64_t max_depth = ~0ull;      // most candidates of one locus (unknown for device batches: assume deep)
    const uint32_t* lfilt = nullptr; // [n_loci][stage::kNumCounters] record-filter counters of a vtx_submit_bam shard (vtx_set_locus_stats)
};

// A persistent grid of a Smith-Waterman kernel: as many blocks as fit on every SM at once, each warp taking tiles from
// a.tile_counter until none are left.  `name` / `cls` (-1: none) name the kernel in the error message.
int launch_sw(vtx_ctx* ctx, void (*kern)(SwArgs), int threads, size_t smem, const SwArgs& a, uint64_t* launches,
              const char* name, int cls)
{
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) {
        if (cls < 0) return set_err(ctx, VTX_E_CUDA, "%s does not fit on an SM (smem %zu)", name, smem);
        return set_err(ctx, VTX_E_CUDA, "%s %d does not fit on an SM (smem %zu)", name, cls, smem);
    }
    kern<<<ctx->n_sm * per_sm, threads, smem, ctx->stream>>>(a);
    CK(cudaGetLastError());
    ++*launches;
    return VTX_OK;
}

template <int CLS> int launch_sw_class(vtx_ctx* ctx, const SwArgs& a, uint64_t* launches)
{
    return launch_sw(ctx, vtx_k_sw_pairs<CLS>, TileClass<CLS>::THREADS,
                     sw_warp_bytes<CLS>(a.mcap, a.multi) * (TileClass<CLS>::THREADS / 32), a, launches,
                     "SW kernel class", CLS);
}
template <int SCLS> int launch_sw_split(vtx_ctx* ctx, const SwArgs& a, uint64_t* launches)
{
    return launch_sw(ctx, vtx_k_sw_split<SCLS>, SplitClass<SCLS>::THREADS,
                     split_warp_bytes<SCLS>(a.mcap) * (SplitClass<SCLS>::THREADS / 32), a, launches,
                     "split SW kernel", SCLS);
}
template <int W, int S, bool SHARED> int launch_sw_fold(vtx_ctx* ctx, const SwArgs& a, uint64_t* launches)
{
    return launch_sw(ctx, vtx_k_sw_fold<W, S, SHARED>, W * 32, fold_cta_bytes<W, S>(), a, launches, "folded SW kernel", -1);
}

// classes + tiles + SW kernels, shared by submit and score_pairs.  pair_start must be ready.
int run_sw(vtx_ctx* ctx, const DevBatch& b, uint32_t n_pairs_ub, const uint32_t* pair_slot, uint32_t* counters,
           uint32_t* pair_scores, uint64_t* launches, uint64_t* sw_launches, TimeRec* tr)
{
    const uint32_t nl = b.n_loci;
    ENS(ctx->tcount, size_t(kNumClasses) * (nl + 1) * 4);
    ENS(ctx->tstart, size_t(kNumClasses) * (nl + 1) * 4);
    ENS(ctx->tile_counters, 64);
    const SwAllow allow = allowed_kernels(ctx->cfg.flags, b.max_read_len, b.max_hap_len);
    vtx_k_locus_prep<<<blocks_for(uint64_t(nl) * 32, 256), 256, 0, ctx->stream>>>(
        nl, b.hap, b.ref_off, b.ref_len, b.alt_off, b.alt_len, P<uint32_t>(ctx->pair_start), P<uint32_t>(ctx->pair_read), b.read_len,
        allow, b.max_read_len, b.max_hap_len, P<unsigned long long>(ctx->d_metrics) + 4, P<uint32_t>(ctx->tcount));
    ++*launches;
    vtx_k_scan_rows<<<kNumClasses, kScanThreads, 0, ctx->stream>>>(P<uint32_t>(ctx->tcount), P<uint32_t>(ctx->tstart), nl, nl + 1);
    ++*launches;
    CK(cudaGetLastError());
    CK(cudaMemsetAsync(ctx->tile_counters.p, 0, 64, ctx->stream));
    ctx->last_tiles_nl = nl;
    ctx->last_tiles_valid = true;
    if (tr) CK(cudaEventRecord(tr->ev[EV_PREP], ctx->stream));

    SwArgs a{};
    a.hap_bytes = b.hap; a.ref_off = b.ref_off; a.ref_len = b.ref_len; a.alt_off = b.alt_off; a.alt_len = b.alt_len;
    a.read_nib = b.read_nib; a.read_off = b.read_off; a.read_len = b.read_len;
    a.pair_read = P<uint32_t>(ctx->pair_read); a.pair_start = P<uint32_t>(ctx->pair_start);
    a.n_loci = nl; a.pair_slot = pair_slot; a.counters = counters; a.pair_scores = pair_scores;
    a.min_score = ctx->cfg.min_score;
    int mcap = int(std::min<uint32_t>(b.max_read_len, kFastMaxRead));
    mcap = std::max(2, (mcap + 1) & ~1);
    a.mcap = mcap;
    a.k64k = 65536u;
    a.multi = allow.multi;
    a.max_hap = b.max_hap_len;

    uint64_t before = *launches;
    if (ctx->cfg.band_mode == VTX_BAND_MODEL) {
        // optional slow path: every pair scored inside the k-mer-chain band model, one warp per pair (vtx_sw_band.cuh)
        BandArgs ba{};
        ba.sw = a; ba.n_pairs_ub = n_pairs_ub; ba.k = ctx->cfg.band_k; ba.w = ctx->cfg.band_w;
        ba.max_read = std::max<uint32_t>(b.max_read_len, 8); ba.max_hap = std::max<uint32_t>(b.max_hap_len, 8);
        const uint64_t all_hits = uint64_t(ba.max_read) * ba.max_hap;          // every position pair can be a hit at most
        ba.hit_cap = uint32_t(std::min<uint64_t>(all_hits, uint64_t(1) << 20));
        ba.hit_cap = std::min<uint32_t>(ba.hit_cap, 65535u * 16u);
        const size_t wb = band_warp_bytes(ba.max_read, ba.max_hap, ba.hit_cap);
        size_t warps = size_t(ctx->n_sm) * 16;
        const size_t budget = size_t(4) << 30;                                  // scratch budget: 4 GiB
        if (warps * wb > budget) warps = std::max<size_t>(size_t(ctx->n_sm), budget / wb);
        warps = std::max<size_t>(warps & ~size_t(3), 4);
        ENS(ctx->band_scratch, warps * wb);
        ba.scratch = P<uint8_t>(ctx->band_scratch);
        if (ba.max_hap >= 65536u || ba.max_read >= 65536u) return set_err(ctx, VTX_E_UNSUPPORTED, "band model: reads and windows must be shorter than 65536");
        ba.overflow = P<unsigned long long>(ctx->d_metrics) + 5;
        ba.bounds_violated = P<unsigned long long>(ctx->d_metrics) + 4;
        ba.cursor = P<uint32_t>(ctx->tile_counters);
        vtx_k_sw_band<<<unsigned(warps / (kBandThreads / 32)), kBandThreads, 0, ctx->stream>>>(ba);
        CK(cudaGetLastError());
        ++*launches;
        *sw_launches += *launches - before;
        return VTX_OK;
    }
    // the kernels of the classes that can get tiles: from the loci's shapes when the host has seen them
    const uint32_t mask = b.have_shapes ? host_class_mask(b.shapes, allow, b.max_read_len) : device_class_mask(allow, b.max_hap_len);
    for (int c = 0; c < kNumClasses; ++c) {
        if (!(mask >> c & 1u)) continue;
        a.tile_start = P<uint32_t>(ctx->tstart) + size_t(c) * (nl + 1);
        a.tile_counter = P<uint32_t>(ctx->tile_counters) + c;
        int rc = VTX_OK;
        switch (c) {
        case 0: rc = launch_sw_class<0>(ctx, a, launches); break;
        case 1: rc = launch_sw_class<1>(ctx, a, launches); break;
        case 2: rc = launch_sw_class<2>(ctx, a, launches); break;
        case 3: rc = launch_sw_class<3>(ctx, a, launches); break;
        case kSlowClass: {
            const unsigned blocks = unsigned(ctx->n_sm) * 4, threads = 128;
            const size_t warps = size_t(blocks) * threads / 32;
            ENS(ctx->scratch, warps * (size_t(b.max_hap_len) + 1) * 32 * 4);
            a.scratch = P<uint32_t>(ctx->scratch);
            vtx_k_sw_generic<<<blocks, threads, 0, ctx->stream>>>(a);
            CK(cudaGetLastError());
            ++*launches;
            break;
        }
        case kSplitClass0: rc = launch_sw_split<0>(ctx, a, launches); break;
        case kSplitClass0 + 1: rc = launch_sw_split<1>(ctx, a, launches); break;
        case kFoldClass: {
            // the depth is taken over all candidates and loci of the shard, which the host knows for host and device
            // batches alike, not over fold tiles: shallow fold loci in a shard of deep loci of other kernels run the deep
            // shape, which is slower on 1-tile loci but still exact
            const bool deep = uint64_t(n_pairs_ub) >= uint64_t(kFoldDeepDepth) * nl;
            rc = deep ? launch_sw_fold<kFoldDeepWarps, kFoldDeepSlots, true>(ctx, a, launches)
                      : launch_sw_fold<kFoldShallowWarps, kFoldShallowWarps, false>(ctx, a, launches);
            break;
        }
        }
        if (rc) return rc;
    }
    *sw_launches += *launches - before;
    return VTX_OK;
}

int grow_results(vtx_ctx* ctx, size_t need)
{
    if (need <= ctx->res_cap) return VTX_OK;
    const size_t ncap = need + need / 4 + 1024;
    for (int i = 0; i < kResArrays; ++i) {
        DBuf& b = ctx->res[i];
        DBuf nb;
        cudaError_t e = cudaMalloc(&nb.p, ncap * kResEsz[i]);
        if (e != cudaSuccess) { nb.p = nullptr; return set_err(ctx, VTX_E_NOMEM, "result cudaMalloc(%zu) failed: %s", ncap * kResEsz[i], cudaGetErrorString(e)); }
        nb.cap = ncap * kResEsz[i];
        if (b.p && ctx->res_ub && !ctx->finished)
            CK(cudaMemcpyAsync(nb.p, b.p, ctx->res_ub * kResEsz[i], cudaMemcpyDeviceToDevice, ctx->stream));
        if (b.p) {
            CK(cudaStreamSynchronize(ctx->stream));
            if (ctx->fetch_stream) CK(cudaStreamSynchronize(ctx->fetch_stream));
            if (ctx->comm_stream) CK(cudaStreamSynchronize(ctx->comm_stream));
            CK(b.release());
        }
        b.swap(nb);
    }
    ctx->res_cap = ncap;
    return VTX_OK;
}

static_assert(sizeof(vtx_locus_stats) == sizeof(uint32_t) * lstats::kFields, "vtx_locus_stats is the kernel's record");

// room for `need` entries of locus statistics; the running entries move along
int grow_stats(vtx_ctx* ctx, size_t need)
{
    if (need <= ctx->lstats_cap) return VTX_OK;
    const size_t ncap = need + need / 2 + 1024;
    DBuf nb;
    const cudaError_t e = cudaMalloc(&nb.p, ncap * sizeof(vtx_locus_stats));
    if (e != cudaSuccess) { nb.p = nullptr; return set_err(ctx, VTX_E_NOMEM, "locus statistics cudaMalloc failed: %s", cudaGetErrorString(e)); }
    nb.cap = ncap * sizeof(vtx_locus_stats);
    if (ctx->lstats.p) {
        if (ctx->stats_n) CK(cudaMemcpyAsync(nb.p, ctx->lstats.p, ctx->stats_n * sizeof(vtx_locus_stats), cudaMemcpyDeviceToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(ctx->lstats.release());
    }
    ctx->lstats.swap(nb);
    ctx->lstats_cap = ncap;
    return VTX_OK;
}

// the per-locus reduction of this shard (vtx_locus_stats.cuh) into entries [stats_n, stats_n + n_loci); after the UMI collapse
int launch_locus_stats(vtx_ctx* ctx, const DevBatch& b, bool have_pairs, uint64_t* launches)
{
    const int use_umi = ctx->cfg.use_umi ? 1 : 0;
    lstats::Inputs in{ b.cand_start, b.cand_read, P<int32_t>(ctx->read_col), use_umi ? b.read_umi : nullptr,
                       have_pairs ? P<uint32_t>(ctx->pair_start) : nullptr, use_umi ? P<uint32_t>(ctx->ucnt) : nullptr,
                       P<uint32_t>(ctx->ccnt), P<uint32_t>(ctx->cslot_col), b.locus_row, b.lfilt };
    const unsigned grid = std::min<unsigned>(b.n_loci, unsigned(ctx->n_sm) * 16);
    lstats::vtx_k_locus_stats<<<grid, lstats::kStatsThreads, 0, ctx->stream>>>(in, b.n_loci, P<uint32_t>(ctx->lstats) + ctx->stats_n * lstats::kFields);
    CK(cudaGetLastError());
    ctx->stats_n += b.n_loci;
    ++*launches;
    return VTX_OK;
}

// the donor accumulator of `cols` columns: H int64 log-likelihoods per column, then 3 u64 counters per column, then the count
// of loci whose row lies outside the dosage table
size_t donor_acc_bytes(uint32_t cols, uint32_t n_hyp) { return size_t(cols) * (size_t(n_hyp) + 3) * 8 + 8; }

// vtx_donors.cuh on this shard's cell slots (slot indices < n_slots_ub, *n_slots of them); after the UMI collapse
int launch_donors(vtx_ctx* ctx, const DevBatch& b, uint32_t n_slots_ub, const uint32_t* n_slots, uint64_t* launches)
{
    using namespace donors;
    cudaStream_t st = ctx->stream;
    const uint32_t H = n_hyp(ctx->n_donors), nc = ctx->donor_cols;
    Inputs in{ P<uint32_t>(ctx->cslot_col), P<uint32_t>(ctx->cslot_locus), b.locus_row, P<uint32_t>(ctx->ccnt),
               P<uint8_t>(ctx->donor_dosage), P<uint8_t>(ctx->donor_usable), ctx->donor_rows, nc, ctx->n_donors, H, ctx->donor_tab };
    int64_t* ll = P<int64_t>(ctx->donor_acc);
    uint64_t* cnt = reinterpret_cast<uint64_t*>(ll + size_t(nc) * H);
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(cnt + size_t(nc) * 3);
    const unsigned grid = grid_for(ctx, std::max<uint64_t>(n_slots_ub, b.n_loci), kDonorThreads);
    ENS(ctx->donor_count, (size_t(nc) + 1) * 4);
    CK(cudaMemsetAsync(ctx->donor_count.p, 0, size_t(nc) * 4, st));
    vtx_k_donor_count<<<grid, kDonorThreads, 0, st>>>(in, n_slots_ub, n_slots, b.n_loci, P<uint32_t>(ctx->donor_count), bad);
    CK(cudaGetLastError());
    ++*launches;
    if (!n_slots) return VTX_OK;
    ENS(ctx->donor_start, (size_t(nc) + 1) * 4);
    ENS(ctx->donor_list, size_t(n_slots_ub) * 4 + 4);
    int rc = scan_u32(ctx, st, ctx->scan_sums, P<uint32_t>(ctx->donor_count), nc, P<uint32_t>(ctx->donor_start), launches);
    if (rc) return rc;
    CK(cudaMemsetAsync(ctx->donor_count.p, 0, size_t(nc) * 4, st));
    vtx_k_donor_scatter<<<grid, kDonorThreads, 0, st>>>(in, n_slots_ub, n_slots, P<uint32_t>(ctx->donor_start),
                                                        P<uint32_t>(ctx->donor_count), P<uint32_t>(ctx->donor_list));
    // one warp per column
    const unsigned ll_grid = grid_for(ctx, uint64_t(nc) * 32, kDonorThreads, 8);
    const uint32_t* cs = P<uint32_t>(ctx->donor_start);
    const uint32_t* lst = P<uint32_t>(ctx->donor_list);
    by_kh(H, [&](auto kh) { vtx_k_donor_ll<decltype(kh)::value><<<ll_grid, kDonorThreads, 0, st>>>(in, cs, lst, ll, cnt); });
    CK(cudaGetLastError());
    *launches += 2;
    return VTX_OK;
}

int process_batch(vtx_ctx* ctx, const DevBatch& b, TimeRec* tr)
{
    const uint64_t nc = b.n_cand;
    const uint32_t nl = b.n_loci, nr = b.n_reads;
    const int use_umi = ctx->cfg.use_umi ? 1 : 0;
    uint64_t launches = 0, sw_launches = 0;
    cudaStream_t st = ctx->stream;

    if (ctx->finished) {      // fresh result set
        CK(cudaMemsetAsync(ctx->d_res_n.p, 0, 8, st));
        CK(cudaMemsetAsync(ctx->d_metrics.p, 0, 48, st));
        ctx->res_ub = 0;
        ctx->stats_n = 0;
        if (ctx->donors) {
            ctx->donor_cols = ctx->n_barcodes;
            const size_t bytes = donor_acc_bytes(ctx->donor_cols, donors::n_hyp(ctx->n_donors));
            ENS(ctx->donor_acc, bytes);
            CK(cudaMemsetAsync(ctx->donor_acc.p, 0, bytes, st));
        }
        ctx->finished = false;
    }
    int rc = grow_results(ctx, ctx->res_ub + nc);
    if (rc) return rc;
    const bool stats = ctx->locus_stats && nl > 0;
    if (stats && (rc = grow_stats(ctx, ctx->stats_n + nl))) return rc;
    const bool donor = ctx->donors && nl > 0;

    const size_t ncp = size_t(nc) + 1;
    ENS(ctx->read_col, size_t(nr ? nr : 1) * 4);
    ENS(ctx->keep, ncp * 4); ENS(ctx->pidx, ncp * 4);
    ENS(ctx->pair_read, ncp * 4); ENS(ctx->pair_col, ncp * 4);
    if (use_umi) ENS(ctx->pair_umi, ncp * 8);
    ENS(ctx->pair_start, size_t(nl + 1) * 4);
    ENS(ctx->pair_first, ncp);
    ENS(ctx->pair_cslot, ncp * 4); ENS(ctx->cslot_col, ncp * 4); ENS(ctx->cslot_locus, ncp * 4);
    ENS(ctx->ccnt, ncp * 16);
    if (use_umi) { ENS(ctx->pair_uslot, ncp * 4); ENS(ctx->uslot_cslot, ncp * 4); ENS(ctx->ucnt, ncp * 16); }
    ENS(ctx->keep2, ncp * 4); ENS(ctx->oidx, ncp * 4);
    uint32_t* pair_scores = nullptr;
    if (ctx->cfg.flags & VTX_F_KEEP_SCORES) { ENS(ctx->pair_scores, ncp * 4); pair_scores = P<uint32_t>(ctx->pair_scores); }

    if (nl == 0 || nc == 0) {
        if (ctx->d_cum && ctx->trec_used - 1 < kMaxCum)     // an empty shard still publishes the running triplet count
            vtx_k_bump<<<1, 32, 0, st>>>(P<unsigned long long>(ctx->d_res_n), nullptr, ctx->d_cum + (ctx->trec_used - 1));
        CK(cudaEventRecord(tr->ev[EV_PREP], st)); CK(cudaEventRecord(tr->ev[EV_SW], st));
        if (stats) {          // loci without candidates still get their entries (the record-filter counters, zeros elsewhere)
            if ((rc = launch_locus_stats(ctx, b, false, &launches))) return rc;
            tr->launches = launches;
        }
        if (donor) {          // no slots, but the loci's rows are still checked against the table
            if ((rc = launch_donors(ctx, b, 0, nullptr, &launches))) return rc;
            tr->launches = launches;
        }
        CK(cudaEventRecord(tr->ev[EV_POST], st));
        ctx->timing_valid = true;
        return VTX_OK;
    }

    Nvtx r_prep("vtx: prep kernels (CB lookup, filter, compaction, slots)");
    // ---- K1: CB lookup, filter, compaction --------------------------------------------------------
    BarcodeTable tab{ P<int32_t>(ctx->bc_slot), ctx->bc_cap - 1, P<uint8_t>(ctx->bc_bytes), P<uint32_t>(ctx->bc_off) };
    if (b.read_cb_key) {
        BarcodeKeyTable kt{ P<uint64_t>(ctx->bck_key), P<uint32_t>(ctx->bck_idx), ctx->bck_cap - 1 };
        vtx_k_cb_lookup_key<<<blocks_for(nr, 256), 256, 0, st>>>(tab, kt, nr, b.read_cb_key, b.cb_bytes, b.cb_off_ex, P<int32_t>(ctx->read_col));
    } else {
        vtx_k_cb_lookup<<<blocks_for(nr, 256), 256, 0, st>>>(tab, nr, b.cb_bytes, b.read_cb_off, b.read_cb_len, P<int32_t>(ctx->read_col));
    }
    vtx_k_cand_filter<<<blocks_for(nc, 256), 256, 0, st>>>(nc, b.cand_read, P<int32_t>(ctx->read_col), b.read_umi, use_umi,
                                                           P<uint32_t>(ctx->keep), P<unsigned long long>(ctx->d_metrics));
    launches += 2;
    rc = scan_u32(ctx, st, ctx->scan_sums, P<uint32_t>(ctx->keep), nc, P<uint32_t>(ctx->pidx), &launches);
    if (rc) return rc;
    vtx_k_compact<<<blocks_for(nc, 256), 256, 0, st>>>(nc, b.cand_read, P<uint32_t>(ctx->keep), P<uint32_t>(ctx->pidx),
                                                       P<int32_t>(ctx->read_col), b.read_umi, use_umi, P<uint32_t>(ctx->pair_read),
                                                       P<uint32_t>(ctx->pair_col), P<uint64_t>(ctx->pair_umi));
    vtx_k_pair_start<<<blocks_for(nl + 1, 256), 256, 0, st>>>(nl, b.cand_start, P<uint32_t>(ctx->pidx), P<uint32_t>(ctx->pair_start));
    launches += 2;
    const uint32_t* n_pairs_ptr = P<uint32_t>(ctx->pidx) + nc;

    // ---- slots: the (row, col[, umi]) structure is independent of the alignment results ----------
    ENS(ctx->big_list, size_t(nc / kSlotSmallMax + 2) * 4);
    CK(cudaMemsetAsync(ctx->big_list.p, 0, 4, st));
    if (b.max_depth > kSlotSmallMax) ENS(ctx->slot_scratch, size_t(kSlotBigWords) * nc * 4);
    CK(cudaMemsetAsync(ctx->cslot_col.p, 0xFF, size_t(nc) * 4, st));
    CK(cudaMemsetAsync(ctx->ccnt.p, 0, size_t(nc) * 16, st));
    if (use_umi) {
        CK(cudaMemsetAsync(ctx->uslot_cslot.p, 0xFF, size_t(nc) * 4, st));
        CK(cudaMemsetAsync(ctx->ucnt.p, 0, size_t(nc) * 16, st));
    }
    vtx_k_slots<<<std::min<uint32_t>(nl, 65535u * 8), kSlotThreads, 0, st>>>(
        nl, P<uint32_t>(ctx->pair_start), P<uint32_t>(ctx->pair_col), P<uint64_t>(ctx->pair_umi), use_umi,
        P<uint8_t>(ctx->pair_first), P<uint32_t>(ctx->pair_cslot), P<uint32_t>(ctx->pair_uslot),
        P<uint32_t>(ctx->cslot_col), P<uint32_t>(ctx->cslot_locus), P<uint32_t>(ctx->uslot_cslot), P<uint32_t>(ctx->big_list));
    ++launches;
    if (nc > kSlotSmallMax) {       // a locus deeper than kSlotSmallMax pairs can only exist in such a shard
        vtx_k_slots_big<<<ctx->n_sm, kSlotBigThreads, 0, st>>>(
            P<uint32_t>(ctx->big_list), P<uint32_t>(ctx->pair_start), P<uint32_t>(ctx->pair_col), P<uint64_t>(ctx->pair_umi), use_umi,
            P<uint32_t>(ctx->slot_scratch), P<uint32_t>(ctx->pair_cslot), P<uint32_t>(ctx->pair_uslot), P<uint32_t>(ctx->cslot_col),
            P<uint32_t>(ctx->cslot_locus), P<uint32_t>(ctx->uslot_cslot));
        ++launches;
    }
    CK(cudaGetLastError());

    // ---- K2 + K3: Smith-Waterman, call, atomic scatter ----------------------------------------------
    nvtxRangePop(); nvtxRangePushA("vtx: Smith-Waterman kernels");
    rc = run_sw(ctx, b, uint32_t(nc), use_umi ? P<uint32_t>(ctx->pair_uslot) : P<uint32_t>(ctx->pair_cslot),
                use_umi ? P<uint32_t>(ctx->ucnt) : P<uint32_t>(ctx->ccnt), pair_scores, &launches, &sw_launches, tr);
    if (rc) return rc;
    CK(cudaEventRecord(tr->ev[EV_SW], st));

    // ---- K4 + K5: UMI collapse, mode value, row-major emit ------------------------------------------
    nvtxRangePop(); nvtxRangePushA("vtx: post kernels (UMI collapse, finalize, emit)");
    if (use_umi) {
        vtx_k_umi_collapse<<<blocks_for(nc, 256), 256, 0, st>>>(uint32_t(nc), n_pairs_ptr, P<uint32_t>(ctx->uslot_cslot),
                                                                P<uint32_t>(ctx->ucnt), P<uint32_t>(ctx->ccnt));
        ++launches;
    }
    if (stats && (rc = launch_locus_stats(ctx, b, true, &launches))) return rc;
    if (donor && (rc = launch_donors(ctx, b, uint32_t(nc), n_pairs_ptr, &launches))) return rc;
    vtx_k_finalize<<<blocks_for(nc, 256), 256, 0, st>>>(uint32_t(nc), n_pairs_ptr, ctx->cfg.mode, P<uint32_t>(ctx->cslot_col),
                                                        P<uint32_t>(ctx->ccnt), P<uint32_t>(ctx->keep2));
    ++launches;
    rc = scan_u32(ctx, st, ctx->scan_sums, P<uint32_t>(ctx->keep2), nc, P<uint32_t>(ctx->oidx), &launches);
    if (rc) return rc;
    if (ctx->gather_guard) {       // a gather started after the previous finish may still be reading the local result arrays
        CK(cudaStreamWaitEvent(st, ctx->ev_gather, 0));
        ctx->gather_guard = false;
    }
    ResultArrays out{ P<uint32_t>(ctx->res[0]), P<uint32_t>(ctx->res[1]), P<uint32_t>(ctx->res[2]), P<uint32_t>(ctx->res[3]),
                      P<uint32_t>(ctx->res[4]), P<double>(ctx->res[5]), P<double>(ctx->res[6]) };
    vtx_k_emit<<<blocks_for(nc, 256), 256, 0, st>>>(uint32_t(nc), ctx->cfg.mode, P<uint32_t>(ctx->keep2), P<uint32_t>(ctx->oidx),
                                                    P<unsigned long long>(ctx->d_res_n), P<uint32_t>(ctx->cslot_col),
                                                    P<uint32_t>(ctx->cslot_locus), b.locus_row, P<uint32_t>(ctx->ccnt), out);
    const size_t sub_idx = ctx->trec_used - 1;       // this submit's slot
    vtx_k_bump<<<1, 32, 0, st>>>(P<unsigned long long>(ctx->d_res_n), P<uint32_t>(ctx->oidx) + nc,
                                 (ctx->d_cum && sub_idx < kMaxCum) ? ctx->d_cum + sub_idx : nullptr);
    launches += 2;
    CK(cudaGetLastError());
    CK(cudaEventRecord(tr->ev[EV_POST], st));
    ctx->res_ub += nc;
    ctx->timing_valid = true;
    tr->sw_launches = sw_launches;
    tr->launches = launches;
    return VTX_OK;
}

// One view of a batch, whichever layout it arrived in.  Building it reads no array, so it serves host and device batches.
struct BatchView {
    uint32_t n_loci = 0, n_reads = 0; uint64_t n_cand = 0;
    const uint32_t *locus_row = nullptr, *ref_off = nullptr, *ref_len = nullptr, *alt_off = nullptr, *alt_len = nullptr;
    const uint64_t* cand_start = nullptr; const uint8_t* hap = nullptr; uint64_t hap_len = 0;
    const uint8_t* read_nib = nullptr; uint64_t nib_len = 0; const uint8_t* cb_bytes = nullptr; uint64_t cb_bytes_len = 0;   // cb_bytes_len: vtx_batch
    const uint64_t* read_off = nullptr; const uint32_t* read_len = nullptr; const uint32_t* cb_off = nullptr; const uint16_t* cb_len = nullptr;   // vtx_batch
    const uint32_t* read_off4 = nullptr; const uint16_t* read_len16 = nullptr; const uint64_t* cb_key = nullptr;                                // vtx_batch2
    uint32_t n_exotic = 0; const uint32_t* cb_off_ex = nullptr;
    const uint64_t* umi = nullptr; const uint32_t* cand_read = nullptr;
    bool v2 = false;
};

BatchView view_of(const vtx_batch* b)
{
    BatchView v;
    v.n_loci = b->n_loci; v.n_reads = b->n_reads; v.n_cand = b->n_cand;
    v.locus_row = b->locus_row; v.ref_off = b->ref_off; v.ref_len = b->ref_len; v.alt_off = b->alt_off; v.alt_len = b->alt_len;
    v.cand_start = b->cand_start; v.hap = b->hap_bytes; v.hap_len = b->hap_bytes_len;
    v.read_nib = b->read_nib; v.nib_len = b->read_nib_len; v.cb_bytes = b->cb_bytes; v.cb_bytes_len = b->cb_bytes_len;
    v.read_off = b->read_off; v.read_len = b->read_len; v.cb_off = b->read_cb_off; v.cb_len = b->read_cb_len;
    v.umi = b->read_umi_key; v.cand_read = b->cand_read;
    return v;
}
BatchView view_of(const vtx_batch2* b)
{
    BatchView v;
    v.v2 = true;
    v.n_loci = b->n_loci; v.n_reads = b->n_reads; v.n_cand = b->n_cand;
    v.locus_row = b->locus_row; v.ref_off = b->ref_off; v.ref_len = b->ref_len; v.alt_off = b->alt_off; v.alt_len = b->alt_len;
    v.cand_start = b->cand_start; v.hap = b->hap_bytes; v.hap_len = b->hap_bytes_len;
    v.read_nib = b->read_nib; v.nib_len = b->read_nib_len; v.cb_bytes = b->cb_bytes;
    v.read_off4 = b->read_off4; v.read_len16 = b->read_len; v.cb_key = b->read_cb_key; v.n_exotic = b->n_exotic_cb; v.cb_off_ex = b->cb_off;
    v.umi = b->read_umi_key; v.cand_read = b->cand_read;
    return v;
}

// the kernels' view of a batch whose arrays are on the device (the slim layout's read arrays come from expand_reads)
DevBatch dev_batch_of(const BatchView& v, uint32_t max_read_len, uint32_t max_hap_len)
{
    DevBatch d{};
    d.n_loci = v.n_loci; d.n_reads = v.n_reads; d.n_cand = v.n_cand;
    d.locus_row = v.locus_row; d.hap = v.hap; d.ref_off = v.ref_off; d.ref_len = v.ref_len; d.alt_off = v.alt_off; d.alt_len = v.alt_len;
    d.cand_start = v.cand_start; d.read_nib = v.read_nib; d.cb_bytes = v.cb_bytes;
    d.read_off = v.read_off; d.read_len = v.read_len; d.read_cb_off = v.cb_off; d.read_cb_len = v.cb_len;
    d.read_cb_key = v.cb_key; d.cb_off_ex = v.cb_off_ex;
    d.read_umi = v.umi; d.cand_read = v.cand_read;
    d.max_read_len = max_read_len; d.max_hap_len = max_hap_len;
    return d;
}

int validate_batch(vtx_ctx* ctx, const BatchView& b)
{
    if (b.n_cand >= 0xFFFFFFF0ull) return set_err(ctx, VTX_E_INVALID, "n_cand %llu exceeds 2^32 per shard; split the shard", (unsigned long long)b.n_cand);
    if (b.n_loci && (!b.locus_row || !b.ref_off || !b.ref_len || !b.alt_off || !b.alt_len || !b.cand_start))
        return set_err(ctx, VTX_E_INVALID, "locus arrays missing");
    if (b.n_reads) {
        const bool reads_ok = b.v2 ? (b.read_len16 && b.cb_key) : (b.read_off && b.read_len && b.cb_off && b.cb_len);
        if (!reads_ok || (!b.umi && ctx->cfg.use_umi)) return set_err(ctx, VTX_E_INVALID, "read arrays missing");
    }
    if (b.v2 && b.n_exotic && !b.cb_off_ex) return set_err(ctx, VTX_E_INVALID, "cb_off missing for the exotic cell tags");
    if (b.n_cand && !b.cand_read && !(b.v2 && b.n_cand == b.n_reads)) return set_err(ctx, VTX_E_INVALID, "cand_read missing (NULL means identity and needs n_cand == n_reads in a vtx_batch2)");
    if (b.hap_len >= 0xFFFFFFFFull) return set_err(ctx, VTX_E_INVALID, "haplotype pool exceeds 4 GiB; split the shard");
    if (b.v2 && b.nib_len >= (uint64_t(1) << 34)) return set_err(ctx, VTX_E_INVALID, "read pool exceeds 16 GiB; split the shard");
    return VTX_OK;
}

// host-side checks that need to touch the (host) arrays; also returns max lengths.  Runs on a few host
// threads while the shard's H2D copies are already in flight (the kernels are only enqueued afterwards).
int scan_host_batch(vtx_ctx* ctx, const BatchView& b, uint32_t* max_read, uint32_t* max_hap, bool check_cands,
                    uint64_t* max_depth = nullptr, uint64_t* shapes_seen = nullptr)
{
    if (check_cands && b.n_loci && (b.cand_start[0] != 0 || b.cand_start[b.n_loci] != b.n_cand))
        return set_err(ctx, VTX_E_INVALID, "cand_start must span [0, n_cand]");
    if (check_cands && !b.n_loci && b.n_cand) return set_err(ctx, VTX_E_INVALID, "candidates without loci");
    if (b.v2 && b.n_exotic) {
        for (uint32_t i = 0; i < b.n_exotic; ++i)
            if (b.cb_off_ex[i] > b.cb_off_ex[i + 1]) return set_err(ctx, VTX_E_INVALID, "cb_off must be ascending (exotic tag %u)", i);
    }
    const bool scan_cands = check_cands && b.cand_read != nullptr;
    const uint64_t work = uint64_t(b.n_reads) + (scan_cands ? b.n_cand : 0) + uint64_t(b.n_loci) * 64;
    unsigned nt = std::min<unsigned>(8u, std::max(1u, std::thread::hardware_concurrency()));
    if (work < (1u << 16)) nt = 1;
    struct Part { uint32_t mr = 0, mh = 0; uint64_t md = 0, units = 0; int bad = 0; uint64_t where = 0, seen = 0; };
    std::vector<Part> parts(nt);
    auto worker = [&](unsigned t) {
        Part& pt = parts[t];
        auto flag = [&](int code, uint64_t where) { if (!pt.bad) { pt.bad = code; pt.where = where; } };
        const uint32_t l0 = uint32_t(uint64_t(b.n_loci) * t / nt), l1 = uint32_t(uint64_t(b.n_loci) * (t + 1) / nt);
        for (uint32_t l = l0; l < l1; ++l) {
            if ((b.ref_off[l] & 15) || (b.alt_off[l] & 15)) { flag(10, l); continue; }
            if (uint64_t(b.ref_off[l]) + b.ref_len[l] > b.hap_len || uint64_t(b.alt_off[l]) + b.alt_len[l] > b.hap_len) { flag(11, l); continue; }
            if (l && b.locus_row[l] <= b.locus_row[l - 1]) flag(12, l);
            if (check_cands && b.cand_start[l] > b.cand_start[l + 1]) flag(13, l);
            if (check_cands) pt.md = std::max<uint64_t>(pt.md, b.cand_start[l + 1] - b.cand_start[l]);
            pt.mh = std::max(pt.mh, std::max(b.ref_len[l], b.alt_len[l]));
            if (shapes_seen) pt.seen |= uint64_t(1) << shape_key(window_shape(b.hap + b.ref_off[l], b.ref_len[l], b.hap + b.alt_off[l], b.alt_len[l]));
        }
        const uint32_t r0 = uint32_t(uint64_t(b.n_reads) * t / nt), r1 = uint32_t(uint64_t(b.n_reads) * (t + 1) / nt);
        for (uint32_t r = r0; r < r1; ++r) {
            uint32_t len;
            if (b.v2) {
                len = b.read_len16[r];
                const uint64_t nb = (uint64_t(len) + 1) / 2;
                if (b.read_off4) { if (uint64_t(b.read_off4[r]) * 4 + nb > b.nib_len) flag(2, r); }
                else pt.units += (nb + 3) / 4;
                const uint64_t k = b.cb_key[r];
                if (k != VTX_NO_CB_KEY && (k & VTX_CB_EXOTIC) && (k & ~VTX_CB_EXOTIC) >= b.n_exotic) flag(3, r);
                else if (k != VTX_NO_CB_KEY && !(k & VTX_CB_EXOTIC) && (k >> 60)) flag(6, r);
            } else {
                len = b.read_len[r];
                if (b.read_off[r] & 15) flag(1, r);
                else if (b.read_off[r] + (uint64_t(len) + 1) / 2 > b.nib_len) flag(2, r);
                else if (b.cb_off[r] != VTX_NO_CB && uint64_t(b.cb_off[r]) + b.cb_len[r] > b.cb_bytes_len) flag(3, r);
            }
            if (b.umi && b.umi[r] != VTX_NO_UMI && b.umi[r] > VTX_UMI_KEY_MAX) flag(4, r);
            pt.mr = std::max(pt.mr, len);
        }
        if (scan_cands) {
            const uint64_t c0 = b.n_cand * t / nt, c1 = b.n_cand * (t + 1) / nt;
            uint32_t worst = 0;
            for (uint64_t c = c0; c < c1; ++c) worst = std::max(worst, b.cand_read[c]);
            if (c1 > c0 && worst >= b.n_reads) flag(5, c0);
        }
    };
    if (nt == 1) worker(0);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 1; t < nt; ++t) th.emplace_back(worker, t);
        worker(0);
        for (auto& x : th) x.join();
    }
    uint32_t mr = 0, mh = 0;
    uint64_t md = 0, units = 0;
    for (const Part& pt : parts) {
        mr = std::max(mr, pt.mr); mh = std::max(mh, pt.mh); md = std::max(md, pt.md); units += pt.units;
        if (shapes_seen) *shapes_seen |= pt.seen;
        const unsigned long long w = (unsigned long long)pt.where;
        switch (pt.bad) {
        case 1: return set_err(ctx, VTX_E_INVALID, "read %llu: read_off must be a multiple of 16", w);
        case 2: return set_err(ctx, VTX_E_INVALID, "read %llu outside read_nib", w);
        case 3: return set_err(ctx, VTX_E_INVALID, "read %llu: CB outside cb_bytes", w);
        case 4: return set_err(ctx, VTX_E_INVALID, "read %llu: UMI key exceeds VTX_UMI_KEY_MAX", w);
        case 5: return set_err(ctx, VTX_E_INVALID, "cand_read out of range near candidate %llu", w);
        case 6: return set_err(ctx, VTX_E_INVALID, "read %llu: read_cb_key is not a vtx_pack_cb code", w);
        case 10: return set_err(ctx, VTX_E_INVALID, "locus %llu: haplotype offsets must be multiples of 16", w);
        case 11: return set_err(ctx, VTX_E_INVALID, "locus %llu: haplotype window outside hap_bytes", w);
        case 12: return set_err(ctx, VTX_E_INVALID, "locus_row must be strictly ascending (locus %llu)", w);
        case 13: return set_err(ctx, VTX_E_INVALID, "cand_start must be ascending (locus %llu)", w);
        default: break;
        }
    }
    if (b.v2 && !b.read_off4 && units * 4 > b.nib_len) return set_err(ctx, VTX_E_INVALID, "dense read pool is shorter than the reads it should hold");
    if (mr > uint32_t(kMaxRead)) return set_err(ctx, VTX_E_UNSUPPORTED, "reads longer than %d bases (biased int16 DP) are not supported (%u)", kMaxRead, mr);
    *max_read = mr; *max_hap = mh;
    if (max_depth) *max_depth = md;
    return VTX_OK;
}

int upload(vtx_ctx* ctx, DBuf& d, const void* h, size_t bytes)
{
    ENS(d, bytes ? bytes : 16);
    if (bytes) CK(cudaMemcpyAsync(d.p, h, bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    return VTX_OK;
}

#define UP(buf, ptr, bytes) do { int rc_ = upload(ctx, buf, ptr, (bytes)); if (rc_) return rc_; } while (0)

// claim the next input slot: its previous user's kernels must have finished before the copy may overwrite it
int claim_slot(vtx_ctx* ctx, InSlot** out)
{
    InSlot* sl = &ctx->slot[ctx->n_submits & 1];
    ++ctx->n_submits;
    if (sl->used) CK(cudaStreamWaitEvent(ctx->copy_stream, sl->free_ev, 0));
    sl->used = true;
    *out = sl;
    return VTX_OK;
}

// the locus arrays and the haplotype pool, both layouts
int upload_loci(vtx_ctx* ctx, InSlot* sl, const BatchView& h, DevBatch& d)
{
    const size_t nl = h.n_loci;
    UP(sl->locus_row, h.locus_row, nl * 4);
    UP(sl->hap, h.hap, h.hap_len);
    UP(sl->ref_off, h.ref_off, nl * 4); UP(sl->ref_len, h.ref_len, nl * 4);
    UP(sl->alt_off, h.alt_off, nl * 4); UP(sl->alt_len, h.alt_len, nl * 4);
    d.n_loci = h.n_loci; d.n_reads = h.n_reads; d.n_cand = h.n_cand;
    d.locus_row = P<uint32_t>(sl->locus_row); d.hap = P<uint8_t>(sl->hap);
    d.ref_off = P<uint32_t>(sl->ref_off); d.ref_len = P<uint32_t>(sl->ref_len);
    d.alt_off = P<uint32_t>(sl->alt_off); d.alt_len = P<uint32_t>(sl->alt_len);
    return VTX_OK;
}

// loci and reads of a vtx_batch (what vtx_score_pairs needs)
int upload_common(vtx_ctx* ctx, InSlot* sl, const BatchView& h, DevBatch& d)
{
    int rc = upload_loci(ctx, sl, h, d);
    if (rc) return rc;
    UP(sl->read_nib, h.read_nib, h.nib_len);
    UP(sl->read_off, h.read_off, size_t(h.n_reads) * 8); UP(sl->read_len, h.read_len, size_t(h.n_reads) * 4);
    d.read_nib = P<uint8_t>(sl->read_nib); d.read_off = P<uint64_t>(sl->read_off); d.read_len = P<uint32_t>(sl->read_len);
    return VTX_OK;
}

// vtx_batch: the rest of the shard
int upload_batch(vtx_ctx* ctx, InSlot* sl, const BatchView& h, DevBatch& d)
{
    int rc = upload_common(ctx, sl, h, d);
    if (rc) return rc;
    const size_t nr = h.n_reads;
    UP(sl->cand_start, h.cand_start, size_t(h.n_loci + 1) * 8);
    UP(sl->cb_bytes, h.cb_bytes, h.cb_bytes_len);
    UP(sl->read_cb_off, h.cb_off, nr * 4); UP(sl->read_cb_len, h.cb_len, nr * 2);
    if (h.umi) UP(sl->read_umi, h.umi, nr * 8);
    UP(sl->cand_read, h.cand_read, size_t(h.n_cand) * 4);
    d.cand_start = P<uint64_t>(sl->cand_start); d.cb_bytes = P<uint8_t>(sl->cb_bytes);
    d.read_cb_off = P<uint32_t>(sl->read_cb_off); d.read_cb_len = P<uint16_t>(sl->read_cb_len);
    d.read_umi = h.umi ? P<uint64_t>(sl->read_umi) : nullptr; d.cand_read = P<uint32_t>(sl->cand_read);
    return VTX_OK;
}

// vtx_batch2: the slim arrays; the engine's read arrays are derived from them on the device (expand_reads)
int upload_batch2(vtx_ctx* ctx, InSlot* sl, const BatchView& h, DevBatch& d)
{
    int rc = upload_loci(ctx, sl, h, d);
    if (rc) return rc;
    const size_t nr = h.n_reads;
    UP(sl->cand_start, h.cand_start, size_t(h.n_loci + 1) * 8);
    UP(sl->read_nib, h.read_nib, h.nib_len);
    if (h.read_off4) UP(sl->read_off4, h.read_off4, nr * 4);
    UP(sl->read_len16, h.read_len16, nr * 2);
    UP(sl->read_cb_key, h.cb_key, nr * 8);
    if (h.n_exotic) { UP(sl->cb_bytes, h.cb_bytes, h.cb_off_ex[h.n_exotic]); UP(sl->cb_off_ex, h.cb_off_ex, size_t(h.n_exotic + 1) * 4); }
    if (h.umi) UP(sl->read_umi, h.umi, nr * 8);
    if (h.cand_read) UP(sl->cand_read, h.cand_read, size_t(h.n_cand) * 4);
    d.cand_start = P<uint64_t>(sl->cand_start); d.read_nib = P<uint8_t>(sl->read_nib);
    d.read_cb_key = P<uint64_t>(sl->read_cb_key);
    d.cb_bytes = h.n_exotic ? P<uint8_t>(sl->cb_bytes) : nullptr; d.cb_off_ex = h.n_exotic ? P<uint32_t>(sl->cb_off_ex) : nullptr;
    d.read_umi = h.umi ? P<uint64_t>(sl->read_umi) : nullptr;
    d.cand_read = h.cand_read ? P<uint32_t>(sl->cand_read) : nullptr;
    return VTX_OK;
}

// slim read arrays (device) -> the engine's internal read_off (u64 bytes) / read_len (u32)
int expand_reads(vtx_ctx* ctx, uint32_t nr, const uint16_t* d_len16, const uint32_t* d_off4, DevBatch& d)
{
    ENS(ctx->x_read_off, size_t(nr ? nr : 1) * 8); ENS(ctx->x_read_len, size_t(nr ? nr : 1) * 4);
    if (nr) {
        if (!d_off4) {          // dense pool: offsets are the running sum of the 4-byte units of the reads before
            ENS(ctx->x_units, size_t(nr) * 4); ENS(ctx->x_off4, size_t(nr + 1) * 4);
            vtx_k_read_units<<<blocks_for(nr, 256), 256, 0, ctx->stream>>>(nr, d_len16, P<uint32_t>(ctx->x_units));
            int rc = scan_u32(ctx, ctx->stream, ctx->scan_sums, P<uint32_t>(ctx->x_units), nr, P<uint32_t>(ctx->x_off4), nullptr);
            if (rc) return rc;
            d_off4 = P<uint32_t>(ctx->x_off4);
        }
        vtx_k_expand_reads<<<blocks_for(nr, 256), 256, 0, ctx->stream>>>(nr, d_len16, d_off4, P<uint64_t>(ctx->x_read_off), P<uint32_t>(ctx->x_read_len));
        CK(cudaGetLastError());
    }
    d.read_off = P<uint64_t>(ctx->x_read_off); d.read_len = P<uint32_t>(ctx->x_read_len);
    return VTX_OK;
}

// Entry checks shared by the submits: barcodes set, batch present, the layout's own checks, the promised read length;
// then the device is selected and the submit gets its timing record.
template <typename Check>
int begin_submit(vtx_ctx* ctx, const void* batch, const char* fn, const char* what, Check check, uint32_t max_read_len, TimeRec** tr)
{
    if (!ctx->have_barcodes) return set_err(ctx, VTX_E_STATE, "vtx_set_barcodes must be called before %s", fn);
    if (!batch) return set_err(ctx, VTX_E_INVALID, "%s is NULL", what);
    int rc = check();
    if (rc) return rc;
    if (max_read_len > uint32_t(kMaxRead)) return set_err(ctx, VTX_E_UNSUPPORTED, "reads longer than %d bases are not supported", kMaxRead);
    CK(cudaSetDevice(ctx->device));
    *tr = new_trec(ctx);
    if (!*tr) return set_err(ctx, VTX_E_CUDA, "cudaEventCreate failed");
    ctx->submitted = true;
    return VTX_OK;
}

// vtx_submit / vtx_submit2: a host batch of either layout
template <typename Batch>
int submit_host(vtx_ctx* ctx, const Batch* hb, const char* fn)
{
    Nvtx nvtx_range(fn);
    BatchView h;
    TimeRec* tr = nullptr;
    int rc = begin_submit(ctx, hb, fn, "batch", [&] { h = view_of(hb); return validate_batch(ctx, h); }, 0, &tr);
    if (rc) return rc;
    InSlot* sl = nullptr;
    rc = claim_slot(ctx, &sl);
    if (rc) return rc;
    // 1. start the copies of this shard on the copy stream (they overlap the previous shard's kernels) ...
    DevBatch d{};
    CK(cudaEventRecord(tr->ev[EV_START], ctx->copy_stream));
    rc = h.v2 ? upload_batch2(ctx, sl, h, d) : upload_batch(ctx, sl, h, d);
    if (rc) return rc;
    CK(cudaEventRecord(tr->ev[EV_H2D], ctx->copy_stream));
    CK(cudaEventRecord(sl->copy_done, ctx->copy_stream));
    tr->had_h2d = true;
    // 2. ... validate the host arrays meanwhile; nothing has been launched on them yet
    { Nvtx r_val("vtx: validate host batch (copies in flight)");
      rc = scan_host_batch(ctx, h, &d.max_read_len, &d.max_hap_len, true, &d.max_depth, &d.shapes); }
    if (rc) { cudaStreamSynchronize(ctx->copy_stream); --ctx->trec_used; return rc; }
    d.have_shapes = true;
    // 3. kernels wait for the copy, and release the slot when done
    CK(cudaStreamWaitEvent(ctx->stream, sl->copy_done, 0));
    CK(cudaEventRecord(tr->ev[EV_C0], ctx->stream));
    if (h.v2) {
        rc = expand_reads(ctx, h.n_reads, P<uint16_t>(sl->read_len16), h.read_off4 ? P<uint32_t>(sl->read_off4) : nullptr, d);
        if (rc) return rc;
    }
    rc = process_batch(ctx, d, tr);
    if (rc) return rc;
    CK(cudaEventRecord(sl->free_ev, ctx->stream));
    return VTX_OK;
}

// vtx_submit_device_ex / vtx_submit2_device: the batch's arrays are already on the device
template <typename Batch>
int submit_resident(vtx_ctx* ctx, const Batch* db, const char* fn, uint32_t max_read_len, uint32_t max_hap_len)
{
    BatchView v;
    TimeRec* tr = nullptr;
    int rc = begin_submit(ctx, db, fn, "batch", [&] { v = view_of(db); return validate_batch(ctx, v); }, max_read_len, &tr);
    if (rc) return rc;
    DevBatch d = dev_batch_of(v, max_read_len, max_hap_len);
    CK(cudaEventRecord(tr->ev[EV_C0], ctx->stream));
    if (v.v2) {
        rc = expand_reads(ctx, v.n_reads, v.read_len16, v.read_off4, d);
        if (rc) return rc;
    }
    return process_batch(ctx, d, tr);
}

void comm_destroy(vtx_ctx* ctx);      // with the NCCL loader below

// The count entries vtx_cluster_cells and vtx_donors_ambient take, validated in one pass: row < n_rows, col < n_cols, (row, col)
// strictly ascending, and at most max_molecules REF + ALT molecules per row (`why` says what a larger sum would break).  Rows are
// contiguous, so per_row(v, i0, i1, molecules) sees each row present once, with its entries [i0, i1).
template <typename PerRow>
int validate_entries(vtx_ctx* ctx, const char* fn, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                            const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, uint64_t max_molecules, const char* why, PerRow per_row)
{
    for (uint64_t i = 0; i < n;) {
        const uint32_t v = row[i];
        if (v >= n_rows) return set_err(ctx, VTX_E_INVALID, "%s: entry %llu has row %u >= n_rows %llu", fn, (unsigned long long)i, v, (unsigned long long)n_rows);
        if (i && v < row[i - 1]) return set_err(ctx, VTX_E_INVALID, "%s: entry %llu: rows are not ascending", fn, (unsigned long long)i);
        uint64_t molecules = 0;
        const uint64_t i0 = i;
        for (; i < n && row[i] == v; ++i) {
            if (col[i] >= n_cols) return set_err(ctx, VTX_E_INVALID, "%s: entry %llu has col %u >= n_cols %u", fn, (unsigned long long)i, col[i], n_cols);
            if (i > i0 && col[i] <= col[i - 1])
                return set_err(ctx, VTX_E_INVALID, "%s: entry %llu: (row, col) is not strictly ascending", fn, (unsigned long long)i);
            molecules += uint64_t(ref_cnt[i]) + alt_cnt[i];
            if (molecules > max_molecules)
                return set_err(ctx, VTX_E_INVALID, "%s: row %u holds more than %llu molecules; %s", fn, v, (unsigned long long)max_molecules, why);
        }
        per_row(v, i0, i, molecules);
    }
    return VTX_OK;
}

// §5h's estimate of m: the coarse grid, then every m within kFineReach of its winner; the largest J wins, ties the smallest m.
// evaluate(list) appends J of every m in `list` to obj and returns a VTX code; ms / obj end with every evaluated m in that order.
template <typename Evaluate>
int estimate_permille(std::vector<uint16_t>& ms, std::vector<int64_t>& obj, Evaluate evaluate, uint32_t* chosen)
{
    using namespace ambient;
    auto best_of = [&]() {
        size_t w = 0;
        for (size_t i = 1; i < ms.size(); ++i)
            if (obj[i] > obj[w] || (obj[i] == obj[w] && ms[i] < ms[w])) w = i;
        return ms[w];
    };
    for (uint32_t m = 0; m <= uint32_t(kMaxPermille); m += kCoarseStep) ms.push_back(uint16_t(m));
    int rc = evaluate(ms);
    if (rc) return rc;
    const uint32_t mc = best_of();
    std::vector<uint16_t> fine;
    for (uint32_t m = mc > kFineReach ? mc - kFineReach : 0; m <= std::min<uint32_t>(kMaxPermille, mc + kFineReach); ++m)
        if (m % kCoarseStep) fine.push_back(uint16_t(m));
    rc = evaluate(fine);
    if (rc) return rc;
    ms.insert(ms.end(), fine.begin(), fine.end());
    *chosen = best_of();
    return VTX_OK;
}

// §5i's fit over touched rows already on the device: A / T [n_t][K], rowA / rowT [n_t], fit [n_fit] (touched indices of the used
// rows).  given = -1 estimates m (ms / obj: every evaluated m in evaluation order), else fixes it.  At the chosen m, LL / GT / PL
// [n_t][K] land in cg_ll / cg_gt / cg_pl.  J uses the first kMaxBatch entries of cg_acc, which the caller has sized.
int cg_fit_device(vtx_ctx* ctx, const ambient::Fractions& fr, uint32_t K, int32_t given, uint32_t n_t, uint32_t n_fit, const uint32_t* d_fit,
                  const unsigned long long* d_rowA, const unsigned long long* d_rowT, const int64_t* d_A, const int64_t* d_T,
                  std::vector<uint16_t>& ms, std::vector<int64_t>& obj, uint32_t* chosen)
{
    using namespace cluster_gt;
    cudaStream_t st = ctx->stream;
    ENS(ctx->cg_ll, size_t(n_t) * K * 24 + 8);
    ENS(ctx->cg_gt, size_t(n_t) * K + 8);
    ENS(ctx->cg_pl, size_t(n_t) * K * 12 + 8);
    unsigned long long* d_J = P<unsigned long long>(ctx->cg_acc);
    // J(m) of every m in the list, one launch per batch of up to kMaxBatch
    std::vector<unsigned long long> h_J(ambient::kMaxBatch);
    auto evaluate = [&](const std::vector<uint16_t>& list) -> int {
        for (size_t o = 0; o < list.size(); o += ambient::kMaxBatch) {
            ambient::Batch bt{};
            bt.n = uint32_t(std::min<size_t>(ambient::kMaxBatch, list.size() - o));
            for (uint32_t b = 0; b < bt.n; ++b) bt.m[b] = list[o + b];
            CK(cudaMemsetAsync(d_J, 0, size_t(ambient::kMaxBatch) * 8, st));
            if (n_fit) {
                const unsigned g = grid_for(ctx, uint64_t(bt.n) * n_fit * 32, kCgThreads);
                vtx_k_cg_fit<<<g, kCgThreads, 0, st>>>(bt, fr, K, n_fit, d_fit, d_rowA, d_rowT, d_A, d_T, d_J);
                CK(cudaGetLastError());
            }
            CK(cudaMemcpyAsync(h_J.data(), d_J, size_t(bt.n) * 8, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (uint32_t b = 0; b < bt.n; ++b) obj.push_back(int64_t(h_J[b]));
        }
        return VTX_OK;
    };
    *chosen = uint32_t(given);
    int rc = VTX_OK;
    if (given < 0) rc = estimate_permille(ms, obj, evaluate, chosen);
    else { ms.assign(1, uint16_t(*chosen)); rc = evaluate(ms); }
    if (rc) return rc;
    if (n_t) {
        const unsigned g = grid_for(ctx, uint64_t(n_t) * 32, kCgThreads);
        vtx_k_cg_call<<<g, kCgThreads, 0, st>>>(*chosen, fr, K, n_t, d_rowA, d_rowT, d_A, d_T, P<int64_t>(ctx->cg_ll), P<uint8_t>(ctx->cg_gt),
                                                 P<uint32_t>(ctx->cg_pl));
        CK(cudaGetLastError());
    }
    return VTX_OK;
}

// ---- the post-passes' shared intake (vtx_cluster_cells*, vtx_donors_ambient, vtx_cluster_genotypes, vtx_cluster_refine) ----

int check_finished(vtx_ctx* ctx, const char* fn)
{
    if (!ctx->finished || ctx->gather_pending)
        return set_err(ctx, VTX_E_STATE, "%s: submits are unfinished (call vtx_finish / vtx_finish_device first)", fn);
    return VTX_OK;
}

int check_error_rate(vtx_ctx* ctx, const char* fn, double error_rate)
{
    if (!(error_rate >= 1e-6 && error_rate <= 0.25))
        return set_err(ctx, VTX_E_INVALID, "%s: error rate %g outside [1e-6, 0.25]", fn, error_rate);
    return VTX_OK;
}

int check_k(vtx_ctx* ctx, const char* fn, uint32_t K)
{
    if (K < clusters::kMinK || K > clusters::kMaxK) return set_err(ctx, VTX_E_INVALID, "%s: k = %u; 2 to 32 clusters are supported", fn, K);
    return VTX_OK;
}

// one row of a dosage table, g[width]: 0, 1, 2 or VTX_GT_MISSING; `noun` names a column ("donor", "sample")
int check_dosage_row(vtx_ctx* ctx, const char* fn, const uint8_t* g, uint32_t width, uint64_t row, const char* noun)
{
    for (uint32_t s = 0; s < width; ++s)
        if (g[s] > 2 && g[s] != donors::kMissing)
            return set_err(ctx, VTX_E_INVALID, "%s: dosage %u at row %llu, %s %u (0, 1, 2 or VTX_GT_MISSING)", fn, unsigned(g[s]),
                           (unsigned long long)row, noun, s);
    return VTX_OK;
}

// row v of a clustering's sums, alt_w / depth_w [K], within §5i's bounds; *total is the depth_w sum over the rows so far
int check_sums_row(vtx_ctx* ctx, const char* fn, const int64_t* alt_w, const int64_t* depth_w, uint32_t K, uint64_t v, uint64_t* total)
{
    for (uint32_t k = 0; k < K; ++k) {
        const int64_t a = alt_w[k], t = depth_w[k];
        if (a < 0 || a > t || t > cluster_gt::kMaxDepthW)
            return set_err(ctx, VTX_E_INVALID, "%s: row %llu, cluster %u: alt_w %lld, depth_w %lld (0 <= alt_w <= depth_w <= 2^51)", fn,
                           (unsigned long long)v, k, (long long)a, (long long)t);
        *total += uint64_t(t);
        if (*total > cluster_gt::kMaxTotalDepthW)
            return set_err(ctx, VTX_E_INVALID, "%s: depth_w sums to more than 2^51 over the rows; the fit's int64 sums would not be exact", fn);
    }
    return VTX_OK;
}

// Refuses a call that needs `need` bytes of device memory when fewer are available: free memory plus the capacity of `held`,
// the buffers the call ensures (ensure frees them before it grows them; a buffer the call does not ensure stays allocated, so a
// null entry counts nothing).  *avail gets the available bytes.
int check_free(vtx_ctx* ctx, const char* fn, double need, std::initializer_list<const DBuf*> held, double* avail = nullptr)
{
    CK(cudaSetDevice(ctx->device));
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    size_t held_b = 0;
    for (const DBuf* b : held) held_b += b ? b->cap : 0;
    const double a = double(free_b) + double(held_b);
    if (avail) *avail = a;
    if (need > a) return set_err(ctx, VTX_E_NOMEM, "%s needs %.0f MB of device memory, %.0f MB are free", fn, need * 1e-6, a * 1e-6);
    return VTX_OK;
}

// Uploads n count entries to cl_row / cl_col / cl_r / cl_a and groups by cell those at rows flagged in cl_used (already on the
// stream) with r + a > 0: §5g's count, scan and scatter into cl_cell_start and cl_c_*
int cell_entries(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt, const uint32_t* alt_cnt,
                 uint32_t n_cols, clusters::CellEntries* ce)
{
    using namespace clusters;
    cudaStream_t st = ctx->stream;
    const size_t nb = size_t(n) * 4 + 4;
    ENS(ctx->cl_row, nb); ENS(ctx->cl_col, nb); ENS(ctx->cl_r, nb); ENS(ctx->cl_a, nb);
    ENS(ctx->cl_c_row, nb); ENS(ctx->cl_c_r, nb); ENS(ctx->cl_c_a, nb);
    ENS(ctx->cl_cell_count, (size_t(n_cols) + 1) * 4);
    ENS(ctx->cl_cell_start, (size_t(n_cols) + 1) * 4);
    if (n) {
        CK(cudaMemcpyAsync(ctx->cl_row.p, row, n * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->cl_col.p, col, n * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->cl_r.p, ref_cnt, n * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->cl_a.p, alt_cnt, n * 4, cudaMemcpyHostToDevice, st));
    }
    const uint32_t nn = uint32_t(n);
    const unsigned grid = grid_for(ctx, n, kClThreads);
    CK(cudaMemsetAsync(ctx->cl_cell_count.p, 0, (size_t(n_cols) + 1) * 4, st));
    vtx_k_cl_count<<<grid, kClThreads, 0, st>>>(nn, P<uint32_t>(ctx->cl_row), P<uint32_t>(ctx->cl_col), P<uint32_t>(ctx->cl_r),
                                                 P<uint32_t>(ctx->cl_a), P<uint8_t>(ctx->cl_used), P<uint32_t>(ctx->cl_cell_count));
    CK(cudaGetLastError());
    const int rc = scan_u32(ctx, st, ctx->scan_sums, P<uint32_t>(ctx->cl_cell_count), n_cols, P<uint32_t>(ctx->cl_cell_start), nullptr);
    if (rc) return rc;
    CK(cudaMemsetAsync(ctx->cl_cell_count.p, 0, (size_t(n_cols) + 1) * 4, st));
    vtx_k_cl_scatter<<<grid, kClThreads, 0, st>>>(nn, P<uint32_t>(ctx->cl_row), P<uint32_t>(ctx->cl_col), P<uint32_t>(ctx->cl_r),
                                                   P<uint32_t>(ctx->cl_a), P<uint8_t>(ctx->cl_used), P<uint32_t>(ctx->cl_cell_start),
                                                   P<uint32_t>(ctx->cl_cell_count), P<uint32_t>(ctx->cl_c_row), P<uint32_t>(ctx->cl_c_r),
                                                   P<uint32_t>(ctx->cl_c_a));
    CK(cudaGetLastError());
    *ce = CellEntries{ P<uint32_t>(ctx->cl_cell_start), P<uint32_t>(ctx->cl_c_row), P<uint32_t>(ctx->cl_c_r), P<uint32_t>(ctx->cl_c_a) };
    return VTX_OK;
}

// §5h's row sums A_v / T_v over the n uploaded entries, into am_sums: *d_A, *d_T [n_rows]
int pool_row_sums(vtx_ctx* ctx, uint64_t n, uint64_t n_rows, const unsigned long long** d_A, const unsigned long long** d_T)
{
    using namespace ambient;
    cudaStream_t st = ctx->stream;
    ENS(ctx->am_sums, size_t(n_rows) * 16 + 16);
    unsigned long long* sums = P<unsigned long long>(ctx->am_sums);
    CK(cudaMemsetAsync(sums, 0, size_t(n_rows) * 16, st));
    if (n) {
        vtx_k_am_rowsum<<<grid_for(ctx, n, kAmThreads), kAmThreads, 0, st>>>(uint32_t(n), P<uint32_t>(ctx->cl_row), P<uint32_t>(ctx->cl_r),
                                                                             P<uint32_t>(ctx->cl_a), sums, sums + n_rows);
        CK(cudaGetLastError());
    }
    *d_A = sums;
    *d_T = sums + n_rows;
    return VTX_OK;
}

// the evaluated m (ms, with obj and, if given, 3 calls per m) in ascending order into m_out / obj_out / calls_out
void sort_grid(const std::vector<uint16_t>& ms, const std::vector<int64_t>& obj, const std::vector<uint64_t>* calls,
               std::vector<uint16_t>& m_out, std::vector<int64_t>& obj_out, std::vector<uint64_t>* calls_out)
{
    std::vector<size_t> order(ms.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](size_t x, size_t y) { return ms[x] < ms[y]; });
    m_out.resize(ms.size()); obj_out.resize(ms.size());
    if (calls_out) calls_out->resize(ms.size() * 3);
    for (size_t i = 0; i < order.size(); ++i) {
        m_out[i] = ms[order[i]];
        obj_out[i] = obj[order[i]];
        if (calls_out) for (int k = 0; k < 3; ++k) (*calls_out)[3 * i + k] = (*calls)[3 * order[i] + k];
    }
}

}  // namespace

// =================================================================================================
extern "C" {

int vtx_abi_version(void) { return VTX_ABI_VERSION; }

const char* vtx_last_error(const vtx_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int vtx_create(const vtx_config* cfg, vtx_ctx** out)
{
    vtx_ctx* ctx = nullptr;   // for CK/set_err before the ctx exists
    if (!cfg || !out) return set_err(nullptr, VTX_E_INVALID, "vtx_create: NULL argument");
    *out = nullptr;
    if (cfg->match != kMatch || cfg->mismatch != kMismatch || cfg->gap_open != kGapOpen || cfg->gap_extend != kGapExtend)
        return set_err(nullptr, VTX_E_UNSUPPORTED, "scoring constants are compiled in: match %d mismatch %d gap_open %d gap_extend %d (main.rs:35-38)",
                       kMatch, kMismatch, kGapOpen, kGapExtend);
    if (cfg->mode < 0 || cfg->mode > 2) return set_err(nullptr, VTX_E_INVALID, "unknown mode %d", cfg->mode);
    if ((cfg->flags & VTX_F_NAME_KEYS) && !cfg->use_umi)
        return set_err(nullptr, VTX_E_INVALID, "VTX_F_NAME_KEYS collapses reads through the UMI path: it needs use_umi");
    if (cfg->band_mode != VTX_BAND_FULL && cfg->band_mode != VTX_BAND_MODEL) return set_err(nullptr, VTX_E_INVALID, "unknown band_mode %d", cfg->band_mode);
    if (cfg->band_k < 0 || cfg->band_k > 8 || cfg->band_w < 0 || cfg->band_w > 4096)
        return set_err(nullptr, VTX_E_UNSUPPORTED, "band constants out of range: K %d (1..8; 0 = %d), W %d (0 = %d; main.rs:33-34)", cfg->band_k, kBandK, cfg->band_w, kBandW);
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0)
        return set_err(nullptr, VTX_E_CUDA, "no CUDA device available (%s); vartrix_b200 has no CPU fallback", cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= n_dev) return set_err(nullptr, VTX_E_INVALID, "device %d out of range (%d devices)", cfg->device, n_dev);
    CK(cudaSetDevice(cfg->device));
    ctx = new vtx_ctx();
    ctx->cfg = *cfg; ctx->device = cfg->device;
    if (ctx->cfg.band_k == 0) ctx->cfg.band_k = kBandK;
    if (ctx->cfg.band_w == 0) ctx->cfg.band_w = kBandW;
    cudaDeviceProp prop{};
    cudaError_t pe = cudaGetDeviceProperties(&prop, cfg->device);
    if (pe != cudaSuccess) { g_create_error = cudaGetErrorString(pe); delete ctx; return VTX_E_CUDA; }
    if (prop.major != 9 || prop.minor != 0) {      // sm_90a code loads on compute capability 9.0 only
        delete ctx;
        return set_err(nullptr, VTX_E_UNSUPPORTED, "vartrix_b200 is built for sm_90a (H100, compute capability 9.0); device %d is %d.%d",
                       cfg->device, prop.major, prop.minor);
    }
    ctx->n_sm = prop.multiProcessorCount;
    if (cfg->stream) { ctx->stream = static_cast<cudaStream_t>(cfg->stream); ctx->own_stream = false; }
    else {
        pe = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        if (pe != cudaSuccess) { g_create_error = cudaGetErrorString(pe); delete ctx; return VTX_E_CUDA; }
        ctx->own_stream = true;
    }
    pe = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    if (pe != cudaSuccess) { g_create_error = cudaGetErrorString(pe); vtx_destroy(ctx); return VTX_E_CUDA; }
    cudaStreamCreateWithFlags(&ctx->fetch_stream, cudaStreamNonBlocking);
    if (ctx->h_cum.alloc(kMaxCum * 8, cudaHostAllocMapped) == cudaSuccess) {
        if (cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->d_cum), ctx->h_cum.p, 0) != cudaSuccess) ctx->d_cum = nullptr;
    } else cudaGetLastError();
    for (auto& sl : ctx->slot) {
        cudaEventCreateWithFlags(&sl.copy_done, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&sl.free_ev, cudaEventDisableTiming);
    }
    bool ok = cudaMalloc(&ctx->d_metrics.p, 64) == cudaSuccess && cudaMalloc(&ctx->d_res_n.p, 64) == cudaSuccess &&
              ctx->h_scalars.alloc(64) == cudaSuccess;
    if (!ok) { g_create_error = "allocation of context scalars failed"; vtx_destroy(ctx); return VTX_E_NOMEM; }
    ctx->d_metrics.cap = 64; ctx->d_res_n.cap = 64;
    cudaMemsetAsync(ctx->d_metrics.p, 0, 64, ctx->stream);
    cudaMemsetAsync(ctx->d_res_n.p, 0, 64, ctx->stream);
    *out = ctx;
    return VTX_OK;
}

void vtx_destroy(vtx_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (cudaStream_t s : { ctx->stream, ctx->comm_stream, ctx->copy_stream, ctx->stage_stream, ctx->fetch_stream })
        if (s) cudaStreamSynchronize(s);
    comm_destroy(ctx);
    for (auto& sl : ctx->slot)
        for (cudaEvent_t e : { sl.copy_done, sl.free_ev }) if (e) cudaEventDestroy(e);
    for (auto& ss : ctx->sslot)
        for (cudaEvent_t e : { ss.staged, ss.free_ev }) if (e) cudaEventDestroy(e);
    for (auto& tr : ctx->trecs) for (auto& ev : tr.ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t e : { ctx->ev_counts, ctx->ev_gather, ctx->ev_results }) if (e) cudaEventDestroy(e);
    for (cudaStream_t s : { ctx->stage_stream, ctx->comm_stream, ctx->copy_stream, ctx->fetch_stream }) if (s) cudaStreamDestroy(s);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;     // frees the device and pinned buffers it owns
}

int vtx_host_alloc(void** out, uint64_t bytes)
{
    if (!out) return VTX_E_INVALID;
    cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault);
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); *out = nullptr; return VTX_E_NOMEM; }
    return VTX_OK;
}

int vtx_host_free(void* p) { return cudaFreeHost(p) == cudaSuccess ? VTX_OK : VTX_E_CUDA; }

int vtx_set_barcodes(vtx_ctx* ctx, const uint8_t* bytes, const uint32_t* off, uint32_t n)
{
    if (!ctx) return VTX_E_INVALID;
    if (!off || (n && !bytes && off[n] > 0)) return set_err(ctx, VTX_E_INVALID, "vtx_set_barcodes: NULL argument");
    if (n == 0) return set_err(ctx, VTX_E_INVALID, "Loaded 0 barcodes (main.rs:712-715)");
    CK(cudaSetDevice(ctx->device));
    uint32_t cap = 16;
    while (cap < 2ull * n + 1) cap <<= 1;
    std::vector<int32_t> slot(cap, -1);
    for (uint32_t i = 0; i < n; ++i) {
        if (off[i + 1] < off[i]) return set_err(ctx, VTX_E_INVALID, "barcode offsets must be ascending");
        const uint32_t len = off[i + 1] - off[i];
        if (len > 0xFFFF) return set_err(ctx, VTX_E_INVALID, "barcode %u longer than 65535 bytes", i);
        uint32_t h = uint32_t(fnv1a64(bytes + off[i], len)) & (cap - 1);
        for (;;) {
            const int32_t s = slot[h];
            if (s < 0) { slot[h] = int32_t(i); break; }
            const uint32_t l2 = off[s + 1] - off[s];
            if (l2 == len && memcmp(bytes + off[s], bytes + off[i], len) == 0)
                return set_err(ctx, VTX_E_INVALID, "duplicate barcode at index %u (first seen at %d); dedup first (main.rs:706-709)", i, s);
            h = (h + 1) & (cap - 1);
        }
    }
    // second table for the slim layout: the barcodes that have a vtx_pack_cb code, keyed by the code
    std::vector<uint64_t> kkey(cap, kNoCbKey);
    std::vector<uint32_t> kidx(cap, 0);
    for (uint32_t i = 0; i < n; ++i) {
        const uint64_t k = stage::pack_cb(bytes + off[i], off[i + 1] - off[i]);
        if (k == kNoCbKey) continue;
        uint32_t h = uint32_t(mix64(k)) & (cap - 1);
        while (kkey[h] != kNoCbKey) h = (h + 1) & (cap - 1);       // codes are injective and the strings distinct: no equal key
        kkey[h] = k; kidx[h] = i;
    }
    UP(ctx->bc_slot, slot.data(), size_t(cap) * 4);
    UP(ctx->bc_bytes, bytes, off[n]);
    UP(ctx->bc_off, off, size_t(n + 1) * 4);
    UP(ctx->bck_key, kkey.data(), size_t(cap) * 8);
    UP(ctx->bck_idx, kidx.data(), size_t(cap) * 4);
    CK(cudaStreamSynchronize(ctx->copy_stream));   // the tables are locals; they must be resident before any submit
    ctx->bc_cap = cap; ctx->bck_cap = cap; ctx->n_barcodes = n; ctx->have_barcodes = true;
    return VTX_OK;
}

int vtx_submit(vtx_ctx* ctx, const vtx_batch* hb)
{
    if (!ctx) return VTX_E_INVALID;
    return submit_host(ctx, hb, "vtx_submit");
}

int vtx_submit_device_ex(vtx_ctx* ctx, const vtx_batch* db, uint32_t max_read_len, uint32_t max_hap_len)
{
    if (!ctx) return VTX_E_INVALID;
    return submit_resident(ctx, db, "vtx_submit_device", max_read_len, max_hap_len);
}

int vtx_submit_device(vtx_ctx* ctx, const vtx_batch* db)
{
    // conservative bounds when the caller does not state them: the largest fast-path read and the
    // widest haplotype any tile class takes (wider inputs need vtx_submit_device_ex)
    return vtx_submit_device_ex(ctx, db, kFastMaxRead, class_max_n(kNumFastClasses - 1));
}

int vtx_submit2(vtx_ctx* ctx, const vtx_batch2* hb)
{
    if (!ctx) return VTX_E_INVALID;
    return submit_host(ctx, hb, "vtx_submit2");
}

int vtx_submit2_device(vtx_ctx* ctx, const vtx_batch2* db, uint32_t max_read_len, uint32_t max_hap_len)
{
    if (!ctx) return VTX_E_INVALID;
    return submit_resident(ctx, db, "vtx_submit2_device", max_read_len, max_hap_len);
}
int vtx_bgzf_inflate(vtx_ctx* ctx, const vtx_bgzf_block* blocks, uint32_t n_blocks, const uint8_t* comp, uint64_t comp_len,
                     uint8_t* out, uint64_t out_len, int32_t* status, uint32_t flags)
{
    if (!ctx) return VTX_E_INVALID;
    Nvtx nvtx_range("vtx_bgzf_inflate");
    if (n_blocks == 0) return VTX_OK;
    if (!blocks || !comp || !status || (!out && out_len)) return set_err(ctx, VTX_E_INVALID, "vtx_bgzf_inflate: NULL argument");
    static_assert(sizeof(vtx_bgzf_block) == sizeof(inflate::BlockDesc), "descriptor layouts must agree");
    for (uint32_t i = 0; i < n_blocks; ++i) {
        const vtx_bgzf_block& b = blocks[i];
        if ((b.in_off & 3) || b.in_off + b.in_len + 8 > comp_len + 8 || b.in_off + b.in_len > comp_len)
            return set_err(ctx, VTX_E_INVALID, "vtx_bgzf_inflate: member %u: payload must start on a 4-byte boundary inside comp", i);
        if (b.out_len > 65536u || b.out_off + b.out_len > out_len) return set_err(ctx, VTX_E_INVALID, "vtx_bgzf_inflate: member %u: output outside out / ISIZE above 64 KiB", i);
    }
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    ENS(ctx->inf_comp, size_t(comp_len) + 16); ENS(ctx->inf_out, size_t(out_len) + 16);
    ENS(ctx->inf_desc, size_t(n_blocks) * sizeof(vtx_bgzf_block)); ENS(ctx->inf_status, size_t(n_blocks) * 4 + 16);
    ENS(ctx->tile_counters, 64);
    CK(cudaMemsetAsync(static_cast<uint8_t*>(ctx->inf_comp.p) + comp_len, 0, 16, st));              // the readable padding
    CK(cudaMemcpyAsync(ctx->inf_comp.p, comp, comp_len, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inf_desc.p, blocks, size_t(n_blocks) * sizeof(vtx_bgzf_block), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ctx->tile_counters.p, 0, 64, st));
    if (int rc = launch_inflate(ctx, st, ctx->inf_desc.p, n_blocks, ctx->inf_comp.p, ctx->inf_out.p, ctx->inf_status.p,
                                P<uint32_t>(ctx->tile_counters), (flags & VTX_BGZF_CHECK_CRC) ? 1 : 0)) return rc;
    if (out_len) CK(cudaMemcpyAsync(out, ctx->inf_out.p, out_len, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(status, ctx->inf_status.p, size_t(n_blocks) * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (uint32_t i = 0; i < n_blocks; ++i)
        if (status[i] != 0) return set_err(ctx, VTX_E_INVALID, "vtx_bgzf_inflate: member %u failed with decoder status %d (corrupt data)", i, status[i]);
    return VTX_OK;
}

// -------------------------------------------------------------------------------------------------
// vtx_submit_bam: inflate + record scan + fetch + filters + tags on the device (vtx_inflate.cuh, vtx_stage.cuh)
// -------------------------------------------------------------------------------------------------

int vtx_submit_bam(vtx_ctx* ctx, const vtx_bam_shard* sh)
{
    if (!ctx) return VTX_E_INVALID;
    Nvtx nvtx_range("vtx_submit_bam");
    uint32_t nl = 0, nm = 0, ne = 0, max_hap = 0;
    uint64_t stream_len = 0;
    auto check = [&]() -> int {
        nl = sh->n_loci; nm = sh->n_members; ne = sh->n_entry;
        if (nl && (!sh->locus_row || !sh->locus_start || !sh->locus_end || !sh->ref_off || !sh->ref_len || !sh->alt_off || !sh->alt_len))
            return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: locus arrays missing");
        if (nm && (!sh->members || !sh->comp)) return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: members missing");
        if ((ne == 1) || (ne && !sh->entry_off)) return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: entry_off needs at least a start and an end");
        if (sh->hap_bytes_len >= 0xFFFFFFFFull) return set_err(ctx, VTX_E_INVALID, "haplotype pool exceeds 4 GiB; split the shard");
        for (uint32_t i = 0; i < nm; ++i) {
            const vtx_bgzf_block& b = sh->members[i];
            if ((b.in_off & 3) || b.in_off + b.in_len > sh->comp_len || b.out_len > 65536u || b.out_off != stream_len)
                return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: member %u: payload on a 4-byte boundary inside comp, out_off = running sum of out_len", i);
            stream_len += b.out_len;
        }
        if (stream_len >= 0xFFFFFFFFull) return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: more than 4 GiB of records in one shard; split the shard");
        for (uint32_t i = 0; i < ne; ++i)
            if (sh->entry_off[i] > stream_len || (i && sh->entry_off[i] <= sh->entry_off[i - 1])) return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: entry_off must ascend inside the stream");
        for (uint32_t l = 0; l < nl; ++l) {
            if ((sh->ref_off[l] & 15) || (sh->alt_off[l] & 15) || uint64_t(sh->ref_off[l]) + sh->ref_len[l] > sh->hap_bytes_len ||
                uint64_t(sh->alt_off[l]) + sh->alt_len[l] > sh->hap_bytes_len) return set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: locus %u: bad haplotype window", l);
            if (l && (sh->locus_row[l] <= sh->locus_row[l - 1])) return set_err(ctx, VTX_E_INVALID, "locus_row must be strictly ascending (locus %u)", l);
            max_hap = std::max(max_hap, std::max(sh->ref_len[l], sh->alt_len[l]));
        }
        return VTX_OK;
    };
    TimeRec* tr = nullptr;
    int rc = begin_submit(ctx, sh, "vtx_submit_bam", "shard", check, 0, &tr);     // the longest read is known after the record scan
    if (rc) return rc;
    if (!ctx->stage_stream) {
        CK(cudaStreamCreateWithFlags(&ctx->stage_stream, cudaStreamNonBlocking));
        for (auto& ss : ctx->sslot) { CK(cudaEventCreateWithFlags(&ss.staged, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ss.free_ev, cudaEventDisableTiming)); }
        ENS(ctx->bam_metrics, sizeof(stage::LocusMetrics));
        CK(cudaMemsetAsync(ctx->bam_metrics.p, 0, sizeof(stage::LocusMetrics), ctx->stage_stream));
        CK(ctx->h_stage.alloc(256));
    }
    cudaStream_t ss = ctx->stage_stream;
    StageSlot& sl = ctx->sslot[ctx->n_bam_submits & 1];
    ++ctx->n_bam_submits;
    if (sl.used_once) CK(cudaEventSynchronize(sl.free_ev));       // the kernels that read this slot's stream two shards ago are done
    sl.used_once = true;
    auto fail_out = [&](int code) { --ctx->trec_used; sl.used_once = false; return code; };

    // ---- copies (staging stream) ----
    auto up = [&](DBuf& d, const void* h, size_t bytes) -> int {
        int rc = ensure(ctx, d, bytes ? bytes + 16 : 16);
        if (rc) return rc;
        if (bytes && cudaMemcpyAsync(d.p, h, bytes, cudaMemcpyHostToDevice, ss) != cudaSuccess) return set_err(ctx, VTX_E_CUDA, "cudaMemcpyAsync failed in vtx_submit_bam");
        return VTX_OK;
    };
    CK(cudaEventRecord(tr->ev[EV_START], ss));
    if ((rc = up(sl.comp, sh->comp, sh->comp_len)) || (rc = up(sl.desc, sh->members, size_t(nm) * sizeof(vtx_bgzf_block))) ||
        (rc = up(sl.entry, sh->entry_off, size_t(ne) * 8)) || (rc = up(sl.l_start, sh->locus_start, size_t(nl) * 8)) ||
        (rc = up(sl.l_end, sh->locus_end, size_t(nl) * 8)) || (rc = up(sl.locus_row, sh->locus_row, size_t(nl) * 4)) ||
        (rc = up(sl.hap, sh->hap_bytes, sh->hap_bytes_len)) || (rc = up(sl.ref_off, sh->ref_off, size_t(nl) * 4)) ||
        (rc = up(sl.ref_len, sh->ref_len, size_t(nl) * 4)) || (rc = up(sl.alt_off, sh->alt_off, size_t(nl) * 4)) ||
        (rc = up(sl.alt_len, sh->alt_len, size_t(nl) * 4))) return fail_out(rc);
    CK(cudaMemsetAsync(static_cast<uint8_t*>(sl.comp.p) + sh->comp_len, 0, 16, ss));
    CK(cudaEventRecord(tr->ev[EV_H2D], ss));
    tr->had_h2d = true;
    // ---- inflate into one contiguous stream ----
    ENS(sl.stream, size_t(stream_len) + stage::kWalkWindow + 64);      // the walkers read whole windows
    ENS(sl.status, size_t(nm) * 4 + 16); ENS(sl.scalars, 256);
    uint32_t* d_sc = P<uint32_t>(sl.scalars);       // [0] walk cursor / inflate cursor, [1] err, [2] max_span, [3] max read, [4..] spare
    CK(cudaMemsetAsync(sl.scalars.p, 0, 256, ss));
    if (nm && (rc = launch_inflate(ctx, ss, sl.desc.p, nm, sl.comp.p, sl.stream.p, sl.status.p, d_sc, 1))) return fail_out(rc);
    stage::Params sp{};
    sp.s = P<uint8_t>(sl.stream); sp.s_len = stream_len; sp.tid = sh->tid;
    sp.mapq_min = sh->mapq; sp.primary_only = sh->primary_only != 0; sp.no_duplicates = sh->no_duplicates != 0;
    sp.min_base_quality = ctx->min_base_quality;
    const bool name_keys = (ctx->cfg.flags & VTX_F_NAME_KEYS) != 0;       // the keys come from vtx_k_name_key, not from UB tags
    sp.want_umi = ctx->cfg.use_umi && !name_keys ? 1 : 0; sp.tag0 = uint8_t(sh->bam_tag[0]); sp.tag1 = uint8_t(sh->bam_tag[1]);
    // ---- record boundaries ----
    const uint32_t n_seg = ne ? ne - 1 : 0;
    ENS(sl.seg_count, size_t(n_seg + 1) * 4); ENS(sl.seg_first, size_t(n_seg + 2) * 4);
    uint32_t n_rec = 0;
    std::vector<int32_t> h_status(nm);
    if (n_seg) {
        stage::vtx_k_walk<<<blocks_for(n_seg, stage::kWalkWarps), stage::kWalkWarps * 32, 0, ss>>>(sp, n_seg, P<uint64_t>(sl.entry), 0, P<uint32_t>(sl.seg_count), nullptr, nullptr, d_sc + 1);
        rc = scan_u32(ctx, ss, ctx->stage_sums, P<uint32_t>(sl.seg_count), n_seg, P<uint32_t>(sl.seg_first), nullptr);
        if (rc) return fail_out(rc);
    }
    // wait #1 (staging stream only): inflate status, walk errors, number of records
    uint32_t* hs = ctx->h_stage.as<uint32_t>();
    if (n_seg) CK(cudaMemcpyAsync(hs, P<uint32_t>(sl.seg_first) + n_seg, 4, cudaMemcpyDeviceToHost, ss)); else hs[0] = 0;
    CK(cudaMemcpyAsync(hs + 1, d_sc + 1, 4, cudaMemcpyDeviceToHost, ss));
    if (nm) CK(cudaMemcpyAsync(h_status.data(), sl.status.p, size_t(nm) * 4, cudaMemcpyDeviceToHost, ss));
    CK(cudaStreamSynchronize(ss));
    for (uint32_t i = 0; i < nm; ++i)
        if (h_status[i] != 0) return fail_out(set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: BGZF member %u failed with decoder status %d (corrupt data)", i, h_status[i]));
    if (hs[1] & (stage::kErrWalk | stage::kErrRecord))
        return fail_out(set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: the record walk did not land on the index's record boundaries (corrupt BAM record or index; flags %u)", hs[1]));
    n_rec = hs[0];
    const size_t nrp = size_t(n_rec) + 1;
    ENS(sl.rec_off, nrp * 8); ENS(sl.rec_tid, nrp * 4); ENS(sl.rec_pos, nrp * 4); ENS(sl.rec_end, nrp * 4); ENS(sl.rec_fm, nrp * 4); ENS(sl.used, nrp * 4);
    ENS(sl.cand_count, size_t(nl + 1) * 4); ENS(sl.cand_first, size_t(nl + 2) * 4); ENS(sl.cand_start, size_t(nl + 2) * 8);
    stage::LocusMetrics* d_met = P<stage::LocusMetrics>(ctx->bam_metrics);
    uint64_t n_cand = 0;
    uint32_t max_read = 0;
    if (n_rec) {
        stage::vtx_k_walk<<<blocks_for(n_seg, stage::kWalkWarps), stage::kWalkWarps * 32, 0, ss>>>(sp, n_seg, P<uint64_t>(sl.entry), 1, nullptr, P<uint32_t>(sl.seg_first), P<uint64_t>(sl.rec_off), d_sc + 1);
        stage::vtx_k_parse<<<blocks_for(n_rec, 256), 256, 0, ss>>>(sp, n_rec, P<uint64_t>(sl.rec_off), P<int32_t>(sl.rec_tid), P<int32_t>(sl.rec_pos),
                                                                   P<int32_t>(sl.rec_end), P<uint32_t>(sl.rec_fm), d_sc + 2);
        CK(cudaMemsetAsync(sl.used.p, 0, nrp * 4, ss));
    }
    if (nl) {
        // counts first; the per-locus metric counters of this pass only become final if the shard is accepted, so they go to a scratch copy
        ENS(sl.status, std::max<size_t>(size_t(nm) * 4 + 16, sizeof(stage::LocusMetrics) + 16));
        stage::LocusMetrics* d_tmp = reinterpret_cast<stage::LocusMetrics*>(sl.status.p);
        CK(cudaMemsetAsync(d_tmp, 0, sizeof(stage::LocusMetrics), ss));
        if (ctx->locus_stats) ENS(sl.lfilt, size_t(nl) * stage::kNumCounters * 4);
        stage::vtx_k_locus_cands<<<blocks_for(nl, 64), 64, 0, ss>>>(sp, nl, P<int64_t>(sl.l_start), P<int64_t>(sl.l_end), n_rec, P<uint64_t>(sl.rec_off),
                                                                   P<int32_t>(sl.rec_tid), P<int32_t>(sl.rec_pos), P<int32_t>(sl.rec_end), P<uint32_t>(sl.rec_fm),
                                                                   d_sc + 2, d_sc + 3, 0, P<uint32_t>(sl.cand_count), nullptr, nullptr, nullptr, d_tmp,
                                                                   ctx->locus_stats ? P<uint32_t>(sl.lfilt) : nullptr);
        rc = scan_u32(ctx, ss, ctx->stage_sums, P<uint32_t>(sl.cand_count), nl, P<uint32_t>(sl.cand_first), nullptr);
        if (rc) return fail_out(rc);
        CK(cudaMemcpyAsync(hs, P<uint32_t>(sl.cand_first) + nl, 4, cudaMemcpyDeviceToHost, ss));
    } else hs[0] = 0;
    CK(cudaMemcpyAsync(hs + 1, d_sc + 1, 12, cudaMemcpyDeviceToHost, ss));      // err, max_span, max read
    CK(cudaStreamSynchronize(ss));                                               // wait #2: number of candidates, longest read
    n_cand = hs[0]; max_read = hs[3];
    if (hs[1] & (stage::kErrWalk | stage::kErrRecord)) return fail_out(set_err(ctx, VTX_E_INVALID, "vtx_submit_bam: corrupt BAM record (flags %u)", hs[1]));
    if (max_read > uint32_t(kMaxRead)) return fail_out(set_err(ctx, VTX_E_UNSUPPORTED, "reads longer than %d bases (biased int16 DP) are not supported (%u)", kMaxRead, max_read));
    if (n_cand >= 0xFFFFFFF0ull) return fail_out(set_err(ctx, VTX_E_INVALID, "n_cand exceeds 2^32 per shard; split the shard"));
    const size_t ncp = size_t(n_cand) + 1;
    ENS(sl.cand_rec, ncp * 4); ENS(sl.read_off, nrp * 8); ENS(sl.read_len, nrp * 4); ENS(sl.read_cb_off, nrp * 4); ENS(sl.read_cb_len, nrp * 2 + 2);
    if (ctx->cfg.use_umi) ENS(sl.read_umi, nrp * 8);
    if (nl) {
        stage::LocusMetrics* d_tmp = reinterpret_cast<stage::LocusMetrics*>(sl.status.p);
        stage::vtx_k_locus_cands<<<blocks_for(nl, 64), 64, 0, ss>>>(sp, nl, P<int64_t>(sl.l_start), P<int64_t>(sl.l_end), n_rec, P<uint64_t>(sl.rec_off),
                                                                   P<int32_t>(sl.rec_tid), P<int32_t>(sl.rec_pos), P<int32_t>(sl.rec_end), P<uint32_t>(sl.rec_fm),
                                                                   d_sc + 2, d_sc + 3, 1, nullptr, P<uint32_t>(sl.cand_first), P<uint32_t>(sl.cand_rec), P<uint32_t>(sl.used), d_tmp,
                                                                   nullptr);
        stage::vtx_k_widen<<<blocks_for(nl + 1, 256), 256, 0, ss>>>(nl + 1, P<uint32_t>(sl.cand_first), P<uint64_t>(sl.cand_start));
    }
    if (n_rec)
        stage::vtx_k_read_emit<<<blocks_for(n_rec, 128), 128, 0, ss>>>(sp, n_rec, P<uint64_t>(sl.rec_off), P<uint32_t>(sl.used), P<uint64_t>(sl.read_off),
                                                                       P<uint32_t>(sl.read_len), P<uint32_t>(sl.read_cb_off), P<uint16_t>(sl.read_cb_len),
                                                                       P<uint64_t>(sl.read_umi), d_sc + 1);
    if (name_keys && n_rec) {             // --collapse-mates: every name can be keyed here, so no wait follows
        uint32_t tab_size = 1;
        while (tab_size < 2 * n_rec) tab_size <<= 1;                   // n_rec < 2^28: the records of < 4 GiB of stream
        ENS(sl.name_tab, size_t(tab_size) * 4);
        CK(cudaMemsetAsync(sl.name_tab.p, 0xFF, size_t(tab_size) * 4, ss));
        stage::vtx_k_name_key<<<blocks_for(n_rec, 128), 128, 0, ss>>>(sp, n_rec, P<uint64_t>(sl.rec_off), P<uint32_t>(sl.used),
                                                                      P<uint32_t>(sl.name_tab), tab_size - 1, P<uint64_t>(sl.read_umi));
    }
    CK(cudaGetLastError());
    if (ctx->cfg.use_umi && !name_keys && n_rec) {      // wait #3 only with --umi: a UB string the device cannot key sends the shard back to the host
        CK(cudaMemcpyAsync(hs + 1, d_sc + 1, 4, cudaMemcpyDeviceToHost, ss));
        CK(cudaStreamSynchronize(ss));
        if (hs[1] & stage::kErrExoticUmi) return fail_out(set_err(ctx, VTX_E_UNSUPPORTED, "vtx_submit_bam: a UB tag outside vtx_pack_umi's alphabet needs the host's interner; stage this shard on the host"));
    }
    if (nl) {                             // the shard is accepted: its filter counters join the running totals
        stage::LocusMetrics* d_tmp = reinterpret_cast<stage::LocusMetrics*>(sl.status.p);
        vtx_k_add_u64<<<1, 32, 0, ss>>>(reinterpret_cast<unsigned long long*>(d_met), reinterpret_cast<const unsigned long long*>(d_tmp),
                                        int(sizeof(stage::LocusMetrics) / 8));
    }
    CK(cudaEventRecord(sl.staged, ss));
    // ---- the usual pipeline, on the engine stream, reading reads and tags inside the stream ----
    DevBatch d{};
    d.n_loci = nl; d.n_reads = n_rec; d.n_cand = n_cand;
    d.locus_row = P<uint32_t>(sl.locus_row); d.hap = P<uint8_t>(sl.hap); d.ref_off = P<uint32_t>(sl.ref_off); d.ref_len = P<uint32_t>(sl.ref_len);
    d.alt_off = P<uint32_t>(sl.alt_off); d.alt_len = P<uint32_t>(sl.alt_len); d.cand_start = P<uint64_t>(sl.cand_start);
    d.read_nib = P<uint8_t>(sl.stream); d.read_off = P<uint64_t>(sl.read_off); d.read_len = P<uint32_t>(sl.read_len);
    d.cb_bytes = P<uint8_t>(sl.stream); d.read_cb_off = P<uint32_t>(sl.read_cb_off); d.read_cb_len = P<uint16_t>(sl.read_cb_len);
    d.read_umi = ctx->cfg.use_umi ? P<uint64_t>(sl.read_umi) : nullptr; d.cand_read = P<uint32_t>(sl.cand_rec);
    d.max_read_len = max_read; d.max_hap_len = max_hap;
    d.lfilt = ctx->locus_stats && nl ? P<uint32_t>(sl.lfilt) : nullptr;
    CK(cudaStreamWaitEvent(ctx->stream, sl.staged, 0));
    CK(cudaEventRecord(tr->ev[EV_C0], ctx->stream));
    rc = process_batch(ctx, d, tr);
    if (rc) return rc;
    CK(cudaEventRecord(sl.free_ev, ctx->stream));
    return VTX_OK;
}

int vtx_bam_metrics_get(vtx_ctx* ctx, vtx_bam_metrics* out)
{
    if (!ctx || !out) return VTX_E_INVALID;
    memset(out, 0, sizeof(*out));
    if (!ctx->stage_stream) return VTX_OK;
    CK(cudaSetDevice(ctx->device));
    static_assert(sizeof(vtx_bam_metrics) == offsetof(stage::LocusMetrics, num_low_base_quality) &&
                  offsetof(stage::LocusMetrics, num_low_base_quality) == stage::kLowBaseQuality * sizeof(unsigned long long),
                  "metric layouts must agree");
    CK(cudaMemcpyAsync(out, ctx->bam_metrics.p, sizeof(*out), cudaMemcpyDeviceToHost, ctx->stage_stream));
    CK(cudaStreamSynchronize(ctx->stage_stream));
    return VTX_OK;
}

int vtx_set_min_base_quality(vtx_ctx* ctx, uint32_t min_q)
{
    if (!ctx) return VTX_E_INVALID;
    if (min_q > stage::kMaxBaseQuality) return set_err(ctx, VTX_E_INVALID, "min base quality %u out of range (0..%u)", min_q, stage::kMaxBaseQuality);
    ctx->min_base_quality = min_q;
    return VTX_OK;
}

int vtx_bam_low_base_quality(vtx_ctx* ctx, uint64_t* out)
{
    if (!ctx || !out) return VTX_E_INVALID;
    *out = 0;
    if (!ctx->stage_stream) return VTX_OK;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(out, static_cast<const uint8_t*>(ctx->bam_metrics.p) + offsetof(stage::LocusMetrics, num_low_base_quality), 8,
                       cudaMemcpyDeviceToHost, ctx->stage_stream));
    CK(cudaStreamSynchronize(ctx->stage_stream));
    return VTX_OK;
}

int vtx_set_locus_stats(vtx_ctx* ctx, int32_t on)
{
    if (!ctx) return VTX_E_INVALID;
    if (ctx->submitted) return set_err(ctx, VTX_E_STATE, "vtx_set_locus_stats must be called before the first submit");
    ctx->locus_stats = on != 0;
    return VTX_OK;
}

int vtx_locus_stats_get(vtx_ctx* ctx, const vtx_locus_stats** out, uint64_t* n)
{
    if (!ctx || !out || !n) return VTX_E_INVALID;
    *out = nullptr; *n = 0;
    if (!ctx->locus_stats) return set_err(ctx, VTX_E_STATE, "locus statistics are off: call vtx_set_locus_stats(ctx, 1) before the first submit");
    if (!ctx->finished) return set_err(ctx, VTX_E_STATE, "vtx_locus_stats_get must follow vtx_finish / vtx_finish_device");
    *out = ctx->stats_last_n ? ctx->h_lstats.as<const vtx_locus_stats>() : nullptr;
    *n = ctx->stats_last_n;
    return VTX_OK;
}

int vtx_set_donors(vtx_ctx* ctx, uint32_t n_donors, uint64_t n_rows, const uint8_t* dosage, double error_rate)
{
    using namespace donors;
    if (!ctx) return VTX_E_INVALID;
    if (ctx->submitted) return set_err(ctx, VTX_E_STATE, "vtx_set_donors must be called before the first submit");
    if (n_donors < kMinDonors || n_donors > kMaxDonors)
        return set_err(ctx, VTX_E_INVALID, "vtx_set_donors: %u donors; 2 to 32 are supported", n_donors);
    if (int rc = check_error_rate(ctx, "vtx_set_donors", error_rate)) return rc;
    if (n_rows && !dosage) return set_err(ctx, VTX_E_INVALID, "vtx_set_donors: dosage is NULL");
    const size_t cells = size_t(n_rows) * n_donors;
    std::vector<uint8_t> usable(size_t(n_rows) + 1, 0);
    for (uint64_t r = 0; r < n_rows; ++r) {
        if (int rc = check_dosage_row(ctx, "vtx_set_donors", dosage + size_t(r) * n_donors, n_donors, r, "donor")) return rc;
        usable[r] = row_usable(dosage + size_t(r) * n_donors, n_donors) ? 1 : 0;
    }
    CK(cudaSetDevice(ctx->device));
    ENS(ctx->donor_dosage, cells + 16);
    ENS(ctx->donor_usable, usable.size());
    if (cells) CK(cudaMemcpy(ctx->donor_dosage.p, dosage, cells, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->donor_usable.p, usable.data(), usable.size(), cudaMemcpyHostToDevice));
    ctx->n_donors = n_donors;
    ctx->donor_rows = n_rows;
    ctx->donor_tab = make_tables(error_rate);
    ctx->donors = true;
    ctx->donor_valid = false;
    return VTX_OK;
}

int vtx_donor_ll_get(vtx_ctx* ctx, const int64_t** ll, const uint64_t** counts, uint32_t* n_cols, uint32_t* n_hyp)
{
    if (!ctx || !ll || !counts || !n_cols || !n_hyp) return VTX_E_INVALID;
    *ll = nullptr; *counts = nullptr; *n_cols = 0; *n_hyp = 0;
    if (!ctx->donors) return set_err(ctx, VTX_E_STATE, "no donors: call vtx_set_donors before the first submit");
    if (!ctx->finished || !ctx->donor_valid) return set_err(ctx, VTX_E_STATE, "vtx_donor_ll_get must follow vtx_finish / vtx_finish_device");
    const uint32_t H = donors::n_hyp(ctx->n_donors);
    *ll = ctx->h_donor.as<const int64_t>();
    *counts = reinterpret_cast<const uint64_t*>(*ll + size_t(ctx->donor_last_cols) * H);
    *n_cols = ctx->donor_last_cols;
    *n_hyp = H;
    return VTX_OK;
}

// The pinned samples of vtx_cluster_cells_pinned (DESIGN.md §5k); J = 0 is vtx_cluster_cells
struct PinSpec {
    uint32_t J = 0, m = 0;
    double error_rate = 0;
    const uint8_t* dosage = nullptr;        // host [n_rows][J]
};

// vtx_cluster_cells and vtx_cluster_cells_pinned: §5g's EM and scoring; with pins, the J pinned clusters' logs are overwritten
// after the init and after every M-step, the pinned clusters keep their indices, and the scoring takes their pinned theta
static int cluster_cells_run(vtx_ctx* ctx, const char* fn, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                             const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const vtx_cluster_params* params,
                             const PinSpec& pin, vtx_clusters* out)
{
    using namespace clusters;
    const uint32_t K = params->k, R = params->restarts, J = pin.J;
    if (n && (!row || !col || !ref_cnt || !alt_cnt)) return set_err(ctx, VTX_E_INVALID, "%s: an entry array is NULL", fn);
    if (n > 0xFFFFFFFFull || n_rows > 0xFFFFFFFFull)
        return set_err(ctx, VTX_E_INVALID, "%s: %llu entries over %llu rows; both must be below 2^32", fn,
                       (unsigned long long)n, (unsigned long long)n_rows);
    const uint32_t H = donors::n_hyp(K);
    // device memory, before any host table of n_rows entries: the by-row entries (16 B) and their by-cell copy (12 B), the
    // weights, the tables, the final sums and the outputs; with pins, the dosage and the row sums
    const double need = double(n) * 28 + double(n_rows) * (5 + 16.0 * K) + double(n_cols) * (12 + 24 + 8.0 * H) +
                        double(R) * n_cols * K * 4 + double(R) * double(n_rows) * K * 8 + (J ? double(n_rows) * (J + 16) : 0.0);
    int rc = check_free(ctx, fn, need, { &ctx->cl_row, &ctx->cl_col, &ctx->cl_r, &ctx->cl_a, &ctx->cl_used, &ctx->cl_used_rows,
                                         &ctx->cl_row_start, &ctx->cl_cell_count, &ctx->cl_cell_start, &ctx->cl_c_row, &ctx->cl_c_r,
                                         &ctx->cl_c_a, &ctx->cl_la, &ctx->cl_lr, &ctx->cl_w, &ctx->cl_flags, &ctx->cl_A, &ctx->cl_T,
                                         &ctx->cl_ll, &ctx->cl_cnt, J ? &ctx->cp_dos : nullptr, J ? &ctx->am_sums : nullptr });
    if (rc) return rc;
    const size_t n_dos = size_t(n_rows) * J;
    for (uint64_t v = 0; J && v < n_rows; ++v)
        if ((rc = check_dosage_row(ctx, fn, pin.dosage + size_t(v) * J, J, v, "sample"))) return rc;
    // validate the entries in one pass; rows are contiguous, so the per-row counts need no table
    std::vector<uint32_t> row_start(size_t(n_rows) + 1, 0);
    ctx->h_cl_used.assign(size_t(n_rows), 0);
    std::vector<uint32_t> used_rows;
    const uint64_t kMaxMolecules = ((1ull << 53) - (1ull << 17)) >> 16;     // molecules x 2^16 + 2^17 stays below 2^53
    rc = validate_entries(ctx, fn, n, row, col, ref_cnt, alt_cnt, n_rows, n_cols, kMaxMolecules,
                          "its weighted sums would not be exact", [&](uint32_t v, uint64_t i0, uint64_t i1, uint64_t) {
        uint32_t with_ref = 0, with_alt = 0;
        for (uint64_t i = i0; i < i1; ++i) { with_ref += ref_cnt[i] > 0; with_alt += alt_cnt[i] > 0; }
        row_start[size_t(v) + 1] = uint32_t(i1 - i0);
        if (with_ref >= kMinCells && with_alt >= kMinCells) { ctx->h_cl_used[v] = 1; used_rows.push_back(v); }
    });
    if (rc) return rc;
    for (uint64_t v = 0; v < n_rows; ++v) row_start[v + 1] += row_start[v];

    cudaStream_t st = ctx->stream;
    ENS(ctx->cl_used, size_t(n_rows) + 1);
    ENS(ctx->cl_used_rows, used_rows.size() * 4 + 4);
    ENS(ctx->cl_row_start, row_start.size() * 4);
    const size_t tab = size_t(R) * size_t(n_rows) * K * 4 + 4;
    ENS(ctx->cl_la, tab); ENS(ctx->cl_lr, tab);
    ENS(ctx->cl_w, size_t(R) * n_cols * K * 4 + 4);
    const size_t flag_bytes = size_t(R + (R & 1)) * 4 + size_t(R) * 8;     // R changed flags, then R scores (8-aligned)
    ENS(ctx->cl_flags, flag_bytes);
    ENS(ctx->cl_A, size_t(n_rows) * K * 8 + 8); ENS(ctx->cl_T, size_t(n_rows) * K * 8 + 8);
    ENS(ctx->cl_ll, size_t(n_cols) * H * 8 + 8); ENS(ctx->cl_cnt, size_t(n_cols) * 24 + 8);
    if (n_rows) CK(cudaMemcpyAsync(ctx->cl_used.p, ctx->h_cl_used.data(), n_rows, cudaMemcpyHostToDevice, st));
    if (!used_rows.empty()) CK(cudaMemcpyAsync(ctx->cl_used_rows.p, used_rows.data(), used_rows.size() * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->cl_row_start.p, row_start.data(), row_start.size() * 4, cudaMemcpyHostToDevice, st));

    // the by-cell index of the used entries
    CellEntries ce;
    if ((rc = cell_entries(ctx, n, row, col, ref_cnt, alt_cnt, n_cols, &ce))) return rc;

    // the pinned samples' dosage and the row sums A_v, T_v over every entry (§5h's kernel)
    cluster_pinned::Pins pins{};
    if (J) {
        ENS(ctx->cp_dos, n_dos + 8);
        if (n_dos) CK(cudaMemcpyAsync(ctx->cp_dos.p, pin.dosage, n_dos, cudaMemcpyHostToDevice, st));
        if ((rc = pool_row_sums(ctx, n, n_rows, &pins.rowA, &pins.rowT))) return rc;
        pins.J = J; pins.m = pin.m; pins.fr = ambient::fractions(pin.error_rate);
        pins.dos = P<uint8_t>(ctx->cp_dos);
    }
    const uint32_t n_used = uint32_t(used_rows.size());
    // the pinned logs of the active restarts over §5g's tables
    auto pin_logs = [&](const Active& a) -> int {
        if (!J || !n_used || !a.n) return VTX_OK;
        const unsigned g = grid_for(ctx, uint64_t(a.n) * n_used * J, cluster_pinned::kCpThreads);
        cluster_pinned::vtx_k_cp_pin<<<g, cluster_pinned::kCpThreads, 0, st>>>(a, pins, n_used, P<uint32_t>(ctx->cl_used_rows), K, n_rows,
                                                                             P<int32_t>(ctx->cl_la), P<int32_t>(ctx->cl_lr));
        CK(cudaGetLastError());
        return VTX_OK;
    };

    // the EM: every active restart in the same launches; the host reads the restarts' flags and scores once per iteration
    if (n_used) {
        const unsigned igrid = grid_for(ctx, uint64_t(R) * n_used * K, kClThreads);
        vtx_k_cl_init<<<igrid, kClThreads, 0, st>>>(params->seed, R, K, n_used, P<uint32_t>(ctx->cl_used_rows), n_rows,
                                                     P<int32_t>(ctx->cl_la), P<int32_t>(ctx->cl_lr));
        CK(cudaGetLastError());
    }
    CK(cudaMemsetAsync(ctx->cl_w.p, 0xFF, size_t(R) * n_cols * K * 4, st));         // no weight is 2^32 - 1: the first E-step changes W
    ctx->h_cl_score.assign(R, 0);
    ctx->h_cl_iters.assign(R, 0);
    Active act{};
    for (uint32_t s = 0; s < R; ++s) act.s[act.n++] = uint8_t(s);
    rc = pin_logs(act);
    if (rc) return rc;
    uint32_t* d_changed = P<uint32_t>(ctx->cl_flags);
    unsigned long long* d_score = reinterpret_cast<unsigned long long*>(d_changed + R + (R & 1));
    std::vector<uint32_t> h_flags(flag_bytes / 4);
    for (uint32_t it = 1; act.n; ++it) {
        CK(cudaMemsetAsync(ctx->cl_flags.p, 0, flag_bytes, st));
        if (n_cols) {
            const unsigned g = grid_for(ctx, uint64_t(act.n) * n_cols * 32, kClThreads);
            vtx_k_cl_estep<<<g, kClThreads, 0, st>>>(act, ce, n_cols, n_rows, K, P<int32_t>(ctx->cl_la), P<int32_t>(ctx->cl_lr),
                                                     P<uint32_t>(ctx->cl_w), d_changed, d_score);
            CK(cudaGetLastError());
        }
        CK(cudaMemcpyAsync(h_flags.data(), ctx->cl_flags.p, flag_bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const uint64_t* h_score = reinterpret_cast<const uint64_t*>(h_flags.data() + R + (R & 1));
        Active next{};
        for (uint32_t i = 0; i < act.n; ++i) {
            const uint32_t s = act.s[i];
            ctx->h_cl_iters[s] = it;
            ctx->h_cl_score[s] = int64_t(h_score[s]);
            if (h_flags[s] && it < kMaxIters) next.s[next.n++] = uint8_t(s);
        }
        act = next;
        if (act.n && n_used) {
            const unsigned g = grid_for(ctx, uint64_t(act.n) * n_used * 32, kClThreads);
            vtx_k_cl_mstep<<<g, kClThreads, 0, st>>>(act, n_used, P<uint32_t>(ctx->cl_used_rows), P<uint32_t>(ctx->cl_row_start),
                                                     P<uint32_t>(ctx->cl_col), P<uint32_t>(ctx->cl_r), P<uint32_t>(ctx->cl_a),
                                                     P<uint32_t>(ctx->cl_w), n_cols, n_rows, K, P<int32_t>(ctx->cl_la), P<int32_t>(ctx->cl_lr));
            CK(cudaGetLastError());
            rc = pin_logs(act);
            if (rc) return rc;
        }
    }
    uint32_t best = 0;
    for (uint32_t s = 1; s < R; ++s)
        if (ctx->h_cl_score[s] > ctx->h_cl_score[best]) best = s;

    // canonical order: the best restart's clusters by sum_c W_ck, descending, ties by EM index (the pinned clusters keep theirs)
    std::vector<uint32_t> w_best(size_t(n_cols) * K);
    if (n_cols) CK(cudaMemcpy(w_best.data(), P<uint32_t>(ctx->cl_w) + size_t(best) * n_cols * K, w_best.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<uint64_t> tot(K, 0);
    for (size_t i = 0; i < w_best.size(); ++i) tot[i % K] += w_best[i];
    std::vector<uint32_t> order(K);
    for (uint32_t k = 0; k < K; ++k) order[k] = k;
    std::stable_sort(order.begin() + J, order.end(), [&](uint32_t x, uint32_t y) { return tot[x] > tot[y]; });
    Perm perm{};
    for (uint32_t j = 0; j < K; ++j) perm.k[j] = uint8_t(order[j]);

    // the final M-step over every row, then the scoring
    if (n_rows) {
        const unsigned g = grid_for(ctx, n_rows * 32, kClThreads);
        vtx_k_cl_final<<<g, kClThreads, 0, st>>>(perm, n_rows, P<uint32_t>(ctx->cl_row_start), P<uint32_t>(ctx->cl_col), P<uint32_t>(ctx->cl_r),
                                                 P<uint32_t>(ctx->cl_a), P<uint32_t>(ctx->cl_w) + size_t(best) * n_cols * K, K,
                                                 P<int64_t>(ctx->cl_A), P<int64_t>(ctx->cl_T));
        CK(cudaGetLastError());
    }
    if (n_cols) {
        const unsigned g = grid_for(ctx, uint64_t(n_cols) * 32, kClThreads, 8);
        const int64_t* A = P<int64_t>(ctx->cl_A);
        const int64_t* T = P<int64_t>(ctx->cl_T);
        int64_t* ll = P<int64_t>(ctx->cl_ll);
        uint64_t* cnt = P<uint64_t>(ctx->cl_cnt);
        // with J = 0 (vtx_cluster_cells) every lane takes theta(A, T)
        by_kh(H, [&](auto kh) {
            cluster_pinned::vtx_k_cl_score_pinned<decltype(kh)::value><<<g, kClThreads, 0, st>>>(ce, n_cols, K, pins, A, T, ll, cnt);
        });
        CK(cudaGetLastError());
    }
    ctx->h_cl_ll.resize(size_t(n_cols) * H);
    ctx->h_cl_cnt.resize(size_t(n_cols) * 3);
    ctx->h_cl_A.resize(size_t(n_rows) * K);
    ctx->h_cl_T.resize(size_t(n_rows) * K);
    if (n_cols) {
        CK(cudaMemcpyAsync(ctx->h_cl_ll.data(), ctx->cl_ll.p, ctx->h_cl_ll.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cl_cnt.data(), ctx->cl_cnt.p, ctx->h_cl_cnt.size() * 8, cudaMemcpyDeviceToHost, st));
    }
    if (n_rows) {
        CK(cudaMemcpyAsync(ctx->h_cl_A.data(), ctx->cl_A.p, ctx->h_cl_A.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cl_T.data(), ctx->cl_T.p, ctx->h_cl_T.size() * 8, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));

    out->k = K; out->n_cols = n_cols; out->n_hyp = H; out->best_restart = best;
    out->n_rows = n_rows; out->rows_used = n_used;
    out->ll = ctx->h_cl_ll.data(); out->counts = ctx->h_cl_cnt.data(); out->row_used = ctx->h_cl_used.data();
    out->alt_w = ctx->h_cl_A.data(); out->depth_w = ctx->h_cl_T.data();
    out->restart_score = ctx->h_cl_score.data(); out->restart_iters = ctx->h_cl_iters.data();
    return VTX_OK;
}

int vtx_cluster_cells(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                      const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const vtx_cluster_params* params, vtx_clusters* out)
{
    if (!ctx || !params || !out) return VTX_E_INVALID;
    *out = vtx_clusters{};
    const char* fn = "vtx_cluster_cells";
    if (int rc = check_finished(ctx, fn)) return rc;
    const uint32_t K = params->k, R = params->restarts;
    if (int rc = check_k(ctx, fn, K)) return rc;
    if (R < 1 || R > clusters::kMaxRestarts) return set_err(ctx, VTX_E_INVALID, "%s: %u restarts; 1 to 64 are supported", fn, R);
    return cluster_cells_run(ctx, fn, n, row, col, ref_cnt, alt_cnt, n_rows, n_cols, params, PinSpec{}, out);
}

int vtx_cluster_cells_pinned(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                             const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const uint8_t* dosage,
                             const vtx_cluster_pinned_params* params, vtx_clusters* out)
{
    if (!ctx || !params || !out) return VTX_E_INVALID;
    *out = vtx_clusters{};
    const char* fn = "vtx_cluster_cells_pinned";
    if (int rc = check_finished(ctx, fn)) return rc;
    const uint32_t K = params->k, R = params->restarts, J = params->n_pinned;
    if (int rc = check_k(ctx, fn, K)) return rc;
    if (R < 1 || R > clusters::kMaxRestarts) return set_err(ctx, VTX_E_INVALID, "%s: %u restarts; 1 to 64 are supported", fn, R);
    if (J < 1 || J >= K) return set_err(ctx, VTX_E_INVALID, "%s: %u pinned samples; 1 to k - 1 = %u are supported", fn, J, K - 1);
    if (!dosage) return set_err(ctx, VTX_E_INVALID, "%s: dosage is NULL", fn);
    if (int rc = check_error_rate(ctx, fn, params->error_rate)) return rc;
    if (params->rho_permille < 0 || params->rho_permille > ambient::kMaxPermille)
        return set_err(ctx, VTX_E_INVALID, "%s: rho_permille %d; 0 to 500", fn, params->rho_permille);
    const vtx_cluster_params cp{ K, R, params->seed };
    PinSpec pin;
    pin.J = J; pin.m = uint32_t(params->rho_permille); pin.error_rate = params->error_rate; pin.dosage = dosage;
    return cluster_cells_run(ctx, fn, n, row, col, ref_cnt, alt_cnt, n_rows, n_cols, &cp, pin, out);
}

int vtx_donors_ambient(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                       const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const uint8_t* dosage,
                       const vtx_ambient_params* params, vtx_ambient* out)
{
    using namespace ambient;
    if (!ctx || !params || !out) return VTX_E_INVALID;
    *out = vtx_ambient{};
    const char* fn = "vtx_donors_ambient";
    int rc = check_finished(ctx, fn);
    if (rc) return rc;
    const uint32_t D = params->n_donors;
    const int32_t given = params->rho_permille;
    if (D < donors::kMinDonors || D > donors::kMaxDonors)
        return set_err(ctx, VTX_E_INVALID, "vtx_donors_ambient: %u donors; 2 to 32 are supported", D);
    if ((rc = check_error_rate(ctx, fn, params->error_rate))) return rc;
    if (given < -1 || given > kMaxPermille)
        return set_err(ctx, VTX_E_INVALID, "vtx_donors_ambient: rho_permille %d; -1 (estimate) or 0 to 500", given);
    if (n && (!row || !col || !ref_cnt || !alt_cnt)) return set_err(ctx, VTX_E_INVALID, "vtx_donors_ambient: an entry array is NULL");
    if (n_rows && !dosage) return set_err(ctx, VTX_E_INVALID, "vtx_donors_ambient: dosage is NULL");
    if (n > 0xFFFFFFFFull || n_rows > 0xFFFFFFFFull)
        return set_err(ctx, VTX_E_INVALID, "vtx_donors_ambient: %llu entries over %llu rows; both must be below 2^32",
                       (unsigned long long)n, (unsigned long long)n_rows);
    const uint32_t H = donors::n_hyp(D);
    // device memory, before any host table of n_rows entries: the entries (16 B) and their by-cell copy (12 B); per row the used
    // flag, the touched index and A, T; per cell the index, the log-likelihoods and the counts.  One m's tables come below.
    // every buffer is allocated with 1/8 to spare (ensure), so both checks and the pass size count that margin
    constexpr double kSlack = 1.125;
    const double need = (double(n) * 28 + double(n_rows) * 21 + double(n_cols) * (8 + 24 + 8.0 * H)) * kSlack;
    double avail = 0;
    rc = check_free(ctx, fn, need, { &ctx->cl_row, &ctx->cl_col, &ctx->cl_r, &ctx->cl_a, &ctx->cl_used, &ctx->cl_cell_count,
                                     &ctx->cl_cell_start, &ctx->cl_c_row, &ctx->cl_c_r, &ctx->cl_c_a, &ctx->cl_ll, &ctx->cl_cnt,
                                     &ctx->am_sums, &ctx->am_tix, &ctx->am_touched, &ctx->am_dos, &ctx->am_tab, &ctx->am_grid }, &avail);
    if (rc) return rc;
    std::vector<uint8_t> usable(size_t(n_rows) + 1, 0);
    uint64_t rows_usable = 0;
    for (uint64_t v = 0; v < n_rows; ++v) {
        if ((rc = check_dosage_row(ctx, fn, dosage + size_t(v) * D, D, v, "donor"))) return rc;
        rows_usable += usable[v] = donors::row_usable(dosage + size_t(v) * D, D) ? 1 : 0;
    }
    // validate the entries in one pass; a usable row with an entry of r + a > 0 is "touched" and gets the next table index
    std::vector<uint32_t> tix(size_t(n_rows) + 1, 0), touched;
    rc = validate_entries(ctx, fn, n, row, col, ref_cnt, alt_cnt, n_rows, n_cols, kMaxRowDepth,
                          "its pool fraction would not be exact", [&](uint32_t v, uint64_t, uint64_t, uint64_t depth) {
        if (depth && usable[v]) { tix[v] = uint32_t(touched.size()); touched.push_back(v); }
    });
    if (rc) return rc;
    const uint32_t n_t = uint32_t(touched.size());
    std::vector<uint8_t> dos(size_t(n_t) * D + 1);
    for (uint32_t t = 0; t < n_t; ++t) memcpy(dos.data() + size_t(t) * D, dosage + size_t(touched[t]) * D, D);
    // the rest of the memory holds the tables of as many m as fit, at least one
    const double fixed = need + double(n_t) * (D + 4) * kSlack, per_m = double(n_t) * 40 * kSlack;
    if (fixed + per_m > avail)
        return set_err(ctx, VTX_E_NOMEM, "%s needs %.0f MB of device memory, %.0f MB are free", fn, (fixed + per_m) * 1e-6, avail * 1e-6);
    uint32_t batch = kMaxBatch;
    if (per_m > 0) batch = uint32_t(std::min(double(kMaxBatch), std::floor((avail - fixed) / per_m)));
    if (params->grid_batch) batch = std::min(batch, params->grid_batch);

    cudaStream_t st = ctx->stream;
    ENS(ctx->cl_used, usable.size());
    ENS(ctx->am_tix, tix.size() * 4);
    ENS(ctx->am_touched, size_t(n_t) * 4 + 4);
    ENS(ctx->am_dos, dos.size());
    ENS(ctx->cl_ll, size_t(n_cols) * H * 8 + 8); ENS(ctx->cl_cnt, size_t(n_cols) * 24 + 8);
    ENS(ctx->am_tab, size_t(batch) * n_t * 40 + 8);
    ENS(ctx->am_grid, size_t(kMaxBatch) * 4 * 8);
    CK(cudaMemcpyAsync(ctx->cl_used.p, usable.data(), usable.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->am_tix.p, tix.data(), tix.size() * 4, cudaMemcpyHostToDevice, st));
    if (n_t) {
        CK(cudaMemcpyAsync(ctx->am_touched.p, touched.data(), size_t(n_t) * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->am_dos.p, dos.data(), size_t(n_t) * D, cudaMemcpyHostToDevice, st));
    }

    // the by-cell index of the kept entries (§5g's kernels with used = the usable rows), then A_v, T_v
    clusters::CellEntries ce;
    if ((rc = cell_entries(ctx, n, row, col, ref_cnt, alt_cnt, n_cols, &ce))) return rc;
    const unsigned long long *d_A, *d_T;
    if ((rc = pool_row_sums(ctx, n, n_rows, &d_A, &d_T))) return rc;

    // J(m) and the calls of every m in `ms`, `batch` m per pass; with `final` (one m), also the cells' log-likelihoods
    const Fractions fr = fractions(params->error_rate);
    unsigned long long* d_J = P<unsigned long long>(ctx->am_grid);
    unsigned long long* d_calls = d_J + kMaxBatch;
    std::vector<unsigned long long> h_grid(size_t(kMaxBatch) * 4);
    auto evaluate = [&](const std::vector<uint16_t>& ms, bool final, std::vector<int64_t>* J, std::vector<uint64_t>* calls) -> int {
        for (size_t o = 0; o < ms.size(); o += batch) {
            Batch bt{};
            bt.n = uint32_t(std::min<size_t>(batch, ms.size() - o));
            for (uint32_t b = 0; b < bt.n; ++b) bt.m[b] = ms[o + b];
            CK(cudaMemsetAsync(ctx->am_grid.p, 0, h_grid.size() * 8, st));
            if (n_t) {
                const unsigned g = grid_for(ctx, uint64_t(bt.n) * n_t, kAmThreads);
                vtx_k_am_tables<<<g, kAmThreads, 0, st>>>(bt, fr, n_t, P<uint32_t>(ctx->am_touched), d_A, d_T, P<int32_t>(ctx->am_tab));
                CK(cudaGetLastError());
            }
            if (n_cols) {
                const unsigned g = grid_for(ctx, uint64_t(bt.n) * n_cols * 32, kAmThreads);
                const uint32_t* tx = P<uint32_t>(ctx->am_tix);
                const uint8_t* dd = P<uint8_t>(ctx->am_dos);
                const int32_t* tb = P<int32_t>(ctx->am_tab);
                int64_t* ll = final ? P<int64_t>(ctx->cl_ll) : nullptr;
                uint64_t* cnt = final ? P<uint64_t>(ctx->cl_cnt) : nullptr;
                by_kh(H, [&](auto kh) {
                    vtx_k_am_score<decltype(kh)::value><<<g, kAmThreads, 0, st>>>(bt, ce, n_cols, D, tx, dd, tb, n_t, d_J, d_calls, ll, cnt);
                });
                CK(cudaGetLastError());
            }
            CK(cudaMemcpyAsync(h_grid.data(), ctx->am_grid.p, h_grid.size() * 8, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (uint32_t b = 0; b < bt.n; ++b) {
                J->push_back(int64_t(h_grid[b]));
                for (int k = 0; k < 3; ++k) calls->push_back(h_grid[kMaxBatch + 3 * size_t(b) + k]);
            }
        }
        return VTX_OK;
    };
    std::vector<uint16_t> ms;
    std::vector<int64_t> obj;
    std::vector<uint64_t> calls;
    uint32_t chosen = uint32_t(given);
    if (given < 0) {
        rc = estimate_permille(ms, obj, [&](const std::vector<uint16_t>& list) { return evaluate(list, false, &obj, &calls); }, &chosen);
        if (rc) return rc;
    }
    std::vector<int64_t> obj_f;
    std::vector<uint64_t> calls_f;
    rc = evaluate({ uint16_t(chosen) }, true, &obj_f, &calls_f);
    if (rc) return rc;
    if (given >= 0) { ms.assign(1, uint16_t(chosen)); obj = obj_f; calls = calls_f; }
    sort_grid(ms, obj, &calls, ctx->h_am_m, ctx->h_am_obj, &ctx->h_am_calls);

    ctx->h_am_ll.resize(size_t(n_cols) * H);
    ctx->h_am_cnt.resize(size_t(n_cols) * 3);
    ctx->h_am_alt.resize(size_t(n_rows));
    ctx->h_am_depth.resize(size_t(n_rows));
    if (n_cols) {
        CK(cudaMemcpyAsync(ctx->h_am_ll.data(), ctx->cl_ll.p, ctx->h_am_ll.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_am_cnt.data(), ctx->cl_cnt.p, ctx->h_am_cnt.size() * 8, cudaMemcpyDeviceToHost, st));
    }
    if (n_rows) {
        CK(cudaMemcpyAsync(ctx->h_am_alt.data(), d_A, size_t(n_rows) * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_am_depth.data(), d_T, size_t(n_rows) * 8, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));

    out->n_donors = D; out->n_cols = n_cols; out->n_hyp = H; out->rho_permille = chosen; out->n_evaluated = uint32_t(ms.size());
    out->n_rows = n_rows; out->rows_usable = rows_usable;
    out->ll = ctx->h_am_ll.data(); out->counts = ctx->h_am_cnt.data();
    out->grid_permille = ctx->h_am_m.data(); out->grid_objective = ctx->h_am_obj.data(); out->grid_calls = ctx->h_am_calls.data();
    out->row_alt = ctx->h_am_alt.data(); out->row_depth = ctx->h_am_depth.data();
    return VTX_OK;
}

int vtx_cluster_genotypes(vtx_ctx* ctx, uint64_t n_rows, const int64_t* alt_w, const int64_t* depth_w, const uint8_t* row_used,
                          const uint64_t* row_alt, const uint64_t* row_depth, const uint8_t* dosage,
                          const vtx_cluster_gt_params* params, vtx_cluster_gt* out)
{
    using namespace cluster_gt;
    if (!ctx || !params || !out) return VTX_E_INVALID;
    *out = vtx_cluster_gt{};
    const char* fn = "vtx_cluster_genotypes";
    int rc = check_finished(ctx, fn);
    if (rc) return rc;
    const uint32_t K = params->k, S = params->n_samples;
    const int32_t given = params->rho_permille;
    if ((rc = check_k(ctx, fn, K))) return rc;
    if (S > kMaxSamples) return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: %u samples; 0 to 1024 are supported", S);
    if (S && !dosage) return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: dosage is NULL");
    if ((rc = check_error_rate(ctx, fn, params->error_rate))) return rc;
    if (given < -1 || given > ambient::kMaxPermille)
        return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: rho_permille %d; -1 (estimate) or 0 to 500", given);
    if (n_rows && (!alt_w || !depth_w || !row_used || !row_alt || !row_depth))
        return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: a row array is NULL");
    if (n_rows > 0xFFFFFFFFull)
        return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: %llu rows; must be below 2^32", (unsigned long long)n_rows);

    // validate in one pass, and list the touched rows (T_kv > 0 for some k), the fitted ones (used and touched) and the compared
    // ones (touched, every sample has a dosage)
    std::vector<uint32_t> touched, fit, cmp;
    uint64_t total = 0, rows_compared = 0;
    for (uint64_t v = 0; v < n_rows; ++v) {
        if ((rc = check_sums_row(ctx, fn, alt_w + v * K, depth_w + v * K, K, v, &total))) return rc;
        const bool reached = std::any_of(depth_w + v * K, depth_w + (v + 1) * K, [](int64_t t) { return t > 0; });
        if (row_alt[v] > row_depth[v] || row_depth[v] > ambient::kMaxRowDepth)
            return set_err(ctx, VTX_E_INVALID, "vtx_cluster_genotypes: row %llu: row_alt %llu, row_depth %llu (row_alt <= row_depth < 2^53 - 2)",
                           (unsigned long long)v, (unsigned long long)row_alt[v], (unsigned long long)row_depth[v]);
        if ((rc = check_dosage_row(ctx, fn, dosage + v * S, S, v, "sample"))) return rc;
        const bool all = S > 0 && std::none_of(dosage + v * S, dosage + (v + 1) * S, [](uint8_t g) { return g == kMissing; });
        rows_compared += all;
        if (!reached) continue;
        if (row_used[v]) fit.push_back(uint32_t(touched.size()));
        if (all) cmp.push_back(uint32_t(touched.size()));
        touched.push_back(uint32_t(v));
    }
    const uint32_t n_t = uint32_t(touched.size()), n_fit = uint32_t(fit.size()), n_cmp = uint32_t(cmp.size());
    // every buffer is allocated with 1/8 to spare (ensure)
    const double need = (double(n_t) * (53.0 * K + 16) + double(n_fit) * 4 + double(n_cmp) * (4.0 + S) + 16.0 * K * (S + 1) + 4096) * 1.125;
    rc = check_free(ctx, fn, need, { &ctx->cg_AT, &ctx->cg_rows, &ctx->cg_fit, &ctx->cg_ll, &ctx->cg_gt, &ctx->cg_pl, &ctx->cg_cmp,
                                     &ctx->cg_dos, &ctx->cg_acc });
    if (rc) return rc;
    // the touched rows' inputs, compacted: A, T [touched][K], then A_v, T_v [touched]; the compared rows' dosages
    std::vector<int64_t> at(size_t(n_t) * K * 2);
    std::vector<uint64_t> rows(size_t(n_t) * 2);
    for (uint32_t i = 0; i < n_t; ++i) {
        const size_t v = touched[i];
        memcpy(at.data() + size_t(i) * K, alt_w + v * K, size_t(K) * 8);
        memcpy(at.data() + (size_t(n_t) + i) * K, depth_w + v * K, size_t(K) * 8);
        rows[i] = row_alt[v];
        rows[n_t + i] = row_depth[v];
    }
    std::vector<uint8_t> dos(size_t(n_cmp) * S);
    for (uint32_t i = 0; i < n_cmp; ++i) memcpy(dos.data() + size_t(i) * S, dosage + size_t(touched[cmp[i]]) * S, S);

    cudaStream_t st = ctx->stream;
    ENS(ctx->cg_AT, at.size() * 8 + 8);
    ENS(ctx->cg_rows, rows.size() * 8 + 8);
    ENS(ctx->cg_fit, size_t(n_fit) * 4 + 4);
    ENS(ctx->cg_cmp, size_t(n_cmp) * 4 + 4);
    ENS(ctx->cg_dos, dos.size() + 8);
    ENS(ctx->cg_acc, (size_t(ambient::kMaxBatch) + 2 * size_t(K) * S + 2 * K) * 8);
    if (n_t) {
        CK(cudaMemcpyAsync(ctx->cg_AT.p, at.data(), at.size() * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->cg_rows.p, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, st));
    }
    if (n_fit) CK(cudaMemcpyAsync(ctx->cg_fit.p, fit.data(), size_t(n_fit) * 4, cudaMemcpyHostToDevice, st));
    if (n_cmp) {
        CK(cudaMemcpyAsync(ctx->cg_cmp.p, cmp.data(), size_t(n_cmp) * 4, cudaMemcpyHostToDevice, st));
        if (S) CK(cudaMemcpyAsync(ctx->cg_dos.p, dos.data(), dos.size(), cudaMemcpyHostToDevice, st));
    }
    const int64_t* d_A = P<int64_t>(ctx->cg_AT);
    const int64_t* d_T = d_A + size_t(n_t) * K;
    const unsigned long long* d_rowA = P<unsigned long long>(ctx->cg_rows);
    const unsigned long long* d_rowT = d_rowA + n_t;
    unsigned long long* d_J = P<unsigned long long>(ctx->cg_acc);
    const ambient::Fractions fr = ambient::fractions(params->error_rate);

    // the fit and the calls at the chosen m, then the match
    std::vector<uint16_t> ms;
    std::vector<int64_t> obj;
    uint32_t chosen = 0;
    rc = cg_fit_device(ctx, fr, K, given, n_t, n_fit, P<uint32_t>(ctx->cg_fit), d_rowA, d_rowT, d_A, d_T, ms, obj, &chosen);
    if (rc) return rc;
    unsigned long long* d_M = d_J + ambient::kMaxBatch;
    const size_t n_acc = 2 * size_t(K) * S + 2 * K;                   // M, discordant [K][S], then rows, called [K]
    CK(cudaMemsetAsync(d_M, 0, n_acc * 8, st));
    if (S && n_cmp) {
        const uint32_t ys = (S + kMatchSamples - 1) / kMatchSamples;
        // about four CTAs per SM in all, each over whole tiles of rows
        const uint64_t xs_want = std::max<uint64_t>(1, uint64_t(ctx->n_sm) * 4 / ys);
        const uint64_t tiles = (n_cmp + kMatchRows - 1) / kMatchRows;
        const uint32_t rows_per_cta = uint32_t((tiles + xs_want - 1) / xs_want) * kMatchRows;
        const uint32_t xs = uint32_t((n_cmp + rows_per_cta - 1) / rows_per_cta);
        vtx_k_cg_match<<<dim3(xs, ys), kCgThreads, 0, st>>>(K, S, n_cmp, rows_per_cta, P<uint32_t>(ctx->cg_cmp), P<uint8_t>(ctx->cg_dos),
                                                             P<int64_t>(ctx->cg_ll), P<uint8_t>(ctx->cg_gt), P<uint32_t>(ctx->cg_pl), d_M,
                                                             d_M + size_t(K) * S, d_M + 2 * size_t(K) * S, d_M + 2 * size_t(K) * S + K);
        CK(cudaGetLastError());
    }
    ctx->h_cg_gt.resize(size_t(n_t) * K);
    ctx->h_cg_pl.resize(size_t(n_t) * K * 3);
    ctx->h_cg_acc.resize(n_acc);
    if (n_t) {
        CK(cudaMemcpyAsync(ctx->h_cg_gt.data(), ctx->cg_gt.p, ctx->h_cg_gt.size(), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cg_pl.data(), ctx->cg_pl.p, ctx->h_cg_pl.size() * 4, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaMemcpyAsync(ctx->h_cg_acc.data(), d_M, n_acc * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));

    sort_grid(ms, obj, nullptr, ctx->h_cg_m, ctx->h_cg_obj, nullptr);
    ctx->h_cg_touched.assign(touched.begin(), touched.end());
    ctx->h_cg_M.resize(size_t(K) * S);
    for (size_t i = 0; i < ctx->h_cg_M.size(); ++i) ctx->h_cg_M[i] = int64_t(ctx->h_cg_acc[i]);

    out->k = K; out->n_samples = S; out->rho_permille = chosen; out->n_evaluated = uint32_t(ms.size());
    out->n_rows = n_rows; out->rows_fit = n_fit; out->n_touched = n_t; out->rows_compared = rows_compared;
    out->grid_permille = ctx->h_cg_m.data(); out->grid_objective = ctx->h_cg_obj.data();
    out->touched = ctx->h_cg_touched.data(); out->gt = ctx->h_cg_gt.data(); out->pl = ctx->h_cg_pl.data();
    out->match_ll = ctx->h_cg_M.data(); out->match_discordant = ctx->h_cg_acc.data() + size_t(K) * S;
    out->match_rows = ctx->h_cg_acc.data() + 2 * size_t(K) * S; out->match_called = out->match_rows + K;
    return VTX_OK;
}

int vtx_cluster_refine(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                       const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const int64_t* alt_w, const int64_t* depth_w,
                       const uint8_t* row_used, const vtx_cluster_calls_params* params, vtx_cluster_calls* out)
{
    using namespace cluster_refine;
    if (!ctx || !params || !out) return VTX_E_INVALID;
    *out = vtx_cluster_calls{};
    const char* fn = "vtx_cluster_refine";
    int rc = check_finished(ctx, fn);
    if (rc) return rc;
    const uint32_t K = params->k, max_rounds = params->max_rounds;
    if ((rc = check_k(ctx, fn, K))) return rc;
    if ((rc = check_error_rate(ctx, fn, params->error_rate))) return rc;
    if (max_rounds > kMaxRounds) return set_err(ctx, VTX_E_INVALID, "vtx_cluster_refine: max_rounds %u; 0 to 32 are supported", max_rounds);
    if (n && (!row || !col || !ref_cnt || !alt_cnt)) return set_err(ctx, VTX_E_INVALID, "vtx_cluster_refine: an entry array is NULL");
    if (n_rows && (!alt_w || !depth_w || !row_used)) return set_err(ctx, VTX_E_INVALID, "vtx_cluster_refine: a row array is NULL");
    if (n > 0xFFFFFFFFull || n_rows > 0xFFFFFFFFull)
        return set_err(ctx, VTX_E_INVALID, "vtx_cluster_refine: %llu entries over %llu rows; both must be below 2^32",
                       (unsigned long long)n, (unsigned long long)n_rows);
    const uint32_t H = donors::n_hyp(K);
    // device memory, before any host table of n_rows entries: the entries (16 B) and their by-cell copy (12 B); per row the flags,
    // scans, row sums and the round's sums, and at most every row touched and scored (the compacted fit, codes and tables); per
    // cell the weights, labels, log-likelihoods and counts.  Every buffer is allocated with 1/8 to spare (ensure).
    const double need = (double(n) * 28 + double(n_rows) * (70.0 * K + 150) + double(n_cols) * (4.0 * K + 8.0 * H + 40) + 4096) * 1.125;
    rc = check_free(ctx, fn, need, { &ctx->cl_row, &ctx->cl_col, &ctx->cl_r, &ctx->cl_a, &ctx->cl_used, &ctx->cl_row_start,
                                     &ctx->cl_cell_count, &ctx->cl_cell_start, &ctx->cl_c_row, &ctx->cl_c_r, &ctx->cl_c_a, &ctx->cl_w,
                                     &ctx->cl_A, &ctx->cl_T, &ctx->cl_ll, &ctx->cl_cnt, &ctx->am_sums, &ctx->cg_AT, &ctx->cg_rows,
                                     &ctx->cg_fit, &ctx->cg_ll, &ctx->cg_gt, &ctx->cg_pl, &ctx->cg_acc, &ctx->cr_rowflags, &ctx->cr_code,
                                     &ctx->cr_sflag, &ctx->cr_scode, &ctx->cr_tab, &ctx->cr_label, &ctx->cr_scal });
    if (rc) return rc;
    // validate once: §5i's bounds on the sums, then the entries, whose total bounds every later round's hard sums
    uint64_t total = 0;
    for (uint64_t v = 0; v < n_rows; ++v)
        if ((rc = check_sums_row(ctx, fn, alt_w + v * K, depth_w + v * K, K, v, &total))) return rc;
    std::vector<uint32_t> row_start(size_t(n_rows) + 1, 0);
    uint64_t molecules = 0;
    rc = validate_entries(ctx, fn, n, row, col, ref_cnt, alt_cnt, n_rows, n_cols, kMaxTotalMolecules,
                          "its hard sums would not be exact", [&](uint32_t v, uint64_t i0, uint64_t i1, uint64_t m) {
        row_start[size_t(v) + 1] = uint32_t(i1 - i0);
        molecules += m;
    });
    if (rc) return rc;
    if (molecules > kMaxTotalMolecules)
        return set_err(ctx, VTX_E_INVALID, "vtx_cluster_refine: the entries hold more than 2^35 molecules; the fit's int64 sums would not be exact");
    for (uint64_t v = 0; v < n_rows; ++v) row_start[v + 1] += row_start[v];

    cudaStream_t st = ctx->stream;
    ENS(ctx->cl_used, size_t(n_rows) + 1);
    ENS(ctx->cl_row_start, row_start.size() * 4);
    ENS(ctx->cl_w, size_t(n_cols) * K * 4 + 4);
    ENS(ctx->cl_A, size_t(n_rows) * K * 8 + 8); ENS(ctx->cl_T, size_t(n_rows) * K * 8 + 8);
    ENS(ctx->cl_ll, size_t(n_cols) * H * 8 + 8); ENS(ctx->cl_cnt, size_t(n_cols) * 24 + 8);
    ENS(ctx->cg_acc, size_t(ambient::kMaxBatch) * 8);
    const size_t rf = size_t(n_rows) + 1;                   // tflag, tpos, fflag, fpos, sidx: n_rows + 1 each
    ENS(ctx->cr_rowflags, rf * 5 * 4);
    ENS(ctx->cr_label, size_t(n_cols) * 8 + 8);
    ENS(ctx->cr_scal, 4 * 8);
    CK(cudaMemcpyAsync(ctx->cl_row_start.p, row_start.data(), row_start.size() * 4, cudaMemcpyHostToDevice, st));
    if (n_rows) {
        CK(cudaMemcpyAsync(ctx->cl_A.p, alt_w, size_t(n_rows) * K * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ctx->cl_T.p, depth_w, size_t(n_rows) * K * 8, cudaMemcpyHostToDevice, st));
    }

    // the by-cell index of every entry with r + a > 0 (§5g's kernels with every row kept), then A_v, T_v; then `used` becomes row_used
    CK(cudaMemsetAsync(ctx->cl_used.p, 1, size_t(n_rows) + 1, st));
    clusters::CellEntries ce;
    if ((rc = cell_entries(ctx, n, row, col, ref_cnt, alt_cnt, n_cols, &ce))) return rc;
    const unsigned long long *d_rowA, *d_rowT;
    if ((rc = pool_row_sums(ctx, n, n_rows, &d_rowA, &d_rowT))) return rc;
    if (n_rows) CK(cudaMemcpyAsync(ctx->cl_used.p, row_used, n_rows, cudaMemcpyHostToDevice, st));
    uint32_t* d_tflag = P<uint32_t>(ctx->cr_rowflags);
    uint32_t* d_tpos = d_tflag + rf;
    uint32_t* d_fflag = d_tpos + rf;
    uint32_t* d_fpos = d_fflag + rf;
    uint32_t* d_sidx = d_fpos + rf;
    uint32_t* d_label = P<uint32_t>(ctx->cr_label);
    uint32_t* d_prev = d_label + n_cols;
    unsigned long long* d_scal = P<unsigned long long>(ctx->cr_scal);       // calls [3], changed
    CK(cudaMemsetAsync(d_prev, 0xFF, size_t(n_cols) * 4, st));              // round 0 compares with VTX_NO_LABEL

    const ambient::Fractions fr = ambient::fractions(params->error_rate);
    const unsigned rgrid = grid_for(ctx, n_rows, kCrThreads);
    clusters::Perm ident{};
    for (uint32_t k = 0; k < K; ++k) ident.k[k] = uint8_t(k);
    ctx->h_cr_rounds.clear();
    bool converged = false;
    uint32_t n_t = 0;
    for (uint32_t r = 0;; ++r) {
        if (r > 0 && n_rows) {       // the previous round's labels' hard sums
            const unsigned g = grid_for(ctx, n_rows * 32, clusters::kClThreads);
            clusters::vtx_k_cl_final<<<g, clusters::kClThreads, 0, st>>>(ident, n_rows, P<uint32_t>(ctx->cl_row_start), P<uint32_t>(ctx->cl_col),
                                                                         P<uint32_t>(ctx->cl_r), P<uint32_t>(ctx->cl_a), P<uint32_t>(ctx->cl_w), K,
                                                                         P<int64_t>(ctx->cl_A), P<int64_t>(ctx->cl_T));
            CK(cudaGetLastError());
        }
        // the touched and fitted rows, compacted on the device
        uint32_t counts[2] = { 0, 0 };
        if (n_rows) {
            vtx_k_cr_touch<<<rgrid, kCrThreads, 0, st>>>(n_rows, K, P<int64_t>(ctx->cl_T), P<uint8_t>(ctx->cl_used), d_tflag, d_fflag);
            CK(cudaGetLastError());
            rc = scan_u32(ctx, st, ctx->scan_sums, d_tflag, n_rows, d_tpos, nullptr);
            if (rc) return rc;
            rc = scan_u32(ctx, st, ctx->scan_sums, d_fflag, n_rows, d_fpos, nullptr);
            if (rc) return rc;
            CK(cudaMemcpyAsync(&counts[0], d_tpos + n_rows, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(&counts[1], d_fpos + n_rows, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        n_t = counts[0];
        const uint32_t n_fit = counts[1];
        ENS(ctx->cg_AT, size_t(n_t) * K * 16 + 8);
        ENS(ctx->cg_rows, size_t(n_t) * 16 + 8);
        ENS(ctx->cg_fit, size_t(n_fit) * 4 + 4);
        ENS(ctx->cr_sflag, (size_t(n_t) * 3 + 1) * 4);        // sflag, spos (n_t + 1), trow
        ENS(ctx->cr_code, size_t(n_t) * K + 8);
        int64_t* d_cA = P<int64_t>(ctx->cg_AT);
        int64_t* d_cT = d_cA + size_t(n_t) * K;
        unsigned long long* d_crow = P<unsigned long long>(ctx->cg_rows);
        uint32_t* d_sflag = P<uint32_t>(ctx->cr_sflag);
        uint32_t* d_spos = d_sflag + n_t;
        uint32_t* d_trow = d_spos + n_t + 1;
        if (n_t) {
            vtx_k_cr_gather<<<rgrid, kCrThreads, 0, st>>>(n_rows, K, n_t, P<int64_t>(ctx->cl_A), P<int64_t>(ctx->cl_T), d_rowA, d_rowT, d_tflag,
                                                          d_tpos, d_fflag, d_fpos, d_cA, d_cT, d_crow, d_trow, P<uint32_t>(ctx->cg_fit));
            CK(cudaGetLastError());
        }
        // §5i's fit and calls, then the codes and the scored rows' tables
        std::vector<uint16_t> ms;
        std::vector<int64_t> obj;
        uint32_t m = 0;
        rc = cg_fit_device(ctx, fr, K, -1, n_t, n_fit, P<uint32_t>(ctx->cg_fit), d_crow, d_crow + n_t, d_cA, d_cT, ms, obj, &m);
        if (rc) return rc;
        uint32_t n_s = 0;
        if (n_t) {
            const unsigned g = grid_for(ctx, n_t, kCrThreads);
            vtx_k_cr_codes<<<g, kCrThreads, 0, st>>>(n_t, K, P<uint8_t>(ctx->cg_gt), P<uint32_t>(ctx->cg_pl), P<uint8_t>(ctx->cr_code), d_sflag);
            CK(cudaGetLastError());
            rc = scan_u32(ctx, st, ctx->scan_sums, d_sflag, n_t, d_spos, nullptr);
            if (rc) return rc;
            CK(cudaMemcpyAsync(&n_s, d_spos + n_t, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        ENS(ctx->cr_scode, size_t(n_s) * K + 8);
        ENS(ctx->cr_tab, size_t(n_s) * kEntries * 8 + 8);
        if (n_rows) CK(cudaMemsetAsync(d_sidx, 0xFF, size_t(n_rows) * 4, st));
        if (n_s) {
            const unsigned g = grid_for(ctx, n_t, kCrThreads);
            vtx_k_cr_tables<<<g, kCrThreads, 0, st>>>(m, fr, n_t, K, d_trow, d_crow, P<uint8_t>(ctx->cr_code), d_sflag, d_spos, d_sidx,
                                                      P<uint8_t>(ctx->cr_scode), P<int32_t>(ctx->cr_tab));
            CK(cudaGetLastError());
        }
        // the cells: scores, calls and labels; the next round's weights and the changed labels
        CK(cudaMemsetAsync(d_scal, 0, 4 * 8, st));
        if (n_cols) {
            const unsigned g = grid_for(ctx, uint64_t(n_cols) * 32, kCrThreads, 8);
            const uint32_t* sx = d_sidx;
            const uint8_t* sc = P<uint8_t>(ctx->cr_scode);
            const int32_t* tb = P<int32_t>(ctx->cr_tab);
            int64_t* ll = P<int64_t>(ctx->cl_ll);
            uint64_t* cnt = P<uint64_t>(ctx->cl_cnt);
            by_kh(H, [&](auto kh) {
                vtx_k_cr_score<decltype(kh)::value><<<g, kCrThreads, 0, st>>>(ce, n_cols, K, sx, sc, tb, ll, cnt, d_label, d_scal);
            });
            CK(cudaGetLastError());
            const unsigned wg = grid_for(ctx, n_cols, kCrThreads);
            vtx_k_cr_weights<<<wg, kCrThreads, 0, st>>>(n_cols, K, d_label, d_prev, P<uint32_t>(ctx->cl_w), d_scal + 3);
            CK(cudaGetLastError());
        }
        unsigned long long h_scal[4];
        CK(cudaMemcpyAsync(h_scal, d_scal, sizeof(h_scal), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        vtx_cluster_calls_round rr{};
        rr.rho_permille = m; rr.rows_fit = n_fit; rr.n_touched = n_t; rr.rows_scored = n_s;
        for (int i = 0; i < 3; ++i) rr.calls[i] = h_scal[i];
        rr.changed = h_scal[3];
        ctx->h_cr_rounds.push_back(rr);
        if (r > 0 && rr.changed == 0) { converged = true; break; }
        if (r == max_rounds) break;
    }

    // the last round's cells and fit
    ctx->h_cr_ll.resize(size_t(n_cols) * H);
    ctx->h_cr_cnt.resize(size_t(n_cols) * 3);
    ctx->h_cr_label.resize(n_cols);
    std::vector<uint32_t> trow(n_t);
    ctx->h_cr_gt.resize(size_t(n_t) * K);
    ctx->h_cr_pl.resize(size_t(n_t) * K * 3);
    if (n_cols) {
        CK(cudaMemcpyAsync(ctx->h_cr_ll.data(), ctx->cl_ll.p, ctx->h_cr_ll.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cr_cnt.data(), ctx->cl_cnt.p, ctx->h_cr_cnt.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cr_label.data(), d_label, size_t(n_cols) * 4, cudaMemcpyDeviceToHost, st));
    }
    if (n_t) {
        CK(cudaMemcpyAsync(trow.data(), P<uint32_t>(ctx->cr_sflag) + 2 * size_t(n_t) + 1, size_t(n_t) * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cr_gt.data(), ctx->cg_gt.p, ctx->h_cr_gt.size(), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_cr_pl.data(), ctx->cg_pl.p, ctx->h_cr_pl.size() * 4, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    ctx->h_cr_touched.assign(trow.begin(), trow.end());

    out->k = K; out->n_cols = n_cols; out->n_hyp = H; out->n_rounds = uint32_t(ctx->h_cr_rounds.size()); out->converged = converged;
    out->n_rows = n_rows; out->n_touched = n_t;
    out->ll = ctx->h_cr_ll.data(); out->counts = ctx->h_cr_cnt.data(); out->label = ctx->h_cr_label.data();
    out->rounds = ctx->h_cr_rounds.data();
    out->touched = ctx->h_cr_touched.data(); out->gt = ctx->h_cr_gt.data(); out->pl = ctx->h_cr_pl.data();
    return VTX_OK;
}

uint64_t vtx_pack_cb(const uint8_t* s, uint32_t len) { return (s || len == 0) ? stage::pack_cb(s, len) : VTX_NO_CB_KEY; }

int vtx_sync(vtx_ctx* ctx)
{
    if (!ctx) return VTX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    return VTX_OK;
}

int vtx_wait_copies(vtx_ctx* ctx)
{
    if (!ctx) return VTX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->copy_stream));
    return VTX_OK;
}

static int finish_scalars(vtx_ctx* ctx)
{
    CK(cudaSetDevice(ctx->device));
    uint64_t* hs = ctx->h_scalars.as<uint64_t>();
    CK(cudaMemcpyAsync(hs, ctx->d_res_n.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(hs + 1, ctx->d_metrics.p, 48, cudaMemcpyDeviceToHost, ctx->stream));
    const uint64_t sn = ctx->finished ? 0 : ctx->stats_n;          // vtx_set_locus_stats: the entries travel with the scalars
    if (sn) {
        if (sn > ctx->h_lstats_cap) {
            const size_t ncap = size_t(sn) + size_t(sn) / 4 + 1024;
            const cudaError_t e = ctx->h_lstats.alloc(ncap * sizeof(vtx_locus_stats));
            if (e != cudaSuccess) { ctx->h_lstats_cap = 0; return set_err(ctx, VTX_E_NOMEM, "pinned locus statistics alloc failed: %s", cudaGetErrorString(e)); }
            ctx->h_lstats_cap = ncap;
        }
        CK(cudaMemcpyAsync(ctx->h_lstats.p, ctx->lstats.p, size_t(sn) * sizeof(vtx_locus_stats), cudaMemcpyDeviceToHost, ctx->stream));
    }
    uint64_t donor_bad = 0;
    if (ctx->donors) {          // vtx_set_donors: the accumulator travels with the scalars too (zeros when nothing was submitted)
        const uint32_t cols = ctx->finished ? ctx->n_barcodes : ctx->donor_cols;
        const size_t bytes = donor_acc_bytes(cols, donors::n_hyp(ctx->n_donors));
        if (bytes > ctx->h_donor_cap) {
            ctx->donor_valid = false;
            const cudaError_t e = ctx->h_donor.alloc(bytes);
            if (e != cudaSuccess) { ctx->h_donor_cap = 0; return set_err(ctx, VTX_E_NOMEM, "pinned donor log-likelihood alloc failed: %s", cudaGetErrorString(e)); }
            ctx->h_donor_cap = bytes;
        }
        if (ctx->finished) memset(ctx->h_donor.p, 0, bytes);
        else CK(cudaMemcpyAsync(ctx->h_donor.p, ctx->donor_acc.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        memcpy(&donor_bad, ctx->h_donor.as<uint8_t>() + bytes - 8, 8);
        ctx->donor_last_cols = cols;
        ctx->donor_valid = true;
    }
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->stats_last_n = sn;
    ctx->stats_n = 0;
    const uint64_t violated = ctx->finished ? 0 : hs[5], band_overflow = ctx->finished ? 0 : hs[6];
    ctx->last_n = ctx->finished ? 0 : hs[0];
    ctx->last_metrics.num_not_cell_bc = ctx->finished ? 0 : hs[1];
    ctx->last_metrics.num_non_umi = ctx->finished ? 0 : hs[2];
    ctx->last_metrics.num_scored = ctx->finished ? 0 : hs[3];
    ctx->t_pairs = ctx->last_metrics.num_scored;
    ctx->finished = true;
    if (band_overflow)
        return set_err(ctx, VTX_E_UNSUPPORTED, "band model: %llu alignments had more k-mer hits than the work buffers hold (reads x windows too large); "
                                               "they were scored with the full matrix", (unsigned long long)band_overflow);
    if (donor_bad)
        return set_err(ctx, VTX_E_INVALID, "%llu loci have a row outside the donor dosage table given to vtx_set_donors (%llu rows); "
                                           "they were left out of the donor log-likelihoods", (unsigned long long)donor_bad,
                       (unsigned long long)ctx->donor_rows);
    if (violated)
        return set_err(ctx, VTX_E_INVALID, "%llu loci of a device batch exceeded the bounds given to vtx_submit_device(_ex) (longest read / widest "
                                           "haplotype window); they were skipped, the result is incomplete", (unsigned long long)violated);
    return VTX_OK;
}

int vtx_finish_device(vtx_ctx* ctx, vtx_result* out)
{
    Nvtx nvtx_range("vtx_finish_device");
    if (!ctx || !out) return VTX_E_INVALID;
    int rc = finish_scalars(ctx);
    if (rc) return rc;
    point_result(out, ptrs(ctx->res), 0x7Fu, ctx->last_n, ctx->last_metrics);
    return VTX_OK;
}

int vtx_fetch(vtx_ctx* ctx, const vtx_result* device_result, vtx_result* out)
{
    Nvtx nvtx_range("vtx_fetch");
    if (!ctx || !device_result || !out) return VTX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    // gathered results get their own host buffers so that a local and a gathered copy can coexist
    const bool gathered = device_result->row == ctx->g_dev[0].p && ctx->g_dev[0].p != nullptr;
    HostResults& h = gathered ? ctx->g_host : ctx->h_res;
    const vtx_result& dev = *device_result;
    const size_t n = dev.n;
    int rc = ensure_host(ctx, h, n);
    if (rc) return rc;
    if (n) {
        rc = copy_results(ctx, h, { dev.row, dev.col, dev.ref_cnt, dev.alt_cnt, dev.unk_cnt, dev.val, dev.val2 }, 0, n, ctx->stream);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
    }
    point_result(out, ptrs(h.a), want_mask(ctx), n, dev.metrics);
    return VTX_OK;
}

int vtx_finish(vtx_ctx* ctx, vtx_result* out)
{
    Nvtx nvtx_range("vtx_finish");
    if (!ctx || !out) return VTX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    // Stream the triplets out submit by submit: the kernels of later submits are usually still running when the
    // host gets here, so the device->host copy of everything but the last shard hides behind them.
    const auto src = ptrs(ctx->res);
    size_t fetched = 0;
    const bool streamed = !ctx->finished && ctx->h_cum.p && ctx->fetch_stream && ctx->trec_used > 0 && ctx->trec_used <= kMaxCum;
    if (streamed) {
        int rc = ensure_host(ctx, ctx->h_res, ctx->res_ub);
        if (rc) return rc;
        for (size_t i = 0; i < ctx->trec_used; ++i) {
            CK(cudaEventSynchronize(ctx->trecs[i].ev[EV_POST]));
            const size_t n_i = size_t(ctx->h_cum.as<unsigned long long>()[i]);
            if (n_i > fetched && n_i <= ctx->h_res.cap) {
                rc = copy_results(ctx, ctx->h_res, src, fetched, n_i, ctx->fetch_stream);
                if (rc) return rc;
                fetched = n_i;
            }
        }
    }
    vtx_result dev{};
    int rc = vtx_finish_device(ctx, &dev);
    if (rc) return rc;
    const size_t n = dev.n;
    rc = ensure_host(ctx, ctx->h_res, n);          // no-op when streamed (res_ub >= n)
    if (rc) return rc;
    cudaStream_t st = ctx->fetch_stream ? ctx->fetch_stream : ctx->stream;
    if (n > fetched) {
        rc = copy_results(ctx, ctx->h_res, src, fetched, n, st);
        if (rc) return rc;
    }
    CK(cudaStreamSynchronize(st));
    point_result(out, ptrs(ctx->h_res.a), want_mask(ctx), n, dev.metrics);
    return VTX_OK;
}
int vtx_last_tile_counts(vtx_ctx* ctx, uint32_t* out, uint32_t n_out)
{
    if (!ctx || !out) return VTX_E_INVALID;
    if (!ctx->last_tiles_valid) return set_err(ctx, VTX_E_STATE, "no Smith-Waterman pass has run yet");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    const uint32_t nl = ctx->last_tiles_nl;
    for (uint32_t c = 0; c < n_out; ++c) {
        out[c] = 0;
        if (c < uint32_t(kNumClasses))
            CK(cudaMemcpy(out + c, P<uint32_t>(ctx->tstart) + size_t(c) * (nl + 1) + nl, 4, cudaMemcpyDeviceToHost));
    }
    return kNumClasses;
}

int vtx_last_timing(vtx_ctx* ctx, vtx_timing* t)
{
    if (!ctx || !t) return VTX_E_INVALID;
    if (!ctx->timing_valid || ctx->trec_used == 0) return set_err(ctx, VTX_E_STATE, "no finished submit to time");
    CK(cudaSetDevice(ctx->device));
    memset(t, 0, sizeof(*t));
    for (size_t i = 0; i < ctx->trec_used; ++i) {      // summed over every submit since the last finish
        TimeRec& r = ctx->trecs[i];
        CK(cudaEventSynchronize(r.ev[EV_POST]));
        float ms = 0;
        if (r.had_h2d) { CK(cudaEventElapsedTime(&ms, r.ev[EV_START], r.ev[EV_H2D])); t->h2d_ms += ms; }
        CK(cudaEventElapsedTime(&ms, r.ev[EV_C0], r.ev[EV_PREP])); t->prep_ms += ms;
        CK(cudaEventElapsedTime(&ms, r.ev[EV_PREP], r.ev[EV_SW])); t->sw_ms += ms;
        CK(cudaEventElapsedTime(&ms, r.ev[EV_SW], r.ev[EV_POST])); t->post_ms += ms;
        t->sw_launches += r.sw_launches; t->total_launches += r.launches;
    }
    t->n_pairs = ctx->t_pairs;
    return VTX_OK;
}

int vtx_score_pairs(vtx_ctx* ctx, const vtx_batch* hb, uint64_t n_pairs, const uint32_t* pair_read,
                    const uint32_t* pair_locus, int16_t* ref_score, int16_t* alt_score)
{
    Nvtx nvtx_range("vtx_score_pairs");
    if (!ctx) return VTX_E_INVALID;
    if (!hb) return set_err(ctx, VTX_E_INVALID, "batch is NULL");
    BatchView hv0 = view_of(hb); hv0.n_cand = 0; hv0.cand_read = nullptr;          // the cand_* fields are ignored here
    int rc = validate_batch(ctx, hv0);
    if (rc) return rc;
    if (n_pairs >= 0xFFFFFFF0ull) return set_err(ctx, VTX_E_INVALID, "too many pairs");
    if (n_pairs && (!pair_read || !pair_locus || !ref_score || !alt_score)) return set_err(ctx, VTX_E_INVALID, "NULL pair arrays");
    DevBatch d{};
    rc = scan_host_batch(ctx, hv0, &d.max_read_len, &d.max_hap_len, false);
    if (rc) return rc;
    if (n_pairs == 0) return VTX_OK;
    const uint32_t nl = hb->n_loci;
    // counting sort by locus (tiles need the pairs of a locus to be contiguous)
    std::vector<uint32_t> start(size_t(nl) + 2, 0), order(n_pairs), s_read(n_pairs), s_locus(n_pairs);
    for (uint64_t i = 0; i < n_pairs; ++i) {
        if (pair_locus[i] >= nl || pair_read[i] >= hb->n_reads) return set_err(ctx, VTX_E_INVALID, "pair %llu out of range", (unsigned long long)i);
        ++start[pair_locus[i] + 1];
    }
    for (uint32_t l = 0; l < nl; ++l) start[l + 1] += start[l];
    {
        std::vector<uint32_t> cur(start.begin(), start.begin() + nl + 1);
        for (uint64_t i = 0; i < n_pairs; ++i) { const uint32_t p = cur[pair_locus[i]]++; order[p] = uint32_t(i); s_read[p] = pair_read[i]; s_locus[p] = pair_locus[i]; }
    }
    CK(cudaSetDevice(ctx->device));
    InSlot* sl = nullptr;
    rc = claim_slot(ctx, &sl);
    if (rc) return rc;
    rc = upload_common(ctx, sl, hv0, d);
    if (rc) return rc;
    CK(cudaEventRecord(sl->copy_done, ctx->copy_stream));
    CK(cudaStreamWaitEvent(ctx->stream, sl->copy_done, 0));
    ENS(ctx->pair_read, n_pairs * 4 + 4); ENS(ctx->pair_locus, n_pairs * 4 + 4); ENS(ctx->pair_start, size_t(nl + 1) * 4);
    ENS(ctx->pair_scores, n_pairs * 4 + 4);
    CK(cudaMemcpyAsync(ctx->pair_read.p, s_read.data(), n_pairs * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->pair_locus.p, s_locus.data(), n_pairs * 4, cudaMemcpyHostToDevice, ctx->stream));
    vtx_k_pair_start_explicit<<<blocks_for(nl + 1, 256), 256, 0, ctx->stream>>>(nl, uint32_t(n_pairs), P<uint32_t>(ctx->pair_locus),
                                                                                P<uint32_t>(ctx->pair_start));
    uint64_t launches = 1, sw_launches = 0;
    rc = run_sw(ctx, d, uint32_t(n_pairs), nullptr, nullptr, P<uint32_t>(ctx->pair_scores), &launches, &sw_launches, nullptr);
    if (rc) return rc;
    CK(cudaEventRecord(sl->free_ev, ctx->stream));
    std::vector<uint32_t> packed(n_pairs);
    CK(cudaMemcpyAsync(packed.data(), ctx->pair_scores.p, n_pairs * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint64_t p = 0; p < n_pairs; ++p) {
        ref_score[order[p]] = int16_t(packed[p] & 0xFFFF);
        alt_score[order[p]] = int16_t(packed[p] >> 16);
    }
    return VTX_OK;
}

uint64_t vtx_pack_umi(const uint8_t* s, uint32_t len) { return stage::pack_umi(s, len); }


// -------------------------------------------------------------------------------------------------
// multi-GPU: one allgatherv of the finished triplets over NCCL (NVLink / NVSwitch).  NCCL has no
// native "v" collective: ncclAllGather of the per-rank counts, then one grouped set of exact-size
// ncclBroadcast calls (7 arrays x n_ranks roots).  NCCL is dlopen'ed so that single-GPU users (and
// CPU-only build hosts) never need the library.
// -------------------------------------------------------------------------------------------------
}  // extern "C"

#include <dlfcn.h>
namespace {
typedef struct { char internal[128]; } nccl_uid;
typedef void* nccl_comm;
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(nccl_uid*) = nullptr;
    int (*CommInitRank)(nccl_comm*, int, nccl_uid, int) = nullptr;
    int (*CommDestroy)(nccl_comm) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm, cudaStream_t) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
NcclApi g_nccl;
constexpr int kNcclUint8 = 1, kNcclUint64 = 5;

bool load_nccl(std::string* why)
{
    if (g_nccl.ok) return true;
    const char* names[] = { "libnccl.so.2", "libnccl.so" };
    for (const char* n : names) { g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (g_nccl.h) break; }
    if (!g_nccl.h) { *why = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
#define SYM(field, name) *(void**)(&g_nccl.field) = dlsym(g_nccl.h, name); if (!g_nccl.field) { *why = std::string("missing symbol ") + name; return false; }
    SYM(GetUniqueId, "ncclGetUniqueId") SYM(CommInitRank, "ncclCommInitRank") SYM(CommDestroy, "ncclCommDestroy")
    SYM(AllGather, "ncclAllGather") SYM(Broadcast, "ncclBroadcast") SYM(GroupStart, "ncclGroupStart")
    SYM(GroupEnd, "ncclGroupEnd") SYM(GetErrorString, "ncclGetErrorString") SYM(Send, "ncclSend") SYM(Recv, "ncclRecv")
#undef SYM
    g_nccl.ok = true;
    return true;
}
#define NK(call) do { int r_ = (call); if (r_ != 0) return set_err(ctx, VTX_E_NCCL, "%s failed: %s", #call, g_nccl.GetErrorString(r_)); } while (0)

void comm_destroy(vtx_ctx* ctx)
{
    if (ctx->comm && g_nccl.ok) g_nccl.CommDestroy(static_cast<nccl_comm>(ctx->comm));
    ctx->comm = nullptr;
}
}  // namespace

extern "C" {

int vtx_comm_unique_id(uint8_t id_out[128])
{
    std::string why;
    if (!id_out) return VTX_E_INVALID;
    if (!load_nccl(&why)) { g_create_error = why; return VTX_E_NCCL; }
    nccl_uid id;
    int r = g_nccl.GetUniqueId(&id);
    if (r != 0) { g_create_error = g_nccl.GetErrorString(r); return VTX_E_NCCL; }
    memcpy(id_out, id.internal, 128);
    return VTX_OK;
}

int vtx_comm_init(vtx_ctx* ctx, const uint8_t id[128], int32_t rank, int32_t n_ranks)
{
    if (!ctx || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return ctx ? set_err(ctx, VTX_E_INVALID, "vtx_comm_init: bad arguments") : VTX_E_INVALID;
    std::string why;
    if (!load_nccl(&why)) return set_err(ctx, VTX_E_NCCL, "%s", why.c_str());
    CK(cudaSetDevice(ctx->device));
    nccl_uid uid; memcpy(uid.internal, id, 128);
    nccl_comm comm = nullptr;
    NK(g_nccl.CommInitRank(&comm, n_ranks, uid, rank));
    ctx->comm = comm; ctx->rank = rank; ctx->n_ranks = n_ranks;
    return VTX_OK;
}

int vtx_gather_start(vtx_ctx* ctx, int32_t root)
{
    Nvtx nvtx_range("vtx_gather_start");
    if (!ctx) return VTX_E_INVALID;
    if (!ctx->finished) return set_err(ctx, VTX_E_STATE, "vtx_gather must follow vtx_finish / vtx_finish_device");
    if (ctx->gather_pending) return set_err(ctx, VTX_E_STATE, "a gather is already in flight: call vtx_gather_wait first");
    const int nrk = ctx->n_ranks;
    if (root != VTX_GATHER_ALL && (root < 0 || root >= nrk)) return set_err(ctx, VTX_E_INVALID, "gather root %d out of range", root);
    if (nrk != 1 && !ctx->comm) return set_err(ctx, VTX_E_STATE, "vtx_comm_init has not been called");
    CK(cudaSetDevice(ctx->device));
    const uint32_t want = want_mask(ctx);       // only these arrays travel
    const DBuf* loc = ctx->res;
    vtx_result& out = ctx->g_out;
    if (nrk == 1) {
        point_result(&out, ptrs(ctx->res), want, ctx->last_n, ctx->last_metrics);
    } else {
        if (!ctx->comm_stream) {
            CK(cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
            CK(cudaEventCreateWithFlags(&ctx->ev_counts, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&ctx->ev_gather, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&ctx->ev_results, cudaEventDisableTiming));
            CK(ctx->h_counts.alloc(size_t(nrk + 1) * 32));
        }
        cudaStream_t cs = ctx->comm_stream;
        nccl_comm comm = static_cast<nccl_comm>(ctx->comm);
        // the local results are complete on the engine stream (vtx_finish synchronised it); order the comm stream behind it anyway
        CK(cudaEventRecord(ctx->ev_results, ctx->stream));
        CK(cudaStreamWaitEvent(cs, ctx->ev_results, 0));
        // 1. counts: {n, not_cell_bc, non_umi, scored} of every rank.  One tiny allgather; the host needs the sizes to post
        //    exact-size receives, and waits for this one event only (tens of microseconds, nothing else is blocked).
        ENS(ctx->g_counts, size_t(nrk + 1) * 32);
        uint64_t* mine = ctx->h_counts.as<uint64_t>() + size_t(nrk) * 4;
        mine[0] = ctx->last_n; mine[1] = ctx->last_metrics.num_not_cell_bc; mine[2] = ctx->last_metrics.num_non_umi; mine[3] = ctx->last_metrics.num_scored;
        uint64_t* dmine = P<uint64_t>(ctx->g_counts) + size_t(nrk) * 4;
        CK(cudaMemcpyAsync(dmine, mine, 32, cudaMemcpyHostToDevice, cs));
        NK(g_nccl.AllGather(dmine, ctx->g_counts.p, 4, kNcclUint64, comm, cs));
        CK(cudaMemcpyAsync(ctx->h_counts.p, ctx->g_counts.p, size_t(nrk) * 32, cudaMemcpyDeviceToHost, cs));
        CK(cudaEventRecord(ctx->ev_counts, cs));
        CK(cudaEventSynchronize(ctx->ev_counts));
        const uint64_t* counts = ctx->h_counts.as<uint64_t>();
        size_t total = 0;
        std::vector<size_t> offs(nrk);
        vtx_metrics met{};
        for (int r = 0; r < nrk; ++r) {
            offs[r] = total; total += counts[size_t(r) * 4];
            met.num_not_cell_bc += counts[size_t(r) * 4 + 1]; met.num_non_umi += counts[size_t(r) * 4 + 2]; met.num_scored += counts[size_t(r) * 4 + 3];
        }
        const bool receiver = root == VTX_GATHER_ALL || root == ctx->rank;
        if (receiver) for (int i = 0; i < kResArrays; ++i) if (want >> i & 1) ENS(ctx->g_dev[i], (total ? total : 1) * kResEsz[i]);
        // 2. the triplets, exact sizes, one NCCL group.  Rooted: ncclSend / ncclRecv, only the writer's GPU receives;
        //    all: one broadcast per (array, rank) = allgatherv.
        NK(g_nccl.GroupStart());
        for (int i = 0; i < kResArrays; ++i) {
            if (!(want >> i & 1)) continue;
            const size_t esz = kResEsz[i];
            if (root == VTX_GATHER_ALL) {
                for (int r = 0; r < nrk; ++r) {
                    const size_t n = counts[size_t(r) * 4];
                    if (n) NK(g_nccl.Broadcast(loc[i].p, static_cast<uint8_t*>(ctx->g_dev[i].p) + offs[r] * esz, n * esz, kNcclUint8, r, comm, cs));
                }
            } else if (ctx->rank == root) {
                for (int r = 0; r < nrk; ++r) {
                    const size_t n = counts[size_t(r) * 4];
                    if (!n) continue;
                    uint8_t* dst = static_cast<uint8_t*>(ctx->g_dev[i].p) + offs[r] * esz;
                    if (r == root) CK(cudaMemcpyAsync(dst, loc[i].p, n * esz, cudaMemcpyDeviceToDevice, cs));
                    else NK(g_nccl.Recv(dst, n * esz, kNcclUint8, r, comm, cs));
                }
            } else if (ctx->last_n) {
                NK(g_nccl.Send(loc[i].p, size_t(ctx->last_n) * esz, kNcclUint8, root, comm, cs));
            }
        }
        NK(g_nccl.GroupEnd());
        CK(cudaEventRecord(ctx->ev_gather, cs));
        ctx->gather_guard = true;
        point_result(&out, ptrs(ctx->g_dev), receiver ? want : 0u, total, met);
    }
    ctx->gather_pending = true;
    return VTX_OK;
}

int vtx_gather_wait(vtx_ctx* ctx, vtx_result* out)
{
    Nvtx nvtx_range("vtx_gather_wait");
    if (!ctx || !out) return VTX_E_INVALID;
    if (!ctx->gather_pending) return set_err(ctx, VTX_E_STATE, "no gather in flight");
    CK(cudaSetDevice(ctx->device));
    if (ctx->n_ranks > 1) CK(cudaEventSynchronize(ctx->ev_gather));
    ctx->gather_pending = false;
    *out = ctx->g_out;
    return VTX_OK;
}

int vtx_gather(vtx_ctx* ctx, vtx_result* out)
{
    if (!ctx || !out) return VTX_E_INVALID;
    const int rc = vtx_gather_start(ctx, VTX_GATHER_ALL);
    return rc ? rc : vtx_gather_wait(ctx, out);
}

}  // extern "C"
