/*
 * vartrix_b200.h -- C ABI of the H100-native per-locus read-scoring engine.
 *
 * Drop-in boundary for the hot path of 10XGenomics/vartrix v1.1.22 (all file:line citations are into
 * vartrix src/main.rs).  The reference has no FFI seam of its own; the seam this ABI sits
 * behind is the rayon block main.rs:279-291 (evaluate_chunk -> evaluate_rec -> evaluate_alns) plus the
 * serial merge main.rs:320-348.  A host (Rust via `extern "C"`, C++, Python ctypes) keeps doing what
 * main.rs does up to and including the record filters (VCF/FASTA/BAM decode, construct_haplotypes
 * main.rs:958-994, mapq/primary/duplicate/useful_alignment filters main.rs:833-865), stages the
 * surviving (read, ref-window, alt-window, CB-tag, UB-tag) candidates into a `vtx_batch`, and this
 * library replaces, on the GPU:
 *     get_cell_barcode + HashMap lookup        main.rs:737-750, 867-877   -> vtx_k_cb_lookup
 *     the --umi gate                           main.rs:879-894            -> vtx_k_cand_filter
 *     banded::Aligner::local x2                main.rs:898-901            -> vtx_k_sw_pairs<...>
 *     Scores push + sort_by_key(cell_index)    main.rs:923-932            -> vtx_k_slots
 *     evaluate_scores                          main.rs:1019-1030          -> SW kernel epilogue (atomicAdd)
 *     parse_scores / UMI collapse              main.rs:1041-1109          -> vtx_k_umi_collapse
 *     consensus_scoring / alt_frac / coverage  main.rs:1111-1164          -> vtx_k_finalize
 *     merge into TriMat (row-major)            main.rs:320-348            -> vtx_k_emit (+ vtx_gather)
 *
 * Conventions: every call returns 0 or a negative VTX_E_* code; no exceptions cross the boundary; no
 * global state except a thread-local message for failed vtx_create; a ctx is single-threaded.
 * All types are plain C (pointers and sizes).  The library is CUDA-only: there is no CPU fallback.
 */
#ifndef VARTRIX_B200_H
#define VARTRIX_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VTX_ABI_VERSION 2     /* 2: vtx_batch2 / vtx_submit2 (slim staging layout), vtx_gather_start / _wait, band fields in vtx_config */

/* error codes */
#define VTX_OK             0
#define VTX_E_INVALID     (-1)   /* bad argument / malformed batch */
#define VTX_E_CUDA        (-2)   /* CUDA runtime failure (message in vtx_last_error) */
#define VTX_E_NOMEM       (-3)
#define VTX_E_UNSUPPORTED (-4)   /* e.g. scoring constants other than the compiled-in ones */
#define VTX_E_STATE       (-5)   /* call order violated */
#define VTX_E_NCCL        (-6)

/* --scoring-method (main.rs:90-95) */
#define VTX_MODE_CONSENSUS 0
#define VTX_MODE_COVERAGE  1
#define VTX_MODE_ALT_FRAC  2

#define VTX_NO_CB   0xFFFFFFFFu             /* read has no Z-typed --bam-tag aux field (main.rs:742-749) */
#define VTX_NO_UMI  0xFFFFFFFFFFFFFFFFull   /* read has no Z-typed UB aux field (main.rs:752-757) */
#define VTX_UMI_KEY_MAX ((1ull << 62) - 1)  /* valid UMI keys are <= this */

typedef struct vtx_ctx vtx_ctx;

typedef struct vtx_config {
    int32_t  device;        /* CUDA device ordinal */
    int32_t  mode;          /* VTX_MODE_* */
    int32_t  use_umi;       /* --umi (main.rs:123-125) */
    int32_t  match;         /* must be  1  (MATCH,      main.rs:35) */
    int32_t  mismatch;      /* must be -5  (MISMATCH,   main.rs:36) */
    int32_t  gap_open;      /* must be -5  (GAP_OPEN,   main.rs:37) */
    int32_t  gap_extend;    /* must be -1  (GAP_EXTEND, main.rs:38) */
    int32_t  min_score;     /* MIN_SCORE, main.rs:30 (25) */
    void*    stream;        /* cudaStream_t to enqueue on; NULL = library-owned non-blocking stream */
    uint32_t flags;         /* VTX_F_* */
    /* The reference aligns with bio 0.30.0's banded aligner, Aligner::new(GAP_OPEN, GAP_EXTEND, score, K, W) (main.rs:27-38,
     * 899).  VTX_BAND_FULL scores the whole matrix: the exact upper bound of every band, equal to the banded score
     * whenever the optimal path stays inside the band, and what reproduces the reference's 12 golden matrices.
     * band_k / band_w: 0 = the reference's constants (6 / 20); they only matter for VTX_BAND_MODEL (K 1..8).
     * VTX_BAND_MODEL scores every pair inside the k-mer-chain band of SURVEY Appendix B ("model B": exact k-mer hits, best
     * chain, +-W around the chain, lazy ends; no hit -> full matrix) -- a restatement of the crate's behaviour from its
     * documentation, NOT a port of its source (unavailable here): consistent with every golden of the reference, otherwise
     * unverified.  It is a slow path (one warp per alignment) for users who prefer the heuristic band in low-complexity
     * sequence; tools/band_exposure.py measures where the two differ. */
    int32_t  band_k;        /* K, main.rs:33 */
    int32_t  band_w;        /* W, main.rs:34 */
    int32_t  band_mode;     /* VTX_BAND_* */
} vtx_config;

#define VTX_BAND_FULL   0   /* full-matrix affine local score (default) */
#define VTX_BAND_MODEL  1   /* score restricted to the k-mer-chain band model of SURVEY Appendix B (oracle: vtxo_sw_band_model) */

#define VTX_F_KEEP_SCORES 1u    /* also keep per-pair raw scores on the device (debug / parity) */
#define VTX_F_NO_SPLIT    2u    /* use only the single-phase Smith-Waterman kernels (neither shared-prefix nor folded) */
#define VTX_F_VALUES_ONLY 4u    /* vtx_finish / vtx_fetch copy only row, col, val (and val2 in coverage mode) to the host;
                                   ref_cnt / alt_cnt / unk_cnt come back NULL (halves the device->host traffic) */
#define VTX_F_NO_FOLD     8u    /* do not use the folded (shared prefix AND suffix) Smith-Waterman kernel */

/*
 * One staged shard of loci.  SoA; for vtx_submit the pointers are HOST pointers (ideally pinned, see
 * vtx_host_alloc) that must stay valid until the next vtx_finish/vtx_sync; for vtx_submit_device they
 * are DEVICE pointers on the ctx's device.
 *
 * loci        : the scored records of this shard, ascending by `locus_row`.  Records the reference
 *               skips before alignment (multi-allelic main.rs:646-653, invalid alt haplotype
 *               main.rs:675-684) are simply not listed; their rows stay empty.
 * hap_bytes   : ASCII haplotype windows exactly as construct_haplotypes builds them (reference window
 *               upper-cased, ALT bytes verbatim).  ref_off/alt_off must be multiples of 16.
 * reads       : each distinct BAM record once.  `read_nib` is the BAM 4-bit encoding (high nibble
 *               first, "=ACMGRSVTWYHKDBN"); read_off must be multiples of 16 and the pool must be padded
 *               to a multiple of 16 bytes.
 * cb / umi    : per read.  CB bytes are compared by exact byte equality with the barcode list.
 *               read_umi_key is any injective encoding of the UB string into [0, VTX_UMI_KEY_MAX]
 *               (equal key <=> equal bytes inside one ctx run); see vtx_pack_umi.
 * candidates  : (read, locus) pairs that survived the host-side filters, locus-major, BAM file order
 *               inside a locus (order only matters for reproducing metrics, not matrices).
 */
typedef struct vtx_batch {
    uint32_t        n_loci;
    const uint32_t* locus_row;     /* [n_loci] matrix row = VCF record index (main.rs:224-233) */
    const uint8_t*  hap_bytes;
    uint64_t        hap_bytes_len;
    const uint32_t* ref_off;       /* [n_loci] */
    const uint32_t* ref_len;       /* [n_loci] */
    const uint32_t* alt_off;       /* [n_loci] */
    const uint32_t* alt_len;       /* [n_loci] */
    const uint64_t* cand_start;    /* [n_loci + 1] */
    uint32_t        n_reads;
    const uint8_t*  read_nib;
    uint64_t        read_nib_len;
    const uint64_t* read_off;      /* [n_reads] */
    const uint32_t* read_len;      /* [n_reads] bases */
    const uint8_t*  cb_bytes;
    uint64_t        cb_bytes_len;
    const uint32_t* read_cb_off;   /* [n_reads] or VTX_NO_CB */
    const uint16_t* read_cb_len;   /* [n_reads] */
    const uint64_t* read_umi_key;  /* [n_reads] or VTX_NO_UMI */
    uint64_t        n_cand;
    const uint32_t* cand_read;     /* [n_cand] */
} vtx_batch;

/*
 * The slim staging layout (ABI 2).  Same content as vtx_batch, ~95 instead of ~138 bytes per candidate on the
 * BASELINE shapes, because host->device bytes are what the end-to-end path pays for:
 *   reads      : `read_nib` holds the reads back to back in id order, each starting on a 4-byte boundary; read_off4 ==
 *                NULL says exactly that (offsets are then derived on the device), else read_off4[r] * 4 is the byte offset
 *                of read r.  read_len is u16 (longer reads: use vtx_batch).
 *   cell tags  : one u64 per read -- vtx_pack_cb() of the tag bytes (an injective code of `[ACGT]{1,24}(-[1-9][0-9]?)?`,
 *                i.e. of every Cell Ranger barcode), VTX_NO_CB_KEY when the read has no Z-typed tag, or
 *                VTX_CB_EXOTIC | i for a tag the code cannot express: its bytes are cb_bytes[cb_off[i] .. cb_off[i+1]).
 *                The comparison with the barcode list stays exact byte equality (main.rs:745): equal strings have equal
 *                codes, and an exotic tag can only equal an exotic barcode.
 *   UMIs       : read_umi_key may be NULL when the ctx was created with use_umi == 0 (the keys are never read).
 *   candidates : cand_read == NULL means candidate c is read c (n_cand == n_reads: no read serves two loci).
 */
#define VTX_NO_CB_KEY  0xFFFFFFFFFFFFFFFFull
#define VTX_CB_EXOTIC  0x8000000000000000ull   /* | index into cb_off */
typedef struct vtx_batch2 {
    uint32_t        n_loci;
    const uint32_t* locus_row;     /* [n_loci] */
    const uint8_t*  hap_bytes;
    uint64_t        hap_bytes_len;
    const uint32_t* ref_off;       /* [n_loci] multiples of 16 */
    const uint32_t* ref_len;
    const uint32_t* alt_off;
    const uint32_t* alt_len;
    const uint64_t* cand_start;    /* [n_loci + 1] */
    uint32_t        n_reads;
    const uint8_t*  read_nib;
    uint64_t        read_nib_len;
    const uint32_t* read_off4;     /* [n_reads] byte offset / 4, or NULL (dense) */
    const uint16_t* read_len;      /* [n_reads] bases */
    const uint64_t* read_cb_key;   /* [n_reads] */
    uint32_t        n_exotic_cb;
    const uint8_t*  cb_bytes;      /* exotic tags only */
    const uint32_t* cb_off;        /* [n_exotic_cb + 1] */
    const uint64_t* read_umi_key;  /* [n_reads] or NULL (use_umi == 0) */
    uint64_t        n_cand;
    const uint32_t* cand_read;     /* [n_cand] or NULL (identity) */
} vtx_batch2;

/* The device-side share of main.rs:449-459 (the host keeps the counters of its own filters). */
typedef struct vtx_metrics {
    uint64_t num_not_cell_bc;      /* main.rs:874 */
    uint64_t num_non_umi;          /* main.rs:886 */
    uint64_t num_scored;           /* pairs that reached the aligner (main.rs:896-930) = the bench unit */
} vtx_metrics;

/*
 * Finished triplets, row-major sorted (row ascending, then col ascending) = TriMat insertion order of
 * main.rs:320-348.  `val` is the out-matrix value of the configured mode, `val2` the --ref-matrix value
 * (coverage mode only, else 0).  Arrays are library-owned and stay valid until the next
 * submit / finish / gather / destroy call on the same ctx.
 */
typedef struct vtx_result {
    uint64_t        n;
    const uint32_t* row;
    const uint32_t* col;
    const uint32_t* ref_cnt;
    const uint32_t* alt_cnt;
    const uint32_t* unk_cnt;
    const double*   val;
    const double*   val2;
    vtx_metrics     metrics;
} vtx_result;

/* ---- lifecycle --------------------------------------------------------------------------------- */
int         vtx_abi_version(void);
int         vtx_create(const vtx_config* cfg, vtx_ctx** out);
void        vtx_destroy(vtx_ctx* ctx);
const char* vtx_last_error(const vtx_ctx* ctx);          /* ctx == NULL: message of the last failed vtx_create */

/* Pinned host memory for staging (north_star: "stages batches into pinned buffers"). */
int         vtx_host_alloc(void** out, uint64_t bytes);
int         vtx_host_free(void* p);

/* ---- barcode list: replaces load_barcodes' HashMap (main.rs:697-718) with a device hash table ---- */
/* keys = n DISTINCT byte strings, key i = bytes[off[i] .. off[i+1]); column id = i (first-seen order).
 * Duplicates are rejected with VTX_E_INVALID (the loader dedups, main.rs:706-709). */
int         vtx_set_barcodes(vtx_ctx* ctx, const uint8_t* bytes, const uint32_t* off, uint32_t n);

/* ---- the hot path --------------------------------------------------------------------------------- */
/* Enqueue one shard (asynchronous on the ctx stream).  Shards must arrive in ascending row order. */
int         vtx_submit(vtx_ctx* ctx, const vtx_batch* host_batch);
int         vtx_submit_device(vtx_ctx* ctx, const vtx_batch* device_batch);
/* The same for the slim layout (host pointers / device pointers). */
int         vtx_submit2(vtx_ctx* ctx, const vtx_batch2* host_batch);
int         vtx_submit2_device(vtx_ctx* ctx, const vtx_batch2* device_batch, uint32_t max_read_len, uint32_t max_hap_len);
/* Device batches cannot be scanned by the host: state the longest read and the widest haplotype window (upper
 * bounds; buffers are sized and kernels selected from them.  A locus with a longer read or a wider window than promised
 * is detected on the device and skipped, and the next vtx_finish / vtx_finish_device returns VTX_E_INVALID.  Plain
 * vtx_submit_device promises reads <= 1024 bases and windows <= 320 bytes). */
int         vtx_submit_device_ex(vtx_ctx* ctx, const vtx_batch* device_batch, uint32_t max_read_len, uint32_t max_hap_len);
/* Wait for everything submitted since the last finish and hand back the triplets (host arrays). */
int         vtx_finish(vtx_ctx* ctx, vtx_result* out);
/* Same, but `out` holds DEVICE pointers (nothing but the 3 counters and `n` crosses PCIe). */
int         vtx_finish_device(vtx_ctx* ctx, vtx_result* out);
/* Copy a device-resident result (from vtx_finish_device or vtx_gather) into library-owned pinned host arrays. */
int         vtx_fetch(vtx_ctx* ctx, const vtx_result* device_result, vtx_result* out);
int         vtx_sync(vtx_ctx* ctx);
/* Wait until every host->device copy enqueued by vtx_submit so far has landed, i.e. until the host buffers
 * of all previous submits may be reused (kernels may still be running). */
int         vtx_wait_copies(vtx_ctx* ctx);

/* Raw scores (Scores.ref_score / alt_score, main.rs:996-1001, 926-927) for an explicit pair list:
 * pair i = (read pair_read[i], locus pair_locus[i]) of `host_batch` (cand_* fields ignored).
 * Synchronous; host pointers.  This is the comparison point of the parity tests. */
int         vtx_score_pairs(vtx_ctx* ctx, const vtx_batch* host_batch, uint64_t n_pairs,
                            const uint32_t* pair_read, const uint32_t* pair_locus,
                            int16_t* ref_score, int16_t* alt_score);

/* Injective UMI key for strings over {A,C,G,T,N} up to 18 bases (3 bits/base + 5-bit length, < 2^59).
 * Returns VTX_NO_UMI if the string does not fit; the caller then interns it as (1 << 61) | id. */
uint64_t    vtx_pack_umi(const uint8_t* s, uint32_t len);

/* ---- BGZF members inflated on the device (SURVEY 8f-1; replaces htslib's bgzf_read_block -> inflate behind
 * main.rs:822-829 for a host that only seeks and reads the compressed file) ------------------------------------------
 * `comp` holds the raw DEFLATE payloads of n_blocks BGZF members (the bytes between the gzip header incl. its extra field
 * and the 8-byte trailer), each starting at a multiple of 4 with at least 8 readable bytes behind it; `blocks[i]` says where
 * member i's payload is, its ISIZE (<= 65536) and CRC-32 from the trailer, and where in `out` its bytes go.  One warp per
 * member; VTX_BGZF_CHECK_CRC verifies the CRC-32 on the device as well.  Host pointers; synchronous.  status[i] = 0 or a
 * decoder error code (1 bad stream, 2 bad code table, 3 input overrun, 4 size mismatch, 5 bad stored block, 6 bad distance,
 * 7 CRC mismatch); returns VTX_E_INVALID if any member failed (the other members are still delivered).  Needs no barcodes. */
typedef struct vtx_bgzf_block {
    uint64_t in_off;
    uint32_t in_len;
    uint32_t out_len;
    uint64_t out_off;
    uint32_t crc32;
    uint32_t reserved;
} vtx_bgzf_block;
#define VTX_BGZF_CHECK_CRC 1u
int         vtx_bgzf_inflate(vtx_ctx* ctx, const vtx_bgzf_block* blocks, uint32_t n_blocks, const uint8_t* comp, uint64_t comp_len,
                             uint8_t* out, uint64_t out_len, int32_t* status, uint32_t flags);

/* ---- a shard of loci straight from the BAM: inflate, record scan, fetch, record filters and tag extraction on the
 * device (SURVEY 8f-1).  The host's part shrinks to what needs the file system and the index: it reads the compressed
 * byte range the loci's index chunks span, walks the BGZF member headers, lists the chunk starts that fall into the range
 * (record boundaries), builds the haplotype windows from the FASTA -- and hands all of it over.  The device then does what
 * csrc/host/stager.hpp does on staging threads and the reference does through rust-htslib: every record of contig `tid`
 * with pos < end and bam_endpos > start per locus, in file order (main.rs:822-829); mapq / primary / duplicate /
 * useful_alignment filters in that order (main.rs:833-865); CB (`bam_tag`) and UB as the first Z-typed aux field of that
 * name (main.rs:737-757); then the same pipeline as vtx_submit.  Loci must be ascending on one contig of a
 * coordinate-sorted BAM.  Asynchronous like vtx_submit (two short waits on the staging stream for sizes).
 *   members / comp : as for vtx_bgzf_inflate, in file order, out_off = running sum of out_len (one contiguous stream)
 *   entry_off      : ascending offsets into that stream; [0] = first record to look at, [n_entry - 1] = end of the
 *                    records to look at; every entry is a record boundary (BAI chunk starts / ends)
 * Returns VTX_E_UNSUPPORTED when the shard needs the host path (a UB string that vtx_pack_umi cannot express, a read
 * above 16 000 bases) and VTX_E_INVALID for corrupt members / records; nothing of the shard has been counted then and
 * the caller may stage it on the host instead (vtx_submit2). */
typedef struct vtx_bam_shard {
    uint32_t        n_loci;
    const uint32_t* locus_row;       /* [n_loci] */
    const int64_t*  locus_start;     /* [n_loci] rec.pos(), 0-based            (main.rs:619-623) */
    const int64_t*  locus_end;       /* [n_loci] start + len(REF) */
    const uint8_t*  hap_bytes;       /* windows as in vtx_batch */
    uint64_t        hap_bytes_len;
    const uint32_t* ref_off;
    const uint32_t* ref_len;
    const uint32_t* alt_off;
    const uint32_t* alt_len;
    int32_t         tid;             /* BAM reference id of the contig */
    uint32_t        n_members;
    const vtx_bgzf_block* members;
    const uint8_t*  comp;
    uint64_t        comp_len;
    uint32_t        n_entry;
    const uint64_t* entry_off;
    uint32_t        mapq;            /* --mapq */
    int32_t         primary_only;    /* --primary-alignments */
    int32_t         no_duplicates;   /* --no-duplicates */
    char            bam_tag[2];      /* --bam-tag */
} vtx_bam_shard;
/* the host-side share of main.rs:449-459, counted on the device for shards that came through vtx_submit_bam */
typedef struct vtx_bam_metrics {
    uint64_t num_reads, num_low_mapq, num_non_primary, num_duplicates, num_not_useful;
} vtx_bam_metrics;
int         vtx_submit_bam(vtx_ctx* ctx, const vtx_bam_shard* shard);
/* Counters of every vtx_submit_bam since the ctx was created (waits for the staging stream). */
int         vtx_bam_metrics_get(vtx_ctx* ctx, vtx_bam_metrics* out);

/* Injective code of a cell-barcode tag of the form [ACGT]{1,24}(-N)? with N = 1..99 written without a leading zero:
 * 2 bits per base, 5 bits length, 7 bits N (0 = no suffix); < 2^60.  Returns VTX_NO_CB_KEY if the bytes have another
 * form -- the caller then lists them as an exotic tag (VTX_CB_EXOTIC | i). */
uint64_t    vtx_pack_cb(const uint8_t* s, uint32_t len);

/* Device-side timings of the last finished submit, milliseconds (CUDA events on the ctx stream). */
typedef struct vtx_timing {
    float h2d_ms;       /* host->device copies of the batch (0 for vtx_submit_device) */
    float prep_ms;      /* CB lookup, filter, compaction, slots, tiling */
    float sw_ms;        /* Smith-Waterman + call + atomic scatter kernels */
    float post_ms;      /* UMI collapse, finalize, emit */
    uint64_t n_pairs;   /* scored pairs of that submit */
    uint64_t sw_launches;
    uint64_t total_launches;
} vtx_timing;
int         vtx_last_timing(vtx_ctx* ctx, vtx_timing* out);
/* Warp tiles each Smith-Waterman kernel class got in the most recent submit / vtx_score_pairs (diagnostic: which
 * kernels took the work).  out[c] for c < n_out: 0..3 single-phase tile classes (4 pairs per tile), 4 generic
 * (16 pairs), 5..6 shared-prefix kernels (8 pairs), 7 folded kernel (4 pairs).  Returns the number of classes. */
int         vtx_last_tile_counts(vtx_ctx* ctx, uint32_t* out, uint32_t n_out);

/* ---- multi-GPU: loci are sharded across ranks; one allgatherv of finished triplets ------------- */
/* Every rank calls vtx_comm_init with the same 128-byte id (made by vtx_comm_unique_id on one rank
 * and shipped by any side channel).  NCCL is dlopen'ed lazily; single-GPU users never need it. */
int         vtx_comm_unique_id(uint8_t id_out[128]);
int         vtx_comm_init(vtx_ctx* ctx, const uint8_t id[128], int32_t rank, int32_t n_ranks);
/* After vtx_finish_device/vtx_finish on every rank: assemble all ranks' triplets, in rank order
 * (= row order when rank r holds the r-th contiguous locus range), on every rank.  `out` holds DEVICE
 * pointers (metrics summed over ranks); the rank that writes the matrix calls vtx_fetch on it. */
int         vtx_gather(vtx_ctx* ctx, vtx_result* out);
/* The same exchange, asynchronous and optionally rooted.  vtx_gather_start enqueues it on the ctx's communication
 * stream and returns; kernels of later submits overlap it (their first write into the local result arrays waits for
 * it on the device).  root = VTX_GATHER_ALL: allgatherv (every rank ends up with everything).  root = r: only rank r
 * -- the one that writes the matrix -- receives (ncclSend / ncclRecv); on the other ranks vtx_gather_wait returns the
 * total `n` and the summed metrics with NULL arrays.  One gather may be in flight per ctx. */
#define VTX_GATHER_ALL (-1)
int         vtx_gather_start(vtx_ctx* ctx, int32_t root);
int         vtx_gather_wait(vtx_ctx* ctx, vtx_result* out);

#ifdef __cplusplus
}
#endif
#endif /* VARTRIX_B200_H */
