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
#define VTX_F_NAME_KEYS  16u    /* vtx_submit_bam keys reads by QNAME, not UB: the records of one template inside one (locus, cell)
                                   are collapsed like the reads of one UMI (--collapse-mates); a QNAME of "*" is a key of its own.
                                   Needs use_umi (vtx_create returns VTX_E_INVALID otherwise).  Host batches are unaffected: their
                                   caller supplies the name keys in read_umi_key. */

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
 *               (equal key <=> equal bytes inside one ctx run); see vtx_pack_umi.  To count each template once
 *               per cell (--collapse-mates), key the reads by QNAME instead: keys only meet inside one locus, so
 *               any code that is injective within the shard will do, with a fresh key for every QNAME "*".
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
 * useful_alignment filters in that order (main.rs:833-865), then the base-quality floor if one was set (see
 * vtx_set_min_base_quality below); CB (`bam_tag`) and UB as the first Z-typed aux field of that
 * name (main.rs:737-757) -- with VTX_F_NAME_KEYS the QNAME instead of UB, interned on the device (a hash table of record
 * indices: key = the index of the first record with that name; "*" keeps its own index); then the same pipeline as
 * vtx_submit.  Loci must be ascending on one contig of a
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
/* --min-base-quality for every later vtx_submit_bam on this ctx (0, the default, turns it off; VTX_E_INVALID above 93).
 * After the four record filters, a (read, locus) pair is dropped when one of its judged bases has a quality below
 * min_q: the bases aligned to the REF span [start, end), and the bases inserted right after a reference base of that span
 * (soft clips, deletions and skips judge nothing).  A pair without judged bases, or a record without qualities (0xFF), is
 * kept.  Host batches (vtx_submit, vtx_submit2 and the device variants) carry no qualities: their callers apply the floor
 * while staging, as the CLI's stager does. */
int         vtx_set_min_base_quality(vtx_ctx* ctx, uint32_t min_q);
/* Pairs the floor above dropped, summed over every vtx_submit_bam since the ctx was created (waits for the staging stream). */
int         vtx_bam_low_base_quality(vtx_ctx* ctx, uint64_t* out);

/* ---- per-locus summary: why each matrix row holds what it holds (the CLI's --out-variant-stats) ---------------------------
 * vtx_set_locus_stats(ctx, 1) before the first submit (VTX_E_STATE after one) makes every submit also reduce, per locus, the
 * counters below on the device; off, the default, launches nothing extra.  After vtx_finish / vtx_finish_device,
 * vtx_locus_stats_get hands back one entry per locus submitted since the previous finish, in submit order (shards in submit
 * order, loci in shard order) -- ascending row when shards arrive in ascending row order, as vtx_submit asks; the library does
 * not sort them.  Library-owned host memory, valid until the next submit or finish.  Entries are plain 32-bit counters (a shard holds fewer than 2^32
 * candidates).  Invariants per locus:
 *     fetched = low_mapq + non_primary + duplicate + not_useful + low_base_quality + no_cell_barcode + no_umi + scored
 *     scored  = reads_ref + reads_alt + reads_unknown + reads_none
 *     calls_* = reads_* without use_umi (with it: molecules after the UMI / name-key collapse, main.rs:1058-1082)
 * The record-filter counters (fetched .. low_base_quality) are counted on the device for vtx_submit_bam shards; host batches
 * (vtx_submit*, which only carry the survivors) leave them 0 -- their caller's stager owns them.  Every other counter comes
 * from the device on every submit path. */
typedef struct vtx_locus_stats {
    uint32_t row;                 /* matrix row = VCF record index */
    uint32_t fetched;             /* records fetch returned (main.rs:831) */
    uint32_t low_mapq;            /* pairs dropped by each filter, counted once at the first that drops them (main.rs:833-865) */
    uint32_t non_primary;
    uint32_t duplicate;
    uint32_t not_useful;
    uint32_t low_base_quality;    /* vtx_set_min_base_quality */
    uint32_t no_cell_barcode;     /* no tag, or a tag not in the barcode list (main.rs:867-877) */
    uint32_t no_umi;              /* use_umi and no UB tag (main.rs:879-894) */
    uint32_t scored;              /* pairs that reached Smith-Waterman */
    uint32_t reads_ref, reads_alt, reads_unknown, reads_none;     /* per-pair calls (evaluate_scores, main.rs:1019-1030) */
    uint32_t calls_ref, calls_alt, calls_unknown;                 /* the counts the matrix is built from */
    uint32_t cells;               /* cells with at least one scored pair (the row's entries in coverage mode) */
    uint32_t cells_ref_only;      /* consensus value 1 */
    uint32_t cells_alt_only;      /* consensus value 2 */
    uint32_t cells_both;          /* consensus value 3 */
    uint32_t cells_multi_unknown; /* calls_unknown > 1 in the cell: "Check this locus manually" (main.rs:1116-1118) */
} vtx_locus_stats;
int         vtx_set_locus_stats(vtx_ctx* ctx, int32_t on);
int         vtx_locus_stats_get(vtx_ctx* ctx, const vtx_locus_stats** out, uint64_t* n);

/* ---- donor log-likelihoods per cell: genotype demultiplexing of pooled cells (the CLI's --out-donors) ----------------------
 * D donors with known genotypes, H = D + D(D-1)/2 hypotheses: h < D the singlet of donor h, then the doublets (0,1), (0,2), ...,
 * (0,D-1), (1,2), ..., (D-2,D-1).  At a row, hypothesis h has s = g_d1 + g_d2 (a singlet d: s = 2 g_d), g the ALT dosage, and
 * the expected ALT fraction q_s = {e, (e + 0.5)/2, 0.5, (1.5 - e)/2, 1 - e} (a doublet is a 50/50 mixture), e = error_rate.
 * A cell with r REF and a ALT molecules at a usable row (ccnt after the UMI / name-key collapse: the counts the matrix is built
 * from; UNKNOWN calls are not used) adds r Lr[s] + a La[s] to hypothesis h, with the int64 constants
 * Lr[s] = llrint(log(1 - q_s) * VTX_DONOR_LL_SCALE) and La[s] = llrint(log(q_s) * VTX_DONOR_LL_SCALE).  A row is usable when every
 * donor has a dosage there.  All sums are int64, so the result is independent of summation order, shard size and device count.
 *
 * vtx_set_donors: before the first submit (VTX_E_STATE after one).  dosage[row * n_donors + d] is 0, 1, 2 or VTX_GT_MISSING
 * for rows 0 .. n_rows - 1 (the matrix rows); 2 <= n_donors <= 32 and 1e-6 <= error_rate <= 0.25, else VTX_E_INVALID.  The table
 * is uploaded once.  Every later submit then reduces its cell slots into a per-column accumulator of
 * n_barcodes x (H + 3) x 8 bytes on the device (420 MB at 100 000 barcodes and 32 donors), zeroed when a submit starts a
 * fresh result set.  A locus whose row is >= n_rows is skipped and makes the next finish return VTX_E_INVALID.
 * vtx_donor_ll_get: after vtx_finish / vtx_finish_device, the sums over the submits since the previous finish:
 * ll[c * n_hyp + h] (int64, x VTX_DONOR_LL_SCALE) in the hypothesis order above, counts[c * 3 + {0, 1, 2}] = rows with
 * r + a > 0, the sum of r, the sum of a.  Library-owned host memory, valid until the next submit or finish. */
#define VTX_GT_MISSING 0xFFu
#define VTX_DONOR_LL_SCALE 16777216      /* 2^24 */
int         vtx_set_donors(vtx_ctx* ctx, uint32_t n_donors, uint64_t n_rows, const uint8_t* dosage, double error_rate);
int         vtx_donor_ll_get(vtx_ctx* ctx, const int64_t** ll, const uint64_t** counts, uint32_t* n_cols, uint32_t* n_hyp);

/* ---- genotype-free clustering of pooled cells (the CLI's --out-clusters; DESIGN.md §5g) ------------------------------------
 * An allele-fraction EM with k clusters over host count entries (row, col, ref_cnt, alt_cnt), e.g. a finished vtx_result:
 * strictly ascending (row, col) in row-major order, row < n_rows, col < n_cols.  Entries with ref + alt = 0 are ignored.  A row
 * is used when at least 4 cells have ref > 0 there and at least 4 have alt > 0.  Cluster k has theta_kv =
 * (A_kv + 2^16) / (T_kv + 2^17) at row v, A / T the cells' ALT / REF + ALT counts weighted by W_ck <= 2^16.  `restarts` EMs
 * start from seeded random thetas and run until W repeats or for 200 iterations; the one with the largest
 * sum_c max_k LL_ck wins (ties: the lowest restart).  Its clusters are ordered by sum_c W_ck, descending (ties: EM index).
 * Everything is integer or correctly rounded double arithmetic: the result is a function of the entries and the parameters.
 *
 * out->ll[c * n_hyp + h] (int64, x VTX_DONOR_LL_SCALE) scores the cell over used rows against the n_hyp = k + k(k-1)/2
 * hypotheses in vtx_set_donors' order (singlet C_h, then the 50/50 doublets); counts[c * 3 + {0, 1, 2}] = used entries, REF, ALT.
 * alt_w / depth_w [row * k + j] are the winner's final A, T over every row (x 2^16); restart_score / restart_iters per restart.
 * Library-owned host memory, valid until the next vtx_cluster_cells or vtx_destroy.  VTX_E_STATE while submits are unfinished
 * (between a submit and its finish); VTX_E_INVALID for k outside 2..32, restarts outside 1..64, a bad entry, or a row whose
 * ref + alt molecules times 2^16 (plus 2^17) reach 2^53; VTX_E_NOMEM when the device cannot hold 28 bytes per entry,
 * restarts x n_cols x k x 4 bytes of weights and restarts x n_rows x k x 8 bytes of tables. */
typedef struct vtx_cluster_params { uint32_t k, restarts; uint64_t seed; } vtx_cluster_params;
typedef struct vtx_clusters {
    uint32_t k, n_cols, n_hyp, best_restart; uint64_t n_rows, rows_used;
    const int64_t* ll;            /* [n_cols][n_hyp] x 2^24, canonical cluster order */
    const uint64_t* counts;       /* [n_cols][3] variants, ref, alt over used rows */
    const uint8_t* row_used;      /* [n_rows] */
    const int64_t* alt_w; const int64_t* depth_w;   /* [n_rows][k] x 2^16: final A, T over all rows */
    const int64_t* restart_score; const uint32_t* restart_iters;   /* [restarts] */
} vtx_clusters;
int         vtx_cluster_cells(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                              const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const vtx_cluster_params* params,
                              vtx_clusters* out);

/* ---- clustering of a pool where some donors are genotyped (the CLI's --known-donors; DESIGN.md §5k) --------------------------
 * vtx_cluster_cells' model over the same entries, with the first n_pinned = J clusters (1 <= J <= k - 1) pinned to samples of
 * known genotype: dosage [row * J + j] is 0, 1, 2 or VTX_GT_MISSING for every row < n_rows.  Where sample j has a dosage g at
 * row v, cluster j is not fitted: it expects vtx_donors_ambient's contaminated fraction theta_jv = (1 - rho) q_2g + rho f_v
 * (q_0, q_2, q_4 = error_rate, 0.5, 1 - error_rate; f_v the pool's ALT fraction over every entry at row v; rho = m / 1000 with
 * m = rho_permille, given), with vtx_donors_ambient's int32 logs, for the whole EM; the scoring mixes that theta into the
 * doublets as it mixes every other cluster's.  Where sample j has no dosage, cluster j is an ordinary cluster of that row.
 * Clusters 0 .. J - 1 keep their indices (the samples' order); clusters J .. k - 1 are free and ordered among themselves by
 * sum_c W_ck, descending (ties: EM index).  alt_w / depth_w hold the winner's final A, T of every cluster, pinned ones included.
 *
 * out is filled as vtx_cluster_cells fills it, library-owned host memory valid until the next vtx_cluster_cells,
 * vtx_cluster_cells_pinned or vtx_destroy.  Device memory: vtx_cluster_cells' plus J + 16 bytes per row.  VTX_E_STATE while
 * submits are unfinished; VTX_E_INVALID for vtx_cluster_cells' refusals, n_pinned outside 1 .. k - 1, a NULL dosage, a dosage
 * other than 0, 1, 2 or VTX_GT_MISSING, error_rate outside [1e-6, 0.25] or rho_permille outside 0 .. 500 (a row's T_v + 2
 * stays below 2^53: vtx_cluster_cells' bound on a row's molecules is far lower); VTX_E_NOMEM when the device cannot hold it. */
typedef struct vtx_cluster_pinned_params {
    uint32_t k, restarts; uint64_t seed;
    uint32_t n_pinned; double error_rate; int32_t rho_permille;
} vtx_cluster_pinned_params;
int         vtx_cluster_cells_pinned(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                                     const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const uint8_t* dosage,
                                     const vtx_cluster_pinned_params* params, vtx_clusters* out);

/* ---- donor assignment against ambient RNA (the CLI's --ambient-rna; DESIGN.md §5h) -----------------------------------------
 * vtx_set_donors' model over host count entries (row, col, ref_cnt, alt_cnt) as vtx_cluster_cells takes them, with the pool's
 * ALT fraction mixed into every hypothesis: at row v, q_vs = (1 - rho) q_s + rho f_v and 1 - q_vs = (1 - rho)(1 - q_s) +
 * rho (1 - f_v), f_v = (A_v + 1) / (T_v + 2) and 1 - f_v = (T_v - A_v + 1) / (T_v + 2) with A_v / T_v the sums of alt / ref + alt
 * over every entry at row v, rho = m / 1000 for m in 0..500.  The constants are llrint(log(q) 2^24) with vtx_cluster_cells'
 * correctly rounded log, so at rho = 0 they equal vtx_set_donors' wherever the two logs round alike.  dosage[row * n_donors + d]
 * as vtx_set_donors takes it, for every row < n_rows; a row is usable when every donor has a dosage there.
 * rho_permille = m fixes rho; -1 estimates it: J(m) = sum over cells with variants of max_h LL_ch is evaluated at m = 0, 10, ...,
 * 500 and then at every m within 9 of the best of those; the largest J wins (ties: the smallest m).  The cells are then scored
 * at the winner.  grid_batch > 0 caps the m values scored per pass (0: as device memory allows); it does not change the result.
 *
 * out->ll [c * n_hyp + h] (x VTX_DONOR_LL_SCALE) and counts [c * 3 + {0, 1, 2}] as vtx_donor_ll_get returns them, at the chosen
 * m (out->rho_permille).  grid_permille / grid_objective / grid_calls [i * 3 + {singlet, doublet, unassigned}] per evaluated m,
 * ascending (the calls use vtx_set_donors' rule with T = 5 nats); row_alt / row_depth [row] = A_v, T_v.  Library-owned host
 * memory, valid until the next vtx_donors_ambient or vtx_destroy.  VTX_E_STATE while submits are unfinished; VTX_E_INVALID for
 * n_donors outside 2..32, error_rate outside [1e-6, 0.25], rho_permille outside -1..500, a dosage other than 0, 1, 2 or
 * VTX_GT_MISSING, a bad entry (as vtx_cluster_cells), or a row whose T_v + 2 reaches 2^53; VTX_E_NOMEM when the device cannot
 * hold the entries (28 bytes each), 21 bytes per row, the cells' log-likelihoods and one m's tables (40 bytes per usable row that
 * an entry touches). */
typedef struct vtx_ambient_params {
    uint32_t n_donors; double error_rate; int32_t rho_permille;      /* -1: estimate */
    uint32_t grid_batch;                                              /* 0: as memory allows; else at most this many m per pass */
} vtx_ambient_params;
typedef struct vtx_ambient {
    uint32_t n_donors, n_cols, n_hyp, rho_permille, n_evaluated; uint64_t n_rows, rows_usable;
    const int64_t* ll; const uint64_t* counts;               /* [n_cols][n_hyp] x 2^24, [n_cols][3]: as vtx_donor_ll_get */
    const uint16_t* grid_permille; const int64_t* grid_objective; const uint64_t* grid_calls;   /* [n_evaluated], ascending m; calls [.][3] */
    const uint64_t* row_alt; const uint64_t* row_depth;       /* [n_rows]: A_v, T_v */
} vtx_ambient;
int         vtx_donors_ambient(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                               const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const uint8_t* dosage,
                               const vtx_ambient_params* params, vtx_ambient* out);

/* ---- genotypes of clusters against ambient RNA, and their match to genotyped samples (the CLI's --out-cluster-genotypes /
 * --out-cluster-matches; DESIGN.md §5i) ---------------------------------------------------------------------------------------
 * Over n_rows matrix rows: alt_w / depth_w [row * k + j] and row_used [row] as vtx_cluster_cells returns them (A_kv, T_kv x 2^16,
 * R_kv = T_kv - A_kv), row_alt / row_depth [row] = A_v, T_v as vtx_donors_ambient returns them (the sums of alt / ref + alt over
 * every entry at the row).  At rho = m / 1000 a dosage g in {0, 1, 2} expects vtx_donors_ambient's q_vs for q_s = error_rate,
 * 0.5 and 1 - error_rate, with its int32 logs La_g / Lr_g, and LL_vkg = floor((A_kv La_g + R_kv Lr_g) / 2^16) exactly (int64,
 * x VTX_DONOR_LL_SCALE).  rho_permille = m fixes rho; -1 estimates it: J(m) = sum over used rows and every cluster of max_g
 * LL_vkg on vtx_donors_ambient's grid (m = 0, 10, ..., 500, then every m within 9 of the best; the largest J wins, ties the
 * smallest m).  At the chosen m each (row, cluster) with T_kv > 0 gets GT = argmax_g LL (ties: the lowest g) and
 * PL_g = floor((10 (LL_max - LL_g) + floor(L10 / 2)) / L10) saturated at 2^31 - 1, L10 = llrint(log(10) 2^24) = 38630967.
 * GQ = min(99, the second-smallest PL).  With n_samples = S > 0, dosage [row * S + s] is 0, 1, 2 or VTX_GT_MISSING; over the
 * rows where every sample has a dosage ("compared"), match_ll [j * S + s] = sum of LL_{v,j,g_sv}, match_discordant [j * S + s]
 * = the compared rows with GQ >= 20 where GT differs from g_sv, match_rows [j] = the compared rows with T_jv > 0 and
 * match_called [j] = the compared rows with GQ >= 20.
 *
 * "Touched" rows are those with T_kv > 0 for some k; gt [t * k + j] (VTX_GT_MISSING where T_jv = 0) and pl [(t * k + j) * 3 + g]
 * follow `touched` (ascending matrix rows).  rows_fit = used rows that are touched.  Library-owned host memory, valid until the
 * next vtx_cluster_genotypes or vtx_destroy.  VTX_E_STATE while submits are unfinished; VTX_E_INVALID for k outside 2..32,
 * n_samples above 1024 (or > 0 with a NULL dosage), error_rate outside [1e-6, 0.25], rho_permille outside -1..500,
 * alt_w < 0 or > depth_w, depth_w > 2^51, depth_w summing over every row and cluster to more than 2^51 (J and match_ll stay
 * in int64), row_alt > row_depth or row_depth + 2 reaching 2^53, a dosage other than 0, 1, 2 or VTX_GT_MISSING, or n_rows
 * reaching 2^32; VTX_E_NOMEM when the device cannot hold about 53 k + 16 bytes per touched row and 4 + S per compared one. */
typedef struct vtx_cluster_gt_params {
    uint32_t k; double error_rate; int32_t rho_permille;             /* -1: estimate */
    uint32_t n_samples;
} vtx_cluster_gt_params;
typedef struct vtx_cluster_gt {
    uint32_t k, n_samples, rho_permille, n_evaluated; uint64_t n_rows, rows_fit, n_touched, rows_compared;
    const uint16_t* grid_permille; const int64_t* grid_objective;  /* [n_evaluated], ascending m */
    const uint64_t* touched;                                       /* [n_touched] ascending matrix rows */
    const uint8_t* gt; const uint32_t* pl;                         /* [n_touched][k], [n_touched][k][3]; VTX_GT_MISSING where T_kv = 0 */
    const int64_t* match_ll; const uint64_t* match_discordant;     /* [k][n_samples] */
    const uint64_t* match_rows; const uint64_t* match_called;      /* [k] */
} vtx_cluster_gt;
int         vtx_cluster_genotypes(vtx_ctx* ctx, uint64_t n_rows, const int64_t* alt_w, const int64_t* depth_w, const uint8_t* row_used,
                                  const uint64_t* row_alt, const uint64_t* row_depth, const uint8_t* dosage,
                                  const vtx_cluster_gt_params* params, vtx_cluster_gt* out);

/* ---- cells called against their clusters' fitted genotypes and ambient RNA, with the clusters refit from their singlets (the
 * CLI's --out-cluster-calls; DESIGN.md §5j) -------------------------------------------------------------------------------------
 * Count entries (row, col, ref_cnt, alt_cnt) as vtx_cluster_cells takes them, and that call's k, alt_w / depth_w [row * k + j] and
 * row_used [row].  Round 0 fits vtx_cluster_genotypes' model (rho estimated, error_rate as there) on alt_w / depth_w; every later
 * round first rebuilds the sums from the previous round's labels: A_kv = 2^16 sum a, T_kv = 2^16 sum (r + a) over the entries of
 * the cells labelled k.  At the round's m a (touched row, cluster) has code GT when GQ >= 20, else P (no called genotype); a row
 * with a called code is scored.  A hypothesis (i, j) in vtx_set_donors' order expects vtx_donors_ambient's q_vs for s = g_i + g_j
 * when both are called, (1 - rho)((q_2g + f_v) / 2) + rho f_v when one is (g its GT), f_v when neither is; cells add r Lr + a La
 * (int32 logs, x VTX_DONOR_LL_SCALE) at scored rows and are called with T = 5 nats.  A singlet on k is labelled k, every other
 * cell VTX_NO_LABEL.  The loop stops when a round's labels equal the previous round's (converged = 1) or after max_rounds rounds
 * after round 0 (converged = 0; max_rounds = 0 runs round 0 only).
 *
 * out->ll [c * n_hyp + h] and counts [c * 3 + {scored rows, ref, alt}] are the last round's, as vtx_donor_ll_get returns them;
 * label [c] its labels; rounds [r] per round; touched / gt / pl the last round's fit as vtx_cluster_genotypes returns them.
 * Library-owned host memory, valid until the next vtx_cluster_refine or vtx_destroy.  VTX_E_STATE while submits are unfinished;
 * VTX_E_INVALID for k outside 2..32, error_rate outside [1e-6, 0.25], max_rounds above 32, a bad entry (as vtx_cluster_cells),
 * 2^16 x the entries' ref + alt summing to more than 2^51, or alt_w / depth_w outside vtx_cluster_genotypes' bounds;
 * VTX_E_NOMEM when the device cannot hold 28 bytes per entry, about 70 k + 150 bytes per row and 4 k + 8 n_hyp + 40 per cell. */
#define VTX_NO_LABEL 0xFFFFFFFFu
typedef struct vtx_cluster_calls_params { uint32_t k; double error_rate; uint32_t max_rounds; } vtx_cluster_calls_params;
typedef struct vtx_cluster_calls_round {
    uint32_t rho_permille, reserved; uint64_t rows_fit, n_touched, rows_scored;
    uint64_t calls[3];                /* singlet, doublet, unassigned */
    uint64_t changed;                 /* labels that differ from the previous round's (round 0: from VTX_NO_LABEL) */
} vtx_cluster_calls_round;
typedef struct vtx_cluster_calls {
    uint32_t k, n_cols, n_hyp, n_rounds; int32_t converged; uint32_t reserved; uint64_t n_rows, n_touched;
    const int64_t* ll; const uint64_t* counts;       /* [n_cols][n_hyp] x 2^24, [n_cols][3] */
    const uint32_t* label;                           /* [n_cols] cluster or VTX_NO_LABEL */
    const vtx_cluster_calls_round* rounds;          /* [n_rounds] */
    const uint64_t* touched;                         /* [n_touched] ascending matrix rows */
    const uint8_t* gt; const uint32_t* pl;           /* [n_touched][k], [n_touched][k][3] */
} vtx_cluster_calls;
int         vtx_cluster_refine(vtx_ctx* ctx, uint64_t n, const uint32_t* row, const uint32_t* col, const uint32_t* ref_cnt,
                               const uint32_t* alt_cnt, uint64_t n_rows, uint32_t n_cols, const int64_t* alt_w, const int64_t* depth_w,
                               const uint8_t* row_used, const vtx_cluster_calls_params* params, vtx_cluster_calls* out);

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
