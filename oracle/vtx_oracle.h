/*
 * vtx_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the per-locus read-scoring path of 10XGenomics/vartrix
 * (reference: vartrix src/main.rs, v1.1.22).  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference leg may load this library.  The product
 * (vartrix_b200/) never links, imports or executes anything in oracle/.
 *
 * Parity status: PINNED at matrix level by the reference's 12 golden .mtx files
 * (oracle/check_goldens.py reproduces all of them through this code).  Raw alignment
 * scores are pinned only through those matrices: the reference delegates Smith-Waterman
 * to the un-vendored crate bio 0.30.0 (Cargo.lock:175-177), a *banded* aligner (k=6, w=20)
 * whose source is not on this machine.  This oracle computes the exact full-matrix affine
 * local score (the upper bound of any band, equal to it whenever the optimal path stays
 * inside the band), which reproduces every golden.
 */
#ifndef VTX_ORACLE_H
#define VTX_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* main.rs:27-38 */
#define VTXO_MIN_SCORE   25
#define VTXO_MATCH        1
#define VTXO_MISMATCH    (-5)
#define VTXO_GAP_OPEN    (-5)
#define VTXO_GAP_EXTEND  (-1)

#define VTXO_MODE_CONSENSUS 0
#define VTXO_MODE_COVERAGE  1
#define VTXO_MODE_ALT_FRAC  2

#define VTXO_NO_CB   0xFFFFFFFFu
#define VTXO_NO_UMI  0xFFFFFFFFFFFFFFFFull

/* Staged batch: same layout as the product's C-ABI (include/vartrix_b200.h, vtx_batch) so
 * identical buffers can be handed to both sides.  Declared independently on purpose. */
typedef struct vtxo_batch {
    uint32_t        n_loci;
    const uint32_t* locus_row;     /* [n_loci] output row (VCF record index) */
    const uint8_t*  hap_bytes;     /* ASCII haplotype pool */
    uint64_t        hap_bytes_len;
    const uint32_t* ref_off;       /* [n_loci] */
    const uint32_t* ref_len;
    const uint32_t* alt_off;
    const uint32_t* alt_len;
    const uint64_t* cand_start;    /* [n_loci+1] candidate range of each locus */
    uint32_t        n_reads;
    const uint8_t*  read_nib;      /* BAM 4-bit bases, high nibble first */
    uint64_t        read_nib_len;
    const uint64_t* read_off;      /* [n_reads] byte offset of each read */
    const uint32_t* read_len;      /* [n_reads] bases */
    const uint8_t*  cb_bytes;      /* cell-barcode tag pool */
    uint64_t        cb_bytes_len;
    const uint32_t* read_cb_off;   /* [n_reads] VTXO_NO_CB = no Z-typed tag */
    const uint16_t* read_cb_len;
    const uint64_t* read_umi_key;  /* [n_reads] injective key of the UB string, VTXO_NO_UMI = absent */
    uint64_t        n_cand;
    const uint32_t* cand_read;     /* [n_cand] read id, locus-major, BAM file order inside a locus */
} vtxo_batch;

typedef struct vtxo_metrics {      /* main.rs:449-459 (device-side subset) */
    uint64_t num_not_cell_bc;
    uint64_t num_non_umi;
    uint64_t num_scored;           /* pairs that reach main.rs:896-930 */
} vtxo_metrics;

/* Affine local Smith-Waterman score, byte equality, full matrix (see header comment). */
int32_t vtxo_sw_full(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n);

/* The same score through the prefix / reversed-suffix / middle / junction decomposition the GPU fold kernel uses
 * (any P + S <= n); exists so that the decomposition is pinned on the CPU against vtxo_sw_full. */
int32_t vtxo_sw_fold(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n, int32_t P, int32_t S);

/* Best-effort model of bio 0.30.0's band (k-mer seeds, sparse chain, +-w band, lazy ends);
 * DIAGNOSTIC ONLY -- used to count pairs whose banded score could differ from the full one. */
int32_t vtxo_sw_band_model(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n, int32_t k, int32_t w);

/* main.rs:1019-1030 with MIN_SCORE = VTXO_MIN_SCORE : 0 = None, 1 = REF, 2 = ALT, -1 = UNKNOWN */
int32_t vtxo_evaluate_scores(int32_t ref_score, int32_t alt_score);

/* rust-htslib 0.36 CigarStringView::read_pos(p, false, true) folded into main.rs:790-806.
 * cigar = BAM-encoded ops (len<<4|op).  Returns 1 useful, 0 not. */
int32_t vtxo_useful_alignment(int64_t pos, const uint32_t* cigar, int32_t n_cigar, int64_t start, int64_t end);

/* BAM nibbles -> ASCII "=ACMGRSVTWYHKDBN" (main.rs:896). */
void vtxo_decode_read(const uint8_t* nib, int32_t len, uint8_t* out);

/* Raw scores for an explicit pair list: pair i = (pair_read[i], pair_locus[i]). */
int32_t vtxo_score_pairs(const vtxo_batch* b, uint64_t n_pairs, const uint32_t* pair_read,
                         const uint32_t* pair_locus, int32_t n_threads,
                         int32_t* ref_score, int32_t* alt_score);

/* Whole path for a staged batch: CB lookup (main.rs:737-750), UMI gate (879-888), 2x SW (898-901),
 * stable sort by cell (932), parse_scores (1041-1109), mode function (1111-1164), row-major merge
 * (320-348).  Loci are split into static contiguous chunks of max(n/threads,1) like main.rs:250-254.
 * min_score is MIN_SCORE of evaluate_scores (main.rs:30, 1019-1030): VTXO_MIN_SCORE in the reference, a run-time
 * setting of the engine (vtx_config.min_score) that this argument mirrors.
 * Output arrays are malloc'ed by the library; free with vtxo_free_result. */
typedef struct vtxo_result {
    uint64_t  n;          /* entries */
    uint32_t* row;
    uint32_t* col;
    uint32_t* ref_cnt;
    uint32_t* alt_cnt;
    uint32_t* unk_cnt;
    double*   val;        /* out-matrix value */
    double*   val2;       /* ref-matrix value (coverage mode), else 0 */
    vtxo_metrics metrics;
} vtxo_result;

int32_t vtxo_run_batch(const vtxo_batch* b,
                       const uint8_t* bc_bytes, const uint32_t* bc_off, uint32_t n_barcodes,
                       int32_t mode, int32_t use_umi, int32_t n_threads, int32_t use_band_model,
                       int32_t min_score, vtxo_result* out);
void vtxo_free_result(vtxo_result* r);

#ifdef __cplusplus
}
#endif
#endif
