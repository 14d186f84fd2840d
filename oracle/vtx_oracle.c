/*
 * vtx_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).  See vtx_oracle.h.
 *
 * Every function cites the reference lines it restates (vartrix src/main.rs unless
 * another file is named).  Third-party arithmetic that is absent from the reference tree:
 *   - bio 0.30.0 (Cargo.lock:175-177) bio::alignment::pairwise::banded::Aligner::local,
 *     called at main.rs:898-901: restated here from the published algorithm (Gotoh affine
 *     local alignment; scoring closure main.rs:898; constants main.rs:33-38).
 *   - rust-htslib 0.36.0 (Cargo.lock:1332-1334) CigarStringView::read_pos, called at main.rs:796.
 * Parity is pinned by the reference's own golden matrices (test/ *.mtx) via oracle/check_goldens.py.
 */
#include "vtx_oracle.h"

#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <stddef.h>

#define NEG_INF (-(1 << 28))

static inline int32_t imax(int32_t a, int32_t b) { return a > b ? a : b; }
static inline int32_t imin(int32_t a, int32_t b) { return a < b ? a : b; }

/* ------------------------------------------------------------------------------------------
 * Smith-Waterman.  x = read (rows), y = haplotype (columns), as in main.rs:900-901
 * (aligner.local(seq, hap)).  Recurrence = bio 0.30.0 pairwise `local` with all clip penalties 0:
 *   I[i][j] = max(I[i-1][j] + ge, S[i-1][j] + go + ge)
 *   D[i][j] = max(D[i][j-1] + ge, S[i][j-1] + go + ge)
 *   S[i][j] = max(S[i-1][j-1] + score(x_i, y_j), I, D, 0)      answer = max S
 * score = +1 on byte equality else -5 (main.rs:898, 35-36), go = -5, ge = -1 (main.rs:37-38).
 * ------------------------------------------------------------------------------------------ */
int32_t vtxo_sw_full(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n)
{
    if (m <= 0 || n <= 0) return 0;
    const int32_t go = VTXO_GAP_OPEN, ge = VTXO_GAP_EXTEND;
    int32_t stack_s[512], stack_d[512];
    int32_t* S = (n + 1 <= 512) ? stack_s : (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    int32_t* I = (n + 1 <= 512) ? stack_d : (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    for (int32_t j = 0; j <= n; ++j) { S[j] = 0; I[j] = NEG_INF; }
    int32_t best = 0;
    for (int32_t i = 1; i <= m; ++i) {
        const uint8_t xi = x[i - 1];
        int32_t diag = S[0];        /* S[i-1][0] = 0 */
        int32_t left = 0;           /* S[i][0]   = 0 */
        int32_t d = NEG_INF;        /* D[i][0] */
        for (int32_t j = 1; j <= n; ++j) {
            int32_t up = S[j];
            int32_t ins = imax(I[j] + ge, up + go + ge);    /* vertical gap (consumes x) */
            d = imax(d + ge, left + go + ge);               /* horizontal gap (consumes y) */
            int32_t s = diag + (xi == y[j - 1] ? VTXO_MATCH : VTXO_MISMATCH);
            s = imax(s, ins);
            s = imax(s, d);
            s = imax(s, 0);
            I[j] = ins;
            diag = up;
            S[j] = s;
            left = s;
            if (s > best) best = s;
        }
    }
    if (S != stack_s) { free(S); free(I); }
    return best;
}

/* ------------------------------------------------------------------------------------------
 * "Fold" decomposition of the same score (CHECKER for the GPU kernel vtx_k_sw_fold, which relies on
 * it; the decomposition itself is proven in DESIGN.md and pinned numerically by tests/test_fold_math_cpu.py):
 *   columns [0, P)      forward DP            -> last column (H, D) per row + maximum
 *   columns [n - S, n)  DP of the REVERSED read against the reversed columns -> (Hr, Dr) per row + maximum
 *   columns [P, n - S)  forward DP continued from the forward boundary
 *   junction            max_i  max( H(i, last) + Hr(i + 1),  D(i, last) + Dr(i + 1) - go )
 * (D = horizontal-gap state; "- go" because a gap running across the junction was opened on both sides).
 * Any P + S <= n gives vtxo_sw_full(x, m, y, n).
 * ------------------------------------------------------------------------------------------ */
static int32_t fold_pass(const uint8_t* x, int32_t m, int32_t xstep, const uint8_t* y, int32_t ncol, int32_t ystep,
                         int32_t* H, int32_t* D /* in: boundary left of the first column; out: last column; [m + 1] */)
{
    /* x[i * xstep], y[j * ystep]: a pass over ncol columns continuing from the boundary column (H, D) */
    const int32_t go = VTXO_GAP_OPEN, ge = VTXO_GAP_EXTEND;
    int32_t best = 0;
    for (int32_t j = 0; j < ncol; ++j) {
        const uint8_t yj = y[(ptrdiff_t)j * ystep];
        int32_t diag = H[0], ins = NEG_INF;           /* row 0: H = 0 */
        for (int32_t i = 1; i <= m; ++i) {
            const int32_t left = H[i];
            const int32_t d = imax(D[i] + ge, left + go + ge);
            ins = imax(ins + ge, H[i - 1] + go + ge);  /* H[i-1] already holds this column */
            int32_t s = diag + (x[(ptrdiff_t)(i - 1) * xstep] == yj ? VTXO_MATCH : VTXO_MISMATCH);
            s = imax(imax(s, ins), imax(d, 0));
            diag = left;
            H[i] = s; D[i] = d;
            if (s > best) best = s;
        }
    }
    return best;
}

int32_t vtxo_sw_fold(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n, int32_t P, int32_t S)
{
    if (m <= 0 || n <= 0) return 0;
    if (P < 0 || S < 0 || P + S > n) return -1;
    int32_t* buf = (int32_t*)malloc(sizeof(int32_t) * 4 * (size_t)(m + 2));
    int32_t *Hf = buf, *Df = Hf + (m + 2), *Hr = Df + (m + 2), *Dr = Hr + (m + 2);
    for (int32_t i = 0; i <= m + 1; ++i) { Hf[i] = 0; Df[i] = NEG_INF; Hr[i] = 0; Dr[i] = NEG_INF; }
    int32_t best = fold_pass(x, m, 1, y, P, 1, Hf, Df);                                   /* prefix */
    if (S > 0) best = imax(best, fold_pass(x + (m - 1), m, -1, y + (n - 1), S, -1, Hr, Dr)); /* reversed suffix */
    best = imax(best, fold_pass(x, m, 1, y + P, n - S - P, 1, Hf, Df));                   /* middle, from the boundary */
    /* junction: forward row i (1-based) meets reversed row m - i */
    for (int32_t i = 1; i <= m - 1; ++i) {
        best = imax(best, Hf[i] + Hr[m - i]);
        if (Df[i] > NEG_INF / 2 && Dr[m - i] > NEG_INF / 2) best = imax(best, Df[i] + Dr[m - i] - VTXO_GAP_OPEN);
    }
    free(buf);
    return best;
}

/* ------------------------------------------------------------------------------------------
 * Band model (DIAGNOSTIC).  Restates, as far as it can be recalled without the crate source,
 * bio 0.30.0 banded::Band::create (SURVEY.md Appendix B, model "B" = the one consistent with
 * every golden): exact k-mer hits, sparse chain with free same-diagonal skips and
 * go + ge*|delta diag| for diagonal changes, band = +-w box swept along chained hits, straight
 * fill between hits, lazy 2k diagonal extension at both ends.  No hits -> full matrix.
 * ------------------------------------------------------------------------------------------ */
typedef struct { int32_t i, j; } hit_t;

static int hit_cmp(const void* a, const void* b)
{
    const hit_t* p = (const hit_t*)a; const hit_t* q = (const hit_t*)b;
    if (p->i != q->i) return p->i < q->i ? -1 : 1;
    if (p->j != q->j) return p->j < q->j ? -1 : 1;
    return 0;
}

static void band_add_box(int32_t* lo, int32_t* hi, int32_t m, int32_t n, int32_t i, int32_t j, int32_t w)
{
    /* cell (i,j) in 1-based DP coordinates (row i, col j); widen every column within +-w */
    int32_t j0 = imax(j - w, 0), j1 = imin(j + w, n);
    int32_t i0 = imax(i - w, 0), i1 = imin(i + w, m);
    for (int32_t c = j0; c <= j1; ++c) {
        if (i0 < lo[c]) lo[c] = i0;
        if (i1 > hi[c]) hi[c] = i1;
    }
}

int32_t vtxo_sw_band_model(const uint8_t* x, int32_t m, const uint8_t* y, int32_t n, int32_t k, int32_t w)
{
    if (m < k || n < k) return vtxo_sw_full(x, m, y, n);
    /* 1. all exact k-mer hits (i,j): x[i..i+k) == y[j..j+k) */
    size_t cap = 1024, nh = 0;
    hit_t* hits = (hit_t*)malloc(cap * sizeof(hit_t));
    for (int32_t i = 0; i + k <= m; ++i)
        for (int32_t j = 0; j + k <= n; ++j)
            if (memcmp(x + i, y + j, (size_t)k) == 0) {
                if (nh == cap) { cap *= 2; hits = (hit_t*)realloc(hits, cap * sizeof(hit_t)); }
                hits[nh].i = i; hits[nh].j = j; ++nh;
            }
    if (nh == 0) { free(hits); return vtxo_sw_full(x, m, y, n); }
    qsort(hits, nh, sizeof(hit_t), hit_cmp);
    /* 2. chain (O(h^2) restatement of the sparse DP; h is a few hundred at most here) */
    int32_t* sc = (int32_t*)malloc(nh * sizeof(int32_t));
    int32_t* pr = (int32_t*)malloc(nh * sizeof(int32_t));
    int32_t best = -1; size_t best_idx = 0;
    for (size_t a = 0; a < nh; ++a) {
        sc[a] = k; pr[a] = -1;
        for (size_t b = 0; b < a; ++b) {
            int32_t di = hits[a].i - hits[b].i, dj = hits[a].j - hits[b].j;
            int32_t cand;
            if (di == 1 && dj == 1) cand = sc[b] + 1;                     /* extend the same run */
            else if (di >= k && dj >= k) {
                int32_t dd = di - dj; if (dd < 0) dd = -dd;
                cand = sc[b] + k + (dd ? VTXO_GAP_OPEN + VTXO_GAP_EXTEND * dd : 0);
            } else continue;
            if (cand > sc[a]) { sc[a] = cand; pr[a] = (int32_t)b; }
        }
        if (sc[a] > best) { best = sc[a]; best_idx = a; }
    }
    /* 3. band as per-column row ranges [lo, hi] over the (m+1) x (n+1) DP matrix */
    int32_t* lo = (int32_t*)malloc((size_t)(n + 1) * sizeof(int32_t));
    int32_t* hi = (int32_t*)malloc((size_t)(n + 1) * sizeof(int32_t));
    for (int32_t c = 0; c <= n; ++c) { lo[c] = m + 1; hi[c] = -1; }
    int32_t cur = (int32_t)best_idx, last_i = -1, last_j = -1, first_i = 0, first_j = 0;
    while (cur >= 0) {
        int32_t hi_i = hits[cur].i, hi_j = hits[cur].j;
        for (int32_t t = 0; t <= k; ++t) band_add_box(lo, hi, m, n, hi_i + t, hi_j + t, w);
        if (last_i >= 0) {
            /* fill between this hit's end and the later hit's start: straight run then diagonal */
            int32_t ai = hi_i + k, aj = hi_j + k;
            while (ai < last_i || aj < last_j) {
                if (last_i - ai > last_j - aj) ++ai;
                else if (last_j - aj > last_i - ai) ++aj;
                else { ++ai; ++aj; }
                band_add_box(lo, hi, m, n, ai, aj, w);
            }
        }
        last_i = hi_i; last_j = hi_j; first_i = hi_i; first_j = hi_j;
        cur = pr[cur];
    }
    /* lazy extension: 2k diagonal cells beyond both ends */
    for (int32_t t = 1; t <= 2 * k; ++t) {
        int32_t ai = first_i - t, aj = first_j - t;
        if (ai >= 0 && aj >= 0) band_add_box(lo, hi, m, n, ai, aj, w);
        ai = hits[best_idx].i + k + t; aj = hits[best_idx].j + k + t;
        if (ai <= m && aj <= n) band_add_box(lo, hi, m, n, ai, aj, w);
    }
    /* 4. banded DP, column-major like the crate; out-of-band predecessors are -inf */
    int32_t* S0 = (int32_t*)malloc((size_t)(m + 1) * sizeof(int32_t) * 6);
    int32_t *S1 = S0 + (m + 1), *I0 = S1 + (m + 1), *I1 = I0 + (m + 1), *D0 = I1 + (m + 1), *D1 = D0 + (m + 1);
    for (int32_t i = 0; i <= m; ++i) { S0[i] = S1[i] = I0[i] = I1[i] = D0[i] = D1[i] = NEG_INF; }
    int32_t ans = 0;
    const int32_t go = VTXO_GAP_OPEN, ge = VTXO_GAP_EXTEND;
    for (int32_t j = 0; j <= n; ++j) {
        int32_t *Sc = (j & 1) ? S1 : S0, *Sp = (j & 1) ? S0 : S1;
        int32_t *Ic = (j & 1) ? I1 : I0;
        int32_t *Dc = (j & 1) ? D1 : D0, *Dp = (j & 1) ? D0 : D1;
        for (int32_t i = 0; i <= m; ++i) { Sc[i] = NEG_INF; Ic[i] = NEG_INF; Dc[i] = NEG_INF; }
        if (hi[j] < 0) continue;
        for (int32_t i = lo[j]; i <= hi[j]; ++i) {
            int32_t s = 0, ins = NEG_INF, del = NEG_INF;
            if (i > 0 && j > 0) {
                if (Sp[i - 1] > NEG_INF / 2)
                    s = imax(s, Sp[i - 1] + (x[i - 1] == y[j - 1] ? VTXO_MATCH : VTXO_MISMATCH));
            }
            if (i > 0) {
                if (Ic[i - 1] > NEG_INF / 2) ins = Ic[i - 1] + ge;
                if (Sc[i - 1] > NEG_INF / 2) ins = imax(ins, Sc[i - 1] + go + ge);
            }
            if (j > 0) {
                if (Dp[i] > NEG_INF / 2) del = Dp[i] + ge;
                if (Sp[i] > NEG_INF / 2) del = imax(del, Sp[i] + go + ge);
            }
            s = imax(s, imax(ins, del));
            Sc[i] = s; Ic[i] = ins; Dc[i] = del;
            if (s > ans) ans = s;
        }
    }
    free(S0); free(lo); free(hi); free(sc); free(pr); free(hits);
    return ans;
}

/* main.rs:1019-1030; min_score = MIN_SCORE (main.rs:30), a run-time setting of the engine (vtx_config.min_score) */
static int32_t evaluate_scores(int32_t ref_score, int32_t alt_score, int32_t min_score)
{
    if (ref_score < min_score && alt_score < min_score) return 0;            /* None */
    if (ref_score > alt_score) return 1;                                     /* REF_VALUE */
    if (alt_score > ref_score) return 2;                                     /* ALT_VALUE */
    return -1;                                                               /* UNKNOWN_VALUE */
}

int32_t vtxo_evaluate_scores(int32_t ref_score, int32_t alt_score)
{
    return evaluate_scores(ref_score, alt_score, VTXO_MIN_SCORE);
}

/* ------------------------------------------------------------------------------------------
 * useful_alignment (main.rs:790-806): true iff some p in start..=end has
 * cigar.read_pos(p, include_softclips=false, include_dels=true) == Ok(Some).  rust-htslib 0.36:
 *  - leading ops: the first of M,=,X,I,S begins the walk; a leading D or N is an error; an H that
 *    is not at either end is an error; nothing but H/P -> Ok(None)
 *  - walk with rpos = record pos: M/=/X and D cover [rpos, rpos+len); N advances; S/I/P do not.
 * An error makes main.rs:799-802 skip the read (returns false).
 * ------------------------------------------------------------------------------------------ */
static int cigar_read_pos_covers(int64_t pos, const uint32_t* cigar, int32_t nc, int64_t p, int* err)
{
    /* BAM op codes: 0 M, 1 I, 2 D, 3 N, 4 S, 5 H, 6 P, 7 =, 8 X */
    int32_t i = 0;
    *err = 0;
    /* leading section */
    while (i < nc) {
        uint32_t op = cigar[i] & 0xF;
        if (op == 0 || op == 7 || op == 8 || op == 1 || op == 4) break;
        if (op == 2 || op == 3) { *err = 1; return 0; }
        if (op == 5) { if (i != 0 && i != nc - 1) { *err = 1; return 0; } ++i; continue; }
        ++i; /* P */
    }
    if (i >= nc) return 0;
    int64_t rpos = pos;
    for (; i < nc; ++i) {
        uint32_t op = cigar[i] & 0xF; int64_t len = cigar[i] >> 4;
        if (rpos > p) break;
        switch (op) {
        case 0: case 7: case 8: case 2:
            if (p >= rpos && p < rpos + len) return 1;
            rpos += len; break;
        case 3: rpos += len; break;
        case 1: case 4: case 6: break;
        case 5: if (i != nc - 1) { *err = 1; return 0; } return 0;
        default: break;
        }
    }
    return 0;
}

int32_t vtxo_useful_alignment(int64_t pos, const uint32_t* cigar, int32_t n_cigar, int64_t start, int64_t end)
{
    for (int64_t p = start; p <= end; ++p) {          /* inclusive end: main.rs:794 */
        int err = 0;
        if (cigar_read_pos_covers(pos, cigar, n_cigar, p, &err)) return 1;
        if (err) return 0;                            /* main.rs:799-802 */
    }
    return 0;
}

/* main.rs:896: rec.seq().as_bytes() */
void vtxo_decode_read(const uint8_t* nib, int32_t len, uint8_t* out)
{
    static const char T[] = "=ACMGRSVTWYHKDBN";
    for (int32_t i = 0; i < len; ++i) {
        uint8_t b = nib[i >> 1];
        out[i] = (uint8_t)T[(i & 1) ? (b & 0xF) : (b >> 4)];
    }
}

/* ---------------------------------- barcode map (main.rs:697-718, 737-750) ------------------ */
typedef struct { const uint8_t* bytes; const uint32_t* off; uint32_t n; uint32_t cap; int32_t* slot; } bcmap_t;

static uint64_t fnv1a(const uint8_t* p, uint32_t n)
{
    uint64_t h = 1469598103934665603ull;
    for (uint32_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

static void bcmap_build(bcmap_t* m, const uint8_t* bytes, const uint32_t* off, uint32_t n)
{
    m->bytes = bytes; m->off = off; m->n = n;
    uint32_t cap = 16; while (cap < 2 * n + 1) cap <<= 1;
    m->cap = cap; m->slot = (int32_t*)malloc(cap * sizeof(int32_t));
    for (uint32_t i = 0; i < cap; ++i) m->slot[i] = -1;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t len = off[i + 1] - off[i];
        uint64_t h = fnv1a(bytes + off[i], len) & (cap - 1);
        for (;;) {
            int32_t s = m->slot[h];
            if (s < 0) { m->slot[h] = (int32_t)i; break; }
            uint32_t l2 = off[s + 1] - off[s];
            if (l2 == len && memcmp(bytes + off[s], bytes + off[i], len) == 0) break;  /* first wins, main.rs:706-709 */
            h = (h + 1) & (cap - 1);
        }
    }
}

static int32_t bcmap_get(const bcmap_t* m, const uint8_t* key, uint32_t len)
{
    uint64_t h = fnv1a(key, len) & (m->cap - 1);
    for (;;) {
        int32_t s = m->slot[h];
        if (s < 0) return -1;
        uint32_t l2 = m->off[s + 1] - m->off[s];
        if (l2 == len && memcmp(m->bytes + m->off[s], key, len) == 0) return s;
        h = (h + 1) & (m->cap - 1);
    }
}

/* ---------------------------------- raw pair scoring ---------------------------------------- */
typedef struct {
    const vtxo_batch* b; uint64_t lo, hi; const uint32_t *pr, *pl; int32_t *rs, *as;
} sp_job;

static void* sp_worker(void* arg)
{
    sp_job* j = (sp_job*)arg; const vtxo_batch* b = j->b;
    uint8_t buf[4096]; uint8_t* seq = buf; size_t cap = sizeof(buf);
    for (uint64_t p = j->lo; p < j->hi; ++p) {
        uint32_t r = j->pr[p], l = j->pl[p];
        uint32_t m = b->read_len[r];
        if (m > cap) { if (seq != buf) free(seq); cap = m; seq = (uint8_t*)malloc(cap); }
        vtxo_decode_read(b->read_nib + b->read_off[r], (int32_t)m, seq);
        j->rs[p] = vtxo_sw_full(seq, (int32_t)m, b->hap_bytes + b->ref_off[l], (int32_t)b->ref_len[l]);
        j->as[p] = vtxo_sw_full(seq, (int32_t)m, b->hap_bytes + b->alt_off[l], (int32_t)b->alt_len[l]);
    }
    if (seq != buf) free(seq);
    return NULL;
}

int32_t vtxo_score_pairs(const vtxo_batch* b, uint64_t n_pairs, const uint32_t* pair_read,
                         const uint32_t* pair_locus, int32_t n_threads,
                         int32_t* ref_score, int32_t* alt_score)
{
    if (n_threads < 1) n_threads = 1;
    if ((uint64_t)n_threads > n_pairs) n_threads = n_pairs ? (int32_t)n_pairs : 1;
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)n_threads);
    sp_job* jobs = (sp_job*)malloc(sizeof(sp_job) * (size_t)n_threads);
    uint64_t per = (n_pairs + (uint64_t)n_threads - 1) / (uint64_t)n_threads;
    for (int32_t t = 0; t < n_threads; ++t) {
        uint64_t lo = per * (uint64_t)t, hi = lo + per; if (lo > n_pairs) lo = n_pairs; if (hi > n_pairs) hi = n_pairs;
        jobs[t] = (sp_job){ b, lo, hi, pair_read, pair_locus, ref_score, alt_score };
        pthread_create(&th[t], NULL, sp_worker, &jobs[t]);
    }
    for (int32_t t = 0; t < n_threads; ++t) pthread_join(th[t], NULL);
    free(th); free(jobs);
    return 0;
}

/* ---------------------------------- whole path ---------------------------------------------- */
typedef struct { uint32_t cell; uint32_t ord; uint64_t umi; int32_t rs, as; } score_t;   /* main.rs:996-1001 */

static int score_cmp(const void* a, const void* b)
{   /* stable sort by cell_index (main.rs:932): ties keep insertion order */
    const score_t* p = (const score_t*)a; const score_t* q = (const score_t*)b;
    if (p->cell != q->cell) return p->cell < q->cell ? -1 : 1;
    return p->ord < q->ord ? -1 : (p->ord > q->ord);
}

typedef struct { uint32_t row, col, r, a, u; double v, v2; } entry_t;
typedef struct { entry_t* e; size_t n, cap; } evec_t;

static void evec_push(evec_t* v, entry_t x)
{
    if (v->n == v->cap) { v->cap = v->cap ? v->cap * 2 : 256; v->e = (entry_t*)realloc(v->e, v->cap * sizeof(entry_t)); }
    v->e[v->n++] = x;
}

/* parse_scores + convert_to_counts + mode function for one locus (main.rs:1041-1164) */
static void aggregate_locus(score_t* sc, size_t n, uint32_t row, int32_t mode, int32_t use_umi, int32_t min_score, evec_t* out)
{
    qsort(sc, n, sizeof(score_t), score_cmp);
    size_t i = 0;
    while (i < n) {
        size_t j = i; while (j < n && sc[j].cell == sc[i].cell) ++j;     /* group_by cell, main.rs:1044 */
        uint32_t r = 0, a = 0, u = 0;
        if (!use_umi) {
            for (size_t k = i; k < j; ++k) {                              /* main.rs:1090-1098 */
                int32_t c = evaluate_scores(sc[k].rs, sc[k].as, min_score);
                if (c == 1) ++r; else if (c == 2) ++a; else if (c == -1) ++u;
            }
        } else {
            /* per-UMI collapse, main.rs:1047-1082; O(g^2) over the (small) cell group */
            for (size_t k = i; k < j; ++k) {
                int seen = 0;
                for (size_t q = i; q < k; ++q) if (sc[q].umi == sc[k].umi) { seen = 1; break; }
                if (seen) continue;
                uint32_t ur = 0, ua = 0, uu = 0;
                for (size_t q = k; q < j; ++q) if (sc[q].umi == sc[k].umi) {
                    int32_t c = evaluate_scores(sc[q].rs, sc[q].as, min_score);
                    if (c == 1) ++ur; else if (c == 2) ++ua; else if (c == -1) ++uu;
                }
                uint32_t t = ur + ua + uu;
                if (t == 0) continue;                         /* no entry in parsed_scores: every call was None */
                double ref_frac = (double)ur / ((double)ua + (double)ur + (double)uu);   /* main.rs:1070-1073 */
                double alt_frac = (double)ua / ((double)ua + (double)ur + (double)uu);
                if (ref_frac < 0.75 && alt_frac < 0.75) ++u;                             /* main.rs:1074-1081 */
                else if (alt_frac >= 0.75) ++a;
                else ++r;
            }
        }
        entry_t e; e.row = row; e.col = sc[i].cell; e.r = r; e.a = a; e.u = u; e.v = 0; e.v2 = 0;
        if (mode == VTXO_MODE_CONSENSUS) {                    /* main.rs:1120-1126 */
            if (r > 0 && a > 0) { e.v = 3; evec_push(out, e); }
            else if (a > 0) { e.v = 2; evec_push(out, e); }
            else if (r > 0) { e.v = 1; evec_push(out, e); }
        } else if (mode == VTXO_MODE_ALT_FRAC) {              /* main.rs:1140-1142 (0/0 -> NaN) */
            e.v = (double)a / ((double)r + (double)a + (double)u);
            evec_push(out, e);
        } else {                                              /* coverage, main.rs:1160-1161 */
            e.v = (double)a; e.v2 = (double)r; evec_push(out, e);
        }
        i = j;
    }
}

typedef struct {
    const vtxo_batch* b; const bcmap_t* bc; uint32_t lo, hi; int32_t mode, use_umi, band, min_score;
    evec_t out; vtxo_metrics met;
} rb_job;

static void rb_chunk(rb_job* J)
{
    const vtxo_batch* b = J->b;
    size_t scap = 256; score_t* sc = (score_t*)malloc(scap * sizeof(score_t));
    size_t qcap = 4096; uint8_t* seq = (uint8_t*)malloc(qcap);
    for (uint32_t l = J->lo; l < J->hi; ++l) {                       /* evaluate_chunk, main.rs:596-607 */
        size_t n = 0;
        const uint8_t* rh = b->hap_bytes + b->ref_off[l]; int32_t nr = (int32_t)b->ref_len[l];
        const uint8_t* ah = b->hap_bytes + b->alt_off[l]; int32_t na = (int32_t)b->alt_len[l];
        for (uint64_t c = b->cand_start[l]; c < b->cand_start[l + 1]; ++c) {   /* evaluate_alns loop, main.rs:829 */
            uint32_t r = b->cand_read[c];
            int32_t cell = -1;
            if (b->read_cb_off[r] != VTXO_NO_CB)
                cell = bcmap_get(J->bc, b->cb_bytes + b->read_cb_off[r], b->read_cb_len[r]);
            if (cell < 0) { J->met.num_not_cell_bc++; continue; }                  /* main.rs:867-876 */
            if (J->use_umi && b->read_umi_key[r] == VTXO_NO_UMI) { J->met.num_non_umi++; continue; }  /* 879-888 */
            uint32_t m = b->read_len[r];
            if (m > qcap) { qcap = m; seq = (uint8_t*)realloc(seq, qcap); }
            vtxo_decode_read(b->read_nib + b->read_off[r], (int32_t)m, seq);                          /* 896 */
            if (n == scap) { scap *= 2; sc = (score_t*)realloc(sc, scap * sizeof(score_t)); }
            sc[n].cell = (uint32_t)cell; sc[n].ord = (uint32_t)n;
            sc[n].umi = J->use_umi ? b->read_umi_key[r] : 1;                                            /* 890-891 */
            if (J->band) {
                sc[n].rs = vtxo_sw_band_model(seq, (int32_t)m, rh, nr, 6, 20);
                sc[n].as = vtxo_sw_band_model(seq, (int32_t)m, ah, na, 6, 20);
            } else {
                sc[n].rs = vtxo_sw_full(seq, (int32_t)m, rh, nr);                                       /* 900 */
                sc[n].as = vtxo_sw_full(seq, (int32_t)m, ah, na);                                       /* 901 */
            }
            ++n; J->met.num_scored++;
        }
        aggregate_locus(sc, n, b->locus_row[l], J->mode, J->use_umi, J->min_score, &J->out);
    }
    free(sc); free(seq);
}

/* the rayon pool of main.rs:279-291: n_threads workers pull chunks until none are left */
typedef struct { rb_job* jobs; uint32_t n_chunks; uint32_t* next; } rb_pool;

static void* rb_worker(void* arg)
{
    rb_pool* P = (rb_pool*)arg;
    for (;;) {
        uint32_t c = __atomic_fetch_add(P->next, 1u, __ATOMIC_RELAXED);
        if (c >= P->n_chunks) break;
        rb_chunk(&P->jobs[c]);
    }
    return NULL;
}

int32_t vtxo_run_batch(const vtxo_batch* b,
                       const uint8_t* bc_bytes, const uint32_t* bc_off, uint32_t n_barcodes,
                       int32_t mode, int32_t use_umi, int32_t n_threads, int32_t use_band_model,
                       int32_t min_score, vtxo_result* out)
{
    memset(out, 0, sizeof(*out));
    bcmap_t bc; bcmap_build(&bc, bc_bytes, bc_off, n_barcodes);
    if (n_threads < 1) n_threads = 1;
    /* static contiguous chunks of max(n / threads, 1) loci -- main.rs:250-254 (may give threads+1 chunks) */
    uint32_t n = b->n_loci;
    uint32_t chunk = n / (uint32_t)n_threads; if (chunk < 1) chunk = 1;
    uint32_t n_chunks = n ? (n + chunk - 1) / chunk : 0;
    rb_job* jobs = (rb_job*)calloc(n_chunks ? n_chunks : 1, sizeof(rb_job));
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (n_chunks ? n_chunks : 1));
    for (uint32_t c = 0; c < n_chunks; ++c) {
        jobs[c].b = b; jobs[c].bc = &bc; jobs[c].lo = c * chunk; jobs[c].hi = imin((int32_t)(c * chunk + chunk), (int32_t)n);
        jobs[c].mode = mode; jobs[c].use_umi = use_umi; jobs[c].band = use_band_model; jobs[c].min_score = min_score;
    }
    uint32_t next = 0; rb_pool pool = { jobs, n_chunks, &next };
    uint32_t nt = (uint32_t)n_threads < n_chunks ? (uint32_t)n_threads : n_chunks;
    for (uint32_t t = 0; t < nt; ++t) pthread_create(&th[t], NULL, rb_worker, &pool);
    for (uint32_t t = 0; t < nt; ++t) pthread_join(th[t], NULL);
    size_t total = 0;
    for (uint32_t c = 0; c < n_chunks; ++c) total += jobs[c].out.n;
    out->n = total;
    size_t al = total ? total : 1;
    out->row = (uint32_t*)malloc(al * 4); out->col = (uint32_t*)malloc(al * 4);
    out->ref_cnt = (uint32_t*)malloc(al * 4); out->alt_cnt = (uint32_t*)malloc(al * 4); out->unk_cnt = (uint32_t*)malloc(al * 4);
    out->val = (double*)malloc(al * 8); out->val2 = (double*)malloc(al * 8);
    size_t k = 0;
    for (uint32_t c = 0; c < n_chunks; ++c) {                 /* serial merge in row order, main.rs:320-348 */
        for (size_t i = 0; i < jobs[c].out.n; ++i, ++k) {
            entry_t* e = &jobs[c].out.e[i];
            out->row[k] = e->row; out->col[k] = e->col; out->ref_cnt[k] = e->r; out->alt_cnt[k] = e->a;
            out->unk_cnt[k] = e->u; out->val[k] = e->v; out->val2[k] = e->v2;
        }
        out->metrics.num_not_cell_bc += jobs[c].met.num_not_cell_bc;
        out->metrics.num_non_umi += jobs[c].met.num_non_umi;
        out->metrics.num_scored += jobs[c].met.num_scored;
        free(jobs[c].out.e);
    }
    free(jobs); free(th); free(bc.slot);
    return 0;
}

void vtxo_free_result(vtxo_result* r)
{
    free(r->row); free(r->col); free(r->ref_cnt); free(r->alt_cnt); free(r->unk_cnt); free(r->val); free(r->val2);
    memset(r, 0, sizeof(*r));
}
