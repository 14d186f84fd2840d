// vartrix_b200 CLI -- keeps the `vartrix` flag surface (vartrix src/main.rs:40-135) and the
// `_main` flow (main.rs:163-418): inputs are decoded and filtered on host threads (stager.hpp), every shard
// of loci is handed to the GPU engine through the C ABI (include/vartrix_b200.h), outputs are the same
// Matrix-Market / label files.  `--dump-staged` stops after staging (no GPU needed; used by the tests).
#include <atomic>
#include <condition_variable>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <malloc.h>
#include <unistd.h>
#include <array>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <sys/stat.h>
#include <chrono>
#include <future>
#include <thread>

#include "stager.hpp"
#include "../vtx_donors.cuh"

using namespace vtxhost;

namespace {

int g_log = 0;      // 0 error, 1 info, 2 debug   (--log-level, main.rs:102-106)
void logf(int level, const char* tag, const char* fmt, ...)
{
    if (level > g_log) return;
    va_list ap; va_start(ap, fmt);
    fprintf(stderr, "[%s] ", tag); vfprintf(stderr, fmt, ap); fputc('\n', stderr);
    va_end(ap);
}
#define LOG_ERR(...) logf(0, "ERROR", __VA_ARGS__)
#define LOG_INFO(...) logf(1, "INFO", __VA_ARGS__)

double now_s()
{
    static const auto t0 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

bool exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0; }

struct Opts {
    std::string vcf, bam, fasta, barcodes, out_matrix = "out_matrix.mtx", ref_matrix = "ref_matrix.mtx", out_variants, out_barcodes;
    std::string scoring = "consensus", bam_tag = "CB", valid_chars = "ATGCatgc", dump_staged, out_variant_stats;
    std::string out_donors, donors;            // --out-donors FILE, --donors NAME,NAME,...
    double donor_error_rate = 0.01;            // --donor-error-rate
    bool donor_error_rate_given = false;
    long padding = 100, threads = 1, mapq = 0, device = 0, shard_loci = 0;      // 0: chosen from the number of loci and threads
    long shard_bytes = 0;       // compressed BAM bytes a shard may span (0: no limit; 192 MB under --gpu-stage)
    uint32_t min_base_quality = 0;     // --min-base-quality (0: off)
    std::vector<int> devices;          // --devices: the loci are sharded over these GPUs (contiguous ranges, main.rs:250-254)
    bool primary = false, no_dups = false, umi = false, collapse_mates = false, ref_matrix_given = false, gpu_inflate = false, gpu_stage = false, cut_at_contigs = false;
};

void usage()
{
    puts("vartrix_b200 -- Variant assignment for single cell genomics (H100-native engine)\n"
         "USAGE: vartrix_b200 --vcf FILE --bam FILE --fasta FILE --cell-barcodes FILE [OPTIONS]\n"
         "  -v, --vcf FILE              Called variant file (VCF)\n"
         "  -b, --bam FILE              Cellranger BAM file\n"
         "  -f, --fasta FILE            Genome fasta file\n"
         "  -c, --cell-barcodes FILE    File with cell barcodes to be evaluated\n"
         "  -o, --out-matrix FILE       Output Matrix Market file [out_matrix.mtx]\n"
         "      --out-variants FILE     Output variant file\n"
         "      --out-barcodes FILE     Output cell barcode file\n"
         "      --out-variant-stats FILE  Per-variant summary table (TSV, one line per VCF record in matrix-row order): the\n"
         "                              reads fetched, dropped by each filter and scored, their calls and the cells covered\n"
         "      --out-donors FILE       Assign each cell to a donor of the VCF's genotypes (TSV, one line per barcode): singlet and\n"
         "                              doublet log-likelihoods from the cell's REF / ALT counts, the best pair and the call\n"
         "      --donors LIST           The VCF samples that are the pool's donors, e.g. S1,S4,S2 (2 to 32) [every sample]\n"
         "      --donor-error-rate E    Per-molecule error rate of the donor model, 1e-6 .. 0.25 [0.01]\n"
         "  -p, --padding INT           Padding on both sides of the variant [100]\n"
         "  -s, --scoring-method M      consensus | coverage | alt_frac [consensus]\n"
         "      --ref-matrix FILE       Reference matrix (coverage mode) [ref_matrix.mtx]\n"
         "      --log-level L           info | debug | error [error]\n"
         "      --threads INT           Host staging threads [1]\n"
         "      --mapq INT              Minimum mapping quality [0]\n"
         "      --primary-alignments    Use primary alignments only\n"
         "      --no-duplicates         Do not consider duplicate alignments\n"
         "      --umi                   Consider UMI information\n"
         "      --collapse-mates        Count each paired-end fragment once per cell: the records of one QNAME at a locus are\n"
         "                              collapsed like the reads of one UMI (not with --umi, which already collapses mates)\n"
         "      --min-base-quality INT  Skip a read at a variant when a base it has there (aligned to the REF span, or\n"
         "                              inserted right after it) has a base quality below INT, 0..93 [0: off]\n"
         "      --bam-tag TAG           BAM tag marking cells [CB]\n"
         "      --valid-chars CHARS     Valid characters in an alternative haplotype [ATGCatgc]\n"
         "      --device INT            CUDA device ordinal [0]\n"
         "      --devices LIST          Shard the loci over several GPUs: e.g. 0-7 or 0,2,5 (one NCCL gather at the end)\n"
         "      --shard-loci INT        VCF records per staged shard [up to 2048, fewer for short VCFs]\n"
         "      --gpu-stage             Decode the BAM on the GPU: the host only reads the compressed ranges the loci's index chunks\n"
         "                              span; inflate, record scan, fetch, record filters and tag extraction run on the device\n"
         "      --shard-bytes INT       End a staged shard when the BAM it spans exceeds INT compressed bytes [192 MB with --gpu-stage]\n"
         "      --cut-at-contigs        End a staged shard where the contig changes (implied by --gpu-stage)\n"
         "      --gpu-inflate           Inflate the BGZF members of every shard on the GPU (one call per shard) instead of on\n"
         "                              the staging threads; for hosts with few cores per GPU\n"
         "      --dump-staged FILE      Stage only, write the shards to FILE (no GPU)");
}

// "0-3", "0,2,5", "1": CUDA device ordinals, no duplicates
bool parse_devices(const std::string& spec, std::vector<int>* out)
{
    out->clear();
    size_t p = 0;
    while (p <= spec.size()) {
        size_t q = spec.find(',', p);
        if (q == std::string::npos) q = spec.size();
        const std::string tok = spec.substr(p, q - p);
        if (tok.empty()) return false;
        const size_t dash = tok.find('-');
        char* end = nullptr;
        const long a = strtol(tok.c_str(), &end, 10);
        long b = a;
        if (dash != std::string::npos) { if (end != tok.c_str() + dash) return false; b = strtol(tok.c_str() + dash + 1, &end, 10); }
        if (*end != 0 || a < 0 || b < a || b > 1023) return false;
        for (long d = a; d <= b; ++d) { if (std::find(out->begin(), out->end(), int(d)) != out->end()) return false; out->push_back(int(d)); }
        p = q + 1;
    }
    return !out->empty();
}

bool parse(int argc, char** argv, Opts* o)
{
    auto need = [&](int& i) -> const char* { if (i + 1 >= argc) { fprintf(stderr, "error: %s needs a value\n", argv[i]); exit(1); } return argv[++i]; };
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        std::string val; bool has_eq = false;
        if (a.rfind("--", 0) == 0) { size_t e = a.find('='); if (e != std::string::npos) { val = a.substr(e + 1); a = a.substr(0, e); has_eq = true; } }
        auto v = [&]() -> std::string { return has_eq ? val : std::string(need(i)); };
        if (a == "-v" || a == "--vcf") o->vcf = v();
        else if (a == "-b" || a == "--bam") o->bam = v();
        else if (a == "-f" || a == "--fasta") o->fasta = v();
        else if (a == "-c" || a == "--cell-barcodes") o->barcodes = v();
        else if (a == "-o" || a == "--out-matrix") o->out_matrix = v();
        else if (a == "--out-variants") o->out_variants = v();
        else if (a == "--out-barcodes") o->out_barcodes = v();
        else if (a == "--out-variant-stats") o->out_variant_stats = v();
        else if (a == "--out-donors") o->out_donors = v();
        else if (a == "--donors") o->donors = v();
        else if (a == "--donor-error-rate") {
            const std::string e = v();
            char* end = nullptr;
            const double x = strtod(e.c_str(), &end);
            if (e.empty() || *end != 0 || !(x >= 1e-6 && x <= 0.25)) {
                fprintf(stderr, "error: --donor-error-rate must be a number from 1e-6 to 0.25, not '%s'\n", e.c_str());
                return false;
            }
            o->donor_error_rate = x;
            o->donor_error_rate_given = true;
        }
        else if (a == "-p" || a == "--padding") o->padding = atol(v().c_str());
        else if (a == "-s" || a == "--scoring-method") o->scoring = v();
        else if (a == "--ref-matrix") { o->ref_matrix = v(); o->ref_matrix_given = true; }
        else if (a == "--log-level") { std::string l = v(); if (l == "info") g_log = 1; else if (l == "debug") g_log = 2; else if (l == "error") g_log = 0; else { puts("Log level not valid"); exit(1); } }
        else if (a == "--threads") o->threads = atol(v().c_str());
        else if (a == "--mapq") o->mapq = atol(v().c_str());
        else if (a == "--primary-alignments") o->primary = true;
        else if (a == "--no-duplicates") o->no_dups = true;
        else if (a == "--umi") o->umi = true;
        else if (a == "--collapse-mates") o->collapse_mates = true;
        else if (a == "--min-base-quality") {
            const std::string q = v();
            char* end = nullptr;
            const long n = strtol(q.c_str(), &end, 10);
            if (q.empty() || *end != 0 || n < 0 || n > long(vtx::stage::kMaxBaseQuality)) {
                fprintf(stderr, "error: --min-base-quality must be an integer from 0 to %u, not '%s'\n", vtx::stage::kMaxBaseQuality, q.c_str());
                return false;
            }
            o->min_base_quality = uint32_t(n);
        }
        else if (a == "--bam-tag") o->bam_tag = v();
        else if (a == "--valid-chars") o->valid_chars = v();
        else if (a == "--device") o->device = atol(v().c_str());
        else if (a == "--devices") { if (!parse_devices(v(), &o->devices)) { fprintf(stderr, "error: bad --devices list\n"); return false; } }
        else if (a == "--shard-loci") o->shard_loci = atol(v().c_str());
        else if (a == "--shard-bytes") o->shard_bytes = std::max(0l, atol(v().c_str()));
        else if (a == "--dump-staged") o->dump_staged = v();
        else if (a == "--gpu-inflate") o->gpu_inflate = true;
        else if (a == "--gpu-stage") { o->gpu_stage = true; o->cut_at_contigs = true; }
        else if (a == "--cut-at-contigs") o->cut_at_contigs = true;
        else if (a == "-h" || a == "--help") { usage(); exit(0); }
        else if (a == "-V" || a == "--version") { puts("vartrix_b200 0.1 (vartrix 1.1.22 surface)"); exit(0); }
        else { fprintf(stderr, "error: unknown argument %s\n", argv[i]); return false; }
    }
    if (o->vcf.empty() || o->bam.empty() || o->fasta.empty() || o->barcodes.empty()) { fprintf(stderr, "error: --vcf, --bam, --fasta and --cell-barcodes are required\n"); return false; }
    if (o->scoring != "consensus" && o->scoring != "coverage" && o->scoring != "alt_frac") { fprintf(stderr, "error: invalid --scoring-method\n"); return false; }
    if (o->bam_tag.size() != 2) { fprintf(stderr, "error: --bam-tag must have two characters\n"); return false; }
    if (o->umi && o->collapse_mates) {
        fprintf(stderr, "error: --collapse-mates cannot be combined with --umi (mates share their UB tag, so --umi already counts a fragment once)\n");
        return false;
    }
    if (!o->out_variant_stats.empty() && !o->dump_staged.empty()) {
        fprintf(stderr, "error: --out-variant-stats counts what the GPU run scores: it cannot be combined with --dump-staged\n");
        return false;
    }
    if (!o->out_donors.empty() && !o->dump_staged.empty()) {
        fprintf(stderr, "error: --out-donors sums what the GPU run counts: it cannot be combined with --dump-staged\n");
        return false;
    }
    if (o->out_donors.empty() && (!o->donors.empty() || o->donor_error_rate_given)) {
        fprintf(stderr, "error: --donors and --donor-error-rate only apply with --out-donors\n");
        return false;
    }
    if (o->threads < 1) o->threads = 1;
    if (o->shard_loci < 0) o->shard_loci = 0;
    if (o->devices.empty()) o->devices.push_back(int(o->device));
    return true;
}

// validate_output_path (main.rs:475-491): refuse to overwrite, parent directory must exist
void validate_output_path(const std::string& p)
{
    if (exists(p)) { LOG_ERR("Output path already exists"); exit(1); }
    size_t s = p.find_last_of('/');
    if (s != std::string::npos && s > 0 && !exists(p.substr(0, s))) { LOG_ERR("Output directory \"%s\" does not exist", p.substr(0, s).c_str()); exit(1); }
}

// check_inputs_exist (main.rs:493-542)
void check_inputs_exist(const Opts& o)
{
    for (const std::string* p : { &o.fasta, &o.vcf, &o.bam, &o.barcodes })
        if (!exists(*p)) { LOG_ERR("Input file %s does not exist", p->c_str()); exit(1); }
    if (o.dump_staged.empty()) { validate_output_path(o.out_matrix); validate_output_path(o.ref_matrix); }
    if (!o.out_variant_stats.empty()) validate_output_path(o.out_variant_stats);
    if (!o.out_donors.empty()) validate_output_path(o.out_donors);
    if (!exists(o.fasta + ".fai")) { LOG_ERR("File %s.fai does not exist", o.fasta.c_str()); exit(1); }
    const size_t dot = o.bam.find_last_of('.');
    const std::string ext = dot == std::string::npos ? "" : o.bam.substr(dot + 1);
    if (ext == "bam") {
        const bool bai = exists(o.bam + ".bai") || exists(o.bam.substr(0, dot) + ".bai");
        if (!bai && exists(o.bam + ".csi")) { LOG_ERR("%s.csi: CSI indices are not supported by this build (no htslib); create a BAI index (samtools index -b)", o.bam.c_str()); exit(1); }
        if (!bai) { LOG_ERR("BAM index does not exist. Expecting %s.bai", o.bam.c_str()); exit(1); }
    } else if (ext == "cram") {
        LOG_ERR("CRAM input is not supported by this build (no htslib); convert to BAM"); exit(1);
    } else { LOG_ERR("BAM file did not end in .bam or .cram. Unable to validate"); exit(1); }
}

// --dump-staged writes the shard in the vtx_batch layout (16-byte aligned reads, tag bytes per read) that the staging
// tests compare with the oracle's decode; the codes are turned back into the tag bytes they stand for.
void dump_shard(FILE* f, const StagedShard& s)
{
    auto put = [&](const void* p, size_t bytes) { uint64_t n = bytes; fwrite(&n, 8, 1, f); if (bytes) fwrite(p, 1, bytes, f); };
#define PUTV(v) put((v).data(), (v).size() * sizeof((v)[0]))
    const size_t nr = s.read_len.size();
    std::vector<uint8_t> nib, cb;
    std::vector<uint64_t> read_off(nr), umi(nr, VTX_NO_UMI);
    std::vector<uint32_t> read_len(nr), cb_off(nr);
    std::vector<uint16_t> cb_len(nr);
    size_t src = 0;
    for (size_t r = 0; r < nr; ++r) {
        const size_t nb = (size_t(s.read_len[r]) + 1) / 2;
        while (nib.size() & 15) nib.push_back(0);
        read_off[r] = nib.size(); read_len[r] = s.read_len[r];
        nib.insert(nib.end(), s.read_nib.begin() + src, s.read_nib.begin() + src + nb);
        src += (nb + 3) / 4 * 4;
        const uint64_t k = s.read_cb_key[r];
        if (k == VTX_NO_CB_KEY) { cb_off[r] = VTX_NO_CB; cb_len[r] = 0; continue; }
        cb_off[r] = uint32_t(cb.size());
        if (k & VTX_CB_EXOTIC) { const uint32_t i = uint32_t(k & 0xFFFFFFFFu); cb.insert(cb.end(), s.cb_bytes.begin() + s.cb_off[i], s.cb_bytes.begin() + s.cb_off[i + 1]); }
        else { const std::string t = unpack_cb(k); cb.insert(cb.end(), t.begin(), t.end()); }
        cb_len[r] = uint16_t(cb.size() - cb_off[r]);
    }
    while (nib.size() & 15) nib.push_back(0);
    if (s.with_umi) umi = s.read_umi_key;
    fwrite("VTXS", 1, 4, f);
    PUTV(s.locus_row); PUTV(s.hap_bytes); PUTV(s.ref_off); PUTV(s.ref_len); PUTV(s.alt_off); PUTV(s.alt_len); PUTV(s.cand_start);
    PUTV(nib); PUTV(read_off); PUTV(read_len); PUTV(cb); PUTV(cb_off); PUTV(cb_len); PUTV(umi); PUTV(s.cand_read);
#undef PUTV
    uint64_t m[7] = { s.met.num_reads, s.met.num_low_mapq, s.met.num_non_primary, s.met.num_duplicates, s.met.num_not_useful,
                      s.met.num_invalid_recs, s.met.num_multiallelic_recs };
    fwrite(m, 8, 7, f);
}

// pinned arena holding one shard for the asynchronous copy
struct Arena {
    uint8_t* base = nullptr; size_t cap = 0;
    bool ensure(size_t bytes)
    {
        if (bytes <= cap) return true;
        if (base) vtx_host_free(base);
        void* p = nullptr;
        if (vtx_host_alloc(&p, bytes + bytes / 4) != VTX_OK) { base = nullptr; cap = 0; return false; }
        base = static_cast<uint8_t*>(p); cap = bytes + bytes / 4;
        return true;
    }
    ~Arena() { if (base) vtx_host_free(base); }
};

// Copies the shard's arrays into the pinned arena.  This runs on the submitting thread while up to `--threads` workers
// stage; with many workers a single memcpy stream (~10 GB/s) would cap the whole pipeline near 70 M reads/s, so shards
// above a few megabytes are copied in 4 MB pieces by the caller plus up to three helper threads.
void stage_into_arena(const StagedShard& s, Arena& a, vtx_batch2* b)
{
    struct Job { uint8_t* dst; const uint8_t* src; size_t bytes; };
    std::vector<Job> jobs;
    size_t off = 0, total = 0;
    auto put = [&](const void* p, size_t bytes) -> const void* {
        off = (off + 15) & ~size_t(15);
        uint8_t* d = a.base + off;
        constexpr size_t kPiece = size_t(4) << 20;
        for (size_t o = 0; o < bytes; o += kPiece) jobs.push_back({ d + o, static_cast<const uint8_t*>(p) + o, std::min(kPiece, bytes - o) });
        off += bytes; total += bytes;
        return d;
    };
    s.fill(b);
#define MV(field, vec) b->field = static_cast<decltype(b->field)>(put((vec).data(), (vec).size() * sizeof((vec)[0])))
    MV(locus_row, s.locus_row); MV(hap_bytes, s.hap_bytes); MV(ref_off, s.ref_off); MV(ref_len, s.ref_len); MV(alt_off, s.alt_off);
    MV(alt_len, s.alt_len); MV(cand_start, s.cand_start); MV(read_nib, s.read_nib); MV(read_len, s.read_len); MV(read_cb_key, s.read_cb_key);
    if (b->n_exotic_cb) { MV(cb_bytes, s.cb_bytes); MV(cb_off, s.cb_off); } else { b->cb_bytes = nullptr; b->cb_off = nullptr; }
    if (s.with_umi) MV(read_umi_key, s.read_umi_key);
    if (!s.identity) MV(cand_read, s.cand_read);
#undef MV
    std::atomic<size_t> next{ 0 };
    auto run = [&]() {
        for (size_t j; (j = next.fetch_add(1)) < jobs.size();) memcpy(jobs[j].dst, jobs[j].src, jobs[j].bytes);
    };
    const size_t helpers = total >= (size_t(8) << 20) ? std::min<size_t>(3, jobs.size() - 1) : 0;
    std::vector<std::thread> pool;
    for (size_t t = 0; t < helpers; ++t) pool.emplace_back(run);
    run();
    for (auto& t : pool) t.join();
}

// --out-variant-stats: one line per VCF record, in matrix-row order.  `dev` holds the engine's entries of every submitted locus
// (each row at most once over all lanes); `host_rows` / `host_filters` the stager's record-filter counters of the host-staged
// loci, which the engine leaves 0.  Records the host never submits are multi-allelic or have an invalid ALT haplotype.
// vtx_locus_stats is 22 u32 counters in declaration order: the writer handles an entry as that array (a copy, not a cast)
constexpr int kStatsWords = 22;
static_assert(sizeof(vtx_locus_stats) == kStatsWords * sizeof(uint32_t), "vtx_locus_stats: 22 counters, no padding");
static_assert(offsetof(vtx_locus_stats, fetched) == 1 * 4 && offsetof(vtx_locus_stats, low_base_quality) == (1 + vtx::stage::kLowBaseQuality) * 4 &&
              offsetof(vtx_locus_stats, scored) == 9 * 4 && offsetof(vtx_locus_stats, cells_multi_unknown) == 21 * 4,
              "vtx_locus_stats field order");
using StatsWords = std::array<uint32_t, kStatsWords>;      // [0] row, [1..6] fetched .. low_base_quality, [7..21] the rest

bool write_variant_stats(const std::string& path, const std::vector<VcfRecord>& recs, const std::vector<vtx_locus_stats>& dev,
                         const std::vector<uint32_t>& host_rows, const std::vector<uint32_t>& host_filters)
{
    std::vector<StatsWords> row(recs.size(), StatsWords{});
    std::vector<char> submitted(recs.size(), 0);
    for (const vtx_locus_stats& e : dev) {
        if (e.row >= recs.size()) return false;
        memcpy(row[e.row].data(), &e, sizeof(e));
        submitted[e.row] = 1;
    }
    for (size_t i = 0; i < host_rows.size(); ++i)
        for (int k = 0; k < vtx::stage::kNumCounters; ++k)      // the stager's record counters, in the columns fetched .. low_base_quality
            row[host_rows[i]][1 + k] += host_filters[i * vtx::stage::kNumCounters + k];
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    fputs("variant\tchrom\tpos\tref\talt\tstatus\tfetched\tlow_mapq\tnon_primary\tduplicate\tnot_useful\tlow_base_quality\t"
          "no_cell_barcode\tno_umi\tscored\treads_ref\treads_alt\treads_unknown\treads_none\tcalls_ref\tcalls_alt\tcalls_unknown\t"
          "cells\tcells_ref_only\tcells_alt_only\tcells_both\tcells_multi_unknown\n", f);
    for (size_t r = 0; r < recs.size(); ++r) {
        const VcfRecord& v = recs[r];
        std::string alt;
        for (size_t k = 1; k < v.alleles.size(); ++k) { if (k > 1) alt += ','; alt += v.alleles[k]; }
        if (v.alleles.size() == 1) alt = ".";
        const char* status = v.alleles.size() > 2 ? "multiallelic" : submitted[r] ? "scored" : "invalid_alt";     // main.rs:646-653, 675-684
        fprintf(f, "%s_%lld\t%s\t%lld\t%s\t%s\t%s", v.chrom.c_str(), (long long)v.pos0, v.chrom.c_str(), (long long)v.pos0 + 1,
                v.alleles[0].c_str(), alt.c_str(), status);
        for (int k = 1; k < kStatsWords; ++k) fprintf(f, "\t%u", row[r][k]);
        fputc('\n', f);
    }
    return fclose(f) == 0;
}

// --out-donors: the selected VCF samples, in --donors order (header order without it), and their dosage table (one row per
// VCF record = matrix row)
struct DonorTable {
    std::vector<std::string> names;
    std::vector<uint8_t> dosage;        // [record][donor]: 0..2 or kGtMissing
    uint64_t usable = 0;                // biallelic rows where every donor has a dosage
};

bool select_donors(const std::string& list, const VcfGenotypes& g, const std::vector<VcfRecord>& recs, DonorTable* t, std::string* err)
{
    std::vector<size_t> idx;
    if (list.empty()) {
        for (size_t i = 0; i < g.samples.size(); ++i) idx.push_back(i);
    } else {
        for (size_t p = 0; p <= list.size();) {
            size_t q = list.find(',', p);
            if (q == std::string::npos) q = list.size();
            const std::string name = list.substr(p, q - p);
            const auto it = std::find(g.samples.begin(), g.samples.end(), name);
            if (it == g.samples.end()) { *err = "--donors: '" + name + "' is not a sample column of the VCF"; return false; }
            const size_t i = size_t(it - g.samples.begin());
            if (std::find(idx.begin(), idx.end(), i) != idx.end()) { *err = "--donors: '" + name + "' is listed twice"; return false; }
            idx.push_back(i);
            p = q + 1;
        }
    }
    if (idx.size() < vtx::donors::kMinDonors || idx.size() > vtx::donors::kMaxDonors) {
        *err = "--out-donors needs 2 to 32 donors, not " + std::to_string(idx.size()) +
               (list.empty() ? " (the VCF's sample columns; choose some with --donors)" : "");
        return false;
    }
    const size_t ns = g.samples.size(), nd = idx.size();
    for (const size_t i : idx) t->names.push_back(g.samples[i]);
    t->dosage.resize(recs.size() * nd);
    for (size_t r = 0; r < recs.size(); ++r) {
        bool all = true;
        for (size_t d = 0; d < nd; ++d) {
            t->dosage[r * nd + d] = g.dosage[r * ns + idx[d]];
            all = all && t->dosage[r * nd + d] != kGtMissing;
        }
        t->usable += all && recs[r].alleles.size() <= 2;
    }
    return true;
}

// The donor file: one line per barcode in column order.  ll [col][H] and cnt [col][3] are the engine's sums over every lane.
// The calls use the fixed threshold T = 5 nats, compared in the integer scale.
bool write_donors(const std::string& path, const std::vector<std::string>& barcodes, const std::vector<std::string>& names,
                  const std::vector<int64_t>& ll, const std::vector<uint64_t>& cnt, uint64_t calls[3])
{
    using namespace vtx::donors;
    const uint32_t D = uint32_t(names.size()), H = n_hyp(D);
    const int64_t T = 5 * int64_t(kScale);
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    fputs("barcode\tvariants\tref\talt\tcall\tassignment\tsinglet_llr\tdoublet_llr\tbest_singlet\tsecond_singlet\tbest_doublet", f);
    for (const std::string& n : names) fprintf(f, "\tll_%s", n.c_str());
    fputc('\n', f);
    auto pair_name = [&](uint32_t h) { uint32_t a, b; hyp_donors(h, D, &a, &b); return names[a] + "+" + names[b]; };
    for (size_t c = 0; c < barcodes.size(); ++c) {
        const int64_t* L = ll.data() + c * H;
        const uint64_t* n = cnt.data() + c * 3;
        uint32_t best = 0, pair = D;
        for (uint32_t h = 1; h < D; ++h) if (L[h] > L[best]) best = h;
        uint32_t second = best == 0 ? 1 : 0;            // ties go to the lowest index: strictly larger replaces
        for (uint32_t h = second + 1; h < D; ++h) if (h != best && L[h] > L[second]) second = h;
        for (uint32_t h = D + 1; h < H; ++h) if (L[h] > L[pair]) pair = h;
        const int64_t s_llr = L[best] - L[second], d_llr = L[pair] - L[best];
        const int call = n[0] == 0 ? 2 : d_llr >= T ? 1 : s_llr >= T ? 0 : 2;        // singlet, doublet, unassigned
        ++calls[call];
        const std::string assignment = call == 0 ? names[best] : call == 1 ? pair_name(pair) : ".";
        fprintf(f, "%s\t%llu\t%llu\t%llu\t%s\t%s\t%.6f\t%.6f\t%s\t%s\t%s", barcodes[c].c_str(), (unsigned long long)n[0],
                (unsigned long long)n[1], (unsigned long long)n[2], call == 0 ? "singlet" : call == 1 ? "doublet" : "unassigned",
                assignment.c_str(), double(s_llr) / kScale, double(d_llr) / kScale, names[best].c_str(), names[second].c_str(),
                pair_name(pair).c_str());
        for (uint32_t d = 0; d < D; ++d) fprintf(f, "\t%.6f", double(L[d]) / kScale);
        fputc('\n', f);
    }
    return fclose(f) == 0;
}

}  // namespace

// One GPU of the run: its own engine context, a contiguous range of shards, a thread that feeds it in order.
struct Lane {
    int device = 0, rank = 0;
    size_t lo = 0, hi = 0;              // shard index range [lo, hi)
    vtx_ctx* ctx = nullptr;
    size_t consumed = 0;                // shards of this lane handed to the engine so far (guarded by the staging mutex)
    Arena arenas[3];
    HostMetrics hm;
    std::string err;
    int rc = 0;
    vtx_result dev{};                   // this lane's triplets on its device
    double ready_s = 0, wait_s = 0, submit_s = 0;      // engine up at; consumer: waiting for staged shards / inside submit calls
    Fasta fb_fa; BamFile fb_bam; bool fb_open = false; size_t host_fallbacks = 0;    // --gpu-stage: shards the device sent back
    std::vector<vtx_locus_stats> stats;                 // --out-variant-stats: the engine's entries after this lane's finish
    std::vector<uint32_t> host_rows, host_filters;      // ... and the stager's filter counters of the loci staged on the host
    std::vector<int64_t> donor_ll;                      // --out-donors: this lane's sums after its finish
    std::vector<uint64_t> donor_cnt;
};

int main(int argc, char** argv)
{
    // staging grows multi-megabyte vectors on many threads: keep them on the heap arenas instead of
    // mmap/munmap per reallocation (which serialises the threads on the process address-space lock)
    mallopt(M_MMAP_THRESHOLD, 1 << 30);
    mallopt(M_TRIM_THRESHOLD, 1 << 30);
    Opts o;
    if (!parse(argc, argv, &o)) { usage(); return 1; }
    check_inputs_exist(o);
    std::string err;
    const bool dumping = !o.dump_staged.empty();

    // Only the requested GPUs become visible to CUDA (unless the caller already chose): on an 8-GPU host, initialising the
    // driver with all devices visible takes 6-7 s even for --device 0, with one visible ~1 s.  `cuda_index` is what CUDA calls
    // the device from here on; logs keep the user's numbering.
    std::vector<int> cuda_index(o.devices.begin(), o.devices.end());
    if (!dumping && !getenv("CUDA_VISIBLE_DEVICES")) {
        std::string vis;
        for (size_t d = 0; d < o.devices.size(); ++d) { vis += (d ? "," : "") + std::to_string(o.devices[d]); cuda_index[d] = int(d); }
        setenv("CUDA_VISIBLE_DEVICES", vis.c_str(), 1);
    }

    BarcodeList bcs;
    if (!load_barcodes(o.barcodes, &bcs, &err)) { LOG_ERR("%s", err.c_str()); return 1; }
    LOG_INFO("Loaded %zu barcodes", bcs.keys.size());

    // --out-donors: the VCF (with its sample columns) is read before any GPU work, so that a bad donor list is refused first
    std::vector<VcfRecord> recs;
    const bool with_donors = !o.out_donors.empty();
    DonorTable donors;
    if (with_donors) {
        VcfGenotypes gts;
        if (!read_vcf(o.vcf, &recs, &err, &gts)) { printf("Vartrix error.\nError: %s\n", err.c_str()); return 1; }
        if (!select_donors(o.donors, gts, recs, &donors, &err)) { fprintf(stderr, "error: %s\n", err.c_str()); return 1; }
    }

    // CUDA context creation takes ~1 s per device: start it now, in the background, while the VCF is parsed and the
    // first shards are staged.  With several devices every lane also joins the engine's NCCL communicator.
    const size_t n_dev = dumping ? 1 : o.devices.size();
    std::vector<Lane> lanes(n_dev);
    uint8_t nccl_id[128] = {};
    if (!dumping && n_dev > 1 && vtx_comm_unique_id(nccl_id) != VTX_OK) { printf("Vartrix error.\nError: %s\n", vtx_last_error(nullptr)); return 1; }
    std::vector<std::future<int>> engine_ready(n_dev);
    if (!dumping) {
        for (size_t d = 0; d < n_dev; ++d) {
            lanes[d].device = o.devices[d]; lanes[d].rank = int(d);
            engine_ready[d] = std::async(std::launch::async, [&, d]() -> int {
                Lane& ln = lanes[d];
                vtx_config cfg{};
                cfg.device = cuda_index[d];
                cfg.mode = o.scoring == "consensus" ? VTX_MODE_CONSENSUS : o.scoring == "coverage" ? VTX_MODE_COVERAGE : VTX_MODE_ALT_FRAC;
                cfg.flags = VTX_F_VALUES_ONLY;       // the writers need row, col and the matrix values only
                if (o.collapse_mates) cfg.flags |= VTX_F_NAME_KEYS;      // name keys through the UMI collapse
                cfg.use_umi = o.umi || o.collapse_mates; cfg.match = 1; cfg.mismatch = -5; cfg.gap_open = -5; cfg.gap_extend = -1; cfg.min_score = 25;
                cfg.band_k = 6; cfg.band_w = 20; cfg.band_mode = VTX_BAND_FULL;          // main.rs:33-34
                if (vtx_create(&cfg, &ln.ctx) != VTX_OK) { ln.err = vtx_last_error(nullptr); return 1; }
                if (o.min_base_quality && vtx_set_min_base_quality(ln.ctx, o.min_base_quality) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); return 1; }
                if (!o.out_variant_stats.empty() && vtx_set_locus_stats(ln.ctx, 1) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); return 1; }
                if (with_donors && vtx_set_donors(ln.ctx, uint32_t(donors.names.size()), recs.size(), donors.dosage.data(), o.donor_error_rate) != VTX_OK) {
                    ln.err = vtx_last_error(ln.ctx); return 1;
                }
                if (vtx_set_barcodes(ln.ctx, bcs.bytes.data(), bcs.off.data(), uint32_t(bcs.keys.size())) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); return 1; }
                if (n_dev > 1 && vtx_comm_init(ln.ctx, nccl_id, int32_t(d), int32_t(n_dev)) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); return 1; }
                ln.ready_s = now_s();
                return 0;
            });
        }
    }

    if (!with_donors && !read_vcf(o.vcf, &recs, &err)) { printf("Vartrix error.\nError: %s\n", err.c_str()); return 1; }
    if (recs.empty()) LOG_ERR("Warning! Zero variants found in input VCF. Output matrices will be by definition empty but will still be generated.");
    LOG_INFO("Initialized a %zu variants x %zu cell barcodes matrix", recs.size(), bcs.keys.size());
    LOG_INFO("[%.3f s] inputs parsed", now_s());

    // validate_inputs (main.rs:545-594): contigs present in FASTA and BAM, record end inside the contig
    Fasta fa0;
    if (!fa0.open(o.fasta, &err)) { LOG_ERR("%s", err.c_str()); return 1; }
    BamFile b0;
    if (!b0.open(o.bam, &err)) { printf("Vartrix error.\nError: error opening bam file: %s (%s)\n", o.bam.c_str(), err.c_str()); return 1; }
    for (const VcfRecord& r : recs) {
        if (!fa0.has(r.chrom)) { LOG_ERR("Sequence %s not seen in FASTA", r.chrom.c_str()); return 1; }
        if (b0.tid_of(r.chrom) < 0) { LOG_ERR("Sequence %s not seen in BAM", r.chrom.c_str()); return 1; }
        const int64_t end = r.pos0 + int64_t(r.alleles[0].size());
        if (end > fa0.length(r.chrom)) {
            LOG_ERR("Record %s:%lld has end position %lld, which is larger than the chromosome length (%lld). Does your FASTA match your VCF?",
                    r.chrom.c_str(), (long long)r.pos0, (long long)end, (long long)fa0.length(r.chrom));
            return 1;
        }
    }

    StageArgs sa;
    sa.padding = o.padding; sa.mapq_min = uint32_t(o.mapq); sa.primary_only = o.primary; sa.no_duplicates = o.no_dups;
    sa.bam_tag[0] = o.bam_tag[0]; sa.bam_tag[1] = o.bam_tag[1];
    sa.with_umi = o.umi || o.collapse_mates || dumping;      // without --umi the engine never looks at the UB keys: they are not staged
    sa.name_keys = o.collapse_mates;
    sa.min_base_quality = o.min_base_quality;
    sa.locus_filters = !o.out_variant_stats.empty();
    for (unsigned char c : o.valid_chars) sa.valid[c] = true;

    // ---- staging: worker threads produce shards of `shard_loci` records; one lane per GPU consumes its range in order ----
    // default shard size: 2048 loci (~100 k candidates at 50x, enough to fill the GPU), smaller when the VCF is short so that
    // every staging thread still gets ~10 shards (load balance; the GPU is idle most of the time anyway)
    // --gpu-stage: the host's share of a shard is small; what counts is the device's fixed cost per shard (three short waits,
    // ~30 launches) and the inflate kernel, which wants thousands of BGZF members per launch to fill the GPU (one warp each):
    // 8192 loci (~400 k reads, ~2 000 members at 50x), fewer only so that every GPU still gets a few shards to pipeline
    if (o.shard_loci == 0 && o.gpu_stage) o.shard_loci = long(std::min<size_t>(8192, std::max<size_t>(256, recs.size() / (o.devices.size() * 6 + 1))));
    if (o.shard_loci == 0) o.shard_loci = long(std::min<size_t>(2048, std::max<size_t>(128, recs.size() / (size_t(o.threads) * 10 + 1))));
    // shard k = records [shard_lo[k], shard_lo[k + 1]).  With --gpu-stage (or --cut-at-contigs) a shard also ends where the contig
    // changes, so that every shard of a sorted VCF can be staged on the device (one contig, ascending positions).
    // A device-staged shard is inflated into one stream (< 4 GiB, vtx_submit_bam) that lives twice in device memory: very deep
    // data must not put gigabytes into one shard, so a shard also ends when the BAM it spans (BAI linear index, compressed
    // bytes) exceeds --shard-bytes [192 MB under --gpu-stage: ~0.8 GB inflated at a BAM's usual ratio].
    if (o.shard_bytes == 0 && o.gpu_stage) o.shard_bytes = 192l << 20;
    std::vector<size_t> shard_lo;
    {
        uint64_t span_begin = 0;
        std::string span_chrom;
        int span_tid = -1;
        for (size_t i = 0, in_shard = 0; i < recs.size(); ++i, ++in_shard) {
            bool cut = i == 0 || in_shard == size_t(o.shard_loci) || (o.cut_at_contigs && recs[i].chrom != recs[i - 1].chrom);
            uint64_t here = 0;
            if (o.shard_bytes > 0) {
                if (recs[i].chrom != span_chrom) { span_chrom = recs[i].chrom; span_tid = b0.tid_of(span_chrom); cut = cut || o.cut_at_contigs; }
                here = b0.linear_offset(span_tid, recs[i].pos0);
                if (!cut && in_shard > 0 && here > span_begin && here - span_begin > uint64_t(o.shard_bytes)) cut = true;
            }
            if (cut) { shard_lo.push_back(i); in_shard = 0; span_begin = here; }
        }
    }
    const size_t n_shards = shard_lo.size();
    shard_lo.push_back(recs.size());

    // Loci -> GPUs: contiguous ranges like the reference's static chunks (main.rs:250-254), balanced by the compressed
    // bytes of BAM each shard spans (BAI linear index) -- a cheap stand-in for the candidate count, known before any decode.
    {
        std::vector<double> w(n_shards, 1.0);
        double total = 0;
        for (size_t k = 0; k < n_shards; ++k) {
            const VcfRecord& a = recs[shard_lo[k]];
            const VcfRecord& z = recs[shard_lo[k + 1] - 1];
            if (a.chrom == z.chrom) {
                const int tid = b0.tid_of(a.chrom);
                const uint64_t f0 = b0.linear_offset(tid, a.pos0), f1 = b0.linear_offset(tid, z.pos0 + int64_t(z.alleles[0].size()) + (1 << 14));
                if (f1 > f0) w[k] = double(f1 - f0);
            }
            total += w[k];
        }
        size_t k = 0;
        double acc = 0;
        for (size_t d = 0; d < n_dev; ++d) {
            lanes[d].lo = k;
            const double target = total * double(d + 1) / double(n_dev);
            while (k < n_shards && (d + 1 == n_dev || acc + w[k] * 0.5 <= target)) acc += w[k++];
            lanes[d].hi = k;
        }
        lanes[n_dev - 1].hi = n_shards;
    }
    // staging order: round robin over the lanes so that every GPU is fed from the start
    std::vector<size_t> order; order.reserve(n_shards);
    std::vector<size_t> lane_of(n_shards, 0);
    for (size_t i = 0, left = n_shards; left; ++i)
        for (size_t d = 0; d < n_dev; ++d)
            if (lanes[d].lo + i < lanes[d].hi) { order.push_back(lanes[d].lo + i); lane_of[lanes[d].lo + i] = d; --left; }

    std::vector<std::unique_ptr<StagedShard>> ready(n_shards);
    std::vector<std::unique_ptr<DeviceShard>> ready_dev(n_shards);         // --gpu-stage: the host's share of a device-staged shard
    const bool gpu_stage = o.gpu_stage;          // with --dump-staged: the host's share of device-staged shards is dumped ("VTXD")
    std::mutex mu; std::condition_variable cv;
    std::atomic<size_t> next{ 0 };
    const size_t window = std::max<size_t>(2, (size_t(o.threads) * 2 + 2 + n_dev - 1) / n_dev);
    bool failed = false; std::string fail_msg;
    UmiInterner umis;
    std::vector<std::unique_ptr<StagedShard>> recycled;      // guarded by mu
    std::atomic<uint64_t> stage_ns{ 0 }, arena_ns{ 0 }, staged_bytes{ 0 };
    std::atomic<int> worker_no{ 0 };
    auto worker = [&]() {
        Fasta fa; BamFile bam; std::string e;
        if (!fa.open(o.fasta, &e) || !bam.open(o.bam, &e)) { std::lock_guard<std::mutex> g(mu); failed = true; fail_msg = e; cv.notify_all(); return; }
        StageArgs sa_w = sa;
        vtx_ctx* ictx = nullptr;                 // --gpu-inflate: this worker's own context for vtx_bgzf_inflate
        std::vector<int32_t> istatus;
        if (o.gpu_inflate && dumping) {
            // --dump-staged never touches a GPU: the bulk path (one compressed range per shard, member walk, serving records out
            // of the bulk buffer) is exercised with the host decoder standing in for vtx_bgzf_inflate (CPU tests)
            sa_w.bulk_inflate = [](const vtx_bgzf_block* b, uint32_t n, const uint8_t* comp, uint64_t, uint8_t* out, uint64_t, std::string* err) {
                for (uint32_t i = 0; i < n; ++i) {
                    if (b[i].out_len && !vtx_inflate_raw(comp + b[i].in_off, b[i].in_len, out + b[i].out_off, b[i].out_len)) { *err = "member " + std::to_string(i) + ": inflate failed"; return false; }
                    if (vtx_crc::crc32_of(out + b[i].out_off, b[i].out_len) != b[i].crc32) { *err = "member " + std::to_string(i) + ": CRC32 mismatch"; return false; }
                }
                return true;
            };
        } else if (o.gpu_inflate) {
            vtx_config c{};
            c.device = cuda_index[size_t(worker_no.fetch_add(1)) % cuda_index.size()];
            c.mode = VTX_MODE_CONSENSUS; c.match = 1; c.mismatch = -5; c.gap_open = -5; c.gap_extend = -1; c.min_score = 25;
            if (vtx_create(&c, &ictx) != VTX_OK) { std::lock_guard<std::mutex> g(mu); failed = true; fail_msg = vtx_last_error(nullptr); cv.notify_all(); return; }
            bam.set_bulk_allocator([](void** q, size_t n) { return vtx_host_alloc(q, n) == VTX_OK; }, [](void* q) { vtx_host_free(q); });
            sa_w.bulk_inflate = [&istatus, ictx](const vtx_bgzf_block* b, uint32_t n, const uint8_t* comp, uint64_t comp_len, uint8_t* out, uint64_t out_len, std::string* err) {
                istatus.resize(n);
                if (vtx_bgzf_inflate(ictx, b, n, comp, comp_len, out, out_len, istatus.data(), VTX_BGZF_CHECK_CRC) == VTX_OK) return true;
                *err = vtx_last_error(ictx);
                return false;
            };
        }
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= n_shards) break;
            const size_t k = order[i];
            Lane& ln = lanes[lane_of[k]];
            { std::unique_lock<std::mutex> g(mu); cv.wait(g, [&] { return failed || k - ln.lo < ln.consumed + window; }); if (failed) return; }
            const size_t lo = shard_lo[k], hi = shard_lo[k + 1];
            if (gpu_stage) {
                auto ds = std::make_unique<DeviceShard>();
                bool supported = true;
                const uint64_t t_stage = StageClock::now();
                const bool ok = stage_loci_device(recs, lo, hi, fa, bam, sa_w, ds.get(), &supported, &e);
                stage_ns += StageClock::now() - t_stage;
                if (!ok) { std::lock_guard<std::mutex> g(mu); failed = true; fail_msg = e; cv.notify_all(); return; }
                if (supported) {
                    { std::lock_guard<std::mutex> g(mu); ready_dev[k] = std::move(ds); }
                    cv.notify_all();
                    continue;
                }
            }
            std::unique_ptr<StagedShard> sh;
            { std::lock_guard<std::mutex> g(mu); if (!recycled.empty()) { sh = std::move(recycled.back()); recycled.pop_back(); } }
            if (!sh) sh = std::make_unique<StagedShard>();
            const uint64_t t_stage = StageClock::now();
            const bool staged_ok = stage_loci(recs, lo, hi, fa, bam, sa_w, umis, sh.get(), &e);
            stage_ns += StageClock::now() - t_stage;
            if (!staged_ok) { std::lock_guard<std::mutex> g(mu); failed = true; fail_msg = e; cv.notify_all(); return; }
            { std::lock_guard<std::mutex> g(mu); ready[k] = std::move(sh); }
            cv.notify_all();
        }
    };

    FILE* dump = nullptr;
    if (dumping) {            // before the pool starts: an early return must not leave joinable threads behind
        dump = fopen(o.dump_staged.c_str(), "wb");
        if (!dump) { LOG_ERR("cannot write %s", o.dump_staged.c_str()); return 1; }
        uint64_t hdr[2] = { recs.size(), bcs.keys.size() };
        fwrite(hdr, 8, 2, dump);
    }
    std::vector<std::thread> pool;
    for (long t = 0; t < o.threads; ++t) pool.emplace_back(worker);

    // one consumer per lane: shards of its range, in order, into its engine (or into the dump file)
    auto take_stats = [&](Lane& ln) -> bool {          // --out-variant-stats: right after the lane's finish
        if (o.out_variant_stats.empty()) return true;
        const vtx_locus_stats* p = nullptr; uint64_t n = 0;
        if (vtx_locus_stats_get(ln.ctx, &p, &n) != VTX_OK) return false;
        ln.stats.assign(p, p + n);
        return true;
    };
    auto take_donors = [&](Lane& ln) -> bool {         // --out-donors: right after the lane's finish
        if (!with_donors) return true;
        const int64_t* ll = nullptr; const uint64_t* cnt = nullptr; uint32_t nc = 0, nh = 0;
        if (vtx_donor_ll_get(ln.ctx, &ll, &cnt, &nc, &nh) != VTX_OK) return false;
        ln.donor_ll.assign(ll, ll + size_t(nc) * nh);
        ln.donor_cnt.assign(cnt, cnt + size_t(nc) * 3);
        return true;
    };
    auto consume = [&](Lane& ln) {
        if (!dumping && engine_ready[size_t(ln.rank)].get() != 0) { ln.rc = 1; std::lock_guard<std::mutex> g(mu); failed = true; cv.notify_all(); return; }
        for (size_t k = ln.lo; k < ln.hi && ln.rc == 0; ++k) {
            std::unique_ptr<StagedShard> sh;
            std::unique_ptr<DeviceShard> ds;
            {
                const double t_w = now_s();
                std::unique_lock<std::mutex> g(mu);
                cv.wait(g, [&] { return failed || ready[k] || ready_dev[k]; });
                if (failed) { ln.rc = 1; break; }
                sh = std::move(ready[k]); ds = std::move(ready_dev[k]);
                ln.consumed = k - ln.lo + 1;
                ln.wait_s += now_s() - t_w;
            }
            cv.notify_all();
            const double t_sub = now_s();
            struct SubmitClock { Lane& l; double t0; ~SubmitClock() { l.submit_s += now_s() - t0; } } submit_clock{ ln, t_sub };
            if (ds && dump) {                   // test dump of the host's share: loci, member table, compressed bytes, record boundaries
                auto put = [&](const void* p, size_t bytes) { uint64_t n = bytes; fwrite(&n, 8, 1, dump); if (bytes) fwrite(p, 1, bytes, dump); };
                fwrite("VTXD", 1, 4, dump);
                const int64_t tid64 = ds->tid;
                put(&tid64, 8);
                put(ds->locus_row.data(), ds->locus_row.size() * 4); put(ds->locus_start.data(), ds->locus_start.size() * 8); put(ds->locus_end.data(), ds->locus_end.size() * 8);
                put(ds->members.data(), ds->members.size() * sizeof(vtx_bgzf_block)); put(ds->comp.data(), ds->comp.size()); put(ds->entry_off.data(), ds->entry_off.size() * 8);
                put(ds->hap_bytes.data(), ds->hap_bytes.size()); put(ds->ref_off.data(), ds->ref_off.size() * 4); put(ds->ref_len.data(), ds->ref_len.size() * 4);
                put(ds->alt_off.data(), ds->alt_off.size() * 4); put(ds->alt_len.data(), ds->alt_len.size() * 4);
                continue;
            }
            if (ds) {
                vtx_bam_shard bs;
                ds->fill(&bs, sa);
                const int brc = vtx_submit_bam(ln.ctx, &bs);
                if (brc == VTX_OK) { ln.hm.add(ds->met); continue; }
                if (brc != VTX_E_UNSUPPORTED) { ln.err = vtx_last_error(ln.ctx); ln.rc = 1; break; }
                // a shard the device cannot key (e.g. a UB string outside vtx_pack_umi's alphabet): stage it here, on the host
                if (!ln.fb_open) {
                    std::string e;
                    if (!ln.fb_fa.open(o.fasta, &e) || !ln.fb_bam.open(o.bam, &e)) { ln.err = e; ln.rc = 1; break; }
                    ln.fb_open = true;
                }
                sh = std::make_unique<StagedShard>();
                std::string e;
                const size_t lo = shard_lo[k], hi = shard_lo[k + 1];
                if (!stage_loci(recs, lo, hi, ln.fb_fa, ln.fb_bam, sa, umis, sh.get(), &e)) { ln.err = e; ln.rc = 1; break; }
                ++ln.host_fallbacks;
            }
            ln.hm.add(sh->met);
            if (!o.out_variant_stats.empty()) {
                ln.host_rows.insert(ln.host_rows.end(), sh->locus_row.begin(), sh->locus_row.end());
                ln.host_filters.insert(ln.host_filters.end(), sh->locus_filters.begin(), sh->locus_filters.end());
            }
            auto recycle = [&]() { sh->clear(); std::lock_guard<std::mutex> g(mu); recycled.push_back(std::move(sh)); };
            if (dump) { dump_shard(dump, *sh); recycle(); continue; }
            Arena& ar = ln.arenas[(k - ln.lo) % 3];
            if (k - ln.lo >= 3 && vtx_wait_copies(ln.ctx) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); ln.rc = 1; break; }     // the arena's previous copy must have landed
            if (!ar.ensure(sh->bytes())) { ln.err = "pinned allocation failed"; ln.rc = 1; break; }
            vtx_batch2 b;
            const uint64_t t_ar = StageClock::now();
            stage_into_arena(*sh, ar, &b);
            arena_ns += StageClock::now() - t_ar; staged_bytes += sh->bytes();
            if (vtx_submit2(ln.ctx, &b) != VTX_OK) { ln.err = vtx_last_error(ln.ctx); ln.rc = 1; }
            recycle();
        }
        if (ln.rc) { std::lock_guard<std::mutex> g(mu); failed = true; cv.notify_all(); return; }
        if (dump || n_dev == 1) return;
        // several GPUs: results stay on the device; one rooted gather over NCCL brings them to lane 0 (the writer)
        vtx_result tmp{};
        if (vtx_finish_device(ln.ctx, &ln.dev) != VTX_OK || !take_stats(ln) || !take_donors(ln) || vtx_gather_start(ln.ctx, 0) != VTX_OK || vtx_gather_wait(ln.ctx, &tmp) != VTX_OK) {
            ln.err = vtx_last_error(ln.ctx); ln.rc = 1; return;
        }
        ln.dev = tmp;
    };
    LOG_INFO("[%.3f s] staging on %ld thread(s) for %zu GPU(s), %zu shards of up to %ld records", now_s(), o.threads, n_dev, n_shards, o.shard_loci);
    {
        std::vector<std::thread> lane_threads;
        for (size_t d = 1; d < n_dev; ++d) lane_threads.emplace_back(consume, std::ref(lanes[d]));
        consume(lanes[0]);
        for (auto& t : lane_threads) t.join();
    }
    int rc = 0;
    HostMetrics hm;
    for (Lane& ln : lanes) {
        hm.add(ln.hm);
        if (ln.rc) rc = 1;
        if (ln.ctx) LOG_INFO("GPU %d: engine up at %.3f s; consumer waited %.3f s for staged shards, spent %.3f s submitting", ln.device, ln.ready_s, ln.wait_s, ln.submit_s);
        if (gpu_stage && ln.ctx && !ln.rc) {          // the record-filter counters of the shards the device staged
            vtx_bam_metrics bm{};
            if (vtx_bam_metrics_get(ln.ctx, &bm) == VTX_OK) {
                hm.num_reads += bm.num_reads; hm.num_low_mapq += bm.num_low_mapq; hm.num_non_primary += bm.num_non_primary;
                hm.num_duplicates += bm.num_duplicates; hm.num_not_useful += bm.num_not_useful;
            }
            uint64_t low_bq = 0;
            if (o.min_base_quality && vtx_bam_low_base_quality(ln.ctx, &low_bq) == VTX_OK) hm.num_low_base_quality += low_bq;
            if (ln.host_fallbacks) LOG_INFO("GPU %d: %zu shard(s) staged on the host after the device declined them", ln.device, ln.host_fallbacks);
        }
    }
    if (rc) { std::lock_guard<std::mutex> g(mu); failed = true; }
    cv.notify_all();
    for (auto& t : pool) t.join();
    if (failed && !fail_msg.empty()) { printf("Vartrix error.\nError: %s\n", fail_msg.c_str()); rc = 1; }
    for (Lane& ln : lanes) if (!ln.err.empty()) { printf("Vartrix error.\nError: %s\n", ln.err.c_str()); rc = 1; }
    if (dump) { fclose(dump); return rc; }
    if (rc) { fflush(nullptr); _exit(rc); }

    LOG_INFO("[%.3f s] all shards staged and submitted", now_s());
    vtx_ctx* ctx = lanes[0].ctx;
    vtx_result res{};
    const int frc = n_dev == 1 ? vtx_finish(ctx, &res) : vtx_fetch(ctx, &lanes[0].dev, &res);
    if (frc != VTX_OK || (n_dev == 1 && (!take_stats(lanes[0]) || !take_donors(lanes[0])))) { printf("Vartrix error.\nError: %s\n", vtx_last_error(ctx)); fflush(nullptr); _exit(1); }

    LOG_INFO("[%.3f s] triplets on the host", now_s());
    {   // where the time went: thread-seconds of the staging pool, device milliseconds of the last finish
        const StageClock& c = stage_clock();
        LOG_INFO("Staging thread-seconds: total %.3f = file read %.3f + inflate %.3f + crc32 %.3f + record scan / filters / packing %.3f; %llu BGZF blocks, %.1f MB inflated; copy into pinned arenas %.3f s (%.1f MB)",
                 stage_ns.load() * 1e-9, c.read_ns.load() * 1e-9, (c.inflate_ns.load() + c.device_inflate_ns.load()) * 1e-9, c.crc_ns.load() * 1e-9,
                 (double(stage_ns.load()) - double(c.read_ns.load()) - double(c.inflate_ns.load()) - double(c.device_inflate_ns.load()) - double(c.crc_ns.load())) * 1e-9,
                 (unsigned long long)c.blocks.load(), c.inflated_bytes.load() * 1e-6, arena_ns.load() * 1e-9, staged_bytes.load() * 1e-6);
        for (Lane& ln : lanes) {
            vtx_timing t{};
            if (vtx_last_timing(ln.ctx, &t) == VTX_OK)
                LOG_INFO("GPU %d device ms: h2d %.2f, prep %.2f, Smith-Waterman %.2f, post %.2f (%llu pairs, %llu launches)", ln.device, t.h2d_ms, t.prep_ms,
                         t.sw_ms, t.post_ms, (unsigned long long)t.n_pairs, (unsigned long long)t.total_launches);
        }
    }
    // metrics (main.rs:350-379)
    LOG_INFO("Number of alignments evaluated: %llu", (unsigned long long)hm.num_reads);
    LOG_INFO("Number of alignments skipped due to low mapping quality: %llu", (unsigned long long)hm.num_low_mapq);
    LOG_INFO("Number of alignments skipped due to not being primary: %llu", (unsigned long long)hm.num_non_primary);
    LOG_INFO("Number of alignments skipped due to being duplicates: %llu", (unsigned long long)hm.num_duplicates);
    LOG_INFO("Number of alignments skipped due to not being associated with a cell barcode: %llu", (unsigned long long)res.metrics.num_not_cell_bc);
    LOG_INFO("Number of alignments skipped due to not intersecting variant: %llu", (unsigned long long)hm.num_not_useful);
    if (o.min_base_quality) LOG_INFO("Number of alignments skipped due to low base quality at the variant: %llu", (unsigned long long)hm.num_low_base_quality);
    LOG_INFO("Number of alignments skipped due to not having a UMI: %llu", (unsigned long long)res.metrics.num_non_umi);
    LOG_INFO("Number of VCF records skipped due to having invalid characters in the alternative haplotype: %llu", (unsigned long long)hm.num_invalid_recs);
    LOG_INFO("Number of VCF records skipped due to being multi-allelic: %llu", (unsigned long long)hm.num_multiallelic_recs);
    LOG_INFO("Number of (read, locus) pairs scored on the GPU: %llu", (unsigned long long)res.metrics.num_scored);

    if (!write_mtx(o.out_matrix, recs.size(), bcs.keys.size(), res.n, res.row, res.col, res.val, &err, unsigned(o.threads))) { printf("Vartrix error.\nError: Error writing out-matrix\n"); rc = 1; }
    if (o.scoring == "coverage")        // clap-2 default_value counts as present (main.rs:100, 385)
        if (!write_mtx(o.ref_matrix, recs.size(), bcs.keys.size(), res.n, res.row, res.col, res.val2, &err, unsigned(o.threads))) { printf("Vartrix error.\nError: Error writing ref-matrix\n"); rc = 1; }

    if (!o.out_variants.empty()) {      // write_variants (main.rs:1166-1179): chrom_pos0
        validate_output_path(o.out_variants);
        FILE* f = fopen(o.out_variants.c_str(), "wb");
        if (!f) { LOG_ERR("error writing variants file"); rc = 1; }
        else { for (const VcfRecord& r : recs) fprintf(f, "%s_%lld\n", r.chrom.c_str(), (long long)r.pos0); fclose(f); }
    }
    if (!o.out_barcodes.empty()) {      // write_barcodes (main.rs:1181-1195): index order
        validate_output_path(o.out_barcodes);
        FILE* f = fopen(o.out_barcodes.c_str(), "wb");
        if (!f) { LOG_ERR("error writing barcodes file"); rc = 1; }
        else { for (const std::string& k : bcs.keys) { fwrite(k.data(), 1, k.size(), f); fputc('\n', f); } fclose(f); }
    }
    if (!o.out_variant_stats.empty()) {
        validate_output_path(o.out_variant_stats);
        std::vector<vtx_locus_stats> dev;
        std::vector<uint32_t> host_rows, host_filters;
        for (const Lane& ln : lanes) {
            dev.insert(dev.end(), ln.stats.begin(), ln.stats.end());
            host_rows.insert(host_rows.end(), ln.host_rows.begin(), ln.host_rows.end());
            host_filters.insert(host_filters.end(), ln.host_filters.begin(), ln.host_filters.end());
        }
        if (!write_variant_stats(o.out_variant_stats, recs, dev, host_rows, host_filters)) { LOG_ERR("error writing variant statistics file"); rc = 1; }
    }
    if (with_donors) {                  // the lanes' int64 sums add up to the one-GPU sums exactly
        validate_output_path(o.out_donors);
        const size_t H = vtx::donors::n_hyp(uint32_t(donors.names.size()));
        std::vector<int64_t> ll(bcs.keys.size() * H, 0);
        std::vector<uint64_t> cnt(bcs.keys.size() * 3, 0);
        for (const Lane& ln : lanes) {
            if (ln.donor_ll.size() != ll.size() || ln.donor_cnt.size() != cnt.size()) { LOG_ERR("donor sums of GPU %d have the wrong size", ln.device); rc = 1; continue; }
            for (size_t i = 0; i < ll.size(); ++i) ll[i] += ln.donor_ll[i];
            for (size_t i = 0; i < cnt.size(); ++i) cnt[i] += ln.donor_cnt[i];
        }
        uint64_t calls[3] = { 0, 0, 0 };
        if (!write_donors(o.out_donors, bcs.keys, donors.names, ll, cnt, calls)) { LOG_ERR("error writing donor file"); rc = 1; }
        std::string list;
        for (const std::string& n : donors.names) list += (list.empty() ? "" : ",") + n;
        LOG_INFO("Donors: %zu (%s), error rate %g; rows with a genotype for every donor: %llu of %zu; cells: %llu singlet, %llu doublet, %llu unassigned",
                 donors.names.size(), list.c_str(), o.donor_error_rate, (unsigned long long)donors.usable, recs.size(),
                 (unsigned long long)calls[0], (unsigned long long)calls[1], (unsigned long long)calls[2]);
    }
    LOG_INFO("[%.3f s] outputs written", now_s());
    double sum = 0;
    for (uint64_t k = 0; k < res.n; ++k) sum += res.val[k];
    if (sum == 0.0) LOG_ERR("The resulting matrix has a sum of 0. Did you use the --umi flag on data without UMIs?");   // main.rs:410-415
    // every output is closed; tearing the CUDA contexts and the pinned arenas down costs 0.5-0.9 s that a one-shot CLI
    // does not need to spend (the driver reclaims everything at process exit)
    fflush(nullptr);
    _exit(rc);
}
