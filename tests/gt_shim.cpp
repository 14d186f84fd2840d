// test shim: the CLI's VCF reader with its genotype sink (vartrix_b200/csrc/host/inputs.hpp) on one file, for
// tests/test_donors_cpu.py.  Writes the sample names (one tab-separated line) and one line of comma-separated dosages per record.
#include "../vartrix_b200/csrc/host/inputs.hpp"

extern "C" int vtx_test_read_genotypes(const char* vcf, const char* out)
{
    std::vector<vtxhost::VcfRecord> recs;
    vtxhost::VcfGenotypes g;
    std::string err;
    FILE* f = fopen(out, "w");
    if (!f) return 2;
    if (!vtxhost::read_vcf(vcf, &recs, &err, &g)) { fprintf(f, "error: %s\n", err.c_str()); fclose(f); return 1; }
    for (size_t i = 0; i < g.samples.size(); ++i) fprintf(f, "%s%s", i ? "\t" : "", g.samples[i].c_str());
    fputc('\n', f);
    const size_t ns = g.samples.size();
    for (size_t r = 0; r < recs.size(); ++r) {
        for (size_t i = 0; i < ns; ++i) fprintf(f, "%s%u", i ? "," : "", unsigned(g.dosage[r * ns + i]));
        fputc('\n', f);
    }
    fclose(f);
    return 0;
}
