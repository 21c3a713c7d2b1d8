// Per-sample stages of rsem-run-gibbs, shared by rsem-run-gibbs and rsem-run-gibbs-batch.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "host.hpp"

namespace host {

std::string gibbs_inputs(const std::string& imdName, int M, uint64_t N0, uint64_t N1, double pseudoC, const std::string* fprior,
                         std::vector<int32_t>& init_counts, std::vector<double>& alpha, double& totc) {
    // load_omit_info (Gibbs.cpp:152-167)
    init_counts.assign(M + 1, 0);
    totc = M + 1;
    {
        FILE* fi = fopen((imdName + ".omit").c_str(), "r");
        if (!fi) return "Cannot open " + imdName + ".omit!";
        int tid;
        while (fscanf(fi, "%d", &tid) == 1) {
            if (tid < 0 || tid > M) { fclose(fi); return "Invalid transcript id in " + imdName + ".omit!"; }
            init_counts[tid] = -1;
            --totc;
        }
        fclose(fi);
    }
    totc = totc * pseudoC + N0 + N1;
    alpha.assign(M + 1, pseudoC);
    if (fprior) {  // load_prior_info (Gibbs.cpp:171-194)
        alpha.assign(M + 1, 0.0);
        // one prior per transcript and line, anything after the number is a comment (Gibbs.cpp:178-184 uses getline:
        // no limit on the line length)
        {
            FILE* fi = fopen(fprior->c_str(), "rb");
            if (!fi) return "Cannot open " + *fprior + "! It may not exist.";
            fclose(fi);
        }
        std::vector<char> buf = slurp(*fprior, false);
        buf.push_back('\0');
        const char* q = buf.data();
        const char* const end = q + buf.size() - 1;
        for (int i = 1; i <= M; ++i) {
            if (q >= end) return "The prior file " + *fprior + " has fewer lines than transcripts!";
            const char* eol = static_cast<const char*>(memchr(q, '\n', (size_t)(end - q)));
            if (!eol) eol = end;
            char* after = nullptr;
            const double prior = strtod(q, &after);
            if (after == q || after > eol) return "Cannot read the prior of transcript " + std::to_string(i) + " from " + *fprior + "!";
            if (init_counts[i] == 0) alpha[i] = prior;
            q = eol < end ? eol + 1 : end;
        }
        totc = 1;
        for (int i = 1; i <= M; ++i)
            if (init_counts[i] == 0) totc += alpha[i];
        totc += N0 + N1;
    }
    return "";
}

void write_countvectors(const std::string& imdName, int M, const std::vector<int32_t>& chain_samples, const int32_t* cvs) {
    size_t at = 0;
    std::vector<char> buf(1 << 20);
    for (size_t t = 0; t < chain_samples.size(); ++t) {
        FILE* fo = fopen((imdName + ".countvectors" + std::to_string(t)).c_str(), "w");
        if (!fo) die("Cannot open " + imdName + ".countvectors" + std::to_string(t) + " for writing!");
        setvbuf(fo, buf.data(), _IOFBF, buf.size());
        for (int s = 0; s < chain_samples[t]; ++s, ++at) {
            const int32_t* c = &cvs[at * (M + 1)];
            for (int i = 0; i < M; ++i) fprintf(fo, "%d ", c[i]);
            fprintf(fo, "%d\n", c[M]);
        }
        fclose(fo);
    }
}

void write_gibbs_results(const std::string& refName, const std::string& imdName, int M, int NSAMPLES, const std::vector<int>& gi,
                         bool alleleS, const std::vector<int>& ta, const int32_t* cvs, const std::vector<double>& sum_c,
                         const std::vector<double>& sum_c2, const std::vector<double>& sum_tpm, const std::vector<double>& sum_fpkm,
                         const std::vector<double>& sum_g2) {
    const int m = (int)gi.size() - 1;
    std::vector<double> pme_c(M + 1), pve_c(M + 1), pme_tpm(M + 1), pme_fpkm(M + 1), pve_g(m), pve_t;
    for (int i = 0; i <= M; ++i) {
        pme_c[i] = sum_c[i] / NSAMPLES;
        pve_c[i] = (sum_c2[i] - double(NSAMPLES) * pme_c[i] * pme_c[i]) / double(NSAMPLES - 1);
        if (pve_c[i] < 0.0) pve_c[i] = 0.0;
        pme_tpm[i] = sum_tpm[i] / NSAMPLES;
        pme_fpkm[i] = sum_fpkm[i] / NSAMPLES;
    }
    for (int i = 0; i < m; ++i) {
        double g = 0.0;
        for (int j = gi[i]; j < gi[i + 1]; ++j) g += pme_c[j];
        pve_g[i] = (sum_g2[i] - double(NSAMPLES) * g * g) / double(NSAMPLES - 1);
        if (pve_g[i] < 0.0) pve_g[i] = 0.0;
    }
    if (alleleS) {  // allele-level variances from the kept count vectors (Gibbs.cpp:338-345, 414-421)
        const int m_trans = (int)ta.size() - 1;
        pve_t.assign(m_trans, 0.0);
        for (int s = 0; s < NSAMPLES; ++s) {
            const int32_t* c = &cvs[(size_t)s * (M + 1)];
            for (int i = 0; i < m_trans; ++i) {
                double x = 0.0;
                for (int j = ta[i]; j < ta[i + 1]; ++j) x += c[j];
                pve_t[i] += x * x;
            }
        }
        for (int i = 0; i < m_trans; ++i) {
            double x = 0.0;
            for (int j = ta[i]; j < ta[i + 1]; ++j) x += pme_c[j];
            pve_t[i] = (pve_t[i] - double(NSAMPLES) * x * x) / double(NSAMPLES - 1);
            if (pve_t[i] < 0.0) pve_t[i] = 0.0;
        }
    }
    write_results_gibbs(refName, imdName, M, pme_c, pme_fpkm, pme_tpm, pve_c, pve_g, pve_t);
}

}  // namespace host
