// Per-sample stages of rsem-run-gibbs, shared by rsem-run-gibbs and rsem-run-gibbs-batch.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>

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

std::string parse_gibbs_args(const std::vector<std::string>& f, GibbsArgs& a) {
    a.imdName = f[0];
    a.statName = f[1];
    a.burnin = atoi(f[2].c_str());
    a.nsamples = atoi(f[3].c_str());
    a.gap = atoi(f[4].c_str());
    for (size_t i = 5; i < f.size(); ++i) {
        const bool arg = i + 1 < f.size();
        if (f[i] == "-p" && arg) a.nThreads = atoi(f[i + 1].c_str());
        if (f[i] == "--seed" && arg) { a.hasSeed = true; a.seed = parse_seed(f[i + 1].c_str()); }
        if (f[i] == "--pseudo-count" && arg) a.pseudoC = atof(f[i + 1].c_str());
        if (f[i] == "-q") a.quiet = true;
        if (f[i] == "--prior" && arg) { a.hasPrior = true; a.fprior = f[i + 1]; }
    }
    if (!(a.nsamples > 1)) return "NSAMPLES must be larger than 1, otherwise the posterior variance cannot be calculated!";
    if (a.gap < 1) return "GAP must be at least 1!";
    return "";
}

void clamp_gibbs_chains(GibbsArgs& a) {
    if (a.nThreads > a.nsamples) {
        a.nThreads = a.nsamples;
        fprintf(stderr, "Warning: Number of samples is less than number of threads! Change the number of threads to %d!\n", a.nThreads);
    }
    if (a.nThreads < 1) a.nThreads = 1;
}

void load_gibbs_ofg(const GibbsArgs& a, int M, GibbsSample& s, const Say& say) {
    load_ofg(a.imdName + ".ofg", M, s.N0, s.row_ptr, s.sid, s.conprb);
    s.N1 = s.row_ptr.size() - 1;
    say("Loading data is finished!\n");
}

void load_gibbs_inputs(const GibbsArgs& a, const RefData& refs, GibbsSample& s, const Say& say) {
    const int M = refs.M;
    const std::string why = gibbs_inputs(a.imdName, M, s.N0, s.N1, a.pseudoC, a.hasPrior ? &a.fprior : nullptr, s.init_counts,
                                         s.alpha, s.totc);
    if (!why.empty()) die(why);
    // init_model_related: eel from the .model's gld, mw copy
    int model_type = 0;
    LenDistH gld;
    HostModel::read_for_gibbs(a.statName + ".model", M, model_type, gld, s.mw);
    calc_eel(refs, gld, s.eel);
    say("Gibbs started!\n");
    // init(): samples per chain and per-chain engines (Gibbs.cpp:207-254)
    s.chain_seeds = engine_seeds(a.hasSeed ? a.seed : (uint32_t)time(NULL), a.nThreads);
    s.chain_samples.resize(a.nThreads);
    const int quotient = a.nsamples / a.nThreads, left = a.nsamples % a.nThreads;
    for (int t = 0; t < a.nThreads; ++t) s.chain_samples[t] = quotient + (t < left ? 1 : 0);
    say("Initialization finished!\n");
}

rsem_b200_gibbs_params gibbs_params(const GibbsArgs& a, const GibbsSample& s, const std::vector<int>& gi) {
    rsem_b200_gibbs_params gp;
    memset(&gp, 0, sizeof gp);
    gp.M = (int)s.init_counts.size() - 1;
    gp.burnin = a.burnin;
    gp.gap = a.gap;
    gp.n_chains = (int)s.chain_samples.size();
    gp.chain_samples = s.chain_samples.data();
    gp.chain_seeds = s.chain_seeds.data();
    gp.n0 = (double)s.N0;
    gp.init_counts = s.init_counts.data();
    gp.pseudo_counts = s.alpha.data();
    gp.totc = s.totc;
    gp.eel = s.eel.data();
    gp.mw = s.mw.data();
    gp.n_genes = (int)gi.size() - 1;
    gp.gene_start = gi.data();
    return gp;
}

namespace {

// imdName.countvectors<t>, one per chain (Gibbs.cpp:257-262); cvs holds the chains' vectors in chain order
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

// release() (Gibbs.cpp:399-422): means and unbiased variances from the sums of all chains and the kept count vectors,
// then imdName.iso_res / gene_res (and the allele file) by write_results_gibbs
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

}  // namespace

void finish_gibbs_sample(const std::string& refName, const GibbsArgs& a, const GibbsSample& s, const std::vector<int>& gi,
                         bool alleleS, const std::vector<int>& ta, const int32_t* cvs, const double* chain_acc, const Say& say) {
    const int M = (int)s.init_counts.size() - 1, m = (int)gi.size() - 1;
    std::vector<double> sum_c(M + 1), sum_c2(M + 1), sum_tpm(M + 1), sum_fpkm(M + 1), sum_g2(m);
    rsem_b200_gibbs_out go;
    go.count_vectors = nullptr;   // not touched by the sums
    go.sum_c = sum_c.data(); go.sum_c2 = sum_c2.data(); go.sum_tpm = sum_tpm.data(); go.sum_fpkm = sum_fpkm.data();
    go.sum_gene_c2 = sum_g2.data();
    const rsem_b200_gibbs_params gp = gibbs_params(a, s, gi);
    check_rc(rsem_b200_gibbs_sum_chains(&gp, chain_acc, &go), "gibbs_sum_chains");
    write_countvectors(a.imdName, M, s.chain_samples, cvs);
    say("Gibbs finished!\n");
    write_gibbs_results(refName, a.imdName, M, a.nsamples, gi, alleleS, ta, cvs, sum_c, sum_c2, sum_tpm, sum_fpkm, sum_g2);
}

}  // namespace host
