// rsem-run-gibbs, H100 edition: same argv and files as the reference (the reference's Gibbs.cpp:425-530).
//
//   rsem-run-gibbs reference_name imdName statName BURNIN NSAMPLES GAP [-p #Threads] [--seed seed]
//                  [--pseudo-count pseudo_count] [--prior file] [-q]
//
// -p keeps its meaning: it is the number of independent chains (the results depend on it, exactly as in
// the reference: NSAMPLES is split over the chains and each chain gets its own mt19937 seed).
// The GPU is chosen with RSEM_B200_DEVICE (default 0); with RSEM_B200_DEVICES=0,1,.. the chains are split into contiguous
// ranges, one per listed device, and the per-chain sums are added up on the host in chain order, so the files are the same
// as on one device.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <ctime>
#include <future>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 7) {
        printf("Usage: rsem-run-gibbs reference_name imdName statName BURNIN NSAMPLES GAP [-p #Threads] [--seed seed] [--pseudo-count pseudo_count] [--prior file] [-q]\n");
        printf("\n");
        printf("Format of the prior file:\n");
        printf("- One isoform's prior per line\n");
        printf("- Priors must be in the same order as in the .ti file\n");
        printf("- Priors for those to-be-omitted isoforms must be included as well\n");
        printf("- Comments can be added after prior separated by space(s)\n");
        exit(-1);
    }
    const std::string refName = argv[1], imdName = argv[2], statName = argv[3];
    const int BURNIN = atoi(argv[4]), NSAMPLES = atoi(argv[5]), GAP = atoi(argv[6]);
    int nThreads = 1;
    bool hasSeed = false, quiet = false, has_prior = false;
    uint32_t seed = 0;
    double pseudoC = 1.0;
    std::string fprior;
    for (int i = 7; i < argc; ++i) {
        if (!strcmp(argv[i], "-p") && i + 1 < argc) nThreads = atoi(argv[i + 1]);
        if (!strcmp(argv[i], "--seed") && i + 1 < argc) { hasSeed = true; seed = parse_seed(argv[i + 1]); }
        if (!strcmp(argv[i], "--pseudo-count") && i + 1 < argc) pseudoC = atof(argv[i + 1]);
        if (!strcmp(argv[i], "-q")) quiet = true;
        if (!strcmp(argv[i], "--prior") && i + 1 < argc) { has_prior = true; fprior = argv[i + 1]; }
    }
    g_verbose = !quiet;
    if (!(NSAMPLES > 1)) die("NSAMPLES must be larger than 1, otherwise the posterior variance cannot be calculated!");
    if (GAP < 1) die("GAP must be at least 1!");
    if (nThreads > NSAMPLES) {
        nThreads = NSAMPLES;
        fprintf(stderr, "Warning: Number of samples is less than number of threads! Change the number of threads to %d!\n", nThreads);
    }
    if (nThreads < 1) nThreads = 1;
    {   // -p means chains here (as in the reference); file parsing uses the host's cores
        const char* e = getenv("RSEM_B200_IO_THREADS");
        const unsigned hw = std::thread::hardware_concurrency();
        g_io_threads = e ? atoi(e) : (int)std::min<unsigned>(hw ? hw : 1, 32);
    }

    // chains are spread over the devices of RSEM_B200_DEVICES (rsem-run-em's list), each device used once: two cooperative
    // grids sized to a whole device must never share one; no device without a chain
    std::vector<int> devices;
    for (int d : gpu_devices())
        if (std::find(devices.begin(), devices.end(), d) == devices.end()) devices.push_back(d);
    if ((int)devices.size() > nThreads) devices.resize(nThreads);
    const int n_dev = (int)devices.size();

    // CUDA context creation takes seconds on a multi-GPU node: overlap it with the .ofg parsing
    struct CtxResult { int rc; rsem_b200_ctx* ctx; std::string err; };
    std::vector<std::future<CtxResult>> ctx_futures;
    for (int d : devices)
        ctx_futures.push_back(std::async(std::launch::async, [d]() {
            CtxResult r{0, nullptr, ""};
            r.rc = rsem_b200_ctx_create(d, &r.ctx);
            if (r.rc != 0) r.err = rsem_b200_last_error();
            return r;
        }));
    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_begin = now();

    // load_data
    RefData refs;
    load_refs(refName + ".seq", false, refs);
    const int M = refs.M;
    uint64_t N0 = 0;
    std::vector<uint64_t> row_ptr;
    std::vector<int32_t> sid;
    std::vector<double> conprb;
    load_ofg(imdName + ".ofg", M, N0, row_ptr, sid, conprb);
    const uint64_t N1 = row_ptr.size() - 1;
    if (g_verbose) printf("Loading data is finished!\n");

    std::vector<int> gi, gt, ta;
    load_groups(refName + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(refName, gt, ta);
    if (g_verbose) printf("Loading group information is finished!\n");

    std::vector<int32_t> init_counts;
    std::vector<double> alpha;
    double totc = 0;
    {
        const std::string why = gibbs_inputs(imdName, M, N0, N1, pseudoC, has_prior ? &fprior : nullptr, init_counts, alpha, totc);
        if (!why.empty()) die(why);
    }

    // init_model_related: eel from the .model's gld, mw copy
    int model_type = 0;
    LenDistH gld;
    std::vector<double> mw, eel;
    HostModel::read_for_gibbs(statName + ".model", M, model_type, gld, mw);
    calc_eel(refs, gld, eel);

    if (g_verbose) printf("Gibbs started!\n");

    // init(): samples per chain and per-chain engines (Gibbs.cpp:207-254)
    std::vector<int32_t> chain_samples(nThreads);
    std::vector<uint32_t> chain_seeds = engine_seeds(hasSeed ? seed : (uint32_t)time(NULL), nThreads);
    {
        const int quotient = NSAMPLES / nThreads, left = NSAMPLES % nThreads;
        for (int i = 0; i < nThreads; ++i) chain_samples[i] = quotient + (i < left ? 1 : 0);
    }
    if (g_verbose) printf("Initialization finished!\n");

    std::vector<rsem_b200_ctx*> ctxs;
    {
        std::vector<CtxResult> rs;
        for (auto& f : ctx_futures) rs.push_back(f.get());   // every creation has returned before the run may stop
        for (const CtxResult& r : rs)
            if (r.rc != 0) die("rsem_b200: ctx_create failed: " + r.err);
        for (const CtxResult& r : rs) ctxs.push_back(r.ctx);
    }
    const double t_loaded = now();
    // the component analysis and the row permutation run once, on the first device; the others copy its layout
    check_rc(rsem_b200_gibbs_upload(ctxs[0], N1, sid.size(), M, row_ptr.data(), sid.data(), conprb.data()), "gibbs_upload");
    const double t_uploaded = now();

    rsem_b200_gibbs_params gp;
    memset(&gp, 0, sizeof gp);
    gp.M = M; gp.burnin = BURNIN; gp.gap = GAP; gp.n_chains = nThreads;
    gp.chain_samples = chain_samples.data();
    gp.chain_seeds = chain_seeds.data();
    gp.n0 = (double)N0;
    gp.init_counts = init_counts.data();
    gp.pseudo_counts = alpha.data();
    gp.totc = totc;
    gp.eel = eel.data();
    gp.mw = mw.data();
    gp.n_genes = m;
    gp.gene_start = gi.data();
    std::vector<int32_t> cvs((size_t)NSAMPLES * (M + 1));
    const size_t acc_per = 4 * ((size_t)M + 1) + (size_t)m;
    std::vector<double> chain_acc((size_t)nThreads * acc_per);
    std::vector<double> sum_c(M + 1), sum_c2(M + 1), sum_tpm(M + 1), sum_fpkm(M + 1), sum_g2(m);

    // one host thread per device, each running a contiguous range of chains into its slice of the count vectors and
    // of the per-chain sums; the ranges depend only on the chain shapes (rsem_b200_gibbs_split_chains)
    std::vector<int32_t> bounds(n_dev + 1);
    check_rc(rsem_b200_gibbs_split_chains(nThreads, chain_samples.data(), BURNIN, GAP, n_dev, bounds.data()), "gibbs_split_chains");
    std::vector<size_t> cv_first(nThreads + 1, 0);   // first count vector of every chain
    for (int t = 0; t < nThreads; ++t) cv_first[t + 1] = cv_first[t] + chain_samples[t];
    std::vector<rsem_b200_gibbs_stats> dev_stats(n_dev);
    std::vector<std::string> dev_err(n_dev);
    auto worker = [&](int d) {
        if (d > 0 && rsem_b200_gibbs_upload_from(ctxs[d], ctxs[0]) != 0) {
            dev_err[d] = std::string("rsem_b200: gibbs_upload_from failed: ") + rsem_b200_last_error();
            return;
        }
        const int t0 = bounds[d], t1 = bounds[d + 1];
        rsem_b200_gibbs_params p = gp;
        p.n_chains = t1 - t0;
        p.chain_samples = chain_samples.data() + t0;
        p.chain_seeds = chain_seeds.data() + t0;
        if (rsem_b200_gibbs_run_chains(ctxs[d], &p, cvs.data() + cv_first[t0] * (M + 1), chain_acc.data() + (size_t)t0 * acc_per,
                                       &dev_stats[d]) != 0)
            dev_err[d] = std::string("rsem_b200: gibbs_run failed: ") + rsem_b200_last_error();
    };
    {
        std::vector<std::thread> pool;
        for (int d = 1; d < n_dev; ++d) pool.emplace_back(worker, d);
        worker(0);
        for (auto& th : pool) th.join();
    }
    for (const std::string& e : dev_err)   // nothing is written unless every device finished its chains
        if (!e.empty()) die(e);
    rsem_b200_gibbs_out go;
    go.count_vectors = cvs.data();
    go.sum_c = sum_c.data(); go.sum_c2 = sum_c2.data(); go.sum_tpm = sum_tpm.data(); go.sum_fpkm = sum_fpkm.data();
    go.sum_gene_c2 = sum_g2.data();
    check_rc(rsem_b200_gibbs_sum_chains(&gp, chain_acc.data(), &go), "gibbs_sum_chains");
    if (timing) {
        fprintf(stderr, "rsem-run-gibbs timing: load+ctx %.3f s, upload+components %.3f s, sampling %.3f s (%d chains)\n",
                t_loaded - t_begin, t_uploaded - t_loaded, now() - t_uploaded, nThreads);
        for (int d = 0; d < n_dev; ++d)
            fprintf(stderr, "rsem-run-gibbs timing: device %d: chains %d..%d, %d worker CTAs per chain, %.3f ms on the device\n",
                    devices[d], bounds[d], bounds[d + 1] - 1, dev_stats[d].worker_ctas, dev_stats[d].device_ms);
    }
    for (rsem_b200_ctx* c : ctxs) rsem_b200_ctx_destroy(c);

    write_countvectors(imdName, M, chain_samples, cvs.data());
    if (g_verbose) printf("Gibbs finished!\n");
    write_gibbs_results(refName, imdName, M, NSAMPLES, gi, alleleS, ta, cvs.data(), sum_c, sum_c2, sum_tpm, sum_fpkm, sum_g2);
    return 0;
}
