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
#include <cstdlib>
#include <future>
#include <thread>

#include "host.hpp"

using namespace host;

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
    const std::string refName = argv[1];
    GibbsArgs a;
    {
        const std::string why = parse_gibbs_args(std::vector<std::string>(argv + 2, argv + argc), a);
        if (!why.empty()) die(why);
    }
    g_verbose = !a.quiet;
    clamp_gibbs_chains(a);
    const int nThreads = a.nThreads;
    {   // -p means chains here (as in the reference); file parsing uses the host's cores
        const unsigned hw = std::thread::hardware_concurrency();
        g_io_threads = env_int("RSEM_B200_IO_THREADS", (int)std::min<unsigned>(hw ? hw : 1, 32));
    }

    // chains are spread over the devices of RSEM_B200_DEVICES (rsem-run-em's list), each device used once: two cooperative
    // grids sized to a whole device must never share one; no device without a chain
    std::vector<int> devices;
    for (int d : gpu_devices())
        if (std::find(devices.begin(), devices.end(), d) == devices.end()) devices.push_back(d);
    if ((int)devices.size() > nThreads) devices.resize(nThreads);
    const int n_dev = (int)devices.size();

    // CUDA context creation takes seconds on a multi-GPU node: overlap it with the .ofg parsing
    std::vector<std::future<LaneContexts>> ctx_futures;
    for (int d : devices) ctx_futures.push_back(std::async(std::launch::async, open_lanes, std::vector<int>{d}));
    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    const double t_begin = now_s();

    auto say = [](const std::string& s) { if (g_verbose) fputs(s.c_str(), stdout); };
    RefData refs;
    load_refs(refName + ".seq", false, refs);
    const int M = refs.M;
    GibbsSample s;
    load_gibbs_ofg(a, M, s, say);
    std::vector<int> gi, gt, ta;
    load_groups(refName + ".grp", gi);
    const bool alleleS = load_allele_groups(refName, gt, ta);
    say("Loading group information is finished!\n");
    load_gibbs_inputs(a, refs, s, say);

    std::vector<rsem_b200_ctx*> ctxs;
    {
        std::vector<LaneContexts> rs;
        for (auto& f : ctx_futures) rs.push_back(f.get());   // every creation has returned before the run may stop
        for (const LaneContexts& r : rs)
            if (!r.err.empty()) die(r.err);
        for (const LaneContexts& r : rs) ctxs.push_back(r.ctx[0]);
    }
    const double t_loaded = now_s();
    // the component analysis and the row permutation run once, on the first device; the others copy its layout
    check_rc(rsem_b200_gibbs_upload(ctxs[0], s.N1, s.sid.size(), M, s.row_ptr.data(), s.sid.data(), s.conprb.data()), "gibbs_upload");
    const double t_uploaded = now_s();

    const rsem_b200_gibbs_params gp = gibbs_params(a, s, gi);
    std::vector<int32_t> cvs((size_t)a.nsamples * (M + 1));
    const size_t acc_per = 4 * ((size_t)M + 1) + gi.size() - 1;
    std::vector<double> chain_acc((size_t)nThreads * acc_per);

    // one host thread per device, each running a contiguous range of chains into its slice of the count vectors and
    // of the per-chain sums; the ranges depend only on the chain shapes (rsem_b200_gibbs_split_chains)
    std::vector<int32_t> bounds(n_dev + 1);
    check_rc(rsem_b200_gibbs_split_chains(nThreads, s.chain_samples.data(), a.burnin, a.gap, n_dev, bounds.data()), "gibbs_split_chains");
    std::vector<size_t> cv_first(nThreads + 1, 0);   // first count vector of every chain
    for (int t = 0; t < nThreads; ++t) cv_first[t + 1] = cv_first[t] + s.chain_samples[t];
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
        p.chain_samples = s.chain_samples.data() + t0;
        p.chain_seeds = s.chain_seeds.data() + t0;
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
    const double t_sampled = now_s();
    finish_gibbs_sample(refName, a, s, gi, alleleS, ta, cvs.data(), chain_acc.data(), say);
    if (timing) {
        fprintf(stderr, "rsem-run-gibbs timing: load+ctx %.3f s, upload+components %.3f s, sampling %.3f s (%d chains)\n",
                t_loaded - t_begin, t_uploaded - t_loaded, t_sampled - t_uploaded, nThreads);
        for (int d = 0; d < n_dev; ++d)
            fprintf(stderr, "rsem-run-gibbs timing: device %d: chains %d..%d, %d worker CTAs per chain, %.3f ms on the device\n",
                    devices[d], bounds[d], bounds[d + 1] - 1, dev_stats[d].worker_ctas, dev_stats[d].device_ms);
    }
    for (rsem_b200_ctx* c : ctxs) rsem_b200_ctx_destroy(c);
    return 0;
}
