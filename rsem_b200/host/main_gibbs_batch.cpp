// rsem-run-gibbs-batch: the Gibbs samplers of many samples against one reference in one process.
//
//   rsem-run-gibbs-batch refName manifest [-q]
//
// Each non-empty manifest line is what rsem-run-gibbs takes after reference_name:
//   imdName statName BURNIN NSAMPLES GAP [-p #chains] [--seed s] [--pseudo-count c] [--prior file]
// and each line gets the files `rsem-run-gibbs refName <line>` writes.  One CUDA context (RSEM_B200_DEVICE) serves the whole
// run.  A sample of 1248 .. 2^19 reads joins a Gibbs batch (K13, rsem_b200_gibbs_batch_*), which runs the chains of all its
// samples in one launch; any other sample runs on the context with rsem_b200_gibbs_upload + rsem_b200_gibbs_run_chains, as in
// rsem-run-gibbs.  When the batch arena is full, the samples in it are run and written before the next one is added; a
// sample that still does not fit then runs on the context.  RSEM_B200_BATCH_ARENA_BYTES sets the arena's size
// (default, or 0: half of the device memory free at the start).  Standard output has one block per sample, in manifest order.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <deque>
#include <future>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

struct Line {
    int no = 0;   // 1-based line number in the manifest
    std::string imdName, statName, fprior;
    int burnin = 0, nsamples = 0, gap = 0, nThreads = 1;
    bool hasSeed = false, hasPrior = false;
    uint32_t seed = 0;
    double pseudoC = 1.0;
};

// a loaded sample, from its .ofg to its written outputs
struct Sample {
    size_t idx = 0;
    uint64_t N0 = 0, N1 = 0;
    std::vector<uint64_t> row_ptr;
    std::vector<int32_t> sid;
    std::vector<double> conprb;
    std::vector<int32_t> init_counts, chain_samples;
    std::vector<uint32_t> chain_seeds;
    std::vector<double> alpha, eel, mw;
    double totc = 0;
};

void usage() {
    printf("Usage: rsem-run-gibbs-batch refName manifest [-q]\n\n");
    printf("  refName: reference name\n");
    printf("  manifest: one sample per line: imdName statName BURNIN NSAMPLES GAP [-p #Threads] [--seed seed] [--pseudo-count pseudo_count] [--prior file]\n");
    printf("  -q: set it quiet\n");
    exit(-1);
}

[[noreturn]] void refuse(const std::string& manifest, int no, const std::string& why) {
    fprintf(stderr, "%s line %d: %s\n", manifest.c_str(), no, why.c_str());
    exit(-1);
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// every manifest line is checked before the context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, int M) {
    std::vector<char> buf = slurp(path);
    std::string text(buf.begin(), buf.end());
    std::istringstream in(text);
    std::vector<Line> lines;
    std::map<std::string, int> seen;
    std::string raw;
    for (int no = 1; std::getline(in, raw); ++no) {
        std::istringstream ls(raw);
        std::vector<std::string> f;
        for (std::string w; ls >> w;) f.push_back(w);
        if (f.empty()) continue;
        if (f.size() < 5) refuse(path, no, "too few fields (imdName statName BURNIN NSAMPLES GAP [options])");
        Line l;
        l.no = no;
        l.imdName = f[0];
        l.statName = f[1];
        l.burnin = atoi(f[2].c_str());
        l.nsamples = atoi(f[3].c_str());
        l.gap = atoi(f[4].c_str());
        for (size_t i = 5; i < f.size(); ++i) {   // the option rules of rsem-run-gibbs
            if (f[i] == "-p" && i + 1 < f.size()) l.nThreads = atoi(f[i + 1].c_str());
            if (f[i] == "--seed" && i + 1 < f.size()) { l.hasSeed = true; l.seed = parse_seed(f[i + 1].c_str()); }
            if (f[i] == "--pseudo-count" && i + 1 < f.size()) l.pseudoC = atof(f[i + 1].c_str());
            if (f[i] == "--prior" && i + 1 < f.size()) { l.hasPrior = true; l.fprior = f[i + 1]; }
        }
        if (!(l.nsamples > 1)) refuse(path, no, "NSAMPLES must be larger than 1, otherwise the posterior variance cannot be calculated!");
        if (l.gap < 1) refuse(path, no, "GAP must be at least 1!");
        auto it = seen.find(l.imdName);
        if (it != seen.end()) refuse(path, no, "its outputs collide with line " + std::to_string(it->second) + " (same imdName)");
        seen[l.imdName] = no;
        {   // .ofg header: M N0
            FILE* fi = fopen((l.imdName + ".ofg").c_str(), "r");
            long long m = -1;
            unsigned long long n0 = 0;
            const int got = fi ? fscanf(fi, "%lld %llu", &m, &n0) : 0;
            if (fi) fclose(fi);
            if (got != 2) refuse(path, no, "cannot read or parse " + l.imdName + ".ofg");
            if (m != M) refuse(path, no, "M in " + l.imdName + ".ofg is not the reference's (M = " + std::to_string(M) + ")");
        }
        {
            std::vector<int32_t> init;
            std::vector<double> alpha;
            double totc = 0;
            const std::string why = gibbs_inputs(l.imdName, M, 0, 0, l.pseudoC, l.hasPrior ? &l.fprior : nullptr, init, alpha, totc);
            if (!why.empty()) refuse(path, no, why);
        }
        {   // .model: model type and orientation (the rest is read with the sample)
            FILE* fi = fopen((l.statName + ".model").c_str(), "r");
            int type = -1;
            double ori = 0;
            const bool ok = fi && fscanf(fi, "%d %lf", &type, &ori) == 2 && type >= 0 && type <= 3;
            if (fi) fclose(fi);
            if (!ok) refuse(path, no, "cannot read or parse " + l.statName + ".model");
        }
        if (l.nThreads > l.nsamples) {
            l.nThreads = l.nsamples;
            fprintf(stderr, "Warning: Number of samples is less than number of threads! Change the number of threads to %d!\n", l.nThreads);
        }
        if (l.nThreads < 1) l.nThreads = 1;
        lines.push_back(l);
    }
    return lines;
}

// RSEM_B200_TIMING=1: wall seconds per phase on stderr at the end
struct Phases {
    double load = 0, device = 0, copy = 0, write = 0;
    double k13_ms = 0;
    uint64_t chain_cycles = 0, sample_cycles = 0, jobs = 0;
    int teams = 0, workers = 0, batched = 0, single = 0, full = 0;
};

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 3) usage();
    const std::string refName = argv[1], manifest = argv[2];
    bool verbose = true;
    for (int i = 3; i < argc; ++i)
        if (!strcmp(argv[i], "-q")) verbose = false;
    g_verbose = false;   // the messages of the shared loaders and writers go into the samples' blocks instead
    {   // as rsem-run-gibbs: file parsing and writing use the host's cores
        const char* e = getenv("RSEM_B200_IO_THREADS");
        const unsigned hw = std::thread::hardware_concurrency();
        g_io_threads = e ? atoi(e) : (int)std::min<unsigned>(hw ? hw : 1, 32);
    }
    RefData refs;
    load_refs(refName + ".seq", false, refs);
    const int M = refs.M;
    const std::vector<Line> lines = read_manifest(manifest, M);

    struct CtxResult { int rc; rsem_b200_ctx* ctx; std::string err; };
    std::future<CtxResult> ctx_future = std::async(std::launch::async, []() {
        CtxResult r{0, nullptr, ""};
        const char* d = getenv("RSEM_B200_DEVICE");
        r.rc = rsem_b200_ctx_create(d ? atoi(d) : 0, &r.ctx);
        if (r.rc != 0) r.err = rsem_b200_last_error();
        return r;
    });
    std::vector<int> gi, gt, ta;
    load_groups(refName + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(refName, gt, ta);
    const size_t acc_per = 4 * ((size_t)M + 1) + (size_t)m;

    Phases ph;
    std::vector<std::string> block(lines.size());
    std::mutex block_mu;
    auto say = [&](size_t i, const std::string& s) {
        if (!verbose) return;
        std::lock_guard<std::mutex> g(block_mu);
        block[i] += s;
    };

    // a sample's inputs (rsem-run-gibbs's load_data, load_omit_info / load_prior_info, init_model_related, init)
    auto load = [&](size_t i) {
        const Line& l = lines[i];
        auto s = std::make_unique<Sample>();
        s->idx = i;
        load_ofg(l.imdName + ".ofg", M, s->N0, s->row_ptr, s->sid, s->conprb);
        s->N1 = s->row_ptr.size() - 1;
        const std::string why = gibbs_inputs(l.imdName, M, s->N0, s->N1, l.pseudoC, l.hasPrior ? &l.fprior : nullptr, s->init_counts,
                                             s->alpha, s->totc);
        if (!why.empty()) die(why);
        int model_type = 0;
        LenDistH gld;
        HostModel::read_for_gibbs(l.statName + ".model", M, model_type, gld, s->mw);
        calc_eel(refs, gld, s->eel);
        s->chain_seeds = engine_seeds(l.hasSeed ? l.seed : (uint32_t)time(NULL), l.nThreads);
        s->chain_samples.resize(l.nThreads);
        const int quotient = l.nsamples / l.nThreads, left = l.nsamples % l.nThreads;
        for (int t = 0; t < l.nThreads; ++t) s->chain_samples[t] = quotient + (t < left ? 1 : 0);
        return s;
    };
    auto params_of = [&](const Sample& s) {
        const Line& l = lines[s.idx];
        rsem_b200_gibbs_params gp;
        memset(&gp, 0, sizeof gp);
        gp.M = M; gp.burnin = l.burnin; gp.gap = l.gap; gp.n_chains = l.nThreads;
        gp.chain_samples = s.chain_samples.data();
        gp.chain_seeds = s.chain_seeds.data();
        gp.n0 = (double)s.N0;
        gp.init_counts = s.init_counts.data();
        gp.pseudo_counts = s.alpha.data();
        gp.totc = s.totc;
        gp.eel = s.eel.data();
        gp.mw = s.mw.data();
        gp.n_genes = m;
        gp.gene_start = gi.data();
        return gp;
    };
    // a sample whose chains have run: the sums of its chains, countvectors<t>, iso_res / gene_res (rsem-run-gibbs from
    // rsem_b200_gibbs_sum_chains on)
    auto finish = [&](const Sample& s, const std::vector<int32_t>& cvs, const std::vector<double>& chain_acc) {
        const Line& l = lines[s.idx];
        std::vector<double> sum_c(M + 1), sum_c2(M + 1), sum_tpm(M + 1), sum_fpkm(M + 1), sum_g2(m);
        rsem_b200_gibbs_out go;
        go.count_vectors = nullptr;
        go.sum_c = sum_c.data(); go.sum_c2 = sum_c2.data(); go.sum_tpm = sum_tpm.data(); go.sum_fpkm = sum_fpkm.data();
        go.sum_gene_c2 = sum_g2.data();
        const rsem_b200_gibbs_params gp = params_of(s);
        check_rc(rsem_b200_gibbs_sum_chains(&gp, chain_acc.data(), &go), "gibbs_sum_chains");
        write_countvectors(l.imdName, M, s.chain_samples, cvs.data());
        say(s.idx, "Gibbs finished!\n");
        write_gibbs_results(refName, l.imdName, M, l.nsamples, gi, alleleS, ta, cvs.data(), sum_c, sum_c2, sum_tpm, sum_fpkm, sum_g2);
        say(s.idx, "Gibbs based expression values are written!\n");
    };

    rsem_b200_ctx* ctx = nullptr;
    {
        CtxResult r = ctx_future.get();
        if (r.rc != 0) die("rsem_b200: ctx_create failed: " + r.err);
        ctx = r.ctx;
    }
    rsem_b200_gibbs_batch* batch = nullptr;
    const char* arena = getenv("RSEM_B200_BATCH_ARENA_BYTES");
    check_rc(rsem_b200_gibbs_batch_create(ctx, arena ? strtoull(arena, nullptr, 10) : 0, 0, &batch), "gibbs_batch_create");

    // the samples in the batch run in one launch; their outputs are copied back one by one and written on worker threads
    std::map<int32_t, std::unique_ptr<Sample>> in_batch;
    const int n_writers = std::max(1, std::min(g_io_threads, 8));
    auto drain = [&]() {
        if (in_batch.empty()) return;
        rsem_b200_gibbs_batch_stats st;
        {
            const double t0 = now_s();
            check_rc(rsem_b200_gibbs_batch_run(batch, &st), "gibbs_batch_run");
            ph.device += now_s() - t0;
        }
        ph.k13_ms += st.device_ms;
        ph.chain_cycles += st.chain_cycles;
        ph.sample_cycles += st.sample_cycles;
        ph.jobs += (uint64_t)st.jobs;
        ph.teams = st.teams;
        ph.workers = st.worker_ctas;
        std::vector<std::pair<int32_t, Sample*>> todo;
        for (auto& kv : in_batch) todo.emplace_back(kv.first, kv.second.get());
        std::atomic<size_t> next{0};
        std::mutex copy_mu;
        std::vector<double> t_copy(n_writers, 0.0), t_write(n_writers, 0.0);
        auto writer = [&](int w) {
            for (size_t k; (k = next.fetch_add(1)) < todo.size();) {
                const Sample& s = *todo[k].second;
                std::vector<int32_t> cvs((size_t)lines[s.idx].nsamples * (M + 1));
                std::vector<double> acc(s.chain_samples.size() * acc_per);
                {
                    std::lock_guard<std::mutex> g(copy_mu);
                    const double t0 = now_s();
                    check_rc(rsem_b200_gibbs_batch_result(batch, todo[k].first, cvs.data(), acc.data()), "gibbs_batch_result");
                    t_copy[w] += now_s() - t0;
                }
                const double t1 = now_s();
                finish(s, cvs, acc);
                t_write[w] += now_s() - t1;
            }
        };
        {
            std::vector<std::thread> pool;
            for (int w = 1; w < n_writers; ++w) pool.emplace_back(writer, w);
            writer(0);
            for (auto& th : pool) th.join();
        }
        for (int w = 0; w < n_writers; ++w) { ph.copy += t_copy[w]; ph.write += t_write[w]; }
        check_rc(rsem_b200_gibbs_batch_clear(batch), "gibbs_batch_clear");
        in_batch.clear();
    };

    // loading runs a few samples ahead of the adds, on host threads
    const size_t ahead = 4;
    std::deque<std::future<std::unique_ptr<Sample>>> loads;
    size_t next_load = 0;
    auto top_up = [&]() {
        while (next_load < lines.size() && loads.size() < ahead) {
            const size_t i = next_load++;
            loads.push_back(std::async(std::launch::async, load, i));
        }
    };
    for (size_t i = 0; i < lines.size(); ++i) {
        const Line& l = lines[i];
        if (verbose) block[i] += "== sample " + l.imdName + " (" + manifest + " line " + std::to_string(l.no) + ")\n";
        top_up();
        const double t_load = now_s();
        std::unique_ptr<Sample> s = loads.front().get();
        loads.pop_front();
        say(i, "Refs.loadRefs finished!\nLoading data is finished!\nLoading group information is finished!\nGibbs started!\nInitialization finished!\n");
        const rsem_b200_gibbs_params gp = params_of(*s);
        int32_t slot = -1;
        int rc = rsem_b200_gibbs_batch_add(batch, s->N1, s->sid.size(), s->row_ptr.data(), s->sid.data(), s->conprb.data(), &gp, &slot);
        ph.load += now_s() - t_load;
        if (rc == RSEM_B200_ERR_FULL) {
            ++ph.full;
            drain();
            const double t0 = now_s();
            rc = rsem_b200_gibbs_batch_add(batch, s->N1, s->sid.size(), s->row_ptr.data(), s->sid.data(), s->conprb.data(), &gp, &slot);
            ph.load += now_s() - t0;
        }
        if (rc == 0) {
            ++ph.batched;
            // the matrix lives in the arena now
            std::vector<uint64_t>().swap(s->row_ptr);
            std::vector<int32_t>().swap(s->sid);
            std::vector<double>().swap(s->conprb);
            in_batch[slot] = std::move(s);
            continue;
        }
        if (rc != RSEM_B200_ERR_UNSUPPORTED && rc != RSEM_B200_ERR_FULL) check_rc(rc, "gibbs_batch_add");
        // outside the batch's size rule (or larger than its whole arena): the single-sample path of rsem-run-gibbs
        ++ph.single;
        const double t0 = now_s();
        check_rc(rsem_b200_gibbs_upload(ctx, s->N1, s->sid.size(), M, s->row_ptr.data(), s->sid.data(), s->conprb.data()), "gibbs_upload");
        std::vector<int32_t> cvs((size_t)l.nsamples * (M + 1));
        std::vector<double> acc(s->chain_samples.size() * acc_per);
        rsem_b200_gibbs_stats gs;
        check_rc(rsem_b200_gibbs_run_chains(ctx, &gp, cvs.data(), acc.data(), &gs), "gibbs_run");
        const double t1 = now_s();
        ph.device += t1 - t0;
        finish(*s, cvs, acc);
        ph.write += now_s() - t1;
    }
    drain();
    if (getenv("RSEM_B200_TIMING")) {
        uint64_t cv_bytes = 0;
        for (const Line& l : lines)
            for (int t = 0; t < l.nThreads; ++t) {
                FILE* f = fopen((l.imdName + ".countvectors" + std::to_string(t)).c_str(), "rb");
                if (!f) continue;
                fseek(f, 0, SEEK_END);
                cv_bytes += (uint64_t)ftell(f);
                fclose(f);
            }
        fprintf(stderr, "rsem-run-gibbs-batch timing: %d samples in the batch, %d on the single-sample path; K13 %.3f ms, %llu jobs, "
                "%d teams of %d worker CTAs, per-kept-draw work %.4f of chain cycles\n", ph.batched, ph.single, ph.k13_ms,
                (unsigned long long)ph.jobs, ph.teams, ph.workers,
                ph.chain_cycles ? (double)ph.sample_cycles / (double)ph.chain_cycles : 0.0);
        fprintf(stderr, "rsem-run-gibbs-batch timing: load+components %.3f s, device %.3f s, copies back %.3f s, writers %.3f s "
                "(thread seconds), count-vector text %llu bytes\n", ph.load, ph.device, ph.copy, ph.write, (unsigned long long)cv_bytes);
        fprintf(stderr, "rsem-run-gibbs-batch timing: arena full %d times\n", ph.full);
    }
    rsem_b200_gibbs_batch_destroy(batch);
    rsem_b200_ctx_destroy(ctx);
    for (const std::string& b : block) fputs(b.c_str(), stdout);
    return 0;
}
