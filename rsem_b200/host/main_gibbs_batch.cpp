// rsem-run-gibbs-batch: the Gibbs samplers of many samples against one reference in one process.
//
//   rsem-run-gibbs-batch refName manifest [-q]
//
// Each non-empty manifest line is what rsem-run-gibbs takes after reference_name:
//   imdName statName BURNIN NSAMPLES GAP [-p #chains] [--seed s] [--pseudo-count c] [--prior file]
// and each line gets the files `rsem-run-gibbs refName <line>` writes.  A lane (a host thread, a CUDA context and a batch
// arena) takes the samples one by one.  A sample of 1248 .. 2^19 reads joins the lane's Gibbs batch (K13,
// rsem_b200_gibbs_batch_*), which runs the chains of all its samples in one launch; any other sample runs on the lane's
// context with rsem_b200_gibbs_upload + rsem_b200_gibbs_run_chains, as in rsem-run-gibbs.  When the batch arena is full,
// the samples in it are run and written before the next one is added; a sample that still does not fit then runs on the
// context.
// There is one lane on RSEM_B200_DEVICE (default 0), or one per entry of RSEM_B200_DEVICES=0,1,... when it lists more
// than one; an entry may repeat a device (0,0 runs two lanes on device 0, whose host stages overlap).  The lanes take the
// manifest lines in manifest order from one counter; a chain's draws depend only on its seed and its sample, so the files
// do not depend on the lane that ran it.  Both kinds of launch are cooperative grids sized to a whole device, so the lanes
// on one device take turns: a per-device mutex is held from before each launch until its stream has finished it.
// RSEM_B200_BATCH_ARENA_BYTES sets each lane's arena (default, or 0: half of the device memory free at the start, shared
// evenly by the lanes on one device).  The first failure of any lane ends the run with exit status -1 once the other lanes
// have finished their current samples.  Standard output has one block per sample, in manifest order.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <future>
#include <map>
#include <memory>
#include <mutex>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

struct Line : GibbsArgs {
    int no = 0;   // 1-based line number in the manifest
};

// a loaded sample, from its .ofg to its written outputs
struct Sample : GibbsSample {
    size_t idx = 0;
};

void usage() {
    printf("Usage: rsem-run-gibbs-batch refName manifest [-q]\n\n");
    printf("  refName: reference name\n");
    printf("  manifest: one sample per line: imdName statName BURNIN NSAMPLES GAP [-p #Threads] [--seed seed] [--pseudo-count pseudo_count] [--prior file]\n");
    printf("  -q: set it quiet\n");
    exit(-1);
}

// every manifest line is checked before the context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, int M) {
    std::vector<Line> lines;
    std::map<std::string, int> seen;
    for (const ManifestLine& ml : manifest_lines(path)) {
        const int no = ml.no;
        if (ml.f.size() < 5) refuse(path, no, "too few fields (imdName statName BURNIN NSAMPLES GAP [options])");
        Line l;
        l.no = no;
        const std::string why = parse_gibbs_args(ml.f, l);
        if (!why.empty()) refuse(path, no, why);
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
        clamp_gibbs_chains(l);
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

// what every lane reads
struct Run {
    std::string refName, manifest;
    bool verbose = true;
    int M = 0;
    size_t acc_per = 0;
    bool alleleS = false;
    std::vector<Line> lines;
    RefData refs;
    std::vector<int> gi, gt, ta;
    std::vector<std::string> block;   // standard output of each sample
    std::mutex block_mu;
};

struct Lane {
    int device = 0;
    rsem_b200_ctx* ctx = nullptr;
    uint64_t arena = 0;
    rsem_b200_gibbs_batch* batch = nullptr;
    std::mutex* launch_mu = nullptr;   // shared by the lanes on this device
    bool isolated = false;             // die() throws on the lane's threads (more than one lane)
    std::string where = "no sample yet";   // what the lane is working on, for the failure message
    Phases ph;
    std::vector<std::pair<double, double>> launches;   // host clock around every cooperative launch, under launch_mu
};

// the samples a lane takes from `claims`, loaded, run and written on the lane's context and batch
void run_lane(Run& R, Lane& L, Claims& claims) {
    const std::vector<Line>& lines = R.lines;
    const std::string& refName = R.refName;
    const int M = R.M;
    const size_t acc_per = R.acc_per;
    const RefData& refs = R.refs;
    const std::vector<int>& gi = R.gi;
    const std::vector<int>& ta = R.ta;
    const bool alleleS = R.alleleS, verbose = R.verbose;
    rsem_b200_ctx* ctx = L.ctx;
    Phases& ph = L.ph;
    check_rc(rsem_b200_gibbs_batch_create(ctx, L.arena, 0, &L.batch), "gibbs_batch_create");
    rsem_b200_gibbs_batch* batch = L.batch;
    auto say = [&](size_t i, const std::string& s) {
        if (!verbose) return;
        std::lock_guard<std::mutex> g(R.block_mu);
        R.block[i] += s;
    };
    auto sample_of = [&](size_t i) { return sample_at(lines[i].imdName, R.manifest, lines[i].no); };
    // a cooperative launch: one at a time per device
    auto launch = [&](const auto& run) {
        std::lock_guard<std::mutex> g(*L.launch_mu);
        const double t0 = now_s();
        run();
        L.launches.emplace_back(t0, now_s());
    };

    // a sample's inputs, with the progress lines of rsem-run-gibbs; the reference and its groups are the run's
    auto load = [&](size_t i) {
        DieThrows throws(L.isolated);
        auto s = std::make_unique<Sample>();
        s->idx = i;
        auto say_i = [&](const std::string& x) { say(i, x); };
        say_i("Refs.loadRefs finished!\n");
        load_gibbs_ofg(lines[i], M, *s, say_i);
        say_i("Loading group information is finished!\n");
        load_gibbs_inputs(lines[i], refs, *s, say_i);
        return s;
    };
    // a sample whose chains have run
    auto finish = [&](const Sample& s, const std::vector<int32_t>& cvs, const std::vector<double>& chain_acc) {
        finish_gibbs_sample(refName, lines[s.idx], s, gi, alleleS, ta, cvs.data(), chain_acc.data(),
                            [&](const std::string& x) { say(s.idx, x); });
        say(s.idx, "Gibbs based expression values are written!\n");
    };

    // the samples in the batch run in one launch; their outputs are copied back one by one and written on worker threads
    std::map<int32_t, std::unique_ptr<Sample>> in_batch;
    const int n_writers = std::max(1, std::min(g_io_threads, 8));
    auto drain = [&]() {
        if (in_batch.empty()) return;
        rsem_b200_gibbs_batch_stats st;
        {
            L.where = "the batch of its " + std::to_string(in_batch.size()) + " samples";
            const double t0 = now_s();
            launch([&]() { check_rc(rsem_b200_gibbs_batch_run(batch, &st), "gibbs_batch_run"); });
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
        std::exception_ptr failed;   // a writer's first failure, raised on the lane's thread once every writer has stopped
        auto writer = [&](int w) {
            DieThrows throws(L.isolated);
            for (size_t k; (k = next.fetch_add(1)) < todo.size();) try {
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
            } catch (...) {
                std::lock_guard<std::mutex> g(copy_mu);
                if (!failed) { failed = std::current_exception(); L.where = sample_of(todo[k].second->idx); }
                next = todo.size();
            }
        };
        {
            std::vector<std::thread> pool;
            for (int w = 1; w < n_writers; ++w) pool.emplace_back(writer, w);
            writer(0);
            for (auto& th : pool) th.join();
        }
        if (failed) std::rethrow_exception(failed);
        for (int w = 0; w < n_writers; ++w) { ph.copy += t_copy[w]; ph.write += t_write[w]; }
        check_rc(rsem_b200_gibbs_batch_clear(batch), "gibbs_batch_clear");
        in_batch.clear();
    };

    // loading runs a few samples ahead of the adds, on host threads; with several lanes, whose loads overlap anyway, one
    // line ahead, so that a lane holds few lines the others could take
    const size_t ahead = L.isolated ? 2 : 4;
    std::deque<std::pair<size_t, std::future<std::unique_ptr<Sample>>>> loads;
    auto top_up = [&]() {
        while (loads.size() < ahead) {
            const size_t i = claims.next();
            if (i >= lines.size()) break;
            loads.emplace_back(i, std::async(std::launch::async, load, i));
        }
    };
    for (top_up(); !loads.empty(); top_up()) {
        const size_t i = loads.front().first;
        L.where = sample_of(i);
        const Line& l = lines[i];
        const double t_load = now_s();
        std::unique_ptr<Sample> s = loads.front().second.get();
        loads.pop_front();
        const rsem_b200_gibbs_params gp = gibbs_params(l, *s, gi);
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
        launch([&]() { check_rc(rsem_b200_gibbs_run_chains(ctx, &gp, cvs.data(), acc.data(), &gs), "gibbs_run"); });
        const double t1 = now_s();
        ph.device += t1 - t0;
        finish(*s, cvs, acc);
        ph.write += now_s() - t1;
    }
    drain();
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 3) usage();
    Run R;
    R.refName = argv[1];
    R.manifest = argv[2];
    for (int i = 3; i < argc; ++i)
        if (!strcmp(argv[i], "-q")) R.verbose = false;
    g_verbose = false;   // the messages of the shared loaders and writers go into the samples' blocks instead
    {   // as rsem-run-gibbs: file parsing and writing use the host's cores
        const unsigned hw = std::thread::hardware_concurrency();
        g_io_threads = env_int("RSEM_B200_IO_THREADS", (int)std::min<unsigned>(hw ? hw : 1, 32));
    }
    load_refs(R.refName + ".seq", false, R.refs);
    R.M = R.refs.M;
    R.lines = read_manifest(R.manifest, R.M);

    const std::vector<int> devices = gpu_devices();
    std::future<LaneContexts> ctx_future = std::async(std::launch::async, open_lanes, devices);
    load_groups(R.refName + ".grp", R.gi);
    R.alleleS = load_allele_groups(R.refName, R.gt, R.ta);
    R.acc_per = 4 * ((size_t)R.M + 1) + R.gi.size() - 1;
    R.block.resize(R.lines.size());
    if (R.verbose)
        for (size_t i = 0; i < R.lines.size(); ++i)
            R.block[i] = "== " + sample_at(R.lines[i].imdName, R.manifest, R.lines[i].no) + "\n";

    std::vector<Lane> lanes(devices.size());
    std::map<int, std::mutex> launch_mu;
    {
        const LaneContexts lc = ctx_future.get();
        if (!lc.err.empty()) die(lc.err);
        for (size_t k = 0; k < lanes.size(); ++k) {
            lanes[k].device = devices[k];
            lanes[k].ctx = lc.ctx[k];
            lanes[k].arena = lc.arena[k];
            lanes[k].launch_mu = &launch_mu[devices[k]];
            lanes[k].isolated = lanes.size() > 1;
        }
    }
    Claims claims(R.lines.size());
    run_lanes("rsem-run-gibbs-batch", lanes, claims, [&](Lane& L) { run_lane(R, L, claims); });
    if (getenv("RSEM_B200_TIMING")) {
        Phases ph;   // the totals
        for (const Lane& L : lanes) {
            ph.load += L.ph.load; ph.device += L.ph.device; ph.copy += L.ph.copy; ph.write += L.ph.write;
            ph.k13_ms += L.ph.k13_ms; ph.chain_cycles += L.ph.chain_cycles; ph.sample_cycles += L.ph.sample_cycles;
            ph.jobs += L.ph.jobs; ph.batched += L.ph.batched; ph.single += L.ph.single; ph.full += L.ph.full;
            if (L.ph.teams) { ph.teams = L.ph.teams; ph.workers = L.ph.workers; }
        }
        uint64_t cv_bytes = 0;
        for (const Line& l : R.lines)
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
        if (lanes.size() > 1)
            for (size_t k = 0; k < lanes.size(); ++k) {   // launches: start-end of each, host monotonic clock in seconds
                const Lane& L = lanes[k];
                std::string stamps;
                char buf[64];
                for (const auto& t : L.launches) {
                    snprintf(buf, sizeof buf, " %.6f-%.6f", t.first, t.second);
                    stamps += buf;
                }
                fprintf(stderr, "rsem-run-gibbs-batch timing: lane %zu, device %d: %d samples in the batch, %d on the single-sample "
                        "path, arena full %d times; device %.3f s; launches%s\n", k, L.device, L.ph.batched, L.ph.single, L.ph.full,
                        L.ph.device, stamps.c_str());
            }
    }
    for (Lane& L : lanes) {
        rsem_b200_gibbs_batch_destroy(L.batch);
        rsem_b200_ctx_destroy(L.ctx);
    }
    for (const std::string& b : R.block) fputs(b.c_str(), stdout);
    return 0;
}
