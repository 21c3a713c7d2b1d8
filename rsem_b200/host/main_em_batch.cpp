// rsem-run-em-batch: the EM of many samples against one reference in one process.
//
//   rsem-run-em-batch refName read_type manifest [-p #Threads] [-q]
//
// Each non-empty manifest line is what rsem-run-em takes after read_type:
//   sampleName imdName statName [-b samInpF has_fai [fai]] [--gibbs-out] [--sampling] [--seed s] [--append-names]
// and each sample gets the files `rsem-run-em refName read_type <line> -p N` writes.  A lane (a host thread, a CUDA context
// holding the reference and a batch arena) takes the samples one by one.  A sample runs its model rounds 1-10 on the
// lane's context as in rsem-run-em; from round 11 on, its frozen rounds join the lane's batch (K12, rsem_b200_batch_*) that
// converges every sample in it with one kernel launch per few dozen rounds.  A sample outside the batch layout
// (rsem_b200_batch_sample_bytes) finishes on the context with rsem_b200_em_rounds right after its round 10.  When the
// batch arena is full, the samples in it are run to the end and written before the next one is added; a sample that
// still does not fit then finishes on the context.
// There is one lane on RSEM_B200_DEVICE (default 0), or one per entry of RSEM_B200_DEVICES=0,1,... when it lists more
// than one; an entry may repeat a device (0,0 runs two lanes on device 0 side by side).  The lanes take the manifest lines
// in manifest order from one counter; every sample runs on one CTA or on one context, so its files do not depend on the
// lane that ran it.  RSEM_B200_BATCH_ARENA_BYTES sets each lane's arena (default, or 0: half of the device memory free at
// the start, shared evenly by the lanes on one device).  The first failure of any lane ends the run with exit status
// -1 once the other lanes have finished their current samples.  Standard output has one block per sample, in manifest
// order.
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <future>
#include <map>
#include <memory>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

struct Line : EmArgs {
    int no = 0;   // 1-based line number in the manifest
    EmCounts n;
};

// a sample from its hand-over to the batch until its outputs are written
struct Pending {
    size_t idx = 0;
    EmSample s;
    EmRounds r;
};

void usage() {
    printf("Usage : rsem-run-em-batch refName read_type manifest [-p #Threads] [-q]\n\n");
    printf("  refName: reference name\n");
    printf("  read_type: 0 single read without quality score; 1 single read with quality score; 2 paired-end read without quality score; 3 paired-end read with quality score.\n");
    printf("  manifest: one sample per line: sampleName imdName statName [-b samInpF has_fai? [fai_file]] [--gibbs-out] [--sampling] [--seed seed] [--append-names]\n");
    printf("  -p: number of threads which user wants to use. (default: 1)\n");
    printf("  -q: set it quiet\n");
    exit(-1);
}

// RSEM_B200_TIMING=1: wall seconds per phase, summed over the samples, on stderr at the end
struct Phases {
    double load = 0, model = 0, frozen = 0, final = 0, write = 0;
};
struct Timed {
    double& acc;
    double t0 = now_s();
    ~Timed() { acc += now_s() - t0; }
};

// every manifest line is checked before the context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, int read_type) {
    std::vector<Line> lines;
    std::map<std::string, int> seen[3];
    for (const ManifestLine& ml : manifest_lines(path)) {
        const int no = ml.no;
        if (ml.f.size() < 3) refuse(path, no, "too few fields (sampleName imdName statName [options])");
        Line l;
        static_cast<EmArgs&>(l) = parse_em_args(ml.f);   // -p and -q are the run's, not the line's
        l.no = no;
        const std::string names[3] = {l.statName, l.imdName, l.outName};
        const char* what[3] = {"statName", "imdName", "sampleName"};
        for (int k = 0; k < 3; ++k) {
            auto it = seen[k].find(names[k]);
            if (it != seen[k].end())
                refuse(path, no, std::string("its outputs collide with line ") + std::to_string(it->second) + " (same " + what[k] + ")");
            seen[k][names[k]] = no;
        }
        if (!load_cnt(l.statName, false, l.n)) refuse(path, no, "cannot read or parse " + l.statName + ".cnt");
        if (l.n.N1 > 0) {
            FILE* fi = fopen((l.imdName + ".dat").c_str(), "r");
            if (fi) {
                long long n1 = 0, nh = 0, rt = -1;
                const int got = fscanf(fi, "%lld %lld %lld", &n1, &nh, &rt);
                fclose(fi);
                if (got != 3 || rt != read_type)
                    refuse(path, no, l.imdName + ".dat does not have the right read type (" + std::to_string(read_type) + ")");
            }
        }
        lines.push_back(l);
    }
    return lines;
}

// what every lane reads
struct Run {
    std::string manifest;
    int read_type = 0, nThreads = 1, MAX_ROUND = 10000, MIN_ROUND = 20;
    std::vector<Line> lines;
    EmReference ref;
    std::vector<std::string> block;   // standard output of each sample, written by the lane that took it
};

struct Lane {
    int device = 0;
    rsem_b200_ctx* ctx = nullptr;
    uint64_t arena = 0;
    rsem_b200_batch* batch = nullptr;
    std::string where = "no sample yet";   // what the lane is working on, for the failure message
    int n_batched = 0, n_single = 0, n_full = 0;   // samples whose frozen rounds ran in the batch / on the context; full arenas
    double k12_ms = 0;
    uint64_t k12_rounds = 0;
    Phases ph;
};

// the samples a lane takes from `claims`, loaded, run and written on the lane's context and batch
void run_lane(Run& R, Lane& L, Claims& claims) {
    const std::vector<Line>& lines = R.lines;
    const std::string& manifest = R.manifest;
    const int read_type = R.read_type, MIN_ROUND = R.MIN_ROUND, MAX_ROUND = R.MAX_ROUND;
    const RefData& refs = R.ref.refs;
    const int M = refs.M;
    rsem_b200_ctx* ctx = L.ctx;
    check_rc(rsem_b200_upload_refs(ctx, M, refs.seq_off.data(), refs.seq.data(), refs.full_len.data(), refs.tot_len.data(),
                                   refs.mask_off.data(), refs.mask_words.data()), "upload_refs");
    check_rc(rsem_b200_batch_create(ctx, L.arena, &L.batch), "batch_create");
    rsem_b200_batch* batch = L.batch;
    Phases& ph = L.ph;
    std::vector<std::string>& block = R.block;
    auto say = [&](size_t i, const std::string& s) { if (g_verbose) block[i] += s; };
    auto sample_of = [&](size_t i) { return sample_at(lines[i].outName, manifest, lines[i].no); };

    // outputs of a sample whose EM has ended
    auto finish = [&](Pending& p) {
        const Line& l = lines[p.idx];
        Timed tw{ph.write};
        finish_em_sample(R.ref, read_type, l, p.s, p.r.totNum, MAX_ROUND, l.outName + ": ", R.nThreads, false);
        if (l.genBam) {
            if (l.bamSampling) say(p.idx, "Begin to sample reads from their posteriors.\nSampling is finished.\n");
            say(p.idx, "Bam output file is generated!\n");
        }
    };

    std::map<int32_t, std::unique_ptr<Pending>> in_batch;   // slot -> sample
    const int CHUNK = 64;
    auto drain = [&]() {
        while (!in_batch.empty()) {
            int32_t n_slots = 0;
            check_rc(rsem_b200_batch_slots(batch, &n_slots), "batch_slots");
            std::vector<rsem_b200_round_stats> st((size_t)n_slots * CHUNK);
            std::vector<int32_t> ran(n_slots), stopped(n_slots);
            L.where = "the batch of its " + std::to_string(in_batch.size()) + " samples";
            {
                Timed tk{ph.frozen};
                check_rc(rsem_b200_batch_run(batch, CHUNK, st.data(), ran.data(), stopped.data()), "batch_run");
            }
            for (auto it = in_batch.begin(); it != in_batch.end();) {
                const int32_t slot = it->first;
                Pending& p = *it->second;
                for (int r = 0; r < ran[slot]; ++r) say(p.idx, round_line(p.r.round + 1 + r, st[(size_t)slot * CHUNK + r]));
                if (ran[slot] > 0) { p.r.round += ran[slot]; p.r.totNum = st[(size_t)slot * CHUNK + ran[slot] - 1].totnum; }
                if (!stopped[slot]) { ++it; continue; }
                L.where = sample_of(p.idx);
                EmSample& s = p.s;
                const bool genBam = lines[p.idx].genBam;
                s.counts.assign(M + 1, 0.0);
                if (genBam) { s.post.resize(s.hits.H); s.post0.resize(s.hits.N); }
                {
                    Timed tf{ph.final};
                    check_rc(rsem_b200_batch_final(batch, slot, s.theta.data(), s.counts.data(), genBam ? s.post.data() : nullptr,
                                                   genBam ? s.post0.data() : nullptr), "batch_final");
                    check_rc(rsem_b200_batch_remove(batch, slot), "batch_remove");
                }
                finish(p);
                it = in_batch.erase(it);
            }
        }
    };

    for (size_t i; (i = claims.next()) < lines.size();) {
        L.where = sample_of(i);
        const Line& l = lines[i];
        if (g_verbose || l.n.N1 == 0) block[i] += "== " + sample_of(i) + "\n";
        if (l.n.N1 == 0) {
            write_no_alignable_reads(R.ref, l, [&](const std::string& s) { block[i] += s; });
            continue;
        }
        const double t_load = now_s();
        auto p = std::make_unique<Pending>();
        p->idx = i;
        EmSample& s = p->s;
        s.n = l.n;
        load_em_hits(l.imdName, read_type, M, s);
        for (int32_t t : s.hits.sid)   // the reference of the run is refName's, not the one this sample was aligned to
            if (t == 0 || std::abs(t) > M)
                refuse(manifest, l.no, "an alignment names transcript " + std::to_string(t) + ", outside " + R.ref.name + " (M = " + std::to_string(M) + ")");
        ReadStore reads;
        load_em_model(l.imdName, read_type, refs, s, reads, [&](const std::string& x) { say(i, x); });
        ph.load += now_s() - t_load;
        const double t_model = now_s();

        const HitStore& hits = s.hits;
        check_rc(rsem_b200_upload_hits(ctx, hits.N, hits.H, M, hits.row_ptr.data(), hits.sid.data(), hits.pos.data(),
                                       read_type >= 2 ? hits.insertL.data() : nullptr), "upload_hits");
        check_rc(rsem_b200_upload_reads(ctx, reads.n_mates, reads.off[0].data(), reads.base[0].data(),
                                        reads.has_qual ? reads.qual[0].data() : nullptr,
                                        reads.n_mates == 2 ? reads.off[1].data() : nullptr,
                                        reads.n_mates == 2 ? reads.base[1].data() : nullptr,
                                        (reads.n_mates == 2 && reads.has_qual) ? reads.qual[1].data() : nullptr,
                                        reads.lowq.data()), "upload_reads");
        check_rc(rsem_b200_set_theta(ctx, s.theta.data()), "set_theta");

        // rounds 1-10 update the model, on the context as in rsem-run-em
        EmRounds& r = p->r;
        r = em_model_rounds(ctx, s.model, l.n.N0, MIN_ROUND, MAX_ROUND, [&](int round, const rsem_b200_round_stats& rs) {
            say(i, round_line(round, rs));
        });
        s.conprb.resize(hits.H);
        s.ncpv.resize(hits.N);
        check_rc(rsem_b200_download_conprb(ctx, s.conprb.data(), s.ncpv.data()), "download_conprb");
        ph.model += now_s() - t_model;
        if (r.keep_going) {   // round 11 on: the batch, or this context when the sample is outside the batch layout
            check_rc(rsem_b200_get_theta(ctx, s.theta.data()), "get_theta");
            auto add = [&](int32_t* slot) {
                return rsem_b200_batch_add(batch, hits.N, hits.H, M, hits.row_ptr.data(), hits.sid.data(), s.conprb.data(),
                                           s.ncpv.data(), s.theta.data(), (double)l.n.N0, r.round + 1, MIN_ROUND, MAX_ROUND, slot);
            };
            int32_t slot = -1;
            int rc = add(&slot);
            if (rc == RSEM_B200_ERR_FULL) {
                ++L.n_full;
                drain();
                rc = add(&slot);
            }
            if (rc == 0) {
                ++L.n_batched;
                in_batch[slot] = std::move(p);
                continue;
            }
            if (rc != RSEM_B200_ERR_UNSUPPORTED && rc != RSEM_B200_ERR_FULL) check_rc(rc, "batch_add");
            ++L.n_single;
            Timed tk{ph.frozen};
            em_frozen_rounds(ctx, l.n.N0, MIN_ROUND, MAX_ROUND, r, [&](int round, const rsem_b200_round_stats& rs) {
                say(i, round_line(round, rs));
            });
        }
        // final pass on the context (EM.cpp:460-478)
        const double t_final = now_s();
        s.counts.assign(M + 1, 0.0);
        check_rc(rsem_b200_get_theta(ctx, s.theta.data()), "get_theta");
        check_rc(rsem_b200_expected_weights(ctx, s.counts.data()), "expected_weights");
        if (l.genBam) {
            s.post.resize(hits.H);
            s.post0.resize(hits.N);
            check_rc(rsem_b200_download_conprb(ctx, s.post.data(), s.post0.data()), "download_conprb");
        }
        ph.final += now_s() - t_final;
        finish(*p);
    }
    drain();
    check_rc(rsem_b200_batch_timing(batch, &L.k12_ms, &L.k12_rounds), "batch_timing");
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 4) usage();
    const time_t t_start = time(NULL);
    Run R;
    const std::string refName = argv[1];
    R.manifest = argv[3];
    R.read_type = atoi(argv[2]);
    for (int i = 4; i < argc; ++i) {
        if (!strcmp(argv[i], "-p") && i + 1 < argc) R.nThreads = atoi(argv[i + 1]);
        if (!strcmp(argv[i], "-q")) g_verbose = false;
    }
    if (R.nThreads <= 0) die("Number of threads should be bigger than 0!");
    g_io_threads = env_int("RSEM_B200_IO_THREADS", R.nThreads);
    if (R.read_type < 0 || R.read_type > 3) { fprintf(stderr, "Unknown Read Type!\n"); exit(-1); }
    R.lines = read_manifest(R.manifest, R.read_type);
    R.MAX_ROUND = env_int("RSEM_MAX_ROUND", 10000);
    R.MIN_ROUND = env_int("RSEM_MIN_ROUND", 20);

    const std::vector<int> devices = gpu_devices();
    std::future<LaneContexts> ctx_future = std::async(std::launch::async, open_lanes, devices);
    load_em_reference(refName, R.ref);
    std::vector<Lane> lanes(devices.size());
    {
        const LaneContexts lc = ctx_future.get();
        if (!lc.err.empty()) die(lc.err);
        for (size_t k = 0; k < lanes.size(); ++k) {
            lanes[k].device = devices[k];
            lanes[k].ctx = lc.ctx[k];
            lanes[k].arena = lc.arena[k];
        }
    }
    R.block.resize(R.lines.size());
    Claims claims(R.lines.size());
    run_lanes("rsem-run-em-batch", lanes, claims, [&](Lane& L) { run_lane(R, L, claims); });
    if (getenv("RSEM_B200_TIMING")) {
        Lane t;   // the totals
        for (const Lane& L : lanes) {
            t.n_batched += L.n_batched; t.n_single += L.n_single; t.n_full += L.n_full;
            t.k12_ms += L.k12_ms; t.k12_rounds += L.k12_rounds;
            t.ph.load += L.ph.load; t.ph.model += L.ph.model; t.ph.frozen += L.ph.frozen; t.ph.final += L.ph.final;
            t.ph.write += L.ph.write;
        }
        fprintf(stderr, "rsem-run-em-batch timing: %d samples in the batch, %d on the single-sample path; K12 %.3f ms over %llu "
                "sample-rounds\n", t.n_batched, t.n_single, t.k12_ms, (unsigned long long)t.k12_rounds);
        fprintf(stderr, "rsem-run-em-batch timing: arena full %d times\n", t.n_full);
        fprintf(stderr, "rsem-run-em-batch timing: load %.3f s, model rounds %.3f s, frozen rounds %.3f s, final pass %.3f s, "
                "writers %.3f s\n", t.ph.load, t.ph.model, t.ph.frozen, t.ph.final, t.ph.write);
        if (lanes.size() > 1)
            for (size_t k = 0; k < lanes.size(); ++k) {
                const Lane& L = lanes[k];
                fprintf(stderr, "rsem-run-em-batch timing: lane %zu, device %d: %d samples in the batch, %d on the single-sample "
                        "path, arena full %d times; K12 %.3f ms; model rounds %.3f s, frozen rounds %.3f s, final pass %.3f s\n", k,
                        L.device, L.n_batched, L.n_single, L.n_full, L.k12_ms, L.ph.model, L.ph.frozen, L.ph.final);
            }
    }
    for (Lane& L : lanes) {
        rsem_b200_batch_destroy(L.batch);
        rsem_b200_ctx_destroy(L.ctx);
    }
    for (const std::string& b : R.block) fputs(b.c_str(), stdout);
    fputs(time_used_line(t_start).c_str(), stdout);
    return 0;
}
