// rsem-run-em-batch: the EM of many samples against one reference in one process.
//
//   rsem-run-em-batch refName read_type manifest [-p #Threads] [-q]
//
// Each non-empty manifest line is what rsem-run-em takes after read_type:
//   sampleName imdName statName [-b samInpF has_fai [fai]] [--gibbs-out] [--sampling] [--seed s] [--append-names]
// and each sample gets the files `rsem-run-em refName read_type <line> -p N` writes.  One CUDA context serves the whole
// run; the reference is uploaded once.  A sample runs its model rounds 1-10 on the context as in rsem-run-em; from round
// 11 on, its frozen rounds join a batch (K12, rsem_b200_batch_*) that converges every sample in it with one kernel
// launch per few dozen rounds.  A sample outside the batch layout (rsem_b200_batch_sample_bytes) finishes on the context
// with rsem_b200_em_rounds right after its round 10.  When the batch arena is full, the samples in it are run to the end
// and written before the next one is added; a sample that still does not fit then finishes on the context.
// RSEM_B200_BATCH_ARENA_BYTES sets the arena's size (default, or 0: half of the device memory free at the start).
// Standard output has one block per sample, in manifest order.
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <future>
#include <map>
#include <memory>
#include <sstream>

#include "host.hpp"

using namespace host;

namespace {

struct Line {
    int no = 0;   // 1-based line number in the manifest
    std::string outName, imdName, statName, inpSamF;
    bool genBam = false, bamSampling = false, gibbsOut = false, hasSeed = false, appendNames = false;
    uint32_t seed = 0;
    uint64_t N0 = 0, N1 = 0, N2 = 0, N_tot = 0;
};

// a sample from its hand-over to the batch until its outputs are written
struct Pending {
    size_t idx = 0;
    HitStore hits;
    HostModel model;
    std::vector<double> conprb, ncpv;
    int round = 10;
    long long totNum = 0;
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

[[noreturn]] void refuse(const std::string& manifest, int no, const std::string& why) {
    fprintf(stderr, "%s line %d: %s\n", manifest.c_str(), no, why.c_str());
    exit(-1);
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// RSEM_B200_TIMING=1: wall seconds per phase, summed over the samples, on stderr at the end
struct Phases {
    double load = 0, model = 0, frozen = 0, final = 0, write = 0;
};
struct Timed {
    double& acc;
    double t0 = now_s();
    ~Timed() { acc += now_s() - t0; }
};

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

uint64_t env_bytes(const char* name) {   // 0 when unset
    const char* v = getenv(name);
    return v ? strtoull(v, nullptr, 10) : 0;
}

std::string round_line(int round, const rsem_b200_round_stats& s) {
    char buf[160];
    snprintf(buf, sizeof buf, "ROUND = %d, SUM = %.15g, bChange = %.6g, totNum = %lld\n", round, s.sum, s.bchange,
             (long long)s.totnum);
    return buf;
}

// every manifest line is checked before the context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, int read_type) {
    std::vector<char> buf = slurp(path);
    std::string text(buf.begin(), buf.end());
    std::istringstream in(text);
    std::vector<Line> lines;
    std::map<std::string, int> seen[3];
    std::string raw;
    for (int no = 1; std::getline(in, raw); ++no) {
        std::istringstream ls(raw);
        std::vector<std::string> f;
        for (std::string w; ls >> w;) f.push_back(w);
        if (f.empty()) continue;
        if (f.size() < 3) refuse(path, no, "too few fields (sampleName imdName statName [options])");
        Line l;
        l.no = no;
        l.outName = f[0];
        l.imdName = f[1];
        l.statName = f[2];
        for (size_t i = 3; i < f.size(); ++i) {   // the option rules of rsem-run-em
            if (f[i] == "-b" && i + 1 < f.size()) { l.genBam = true; l.inpSamF = f[i + 1]; }
            if (f[i] == "--gibbs-out") l.gibbsOut = true;
            if (f[i] == "--sampling") l.bamSampling = true;
            if (f[i] == "--seed" && i + 1 < f.size()) { l.hasSeed = true; l.seed = parse_seed(f[i + 1].c_str()); }
            if (f[i] == "--append-names") l.appendNames = true;
        }
        const std::string names[3] = {l.statName, l.imdName, l.outName};
        const char* what[3] = {"statName", "imdName", "sampleName"};
        for (int k = 0; k < 3; ++k) {
            auto it = seen[k].find(names[k]);
            if (it != seen[k].end())
                refuse(path, no, std::string("its outputs collide with line ") + std::to_string(it->second) + " (same " + what[k] + ")");
            seen[k][names[k]] = no;
        }
        std::vector<char> cnt = slurp(l.statName + ".cnt", false);
        cnt.push_back(0);
        unsigned long long v[4];
        if (cnt.size() < 2 || sscanf(cnt.data(), "%llu %llu %llu %llu", &v[0], &v[1], &v[2], &v[3]) != 4)
            refuse(path, no, "cannot read or parse " + l.statName + ".cnt");
        l.N0 = v[0]; l.N1 = v[1]; l.N2 = v[2]; l.N_tot = v[3];
        if (l.N1 > 0) {
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

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 4) usage();
    const time_t t_start = time(NULL);
    const std::string refName = argv[1], manifest = argv[3];
    const int read_type = atoi(argv[2]);
    int nThreads = 1;
    for (int i = 4; i < argc; ++i) {
        if (!strcmp(argv[i], "-p") && i + 1 < argc) nThreads = atoi(argv[i + 1]);
        if (!strcmp(argv[i], "-q")) g_verbose = false;
    }
    if (nThreads <= 0) die("Number of threads should be bigger than 0!");
    g_io_threads = env_int("RSEM_B200_IO_THREADS", nThreads);
    if (read_type < 0 || read_type > 3) { fprintf(stderr, "Unknown Read Type!\n"); exit(-1); }
    std::vector<Line> lines = read_manifest(manifest, read_type);
    const int MAX_ROUND = env_int("RSEM_MAX_ROUND", 10000), MIN_ROUND = env_int("RSEM_MIN_ROUND", 20);

    struct CtxResult { int rc; rsem_b200_ctx* ctx; std::string err; };
    std::future<CtxResult> ctx_future = std::async(std::launch::async, []() {
        CtxResult r{0, nullptr, ""};
        r.rc = rsem_b200_ctx_create(env_int("RSEM_B200_DEVICE", 0), &r.ctx);
        if (r.rc != 0) r.err = rsem_b200_last_error();
        return r;
    });
    RefData refs;
    load_refs(refName + ".seq", true, refs);
    const int M = refs.M;
    std::vector<TranscriptInfo> transcripts;
    int ti_type = 0;
    load_transcripts(refName + ".ti", transcripts, &ti_type);
    rsem_b200_ctx* ctx = nullptr;
    {
        CtxResult r = ctx_future.get();
        if (r.rc != 0) die("rsem_b200: ctx_create failed: " + r.err);
        ctx = r.ctx;
    }
    check_rc(rsem_b200_upload_refs(ctx, M, refs.seq_off.data(), refs.seq.data(), refs.full_len.data(), refs.tot_len.data(),
                                   refs.mask_off.data(), refs.mask_words.data()), "upload_refs");
    rsem_b200_batch* batch = nullptr;
    check_rc(rsem_b200_batch_create(ctx, env_bytes("RSEM_B200_BATCH_ARENA_BYTES"), &batch), "batch_create");
    int n_batched = 0, n_single = 0, n_full = 0;   // samples whose frozen rounds ran in the batch / on the context; full arenas

    Phases ph;
    std::vector<std::string> block(lines.size());
    auto say = [&](size_t i, const std::string& s) { if (g_verbose) block[i] += s; };

    // outputs of a sample whose EM has ended: counts without N0, posteriors only with -b
    auto finish = [&](size_t i, const HitStore& hits, const HostModel& model, const std::vector<double>& theta,
                      std::vector<double> counts, std::vector<double>& post, const std::vector<double>& post0,
                      const std::vector<double>& conprb, const std::vector<double>& ncpv, long long totNum) {
        const Line& l = lines[i];
        Timed tw{ph.write};
        if (totNum > 0)
            fprintf(stderr, "%s: Warning: RSEM reaches %d iterations before meeting the convergence criteria.\n",
                    l.outName.c_str(), MAX_ROUND);
        if (l.gibbsOut) write_ofg(l.imdName + ".ofg", M, l.N0, hits, conprb, ncpv);
        counts[0] += l.N0;
        write_em_outputs(refName, l.imdName, l.statName, refs, transcripts, model, theta, counts, l.appendNames);
        if (l.genBam) {
            write_posterior_bam(l.inpSamF, l.outName, read_type, l.bamSampling, l.hasSeed, l.seed, transcripts, ti_type,
                                hits, post, post0, nThreads, false);
            if (l.bamSampling) say(i, "Begin to sample reads from their posteriors.\nSampling is finished.\n");
            say(i, "Bam output file is generated!\n");
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
            {
                Timed tk{ph.frozen};
                check_rc(rsem_b200_batch_run(batch, CHUNK, st.data(), ran.data(), stopped.data()), "batch_run");
            }
            for (auto it = in_batch.begin(); it != in_batch.end();) {
                const int32_t s = it->first;
                Pending& p = *it->second;
                for (int r = 0; r < ran[s]; ++r) say(p.idx, round_line(p.round + 1 + r, st[(size_t)s * CHUNK + r]));
                if (ran[s] > 0) { p.round += ran[s]; p.totNum = st[(size_t)s * CHUNK + ran[s] - 1].totnum; }
                if (!stopped[s]) { ++it; continue; }
                const Line& l = lines[p.idx];
                std::vector<double> theta(M + 1), counts(M + 1), post, post0;
                if (l.genBam) { post.resize(p.hits.H); post0.resize(p.hits.N); }
                {
                    Timed tf{ph.final};
                    check_rc(rsem_b200_batch_final(batch, s, theta.data(), counts.data(), l.genBam ? post.data() : nullptr,
                                                   l.genBam ? post0.data() : nullptr), "batch_final");
                    check_rc(rsem_b200_batch_remove(batch, s), "batch_remove");
                }
                finish(p.idx, p.hits, p.model, theta, counts, post, post0, p.conprb, p.ncpv, p.totNum);
                it = in_batch.erase(it);
            }
        }
    };

    for (size_t i = 0; i < lines.size(); ++i) {
        const Line& l = lines[i];
        if (g_verbose || l.N1 == 0) block[i] += "== sample " + l.outName + " (" + manifest + " line " + std::to_string(l.no) + ")\n";
        if (l.N1 == 0) {  // EM.cpp:615-638
            block[i] += "Warning: There are no alignable reads!\n";
            FILE* fo = fopen((l.statName + ".theta").c_str(), "w");
            if (fo) fclose(fo);
            fo = fopen((l.statName + ".model").c_str(), "w");
            if (fo) fclose(fo);
            std::vector<double> theta(M + 1, 0.0), eel(M + 1, 0.0), countv(M + 1, 0.0);
            for (int t = 1; t <= M; ++t) eel[t] = transcripts[t].length;
            write_results_em(refName, l.imdName, transcripts, theta, eel, countv.data(), l.appendNames);
            if (l.genBam) {  // EM.cpp:627-633: the input is copied as it is
                const std::string command = "cp " + l.inpSamF + " " + l.outName + ".transcript.bam";
                block[i] += command + "\n";
                if (system(command.c_str()) != 0) die("Cannot copy " + l.inpSamF + "!");
            }
            continue;
        }
        const double t_load = now_s();
        ModelParamsH mp;
        mp.M = M;
        mp.N[0] = l.N0; mp.N[1] = l.N1; mp.N[2] = l.N2;
        load_mparams(l.imdName + ".mparams", mp);
        auto p = std::make_unique<Pending>();
        p->idx = i;
        HitStore& hits = p->hits;
        Sidecar sidecar;
        bool have_sidecar = load_sidecar(l.imdName, read_type, sidecar);
        if (have_sidecar && (sidecar.hits.N != l.N1 || sidecar.reads[0].n != l.N0 || sidecar.reads[2].n != l.N2 || mp.seedLen > kSidecarShortLen))
            have_sidecar = false;
        if (have_sidecar) hits = std::move(sidecar.hits);
        else load_dat(l.imdName + ".dat", read_type, l.N1, hits);
        for (int32_t t : hits.sid)   // the reference of the run is refName's, not the one this sample was aligned to
            if (t == 0 || std::abs(t) > M)
                refuse(manifest, l.no, "an alignment names transcript " + std::to_string(t) + ", outside " + refName + " (M = " + std::to_string(M) + ")");
        say(i, "Thread 0 : N = " + std::to_string(hits.N) + ", NHit = " + std::to_string(hits.H) + "\nEM_init finished!\n");
        if (!(l.N_tot > l.N2)) die("N_tot must be larger than N2!");
        std::vector<double> theta(M + 1);
        theta[0] = std::max(l.N0 * 1.0 / (l.N_tot - l.N2), 1e-8);   // EM.cpp:342-346
        for (int t = 1; t <= M; ++t) theta[t] = (1.0 - theta[0]) / M;
        HostModel& mdl = p->model;
        mdl.init_master(read_type, mp, &refs);
        ReadStore reads;
        mdl.estimate_from_reads(l.imdName, reads, have_sidecar ? &sidecar : nullptr);
        if (reads.n != l.N1) die("Read indices files do not match!");
        ph.load += now_s() - t_load;
        const double t_model = now_s();

        check_rc(rsem_b200_upload_hits(ctx, hits.N, hits.H, M, hits.row_ptr.data(), hits.sid.data(), hits.pos.data(),
                                       read_type >= 2 ? hits.insertL.data() : nullptr), "upload_hits");
        check_rc(rsem_b200_upload_reads(ctx, reads.n_mates, reads.off[0].data(), reads.base[0].data(),
                                        reads.has_qual ? reads.qual[0].data() : nullptr,
                                        reads.n_mates == 2 ? reads.off[1].data() : nullptr,
                                        reads.n_mates == 2 ? reads.base[1].data() : nullptr,
                                        (reads.n_mates == 2 && reads.has_qual) ? reads.qual[1].data() : nullptr,
                                        reads.lowq.data()), "upload_reads");
        check_rc(rsem_b200_set_theta(ctx, theta.data()), "set_theta");

        // rounds 1-10 update the model (EM.cpp:364-416), on the context as in rsem-run-em
        std::vector<double> st_prof(mdl.n_prof()), st_noise(mdl.n_noise()), st_gld(mp.maxL - (mp.minL - 1) + 1), st_rspd(mp.B + 2);
        rsem_b200_model_stats mstats;
        mstats.profile = st_prof.data();
        mstats.noise_profile = st_noise.data();
        mstats.gld_pdf = st_gld.data();
        mstats.gld_lb = mp.minL - 1;
        mstats.gld_span = mp.maxL - (mp.minL - 1);
        mstats.rspd_pdf = st_rspd.data();
        auto push_model = [&]() {
            rsem_b200_model abi;
            mdl.fill_abi(abi);
            check_rc(rsem_b200_set_model(ctx, &abi), "set_model");
        };
        bool keep_going = true;
        int ROUND = 0;
        long long tot = 0;
        while (keep_going && ROUND < 10) {
            ++ROUND;
            push_model();
            rsem_b200_round_stats rs;
            check_rc(rsem_b200_em_model_round(ctx, (double)l.N0, &mstats, &rs), "em_model_round");
            mdl.rebuild(mstats);
            say(i, round_line(ROUND, rs));
            tot = rs.totnum;
            keep_going = ROUND < MIN_ROUND || (tot > 0 && ROUND < MAX_ROUND);
        }
        push_model();
        check_rc(rsem_b200_calc_conprb(ctx), "calc_conprb");
        p->conprb.resize(hits.H);
        p->ncpv.resize(hits.N);
        check_rc(rsem_b200_download_conprb(ctx, p->conprb.data(), p->ncpv.data()), "download_conprb");
        p->round = ROUND;
        p->totNum = tot;
        ph.model += now_s() - t_model;
        if (keep_going) {   // round 11 on: the batch, or this context when the sample is outside the batch layout
            check_rc(rsem_b200_get_theta(ctx, theta.data()), "get_theta");
            int32_t slot = -1;
            int rc = rsem_b200_batch_add(batch, hits.N, hits.H, M, hits.row_ptr.data(), hits.sid.data(), p->conprb.data(),
                                         p->ncpv.data(), theta.data(), (double)l.N0, ROUND + 1, MIN_ROUND, MAX_ROUND, &slot);
            if (rc == RSEM_B200_ERR_FULL) {
                ++n_full;
                drain();
                rc = rsem_b200_batch_add(batch, hits.N, hits.H, M, hits.row_ptr.data(), hits.sid.data(), p->conprb.data(),
                                         p->ncpv.data(), theta.data(), (double)l.N0, ROUND + 1, MIN_ROUND, MAX_ROUND, &slot);
            }
            if (rc == 0) {
                ++n_batched;
                in_batch[slot] = std::move(p);
                continue;
            }
            if (rc != RSEM_B200_ERR_UNSUPPORTED && rc != RSEM_B200_ERR_FULL) check_rc(rc, "batch_add");
            ++n_single;
            std::vector<rsem_b200_round_stats> cs(32);
            Timed tk{ph.frozen};
            while (keep_going) {
                int32_t ran = 0, stopped = 0;
                check_rc(rsem_b200_em_rounds(ctx, ROUND + 1, 32, MIN_ROUND, MAX_ROUND, (double)l.N0, cs.data(), &ran, &stopped), "em_rounds");
                for (int r = 0; r < ran; ++r) say(i, round_line(ROUND + 1 + r, cs[r]));
                if (ran > 0) { ROUND += ran; tot = cs[ran - 1].totnum; }
                keep_going = !stopped;
            }
        }
        // final pass on the context (EM.cpp:460-478)
        const double t_final = now_s();
        std::vector<double> counts(M + 1), post, post0;
        check_rc(rsem_b200_get_theta(ctx, theta.data()), "get_theta");
        check_rc(rsem_b200_expected_weights(ctx, counts.data()), "expected_weights");
        if (l.genBam) {
            post.resize(hits.H);
            post0.resize(hits.N);
            check_rc(rsem_b200_download_conprb(ctx, post.data(), post0.data()), "download_conprb");
        }
        ph.final += now_s() - t_final;
        finish(i, hits, mdl, theta, counts, post, post0, p->conprb, p->ncpv, tot);
    }
    drain();
    double k12_ms = 0;
    uint64_t k12_rounds = 0;
    check_rc(rsem_b200_batch_timing(batch, &k12_ms, &k12_rounds), "batch_timing");
    if (getenv("RSEM_B200_TIMING")) {
        fprintf(stderr, "rsem-run-em-batch timing: %d samples in the batch, %d on the single-sample path; K12 %.3f ms over %llu "
                "sample-rounds\n", n_batched, n_single, k12_ms, (unsigned long long)k12_rounds);
        fprintf(stderr, "rsem-run-em-batch timing: arena full %d times\n", n_full);
        fprintf(stderr, "rsem-run-em-batch timing: load %.3f s, model rounds %.3f s, frozen rounds %.3f s, final pass %.3f s, "
                "writers %.3f s\n", ph.load, ph.model, ph.frozen, ph.final, ph.write);
    }
    rsem_b200_batch_destroy(batch);
    rsem_b200_ctx_destroy(ctx);
    for (const std::string& b : block) fputs(b.c_str(), stdout);
    const time_t t_end = time(NULL);
    printf("Time Used for EM.cpp : %d h %02d m %02d s\n", int((t_end - t_start) / 3600), int((t_end - t_start) % 3600 / 60), int((t_end - t_start) % 60));
    return 0;
}
