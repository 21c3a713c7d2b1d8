// rsem-run-em, H100 edition: same argv, same input and output files as the reference executable
// (/root/reference/EM.cpp:541-675), so it drops in beside the unmodified rsem-calculate-expression.
//
//   rsem-run-em refName read_type sampleName imdName statName [-p #Threads] [-b samInpF has_fai? [fai_file]]
//               [-q] [--gibbs-out] [--sampling] [--seed seed] [--append-names]
//
// Differences from the reference, all outside the results:
//   * -p is accepted and ignored for the EM (the result of the reference does not depend on it);
//     the GPU is chosen with RSEM_B200_DEVICE (default 0), several GPUs with RSEM_B200_DEVICES=0,1,..:
//     reads are sharded over them like the reference shards them over threads, counts and model
//     statistics are summed with ncclAllReduce.
//   * -b: the input SAM / BAM is re-read and written to sampleName.transcript.bam with MAPQ and ZW:f set from the
//     posteriors (EM.cpp:504-536, BamWriter.h); SAM and BAM are read and BAM is written by this program's own
//     BGZF / BAM code (host/bam.cpp) - CRAM input and the has_fai / fai_file arguments (which the reference parses but
//     never applies, BamWriter.h:56) are not supported.  -p sets the BGZF compression threads like hts_set_threads.
//   * RSEM_MAX_ROUND / RSEM_MIN_ROUND override the compile-time constants MAX_ROUND = 10000 and
//     MIN_ROUND = 20 (EM.cpp:54-55), like oracle/_ref/rsem-run-em-rounds, for fixed-round parity runs.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <ctime>
#include <future>
#include <map>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

struct Args {
    std::string refName, outName, imdName, statName;
    int read_type = 0;
    bool genBam = false, bamSampling = false, gibbsOut = false, hasSeed = false, appendNames = false;
    uint32_t seed = 0;
    std::string inpSamF;
};

void usage() {
    printf("Usage : rsem-run-em refName read_type sampleName imdName statName [-p #Threads] [-b samInpF has_fai? [fai_file]] [-q] [--gibbs-out] [--sampling] [--seed seed] [--append-names]\n\n");
    printf("  refName: reference name\n");
    printf("  read_type: 0 single read without quality score; 1 single read with quality score; 2 paired-end read without quality score; 3 paired-end read with quality score.\n");
    printf("  sampleName: sample's name, including the path\n");
    printf("  sampleToken: sampleName excludes the path\n");
    printf("  -p: number of threads which user wants to use. (default: 1)\n");
    printf("  -b: produce bam format output file. (default: off)\n");
    printf("  -q: set it quiet\n");
    printf("  --gibbs-out: generate output file used by Gibbs sampler. (default: off)\n");
    printf("  --sampling: sample each read from its posterior distribution when BAM file is generated. (default: off)\n");
    printf("  --seed uint32: the seed used for the BAM sampling. (default: off)\n");
    printf("  --append-names: append transcript_name/gene_name when available. (default: off)\n");
    printf("// model parameters should be in imdName.mparams.\n");
    exit(-1);
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
double g_t0 = 0;
void stamp(const char* what) {   // RSEM_B200_TIMING=1: phase timestamps on stderr
    static const bool on = getenv("RSEM_B200_TIMING") != nullptr;
    if (on) fprintf(stderr, "rsem-run-em timing: %8.3f s  %s\n", now_s() - g_t0, what);
}

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

void print_round(int round, const rsem_b200_round_stats& s) {
    if (g_verbose) {  // the reference ends the line with std::endl, i.e. flushes it (EM.cpp:415); harnesses timestamp these lines
        printf("ROUND = %d, SUM = %.15g, bChange = %.6g, totNum = %lld\n", round, s.sum, s.bchange, (long long)s.totnum);
        fflush(stdout);
    }
}

// Contiguous read ranges with about nHits / world hits each: the reference's thread-sharding rule (EM.cpp:135-157),
// implemented once in the library (rsem_b200_shard_reads) so that bench.py and the tests exercise the same code.
std::vector<std::pair<uint64_t, uint64_t>> shard_reads(const std::vector<uint64_t>& row_ptr, int world) {
    std::vector<uint64_t> bounds((size_t)world + 1);
    check_rc(rsem_b200_shard_reads(row_ptr.size() - 1, row_ptr.data(), world, bounds.data()), "shard_reads");
    std::vector<std::pair<uint64_t, uint64_t>> out;
    for (int i = 0; i < world; ++i) out.emplace_back(bounds[i], bounds[i + 1]);
    return out;
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 6) usage();
    const time_t t_start = time(NULL);
    g_t0 = now_s();
    Args a;
    a.refName = argv[1];
    a.read_type = atoi(argv[2]);
    a.outName = argv[3];
    a.imdName = argv[4];
    a.statName = argv[5];
    int nThreads = 1;
    for (int i = 6; i < argc; ++i) {
        if (!strcmp(argv[i], "-p") && i + 1 < argc) nThreads = atoi(argv[i + 1]);
        if (!strcmp(argv[i], "-b") && i + 1 < argc) { a.genBam = true; a.inpSamF = argv[i + 1]; }
        if (!strcmp(argv[i], "-q")) g_verbose = false;
        if (!strcmp(argv[i], "--gibbs-out")) a.gibbsOut = true;
        if (!strcmp(argv[i], "--sampling")) a.bamSampling = true;
        if (!strcmp(argv[i], "--seed") && i + 1 < argc) { a.hasSeed = true; a.seed = parse_seed(argv[i + 1]); }
        if (!strcmp(argv[i], "--append-names")) a.appendNames = true;
    }
    if (nThreads <= 0) die("Number of threads should be bigger than 0!");
    g_io_threads = env_int("RSEM_B200_IO_THREADS", nThreads);   // -p: host threads for parsing / formatting
    if (a.read_type < 0 || a.read_type > 3) { fprintf(stderr, "Unknown Read Type!\n"); exit(-1); }

    // CUDA context creation takes seconds on a multi-GPU node: start it now, overlap it with the file parsing
    struct CtxResult { int rc; rsem_b200_ctx* ctx; std::string err; };
    std::future<CtxResult> ctx_future = std::async(std::launch::async, []() {
        CtxResult r{0, nullptr, ""};
        r.rc = rsem_b200_ctx_create(env_int("RSEM_B200_DEVICE", 0), &r.ctx);
        if (r.rc != 0) r.err = rsem_b200_last_error();  // the message is thread-local: take it here
        return r;
    });

    RefData refs;
    load_refs(a.refName + ".seq", true, refs);
    const int M = refs.M;
    std::vector<TranscriptInfo> transcripts;
    int ti_type = 0;
    load_transcripts(a.refName + ".ti", transcripts, &ti_type);
    stamp("refs + transcripts loaded");

    uint64_t N0, N1, N2, N_tot;
    {
        std::vector<char> b = slurp(a.statName + ".cnt");
        b.push_back(0);
        unsigned long long v[4];
        if (sscanf(b.data(), "%llu %llu %llu %llu", &v[0], &v[1], &v[2], &v[3]) != 4) die("Cannot parse " + a.statName + ".cnt!");
        N0 = v[0]; N1 = v[1]; N2 = v[2]; N_tot = v[3];
    }

    std::vector<double> theta(M + 1, 0.0), eel;
    if (N1 == 0) {  // EM.cpp:615-638
        printf("Warning: There are no alignable reads!\n");
        FILE* fo = fopen((a.statName + ".theta").c_str(), "w");
        if (fo) fclose(fo);
        fo = fopen((a.statName + ".model").c_str(), "w");
        if (fo) fclose(fo);
        eel.assign(M + 1, 0.0);
        for (int i = 1; i <= M; ++i) eel[i] = transcripts[i].length;
        std::vector<double> countv(M + 1, 0.0);
        write_results_em(a.refName, a.imdName, transcripts, theta, eel, countv.data(), a.appendNames);
        if (a.genBam) {  // EM.cpp:627-633: the input is copied as it is
            const std::string command = "cp " + a.inpSamF + " " + a.outName + ".transcript.bam";
            printf("%s\n", command.c_str());
            if (system(command.c_str()) != 0) die("Cannot copy " + a.inpSamF + "!");
        }
        const time_t t_end = time(NULL);
        printf("Time Used for EM.cpp : %d h %02d m %02d s\n", int((t_end - t_start) / 3600), int((t_end - t_start) % 3600 / 60), int((t_end - t_start) % 60));
        return 0;
    }

    ModelParamsH mp;
    mp.M = M;
    mp.N[0] = N0; mp.N[1] = N1; mp.N[2] = N2;
    load_mparams(a.imdName + ".mparams", mp);

    const int MAX_ROUND = env_int("RSEM_MAX_ROUND", 10000), MIN_ROUND = env_int("RSEM_MIN_ROUND", 20);

    // ---- init (EM.cpp:97-174): hits from .dat; the GPU holds the whole read range ----
    HitStore hits;
    Sidecar sidecar;   // imd.b200, written by bin/rsem-parse-alignments: the same content as .dat + the read files, decoded
    bool have_sidecar = load_sidecar(a.imdName, a.read_type, sidecar);
    if (have_sidecar && (sidecar.hits.N != N1 || sidecar.reads[0].n != N0 || sidecar.reads[2].n != N2 || mp.seedLen > kSidecarShortLen))
        have_sidecar = false;   // does not describe this run: parse the text files
    if (have_sidecar) {
        hits = std::move(sidecar.hits);
        stamp("binary side-car loaded (.dat and read files not parsed)");
    } else {
        load_dat(a.imdName + ".dat", a.read_type, N1, hits);
        stamp(".dat parsed");
    }
    if (g_verbose) {
        printf("Thread 0 : N = %llu, NHit = %llu\n", (unsigned long long)hits.N, (unsigned long long)hits.H);
        printf("EM_init finished!\n");
    }

    // initial theta (EM.cpp:342-346)
    if (!(N_tot > N2)) die("N_tot must be larger than N2!");
    theta[0] = std::max(N0 * 1.0 / (N_tot - N2), 1e-8);
    for (int i = 1; i <= M; ++i) theta[i] = (1.0 - theta[0]) / M;

    HostModel model;
    model.init_master(a.read_type, mp, &refs);
    ReadStore reads;
    model.estimate_from_reads(a.imdName, reads, have_sidecar ? &sidecar : nullptr);
    if (reads.n != N1) die("Read indices files do not match!");
    stamp("reads parsed, initial model estimated");

    // ---- device set-up: one worker (host thread + context) per GPU, reads sharded like the reference's threads ----
    std::vector<int> devices = gpu_devices();
    if ((uint64_t)devices.size() > N1) devices.resize((size_t)N1);
    const int world = (int)devices.size();
    std::vector<std::pair<uint64_t, uint64_t>> shards = shard_reads(hits.row_ptr, world);
    if (g_verbose && world > 1)
        for (int r = 0; r < world; ++r)
            printf("GPU %d : N = %llu, NHit = %llu\n", devices[r], (unsigned long long)(shards[r].second - shards[r].first),
                   (unsigned long long)(hits.row_ptr[shards[r].second] - hits.row_ptr[shards[r].first]));

    unsigned char uid[RSEM_B200_UNIQUE_ID_BYTES] = {0};
    rsem_b200_ctx* ctx0 = nullptr;
    {
        CtxResult r = ctx_future.get();
        if (r.rc != 0) die("rsem_b200: ctx_create failed: " + r.err);
        ctx0 = r.ctx;
    }
    if (world > 1) check_rc(rsem_b200_comm_unique_id(uid), "comm_unique_id");

    std::vector<double> conprb(hits.H), ncpv(hits.N), counts(M + 1, 0.0);
    std::vector<double> post, post0;  // posteriors in hit / read order, only kept for -b
    if (a.genBam) { post.resize(hits.H); post0.resize(hits.N); }
    HostModel final_model;
    long long totNum = 0;

    auto worker = [&](int rank) {
        rsem_b200_ctx* ctx = rank == 0 ? ctx0 : nullptr;
        if (rank != 0) check_rc(rsem_b200_ctx_create(devices[rank], &ctx), "ctx_create");
        if (world > 1) check_rc(rsem_b200_comm_init(ctx, uid, world, rank), "comm_init");
        const uint64_t r0 = shards[rank].first, r1 = shards[rank].second;
        const uint64_t h0 = hits.row_ptr[r0], h1 = hits.row_ptr[r1];
        // shard-local CSR and read offsets (rebased to 0)
        std::vector<uint64_t> rp(r1 - r0 + 1), off[2];
        for (uint64_t i = r0; i <= r1; ++i) rp[i - r0] = hits.row_ptr[i] - h0;
        for (int m = 0; m < reads.n_mates; ++m) {
            off[m].resize(r1 - r0 + 1);
            for (uint64_t i = r0; i <= r1; ++i) off[m][i - r0] = reads.off[m][i] - reads.off[m][r0];
        }
        check_rc(rsem_b200_upload_hits(ctx, r1 - r0, h1 - h0, M, rp.data(), hits.sid.data() + h0, hits.pos.data() + h0,
                                       a.read_type >= 2 ? hits.insertL.data() + h0 : nullptr), "upload_hits");
        auto mate = [&](const std::vector<uint8_t>& v, int m) { return v.data() + reads.off[m][r0]; };
        check_rc(rsem_b200_upload_reads(ctx, reads.n_mates, off[0].data(), mate(reads.base[0], 0),
                                        reads.has_qual ? mate(reads.qual[0], 0) : nullptr,
                                        reads.n_mates == 2 ? off[1].data() : nullptr,
                                        reads.n_mates == 2 ? mate(reads.base[1], 1) : nullptr,
                                        (reads.n_mates == 2 && reads.has_qual) ? mate(reads.qual[1], 1) : nullptr,
                                        reads.lowq.data() + r0), "upload_reads");
        check_rc(rsem_b200_upload_refs(ctx, M, refs.seq_off.data(), refs.seq.data(), refs.full_len.data(), refs.tot_len.data(),
                                       refs.mask_off.data(), refs.mask_words.data()), "upload_refs");
        check_rc(rsem_b200_set_theta(ctx, theta.data()), "set_theta");
        if (rank == 0) stamp("context ready, inputs uploaded");

        // ---- EM loop (EM.cpp:364-416).  Every rank keeps its own copy of the master model and rebuilds it from the
        // (allreduced, hence identical) statistics: no broadcast is needed.
        HostModel mdl = model;
        std::vector<double> st_prof(mdl.n_prof()), st_noise(mdl.n_noise()), st_gld(mp.maxL - (mp.minL - 1) + 1), st_rspd(mp.B + 2);
        rsem_b200_model_stats mstats;
        mstats.profile = st_prof.data();
        mstats.noise_profile = st_noise.data();
        mstats.gld_pdf = st_gld.data();
        mstats.gld_lb = mp.minL - 1;
        mstats.gld_span = mp.maxL - (mp.minL - 1);
        mstats.rspd_pdf = st_rspd.data();

        bool model_dirty = true;  // device copy of the model tables / conprb is stale (needCalcConPrb)
        auto push_model = [&]() {
            rsem_b200_model abi;
            mdl.fill_abi(abi);
            check_rc(rsem_b200_set_model(ctx, &abi), "set_model");
        };
        int ROUND = 0;
        long long tot = 0;
        const int CHUNK = 32;
        std::vector<rsem_b200_round_stats> chunk_stats(CHUNK);
        bool keep_going = true;
        while (keep_going) {
            ++ROUND;
            if (ROUND <= 10) {  // doesUpdateModel, EM.cpp:307-310
                if (model_dirty) { push_model(); model_dirty = false; }
                rsem_b200_round_stats rs;
                check_rc(rsem_b200_em_model_round(ctx, (double)N0, &mstats, &rs), "em_model_round");
                mdl.rebuild(mstats);  // model.init(); collect(); finish()
                model_dirty = true;
                if (rank == 0) print_round(ROUND, rs);
                tot = rs.totnum;
                keep_going = ROUND < MIN_ROUND || (tot > 0 && ROUND < MAX_ROUND);
            } else {
                if (model_dirty) {
                    push_model();
                    check_rc(rsem_b200_calc_conprb(ctx), "calc_conprb");
                    model_dirty = false;
                }
                int32_t ran = 0, stopped = 0;
                check_rc(rsem_b200_em_rounds(ctx, ROUND, CHUNK, MIN_ROUND, MAX_ROUND, (double)N0, chunk_stats.data(), &ran, &stopped), "em_rounds");
                if (rank == 0) for (int r = 0; r < ran; ++r) print_round(ROUND + r, chunk_stats[r]);
                if (ran > 0) { ROUND += ran - 1; tot = chunk_stats[ran - 1].totnum; }
                keep_going = !stopped;
            }
        }
        if (rank == 0) stamp("EM loop finished");
        // ---- .ofg inputs (EM.cpp:421-457): calcConProbs when the loop ended inside the model rounds
        if (model_dirty) {
            push_model();
            check_rc(rsem_b200_calc_conprb(ctx), "calc_conprb");
            model_dirty = false;
        }
        if (a.gibbsOut) check_rc(rsem_b200_download_conprb(ctx, conprb.data() + h0, ncpv.data() + r0), "download_conprb");
        // ---- expected weights with the learned parameters (EM.cpp:460-478); counts are summed over ranks by the library
        std::vector<double> th(M + 1), cnt(M + 1);
        check_rc(rsem_b200_get_theta(ctx, th.data()), "get_theta");
        check_rc(rsem_b200_expected_weights(ctx, cnt.data()), "expected_weights");
        if (a.genBam) check_rc(rsem_b200_download_conprb(ctx, post.data() + h0, post0.data() + r0), "download_conprb");  // now the posteriors
        if (rank == 0) {
            theta = th;
            counts = cnt;
            final_model = mdl;
            totNum = tot;
        }
        rsem_b200_ctx_destroy(ctx);
    };
    if (world == 1) worker(0);
    else {
        std::vector<std::thread> pool;
        for (int r = 0; r < world; ++r) pool.emplace_back(worker, r);
        for (auto& t : pool) t.join();
    }
    model = final_model;
    if (totNum > 0) fprintf(stderr, "Warning: RSEM reaches %d iterations before meeting the convergence criteria.\n", MAX_ROUND);
    stamp("final pass done, outputs downloaded");
    if (a.gibbsOut) write_ofg(a.imdName + ".ofg", M, N0, hits, conprb, ncpv);
    stamp(".ofg written");
    counts[0] += N0;

    write_em_outputs(a.refName, a.imdName, a.statName, refs, transcripts, model, theta, counts, a.appendNames);
    stamp(".theta / .model / result rows written");
    if (a.genBam) {
        write_posterior_bam(a.inpSamF, a.outName, a.read_type, a.bamSampling, a.hasSeed, a.seed, transcripts, ti_type, hits,
                            post, post0, nThreads, g_verbose);
        stamp("transcript BAM written");
    }

    const time_t t_end = time(NULL);
    printf("Time Used for EM.cpp : %d h %02d m %02d s\n", int((t_end - t_start) / 3600), int((t_end - t_start) % 3600 / 60), int((t_end - t_start) % 60));
    return 0;
}
