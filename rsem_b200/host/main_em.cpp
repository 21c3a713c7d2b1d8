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
#include <cstdlib>
#include <ctime>
#include <future>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

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

double g_t0 = 0;
void stamp(const char* what) {   // RSEM_B200_TIMING=1: phase timestamps on stderr
    static const bool on = getenv("RSEM_B200_TIMING") != nullptr;
    if (on) fprintf(stderr, "rsem-run-em timing: %8.3f s  %s\n", now_s() - g_t0, what);
}

void print_round(int round, const rsem_b200_round_stats& s) {
    if (g_verbose) {  // the reference ends the line with std::endl, i.e. flushes it (EM.cpp:415); harnesses timestamp these lines
        fputs(round_line(round, s).c_str(), stdout);
        fflush(stdout);
    }
}

void put(const std::string& s) { fputs(s.c_str(), stdout); }

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
    const std::string refName = argv[1];
    const int read_type = atoi(argv[2]);
    EmArgs a = parse_em_args(std::vector<std::string>(argv + 3, argv + argc));
    if (a.quiet) g_verbose = false;
    if (a.nThreads <= 0) die("Number of threads should be bigger than 0!");
    g_io_threads = env_int("RSEM_B200_IO_THREADS", a.nThreads);   // -p: host threads for parsing / formatting
    if (read_type < 0 || read_type > 3) { fprintf(stderr, "Unknown Read Type!\n"); exit(-1); }

    // CUDA context creation takes seconds on a multi-GPU node: start it now (rank 0's), overlap it with the file parsing
    std::vector<int> devices = gpu_devices();
    std::future<LaneContexts> ctx_future = std::async(std::launch::async, open_lanes, std::vector<int>{devices[0]});

    EmReference ref;
    load_em_reference(refName, ref);
    const int M = ref.refs.M;
    stamp("refs + transcripts loaded");

    EmSample s;
    if (!load_cnt(a.statName, true, s.n)) die("Cannot parse " + a.statName + ".cnt!");
    if (s.n.N1 == 0) {
        write_no_alignable_reads(ref, a, put);
        put(time_used_line(t_start));
        return 0;
    }
    const int MAX_ROUND = env_int("RSEM_MAX_ROUND", 10000), MIN_ROUND = env_int("RSEM_MIN_ROUND", 20);

    // ---- init (EM.cpp:97-174): hits from .dat; the GPU holds the whole read range ----
    load_em_hits(a.imdName, read_type, M, s);
    stamp(s.have_sidecar ? "binary side-car loaded (.dat and read files not parsed)" : ".dat parsed");
    ReadStore reads;
    load_em_model(a.imdName, read_type, ref.refs, s, reads, put);
    stamp("reads parsed, initial model estimated");
    const HitStore& hits = s.hits;
    const RefData& refs = ref.refs;

    // ---- device set-up: one worker (host thread + context) per GPU, reads sharded like the reference's threads ----
    if ((uint64_t)devices.size() > s.n.N1) devices.resize((size_t)s.n.N1);
    const int world = (int)devices.size();
    std::vector<std::pair<uint64_t, uint64_t>> shards = shard_reads(hits.row_ptr, world);
    if (g_verbose && world > 1)
        for (int r = 0; r < world; ++r)
            printf("GPU %d : N = %llu, NHit = %llu\n", devices[r], (unsigned long long)(shards[r].second - shards[r].first),
                   (unsigned long long)(hits.row_ptr[shards[r].second] - hits.row_ptr[shards[r].first]));

    unsigned char uid[RSEM_B200_UNIQUE_ID_BYTES] = {0};
    rsem_b200_ctx* ctx0 = nullptr;
    {
        const LaneContexts lc = ctx_future.get();
        if (!lc.err.empty()) die(lc.err);
        ctx0 = lc.ctx[0];
    }
    if (world > 1) check_rc(rsem_b200_comm_unique_id(uid), "comm_unique_id");

    if (a.gibbsOut) { s.conprb.resize(hits.H); s.ncpv.resize(hits.N); }
    if (a.genBam) { s.post.resize(hits.H); s.post0.resize(hits.N); }   // posteriors in hit / read order
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
                                       read_type >= 2 ? hits.insertL.data() + h0 : nullptr), "upload_hits");
        auto mate = [&](const std::vector<uint8_t>& v, int m) { return v.data() + reads.off[m][r0]; };
        check_rc(rsem_b200_upload_reads(ctx, reads.n_mates, off[0].data(), mate(reads.base[0], 0),
                                        reads.has_qual ? mate(reads.qual[0], 0) : nullptr,
                                        reads.n_mates == 2 ? off[1].data() : nullptr,
                                        reads.n_mates == 2 ? mate(reads.base[1], 1) : nullptr,
                                        (reads.n_mates == 2 && reads.has_qual) ? mate(reads.qual[1], 1) : nullptr,
                                        reads.lowq.data() + r0), "upload_reads");
        check_rc(rsem_b200_upload_refs(ctx, M, refs.seq_off.data(), refs.seq.data(), refs.full_len.data(), refs.tot_len.data(),
                                       refs.mask_off.data(), refs.mask_words.data()), "upload_refs");
        check_rc(rsem_b200_set_theta(ctx, s.theta.data()), "set_theta");
        if (rank == 0) stamp("context ready, inputs uploaded");

        // ---- EM loop (EM.cpp:364-416).  Every rank keeps its own copy of the master model and rebuilds it from the
        // (allreduced, hence identical) statistics: no broadcast is needed.
        HostModel mdl = s.model;
        auto on_round = [&](int round, const rsem_b200_round_stats& rs) { if (rank == 0) print_round(round, rs); };
        EmRounds r = em_model_rounds(ctx, mdl, s.n.N0, MIN_ROUND, MAX_ROUND, on_round);
        em_frozen_rounds(ctx, s.n.N0, MIN_ROUND, MAX_ROUND, r, on_round);
        if (rank == 0) stamp("EM loop finished");
        if (a.gibbsOut) check_rc(rsem_b200_download_conprb(ctx, s.conprb.data() + h0, s.ncpv.data() + r0), "download_conprb");
        // ---- expected weights with the learned parameters (EM.cpp:460-478); counts are summed over ranks by the library
        std::vector<double> th(M + 1), cnt(M + 1);
        check_rc(rsem_b200_get_theta(ctx, th.data()), "get_theta");
        check_rc(rsem_b200_expected_weights(ctx, cnt.data()), "expected_weights");
        if (a.genBam) check_rc(rsem_b200_download_conprb(ctx, s.post.data() + h0, s.post0.data() + r0), "download_conprb");  // now the posteriors
        if (rank == 0) {
            s.theta = th;
            s.counts = cnt;
            final_model = mdl;
            totNum = r.totNum;
        }
        rsem_b200_ctx_destroy(ctx);
    };
    if (world == 1) worker(0);
    else {
        std::vector<std::thread> pool;
        for (int r = 0; r < world; ++r) pool.emplace_back(worker, r);
        for (auto& t : pool) t.join();
    }
    s.model = final_model;
    stamp("final pass done, outputs downloaded");
    finish_em_sample(ref, read_type, a, s, totNum, MAX_ROUND, "", a.nThreads, g_verbose, stamp);
    put(time_used_line(t_start));
    return 0;
}
