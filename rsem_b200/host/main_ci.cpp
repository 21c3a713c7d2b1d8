// bin/rsem-calculate-credibility-intervals: drop-in for the reference's tool of that name (calcCI.cpp).
//
//   rsem-calculate-credibility-intervals reference_name imdName statName confidence nCV nSpC nMB [-p #Threads]
//                                        [--seed seed] [--pseudo-count pseudo_count] [-q]
//
// Phase I (calcCI.cpp:93-216) runs on host threads, one per count-vector file, in host/ffm/ci_sample.cpp: the Gamma draws
// compare glibc's libm against uniforms and must stay bit-exact.  Each thread pushes its finished sample rows to the
// device while it keeps sampling.  Phase II (calcCI.cpp:218-508: transpose, FPKM, gene and isoform sums, sorting and
// the intervals) runs on the device (csrc/ci_kernels.cu).  The appended rows of imd.iso_res / imd.gene_res (and
// imd.allele_res) are the reference's for the same --seed.
//
// Samples are stored at fixed positions (thread t's after those of the count vectors of threads 0 .. t - 1) where the
// reference's buffer takes them in the order its threads get the lock; only the isoform rows of an allele-specific
// reference depend on that order (their running sums, calcCI.cpp:308-345), and with -p 1 both orders are the same.
// The one difference in files: imd.tmp, the reference's transposed sample file that nothing reads afterwards, is
// not written.
//
// RSEM_B200_CI_DEVICE_BYTES=<bytes> caps the device memory K8 uses (tests force the blocked path with it);
// RSEM_B200_TIMING=1 prints the host sampling time and the device time of each phase to stderr.
// The stages are in host/ci_stages.cpp, shared with rsem-calculate-credibility-intervals-batch.
#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <string>
#include <vector>

#include "host.hpp"

using namespace host;

int main(int argc, char* argv[]) {
    if (argc < 8) {
        printf("Usage: rsem-calculate-credibility-intervals reference_name imdName statName confidence nCV nSpC nMB [-p #Threads] [--seed seed] [--pseudo-count pseudo_count] [-q]\n");
        exit(-1);
    }
    CiArgs a;
    std::string why = parse_ci_args(std::vector<std::string>(argv + 2, argv + argc), a, false);
    g_verbose = !a.quiet;
    if (!why.empty()) die(why);
    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    const Say out = [](const std::string& line) { fputs(line.c_str(), stdout); };
    const Say* say = g_verbose ? &out : nullptr;

    CiReference ref;
    load_ci_reference(argv[1], ref);
    const int M = ref.refs.M;
    why = ci_sample_count_error(a, M);
    if (!why.empty()) die(why);
    CiSample s;
    load_ci_model(ref, a, s.eel, s.mw);
    why = ci_memory_error(a, M);
    if (!why.empty()) die(why);
    const uint32_t seed = a.hasSeed ? a.seed : (uint32_t)time(NULL);
    load_ci_vectors(a, M, s, false);
    const std::vector<int32_t> parts = ci_parts(a.nThreads, M, ref.gi);

    rsem_b200_ctx* ctx = nullptr;
    const char* dev = getenv("RSEM_B200_DEVICE");
    check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
    const char* budget = getenv("RSEM_B200_CI_DEVICE_BYTES");
    const rsem_b200_ci_params cp = ci_params(ref, a, parts, budget ? strtoull(budget, nullptr, 10) : 0);
    check_rc(rsem_b200_ci_begin(ctx, &cp), "ci_begin");

    // Phase I: each sampler pushes its rows as it draws them; the device copy overlaps with the sampling
    const double t0 = now_s();
    ci_sample_rows(ctx, a, M, s, seed, say, false);
    const double t1 = now_s();
    if (say) out("Sampling is finished!\n");

    CiIntervals r;
    ci_intervals(ctx, ref, r);
    rsem_b200_ctx_destroy(ctx);
    const double t2 = now_s();
    write_ci_sample(ref, a, parts, r, say);
    if (timing)
        fprintf(stderr,
                "rsem-calculate-credibility-intervals timing: sampling (host, %d threads) %.3f s, intervals %.3f s; device: "
                "transpose %.3f s, sums %.3f s, sort %.3f s, intervals %.3f s, %llu blocks, sample matrix %s\n",
                a.samplers(), t1 - t0, t2 - t1, r.st.transpose_ms / 1e3, r.st.sums_ms / 1e3, r.st.sort_ms / 1e3,
                r.st.interval_ms / 1e3, (unsigned long long)r.st.blocks, r.st.resident ? "on the device" : "in host memory");
    return 0;
}
