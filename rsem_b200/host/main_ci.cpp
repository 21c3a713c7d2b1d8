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
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <string>
#include <thread>
#include <vector>

#include "host.hpp"

namespace host {
void ci_sample_vectors(const int32_t* cvs, int n_cv, int M, int nSpC, double pseudoC, uint32_t seed, const double* eel,
                       const double* mw, int thread_no, bool verbose,
                       const std::function<void(int64_t, const float*, float)>& emit);
}  // namespace host

using namespace host;

namespace {

// the count vectors of one file, M + 1 integers each, whitespace-separated as fscanf("%d") reads them (calcCI.cpp:112-114)
std::vector<int32_t> read_count_vectors(const std::string& path, int M) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) die("Cannot open " + path + "! It may not exist.");
    fclose(f);
    std::vector<char> buf = slurp(path);
    buf.push_back('\0');
    std::vector<int32_t> out;
    const char* p = buf.data();
    for (;;) {
        char* end = nullptr;
        const long v = strtol(p, &end, 10);
        if (end == p) break;
        out.push_back((int32_t)v);
        p = end;
    }
    while (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r') ++p;
    if (*p) die("Cannot parse " + path + "!");
    if (out.size() % (size_t)(M + 1)) die(path + " holds a count vector with fewer than " + std::to_string(M + 1) + " entries!");
    for (size_t i = 0; i < out.size(); i += M + 1)
        if (out[i] < 0) die(path + ": a count vector has a negative noise count!");
    return out;
}

void write_rows(const std::string& path, const float* v, int n) {
    FILE* fo = fopen(path.c_str(), "a");
    if (!fo) die("Cannot open " + path + "!");
    for (int f = 0; f < 6; ++f)
        for (int i = 0; i < n; ++i) fprintf(fo, "%.6g%c", v[(size_t)i * 6 + f], (i < n - 1 ? '\t' : '\n'));
    if (fclose(fo) != 0) die("Cannot write " + path + "!");
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 8) {
        printf("Usage: rsem-calculate-credibility-intervals reference_name imdName statName confidence nCV nSpC nMB [-p #Threads] [--seed seed] [--pseudo-count pseudo_count] [-q]\n");
        exit(-1);
    }
    const std::string refName = argv[1], imdName = argv[2], statName = argv[3];
    const double confidence = atof(argv[4]);
    const int nCV = atoi(argv[5]), nSpC = atoi(argv[6]), nMB = atoi(argv[7]);
    int nThreads = 1;
    bool quiet = false, hasSeed = false;
    uint32_t seed = 0;
    double pseudoC = 1.0;
    for (int i = 8; i < argc; i++) {
        if (!strcmp(argv[i], "-p") && i + 1 < argc) nThreads = atoi(argv[i + 1]);
        if (!strcmp(argv[i], "--seed") && i + 1 < argc) { hasSeed = true; seed = parse_seed(argv[i + 1]); }
        if (!strcmp(argv[i], "--pseudo-count") && i + 1 < argc) pseudoC = atof(argv[i + 1]);
        if (!strcmp(argv[i], "-q")) quiet = true;
    }
    g_verbose = !quiet;
    if (nThreads < 1) die("Number of threads should be bigger than 0!");
    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };

    RefData refs;
    load_refs(refName + ".seq", false, refs);
    const int M = refs.M;
    std::vector<int> gi, gt, ta;
    load_groups(refName + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(refName, gt, ta);
    const int m_trans = alleleS ? (int)ta.size() - 1 : 0;
    const int64_t nSamples = (int64_t)nCV * nSpC;
    if (!(nCV > 0 && nSpC > 0 && M > 0)) die("nCV and nSpC must be positive!");
    if (nSamples > INT32_MAX) die("nCV * nSpC must be below 2^31!");

    int model_type = 0;
    LenDistH gld;
    std::vector<double> mw, eel;
    HostModel::read_for_gibbs(statName + ".model", M, model_type, gld, mw);
    calc_eel(refs, gld, eel);

    {   // Buffer.h:18-20, in its unsigned 64-bit arithmetic (a negative nMB wraps to a large size and passes)
        uint64_t size = (uint64_t)(int64_t)nMB * 1024 * 1024 / sizeof(float) / (uint64_t)M;
        if (size > (uint64_t)nSamples) size = nSamples;
        if (size == 0) die("Memory allocated for credibility intervals is not enough!");
    }

    // one reader per count-vector file, engines from the engineFactory sequence (calcCI.cpp:172-188)
    const int num_threads = std::min(nThreads, nCV);
    const std::vector<uint32_t> seeds = engine_seeds(hasSeed ? seed : (uint32_t)time(NULL), num_threads);
    std::vector<std::vector<int32_t>> cvs(num_threads);
    {
        std::vector<std::thread> th;
        for (int t = 0; t < num_threads; ++t)
            th.emplace_back([&, t]() { cvs[t] = read_count_vectors(imdName + ".countvectors" + std::to_string(t), M); });
        for (auto& x : th) x.join();
    }
    std::vector<int64_t> first(num_threads + 1, 0);
    for (int t = 0; t < num_threads; ++t) first[t + 1] = first[t] + (int64_t)(cvs[t].size() / (M + 1)) * nSpC;
    if (first[num_threads] != nSamples)
        die("The count-vector files hold " + std::to_string(first[num_threads] / nSpC) + " count vectors, not nCV = " +
            std::to_string(nCV) + "!");

    // the gene ranges of the reference's Phase II threads (calcCI.cpp:402-420)
    std::vector<int32_t> parts{0};
    {
        int n_parts = nThreads, quotient = M / n_parts;
        if (quotient < 1) { n_parts = M; quotient = 1; }
        int cur = 0;
        for (int i = 0; i < n_parts; i++) {
            int num_isoforms = 0;
            while ((m - cur > n_parts - i - 1) && (i == n_parts - 1 || num_isoforms < quotient)) {
                num_isoforms += gi[cur + 1] - gi[cur];
                ++cur;
            }
            parts.push_back(cur);
        }
    }

    rsem_b200_ctx* ctx = nullptr;
    const char* dev = getenv("RSEM_B200_DEVICE");
    check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
    rsem_b200_ci_params cp;
    memset(&cp, 0, sizeof cp);
    cp.M = M;
    cp.n_genes = m;
    cp.gene_start = gi.data();
    cp.n_isoforms = m_trans;
    cp.isoform_start = alleleS ? ta.data() : nullptr;
    cp.n_parts = (int)parts.size() - 1;
    cp.part_gene_start = parts.data();
    cp.n_samples = nSamples;
    cp.threshold = (int)(nSamples - ((int)(confidence * nSamples - 1e-8) + 1));
    const char* budget = getenv("RSEM_B200_CI_DEVICE_BYTES");
    cp.device_budget = budget ? strtoull(budget, nullptr, 10) : 0;
    check_rc(rsem_b200_ci_begin(ctx, &cp), "ci_begin");

    // Phase I: each thread fills its own chunk of rows and pushes it; the device copy overlaps with the sampling
    const double t0 = now();
    {
        const int64_t chunk = std::max<int64_t>(1, (16 << 20) / ((int64_t)M * 4));
        std::vector<std::thread> th;
        std::vector<std::string> errors(num_threads);
        for (int t = 0; t < num_threads; ++t)
            th.emplace_back([&, t]() {
                std::vector<float> rows((size_t)chunk * M), lbars(chunk);
                int64_t held = 0, at = first[t];
                auto flush = [&]() {
                    if (held && errors[t].empty() && rsem_b200_ci_push(ctx, rows.data(), lbars.data(), at, held) != 0)
                        errors[t] = rsem_b200_last_error();
                    at += held;
                    held = 0;
                };
                ci_sample_vectors(cvs[t].data(), (int)(cvs[t].size() / (M + 1)), M, nSpC, pseudoC, seeds[t], eel.data(),
                                  mw.data(), t, g_verbose, [&](int64_t, const float* tpm, float l_bar) {
                                      memcpy(&rows[(size_t)held * M], tpm, (size_t)M * 4);
                                      lbars[held] = l_bar;
                                      if (++held == chunk) flush();
                                  });
                flush();
                std::vector<int32_t>().swap(cvs[t]);
            });
        for (auto& x : th) x.join();
        for (const std::string& e : errors)
            if (!e.empty()) die("rsem_b200: ci_push failed: " + e);
    }
    const double t1 = now();
    if (g_verbose) printf("Sampling is finished!\n");

    std::vector<float> tr((size_t)M * 6), gene((size_t)m * 6), iso((size_t)m_trans * 6);
    rsem_b200_ci_stats st;
    check_rc(rsem_b200_ci_end(ctx, tr.data(), gene.data(), alleleS ? iso.data() : nullptr, &st), "ci_end");
    rsem_b200_ctx_destroy(ctx);
    const double t2 = now();
    if (g_verbose)  // calcCI.cpp:360, per Phase II thread range
        for (size_t i = 0; i + 1 < parts.size(); ++i)
            for (int cnt = 1000; cnt <= parts[i + 1] - parts[i]; cnt += 1000)
                printf("In thread %d, %d genes are processed for CI calculation!\n", (int)i, cnt);

    write_rows(imdName + (alleleS ? ".allele_res" : ".iso_res"), tr.data(), M);
    if (alleleS) write_rows(imdName + ".iso_res", iso.data(), m_trans);
    write_rows(imdName + ".gene_res", gene.data(), m);
    if (g_verbose) printf("All credibility intervals are calculated!\n");
    if (timing)
        fprintf(stderr,
                "rsem-calculate-credibility-intervals timing: sampling (host, %d threads) %.3f s, intervals %.3f s; device: "
                "transpose %.3f s, sums %.3f s, sort %.3f s, intervals %.3f s, %llu blocks, sample matrix %s\n",
                num_threads, t1 - t0, t2 - t1, st.transpose_ms / 1e3, st.sums_ms / 1e3, st.sort_ms / 1e3,
                st.interval_ms / 1e3, (unsigned long long)st.blocks, st.resident ? "on the device" : "in host memory");
    return 0;
}
