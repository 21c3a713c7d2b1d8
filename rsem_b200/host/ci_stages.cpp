// The per-sample stages of rsem-calculate-credibility-intervals (calcCI.cpp), which rsem-calculate-credibility-intervals
// runs once and rsem-calculate-credibility-intervals-batch runs for each manifest line.  Phase I's draws are in
// ffm/ci_sample.cpp (compiled with the reference's flags); Phase II is K8 on the device (csrc/ci_kernels.cu).
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <thread>

#include "host.hpp"

namespace host {

void ci_sample_vectors(const int32_t* cvs, int n_cv, int M, int nSpC, double pseudoC, uint32_t seed, const double* eel,
                       const double* mw, int thread_no, const Say* progress,
                       const std::function<void(int64_t, const float*, float)>& emit);

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

// fn(t) on one thread per t < n; with isolate, die() throws on those threads and the first failure is raised here
void on_threads(int n, bool isolate, const std::function<void(int)>& fn) {
    std::vector<std::string> errors(n);
    std::vector<std::thread> th;
    for (int t = 0; t < n; ++t)
        th.emplace_back([&, t]() {
            DieThrows throws(isolate);
            try {
                fn(t);
            } catch (const std::exception& e) {
                errors[t] = e.what();
            }
        });
    for (auto& x : th) x.join();
    for (const std::string& e : errors)
        if (!e.empty()) die(e);
}

}  // namespace

void load_ci_reference(const std::string& refName, CiReference& ref) {
    ref.name = refName;
    load_refs(refName + ".seq", false, ref.refs);
    load_groups(refName + ".grp", ref.gi);
    ref.alleleS = load_allele_groups(refName, ref.gt, ref.ta);
}

std::string parse_ci_args(const std::vector<std::string>& f, CiArgs& a, bool whole_seed) {
    a.imdName = f[0];
    a.statName = f[1];
    a.confidence = atof(f[2].c_str());
    a.nCV = atoi(f[3].c_str());
    a.nSpC = atoi(f[4].c_str());
    a.nMB = atoi(f[5].c_str());
    for (size_t i = 6; i < f.size(); ++i) {
        const bool arg = i + 1 < f.size();
        if (f[i] == "-p" && arg) a.nThreads = atoi(f[i + 1].c_str());
        if (f[i] == "--seed") {
            if (whole_seed && (!arg || f[i + 1].find_first_not_of("0123456789") != std::string::npos))
                return arg ? "cannot parse seed " + f[i + 1] : "--seed needs a value";
            if (arg) { a.hasSeed = true; a.seed = parse_seed(f[i + 1].c_str()); }
        }
        if (f[i] == "--pseudo-count" && arg) a.pseudoC = atof(f[i + 1].c_str());
        if (f[i] == "-q") a.quiet = true;
    }
    if (a.nThreads < 1) return "Number of threads should be bigger than 0!";
    return "";
}

std::string ci_sample_count_error(const CiArgs& a, int M) {
    if (!(a.nCV > 0 && a.nSpC > 0 && M > 0)) return "nCV and nSpC must be positive!";
    if (a.n_samples() > INT32_MAX) return "nCV * nSpC must be below 2^31!";
    return "";
}

std::string ci_memory_error(const CiArgs& a, int M) {
    // Buffer.h:18-20, in its unsigned 64-bit arithmetic (a negative nMB wraps to a large size and passes)
    uint64_t size = (uint64_t)(int64_t)a.nMB * 1024 * 1024 / sizeof(float) / (uint64_t)M;
    if (size > (uint64_t)a.n_samples()) size = a.n_samples();
    return size == 0 ? "Memory allocated for credibility intervals is not enough!" : "";
}

void load_ci_model(const CiReference& ref, const CiArgs& a, std::vector<double>& eel, std::vector<double>& mw) {
    int model_type = 0;
    LenDistH gld;
    HostModel::read_for_gibbs(a.statName + ".model", ref.refs.M, model_type, gld, mw);
    calc_eel(ref.refs, gld, eel);
}

void load_ci_vectors(const CiArgs& a, int M, CiSample& s, bool isolate) {
    const int n = a.samplers();
    s.cvs.assign(n, {});
    on_threads(n, isolate, [&](int t) { s.cvs[t] = read_count_vectors(a.imdName + ".countvectors" + std::to_string(t), M); });
    s.first.assign(n + 1, 0);
    for (int t = 0; t < n; ++t) s.first[t + 1] = s.first[t] + (int64_t)(s.cvs[t].size() / (M + 1)) * a.nSpC;
    if (s.first[n] != a.n_samples())
        die("The count-vector files hold " + std::to_string(s.first[n] / a.nSpC) + " count vectors, not nCV = " +
            std::to_string(a.nCV) + "!");
}

std::vector<int32_t> ci_parts(int nThreads, int M, const std::vector<int>& gi) {
    const int m = (int)gi.size() - 1;
    std::vector<int32_t> parts{0};
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
    return parts;
}

rsem_b200_ci_params ci_params(const CiReference& ref, const CiArgs& a, const std::vector<int32_t>& parts, uint64_t budget) {
    rsem_b200_ci_params cp;
    memset(&cp, 0, sizeof cp);
    const int64_t nSamples = a.n_samples();
    cp.M = ref.refs.M;
    cp.n_genes = ref.m();
    cp.gene_start = ref.gi.data();
    cp.n_isoforms = ref.m_trans();
    cp.isoform_start = ref.alleleS ? ref.ta.data() : nullptr;
    cp.n_parts = (int)parts.size() - 1;
    cp.part_gene_start = parts.data();
    cp.n_samples = nSamples;
    cp.threshold = (int)(nSamples - ((int)(a.confidence * nSamples - 1e-8) + 1));
    cp.device_budget = budget;
    return cp;
}

double ci_sample_rows(rsem_b200_ctx* ctx, const CiArgs& a, int M, CiSample& s, uint32_t seed, const Say* progress, bool isolate) {
    // one reader per count-vector file, engines from the engineFactory sequence (calcCI.cpp:172-188)
    const int n = a.samplers();
    const std::vector<uint32_t> seeds = engine_seeds(seed, n);
    const int64_t chunk = std::max<int64_t>(1, (16 << 20) / ((int64_t)M * 4));
    std::vector<double> seconds(n, 0.0);
    std::vector<std::string> push_errors(n);
    // each thread fills its own chunk of rows and pushes it; the device copy overlaps with the sampling
    on_threads(n, isolate, [&](int t) {
        const double t0 = now_s();
        std::vector<float> rows((size_t)chunk * M), lbars(chunk);
        int64_t held = 0, at = s.first[t];
        std::string& error = push_errors[t];
        auto flush = [&]() {
            if (held && error.empty() && rsem_b200_ci_push(ctx, rows.data(), lbars.data(), at, held) != 0)
                error = rsem_b200_last_error();
            at += held;
            held = 0;
        };
        ci_sample_vectors(s.cvs[t].data(), (int)(s.cvs[t].size() / (M + 1)), M, a.nSpC, a.pseudoC, seeds[t], s.eel.data(),
                          s.mw.data(), t, progress, [&](int64_t, const float* tpm, float l_bar) {
                              memcpy(&rows[(size_t)held * M], tpm, (size_t)M * 4);
                              lbars[held] = l_bar;
                              if (++held == chunk) flush();
                          });
        flush();
        std::vector<int32_t>().swap(s.cvs[t]);
        seconds[t] = now_s() - t0;
    });
    for (const std::string& e : push_errors)
        if (!e.empty()) die("rsem_b200: ci_push failed: " + e);
    double sum = 0;
    for (double x : seconds) sum += x;
    return sum;
}

void ci_intervals(rsem_b200_ctx* ctx, const CiReference& ref, CiIntervals& out) {
    out.tr.assign((size_t)ref.refs.M * 6, 0.0f);
    out.gene.assign((size_t)ref.m() * 6, 0.0f);
    out.iso.assign((size_t)ref.m_trans() * 6, 0.0f);
    check_rc(rsem_b200_ci_end(ctx, out.tr.data(), out.gene.data(), ref.alleleS ? out.iso.data() : nullptr, &out.st), "ci_end");
}

void write_ci_sample(const CiReference& ref, const CiArgs& a, const std::vector<int32_t>& parts, const CiIntervals& r,
                     const Say* say) {
    if (say)  // calcCI.cpp:360, per Phase II thread range
        for (size_t i = 0; i + 1 < parts.size(); ++i)
            for (int cnt = 1000; cnt <= parts[i + 1] - parts[i]; cnt += 1000)
                (*say)("In thread " + std::to_string(i) + ", " + std::to_string(cnt) + " genes are processed for CI calculation!\n");
    write_rows(a.imdName + (ref.alleleS ? ".allele_res" : ".iso_res"), r.tr.data(), ref.refs.M);
    if (ref.alleleS) write_rows(a.imdName + ".iso_res", r.iso.data(), ref.m_trans());
    write_rows(a.imdName + ".gene_res", r.gene.data(), ref.m());
    if (say) (*say)("All credibility intervals are calculated!\n");
}

}  // namespace host
