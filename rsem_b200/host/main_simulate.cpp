// bin/rsem-simulate-reads: drop-in for the reference's rsem-simulate-reads (simulation.cpp).
//
//   rsem-simulate-reads reference_name estimated_model_file estimated_isoform_results theta0 N output_name
//                       [--seed seed] [-q]
//
// Same argv, files and output as the reference for the same --seed: the reads are drawn on the GPU from the same
// mt19937 stream (csrc/sim_kernels.cu); this file reads the inputs, builds the cumulative tables, writes the read text
// the device returns and the .sim.*.results tables.
//
// RSEM_B200_SIM_WINDOW=<words> sets the device's stream window (tests use small windows to cross many window bounds);
// RSEM_B200_TIMING=1 prints the device time of each phase and the time spent waiting for file writes to stderr.
// RSEM_B200_DEVICES=a,b,... with more than one entry spreads the stream's windows over those devices (an entry may
// repeat: several contexts on one card), with the same output; otherwise RSEM_B200_DEVICE picks the one device.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <future>
#include <sstream>
#include <string>
#include <vector>

#include "host.hpp"

namespace host {
double sim_theta(const std::string& results_path, int M, int offsite, const std::vector<double>& eel,
                 std::vector<double>& theta);
void sim_prefix(const double* in, double* out, int n);
void sim_profile_cdf(const std::vector<double>& p, int rows, std::vector<double>& pc);
void sim_noiseq_cdf(const std::vector<double>& p, std::vector<double>& pc);
void sim_rspd_cdf(const std::vector<double>& pdf, const std::vector<double>& cdf, int B,
                  const std::vector<int32_t>& full_len, std::vector<uint64_t>& off, std::vector<double>& out);
}  // namespace host

using namespace host;

namespace {

// true when a table row that sums to 0 can be sampled: simul::sample then draws a second word (simul.h:29-32), so
// an attempt's length depends on its qualities.  Qualities are followed through the QualDist chain from the initial
// distribution; profile rows are checked for every reachable quality and every reference base.
bool reachable_zero_row(const HostModel& m, const std::vector<double>& qd_init, const std::vector<double>& qd_tran,
                        const std::vector<double>& pro, int pro_rows, const std::vector<double>& noise) {
    auto row_zero = [](const double* row, int n) { return !(row[n - 1] > 0.0); };
    if (!m.hasq()) {
        if (row_zero(noise.data(), 5)) return true;
        for (int i = 0; i < pro_rows * 5; ++i)
            if (row_zero(&pro[(size_t)i * 5], 5)) return true;
        return false;
    }
    if (row_zero(qd_init.data(), 100)) return true;
    std::vector<char> seen(100, 0);
    std::vector<int> todo;
    auto visit = [&](const double* row) {
        for (int q = 0; q < 100; ++q)
            if (row[q] > (q ? row[q - 1] : 0.0) && !seen[q]) { seen[q] = 1; todo.push_back(q); }
    };
    visit(qd_init.data());
    while (!todo.empty()) {
        const int q = todo.back();
        todo.pop_back();
        const double* row = &qd_tran[(size_t)q * 100];
        if (row_zero(row, 100)) return true;
        visit(row);
    }
    for (int q = 0; q < 100; ++q) {
        if (!seen[q]) continue;
        if (row_zero(&noise[(size_t)q * 5], 5)) return true;
        for (int r = 0; r < 5; ++r)
            if (row_zero(&pro[((size_t)q * 5 + r) * 5], 5)) return true;
    }
    return false;
}

void usage() {
    printf("Usage: rsem-simulate-reads reference_name estimated_model_file estimated_isoform_results theta0 N output_name [--seed seed] [-q]\n\n");
    printf("Outputs output_name.fa / .fq (single-end) or output_name_1 / _2 (paired-end), and output_name.sim.isoforms.results, "
           "output_name.sim.genes.results (and output_name.sim.alleles.results for allele-specific references).\n"
           "Read names are rid_dir_sid_pos[_insertL].\n");
    exit(-1);
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 7 || argc > 10) usage();
    bool quiet = false, have_seed = false;
    uint32_t seed = 0;
    for (int i = 7; i < argc; i++) {
        if (!strcmp(argv[i], "-q")) quiet = true;
        if (!strcmp(argv[i], "--seed")) {  // simulation.cpp:176-182: istringstream >> unsigned
            if (i + 1 >= argc) { fprintf(stderr, "rsem-simulate-reads: --seed needs a value\n"); abort(); }
            std::istringstream reader(argv[i + 1]);
            unsigned int s;
            if (!(reader >> s)) { fprintf(stderr, "rsem-simulate-reads: cannot parse seed %s\n", argv[i + 1]); abort(); }
            seed = s;
            have_seed = true;
        }
    }
    g_verbose = !quiet;
    if (!have_seed) seed = (uint32_t)time(NULL);

    const std::string refName = argv[1], modelF = argv[2], resultsF = argv[3], outName = argv[6];
    std::vector<int> gt, ta;
    const bool alleleS = load_allele_groups(refName, gt, ta);
    const int offsite = alleleS ? 6 : 5;

    RefData refs;
    load_refs(refName + ".seq", true, refs);
    const int M = refs.M;
    std::vector<TranscriptInfo> transcripts;
    load_transcripts(refName + ".ti", transcripts);

    int model_type;
    {
        FILE* fi = fopen(modelF.c_str(), "r");
        if (!fi) { fprintf(stderr, "Cannot open %s! It may not exist.\n", modelF.c_str()); exit(-1); }
        if (fscanf(fi, "%d", &model_type) != 1 || model_type < 0 || model_type > 3) die("Cannot parse " + modelF + "!");
        fclose(fi);
    }
    std::vector<double> theta((size_t)M + 1, 0.0);
    theta[0] = atof(argv[4]);
    const long long N = atoi(argv[5]);

    // genOutReadStreams (simulation.cpp:60-84): the read files are created before the model is read
    const bool paired = model_type >= 2, hasq = model_type & 1;
    const int n_os = paired ? 2 : 1;
    FILE* os[2] = {nullptr, nullptr};
    for (int i = 0; i < n_os; ++i) {
        const std::string f = outName + (paired ? "_" + std::to_string(i + 1) : "") + (hasq ? ".fq" : ".fa");
        os[i] = fopen(f.c_str(), "w");
        if (!os[i]) die("Cannot open " + f + "!");
    }

    HostModel model;
    model.read(modelF, M);
    std::vector<double> eel;
    calc_eel(refs, model.gld, eel);
    const double denom = sim_theta(resultsF, M, offsite, eel, theta);
    if (!(denom > kEps)) {  // simulation.cpp:113
        fprintf(stderr, "rsem-simulate-reads: the results file gives every transcript TPM * effective length 0\n");
        abort();
    }

    // startSimulation tables
    std::vector<double> theta_cdf((size_t)M + 1);
    sim_prefix(theta.data(), theta_cdf.data(), M + 1);
    std::vector<double> qd_init, qd_tran, pro, noise;
    if (hasq) {
        qd_init.resize(100);
        qd_tran.resize(100 * 100);
        sim_prefix(model.qd_init.data(), qd_init.data(), 100);
        for (int i = 0; i < 100; ++i) sim_prefix(&model.qd_tran[(size_t)i * 100], &qd_tran[(size_t)i * 100], 100);
        sim_noiseq_cdf(model.noise_p, noise);
    } else {
        noise.resize(5);
        sim_prefix(model.noise_p.data(), noise.data(), 5);
    }
    const int pro_rows = hasq ? 100 : model.pro_len;
    sim_profile_cdf(model.profile, pro_rows, pro);
    std::vector<uint64_t> rspd_off;
    std::vector<double> rspd_cdf;
    if (model.mp.estRSPD) sim_rspd_cdf(model.rspd_pdf, model.rspd_cdf, model.mp.B, refs.full_len, rspd_off, rspd_cdf);
    std::vector<uint64_t> seq_off(refs.seq_off.begin(), refs.seq_off.end());

    rsem_b200_sim_params p;
    memset(&p, 0, sizeof p);
    p.model_type = model_type;
    p.M = M;
    p.seed = seed;
    p.exact_body = reachable_zero_row(model, qd_init, qd_tran, pro, pro_rows, noise);
    p.N = N > 0 ? (uint64_t)N : 0;
    const char* win = getenv("RSEM_B200_SIM_WINDOW");
    p.window_words = win ? strtoull(win, nullptr, 10) : 0;
    p.theta_cdf = theta_cdf.data();
    p.ori_prob0 = model.ori[0];
    p.gld = rsem_b200_lendist{model.gld.lb, model.gld.ub, model.gld.span, model.gld.pdf.data(), model.gld.cdf.data()};
    p.has_mld = model.has_mld;
    if (model.has_mld)
        p.mld = rsem_b200_lendist{model.mld.lb, model.mld.ub, model.mld.span, model.mld.pdf.data(), model.mld.cdf.data()};
    p.est_rspd = model.mp.estRSPD;
    p.rspd_off = rspd_off.data();
    p.rspd_cdf = rspd_cdf.data();
    p.qd_init_cdf = qd_init.data();
    p.qd_tran_cdf = qd_tran.data();
    p.pro_rows = pro_rows;
    p.profile_cdf = pro.data();
    p.noise_cdf = noise.data();
    p.seq_off = seq_off.data();
    p.seq = refs.seq.data();
    p.tot_len = refs.tot_len.data();
    p.full_len = refs.full_len.data();

    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t_dev = 0, t_io = 0;

    const std::vector<int> devices = gpu_devices();
    rsem_b200_ctx* ctx = nullptr;
    LaneContexts lanes;
    rsem_b200_sim_multi* multi = nullptr;
    if (devices.size() > 1) {
        lanes = open_lanes(devices);
        if (!lanes.err.empty()) die(lanes.err);
        check_rc(rsem_b200_sim_begin_devices(lanes.ctx.data(), (int)lanes.ctx.size(), &p, &multi), "sim_begin_devices");
    } else {
        const char* dev = getenv("RSEM_B200_DEVICE");
        check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
        check_rc(rsem_b200_sim_begin(ctx, &p), "sim_begin");
    }
    // the read text of one chunk is written on a second thread while the device produces the next chunk (the library
    // keeps a chunk's buffers until the second following sim_next)
    uint64_t done = 0;
    std::future<bool> writing;
    auto finish_write = [&]() {
        if (writing.valid() && !writing.get()) die("Cannot write the simulated reads!");
    };
    for (;;) {
        const char* text[2];
        uint64_t bytes[2], n = 0;
        double t0 = now();
        if (multi) check_rc(rsem_b200_sim_next_devices(multi, text, bytes, &n), "sim_next_devices");
        else check_rc(rsem_b200_sim_next(ctx, text, bytes, &n), "sim_next");
        t_dev += now() - t0;
        t0 = now();
        finish_write();
        t_io += now() - t0;  // time the device loop waited for the previous chunk's write
        if (n == 0) break;
        if (g_verbose)  // simulation.cpp:125
            for (uint64_t k = done / 1000000 + 1; k * 1000000 <= done + n; ++k) {
                printf("GEN %llu\n", (unsigned long long)(k * 1000000));
                fflush(stdout);
            }
        done += n;
        writing = std::async(std::launch::async, [&os, n_os, text0 = text[0], text1 = text[1], b0 = bytes[0], b1 = bytes[1]]() {
            const char* tx[2] = {text0, text1};
            const uint64_t by[2] = {b0, b1};
            for (int i = 0; i < n_os; ++i)
                if (fwrite(tx[i], 1, by[i], os[i]) != by[i]) return false;
            return true;
        });
    }
    std::vector<double> counts((size_t)M + 1, 0.0);
    uint64_t resim = 0;
    rsem_b200_sim_stats st;
    rsem_b200_sim_devices_stats dst{};
    std::vector<rsem_b200_sim_stats> per(lanes.ctx.size());
    if (multi) {
        check_rc(rsem_b200_sim_end_devices(multi, counts.data(), &resim, &dst, per.data()), "sim_end_devices");
        st = dst.sum;
        for (rsem_b200_ctx* c : lanes.ctx) rsem_b200_ctx_destroy(c);
    } else {
        check_rc(rsem_b200_sim_end(ctx, counts.data(), &resim, &st), "sim_end");
        rsem_b200_ctx_destroy(ctx);
    }
    printf("Total number of resimulation is %llu\n", (unsigned long long)resim);
    fflush(stdout);

    write_results_simulation(refName, outName, transcripts, eel, counts);
    for (int i = 0; i < n_os; ++i) {
        const double t0 = now();
        if (fclose(os[i]) != 0) die("Cannot write the simulated reads!");
        t_io += now() - t0;
    }
    if (timing)
        fprintf(stderr,
                "rsem-simulate-reads timing: reads %llu, sim_next %.3f s, waiting for read-file writes %.3f s; device: "
                "stream generation %.3f s (%llu words, %.3g words/s, overlapped), boundary resolution %.3f s, read "
                "generation + formatting %.3f s, copy to host %.3f s, windows %llu\n",
                (unsigned long long)done, t_dev, t_io, st.generate_ms / 1e3, (unsigned long long)st.words,
                st.generate_ms > 0 ? st.words / (st.generate_ms / 1e3) : 0.0, st.resolve_ms / 1e3, st.reads_ms / 1e3,
                st.copy_ms / 1e3, (unsigned long long)st.windows);
    if (timing && multi) {
        fprintf(stderr, "rsem-simulate-reads timing: %zu devices (times summed over them): mt19937 jumps %.3f s "
                "(overlapped), waiting for each window's entry point %.3f s\n", per.size(), dst.jump_ms / 1e3,
                dst.handoff_ms / 1e3);
        for (size_t g = 0; g < per.size(); ++g)
            fprintf(stderr, "rsem-simulate-reads timing: device %d (entry %zu): stream generation %.3f s (%llu words), "
                    "boundary resolution %.3f s, read generation + formatting %.3f s, copy to host %.3f s, windows %llu\n",
                    devices[g], g, per[g].generate_ms / 1e3, (unsigned long long)per[g].words, per[g].resolve_ms / 1e3,
                    per[g].reads_ms / 1e3, per[g].copy_ms / 1e3, (unsigned long long)per[g].windows);
    }
    return 0;
}
