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
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <string>
#include <vector>

#include "host.hpp"

using namespace host;

namespace {

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
    SimArgs a;
    {
        const std::string why = parse_sim_args(std::vector<std::string>(argv + 2, argv + argc), a);
        if (!why.empty()) { fprintf(stderr, "rsem-simulate-reads: %s\n", why.c_str()); abort(); }
    }
    g_verbose = !a.quiet;
    const uint32_t seed = a.hasSeed ? a.seed : (uint32_t)time(NULL);

    SimReference ref;
    load_sim_reference(argv[1], ref);
    const int M = ref.refs.M;

    const int model_type = sim_model_type(a.modelF);
    if (model_type == -1) { fprintf(stderr, "Cannot open %s! It may not exist.\n", a.modelF.c_str()); exit(-1); }
    if (model_type < 0) die("Cannot parse " + a.modelF + "!");

    // genOutReadStreams (simulation.cpp:60-84): the read files are created before the model is read
    const std::vector<std::string> files = sim_read_files(a.outName, model_type);
    const int n_os = (int)files.size();
    FILE* os[2] = {nullptr, nullptr};
    for (int i = 0; i < n_os; ++i) {
        os[i] = fopen(files[i].c_str(), "w");
        if (!os[i]) die("Cannot open " + files[i] + "!");
    }

    SimSample sample;
    if (!load_sim_sample(ref, a, sample)) {
        fprintf(stderr, "rsem-simulate-reads: the results file gives every transcript TPM * effective length 0\n");
        abort();
    }
    const rsem_b200_sim_params p = sim_params(ref, sample, seed, a.N, true);

    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
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
    const Say gen = [](const std::string& line) {
        fputs(line.c_str(), stdout);
        fflush(stdout);
    };
    const uint64_t done = write_sim_reads(
        [&](const char* text[2], uint64_t bytes[2], uint64_t* n) {
            if (multi) check_rc(rsem_b200_sim_next_devices(multi, text, bytes, n), "sim_next_devices");
            else check_rc(rsem_b200_sim_next(ctx, text, bytes, n), "sim_next");
        },
        os, n_os, g_verbose ? &gen : nullptr, t_dev, t_io);
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

    write_results_simulation(ref.name, a.outName, ref.transcripts, sample.eel, counts);
    for (int i = 0; i < n_os; ++i) {
        const double t0 = now_s();
        if (fclose(os[i]) != 0) die("Cannot write the simulated reads!");
        t_io += now_s() - t0;
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
