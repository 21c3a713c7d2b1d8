// rsem-simulate-reads-batch: many rsem-simulate-reads runs against one reference in one process.
//
//   rsem-simulate-reads-batch reference_name manifest [-q]
//
// Each non-empty manifest line is what rsem-simulate-reads takes after reference_name:
//   estimated_model_file estimated_isoform_results theta0 N output_name [--seed seed] [-q]
// and each line gets the files `rsem-simulate-reads reference_name <line>` writes, byte for byte for the same seed; a
// line without --seed takes time(NULL) when its lane starts it.  The reference is read once and uploaded once to each
// lane's context (rsem_b200_sim_upload_refs); a lane (a host thread and a CUDA context) runs its samples one after the
// other on that context, which keeps the run's device buffers from one sample to the next.  While the device draws one
// sample, a helper thread loads the lane's next one (model, theta, cumulative tables); the read text is written on a
// second thread one chunk behind the device, as in rsem-simulate-reads.
// There is one lane on RSEM_B200_DEVICE (default 0), or one per entry of RSEM_B200_DEVICES=0,1,... when it lists more
// than one; an entry may repeat a device (0,0,0,0 runs four samples side by side on one card, whose kernels overlap).
// The lanes take the manifest lines in manifest order from one counter.  A sample runs whole on one context, so its
// files do not depend on the lane.  RSEM_B200_SIM_WINDOW applies to every sample.
// Every manifest line is checked before a context is created or a file written; a refused line ends the run with exit
// status 255 and names the line.  The first failure of a lane ends the run (exit status 255) once the other lanes have
// finished their current samples.  Standard output has one block per sample, in manifest order: "== <sample>" and what
// rsem-simulate-reads prints for the line; -q drops the headers and sets every line's -q.
// RSEM_B200_TIMING=1 prints one line per lane to stderr: its device, its samples, the summed device phase times and the
// host time spent loading and writing.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <filesystem>
#include <future>
#include <map>
#include <memory>
#include <mutex>

#include "host.hpp"

using namespace host;

namespace {

struct Line : SimArgs {
    int no = 0;   // 1-based line number in the manifest
};

void usage() {
    printf("Usage: rsem-simulate-reads-batch reference_name manifest [-q]\n\n");
    printf("  reference_name: reference name\n");
    printf("  manifest: one sample per line: estimated_model_file estimated_isoform_results theta0 N output_name [--seed seed] [-q]\n");
    printf("  -q: set it quiet\n");
    printf("Each line writes the files rsem-simulate-reads writes for it.\n");
    exit(-1);
}

// every manifest line is checked before a context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, int M) {
    std::vector<Line> lines;
    std::map<std::string, int> seen;   // output file -> the line that writes it
    for (const ManifestLine& ml : manifest_lines(path)) {
        const int no = ml.no;
        if (ml.f.size() < 5 || ml.f.size() > 8)
            refuse(path, no, "expected 5 to 8 fields (estimated_model_file estimated_isoform_results theta0 N output_name "
                             "[--seed seed] [-q]), got " + std::to_string(ml.f.size()));
        Line l;
        l.no = no;
        const std::string why = parse_sim_args(ml.f, l);
        if (!why.empty()) refuse(path, no, why);
        const int type = sim_model_type(l.modelF);
        if (type == -1) refuse(path, no, "cannot open " + l.modelF);
        if (type < 0) refuse(path, no, "the model type in " + l.modelF + " is not 0, 1, 2 or 3");
        {   // the whole model, as the line's run will read it; its mw block names the reference it was estimated on
            std::string bad;
            int file_M = 0;
            {
                DieThrows throws(true);
                try {
                    HostModel model;
                    model.read(l.modelF, M, &file_M);
                } catch (const std::exception& e) {
                    bad = e.what();
                }
            }
            if (!bad.empty()) refuse(path, no, bad);
            if (file_M != 0 && file_M != M)
                refuse(path, no, "M in " + l.modelF + " is " + std::to_string(file_M) + ", not the reference's (M = " +
                                 std::to_string(M) + ")");
        }
        if (FILE* fi = fopen(l.resultsF.c_str(), "r")) fclose(fi);
        else refuse(path, no, "cannot open " + l.resultsF);
        std::vector<std::string> outs = sim_read_files(l.outName, type);
        for (const char* ext : {".sim.isoforms.results", ".sim.genes.results", ".sim.alleles.results"})
            outs.push_back(l.outName + ext);
        for (const std::string& f : outs) {
            const std::string key = std::filesystem::absolute(f).lexically_normal().string();
            auto it = seen.find(key);
            if (it != seen.end()) refuse(path, no, "its output " + f + " collides with line " + std::to_string(it->second));
            seen[key] = no;
        }
        lines.push_back(l);
    }
    return lines;
}

// what every lane reads
struct Run {
    std::string manifest;
    bool verbose = true;
    SimReference ref;
    std::vector<Line> lines;
    std::vector<std::string> block;   // standard output of each sample, written by the lane that ran it
};

struct Lane {
    int device = 0;
    rsem_b200_ctx* ctx = nullptr;
    bool isolated = false;                 // die() throws on the lane's threads (more than one lane)
    std::string where = "no sample yet";   // what the lane is working on, for the failure message
    // RSEM_B200_TIMING=1
    int samples = 0;
    uint64_t reads = 0;
    rsem_b200_sim_stats st{};
    double load = 0;        // helper-thread seconds loading samples
    double load_wait = 0;   // seconds the lane waited for a load
    double calls = 0;       // seconds in sim_begin / sim_next / sim_end
    double write = 0;       // seconds waiting for read-file writes, and writing the results tables
};

struct Loaded {
    SimSample s;
    double seconds = 0;
};

// the samples a lane takes from `claims`, each loaded one sample ahead, run and written on the lane's context
void run_lane(Run& R, Lane& L, Claims& claims) {
    const std::vector<Line>& lines = R.lines;
    const SimReference& ref = R.ref;
    const RefData& refs = ref.refs;
    const int M = refs.M;
    check_rc(rsem_b200_sim_upload_refs(L.ctx, M, refs.seq_off.data(), refs.seq.data(), refs.tot_len.data(),
                                       refs.full_len.data()), "sim_upload_refs");
    auto sample_of = [&](size_t i) { return sample_at(lines[i].outName, R.manifest, lines[i].no); };
    auto load = [&](size_t i) {
        DieThrows throws(L.isolated);
        auto x = std::make_unique<Loaded>();
        const double t0 = now_s();
        if (!load_sim_sample(ref, lines[i], x->s))
            die(sample_of(i) + ": the results file gives every transcript TPM * effective length 0");
        x->seconds = now_s() - t0;
        return x;
    };
    std::future<std::unique_ptr<Loaded>> loading;
    size_t i = claims.next();
    if (i < lines.size()) loading = std::async(std::launch::async, load, i);
    while (i < lines.size()) {
        const Line& l = lines[i];
        L.where = sample_of(i);
        double t0 = now_s();
        std::unique_ptr<Loaded> x = loading.get();
        L.load_wait += now_s() - t0;
        L.load += x->seconds;
        const size_t next = claims.next();
        if (next < lines.size()) loading = std::async(std::launch::async, load, next);
        const SimSample& s = x->s;

        const uint32_t seed = l.hasSeed ? l.seed : (uint32_t)time(NULL);
        const std::vector<std::string> files = sim_read_files(l.outName, s.model.type);
        const int n_os = (int)files.size();
        FILE* os[2] = {nullptr, nullptr};
        for (int k = 0; k < n_os; ++k) {
            os[k] = fopen(files[k].c_str(), "w");
            if (!os[k]) die("Cannot open " + files[k] + "!");
        }
        std::string& block = R.block[i];   // this lane's alone until the lanes have stopped
        if (R.verbose && !l.quiet) block += "Refs.loadRefs finished!\n";   // rsem-simulate-reads has read the reference
        const Say gen = [&](const std::string& line) { block += line; };
        const rsem_b200_sim_params p = sim_params(ref, s, seed, l.N, false);
        t0 = now_s();
        check_rc(rsem_b200_sim_begin(L.ctx, &p), "sim_begin");
        L.calls += now_s() - t0;
        L.reads += write_sim_reads(
            [&](const char* text[2], uint64_t bytes[2], uint64_t* n) { check_rc(rsem_b200_sim_next(L.ctx, text, bytes, n), "sim_next"); },
            os, n_os, R.verbose && !l.quiet ? &gen : nullptr, L.calls, L.write);
        std::vector<double> counts((size_t)M + 1, 0.0);
        uint64_t resim = 0;
        rsem_b200_sim_stats st{};
        t0 = now_s();
        check_rc(rsem_b200_sim_end(L.ctx, counts.data(), &resim, &st), "sim_end");
        L.calls += now_s() - t0;
        block += "Total number of resimulation is " + std::to_string(resim) + "\n";
        t0 = now_s();
        write_results_simulation(ref.name, l.outName, ref.transcripts, s.eel, counts);
        for (int k = 0; k < n_os; ++k)
            if (fclose(os[k]) != 0) die("Cannot write the simulated reads!");
        L.write += now_s() - t0;
        L.st.generate_ms += st.generate_ms;
        L.st.resolve_ms += st.resolve_ms;
        L.st.reads_ms += st.reads_ms;
        L.st.copy_ms += st.copy_ms;
        L.st.words += st.words;
        L.st.windows += st.windows;
        ++L.samples;
        i = next;
    }
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 3) usage();
    Run R;
    R.manifest = argv[2];
    for (int i = 3; i < argc; ++i)
        if (!strcmp(argv[i], "-q")) R.verbose = false;
    g_verbose = false;   // the lines the run prints go into the samples' blocks
    load_sim_reference(argv[1], R.ref);
    R.lines = read_manifest(R.manifest, R.ref.refs.M);
    R.block.resize(R.lines.size());
    if (R.verbose)
        for (size_t i = 0; i < R.lines.size(); ++i)
            R.block[i] = "== " + sample_at(R.lines[i].outName, R.manifest, R.lines[i].no) + "\n";
    if (R.lines.empty()) return 0;

    const std::vector<int> devices = gpu_devices();
    std::vector<Lane> lanes(devices.size());
    {
        const LaneContexts lc = open_lanes(devices);
        if (!lc.err.empty()) die(lc.err);
        for (size_t k = 0; k < lanes.size(); ++k) {
            lanes[k].device = devices[k];
            lanes[k].ctx = lc.ctx[k];
            lanes[k].isolated = lanes.size() > 1;
        }
    }
    Claims claims(R.lines.size());
    const double t0 = now_s();
    run_lanes("rsem-simulate-reads-batch", lanes, claims, [&](Lane& L) { run_lane(R, L, claims); });
    const double wall = now_s() - t0;
    if (getenv("RSEM_B200_TIMING"))
        for (size_t k = 0; k < lanes.size(); ++k) {
            const Lane& L = lanes[k];
            fprintf(stderr, "rsem-simulate-reads-batch timing: lane %zu, device %d: %d samples, %llu reads, run %.3f s; device: "
                    "stream generation %.3f s (%llu words, overlapped), boundary resolution %.3f s, read generation + "
                    "formatting %.3f s, copy to host %.3f s, windows %llu; host: sim calls %.3f s, loading %.3f s (helper "
                    "thread; waited for %.3f s), waiting for read-file writes + results %.3f s\n",
                    k, L.device, L.samples, (unsigned long long)L.reads, wall, L.st.generate_ms / 1e3,
                    (unsigned long long)L.st.words, L.st.resolve_ms / 1e3, L.st.reads_ms / 1e3, L.st.copy_ms / 1e3,
                    (unsigned long long)L.st.windows, L.calls, L.load, L.load_wait, L.write);
        }
    for (Lane& L : lanes) rsem_b200_ctx_destroy(L.ctx);
    for (const std::string& b : R.block) fputs(b.c_str(), stdout);
    return 0;
}
