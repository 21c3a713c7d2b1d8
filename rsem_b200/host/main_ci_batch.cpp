// rsem-calculate-credibility-intervals-batch: many rsem-calculate-credibility-intervals runs against one reference in one
// process.
//
//   rsem-calculate-credibility-intervals-batch reference_name manifest [-q]
//
// Each non-empty manifest line is what rsem-calculate-credibility-intervals takes after reference_name:
//   imdName statName confidence nCV nSpC nMB [-p #Threads] [--seed seed] [--pseudo-count c] [-q]
// and each line appends the rows `rsem-calculate-credibility-intervals reference_name <line>` appends to imdName.iso_res,
// imdName.gene_res (and imdName.allele_res), byte for byte for the same seed; a line without --seed takes time(NULL)
// when its lane starts it.  The reference (.seq lengths, .grp, .gt / .ta) is read once.
//
// There is one lane on RSEM_B200_DEVICE (default 0), or one per entry of RSEM_B200_DEVICES=0,1,... when it lists more
// than one; an entry may repeat a device (0,0,0,0 samples four lines side by side on one card).  The lanes take the
// manifest lines in manifest order from one counter, and a lane runs one sample at a time on its context, which keeps
// K8's buffers from one sample to the next.  Phase I of a sample runs on the line's min(-p, nCV) sampler threads, as in
// rsem-calculate-credibility-intervals; while it samples, runs Phase II and writes, a helper thread loads the lane's next
// sample (the .model and the expected effective lengths, and its count vectors with one parser thread per file).  So a
// run samples on up to (lanes) x min(-p, nCV) host threads at once, next to one thread per lane and, while they load,
// the helper and parser threads: with -p 8, about 8 host cores per lane.
// Each lane's device budget is RSEM_B200_CI_DEVICE_BYTES when it is set, else the device memory free before the first
// context on its device, less 512 MB, divided by the lanes on that device, so that the lanes of one card cannot
// over-commit it.  A sample whose matrix does not fit its lane's budget keeps it in pinned host memory (same rows).
//
// Every manifest line is checked before a context is created or a file written; a refused line ends the run with exit
// status 255 and names the line.  Whether a count-vector file holds the line's count vectors is known only once it has
// been parsed: a failure there, or any other failure of a lane, ends the run (exit status 255) as "device D, sample X
// (<manifest> line N): why" once the other lanes have finished their current samples.  Standard output has one block per
// sample, in manifest order: "== <sample>" and what rsem-calculate-credibility-intervals prints for the line (inside a
// block, the sampler threads' lines in the order they were printed); -q drops the headers and sets every line's -q.
// RSEM_B200_TIMING=1 prints one line per lane to stderr: its device and budget, its samples, the host sampling
// thread-seconds, the summed device phase times and the host time spent loading and in Phase II.
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

constexpr const char* kTool = "rsem-calculate-credibility-intervals-batch";

struct Line : CiArgs {
    int no = 0;   // 1-based line number in the manifest
};

void usage() {
    printf("Usage: rsem-calculate-credibility-intervals-batch reference_name manifest [-q]\n\n");
    printf("  reference_name: reference name\n");
    printf("  manifest: one sample per line: imdName statName confidence nCV nSpC nMB [-p #Threads] [--seed seed] "
           "[--pseudo-count pseudo_count] [-q]\n");
    printf("  -q: set it quiet\n");
    printf("Each line appends the rows rsem-calculate-credibility-intervals appends for it.\n");
    exit(-1);
}

// every manifest line is checked before a context is created and before any output is written
std::vector<Line> read_manifest(const std::string& path, const CiReference& ref) {
    const int M = ref.refs.M;
    std::vector<Line> lines;
    std::map<std::string, int> seen;   // imdName -> the line that appends to its files
    for (const ManifestLine& ml : manifest_lines(path)) {
        const int no = ml.no;
        if (ml.f.size() < 6)
            refuse(path, no, "expected at least 6 fields (imdName statName confidence nCV nSpC nMB [-p #Threads] "
                             "[--seed seed] [--pseudo-count c] [-q]), got " + std::to_string(ml.f.size()));
        Line l;
        l.no = no;
        std::string why = parse_ci_args(ml.f, l, true);
        if (why.empty()) why = ci_sample_count_error(l, M);
        if (why.empty()) why = ci_memory_error(l, M);
        if (!why.empty()) refuse(path, no, why);
        {   // the whole model, as the line's run will read it for the reference's M
            DieThrows throws(true);
            try {
                std::vector<double> eel, mw;
                load_ci_model(ref, l, eel, mw);
            } catch (const std::exception& e) {
                why = e.what();
            }
        }
        if (!why.empty()) refuse(path, no, why);
        for (int t = 0; t < l.samplers(); ++t) {
            const std::string f = l.imdName + ".countvectors" + std::to_string(t);
            if (FILE* fi = fopen(f.c_str(), "r")) fclose(fi);
            else refuse(path, no, "cannot open " + f);
        }
        const std::string key = std::filesystem::absolute(l.imdName).lexically_normal().string();
        auto it = seen.find(key);
        if (it != seen.end())
            refuse(path, no, "imdName " + l.imdName + " is line " + std::to_string(it->second) +
                             "'s too: both would append to its result files");
        seen[key] = no;
        lines.push_back(l);
    }
    return lines;
}

// what every lane reads
struct Run {
    std::string manifest;
    bool verbose = true;
    CiReference ref;
    std::vector<Line> lines;
    std::vector<std::string> block;   // standard output of each sample, written by the lane that ran it
};

struct Lane {
    int device = 0;
    rsem_b200_ctx* ctx = nullptr;
    uint64_t budget = 0;
    std::string where = "no sample yet";   // what the lane is working on, for the failure message
    // RSEM_B200_TIMING=1
    int samples = 0, in_host_memory = 0;
    rsem_b200_ci_stats st{};
    double sampling = 0;      // sampler thread-seconds
    double sampling_wall = 0; // seconds from ci_begin to the end of Phase I
    double intervals = 0;     // seconds in ci_end and writing the rows
    double load = 0;          // helper-thread seconds loading samples
    double load_wait = 0;     // seconds the lane waited for a load
};

struct Loaded {
    CiSample s;
    std::vector<int32_t> parts;
    double seconds = 0;
};

// the samples a lane takes from `claims`, each loaded one sample ahead, run and written on the lane's context.  die()
// throws on the lane's threads (the caller reports the failure with the lane and the sample).
void run_lane(Run& R, Lane& L, Claims& claims) {
    const std::vector<Line>& lines = R.lines;
    const CiReference& ref = R.ref;
    const int M = ref.refs.M;
    auto load = [&](size_t i) {
        DieThrows throws(true);
        auto x = std::make_unique<Loaded>();
        const double t0 = now_s();
        load_ci_model(ref, lines[i], x->s.eel, x->s.mw);
        load_ci_vectors(lines[i], M, x->s, true);
        x->parts = ci_parts(lines[i].nThreads, M, ref.gi);
        x->seconds = now_s() - t0;
        return x;
    };
    std::future<std::unique_ptr<Loaded>> loading;
    size_t i = claims.next();
    if (i < lines.size()) loading = std::async(std::launch::async, load, i);
    while (i < lines.size()) {
        const Line& l = lines[i];
        L.where = sample_at(l.imdName, R.manifest, l.no);
        double t0 = now_s();
        std::unique_ptr<Loaded> x = loading.get();
        L.load_wait += now_s() - t0;
        L.load += x->seconds;
        const size_t next = claims.next();
        if (next < lines.size()) loading = std::async(std::launch::async, load, next);

        const uint32_t seed = l.hasSeed ? l.seed : (uint32_t)time(NULL);
        std::string& block = R.block[i];   // this lane's alone until the lanes have stopped
        std::mutex block_mu;               // the sampler threads print into it side by side
        const Say gen = [&](const std::string& line) {
            std::lock_guard<std::mutex> g(block_mu);
            block += line;
        };
        const Say* say = R.verbose && !l.quiet ? &gen : nullptr;
        if (say) gen("Refs.loadRefs finished!\n");   // rsem-calculate-credibility-intervals has read the reference
        const rsem_b200_ci_params cp = ci_params(ref, l, x->parts, L.budget);
        t0 = now_s();
        check_rc(rsem_b200_ci_begin(L.ctx, &cp), "ci_begin");
        L.sampling += ci_sample_rows(L.ctx, l, M, x->s, seed, say, true);
        const double t1 = now_s();
        if (say) gen("Sampling is finished!\n");
        CiIntervals r;
        ci_intervals(L.ctx, ref, r);
        write_ci_sample(ref, l, x->parts, r, say);
        L.sampling_wall += t1 - t0;
        L.intervals += now_s() - t1;
        L.st.transpose_ms += r.st.transpose_ms;
        L.st.sums_ms += r.st.sums_ms;
        L.st.sort_ms += r.st.sort_ms;
        L.st.interval_ms += r.st.interval_ms;
        L.st.blocks += r.st.blocks;
        L.in_host_memory += r.st.resident ? 0 : 1;
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
    load_ci_reference(argv[1], R.ref);
    R.lines = read_manifest(R.manifest, R.ref);
    R.block.resize(R.lines.size());
    if (R.verbose)
        for (size_t i = 0; i < R.lines.size(); ++i)
            R.block[i] = "== " + sample_at(R.lines[i].imdName, R.manifest, R.lines[i].no) + "\n";
    if (R.lines.empty()) return 0;

    const std::vector<int> devices = gpu_devices();
    std::vector<Lane> lanes(devices.size());
    {
        const LaneContexts lc = open_lanes_measured(devices);
        if (!lc.err.empty()) die(lc.err);
        const char* e = getenv("RSEM_B200_CI_DEVICE_BYTES");
        const uint64_t set = e ? strtoull(e, nullptr, 10) : 0;   // 0 is the default, as unset
        const uint64_t reserve = 512ull << 20;
        for (size_t k = 0; k < lanes.size(); ++k) {
            lanes[k].device = devices[k];
            lanes[k].ctx = lc.ctx[k];
            const uint64_t sharing = std::count(devices.begin(), devices.end(), devices[k]);
            // at least 1: a budget of 0 would have ci_begin read the free memory again
            lanes[k].budget = set ? set : std::max<uint64_t>(1, (lc.free[k] > reserve ? lc.free[k] - reserve : 0) / sharing);
        }
    }
    Claims claims(R.lines.size());
    const double t0 = now_s();
    run_lanes(kTool, lanes, claims, [&](Lane& L) {
        if (lanes.size() > 1) return run_lane(R, L, claims);   // run_lanes reports a failure with the lane
        std::string failed;
        {
            DieThrows throws(true);
            try {
                run_lane(R, L, claims);
            } catch (const std::exception& x) {
                failed = std::string(kTool) + ": device " + std::to_string(L.device) + ", " + L.where + ": " + x.what();
            }
        }
        if (!failed.empty()) die(failed);
    });
    const double wall = now_s() - t0;
    if (getenv("RSEM_B200_TIMING"))
        for (size_t k = 0; k < lanes.size(); ++k) {
            const Lane& L = lanes[k];
            fprintf(stderr, "%s timing: lane %zu, device %d: budget %llu bytes, %d samples (%d with the matrix in host "
                    "memory), run %.3f s; host: sampling %.3f thread-s (%.3f s from ci_begin), intervals + rows %.3f s, "
                    "loading %.3f s (helper thread; waited for %.3f s); device: transpose %.3f s, sums %.3f s, sort %.3f s, "
                    "intervals %.3f s, %llu blocks\n",
                    kTool, k, L.device, (unsigned long long)L.budget, L.samples, L.in_host_memory, wall, L.sampling,
                    L.sampling_wall, L.intervals, L.load, L.load_wait, L.st.transpose_ms / 1e3, L.st.sums_ms / 1e3,
                    L.st.sort_ms / 1e3, L.st.interval_ms / 1e3, (unsigned long long)L.st.blocks);
        }
    for (Lane& L : lanes) rsem_b200_ctx_destroy(L.ctx);
    for (const std::string& b : R.block) fputs(b.c_str(), stdout);
    return 0;
}
