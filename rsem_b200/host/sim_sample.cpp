// The per-sample stages of rsem-simulate-reads (simulation.cpp), shared by bin/rsem-simulate-reads and
// bin/rsem-simulate-reads-batch: the arguments, the reference, the model and the cumulative tables of a sample, the run's
// parameters, and the loop that writes the read text the device returns.
#include <cstdlib>
#include <cstring>
#include <future>
#include <sstream>

#include "host.hpp"

namespace host {
double sim_theta(const std::string& results_path, int M, int offsite, const std::vector<double>& eel,
                 std::vector<double>& theta);
void sim_prefix(const double* in, double* out, int n);
void sim_profile_cdf(const std::vector<double>& p, int rows, std::vector<double>& pc);
void sim_noiseq_cdf(const std::vector<double>& p, std::vector<double>& pc);
void sim_rspd_cdf(const std::vector<double>& pdf, const std::vector<double>& cdf, int B,
                  const std::vector<int32_t>& full_len, std::vector<uint64_t>& off, std::vector<double>& out);

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

}  // namespace

void load_sim_reference(const std::string& refName, SimReference& ref) {
    ref.name = refName;
    ref.alleleS = load_allele_groups(refName, ref.gt, ref.ta);
    ref.offsite = ref.alleleS ? 6 : 5;
    load_refs(refName + ".seq", true, ref.refs);
    load_transcripts(refName + ".ti", ref.transcripts);
}

std::string parse_sim_args(const std::vector<std::string>& f, SimArgs& a) {
    a.modelF = f[0];
    a.resultsF = f[1];
    a.theta0 = atof(f[2].c_str());
    a.N = atoi(f[3].c_str());
    a.outName = f[4];
    for (size_t i = 5; i < f.size(); ++i) {
        if (f[i] == "-q") a.quiet = true;
        if (f[i] == "--seed") {  // simulation.cpp:176-182: istringstream >> unsigned
            if (i + 1 >= f.size()) return "--seed needs a value";
            std::istringstream reader(f[i + 1]);
            unsigned int s;
            if (!(reader >> s)) return "cannot parse seed " + f[i + 1];
            a.seed = s;
            a.hasSeed = true;
        }
    }
    return "";
}

int sim_model_type(const std::string& modelF) {
    FILE* fi = fopen(modelF.c_str(), "r");
    if (!fi) return -1;
    int type = -1;
    const bool ok = fscanf(fi, "%d", &type) == 1 && type >= 0 && type <= 3;
    fclose(fi);
    return ok ? type : -2;
}

std::vector<std::string> sim_read_files(const std::string& outName, int model_type) {
    const bool paired = model_type >= 2, hasq = model_type & 1;
    std::vector<std::string> files;
    for (int i = 0; i < (paired ? 2 : 1); ++i)
        files.push_back(outName + (paired ? "_" + std::to_string(i + 1) : "") + (hasq ? ".fq" : ".fa"));
    return files;
}

bool load_sim_sample(const SimReference& ref, const SimArgs& a, SimSample& s) {
    const RefData& refs = ref.refs;
    const int M = refs.M;
    HostModel& model = s.model;
    model.read(a.modelF, M);
    calc_eel(refs, model.gld, s.eel);
    s.theta.assign((size_t)M + 1, 0.0);
    s.theta[0] = a.theta0;
    const double denom = sim_theta(a.resultsF, M, ref.offsite, s.eel, s.theta);
    if (!(denom > kEps)) return false;  // simulation.cpp:113

    // startSimulation tables
    const bool hasq = model.hasq();
    s.theta_cdf.resize((size_t)M + 1);
    sim_prefix(s.theta.data(), s.theta_cdf.data(), M + 1);
    if (hasq) {
        s.qd_init.resize(100);
        s.qd_tran.resize(100 * 100);
        sim_prefix(model.qd_init.data(), s.qd_init.data(), 100);
        for (int i = 0; i < 100; ++i) sim_prefix(&model.qd_tran[(size_t)i * 100], &s.qd_tran[(size_t)i * 100], 100);
        sim_noiseq_cdf(model.noise_p, s.noise);
    } else {
        s.noise.resize(5);
        sim_prefix(model.noise_p.data(), s.noise.data(), 5);
    }
    s.pro_rows = hasq ? 100 : model.pro_len;
    sim_profile_cdf(model.profile, s.pro_rows, s.pro);
    if (model.mp.estRSPD) sim_rspd_cdf(model.rspd_pdf, model.rspd_cdf, model.mp.B, refs.full_len, s.rspd_off, s.rspd_cdf);
    s.exact_body = reachable_zero_row(model, s.qd_init, s.qd_tran, s.pro, s.pro_rows, s.noise);
    return true;
}

rsem_b200_sim_params sim_params(const SimReference& ref, const SimSample& s, uint32_t seed, long long N, bool with_seq) {
    const HostModel& model = s.model;
    const RefData& refs = ref.refs;
    rsem_b200_sim_params p;
    memset(&p, 0, sizeof p);
    p.model_type = model.type;
    p.M = refs.M;
    p.seed = seed;
    p.exact_body = s.exact_body;
    p.N = N > 0 ? (uint64_t)N : 0;
    const char* win = getenv("RSEM_B200_SIM_WINDOW");
    p.window_words = win ? strtoull(win, nullptr, 10) : 0;
    p.theta_cdf = s.theta_cdf.data();
    p.ori_prob0 = model.ori[0];
    p.gld = rsem_b200_lendist{model.gld.lb, model.gld.ub, model.gld.span, model.gld.pdf.data(), model.gld.cdf.data()};
    p.has_mld = model.has_mld;
    if (model.has_mld)
        p.mld = rsem_b200_lendist{model.mld.lb, model.mld.ub, model.mld.span, model.mld.pdf.data(), model.mld.cdf.data()};
    p.est_rspd = model.mp.estRSPD;
    p.rspd_off = s.rspd_off.data();
    p.rspd_cdf = s.rspd_cdf.data();
    p.qd_init_cdf = s.qd_init.data();
    p.qd_tran_cdf = s.qd_tran.data();
    p.pro_rows = s.pro_rows;
    p.profile_cdf = s.pro.data();
    p.noise_cdf = s.noise.data();
    if (with_seq) {
        p.seq_off = refs.seq_off.data();
        p.seq = refs.seq.data();
        p.tot_len = refs.tot_len.data();
        p.full_len = refs.full_len.data();
    }
    return p;
}

uint64_t write_sim_reads(const SimNext& next, FILE* const* os, int n_os, const Say* gen, double& t_next, double& t_write) {
    // the library keeps a chunk's buffers until the second following call, so one chunk is written while the device
    // produces the next
    uint64_t done = 0;
    std::future<bool> writing;
    auto finish_write = [&]() {
        if (writing.valid() && !writing.get()) die("Cannot write the simulated reads!");
    };
    for (;;) {
        const char* text[2];
        uint64_t bytes[2], n = 0;
        double t0 = now_s();
        next(text, bytes, &n);
        t_next += now_s() - t0;
        t0 = now_s();
        finish_write();
        t_write += now_s() - t0;  // time the device loop waited for the previous chunk's write
        if (n == 0) break;
        if (gen)  // simulation.cpp:125
            for (uint64_t k = done / 1000000 + 1; k * 1000000 <= done + n; ++k)
                (*gen)("GEN " + std::to_string(k * 1000000) + "\n");
        done += n;
        writing = std::async(std::launch::async, [os, n_os, text0 = text[0], text1 = text[1], b0 = bytes[0], b1 = bytes[1]]() {
            const char* tx[2] = {text0, text1};
            const uint64_t by[2] = {b0, b1};
            for (int i = 0; i < n_os; ++i)
                if (fwrite(tx[i], 1, by[i], os[i]) != by[i]) return false;
            return true;
        });
    }
    return done;
}

}  // namespace host
