// Per-sample stages of rsem-run-em, shared by rsem-run-em and rsem-run-em-batch.
#include <algorithm>
#include <cstdlib>
#include <ctime>

#include "host.hpp"

namespace host {

void load_em_reference(const std::string& refName, EmReference& ref) {
    ref.name = refName;
    load_refs(refName + ".seq", true, ref.refs);
    load_transcripts(refName + ".ti", ref.transcripts, &ref.ti_type);
}

EmArgs parse_em_args(const std::vector<std::string>& f) {
    EmArgs a;
    a.outName = f[0];
    a.imdName = f[1];
    a.statName = f[2];
    for (size_t i = 3; i < f.size(); ++i) {
        const bool arg = i + 1 < f.size();
        if (f[i] == "-p" && arg) a.nThreads = atoi(f[i + 1].c_str());
        if (f[i] == "-b" && arg) { a.genBam = true; a.inpSamF = f[i + 1]; }
        if (f[i] == "-q") a.quiet = true;
        if (f[i] == "--gibbs-out") a.gibbsOut = true;
        if (f[i] == "--sampling") a.bamSampling = true;
        if (f[i] == "--seed" && arg) { a.hasSeed = true; a.seed = parse_seed(f[i + 1].c_str()); }
        if (f[i] == "--append-names") a.appendNames = true;
    }
    return a;
}

bool load_cnt(const std::string& statName, bool must_exist, EmCounts& n) {
    std::vector<char> b = slurp(statName + ".cnt", must_exist);
    b.push_back(0);
    unsigned long long v[4];
    if (sscanf(b.data(), "%llu %llu %llu %llu", &v[0], &v[1], &v[2], &v[3]) != 4) return false;
    n.N0 = v[0]; n.N1 = v[1]; n.N2 = v[2]; n.N_tot = v[3];
    return true;
}

void write_no_alignable_reads(const EmReference& ref, const EmArgs& a, const Say& say) {
    say("Warning: There are no alignable reads!\n");
    FILE* fo = fopen((a.statName + ".theta").c_str(), "w");
    if (fo) fclose(fo);
    fo = fopen((a.statName + ".model").c_str(), "w");
    if (fo) fclose(fo);
    const int M = ref.refs.M;
    std::vector<double> theta(M + 1, 0.0), eel(M + 1, 0.0), countv(M + 1, 0.0);
    for (int i = 1; i <= M; ++i) eel[i] = ref.transcripts[i].length;
    write_results_em(ref.name, a.imdName, ref.transcripts, theta, eel, countv.data(), a.appendNames);
    if (a.genBam) {  // EM.cpp:627-633: the input is copied as it is
        const std::string command = "cp " + a.inpSamF + " " + a.outName + ".transcript.bam";
        say(command + "\n");
        if (system(command.c_str()) != 0) die("Cannot copy " + a.inpSamF + "!");
    }
}

void load_em_hits(const std::string& imdName, int read_type, int M, EmSample& s) {
    s.mp.M = M;
    s.mp.N[0] = s.n.N0; s.mp.N[1] = s.n.N1; s.mp.N[2] = s.n.N2;
    load_mparams(imdName + ".mparams", s.mp);
    // imd.b200, written by bin/rsem-parse-alignments: the same content as .dat + the read files, decoded
    s.have_sidecar = load_sidecar(imdName, read_type, s.sidecar);
    if (s.have_sidecar && (s.sidecar.hits.N != s.n.N1 || s.sidecar.reads[0].n != s.n.N0 || s.sidecar.reads[2].n != s.n.N2 ||
                           s.mp.seedLen > kSidecarShortLen))
        s.have_sidecar = false;   // does not describe this run: parse the text files
    if (s.have_sidecar) s.hits = std::move(s.sidecar.hits);
    else load_dat(imdName + ".dat", read_type, s.n.N1, s.hits);
}

void load_em_model(const std::string& imdName, int read_type, const RefData& refs, EmSample& s, ReadStore& reads, const Say& say) {
    if (g_verbose)
        say("Thread 0 : N = " + std::to_string(s.hits.N) + ", NHit = " + std::to_string(s.hits.H) + "\nEM_init finished!\n");
    if (!(s.n.N_tot > s.n.N2)) die("N_tot must be larger than N2!");
    const int M = refs.M;
    s.theta.assign(M + 1, 0.0);
    s.theta[0] = std::max(s.n.N0 * 1.0 / (s.n.N_tot - s.n.N2), 1e-8);
    for (int i = 1; i <= M; ++i) s.theta[i] = (1.0 - s.theta[0]) / M;
    s.model.init_master(read_type, s.mp, &refs);
    s.model.estimate_from_reads(imdName, reads, s.have_sidecar ? &s.sidecar : nullptr);
    s.sidecar = Sidecar();
    if (reads.n != s.n.N1) die("Read indices files do not match!");
}

std::string round_line(int round, const rsem_b200_round_stats& s) {
    char buf[160];
    snprintf(buf, sizeof buf, "ROUND = %d, SUM = %.15g, bChange = %.6g, totNum = %lld\n", round, s.sum, s.bchange,
             (long long)s.totnum);
    return buf;
}

EmRounds em_model_rounds(rsem_b200_ctx* ctx, HostModel& model, uint64_t N0, int MIN_ROUND, int MAX_ROUND, const OnRound& on_round) {
    const ModelParamsH& mp = model.mp;
    std::vector<double> st_prof(model.n_prof()), st_noise(model.n_noise()), st_gld(mp.maxL - (mp.minL - 1) + 1), st_rspd(mp.B + 2);
    rsem_b200_model_stats mstats;
    mstats.profile = st_prof.data();
    mstats.noise_profile = st_noise.data();
    mstats.gld_pdf = st_gld.data();
    mstats.gld_lb = mp.minL - 1;
    mstats.gld_span = mp.maxL - (mp.minL - 1);
    mstats.rspd_pdf = st_rspd.data();
    auto push_model = [&]() {
        rsem_b200_model abi;
        model.fill_abi(abi);
        check_rc(rsem_b200_set_model(ctx, &abi), "set_model");
    };
    EmRounds r;
    while (r.keep_going && r.round < 10) {   // doesUpdateModel, EM.cpp:307-310
        ++r.round;
        push_model();
        rsem_b200_round_stats rs;
        check_rc(rsem_b200_em_model_round(ctx, (double)N0, &mstats, &rs), "em_model_round");
        model.rebuild(mstats);   // model.init(); collect(); finish()
        on_round(r.round, rs);
        r.totNum = rs.totnum;
        r.keep_going = r.round < MIN_ROUND || (r.totNum > 0 && r.round < MAX_ROUND);
    }
    // calcConProbs with the last model: for the frozen rounds, and for the .ofg when the EM ends here (EM.cpp:421-457)
    push_model();
    check_rc(rsem_b200_calc_conprb(ctx), "calc_conprb");
    return r;
}

void em_frozen_rounds(rsem_b200_ctx* ctx, uint64_t N0, int MIN_ROUND, int MAX_ROUND, EmRounds& r, const OnRound& on_round) {
    const int CHUNK = 32;
    std::vector<rsem_b200_round_stats> cs(CHUNK);
    while (r.keep_going) {
        int32_t ran = 0, stopped = 0;
        check_rc(rsem_b200_em_rounds(ctx, r.round + 1, CHUNK, MIN_ROUND, MAX_ROUND, (double)N0, cs.data(), &ran, &stopped), "em_rounds");
        for (int k = 0; k < ran; ++k) on_round(r.round + 1 + k, cs[k]);
        if (ran > 0) { r.round += ran; r.totNum = cs[ran - 1].totnum; }
        r.keep_going = !stopped;
    }
}

void finish_em_sample(const EmReference& ref, int read_type, const EmArgs& a, EmSample& s, long long totNum, int MAX_ROUND,
                      const std::string& who, int threads, bool verbose, void (*stamp)(const char*)) {
    auto mark = [&](const char* what) { if (stamp) stamp(what); };
    if (totNum > 0)
        fprintf(stderr, "%sWarning: RSEM reaches %d iterations before meeting the convergence criteria.\n", who.c_str(), MAX_ROUND);
    if (a.gibbsOut) write_ofg(a.imdName + ".ofg", ref.refs.M, s.n.N0, s.hits, s.conprb, s.ncpv);
    mark(".ofg written");
    s.counts[0] += s.n.N0;
    write_em_outputs(ref.name, a.imdName, a.statName, ref.refs, ref.transcripts, s.model, s.theta, s.counts, a.appendNames);
    mark(".theta / .model / result rows written");
    if (a.genBam) {
        write_posterior_bam(a.inpSamF, a.outName, read_type, a.bamSampling, a.hasSeed, a.seed, ref.transcripts, ref.ti_type, s.hits,
                            s.post, s.post0, threads, verbose);
        mark("transcript BAM written");
    }
}

std::string time_used_line(time_t t_start) {
    const long t = (long)(time(NULL) - t_start);
    char buf[96];
    snprintf(buf, sizeof buf, "Time Used for EM.cpp : %d h %02d m %02d s\n", int(t / 3600), int(t % 3600 / 60), int(t % 60));
    return buf;
}

// EM.cpp:504-536 + BamWriter::work (BamWriter.h:82-146): every mapped alignment line (pair of lines for paired-end
// reads) takes the next hit's posterior, in .dat order; all lines are written back, mates with read 1 first.
void write_posterior_bam(const std::string& inpSamF, const std::string& outName, int read_type, bool sampling, bool hasSeed,
                         uint32_t seed, const std::vector<TranscriptInfo>& tr, int ti_type, const HitStore& hits,
                         std::vector<double>& post, const std::vector<double>& post0, int threads, bool verbose) {
    if (sampling) {  // one alignment (or the noise entry) per read, drawn from its posterior (EM.cpp:507-531)
        Mt engine(hasSeed ? seed : (uint32_t)time(NULL));
        if (verbose) printf("Begin to sample reads from their posteriors.\n");
        std::vector<double> arr;
        for (uint64_t j = 0; j < hits.N; ++j) {
            const uint64_t fr = hits.row_ptr[j], to = hits.row_ptr[j + 1];
            const int len = (int)(to - fr + 1);
            arr.assign(len, 0.0);
            arr[0] = post0[j];
            for (uint64_t k = fr; k < to; ++k) arr[k - fr + 1] = arr[k - fr] + post[k];
            int id = -1;
            if (!(arr[len - 1] < kEps)) {  // sample(): first index with arr[index] > u * total (sampling.h:50-65)
                const double prb = engine.uniform01() * arr[len - 1];
                int l = 0, r = len - 1;
                while (l <= r) {
                    const int mid = (l + r) / 2;
                    if (arr[mid] <= prb) l = mid + 1;
                    else r = mid - 1;
                }
                if (l >= len) die("sampling: the draw fell outside the cumulative posterior (reference: assert(l < len))");
                id = l;
            }
            for (uint64_t k = fr; k < to; ++k) post[k] = ((int)(k - fr + 1) == id ? 1.0 : 0.0);
        }
        if (verbose) printf("Sampling is finished.\n");
    }
    AlnReader in(inpSamF);
    const std::vector<int> e2i = map_bam_targets(in.ref_names(), tr, ti_type);
    BamWriter out(outName + ".transcript.bam", rsem_bam_header_text(in.header_text()), threads);
    const bool paired = read_type >= 2;
    uint64_t next_hit = 0, cnt = 0;
    auto take_hit = [&](const BamRecord& b) {
        if (next_hit >= hits.H) die("The alignment file has more aligned lines than the .dat file has alignments (reference: assert(hit != NULL))!");
        const int32_t t = b.tid();
        if (t < 0 || t >= (int32_t)e2i.size() || e2i[t] != std::abs(hits.sid[next_hit]))
            die("The alignment file does not match the .dat file (reference: assert(getInternalSid(tid + 1) == hit->getSid()))!");
        return post[next_hit++];
    };
    BamRecord b, b2;
    if (!paired) {
        while (in.next(b)) {
            ++cnt;
            if (verbose && cnt % 1000000 == 0) printf("%llu alignment lines are loaded!\n", (unsigned long long)cnt);
            if (b.mapped()) b.set_alignment_weight(take_hit(b));
            out.write(b);
        }
    } else {
        while (in.next(b) && in.next(b2)) {
            cnt += 2;
            if (verbose && cnt % 1000000 == 0) printf("%llu alignment lines are loaded!\n", (unsigned long long)cnt);
            if (!b.read1()) b.data.swap(b2.data);
            if (b.mapped() && b2.mapped()) {
                const double w = take_hit(b);
                if (b2.tid() != b.tid()) die("The two mates of a read pair align to different transcripts in the alignment file!");
                b.set_alignment_weight(w);
                b2.set_alignment_weight(w);
            }
            out.write(b);
            out.write(b2);
        }
    }
    if (next_hit != hits.H) die("The alignment file has fewer aligned lines than the .dat file has alignments (reference: assert(wrapper.getNextHit() == NULL))!");
    out.close();
    if (verbose) printf("Bam output file is generated!\n");
}


// .theta (EM.cpp:484-500), .model and the result rows (EM.cpp:480-502); counts[0] already holds N0
void write_em_outputs(const std::string& refName, const std::string& imdName, const std::string& statName,
                      const RefData& refs, const std::vector<TranscriptInfo>& transcripts, const HostModel& model,
                      std::vector<double> theta, const std::vector<double>& counts, bool appendNames) {
    FILE* fo = fopen((statName + ".theta").c_str(), "w");
    if (!fo) die("Cannot open " + statName + ".theta for writing!");
    const int M = refs.M;
    std::vector<double> eel;
    fprintf(fo, "%d\n", M + 1);
    for (int i = 0; i < M; ++i) fprintf(fo, "%.15g ", theta[i]);
    fprintf(fo, "%.15g\n", theta[M]);
    calc_eel(refs, model.gld, eel);
    polish_theta(theta, eel, model.mw);
    for (int i = 0; i < M; ++i) fprintf(fo, "%.15g ", theta[i]);
    fprintf(fo, "%.15g\n", theta[M]);
    fclose(fo);
    model.write(statName + ".model");
    write_results_em(refName, imdName, transcripts, theta, eel, counts.data(), appendNames);
}

}  // namespace host
