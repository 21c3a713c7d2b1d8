// Host side of the drop-in executables rsem-run-em / rsem-run-gibbs.
//
// Everything here is O(input) parsing, O(table) model bookkeeping and O(M) output math; all per-hit
// and per-read arithmetic runs on the GPU through the C ABI (include/rsem_b200.h).
// File formats and semantics follow the reference (citations per function, paths relative to
// /root/reference); the code structure does not: one table-oriented HostModel instead of four
// template classes, SoA read/hit stores instead of streams of objects.
#pragma once

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <ctime>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "rsem_b200.h"

namespace host {

constexpr double kEps = 1e-300;     // utils.h:18 EPSILON
constexpr double kMinEel = 1.0;     // utils.h:19 MINEEL
constexpr int kOlen = 25;           // utils.h:23 OLEN
constexpr int kRange = 201;         // utils.h:22 RANGE

extern bool g_verbose;
extern int g_io_threads;  // host threads used for parsing / formatting (rsem-run-em: -p; RSEM_B200_IO_THREADS overrides)

// fn(begin, end, part) over [0, n) split into `parts` contiguous ranges, one std::thread each
void parallel_ranges(size_t n, int parts, const std::function<void(size_t, size_t, int)>& fn);

[[noreturn]] void die(const std::string& msg);          // message to stderr, exit(-1) (my_assert.h:34-41)
void check_rc(int rc, const char* what);                // C-ABI error -> die(rsem_b200_last_error())

// ---- reference transcripts: ref.seq (RefSeq.h:108-127), ref.ti (Transcript.h:119-146), ref.grp ----
struct RefData {
    int M = 0;
    bool has_polyA = false;
    std::vector<uint64_t> seq_off;   // M + 2 (index 0 unused)
    std::vector<uint8_t> seq;        // base codes, forward strand, totLen per transcript
    std::vector<int32_t> full_len, tot_len;  // M + 1
    std::vector<uint64_t> mask_off;  // M + 1
    std::vector<uint32_t> mask_words;
    bool mask(int sid, int p) const { return (mask_words[mask_off[sid] + p / 32] >> (p % 32)) & 1u; }
};
void load_refs(const std::string& path, bool with_seqs, RefData& out);  // Refs::loadRefs, Refs.h:118-145

struct TranscriptInfo {
    std::string transcript_id, transcript_name, gene_id, gene_name, seqname;
    int length = 0;
    char strand = '+';
    std::vector<std::pair<int, int>> exons;   // (start, end), 1-based inclusive, as the file lists them
    int exon_length = 0;                      // sum of the exon lengths
};
// index 1..M; *type = 0 from a genome, 1 stand-alone transcriptome, 2 allele-specific (Transcripts.h:75)
void load_transcripts(const std::string& path, std::vector<TranscriptInfo>& out, int* type = nullptr);
void load_groups(const std::string& path, std::vector<int>& starts);               // GroupInfo.h:34-53
bool load_allele_groups(const std::string& ref_name, std::vector<int>& gt, std::vector<int>& ta);  // WriteResults.h:106-123
// Transcripts::buildMappings (Transcripts.h:105-143): BAM reference index -> transcript id 1..M (by transcript_id, by
// seqname for an allele-specific reference), with the reference's errors and warning
std::vector<int> map_bam_targets(const std::vector<std::string>& names, const std::vector<TranscriptInfo>& tr, int ti_type);

// ---- reads (SingleRead(Q).h, PairedEndRead(Q).h, ReadReader.h) ------------------------------------
struct ReadStore {
    int n_mates = 1;
    bool has_qual = false;
    uint64_t n = 0;
    std::vector<uint64_t> off[2];
    std::vector<uint8_t> base[2], qual[2];
    std::vector<uint8_t> lowq;
};
// Parses a whole read set (tag 0 "un", 1 "alignable", 2 "max"; utils.h:129-149) with g_io_threads threads.
// calc_lq as SingleReadQ.h:63-95 / PairedEndReadQ.h:58-65.
void parse_reads(const std::string& imd_name, int tag, int read_type, bool has_polyA, int seed_len, ReadStore& out,
                 std::vector<std::string>* short_names, uint64_t* n_short);

// ---- hits: imd.dat (HitContainer.h:62-79, parseIt.cpp:197-211) -----------------------------------
struct HitStore {
    uint64_t N = 0, H = 0;
    std::vector<uint64_t> row_ptr;
    std::vector<int32_t> sid, pos, insertL;
};
void load_dat(const std::string& path, int read_type, uint64_t expect_n1, HitStore& out);

// ---- binary side-car imd.b200 (sidecar.cpp): the hand-off from bin/rsem-parse-alignments to bin/rsem-run-em -----------
// The text files (.dat, read files) stay the contract and are always written; the side-car holds the same content in the
// layout rsem-run-em uploads (CSR + SoA hit fields, base / quality codes with offsets), so the text parse
// (HitContainer.h:62-79, the ReadReader loops of EM.cpp:195-202) is skipped when it is present and still describes
// the text files (sizes recorded in its header).  RSEM_B200_SIDECAR=0 disables writing and reading it.
struct ShortRead { uint64_t index; std::string name; };
struct Sidecar {
    int read_type = 0;
    HitStore hits;
    ReadStore reads[3];                    // tag 0 "un", 1 "alignable", 2 "max"; lowq is NOT stored (needs seedLen / polyA)
    std::vector<ShortRead> shorts[3];      // names of the reads with a mate shorter than kSidecarShortLen (for the warnings)
};
constexpr int kSidecarShortLen = 64;
bool sidecar_enabled();
void write_sidecar(const std::string& imd_name, const Sidecar& sc);
bool load_sidecar(const std::string& imd_name, int read_type, Sidecar& out);   // false: absent, stale or disabled
// lowq flags and the short-read names from codes, as parse_reads derives them from text
void finish_sidecar_reads(ReadStore& rs, const std::vector<ShortRead>& shorts, bool has_polyA, int seed_len,
                          std::vector<std::string>* short_names, uint64_t* n_short);

// imd.ofg (EM.cpp:435-457 writer, Gibbs.cpp:101-137 reader); both split the rows over g_io_threads
void write_ofg(const std::string& path, int M, uint64_t N0, const HitStore& h, const std::vector<double>& conprb,
               const std::vector<double>& ncpv);
// load_ofg first tries the binary side-car `path`.b200 that write_ofg leaves next to the text (same rows, the doubles
// the text denotes); it is used only while its recorded size of the text file still matches
void load_ofg(const std::string& path, int M, uint64_t& N0, std::vector<uint64_t>& row_ptr, std::vector<int32_t>& sid,
              std::vector<double>& conprb, bool allow_sidecar = true);

// ---- model -------------------------------------------------------------------------------------
struct LenDistH {  // LenDist.h
    int lb = 0, ub = 1000, span = 1000;
    std::vector<double> pdf, cdf;
    LenDistH() { reset(1, 1000); }
    void reset(int minL, int maxL);         // constructor LenDist.h:17-32 (uniform)
    void zero();                            // init()
    void finish();                          // normalise + cdf + trim (LenDist.h:186-200)
    void trim();                            // LenDist.h:265-294
    void set_as_normal(double mean, double sd, int minL, int maxL);  // LenDist.h:91-179
    double prob(int len) const { return pdf[len - lb]; }
    double adj(int len, int refL) const;    // getAdjustedProb
    double adj_cum(int len, int refL) const;  // getAdjustedCumulativeProb
    int minL() const { return lb + 1; }
    int maxL() const { return ub; }
    void write(FILE* fo) const;             // LenDist.h:237-243
    void read(FILE* fi);                    // LenDist.h:221-235
};

struct ModelParamsH {  // ModelParams.h + imd.mparams
    int M = 0;
    uint64_t N[3] = {0, 0, 0};
    int minL = 1, maxL = 1000, B = 20, mate_minL = 1, mate_maxL = 1000, seedLen = 0;
    bool estRSPD = false;
    double probF = 0.5, mean = -1, sd = 0;
};
void load_mparams(const std::string& path, ModelParamsH& p);  // EM.cpp:647-658

struct HostModel {
    int type = 0;  // 0..3
    ModelParamsH mp;
    const RefData* refs = nullptr;
    double ori[2] = {0.5, 0.5};
    LenDistH gld, mld;
    bool has_mld = false;
    // RSPD (RSPD.h)
    std::vector<double> rspd_pdf, rspd_cdf;  // B + 2
    // QualDist (QualDist.h), Q models only
    std::vector<double> qd_init, qd_tran;
    // Profile / QProfile
    int pro_len = 0;
    std::vector<double> profile;
    // Noise(Q)Profile: p and the N0 counts c
    std::vector<double> noise_p, noise_c;
    std::vector<double> mw;  // M + 1

    bool hasq() const { return type & 1; }
    bool paired() const { return type >= 2; }
    size_t n_prof() const { return hasq() ? 2500 : (size_t)pro_len * 25; }
    size_t n_noise() const { return hasq() ? 500 : 5; }

    void init_master(int model_type, const ModelParamsH& p, const RefData* refs);  // Model(ModelParams&, true)
    // estimateFromReads; `sc` (optional) supplies the read sets already decoded (binary side-car)
    void estimate_from_reads(const std::string& imd_name, ReadStore& alignable, Sidecar* sc = nullptr);
    // init(); collect(helpers); finish()  (EM.cpp:400-404) from the device sufficient statistics
    void rebuild(const rsem_b200_model_stats& st);
    void calc_mw();
    double rspd_eval_cdf(int fpos, int fullLen) const;
    double rspd_adj(int fpos, int effL, int fullLen) const;
    void fill_abi(rsem_b200_model& m) const;
    void write(const std::string& path) const;   // Model::write
    // Model::read for rsem-run-gibbs: only gld and mw are needed afterwards, but the whole file is parsed
    static void read_for_gibbs(const std::string& path, int M, int& model_type, LenDistH& gld, std::vector<double>& mw);
    // the whole .model file, every model type (rsem-simulate-reads); mw stays empty when the file has none for M.
    // file_M (optional): the transcript count the file's mw block is written for, 0 when it has none
    void read(const std::string& path, int M, int* file_M = nullptr);
};

// ---- O(M) result math (WriteResults.h:24-104) ------------------------------------------------------
void calc_eel(const RefData& refs, const LenDistH& gld, std::vector<double>& eel);
void polish_theta(std::vector<double>& theta, const std::vector<double>& eel, const std::vector<double>& mw);
void expression_values(const std::vector<double>& theta, const std::vector<double>& eel, std::vector<double>& tpm,
                       std::vector<double>& fpkm);
void write_results_em(const std::string& ref_name, const std::string& imd_name, const std::vector<TranscriptInfo>& tr,
                      const std::vector<double>& theta, const std::vector<double>& eel, const double* counts,
                      bool append_names);  // WriteResults.h:125-355
// Where a per-sample stage sends its progress lines: stdout for the single-sample tools, the sample's block in the batch tools
using Say = std::function<void(const std::string&)>;

// ---- em_sample.cpp: the per-sample stages of rsem-run-em, which rsem-run-em-batch runs for each manifest line ----------
struct EmReference {   // refName.seq (with the sequences) and refName.ti
    std::string name;
    RefData refs;
    std::vector<TranscriptInfo> transcripts;
    int ti_type = 0;
};
void load_em_reference(const std::string& refName, EmReference& ref);
// rsem-run-em's arguments from sampleName on: sampleName imdName statName [options] (EM.cpp:578-600); -p and -q are only
// recorded here, rsem-run-em-batch ignores them on a manifest line
struct EmArgs {
    std::string outName, imdName, statName, inpSamF;
    bool genBam = false, bamSampling = false, gibbsOut = false, hasSeed = false, appendNames = false, quiet = false;
    uint32_t seed = 0;
    int nThreads = 1;
};
EmArgs parse_em_args(const std::vector<std::string>& f);   // f.size() >= 3
struct EmCounts { uint64_t N0 = 0, N1 = 0, N2 = 0, N_tot = 0; };
bool load_cnt(const std::string& statName, bool must_exist, EmCounts& n);   // statName.cnt; false: cannot be parsed
// N1 == 0 (EM.cpp:615-638): empty .theta / .model, zero result rows, with -b the input copied as it is; `say` gets the
// warning and the cp command
void write_no_alignable_reads(const EmReference& ref, const EmArgs& a, const Say& say);
// a sample from its counts to its outputs
struct EmSample {
    EmCounts n;
    ModelParamsH mp;
    Sidecar sidecar;             // imdName.b200 while it describes this sample, until the model is estimated
    bool have_sidecar = false;
    HitStore hits;
    HostModel model;
    std::vector<double> theta;   // the initial θ (EM.cpp:342-346), then the final one
    std::vector<double> counts, conprb, ncpv, post, post0;   // expected counts without N0, .ofg inputs, -b posteriors
};
// imdName.mparams and the hits: from the side-car when it describes this sample, else from imdName.dat
void load_em_hits(const std::string& imdName, int read_type, int M, EmSample& s);
// then the initial θ, the master model and estimateFromReads (EM.cpp:97-174, 342-346); the alignable reads go to `reads`
void load_em_model(const std::string& imdName, int read_type, const RefData& refs, EmSample& s, ReadStore& reads, const Say& say);
using OnRound = std::function<void(int round, const rsem_b200_round_stats&)>;
std::string round_line(int round, const rsem_b200_round_stats& s);   // "ROUND = ..." as EM.cpp:415 prints it
struct EmRounds {
    int round = 0;          // the last round run
    long long totNum = 0;
    bool keep_going = true;
};
// rounds 1-10, which update the model (EM.cpp:364-416), on ctx; they end with the model pushed and conprb computed
EmRounds em_model_rounds(rsem_b200_ctx* ctx, HostModel& model, uint64_t N0, int MIN_ROUND, int MAX_ROUND, const OnRound& on_round);
// the frozen rounds that follow on ctx, 32 per rsem_b200_em_rounds call, until the stop rule holds
void em_frozen_rounds(rsem_b200_ctx* ctx, uint64_t N0, int MIN_ROUND, int MAX_ROUND, EmRounds& r, const OnRound& on_round);
// the end of a sample whose EM has ended: the convergence warning (prefixed with `who`), .ofg with --gibbs-out,
// counts[0] += N0, write_em_outputs and with -b the posterior BAM (`threads` BGZF threads, its messages when `verbose`)
void finish_em_sample(const EmReference& ref, int read_type, const EmArgs& a, EmSample& s, long long totNum, int MAX_ROUND,
                      const std::string& who, int threads, bool verbose, void (*stamp)(const char*) = nullptr);
// .theta, .model and the result rows of a sample; counts[0] already holds N0
void write_em_outputs(const std::string& refName, const std::string& imdName, const std::string& statName,
                      const RefData& refs, const std::vector<TranscriptInfo>& transcripts, const HostModel& model,
                      std::vector<double> theta, const std::vector<double>& counts, bool appendNames);
std::string time_used_line(time_t t_start);   // "Time Used for EM.cpp : ..." (EM.cpp:673)

// ---- gibbs_sample.cpp: the per-sample stages of rsem-run-gibbs, which rsem-run-gibbs-batch runs for each manifest line --
struct GibbsArgs {   // rsem-run-gibbs's arguments after reference_name
    std::string imdName, statName, fprior;
    int burnin = 0, nsamples = 0, gap = 0, nThreads = 1;
    bool hasSeed = false, hasPrior = false, quiet = false;
    uint32_t seed = 0;
    double pseudoC = 1.0;
};
// imdName statName BURNIN NSAMPLES GAP [options] (f.size() >= 5); returns "" or why they are refused
std::string parse_gibbs_args(const std::vector<std::string>& f, GibbsArgs& a);
void clamp_gibbs_chains(GibbsArgs& a);   // -p: at most NSAMPLES chains (with the reference's warning), at least one
struct GibbsSample {
    uint64_t N0 = 0, N1 = 0;
    std::vector<uint64_t> row_ptr;   // imdName.ofg
    std::vector<int32_t> sid;
    std::vector<double> conprb;
    std::vector<int32_t> init_counts, chain_samples;
    std::vector<uint32_t> chain_seeds;
    std::vector<double> alpha, eel, mw;
    double totc = 0;
};
// load_data's imdName.ofg (Gibbs.cpp:101-137); `say` gets "Loading data is finished!"
void load_gibbs_ofg(const GibbsArgs& a, int M, GibbsSample& s, const Say& say);
// after the groups: load_omit_info / load_prior_info, init_model_related and init()'s chains and seeds (Gibbs.cpp:152-254)
void load_gibbs_inputs(const GibbsArgs& a, const RefData& refs, GibbsSample& s, const Say& say);
rsem_b200_gibbs_params gibbs_params(const GibbsArgs& a, const GibbsSample& s, const std::vector<int>& gi);
// a sample whose chains have run: the sums of its chains, imdName.countvectors<t>, iso_res / gene_res
void finish_gibbs_sample(const std::string& refName, const GibbsArgs& a, const GibbsSample& s, const std::vector<int>& gi,
                         bool alleleS, const std::vector<int>& ta, const int32_t* cvs, const double* chain_acc, const Say& say);
// load_omit_info / load_prior_info (Gibbs.cpp:152-194): init_counts (-1 = omitted), alpha and totc of a sample with N0 + N1
// reads; returns "" or why imdName.omit or the prior file cannot be used.
std::string gibbs_inputs(const std::string& imdName, int M, uint64_t N0, uint64_t N1, double pseudoC, const std::string* fprior,
                         std::vector<int32_t>& init_counts, std::vector<double>& alpha, double& totc);
void write_results_gibbs(const std::string& ref_name, const std::string& imd_name, int M, const std::vector<double>& pme_c,
                         const std::vector<double>& pme_fpkm, const std::vector<double>& pme_tpm,
                         const std::vector<double>& pve_c, const std::vector<double>& pve_c_genes,
                         const std::vector<double>& pve_c_trans);  // WriteResults.h:357-479
void write_results_simulation(const std::string& ref_name, const std::string& out_name,
                              const std::vector<TranscriptInfo>& tr, const std::vector<double>& eel,
                              const std::vector<double>& counts);  // WriteResults.h:481-635

// ---- sim_sample.cpp: the per-sample stages of rsem-simulate-reads, which rsem-simulate-reads-batch runs for each line -----
struct SimReference {   // refName.seq with the sequences, refName.ti and the allele groups (WriteResults.h:106-123)
    std::string name;
    RefData refs;
    std::vector<TranscriptInfo> transcripts;
    std::vector<int> gt, ta;
    bool alleleS = false;
    int offsite = 5;     // column of the TPM in the results file (simulation.cpp:94-100)
};
void load_sim_reference(const std::string& refName, SimReference& ref);
// rsem-simulate-reads's arguments after reference_name (simulation.cpp:160-182)
struct SimArgs {
    std::string modelF, resultsF, outName;
    double theta0 = 0;
    long long N = 0;
    bool hasSeed = false, quiet = false;
    uint32_t seed = 0;
};
// estimated_model_file estimated_isoform_results theta0 N output_name [--seed seed] [-q] (f.size() >= 5): atof theta0,
// atoi N, istringstream for the seed; returns "" or why the seed cannot be taken
std::string parse_sim_args(const std::vector<std::string>& f, SimArgs& a);
// the model type on the first line of a .model file: -1 when the file cannot be opened, -2 when it is not 0..3
int sim_model_type(const std::string& modelF);
// the read file(s) a run writes (genOutReadStreams, simulation.cpp:60-84)
std::vector<std::string> sim_read_files(const std::string& outName, int model_type);
// what rsem-simulate-reads derives from the model and the results file before it draws (simulation.cpp:86-120)
struct SimSample {
    HostModel model;
    std::vector<double> eel, theta, theta_cdf, qd_init, qd_tran, pro, noise, rspd_cdf;
    std::vector<uint64_t> rspd_off;
    int pro_rows = 0;
    bool exact_body = false;
};
// the model, the expected effective lengths, theta and the cumulative tables; false when the results file gives every
// transcript TPM * effective length 0 (simulation.cpp:113)
bool load_sim_sample(const SimReference& ref, const SimArgs& a, SimSample& s);
// the run's parameters; with_seq false leaves the reference out (the context's rsem_b200_sim_upload_refs copy is used).
// RSEM_B200_SIM_WINDOW sets the window.  The pointers are into ref and s.
rsem_b200_sim_params sim_params(const SimReference& ref, const SimSample& s, uint32_t seed, long long N, bool with_seq);
// The chunk loop of a run: next() is rsem_b200_sim_next or _next_devices; the text of one chunk is written to the
// read files on a second thread while the device produces the next one.  `gen` (may be null) gets the GEN lines
// (simulation.cpp:125).  Returns the reads written; t_next adds the time in next(), t_write the time spent waiting for
// the writes.
using SimNext = std::function<void(const char* text[2], uint64_t bytes[2], uint64_t* n)>;
uint64_t write_sim_reads(const SimNext& next, FILE* const* os, int n_os, const Say* gen, double& t_next, double& t_write);

// ---- ci_stages.cpp: the per-sample stages of rsem-calculate-credibility-intervals, which
// rsem-calculate-credibility-intervals-batch runs for each manifest line --------------------------------------------------
struct CiReference {   // refName.seq (lengths), refName.grp and, for an allele-specific reference, .gt / .ta
    std::string name;
    RefData refs;
    std::vector<int> gi, gt, ta;
    bool alleleS = false;
    int m() const { return (int)gi.size() - 1; }
    int m_trans() const { return alleleS ? (int)ta.size() - 1 : 0; }
};
void load_ci_reference(const std::string& refName, CiReference& ref);
// the arguments after reference_name (calcCI.cpp:520-540)
struct CiArgs {
    std::string imdName, statName;
    double confidence = 0, pseudoC = 1.0;
    int nCV = 0, nSpC = 0, nMB = 0, nThreads = 1;
    bool hasSeed = false, quiet = false;
    uint32_t seed = 0;
    int64_t n_samples() const { return (int64_t)nCV * nSpC; }
    int samplers() const { return std::min(nThreads, nCV); }   // one per count-vector file (calcCI.cpp:172)
};
// imdName statName confidence nCV nSpC nMB [-p #Threads] [--seed seed] [--pseudo-count c] [-q] (f.size() >= 6); returns
// "" or why -p is refused.  whole_seed: refuse a --seed without a value or with anything but digits (the batch); else the
// seed is read digit by digit whatever it holds, as the reference does
std::string parse_ci_args(const std::vector<std::string>& f, CiArgs& a, bool whole_seed);
std::string ci_sample_count_error(const CiArgs& a, int M);   // nCV, nSpC positive, nCV * nSpC below 2^31; "" or why
std::string ci_memory_error(const CiArgs& a, int M);         // nMB holds one sample row (Buffer.h:18-20); "" or why
// statName.model -> the expected effective lengths and mw (dies as the reference does on a file it cannot read)
void load_ci_model(const CiReference& ref, const CiArgs& a, std::vector<double>& eel, std::vector<double>& mw);
// imdName.countvectors<t> for t < samplers(), one parser thread per file; dies when a file is missing or cannot be
// parsed, or when the files do not hold nCV vectors (with isolate, die() throws on the parser threads and the first
// failure is raised on the calling thread).  first[t]: the index of file t's first sample.
struct CiSample {
    std::vector<double> eel, mw;
    std::vector<std::vector<int32_t>> cvs;
    std::vector<int64_t> first;
};
void load_ci_vectors(const CiArgs& a, int M, CiSample& s, bool isolate);
// the gene ranges of the reference's Phase II threads (calcCI.cpp:402-420), from the line's -p
std::vector<int32_t> ci_parts(int nThreads, int M, const std::vector<int>& gi);
// the run's parameters; the pointers are into ref and parts
rsem_b200_ci_params ci_params(const CiReference& ref, const CiArgs& a, const std::vector<int32_t>& parts, uint64_t budget);
// Phase I after ci_begin: one sampler thread per file pushes its rows as it draws them; the count vectors are released
// as each thread ends.  progress (may be null) gets the samplers' lines from their threads.  With isolate, die() throws
// on the sampler threads and the first failure is raised on the calling thread.  Returns the samplers' summed seconds.
double ci_sample_rows(rsem_b200_ctx* ctx, const CiArgs& a, int M, CiSample& s, uint32_t seed, const Say* progress, bool isolate);
// ci_end: the intervals of every transcript, gene and isoform, 6 floats each
struct CiIntervals {
    std::vector<float> tr, gene, iso;
    rsem_b200_ci_stats st{};
};
void ci_intervals(rsem_b200_ctx* ctx, const CiReference& ref, CiIntervals& out);
// the Phase II threads' progress lines (calcCI.cpp:360), the rows appended to imdName.iso_res / .gene_res (and
// .allele_res) and "All credibility intervals are calculated!"; `say` (may be null) gets the lines
void write_ci_sample(const CiReference& ref, const CiArgs& a, const std::vector<int32_t>& parts, const CiIntervals& r,
                     const Say* say);

// ---- alignment files for -b: SAM / BAM in, BAM out (bam.cpp; BamWriter.h, sam_utils.h, SamHeader.cpp) -----------------
struct BamRecord {
    std::vector<uint8_t> data;  // the record as BAM stores it, without the leading block_size
    uint16_t flag() const;
    int32_t tid() const;
    bool mapped() const { return !(flag() & 0x4); }
    bool read1() const { return flag() & 0x40; }
    bool read2() const { return flag() & 0x80; }
    bool paired() const { return flag() & 0x1; }
    bool reverse() const { return flag() & 0x10; }
    int32_t pos() const;          // 0-based leftmost position
    int32_t l_seq() const;
    const char* qname() const;    // NUL-terminated
    uint32_t n_cigar() const;
    uint32_t cigar(uint32_t i) const;   // len << 4 | op
    int base4(int32_t i) const;   // 4-bit base code (1 A, 2 C, 4 G, 8 T, 15 N)
    const uint8_t* qual() const;  // l_seq phred values (0xff = absent)
    bool aux_int(const char tag[2], long long& value) const;  // bam_aux_get + bam_aux2i (0 for non-integer types)
    void set_alignment_weight(double prb);  // MAPQ + ZW:f (BamWriter.h:39-48)
};
uint8_t prb_to_mapq(double prb);            // bam_prb_to_mapq (sam_utils.h:72-76)
// t[m] = the smallest float p >= 0 with prb_to_mapq(p) >= m, m = 1..100 (t[0] = 0): MAPQ(p) = #{m >= 1 : p >= t[m]}
// for every float p >= 0, because prb_to_mapq does not decrease with p (checked for every float in [0, 2] by
// rsem-b200-host-selftest mapq-table; from 1 on it is 100)
std::vector<float> mapq_thresholds();

class AlnReader {
public:
    // tool: the executable named in the refusal of CRAM input (nullptr: rsem-run-em's message for -b).  htslib_header:
    // a BAM header cut short is reported as htslib 1.3's bam_hdr_read and the reference's build_wiggles report it
    // ("Cannot load SAM header!", wiggle.cpp:52) instead of "Truncated BAM header!"
    explicit AlnReader(const std::string& path, const char* tool = nullptr, bool htslib_header = false);
    ~AlnReader();
    AlnReader(const AlnReader&) = delete;
    AlnReader& operator=(const AlnReader&) = delete;
    const std::string& header_text() const { return text_; }
    const std::vector<std::string>& ref_names() const { return ref_names_; }
    const std::vector<uint32_t>& ref_lens() const { return ref_lens_; }
    bool next(BamRecord& rec);  // false at the end of the file

private:
    struct Source;
    struct Conv;          // SAM text -> BAM records on worker threads, ahead of next()
    Source* src_;
    Conv* conv_ = nullptr;
    bool is_bam_ = false, have_pending_ = false;
    std::string text_, pending_;
    std::vector<std::string> ref_names_;
    std::vector<uint32_t> ref_lens_;
    std::map<std::string, int> ref_index_;
    std::string spill_;           // a line that crosses a buffer boundary
    // last_ref: RNAME of the caller's previous line (alignments of a read mostly share it or repeat it)
    void parse_sam_line(const char* ln, size_t len, BamRecord& rec, int& last_ref) const;
    void conv_run();
    bool conv_next(BamRecord& rec);
};

// SamHeader(text) (SamHeader.cpp:48-114) + insertPG(pg_id, pg_cl) (SamHeader.hpp:39-46), with the @SQ block replaced by
// *sq when given (replaceSQ).  reference_pg_ids: take @PG IDs the way SamHeader::parse_line does, where a field followed
// by others reads as ID:<value>\t<the first characters after it> (substr with an end index used as a count), and refuse
// a @PG line without ID; otherwise the ID is the field's own value (what rsem-run-em -b has always written).
std::string rsem_bam_header_text(const std::string& in_text, const std::string& pg_id = "RSEM", const std::string& pg_cl = "",
                                 const std::string* sq = nullptr, bool reference_pg_ids = false);

class BamWriter {
public:
    BamWriter(const std::string& path, const std::string& header_text, int threads);
    ~BamWriter();
    BamWriter(const BamWriter&) = delete;
    BamWriter& operator=(const BamWriter&) = delete;
    void write(const BamRecord& rec);
    void write_encoded(const uint8_t* p, size_t n);   // records already framed as block_size + bytes
    void close();

private:
    FILE* fo_ = nullptr;
    int threads_ = 1;
    std::vector<uint8_t> pending_;
    void append(const uint8_t* p, size_t n);
    void flush_pending(bool all);
};

// ---- rsem-bam2wig / rsem-bam2readdepth (wiggle.cpp; the reference's wiggle.cpp:16-130) ------------------------------
struct WigTarget {
    std::string name;
    uint64_t length = 0;              // target_len
    const double* depth = nullptr;    // length values, or nullptr for the reference's empty read_depth
};
// What UCSCWiggleTrackWriter::process (wig) or ReadDepthWriter::process (!wig) writes for every target, in order,
// split into chunks of about chunk_positions positions that `threads` threads format with glibc's snprintf; the
// chunks concatenated in order are the text, whatever chunk_positions and threads are.
void format_wiggles(const std::vector<WigTarget>& targets, bool wig, size_t chunk_positions, int threads,
                    std::vector<std::string>& chunks);
// build_wiggles (wiggle.cpp:16-83) with one of the two writers, onto `out` (already holding what the tool wrote first).
// Prints the progress lines on stdout; refusals stop the run with exit status 255.
void run_wiggles(const char* tool, const std::string& in_path, bool wig, bool no_fractional_weight, FILE* out);

// boost::random::mt19937 as the reference uses it (sampling.h:12-16): engine(seed), 32-bit draws; uniform_01 = x * 2^-32
struct Mt {
    uint32_t mt[624];
    int idx;
    explicit Mt(uint32_t seed) {
        mt[0] = seed;
        for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
        idx = 624;
    }
    uint32_t next() {
        if (idx >= 624) {
            for (int k = 0; k < 624; ++k) {
                const uint32_t y = (mt[k] & 0x80000000u) | (mt[(k + 1) % 624] & 0x7fffffffu);
                mt[k] = mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            idx = 0;
        }
        uint32_t y = mt[idx++];
        y ^= y >> 11;
        y ^= (y << 7) & 0x9d2c5680u;
        y ^= (y << 15) & 0xefc60000u;
        y ^= y >> 18;
        return y;
    }
    double uniform01() { return next() * (1.0 / 4294967296.0); }  // boost uniform_01 on a 32-bit engine
};

// em_sample.cpp: sampleName.transcript.bam with the posteriors of the final pass (EM.cpp:504-536, BamWriter.h)
void write_posterior_bam(const std::string& inpSamF, const std::string& outName, int read_type, bool sampling, bool hasSeed,
                         uint32_t seed, const std::vector<TranscriptInfo>& tr, int ti_type, const HitStore& hits,
                         std::vector<double>& post, const std::vector<double>& post0, int threads, bool verbose);


// ---- small utilities -----------------------------------------------------------------------------
// engineFactory (sampling.h:19-40): n engine seeds drawn from mt19937(seed), a seed already handed out is skipped
std::vector<uint32_t> engine_seeds(uint32_t seed, int n);
std::vector<char> slurp(const std::string& path, bool must_exist = true);
void read_type_files(const std::string& imd_name, int tag, int read_type, std::vector<std::string>& files);
uint32_t parse_seed(const char* s);  // digit-by-digit as EM.cpp:588-593
double now_s();                      // steady clock, seconds
int env_int(const char* name, int dflt);

// ---- lanes.cpp: devices, and the lanes of the batch executables (one host thread, context and batch arena each) ----
// CUDA devices of a multi-GPU run: RSEM_B200_DEVICES=0,1,... in the order given; with at most one entry there,
// RSEM_B200_DEVICE when it is set, else that entry, else device 0
std::vector<int> gpu_devices();
// While a DieThrows(true) lives on a thread, die() and check_rc() there throw std::runtime_error instead of ending the
// process, so that a failing lane can be reported once the other lanes have stopped.
struct DieThrows {
    explicit DieThrows(bool on);
    ~DieThrows();
    bool prev;
};
// One context per entry of `devices`, created on host threads.  arena[k] is lane k's batch arena: RSEM_B200_BATCH_ARENA_BYTES
// when it is set and not 0; else, with one entry, 0 (the batch's own default); else half of the device memory free before the first
// context on the lane's device, divided by the entries naming that device.  free[k]: from open_lanes_measured, the
// device memory free on lane k's device before its first context (from open_lanes, 0 unless arena needed it).  err: the
// first device that could not be opened, once every creation has returned (the caller ends the run).
struct LaneContexts {
    std::vector<rsem_b200_ctx*> ctx;
    std::vector<uint64_t> arena, free;
    std::string err;
};
LaneContexts open_lanes(const std::vector<int>& devices);
LaneContexts open_lanes_measured(const std::vector<int>& devices);
// The manifest lines, handed to the lanes in manifest order; the first failure stops the handing out.
class Claims {
  public:
    explicit Claims(size_t n) : n_(n) {}
    size_t next();                          // n once every line is handed out or a lane has failed
    void fail(const std::string& msg);      // keeps the first message
    bool failed();
    std::string message();
  private:
    const size_t n_;
    std::atomic<size_t> i_{0};
    std::atomic<bool> failed_{false};
    std::mutex mu_;
    std::string msg_;
};
// Runs run(lane) for every lane: the only one on this thread, or each on its own thread with die() throwing.  The first
// failure ends the run (exit status -1) as "<tool>: device D, <where>: <what>" once every lane has stopped; a Lane
// needs `device` and `where` (what it is working on) for it.
template <class Lane, class Run>
void run_lanes(const char* tool, std::vector<Lane>& lanes, Claims& claims, Run run) {
    if (lanes.size() == 1) return run(lanes[0]);
    auto lane_main = [&](Lane& L) {
        DieThrows throws(true);
        try {
            run(L);
        } catch (const std::exception& e) {
            claims.fail(std::string(tool) + ": device " + std::to_string(L.device) + ", " + L.where + ": " + e.what());
        }
    };
    std::vector<std::thread> pool;
    for (size_t k = 1; k < lanes.size(); ++k) pool.emplace_back(lane_main, std::ref(lanes[k]));
    lane_main(lanes[0]);
    for (auto& th : pool) th.join();
    if (claims.failed()) die(claims.message());
}
// The non-empty lines of a manifest: 1-based line number and whitespace-separated fields
struct ManifestLine {
    int no;
    std::vector<std::string> f;
};
std::vector<ManifestLine> manifest_lines(const std::string& path);
[[noreturn]] void refuse(const std::string& manifest, int no, const std::string& why);   // "<manifest> line N: why"
std::string sample_at(const std::string& name, const std::string& manifest, int no);     // "sample X (<manifest> line N)"

}  // namespace host
