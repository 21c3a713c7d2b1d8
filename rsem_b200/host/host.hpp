// Host side of the drop-in executables rsem-run-em / rsem-run-gibbs.
//
// Everything here is O(input) parsing, O(table) model bookkeeping and O(M) output math; all per-hit
// and per-read arithmetic runs on the GPU through the C ABI (include/rsem_b200.h).
// File formats and semantics follow the reference (citations per function, paths relative to
// /root/reference); the code structure does not: one table-oriented HostModel instead of four
// template classes, SoA read/hit stores instead of streams of objects.
#pragma once

#include <cstdint>
#include <cstdio>
#include <functional>
#include <map>
#include <string>
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
    // the whole .model file, every model type (rsem-simulate-reads); mw stays empty when the file has none for M
    void read(const std::string& path, int M);
};

// ---- O(M) result math (WriteResults.h:24-104) ------------------------------------------------------
void calc_eel(const RefData& refs, const LenDistH& gld, std::vector<double>& eel);
void polish_theta(std::vector<double>& theta, const std::vector<double>& eel, const std::vector<double>& mw);
void expression_values(const std::vector<double>& theta, const std::vector<double>& eel, std::vector<double>& tpm,
                       std::vector<double>& fpkm);
void write_results_em(const std::string& ref_name, const std::string& imd_name, const std::vector<TranscriptInfo>& tr,
                      const std::vector<double>& theta, const std::vector<double>& eel, const double* counts,
                      bool append_names);  // WriteResults.h:125-355
// em_sample.cpp: the per-sample output stages of rsem-run-em (also used by rsem-run-em-batch)
void write_em_outputs(const std::string& refName, const std::string& imdName, const std::string& statName,
                      const RefData& refs, const std::vector<TranscriptInfo>& transcripts, const HostModel& model,
                      std::vector<double> theta, const std::vector<double>& counts, bool appendNames);
// gibbs_sample.cpp: the per-sample stages of rsem-run-gibbs (also used by rsem-run-gibbs-batch)
// load_omit_info / load_prior_info (Gibbs.cpp:152-194): init_counts (-1 = omitted), alpha and totc of a sample with N0 + N1
// reads; returns "" or why imdName.omit or the prior file cannot be used.
std::string gibbs_inputs(const std::string& imdName, int M, uint64_t N0, uint64_t N1, double pseudoC, const std::string* fprior,
                         std::vector<int32_t>& init_counts, std::vector<double>& alpha, double& totc);
// imdName.countvectors<t>, one per chain (Gibbs.cpp:257-262); cvs holds the chains' vectors in chain order
void write_countvectors(const std::string& imdName, int M, const std::vector<int32_t>& chain_samples, const int32_t* cvs);
// release() (Gibbs.cpp:399-422): means and unbiased variances from the sums of all chains and the kept count vectors,
// then imdName.iso_res / gene_res (and the allele file) by write_results_gibbs
void write_gibbs_results(const std::string& refName, const std::string& imdName, int M, int NSAMPLES, const std::vector<int>& gi,
                         bool alleleS, const std::vector<int>& ta, const int32_t* cvs, const std::vector<double>& sum_c,
                         const std::vector<double>& sum_c2, const std::vector<double>& sum_tpm, const std::vector<double>& sum_fpkm,
                         const std::vector<double>& sum_g2);
void write_results_gibbs(const std::string& ref_name, const std::string& imd_name, int M, const std::vector<double>& pme_c,
                         const std::vector<double>& pme_fpkm, const std::vector<double>& pme_tpm,
                         const std::vector<double>& pve_c, const std::vector<double>& pve_c_genes,
                         const std::vector<double>& pve_c_trans);  // WriteResults.h:357-479
void write_results_simulation(const std::string& ref_name, const std::string& out_name,
                              const std::vector<TranscriptInfo>& tr, const std::vector<double>& eel,
                              const std::vector<double>& counts);  // WriteResults.h:481-635

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
// CUDA devices of a multi-GPU run: RSEM_B200_DEVICES=0,1,... in the order given; with at most one entry there,
// RSEM_B200_DEVICE when it is set, else that entry, else device 0
std::vector<int> gpu_devices();

}  // namespace host
