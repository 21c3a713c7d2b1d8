/*
 * rsem_b200.h - C ABI of librsem_b200.so: the H100 (sm_90a) implementation of RSEM's
 * expression-estimation hot path (rsem-run-em E/M loop and rsem-run-gibbs sampler).
 *
 * The reference has no in-process plugin/FFI interface for this path: its boundary is the
 * process boundary of `rsem-run-em` / `rsem-run-gibbs` (argv + files, SURVEY.md section 8(b)).
 * The drop-in executables in rsem_b200/host/ keep that boundary byte for byte and call ONLY the
 * functions below for compute.  Every entry point cites the reference code it replaces
 * (paths relative to /root/reference).
 *
 * Conventions
 *   - all functions return 0 on success, non-zero on error; rsem_b200_last_error() returns a
 *     thread-local message.  Host callers print it and exit(-1) (reference convention,
 *     my_assert.h:34-41).
 *   - all pointer arguments are HOST pointers owned by the caller unless stated otherwise;
 *     device buffers are owned by the context.
 *   - calls are synchronous with respect to the host unless stated otherwise.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 *   - transcript ids are the reference's: 0 = noise "transcript", 1..M = isoforms.
 *   - `sid` is signed exactly as SingleHit stores it: |sid| = transcript id, sid < 0 = reverse
 *     strand (SingleHit.h:24-26).
 */
#ifndef RSEM_B200_H_
#define RSEM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSEM_B200_VERSION 100 /* 0.1.0 */

/* error codes */
#define RSEM_B200_OK 0
#define RSEM_B200_ERR_CUDA 1     /* CUDA runtime / driver failure, or no device */
#define RSEM_B200_ERR_ARG 2      /* invalid argument / call order */
#define RSEM_B200_ERR_NCCL 3     /* NCCL failure or libnccl not loadable */
#define RSEM_B200_ERR_UNSUPPORTED 4
#define RSEM_B200_ERR_FULL 5       /* rsem_b200_batch_add: the sample does not fit the arena's remaining bytes */

typedef struct rsem_b200_batch rsem_b200_batch;

typedef struct rsem_b200_ctx rsem_b200_ctx;

/* ------------------------------------------------------------------------------------------------
 * Model tables handed to the device (read-only during an E-step).
 * Replaces the per-thread shared `ModelType& model` read by E_STEP (EM.cpp:176-247):
 *   Orientation.h:12-25, LenDist.h:57-77, RSPD.h:63-75, Profile.h:114-124, QProfile.h:111-120,
 *   NoiseProfile.h:104-113, NoiseQProfile.h:115-124 and `mw` (SingleQModel.h:482-544).
 * ---------------------------------------------------------------------------------------------- */
typedef struct rsem_b200_lendist {
    int32_t lb, ub, span;  /* support is (lb, ub], span = ub - lb (LenDist.h:17-32)            */
    const double* pdf;     /* span + 1 entries, pdf[0] = 0                                     */
    const double* cdf;     /* span + 1 entries                                                 */
} rsem_b200_lendist;

typedef struct rsem_b200_model {
    int32_t model_type;   /* 0 SingleModel, 1 SingleQModel, 2 PairedEndModel, 3 PairedEndQModel (EM.cpp:661-667) */
    int32_t M;            /* number of transcripts                                             */
    int32_t seed_len;     /* ModelParams::seedLen                                              */
    int32_t est_rspd;     /* 0/1                                                               */
    int32_t rspd_B;       /* number of RSPD bins                                               */
    int32_t has_mld;      /* single-end: 1 iff --fragment-length-mean given (mld != NULL);
                             paired-end: always 1 (mld = mate length distribution)             */
    int32_t pro_len;      /* no-quality models: Profile::proLen (= mparams.maxL); else 0       */
    int32_t reserved;
    double ori[2];        /* P(forward), P(reverse)                                            */
    rsem_b200_lendist gld;
    rsem_b200_lendist mld;        /* valid iff has_mld                                         */
    const double* rspd_pdf;       /* B + 2 entries (RSPD.h:21-33)                              */
    const double* rspd_cdf;       /* B + 2 entries                                             */
    const double* profile;        /* Q models: [100][5][5]; no-Q: [pro_len][5][5], p[.][ref][read] */
    const double* noise_profile;  /* Q models: [100][5];    no-Q: [5]                          */
    const double* mw;             /* M + 1 mask weights, mw[0] = 1                             */
} rsem_b200_model;

/* Sufficient statistics produced by one model-update E-step (rounds 1-10).
 * Replaces the helper models `mhps[t]` filled by update/updateNoise (e.g. SingleQModel.h:168-221,
 * PairedEndQModel.h:161-188) and summed by Model::collect (EM.cpp:400-404).
 * The caller provides the buffers; entries the model does not estimate are left untouched.   */
typedef struct rsem_b200_model_stats {
    double* profile;        /* same shape as rsem_b200_model.profile, raw (un-normalised) sums  */
    double* noise_profile;  /* same shape as rsem_b200_model.noise_profile, raw sums WITHOUT the N0 counts `c` */
    double* gld_pdf;        /* paired-end only: gld_span + 1 sums indexed by len - gld_lb      */
    int32_t gld_lb, gld_span; /* support the helper histogram uses: the ORIGINAL (minL-1, maxL] (PairedEndQModel.h:72) */
    double* rspd_pdf;       /* est_rspd only: B + 2 sums (RSPD.h:43-59)                        */
} rsem_b200_model_stats;

/* per-round scalars printed on the reference's "ROUND = ..." line (EM.cpp:406-415) */
typedef struct rsem_b200_round_stats {
    double sum;      /* sum of counts incl. N0  */
    double bchange;  /* biggest relative change */
    int64_t totnum;  /* #transcripts with probv >= 1e-7 and relative change >= 1e-3 */
} rsem_b200_round_stats;

/* ------------------------------------------------------------------------------------------------ */
int rsem_b200_version(void);
const char* rsem_b200_last_error(void);
int rsem_b200_device_count(int* n_devices);
/* bytes of device memory free on `device` now; the batch executables size their arenas from it */
int rsem_b200_device_free_bytes(int device, uint64_t* free_bytes);

/* One context per GPU (one host thread or process per context). */
int rsem_b200_ctx_create(int device, rsem_b200_ctx** out);
int rsem_b200_ctx_destroy(rsem_b200_ctx* ctx);
/* Run all subsequent work on `cuda_stream` (a cudaStream_t owned by the caller, e.g. a
 * torch.cuda.Stream handle) instead of the context's own stream.  NULL restores the default.  */
int rsem_b200_ctx_set_stream(rsem_b200_ctx* ctx, void* cuda_stream);
int rsem_b200_ctx_sync(rsem_b200_ctx* ctx);
/* bytes of device memory currently held by the context */
int rsem_b200_ctx_device_bytes(rsem_b200_ctx* ctx, uint64_t* bytes);

/* ---- multi-GPU: reads are sharded across contexts; the per-transcript count vector (and, in
 * rounds 1-10, the model sufficient statistics) are summed with ncclAllReduce over NVLink.
 * Replaces the serial merge `countvs[0][j] += countvs[i][j]` (EM.cpp:385-389) and
 * Model::collect (EM.cpp:402).  libnccl.so.2 is dlopen()ed on first use.                       */
#define RSEM_B200_UNIQUE_ID_BYTES 128
int rsem_b200_comm_unique_id(void* id_out /* 128 bytes */);
int rsem_b200_comm_init(rsem_b200_ctx* ctx, const void* id /* 128 bytes */, int n_ranks, int rank);

/* Read sharding over GPUs = the reference's read sharding over threads (init<>, EM.cpp:135-157): shard i gets the
 * contiguous reads [bounds[i], bounds[i + 1]) holding about nHits / n_shards hits, every shard at least one read while
 * reads are left.  Pure host arithmetic (no device needed); bounds has n_shards + 1 entries.                      */
int rsem_b200_shard_reads(uint64_t N, const uint64_t* row_ptr /* N + 1 */, int32_t n_shards, uint64_t* bounds);

/* ---- data upload ------------------------------------------------------------------------------
 * Hit buffer = HitContainer<SingleHit|PairedEndHit> (HitContainer.h:12-59) as SoA CSR.
 * row_ptr has N + 1 entries, row_ptr[0] = 0, row_ptr[N] = H.  insertL may be NULL (single-end).
 * pos/insertL may both be NULL when only frozen-conprb rounds / Gibbs are going to run.        */
int rsem_b200_upload_hits(rsem_b200_ctx* ctx, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr,
                          const int32_t* sid, const int32_t* pos, const int32_t* insertL);
/* Directly set hit.conprb / ncpv (used when resuming from an .ofg-like matrix, by tests and the
 * benchmark).  conprb: H doubles, ncpv: N doubles.  The copies run on a second stream; meanwhile the
 * directory of the equivalence-class layout the frozen-conprb rounds use (it depends on row_ptr / sid
 * only) is built on the device, so a following rsem_b200_em_rounds starts without that latency.    */
int rsem_b200_upload_conprb(rsem_b200_ctx* ctx, const double* conprb, const double* ncpv);
int rsem_b200_download_conprb(rsem_b200_ctx* ctx, double* conprb, double* ncpv);
/* Same as upload_hits + upload_conprb but from DEVICE pointers already resident on ctx's GPU
 * (no copy across PCIe; buffers are copied device-to-device into the context, on the context's
 * stream: work that produces them on another stream must have completed before the call).      */
int rsem_b200_adopt_device_matrix(rsem_b200_ctx* ctx, uint64_t N, uint64_t H, int32_t M, const uint64_t* d_row_ptr,
                                  const int32_t* d_sid, const double* d_conprb, const double* d_ncpv);

/* Reads, parsed once and kept resident (the reference re-parses the FASTA/FASTQ text every round
 * 1-11: ReadReader.h:34-38, EM.cpp:195-202).  mate m of read i occupies
 * base[m][off[m][i] .. off[m][i+1]) with codes A0 C1 G2 T3 N4 (utils.h:36-55); qual holds
 * phred+33 - 33 (QProfile.h:42) or is NULL for no-quality read types.  low_quality[i] is the
 * result of calc_lq (SingleReadQ.h:63-95, PairedEndReadQ.h:58-65).                             */
int rsem_b200_upload_reads(rsem_b200_ctx* ctx, int32_t n_mates, const uint64_t* off1, const uint8_t* base1,
                           const uint8_t* qual1, const uint64_t* off2, const uint8_t* base2, const uint8_t* qual2,
                           const uint8_t* low_quality);
/* Reference transcripts (Refs.h / RefSeq.h): forward-strand base codes of transcript t in
 * seq[seq_off[t] .. seq_off[t] + totLen[t]) for t = 1..M (index 0 unused), seed masks as the
 * 32-bit words of RefSeq::fmasks (RefSeq.h:89-97) at mask_words[mask_off[t] ..).               */
int rsem_b200_upload_refs(rsem_b200_ctx* ctx, int32_t M, const uint64_t* seq_off, const uint8_t* seq,
                          const int32_t* full_len, const int32_t* tot_len, const uint64_t* mask_off,
                          const uint32_t* mask_words);
int rsem_b200_set_model(rsem_b200_ctx* ctx, const rsem_b200_model* model);

/* ---- compute ----------------------------------------------------------------------------------- */
/* K1: hit.conprb = model.getConPrb(read, hit), ncpv = model.getNoiseConPrb(read) for every hit
 * (calcConProbs, EM.cpp:249-278; getConPrb e.g. SingleQModel.h:101-151).                       */
int rsem_b200_calc_conprb(rsem_b200_ctx* ctx);

int rsem_b200_set_theta(rsem_b200_ctx* ctx, const double* theta /* M + 1 */);
int rsem_b200_get_theta(rsem_b200_ctx* ctx, double* theta /* M + 1 */);

/* K2 + (allreduce) + K4, repeated: frozen-conprb EM rounds (ROUND >= 12 of EM.cpp:364-416).
 * Runs rounds first_round, first_round + 1, ... without host round trips until either
 * `max_rounds_this_call` rounds ran or the reference's loop condition
 *     ROUND < min_round || (totNum > 0 && ROUND < max_round)           (EM.cpp:416)
 * became false (the stop test runs on the device).  n0 is N0 of the .cnt file (EM.cpp:392).
 * stats_out receives one entry per executed round; *rounds_run their number; *stopped = 1 if
 * the loop condition ended the run.  With a communicator every rank must make the same call.   */
int rsem_b200_em_rounds(rsem_b200_ctx* ctx, int32_t first_round, int32_t max_rounds_this_call, int32_t min_round,
                        int32_t max_round, double n0, rsem_b200_round_stats* stats_out, int32_t* rounds_run,
                        int32_t* stopped);

/* One model-updating round (ROUND <= 10, EM.cpp:368-404): [K1 if conprb is stale] + K2 with
 * posterior write-back + K3 (update/updateNoise) + allreduce + K4.  The caller then rebuilds the
 * master model from `stats` (Model::finish) and calls rsem_b200_set_model again, which marks
 * conprb stale (needCalcConPrb).                                                                */
int rsem_b200_em_model_round(rsem_b200_ctx* ctx, double n0, rsem_b200_model_stats* stats,
                             rsem_b200_round_stats* round_stats);

/* Final pass with calcExpectedWeights = true (EM.cpp:460-478): E-step with the current theta that
 * overwrites hit.conprb / ncpv with the posteriors and returns the expected counts
 * (M + 1, summed over ranks, WITHOUT adding N0).  theta is not changed.  Afterwards conprb / ncpv
 * hold posteriors (read them with download_conprb): further E-steps on this context need a new
 * upload_conprb / calc_conprb first and fail with RSEM_B200_ERR_ARG otherwise.                   */
int rsem_b200_expected_weights(rsem_b200_ctx* ctx, double* counts_out);

/* ---- Gibbs (rsem-run-gibbs, Gibbs.cpp:265-353) ------------------------------------------------
 * The .ofg matrix: rows of (sid, conprb) with the noise entry (sid 0) first when present
 * (Gibbs.cpp:119-131).                                                                          */
typedef struct rsem_b200_gibbs_params {
    int32_t M;
    int32_t burnin, gap;
    int32_t n_chains;             /* = the reference's nThreads after clamping (Gibbs.cpp:478-481)       */
    const int32_t* chain_samples; /* n_chains entries: samples kept by chain t (Gibbs.cpp:211-223)       */
    const uint32_t* chain_seeds;  /* n_chains entries: mt19937 seeds from engineFactory (sampling.h:19-42) */
    double n0;                    /* N0 from the .ofg header                                             */
    const int32_t* init_counts;   /* M + 1: 0, or -1 for omitted transcripts (Gibbs.cpp:152-167)         */
    const double* pseudo_counts;  /* M + 1: pseudoC or the --prior values (Gibbs.cpp:298-306)            */
    double totc;                  /* Gibbs.cpp:166 / 186-193                                             */
    const double* eel;            /* M + 1 expected effective lengths (WriteResults.h:24-53)             */
    const double* mw;             /* M + 1                                                               */
    int32_t n_genes;              /* m                                                                   */
    const int32_t* gene_start;    /* m + 1 (GroupInfo::spAt)                                             */
} rsem_b200_gibbs_params;

typedef struct rsem_b200_gibbs_out {
    /* per chain, concatenated in chain order: chain_samples[t] count vectors of M + 1 int32 each,
     * i.e. the lines of imd.countvectors<t> (Gibbs.cpp:257-262)                                 */
    int32_t* count_vectors;
    /* sums over ALL kept samples of all chains (Gibbs.cpp:325-345, 372-397)                     */
    double* sum_c;        /* M + 1 */
    double* sum_c2;       /* M + 1 */
    double* sum_tpm;      /* M + 1 */
    double* sum_fpkm;     /* M + 1 */
    double* sum_gene_c2;  /* n_genes */
} rsem_b200_gibbs_out;

int rsem_b200_gibbs_upload(rsem_b200_ctx* ctx, uint64_t N1, uint64_t E, int32_t M, const uint64_t* row_ptr,
                           const int32_t* sid, const double* conprb);
/* = rsem_b200_gibbs_run_chains followed by rsem_b200_gibbs_sum_chains */
int rsem_b200_gibbs_run(rsem_b200_ctx* ctx, const rsem_b200_gibbs_params* params, rsem_b200_gibbs_out* out);

/* ---- Gibbs over several GPUs: the reference's threads are independent chains (Gibbs.cpp:265-353), so a run's chains can
 * be split into contiguous ranges, one per device, and their per-chain sums added up on the host in chain order.
 * A chain's draws depend only on its own seed and sample count, never on the other chains of the call.               */
/* device time and shape of one rsem_b200_gibbs_run_chains call */
typedef struct rsem_b200_gibbs_stats {
    double device_ms;      /* CUDA events around the sampler's launches                                         */
    int32_t worker_ctas;   /* worker CTAs per chain of the component-parallel kernel; 0 when the serial kernel ran */
    int32_t launches;      /* kernel launches (waves of chains)                                                 */
} rsem_b200_gibbs_stats;
/* Runs the chains params describes (any contiguous range of a run: the caller passes the sub-arrays of chain_samples /
 * chain_seeds).  count_vectors: as rsem_b200_gibbs_out.count_vectors, for these chains.  chain_acc: n_chains blocks of
 * 4 (M + 1) + n_genes doubles in chain order, each holding one chain's sum_c, sum_c2, sum_tpm, sum_fpkm (M + 1 each)
 * and sum_gene_c2 (n_genes).  stats may be NULL.                                                                    */
int rsem_b200_gibbs_run_chains(rsem_b200_ctx* ctx, const rsem_b200_gibbs_params* params, int32_t* count_vectors,
                               double* chain_acc, rsem_b200_gibbs_stats* stats);
/* out's sums (count_vectors is not touched) = the params->n_chains blocks of chain_acc added up in chain order
 * (Gibbs.cpp:372-397).  Pure host arithmetic (no device needed).                                                    */
int rsem_b200_gibbs_sum_chains(const rsem_b200_gibbs_params* params, const double* chain_acc, rsem_b200_gibbs_out* out);
/* Contiguous chain ranges for n_parts devices: part i runs chains [bounds[i], bounds[i + 1]).  A chain costs
 * burnin + 1 + (chain_samples[t] - 1) gap sweeps; bound i is the chain boundary whose prefix of sweeps is nearest to
 * i / n_parts of the total (the lower one on a tie), every part at least one chain while chains are left.  More parts
 * than chains: the surplus parts are empty.  Pure host arithmetic; bounds has n_parts + 1 entries.                    */
int rsem_b200_gibbs_split_chains(int32_t n_chains, const int32_t* chain_samples, int32_t burnin, int32_t gap,
                                 int32_t n_parts, int32_t* bounds);
/* Gives dst (any device, another context) the matrix uploaded to src with rsem_b200_gibbs_upload, component layout
 * included, by device-to-device copies (over NVLink where the two devices can map each other's memory): the host-side
 * component analysis and the row permutation run once, on src.  dst's previous matrix is released.  A src without a
 * completed upload, or src == dst, is refused with RSEM_B200_ERR_ARG.                                                */
int rsem_b200_gibbs_upload_from(rsem_b200_ctx* dst, const rsem_b200_ctx* src);

/* ---- K13: the Gibbs chains of many samples at once (rsem-run-gibbs-batch) --------------------------------------------
 * A Gibbs batch holds the .ofg matrices of several samples, their per-sample inputs (rsem_b200_gibbs_params) and room for
 * their outputs in one device arena, and runs every (sample, chain) job in one cooperative launch.  A team of
 * worker_ctas worker CTAs and 1 generator CTA runs one job at a time with the component-parallel chain of
 * rsem_b200_gibbs_run_chains; teams claim jobs from a device counter, largest first (sweeps x reads).  A job's count
 * vectors and chain_acc block are bit-identical to that chain run by rsem_b200_gibbs_run_chains on the sample alone.
 *
 * Size rule: a sample takes the batch when 1248 <= N1 <= 2^19 reads.  Smaller ones run the serial kernel of
 * rsem_b200_gibbs_run_chains (its generator runs one sweep ahead, which needs 624 outputs to span at most two sweeps);
 * larger ones have enough reads to spread over a whole-GPU cooperative launch of their own, which one team cannot use.
 * Both are refused with RSEM_B200_ERR_UNSUPPORTED and run with rsem_b200_gibbs_upload + rsem_b200_gibbs_run_chains.
 * The batch lives on `ctx`'s device and stream; destroy it before the context.                                        */
typedef struct rsem_b200_gibbs_batch rsem_b200_gibbs_batch;
#define RSEM_B200_GIBBS_BATCH_MIN_READS 1248ull
#define RSEM_B200_GIBBS_BATCH_MAX_READS 524288ull
/* capacity_bytes = 0: half of the device memory free at the call.  worker_ctas: worker CTAs per team, 1..8, or 0 for the
 * library's choice (2).                                                                                                */
int rsem_b200_gibbs_batch_create(rsem_b200_ctx* ctx, uint64_t capacity_bytes, int32_t worker_ctas,
                                 rsem_b200_gibbs_batch** out);
int rsem_b200_gibbs_batch_destroy(rsem_b200_gibbs_batch* batch);
/* Arena bytes of a sample of N1 reads, E entries, M transcripts, n_genes genes and n_samples count vectors over n_chains
 * chains (layout, inputs, count vectors, per-chain sums and state), or RSEM_B200_ERR_UNSUPPORTED outside the size rule
 * above.  No GPU needed.                                                                                               */
int rsem_b200_gibbs_batch_sample_bytes(uint64_t N1, uint64_t E, int32_t M, int32_t n_genes, int32_t n_samples,
                                       int32_t n_chains, uint64_t* bytes);
/* Adds a sample: its .ofg matrix as for rsem_b200_gibbs_upload and its chains' parameters (copied; every pointer of
 * params is read during the call only).  Every sample of a batch has the M and n_genes of the first.  Refused with
 * RSEM_B200_ERR_ARG for a read without entries or a bad id, RSEM_B200_ERR_FULL when the arena has no room left,
 * RSEM_B200_ERR_UNSUPPORTED outside the size rule.  *slot receives its handle.                                          */
int rsem_b200_gibbs_batch_add(rsem_b200_gibbs_batch* batch, uint64_t N1, uint64_t E, const uint64_t* row_ptr,
                              const int32_t* sid, const double* conprb, const rsem_b200_gibbs_params* params,
                              int32_t* slot);
typedef struct rsem_b200_gibbs_batch_stats {
    double device_ms;         /* CUDA events around the launch                                                        */
    int32_t worker_ctas;      /* worker CTAs per team                                                                 */
    int32_t teams;            /* co-resident teams of the launch                                                      */
    int64_t jobs;             /* (sample, chain) jobs run                                                             */
    uint64_t chain_cycles;    /* SM cycles of worker CTA 0 summed over the jobs: whole sweeps (ChainSync::prof[0,2,3]) */
    uint64_t sample_cycles;   /* of which the per-kept-draw O(M) work (ChainSync::prof[3])                            */
} rsem_b200_gibbs_batch_stats;
/* Runs every sample added since the last run, in one launch.  stats may be NULL. */
int rsem_b200_gibbs_batch_run(rsem_b200_gibbs_batch* batch, rsem_b200_gibbs_batch_stats* stats);
/* A sample's outputs after its run, as rsem_b200_gibbs_run_chains gives them: count_vectors (sum of chain_samples
 * vectors of M + 1), chain_acc (n_chains blocks of 4 (M + 1) + n_genes).                                              */
int rsem_b200_gibbs_batch_result(rsem_b200_gibbs_batch* batch, int32_t slot, int32_t* count_vectors, double* chain_acc);
/* Frees every sample (the arena is empty again). */
int rsem_b200_gibbs_batch_clear(rsem_b200_gibbs_batch* batch);

typedef struct rsem_b200_sim_stats rsem_b200_sim_stats;

/* ---- read simulation (rsem-simulate-reads, simulation.cpp:86-130) ------------------------------
 * All tables are the cumulative arrays the reference's startSimulation builds, in its layout:
 *   theta_cdf       M + 1: prefix sums of theta (SingleModel.h / PairedEndQModel.h startSimulation)
 *   gld, mld        LenDist (LenDist.h:255-262 samples cdf + 1); mld only when the model has one
 *   rspd_cdf        estRSPD only: transcript i's fullLen values evalCDF(j + 1, fullLen) at rspd_off[i]
 *                   (RSPD.h:182-193); rspd_off has M + 2 entries
 *   qd_*_cdf        QualDist, Q models: 100 and 100 x 100 (QualDist.h:116-130)
 *   profile_cdf     pro_rows x 5 x 5: QProfile (100 rows, QProfile.h:151-193) or Profile (proLen rows,
 *                   Profile.h:163-205), after the reference's zero-row repair
 *   noise_cdf       NoiseQProfile 100 x 5 (NoiseQProfile.h:153-166) or NoiseProfile 5 (NoiseProfile.h:137-144)
 *   seq / seq_off   forward-strand base codes 0..4 (A C G T N) per transcript, as upload_refs takes them; seq ==
 *                   NULL: the reference of rsem_b200_sim_upload_refs (seq_off, tot_len and full_len are then not read)
 * exact_body = 1 when a reachable table row sums to 0 (simul.h:29-32 then draws a second word), so the number of
 * words an attempt takes depends on the drawn qualities.  With 0 the attempt lengths are computed from the first
 * draws only; a wrong 0 gives wrong reads.
 * window_words: stream words per device window (0 = default); small values are for tests.                  */
typedef struct rsem_b200_sim_params {
    int32_t model_type;  /* 0 SingleModel, 1 SingleQModel, 2 PairedEndModel, 3 PairedEndQModel */
    int32_t M;
    uint32_t seed;       /* boost::mt19937(seed), simul.h:11 */
    int32_t exact_body;
    uint64_t N;          /* reads to simulate */
    uint64_t window_words;
    const double* theta_cdf;
    double ori_prob0;    /* Orientation prob[0] (Orientation.h:36) */
    rsem_b200_lendist gld, mld; /* pdf is not read */
    int32_t has_mld;
    int32_t est_rspd;
    const uint64_t* rspd_off;
    const double* rspd_cdf;
    const double* qd_init_cdf;
    const double* qd_tran_cdf;
    int32_t pro_rows;
    int32_t reserved;
    const double* profile_cdf;
    const double* noise_cdf;
    const uint64_t* seq_off;   /* M + 2 */
    const uint8_t* seq;
    const int32_t* tot_len;    /* M + 1 */
    const int32_t* full_len;   /* M + 1 */
} rsem_b200_sim_params;

/* Keeps a reference on the context for the runs that follow: rsem_b200_sim_begin with params->seq == NULL uses it
 * (its M must be params->M) instead of uploading the params' own.  Replaces an earlier upload; freed with the context.
 * Not while a run is between sim_begin and sim_end.                                                          */
int rsem_b200_sim_upload_refs(rsem_b200_ctx* ctx, int32_t M, const uint64_t* seq_off, const uint8_t* seq,
                              const int32_t* tot_len, const int32_t* full_len);
/* uploads the tables and seeds the stream (simulation.cpp:117-120, simul.h:11).  The device buffers of a run stay on
 * the context after sim_end and are reused by its next run (grown when that run needs more), so a context that runs
 * sample after sample allocates nothing after its largest one; rsem_b200_ctx_destroy frees them.              */
int rsem_b200_sim_begin(rsem_b200_ctx* ctx, const rsem_b200_sim_params* params);
/* the next chunk of reads, in order (simulation.cpp:121-126): *n_reads reads as the text of the read file(s)
 * (SingleRead(Q)::write, PairedEndRead(Q)::write: mate 1 in text[0], mate 2 in text[1]).  The buffers belong to the
 * context and stay valid until the second following call, so a caller can write one chunk while it asks for the
 * next.  *n_reads == 0: all N reads were returned.                                                          */
int rsem_b200_sim_next(rsem_b200_ctx* ctx, const char* text[2], uint64_t bytes[2], uint64_t* n_reads);
/* device time per phase, summed over the windows (CUDA events) */
typedef struct rsem_b200_sim_stats {
    double generate_ms;  /* mt19937 stream generation (on its own stream, overlapped with the other phases) */
    double resolve_ms;   /* attempt lengths + chain resolution                                           */
    double reads_ms;     /* read heads, offsets, text formatting                                         */
    double copy_ms;      /* read text to the host                                                        */
    uint64_t words;      /* stream words generated                                                       */
    uint64_t windows;
} rsem_b200_sim_stats;
/* counts[sid] of the simulated reads (M + 1), the number of failed attempts ("resimulation") and, when stats is not
 * NULL, the phase times; ends the run (its buffers stay on the context)                                      */
int rsem_b200_sim_end(rsem_b200_ctx* ctx, double* counts, uint64_t* resim, rsem_b200_sim_stats* stats);

/* ---- read simulation over several contexts (RSEM_B200_DEVICES) ----------------------------------------------------
 * The same reads as rsem_b200_sim_begin / _next / _end on one context for the same params, byte for byte.  Stream
 * window w (words [w W, (w + 1) W + L)) belongs to context w mod n: each context generates the W + L words of its
 * windows and jumps its mt19937 state ahead to its next one (rsem_b200_mt19937_jump's scheme, on the device).  The
 * attempt lengths of all windows are worked out side by side; the chain of attempts crosses the windows in order, each
 * window's entry point handed from one context to the next.  n >= 2; contexts may share a device.  The handle does not
 * own the contexts; each holds its part of the run as after rsem_b200_sim_begin until rsem_b200_sim_end_devices.     */
typedef struct rsem_b200_sim_multi rsem_b200_sim_multi;
int rsem_b200_sim_begin_devices(rsem_b200_ctx* const* ctxs, int n, const rsem_b200_sim_params* params,
                                rsem_b200_sim_multi** out);
/* as rsem_b200_sim_next: chunks in read order, each valid until the second following call */
int rsem_b200_sim_next_devices(rsem_b200_sim_multi* multi, const char* text[2], uint64_t bytes[2], uint64_t* n_reads);
typedef struct rsem_b200_sim_devices_stats {
    rsem_b200_sim_stats sum;  /* summed over the contexts; generate_ms excludes the jumps                       */
    double jump_ms;           /* mt19937 jumps between a context's windows (on the generator streams, overlapped) */
    double handoff_ms;        /* host time waiting for each window's chain resolution, whose exit is the next
                                 window's entry point                                                         */
} rsem_b200_sim_devices_stats;
/* counts and failed attempts summed over the contexts, stats (may be NULL), per_device (n entries, may be NULL: each
 * context's own phases); ends every context's run and frees the handle                                     */
int rsem_b200_sim_end_devices(rsem_b200_sim_multi* multi, double* counts, uint64_t* resim,
                              rsem_b200_sim_devices_stats* stats, rsem_b200_sim_stats* per_device);
/* Device-free: state_out = the boost::mt19937 state after J draws from state_in.  state[0..623] are the words,
 * state[624] the index (624: twist before the next draw).  Runs on the host; needs no GPU.                     */
int rsem_b200_mt19937_jump(const uint32_t state_in[625], uint64_t J, uint32_t state_out[625]);

/* ---- rsem-calculate-credibility-intervals, Phase II (K8, ci_kernels.cu) ------------------------------------------------
 * Replaces the reference's temp-file transpose (Buffer.h:41-80, calcCI.cpp:302-305) and calculate_credibility_intervals
 * (calcCI.cpp:286-508).  The caller draws the samples (calcCI.cpp:93-164) and pushes each one's TPM row and l_bar at a
 * fixed sample index; ci_end returns the intervals of every transcript, gene and (allele-specific references) isoform.
 * gene_start / isoform_start are GroupInfo start arrays (1-based transcript ids, n + 1 entries, GroupInfo.h:34-53);
 * part_gene_start are the gene ranges of the reference's Phase II threads (calcCI.cpp:402-420): the isoform sums of an
 * allele-specific reference run on across the isoforms of one range (calcCI.cpp:308-345), so their ranges matter.
 * threshold = nSamples - (int(confidence * nSamples - 1e-8) + 1) (calcCI.cpp:221).
 * device_budget: bytes of device memory to use (0 = what is free less 512 MB); when the sample matrix does not fit next
 * to the rows of the largest gene it is kept in pinned host memory and gathered block by block.                   */
typedef struct rsem_b200_ci_params {
    int32_t M;
    int32_t n_genes;
    const int32_t* gene_start;       /* n_genes + 1 */
    int32_t n_isoforms;              /* 0 unless allele-specific */
    int32_t n_parts;
    const int32_t* isoform_start;    /* n_isoforms + 1, or NULL */
    const int32_t* part_gene_start;  /* n_parts + 1: 0 ... n_genes */
    int64_t n_samples;
    int32_t threshold;
    int32_t reserved;
    uint64_t device_budget;
} rsem_b200_ci_params;
/* device time per phase, summed over the blocks (CUDA events) */
typedef struct rsem_b200_ci_stats {
    double transpose_ms;  /* sample-major -> transcript-major rows (with the column gather when not resident) */
    double sums_ms;       /* FPKM rows, gene sums, isoform sums                                                 */
    double sort_ms;       /* segmented sort of every row                                                        */
    double interval_ms;   /* calcCI per row                                                                     */
    uint64_t blocks;
    int32_t resident;     /* 1: the sample matrix was kept on the device                                        */
    int32_t reserved;
} rsem_b200_ci_stats;
/* sets up a run and its sample matrix (Buffer.h:16-31 sizes a host buffer instead).  The context keeps K8's buffers
 * from one run to the next and grows them only when a run needs more, so a run whose shape it has already held makes no
 * allocation; when the kept buffers would then exceed both the budget and what this run needs, the larger ones are
 * released first.  With device_budget = 0 the memory the context keeps for K8 counts as free.  ctx_destroy frees them. */
int rsem_b200_ci_begin(rsem_b200_ctx* ctx, const rsem_b200_ci_params* params);
/* count samples from index first: rows = count x M TPMs (tpm + 1 of calcCI.cpp:146), l_bars = count values.  Thread
 * safe; the buffers may be reused when it returns (Buffer::write, Buffer.h:41-49)                                 */
int rsem_b200_ci_push(rsem_b200_ctx* ctx, const float* rows, const float* l_bars, int64_t first, int64_t count);
/* intervals as (lb, ub, cqv) of TPM then of FPKM, 6 floats per item: transcripts (M), genes (n_genes), isoforms
 * (n_isoforms; may be NULL when 0) (calcCI.cpp:313-385, 446-496 prints them); ends the run and keeps its buffers  */
int rsem_b200_ci_end(rsem_b200_ctx* ctx, float* transcripts, float* genes, float* isoforms, rsem_b200_ci_stats* stats);

/* ---- rsem-for-ebseq-calculate-clustering-info (K9, kmer_kernels.cu) ----------------------------------------------------
 * Replaces the k-mer candidate list, its std::sort and the pass over groups of equal k-mers
 * (EBSeq/calcClusteringInfo.cpp:101-130).  Transcript t (0-based, input order) is bases[offsets[t] .. offsets[t + 1]), one
 * code per base: 0 A, 1 C, 2 G, 3 T, 4 N (the caller maps every other letter to N, as convert() does, :51-59).  For each
 * t, shared_counts[t] = the number of start positions j in [0, len_t - k + 1) whose k-mer (forward strand) also starts at
 * some position of a different transcript: the sum of the group runs with numerator < denominator (:117-130).  Repeats
 * inside one transcript do not count; N matches N.  The ratio the tool prints is shared_counts[t] / effL_t (:132-134).
 * max_device_bytes: device memory for the packed bases, the offsets, the counts and the hash table (0 = what is free
 * less 512 MB).  When a table of 2 slots (12 bytes each) per position does not fit, the k-mers are split by hash into
 * passes = ceil(2 positions / table slots) passes over one table; the counts are the same for every budget.
 * fingerprint_bits: bits of the hash kept in a slot beside the position (0 = 24; 1..24).  Equal fingerprints are
 * verified base by base, so the counts do not depend on it; small values make most probes verify (tests).          */
typedef struct rsem_b200_kmer_params {
    int32_t k;                   /* >= 1 */
    int32_t fingerprint_bits;
    uint64_t n_transcripts;
    const uint64_t* offsets;     /* n_transcripts + 1, offsets[0] = 0, non-decreasing */
    const uint8_t* bases;        /* offsets[n_transcripts] codes 0..4 */
    uint64_t max_device_bytes;
} rsem_b200_kmer_params;
/* device time per phase (CUDA events), summed over the passes */
typedef struct rsem_b200_kmer_stats {
    uint64_t positions;     /* k-mer start positions (the reference's cands.size()) */
    uint64_t table_slots;
    uint64_t input_bytes;   /* packed bases (2 + 1 bits per base), offsets and counts */
    uint64_t table_bytes;
    int32_t passes;         /* 0 when there are no positions (no device work) */
    int32_t reserved;
    double pack_ms;         /* bases to the device and packing */
    double insert_ms;       /* table clearing and the insert pass */
    double count_ms;        /* the count pass */
} rsem_b200_kmer_stats;
int rsem_b200_kmer_shared(rsem_b200_ctx* ctx, const rsem_b200_kmer_params* params, uint64_t* shared_counts,
                          rsem_b200_kmer_stats* stats /* may be NULL */);

/* ---- rsem-tbam2gbam (K10, gbam_kernels.cu) -----------------------------------------------------------------------------
 * Replaces the per-alignment work of BamConverter::process (BamConverter.h:92-303): convert() with tr2chr
 * (sam_utils.h:137-208), flipSeq / flipQual, modifyTags, the CollapseMap of each read (bc_aux.h) and
 * writeCollapsedLines.  One call converts one batch of whole groups and returns the output records in output order.
 *
 * Batch: every record as BAM stores it, preceded by its u32 block_size, at data + rec_off[r].  A unit is one record or
 * a mate pair (mate 1 first): records [unit_rec[u], unit_rec[u + 1]).  unit_tr[u] = the transcript (1..M) of a mapped
 * unit, 0 for an unmapped unit, which is written through unchanged.  unit_group[u] is non-decreasing; the mapped units
 * of one group (a run of one read name) collapse as in CollapseMap; an unmapped unit is a group of its own.
 * The caller does the framing and the validation the reference does while it reads (BamConverter.h:110-150).
 *
 * Tables (uploaded on the first call with a given `tables` pointer and kept until the context is destroyed):
 * out_tid[t] = the chrlist index of transcript t's seqname (-1: not in the chrlist); minus[t] = 1 on '-' strand;
 * exons of t are [exon_off[t], exon_off[t + 1]) as 1-based inclusive (start, end), ascending (Transcript.h:119-148).
 * mapq_prb[m] = the smallest float prb >= 0 with bam_prb_to_mapq(prb) >= m, m = 1..100 (sam_utils.h:72-76, built on
 * the host with the host's log10); the device gives MAPQ = #{m : prb >= mapq_prb[m]}.
 *
 * out: out_cap bytes; *out_bytes = what the batch wrote (block_size + record, in output order).  On a record the
 * reference would abort on (a base code other than 1/2/4/8/15, a negative genomic position, a read outside the exons,
 * a transcript without a chrlist entry, a kept pair whose mate 2 lacks the ZW of mate 1, a ZW sum below 0 or NaN,
 * an optional field of unknown type) the call returns RSEM_B200_ERR_ARG with stats->bad_unit = the first such unit. */
typedef struct rsem_b200_gbam_tables {
    int32_t M;
    int32_t reserved;
    const int32_t* out_tid;     /* M + 1 */
    const uint8_t* minus;       /* M + 1 */
    const int32_t* length;      /* M + 1: Transcript::length */
    const int64_t* exon_off;    /* M + 2 */
    const int32_t* exon_start;  /* exon_off[M + 1] */
    const int32_t* exon_end;
    const float* mapq_prb;      /* 101; [0] unused */
} rsem_b200_gbam_tables;
typedef struct rsem_b200_gbam_batch {
    uint64_t n_records, n_units, n_bytes;
    const uint8_t* data;        /* n_bytes */
    const uint64_t* rec_off;    /* n_records */
    const uint32_t* unit_rec;   /* n_units + 1 */
    const uint32_t* unit_group; /* n_units */
    const int32_t* unit_tr;     /* n_units */
} rsem_b200_gbam_batch;
typedef struct rsem_b200_gbam_stats {
    double device_ms;           /* CUDA events: copies in, convert, sort, collapse, emit, copy out */
    uint64_t units_written;     /* kept + written-through units */
    int64_t bad_unit;           /* -1 unless the call failed on a record */
} rsem_b200_gbam_stats;
int rsem_b200_gbam_convert(rsem_b200_ctx* ctx, const rsem_b200_gbam_tables* tables, const rsem_b200_gbam_batch* batch,
                           uint8_t* out, uint64_t out_cap, uint64_t* out_bytes, rsem_b200_gbam_stats* stats /* may be NULL */);

/* ---- rsem-bam2wig / rsem-bam2readdepth (K11, wiggle_kernels.cu) ------------------------------------------------------
 * Replaces the per-alignment work of build_wiggles (wiggle.cpp:16-83): for every mapped record, w (bam_aux2f of its
 * first ZW: 'f' widened, 'd', any other type 0.0; no ZW: the record adds nothing; 1.0 with no_fractional_weight, the
 * optional fields then not read) is added to every position of every M operation of its CIGAR; D, N, = and X advance
 * the position, every other operation neither adds nor advances.  Each position's value is the double sum, from +0.0,
 * of its contributions in record order (x86 SSE rules for NaN and infinities); nothing is reassociated.
 *
 * Batch: every mapped record as BAM stores it, preceded by its u32 block_size, at data + rec_off[r].  A run is a
 * maximal stretch of records on one target; rec_run[r] is the record's run (non-decreasing, < n_runs) and run_len[i]
 * the target's length.  The caller checks tid and pos >= 0 (the device does not see tid).  continues = 1: run 0 is the
 * run the previous call left resident.  keep_last = 1: the last run stays resident for the next call, which may
 * continue it.  A call with n_runs = 0 and keep_last = 0 returns the resident run.
 *
 * out: the depth arrays of the runs this call finishes, concatenated in order: the previously resident run first when
 * this call does not continue it, then runs 0 .. n_runs - 1 - keep_last.  *out_len = doubles written (<= out_cap).
 * On a record the reference has no defined result for (an M operation that ends past run_len, an optional field of
 * unknown type or one cut short by the record's end before the first ZW, a CIGAR past the record's end) the call
 * returns RSEM_B200_ERR_ARG with stats->bad_record = the first such record and stats->bad_code its kind (1 M past the
 * end, 2 unknown optional field type, 3 truncated record); the resident run is then dropped.  On every other failure
 * (arguments, a run the device cannot allocate, CUDA errors) stats->bad_record is -1.                                                                                            */
typedef struct rsem_b200_wig_batch {
    uint64_t n_records, n_bytes;
    const uint8_t* data;        /* n_bytes */
    const uint64_t* rec_off;    /* n_records */
    const uint32_t* rec_run;    /* n_records */
    const uint32_t* run_len;    /* n_runs */
    uint32_t n_runs;
    int32_t continues;
    int32_t keep_last;
    int32_t no_fractional_weight;
} rsem_b200_wig_batch;
typedef struct rsem_b200_wig_stats {
    double device_ms;           /* CUDA events: copies in, parse, scans, emit, sort, accumulate, copies out */
    uint64_t blocks;            /* M operations that add */
    uint64_t entries;           /* (tile, block) pairs */
    int64_t bad_record;         /* -1 unless the call failed on a record */
    int32_t bad_code;
    int32_t reserved;
} rsem_b200_wig_stats;
int rsem_b200_wig_depth(rsem_b200_ctx* ctx, const rsem_b200_wig_batch* batch, double* out, uint64_t out_cap,
                        uint64_t* out_len, rsem_b200_wig_stats* stats /* may be NULL */);

/* ---- instrumentation (bench / tests) ----------------------------------------------------------- */
/* number of kernels this library launched on ctx since creation */
/* ---- K12: frozen-conprb rounds of many samples at once (rsem-run-em-batch) --------------------------------------
 * A batch holds the frozen matrices (conprb, ncpv of ROUND >= 11) of several samples in one device arena and runs their
 * rounds of EM.cpp:364-416 (E_STEP EM.cpp:199-244, M-step EM.cpp:385-398, bChange / totNum EM.cpp:406-413, stop test
 * EM.cpp:416) in one kernel: a CTA owns a sample and runs its rounds back to back.  Each sample is kept in the space
 * of the transcripts its hits name; this is exact from round 2 on, where theta is 0 for every other transcript.
 * The batch lives on `ctx`'s device and stream; destroy it before the context.                                      */

/* capacity_bytes = 0: half of the device memory free at the call. */
int rsem_b200_batch_create(rsem_b200_ctx* ctx, uint64_t capacity_bytes, rsem_b200_batch** out);
int rsem_b200_batch_destroy(rsem_b200_batch* batch);

/* Device bytes a sample of this shape takes in an arena (m = its number of distinct transcripts), or
 * RSEM_B200_ERR_UNSUPPORTED when it is outside the batch layout (more than 2^20 hits, more than 12287 distinct
 * transcripts, or a read with more than 2048 alignments): such a sample runs with rsem_b200_em_rounds.  No GPU needed. */
int rsem_b200_batch_sample_bytes(uint64_t N, uint64_t H, const uint64_t* row_ptr, int32_t m, uint64_t* bytes);

/* Adds a sample whose next round is `first_round` (>= 2): its CSR matrix (row_ptr N + 1, sid H, signed as in the .dat),
 * frozen conprb (H) / ncpv (N), theta (M + 1) after round first_round - 1 and N0.  Refused with RSEM_B200_ERR_ARG when
 * theta is not exactly 0 for a transcript no hit names, RSEM_B200_ERR_FULL when the arena has no room left for it,
 * RSEM_B200_ERR_UNSUPPORTED as rsem_b200_batch_sample_bytes.  *slot receives its handle.                            */
int rsem_b200_batch_add(rsem_b200_batch* batch, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr,
                        const int32_t* sid, const double* conprb, const double* ncpv, const double* theta, double n0,
                        int32_t first_round, int32_t min_round, int32_t max_round, int32_t* slot);

/* One launch: every sample that has not stopped runs up to `max_rounds` rounds.  Arrays are indexed by slot and sized
 * by rsem_b200_batch_slots: stats (slots x max_rounds, may be NULL) receives each round's (sum, bChange, totNum) of
 * the "ROUND = ..." line (EM.cpp:415), rounds_run the number of rounds the slot ran, stopped 1 once the slot's loop
 * condition ROUND < min_round || (totNum > 0 && ROUND < max_round) became false.                                   */
int rsem_b200_batch_run(rsem_b200_batch* batch, int32_t max_rounds, rsem_b200_round_stats* stats, int32_t* rounds_run,
                        int32_t* stopped);
int rsem_b200_batch_slots(rsem_b200_batch* batch, int32_t* n_slots);

/* Final pass with calcExpectedWeights = true (EM.cpp:460-478) for one sample: theta (M + 1) and the expected counts
 * (M + 1, WITHOUT N0) scattered back to transcript ids, and when not NULL the posteriors per hit (H) and of the noise
 * entry per read (N), as rsem_b200_expected_weights gives them.  theta is not changed; the sample stays in the batch. */
int rsem_b200_batch_final(rsem_b200_batch* batch, int32_t slot, double* theta, double* counts, double* post,
                          double* post0);
/* Frees a sample's bytes in the arena. */
int rsem_b200_batch_remove(rsem_b200_batch* batch, int32_t slot);
/* K12 device time summed over launches (CUDA events) and the sample-rounds they ran. */
int rsem_b200_batch_timing(rsem_b200_batch* batch, double* total_ms, uint64_t* sample_rounds);

int rsem_b200_launch_count(rsem_b200_ctx* ctx, uint64_t* launches);
/* device time (ms, CUDA events on the context's stream) spent in the E/M kernel (K2) launches and
 * their number since the last reset; used for the roofline figure.                              */
int rsem_b200_estep_timing(rsem_b200_ctx* ctx, double* total_ms, uint64_t* launches, int32_t reset);
/* enable per-launch event timing of K2 (off by default: it adds two event records per round)    */
int rsem_b200_set_profiling(rsem_b200_ctx* ctx, int32_t enabled);
/* select the E/M kernel variant: 0 = auto (equivalence-class layout for frozen-conprb rounds, row groups when
 * posteriors are written), 2 = direct (no smem staging), 4 = row groups on CTA-staged tiles (TMA, no CTA
 * barriers, dynamic row batches), 5 = equivalence-class layout, fail if the matrix is outside its limits.
 * Any other value returns RSEM_B200_ERR_ARG.                                                          */
int rsem_b200_set_estep_variant(rsem_b200_ctx* ctx, int32_t variant);

/* Equivalence-class layout the frozen-conprb rounds run on (derived from the hit matrix on first use; reads with
 * identical transcript lists - the reference has no counterpart, it walks HitContainer row by row, EM.cpp:199-244).
 * out[10] = { built (0/1), rows in the layout, rows handled by the long-row launch, segments, batches, tiles,
 *             staged doubles (conprb + ncpv), staged ids, tiles of the main launch, hits in run batches }.  Streamed
 *             bytes per round = 8 out[6] + 4 out[7] + 16 out[4].  Tiles [0, out[8]) hold the rows of at most 127
 *             hits; the other out[5] - out[8] tiles (rows of 128..2047 hits) run in a second launch.  A run batch's
 *             rows hit consecutive transcripts, and it stages one id (the first) per segment, or one per batch when
 *             all its segments belong to one class, instead of every id.                                          */
int rsem_b200_class_layout_info(rsem_b200_ctx* ctx, uint64_t* out /* 10 */);
/* CSR layout the row-group and direct E-steps run on (built by upload_hits / adopt_device_matrix).  out[6] =
 * { tiles of the row kernel (0: every CSR pass runs the direct kernel), tile weight C (a tile holds the rows r with
 *   row_ptr[r] + C r in [k W, (k + 1) W), W = 4094 - longest row; 0 without tiles), lanes per row of the row kernel,
 *   lanes per row of the direct kernel, longest row, 1 if some row has no hits }.  No GPU work.                  */
int rsem_b200_csr_layout_info(rsem_b200_ctx* ctx, uint64_t* out /* 6 */);
/* Busy time (ns, %globaltimer) of every persistent CTA in the latest class-layout E-step launch over the main tiles
 * (see rsem_b200_class_layout_info): the evidence for the segmented reduction's load balance on skewed matrices
 * (BASELINE configs[4]).  *n = CTAs written (<= cap); 0 when the layout has no main tiles.                         */
int rsem_b200_estep_cta_times(rsem_b200_ctx* ctx, uint64_t* out_ns, int32_t cap, int32_t* n);
/* Where the class-layout E-step's time went in its latest main launch with profiling on (rsem_b200_set_profiling):
 * out_ns[8 i .. 8 i + 7] = { ns the consumer warps of CTA i spent blocked on staged data (summed over the warps),
 * ns a separate copy-issuing warp spent blocked on a free stage (0 when the consumer warps issue their own copies),
 * consumer warps of CTA i, then in SM cycles, summed over the consumer warps: front (a batch's descriptor, ids and
 * theta gather until theta is usable), rows (the row walk),
 * flush (fold + reductions on the count vector), hand-over (releasing a stage -> the next stage's data seen), and
 * last the SM cycles CTA i was busy }.  out_ns holds 8 cap entries.  *n = CTAs written (<= cap); 0 when the latest
 * launch ran without profiling.                                                                                    */
int rsem_b200_estep_wait_times(rsem_b200_ctx* ctx, uint64_t* out_ns, int32_t cap, int32_t* n);

#ifdef __cplusplus
}
#endif
#endif /* RSEM_B200_H_ */
