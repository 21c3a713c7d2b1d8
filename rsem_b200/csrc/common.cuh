// Internal declarations shared by the translation units of librsem_b200.so.
// Nothing here is part of the public ABI (see include/rsem_b200.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/rsem_b200.h"

namespace rsem_b200 {

// The reference's clamp constant (utils.h:18): values below it are treated as exactly 0.
constexpr double kEpsilon = 1e-300;

void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define RB_CUDA(call)                                                       \
    do {                                                                    \
        cudaError_t _e = (call);                                            \
        if (_e != cudaSuccess) return ::rsem_b200::cuda_fail(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define RB_ARG(cond, msg)                         \
    do {                                          \
        if (!(cond)) {                            \
            ::rsem_b200::set_error(msg);          \
            return RSEM_B200_ERR_ARG;             \
        }                                         \
    } while (0)

// ---- NCCL, loaded at run time (nccl_dyn.cpp) -----------------------------------------------
struct NcclApi;
const NcclApi* nccl_api();  // nullptr + last_error set when libnccl.so.2 cannot be loaded
int nccl_unique_id(void* id128);
int nccl_comm_init(void** comm, const void* id128, int n_ranks, int rank);
int nccl_allreduce_sum_f64(void* comm, double* buf, size_t n, cudaStream_t stream);
int nccl_allgather_bytes(void* comm, const void* send, void* recv, size_t bytes_per_rank, cudaStream_t stream);
int nccl_comm_destroy(void* comm);

// ---- device-side model (pointers into one packed device buffer) -----------------------------
struct DevLenDist {
    int lb, ub, span;
    const double* pdf;
    const double* cdf;
};

struct DevModel {
    int model_type, M, seed_len, est_rspd, rspd_B, has_mld, pro_len;
    double ori[2];
    DevLenDist gld, mld;
    const double* rspd_pdf;
    const double* rspd_cdf;
    const double* profile;
    const double* noise_profile;
    const double* mw;
};

// raw accumulation targets of the model-update kernel (K3)
struct DevStats {
    double* profile;        // [100|pro_len][5][5]
    double* noise_profile;  // [100][5] or [5]
    double* gld_pdf;        // gld_span + 1
    int gld_lb, gld_span;
    double* rspd_pdf;       // B + 2
    size_t total_doubles;   // size of the packed buffer all four point into
};

struct DevReads {
    int n_mates = 0;
    bool has_qual = false;
    uint64_t* off[2] = {nullptr, nullptr};
    uint8_t* base[2] = {nullptr, nullptr};
    uint8_t* qual[2] = {nullptr, nullptr};
    uint8_t* lowq = nullptr;
    uint8_t* uni = nullptr;                 // per read: all hits show the same bases (model_kernels.cu); needs hits + refs too
    bool uni_valid = false;
    int max_len = 0;
    int qmax = -1;                          // largest quality value (computed on first use)
    unsigned long long total_bases[2] = {0, 0};
};

struct DevRefs {
    int M = 0;
    uint64_t* seq_off = nullptr;
    uint8_t* seq = nullptr;
    int32_t* full_len = nullptr;
    int32_t* tot_len = nullptr;
    uint64_t* mask_off = nullptr;
    uint32_t* mask_words = nullptr;
};

struct DevGibbs {
    uint64_t N1 = 0, E = 0;
    int M = 0;
    uint64_t* row_ptr = nullptr;
    int32_t* sid = nullptr;
    double* conprb = nullptr;
    // component-parallel sampler (gibbs_kernels.cu): reads grouped by connected component
    int32_t* order = nullptr;      // N1 read ids: component by component (longest first), read order inside
    uint64_t* p_off = nullptr;     // rows re-laid in that slot order
    int32_t* p_sid = nullptr;
    double* p_con = nullptr;
    int32_t* seg_start = nullptr;  // n_segs + 1 offsets into `order`
    int32_t* seg_ntr = nullptr;    // transcripts per component; < 32: rows (p_sid) and assignments hold local ids
    int32_t* seg_tid_off = nullptr;
    int32_t* comp_tids = nullptr;  // sorted transcript ids of every component
    size_t n_comp_tids = 0;        // entries of comp_tids
    int32_t n_segs = 0;
    uint32_t max_len = 0;
    bool empty_row = false;        // some read has no entry: gibbs_run refuses the matrix before any launch
    bool ready = false;            // the upload, component layout included, completed (a source for gibbs_upload_from)
};

// count reduction over NVLink peer memory (p2p.cu)
constexpr int kMaxP2PRanks = 8;
struct P2PState {
    bool on = false;
    int n = 0;
    uint64_t seq = 0;                       // rounds reduced so far (same on every rank): buffer parity + flag value
    double* count_buf = nullptr;            // 2 x (M + 1): K2 accumulates into [(seq + 1) & 1]
    unsigned long long* flags = nullptr;    // flags[r] = last round rank r has completed
    double* peer_count[kMaxP2PRanks] = {};
    unsigned long long* peer_flags[kMaxP2PRanks] = {};
    void* opened_count[kMaxP2PRanks] = {};  // cudaIpcOpenMemHandle results to close
    void* opened_flags[kMaxP2PRanks] = {};
};

// equivalence-class layout of the hit matrix for the frozen-conprb rounds (class_kernels.cu)
constexpr int kWaitRecord = 8;  // uint64 entries per CTA in ClassLayout::wait_ns
struct ClassLayout {
    bool built = false;
    uint64_t vals_epoch = 0;        // conprb epoch the value stream was gathered at (0 = never)
    uint32_t n_rows = 0, n_long = 0, n_segs = 0, n_batches = 0, n_tiles = 0, R = 0;
    uint32_t n_tiles_main = 0;      // tiles [0, n_tiles_main): rows of <= 127 hits; the rest: longer rows (own launch)
    uint64_t n_vals = 0, n_ids = 0;
    uint64_t n_run_hits = 0;        // hits in batches whose segments hit consecutive transcripts (ids stored as firsts)
    double* vals = nullptr;         // per batch: ncpv [row][segment], then conprb [(row, column)][segment]
    int32_t* ids = nullptr;         // per batch: transcript ids [column][segment] (or [column] for a one-class batch);
                                    // a run batch: first id [segment] (or one for a one-class batch)
    void* desc = nullptr;           // BatchDesc[n_batches]
    void* tile = nullptr;           // TileRec[n_tiles + 1]
    uint32_t* batch_first = nullptr;  // first segment (final order) of every batch
    uint32_t* fseg_first = nullptr;   // first sorted row position of every segment (final order)
    uint32_t* rows = nullptr;         // sorted position -> original row
    uint32_t* long_rows = nullptr;    // original rows with more than kLongDeg hits
    uint32_t* claim = nullptr;        // {next tile, CTAs done} of the class-kernel launch in flight; 0 between launches
    uint64_t* cta_ns = nullptr;       // per-CTA busy time (ns) of the latest class-kernel launch over the main tiles
    uint64_t* wait_ns = nullptr;      // per-CTA wait and phase accounting of the latest profiled main launch
                                      // (kWaitRecord entries per CTA, see rsem_b200_estep_wait_times)
    uint32_t last_grid = 0;
    bool last_profiled = false;       // the latest class-kernel launch ran with profiling on (wait_ns is current)
};

// skip_aux of htslib 1.3 (sam.c): bytes of the optional-field value whose type byte is at s, type byte included;
// 0 = unknown type.  A 'Z' / 'H' value without its NUL before `end` gives a length that runs past `end`.  Used by K10
// and K11 to walk a record's optional fields.
#ifdef __CUDACC__
__device__ __forceinline__ int aux_len(const uint8_t* s, const uint8_t* end) {
    const uint8_t t = *s;
    switch (t) {
        case 'A': case 'c': case 'C': return 2;
        case 's': case 'S': return 3;
        case 'i': case 'I': case 'f': return 5;
        case 'd': return 9;
        case 'Z': case 'H': {
            const uint8_t* q = s + 1;
            while (q < end && *q) ++q;
            return (int)(q - s) + 1;
        }
        case 'B': {
            const uint8_t sub = s[1];
            const int sz = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : (sub == 'i' || sub == 'I' || sub == 'f') ? 4 : 0;
            if (sz == 0) return 0;
            const uint32_t n = s[2] | (s[3] << 8) | (s[4] << 16) | ((uint32_t)s[5] << 24);
            return 6 + sz * (int)n;
        }
    }
    return 0;
}
#endif

struct SimState;  // sim_kernels.cu
struct CiState;   // ci_kernels.cu
struct GbamState; // gbam_kernels.cu
struct WigState;  // batch_kernels.cu
int batch_create(rsem_b200_ctx* ctx, uint64_t capacity, rsem_b200_batch** out);
void batch_destroy(rsem_b200_batch* b);
int batch_sample_bytes(uint64_t N, uint64_t H, const uint64_t* row_ptr, int32_t m, uint64_t* bytes);
int batch_add(rsem_b200_batch* b, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr, const int32_t* sid,
              const double* conprb, const double* ncpv, const double* theta, double n0, int32_t first_round,
              int32_t min_round, int32_t max_round, int32_t* slot);
int batch_run(rsem_b200_batch* b, int32_t rounds, rsem_b200_round_stats* stats, int32_t* rounds_run, int32_t* stopped);
int batch_final(rsem_b200_batch* b, int32_t slot, double* theta, double* counts, double* post, double* post0);
void batch_remove(rsem_b200_batch* b, int slot);
int batch_slots(const rsem_b200_batch* b);
bool batch_slot_live(const rsem_b200_batch* b, int slot);
int batch_timing(const rsem_b200_batch* b, double* ms, uint64_t* sample_rounds);

// wiggle_kernels.cu

}  // namespace rsem_b200

struct rsem_b200_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;   // host -> device copies that overlap with work on `stream` (upload_conprb)
    uint64_t launches = 0;
    uint64_t dev_bytes = 0;

    // device block cache (capi.cu: block_alloc / block_free): the buffers of a released hit matrix and of its derived
    // layouts are kept and handed out again to requests of exactly the same size, so that repeated jobs of one shape pay
    // neither cudaMalloc nor the device-wide synchronisation of cudaFree.  All users order their work on `stream`.
    std::vector<std::pair<size_t, void*>> idle_blocks;
    std::unordered_map<void*, size_t> live_blocks;
    size_t idle_bytes = 0;

    // hit matrix
    uint64_t N = 0, H = 0;
    int M = 0;
    uint32_t max_deg = 0;
    uint64_t* row_ptr = nullptr;
    int32_t* sid = nullptr;      // signed: sign = strand (K1 / K3)
    int32_t* sid_abs = nullptr;  // |sid|: the stream K2 reads
    int32_t* pos = nullptr;
    int32_t* insertL = nullptr;
    double* conprb = nullptr;
    double* ncpv = nullptr;
    double* post = nullptr;   // posterior / frac per hit (lazily allocated)
    double* post0 = nullptr;  // posterior of the noise entry per read
    bool conprb_valid = false;
    uint64_t conprb_epoch = 1;  // bumped whenever conprb / ncpv change (derived layouts compare it)
    rsem_b200::ClassLayout cls;

    // E-step tiling (em_kernels.cu)
    uint64_t* tile_row = nullptr;
    uint64_t* tile_hit = nullptr;
    uint32_t n_tiles = 0;
    int group = 16;       // lanes cooperating on one row (K1 / K3 / direct K2)
    int rows_group = 8;   // lanes per row of the row-group K2 (variant 4)
    int variant = 0;      // 0 auto, 2 direct, 4 row groups, 5 class layout

    // EM state
    double* theta = nullptr;   // M + 1
    double* count = nullptr;   // M + 1
    int* done_flag = nullptr;  // device int: 1 once the loop condition ended the run
    int* err_flag = nullptr;
    rsem_b200_round_stats* d_stats = nullptr;
    int stats_cap = 0;

    // model + reads + refs
    rsem_b200::DevModel model{};
    double* model_buf = nullptr;
    size_t model_buf_doubles = 0;
    bool model_set = false;
    rsem_b200::DevStats stats{};
    double* stats_buf = nullptr;
    size_t stats_buf_doubles = 0;
    rsem_b200::DevReads reads;
    rsem_b200::DevRefs refs;

    rsem_b200::DevGibbs gibbs;
    rsem_b200::SimState* sim = nullptr;  // rsem-simulate-reads between sim_begin and sim_end
    rsem_b200::CiState* ci = nullptr;    // rsem-calculate-credibility-intervals between ci_begin and ci_end
    rsem_b200::GbamState* gbam = nullptr;  // rsem-tbam2gbam: transcript tables and batch scratch
    rsem_b200::WigState* wig = nullptr;    // rsem-bam2wig / rsem-bam2readdepth: the resident run and batch scratch

    // multi-GPU
    void* comm = nullptr;
    int n_ranks = 1, rank = 0;
    rsem_b200::P2PState p2p;
    double* k2_target = nullptr;   // where K2 accumulates (count, or the peer-mapped buffer of the round)

    // RSEM_B200_PHASE_TIMING=1: device time per kernel of the model rounds (K1, K2 with posteriors, K3), printed at destroy
    bool phase_timing = false;
    cudaEvent_t ph_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double ph_ms[3] = {0, 0, 0};
    uint64_t ph_n[3] = {0, 0, 0};

    // profiling of K2
    bool profiling = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pool;
    size_t ev_used = 0;
    double estep_ms = 0;
    uint64_t estep_launches = 0;
};

namespace rsem_b200 {

// allocation with accounting; every array gets 256 B of tail padding so that 16-byte granular
// bulk copies may over-read the last tile.
// capi.cu: cached device blocks (see rsem_b200_ctx::idle_blocks)
cudaError_t block_alloc(rsem_b200_ctx* ctx, void** p, size_t bytes);
void block_free(rsem_b200_ctx* ctx, void* p);
void block_cache_flush(rsem_b200_ctx* ctx);

template <class T>
int dev_alloc(rsem_b200_ctx* ctx, T** p, size_t n) {
    size_t bytes = n * sizeof(T) + 256;
    void* q = nullptr;
    cudaError_t e = block_alloc(ctx, &q, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
    // the padding is read (never used) by the E-step's bulk copies, which round up to 16 B: keep it defined
    cudaMemset(static_cast<char*>(q) + n * sizeof(T), 0, 256);
    ctx->dev_bytes += bytes;
    *p = static_cast<T*>(q);
    return 0;
}
template <class T>
void dev_free(rsem_b200_ctx* ctx, T** p, size_t n) {
    if (*p) {
        block_free(ctx, *p);
        ctx->dev_bytes -= n * sizeof(T) + 256;
        *p = nullptr;
    }
}

// em_kernels.cu
int em_build_tiles(rsem_b200_ctx* ctx);
int em_launch_estep(rsem_b200_ctx* ctx, bool write_post);
int em_prepare_frozen_layout(rsem_b200_ctx* ctx);
int em_launch_theta_update(rsem_b200_ctx* ctx, double n0, int round, int min_round, int max_round, int stats_slot);
int em_max_degree(rsem_b200_ctx* ctx, uint32_t* max_deg);
int em_make_abs_sid(rsem_b200_ctx* ctx);

// class_kernels.cu
void class_free(rsem_b200_ctx* ctx);
int class_build(rsem_b200_ctx* ctx);
int class_fill_vals(rsem_b200_ctx* ctx);
int class_launch_estep(rsem_b200_ctx* ctx);

// p2p.cu
void p2p_release(rsem_b200_ctx* ctx);
int p2p_setup(rsem_b200_ctx* ctx);
double* p2p_k2_target(rsem_b200_ctx* ctx);
int p2p_reduce(rsem_b200_ctx* ctx);

// model_kernels.cu
int model_launch_conprb(rsem_b200_ctx* ctx);
int model_launch_update(rsem_b200_ctx* ctx);

// gibbs_kernels.cu
int gibbs_run(rsem_b200_ctx* ctx, const rsem_b200_gibbs_params* p, int32_t* count_vectors, double* chain_acc,
              rsem_b200_gibbs_stats* stats);
int gibbs_prepare(rsem_b200_ctx* ctx, const uint64_t* row_ptr, const int32_t* sid);
// host side of the component-parallel sampler's layout (gibbs_kernels.cu): components, segments longest first, local
// ids of register-resident components, rows in slot order.  gibbs_prepare and the Gibbs batch (K13) both build it.
struct GibbsLayout {
    uint64_t N1 = 0;
    std::vector<int32_t> order;        // N1 read ids in slot order
    std::vector<uint64_t> p_off;       // N1 + 1 entry offsets of the slots
    std::vector<int32_t> p_sid;        // E ids (local ids in register-resident components)
    std::vector<int32_t> seg_start;    // n_segs + 1
    std::vector<int32_t> seg_ntr;      // n_segs
    std::vector<int32_t> seg_tid_off;  // n_segs + 1
    std::vector<int32_t> comp_tids;
    int32_t n_segs = 0;
    uint32_t max_len = 0;
    bool empty_row = false;
};
int gibbs_layout(const uint64_t* row_ptr, const int32_t* sid, uint64_t N1, int M, GibbsLayout& L);
int gibbs_batch_create(rsem_b200_ctx* c, uint64_t capacity, int worker_ctas, rsem_b200_gibbs_batch** out);
void gibbs_batch_destroy(rsem_b200_gibbs_batch* b);
int gibbs_batch_sample_bytes(uint64_t N1, uint64_t E, int32_t M, int32_t n_genes, int32_t n_samples, int32_t n_chains,
                             uint64_t* bytes);
int gibbs_batch_add(rsem_b200_gibbs_batch* b, uint64_t N1, uint64_t E, const uint64_t* row_ptr, const int32_t* sid,
                    const double* conprb, const rsem_b200_gibbs_params* p, int32_t* slot);
int gibbs_batch_run(rsem_b200_gibbs_batch* b, rsem_b200_gibbs_batch_stats* stats);
int gibbs_batch_result(rsem_b200_gibbs_batch* b, int32_t slot, int32_t* count_vectors, double* chain_acc);
void gibbs_batch_clear(rsem_b200_gibbs_batch* b);

// sim_kernels.cu
int sim_begin(rsem_b200_ctx* ctx, const rsem_b200_sim_params* p);
int sim_next(rsem_b200_ctx* ctx, const char* text[2], uint64_t bytes[2], uint64_t* n_reads);
int sim_end(rsem_b200_ctx* ctx, double* counts, uint64_t* resim, rsem_b200_sim_stats* stats);
void sim_free(rsem_b200_ctx* ctx);

// ci_kernels.cu
int ci_begin(rsem_b200_ctx* ctx, const rsem_b200_ci_params* p);
int ci_push(rsem_b200_ctx* ctx, const float* rows, const float* l_bars, int64_t first, int64_t count);
int ci_end(rsem_b200_ctx* ctx, float* transcripts, float* genes, float* isoforms, rsem_b200_ci_stats* stats);
void ci_free(rsem_b200_ctx* ctx);

// kmer_kernels.cu
int kmer_shared(rsem_b200_ctx* ctx, const rsem_b200_kmer_params* p, uint64_t* counts, rsem_b200_kmer_stats* stats);

// gbam_kernels.cu
int gbam_convert(rsem_b200_ctx* ctx, const rsem_b200_gbam_tables* t, const rsem_b200_gbam_batch* b, uint8_t* out,
                 uint64_t out_cap, uint64_t* out_bytes, rsem_b200_gbam_stats* stats);
void gbam_free(rsem_b200_ctx* ctx);

// wiggle_kernels.cu
int wig_depth(rsem_b200_ctx* ctx, const rsem_b200_wig_batch* b, double* out, uint64_t out_cap, uint64_t* out_len,
              rsem_b200_wig_stats* stats);
void wig_free(rsem_b200_ctx* ctx);

}  // namespace rsem_b200
