// C ABI glue (include/rsem_b200.h): argument checking, device buffer ownership, stream / NCCL
// sequencing.  All arithmetic lives in the *_kernels.cu files.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>

#include "common.cuh"

namespace rsem_b200 {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    char buf[512];
    snprintf(buf, sizeof buf, "CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    g_last_error = buf;
    return RSEM_B200_ERR_CUDA;
}

// ---- device block cache ---------------------------------------------------------------------------------------------
// RSEM_B200_BLOCK_CACHE=0 turns it off (every request goes to cudaMalloc / cudaFree as before).
static bool block_cache_on() {
    static const bool on = !(getenv("RSEM_B200_BLOCK_CACHE") && !strcmp(getenv("RSEM_B200_BLOCK_CACHE"), "0"));
    return on;
}

cudaError_t block_alloc(rsem_b200_ctx* ctx, void** p, size_t bytes) {
    if (bytes == 0) bytes = 1;
    if (block_cache_on()) {
        for (size_t k = 0; k < ctx->idle_blocks.size(); ++k)
            if (ctx->idle_blocks[k].first == bytes) {
                *p = ctx->idle_blocks[k].second;
                ctx->idle_blocks[k] = ctx->idle_blocks.back();
                ctx->idle_blocks.pop_back();
                ctx->idle_bytes -= bytes;
                ctx->live_blocks[*p] = bytes;
                return cudaSuccess;
            }
    }
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaErrorMemoryAllocation && !ctx->idle_blocks.empty()) {   // give the cached blocks back and try again
        cudaGetLastError();
        block_cache_flush(ctx);
        e = cudaMalloc(p, bytes);
    }
    if (e == cudaSuccess) ctx->live_blocks[*p] = bytes;
    return e;
}

void block_free(rsem_b200_ctx* ctx, void* p) {
    if (!p) return;
    auto it = ctx->live_blocks.find(p);
    if (it == ctx->live_blocks.end()) { cudaFree(p); return; }   // not ours (allocated before the cache existed)
    const size_t bytes = it->second;
    ctx->live_blocks.erase(it);
    if (block_cache_on() && bytes >= (1u << 16)) {   // small blocks are not worth keeping
        ctx->idle_blocks.emplace_back(bytes, p);
        ctx->idle_bytes += bytes;
    } else {
        cudaFree(p);
    }
}

void block_cache_flush(rsem_b200_ctx* ctx) {
    if (!ctx->idle_blocks.empty()) cudaStreamSynchronize(ctx->stream);
    for (auto& b : ctx->idle_blocks) cudaFree(b.second);
    ctx->idle_blocks.clear();
    ctx->idle_bytes = 0;
}

namespace {

template <class T>
int upload(rsem_b200_ctx* ctx, T** dst, const T* src, size_t n) {
    if (int rc = dev_alloc(ctx, dst, n)) return rc;
    if (n) RB_CUDA(cudaMemcpyAsync(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

void free_hits(rsem_b200_ctx* c) {
    dev_free(c, &c->row_ptr, c->N + 1);
    dev_free(c, &c->sid, c->H);
    if (c->sid_abs) dev_free(c, &c->sid_abs, c->H);
    if (c->pos) dev_free(c, &c->pos, c->H);
    if (c->insertL) dev_free(c, &c->insertL, c->H);
    dev_free(c, &c->conprb, c->H);
    dev_free(c, &c->ncpv, c->N);
    if (c->post) dev_free(c, &c->post, c->H);
    if (c->post0) dev_free(c, &c->post0, c->N);
    if (c->theta) dev_free(c, &c->theta, (size_t)c->M + 1);
    if (c->count) dev_free(c, &c->count, (size_t)c->M + 1);
    if (c->tile_row) { cudaFree(c->tile_row); c->tile_row = nullptr; }   // small (16 B per ~4000 hits)
    if (c->tile_hit) { cudaFree(c->tile_hit); c->tile_hit = nullptr; }
    c->n_tiles = 0;
    class_free(c);
    if (c->reads.uni) { cudaFree(c->reads.uni); c->reads.uni = nullptr; }   // sized by N, derived from the hits
    c->reads.uni_valid = false;
    c->N = c->H = 0;
    c->conprb_valid = false;
    c->conprb_epoch++;
}

void free_reads(rsem_b200_ctx* c) {
    for (int m = 0; m < 2; ++m) {
        if (c->reads.off[m]) { cudaFree(c->reads.off[m]); c->reads.off[m] = nullptr; }
        if (c->reads.base[m]) { cudaFree(c->reads.base[m]); c->reads.base[m] = nullptr; }
        if (c->reads.qual[m]) { cudaFree(c->reads.qual[m]); c->reads.qual[m] = nullptr; }
    }
    if (c->reads.lowq) { cudaFree(c->reads.lowq); c->reads.lowq = nullptr; }
    if (c->reads.uni) { cudaFree(c->reads.uni); c->reads.uni = nullptr; }
    c->reads.uni_valid = false;
    c->reads.n_mates = 0;
}

void free_refs(rsem_b200_ctx* c) {
    if (c->refs.seq_off) cudaFree(c->refs.seq_off);
    if (c->refs.seq) cudaFree(c->refs.seq);
    if (c->refs.full_len) cudaFree(c->refs.full_len);
    if (c->refs.tot_len) cudaFree(c->refs.tot_len);
    if (c->refs.mask_off) cudaFree(c->refs.mask_off);
    if (c->refs.mask_words) cudaFree(c->refs.mask_words);
    c->refs = DevRefs{};
    c->reads.uni_valid = false;
}

void free_gibbs(rsem_b200_ctx* c) {
    if (c->gibbs.row_ptr) cudaFree(c->gibbs.row_ptr);
    if (c->gibbs.sid) cudaFree(c->gibbs.sid);
    if (c->gibbs.conprb) cudaFree(c->gibbs.conprb);
    if (c->gibbs.order) cudaFree(c->gibbs.order);
    if (c->gibbs.p_off) cudaFree(c->gibbs.p_off);
    if (c->gibbs.p_sid) cudaFree(c->gibbs.p_sid);
    if (c->gibbs.p_con) cudaFree(c->gibbs.p_con);
    if (c->gibbs.seg_start) cudaFree(c->gibbs.seg_start);
    if (c->gibbs.seg_ntr) cudaFree(c->gibbs.seg_ntr);
    if (c->gibbs.seg_tid_off) cudaFree(c->gibbs.seg_tid_off);
    if (c->gibbs.comp_tids) cudaFree(c->gibbs.comp_tids);
    c->gibbs = DevGibbs{};
}

int ensure_post(rsem_b200_ctx* c) {
    if (!c->post) {
        if (int rc = dev_alloc(c, &c->post, c->H)) return rc;
        if (int rc = dev_alloc(c, &c->post0, c->N)) return rc;
    }
    return 0;
}

int ensure_stats(rsem_b200_ctx* c, int n) {
    if (c->stats_cap >= n) return 0;
    if (c->d_stats) cudaFree(c->d_stats);
    RB_CUDA(cudaMalloc(&c->d_stats, sizeof(rsem_b200_round_stats) * n));
    c->stats_cap = n;
    return 0;
}

int finish_matrix_setup(rsem_b200_ctx* ctx) {
    if (int rc = dev_alloc(ctx, &ctx->sid_abs, (size_t)ctx->H)) return rc;
    if (int rc = em_make_abs_sid(ctx)) return rc;
    if (int rc = dev_alloc(ctx, &ctx->theta, (size_t)ctx->M + 1)) return rc;
    if (int rc = dev_alloc(ctx, &ctx->count, (size_t)ctx->M + 1)) return rc;
    RB_CUDA(cudaMemsetAsync(ctx->theta, 0, ((size_t)ctx->M + 1) * sizeof(double), ctx->stream));
    RB_CUDA(cudaMemsetAsync(ctx->count, 0, ((size_t)ctx->M + 1) * sizeof(double), ctx->stream));
    RB_CUDA(cudaMemsetAsync(ctx->done_flag, 0, sizeof(int), ctx->stream));
    ctx->k2_target = ctx->count;
    if (ctx->comm) if (int rc = p2p_setup(ctx)) return rc;   // collective: every rank uploads its shard
    return em_build_tiles(ctx);
}

// collect event timings recorded by em_launch_estep (after a stream sync)
void harvest_events(rsem_b200_ctx* ctx) {
    for (size_t i = 0; i < ctx->ev_used; ++i) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ctx->ev_pool[i].first, ctx->ev_pool[i].second) == cudaSuccess) {
            ctx->estep_ms += ms;
            ctx->estep_launches++;
        }
    }
    if (ctx->ev_used > 1 && getenv("RSEM_B200_TIMING_GAPS")) {  // time between consecutive K2 launches (K4, allreduce, launch gaps)
        double gap = 0.0;
        for (size_t i = 0; i + 1 < ctx->ev_used; ++i) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ctx->ev_pool[i].second, ctx->ev_pool[i + 1].first) == cudaSuccess) gap += ms;
        }
        fprintf(stderr, "rsem_b200: mean time between K2 launches %.4f ms over %zu gaps\n", gap / (double)(ctx->ev_used - 1),
                ctx->ev_used - 1);
    }
    ctx->ev_used = 0;
}

int check_err_flag(rsem_b200_ctx* ctx) {
    int e = 0;
    RB_CUDA(cudaMemcpyAsync(&e, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (e) {
        RB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
        if (e == 4) {
            set_error("a peer GPU never reported its counts of the round (count reduction over NVLink peer memory): a rank has failed");
            return RSEM_B200_ERR_NCCL;
        }
        set_error(e == 2 ? "an alignment lies outside its transcript (the reference aborts here: general_assert in "
                           "getConPrb, e.g. SingleQModel.h:116-121); the aligner may have reported different read "
                           "lengths for the same read"
                         : "sum of expected counts < 1e-300 (reference: assert(sum >= EPSILON), EM.cpp:397)");
        return RSEM_B200_ERR_ARG;
    }
    return 0;
}

}  // namespace
}  // namespace rsem_b200

using namespace rsem_b200;

extern "C" {

int rsem_b200_version(void) { return RSEM_B200_VERSION; }

const char* rsem_b200_last_error(void) { return g_last_error.c_str(); }

int rsem_b200_device_count(int* n) {
    RB_ARG(n, "n_devices is NULL");
    *n = 0;
    RB_CUDA(cudaGetDeviceCount(n));
    return 0;
}

int rsem_b200_ctx_create(int device, rsem_b200_ctx** out) {
    RB_ARG(out, "out is NULL");
    int n = 0;
    RB_CUDA(cudaGetDeviceCount(&n));
    if (n <= 0) {
        set_error("no CUDA device available (librsem_b200 has no CPU fallback)");
        return RSEM_B200_ERR_CUDA;
    }
    RB_ARG(device >= 0 && device < n, "device index out of range");
    RB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    RB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        char buf[256];
        snprintf(buf, sizeof buf, "device %d is sm_%d%d; librsem_b200 contains sm_90a code only", device, prop.major,
                 prop.minor);
        set_error(buf);
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    rsem_b200_ctx* c = new rsem_b200_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    RB_CUDA(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    RB_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    c->stream = c->own_stream;
    RB_CUDA(cudaMalloc(&c->done_flag, sizeof(int)));
    RB_CUDA(cudaMalloc(&c->err_flag, sizeof(int)));
    RB_CUDA(cudaMemset(c->done_flag, 0, sizeof(int)));
    RB_CUDA(cudaMemset(c->err_flag, 0, sizeof(int)));
    if (getenv("RSEM_B200_PHASE_TIMING")) {
        c->phase_timing = true;
        for (auto& e : c->ph_ev) RB_CUDA(cudaEventCreate(&e));
    }
    *out = c;
    return 0;
}

int rsem_b200_ctx_destroy(rsem_b200_ctx* c) {
    if (!c) return 0;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    p2p_release(c);
    if (c->comm) nccl_comm_destroy(c->comm);
    if (c->phase_timing) {
        static const char* names[3] = {"K1 conprb_kernel", "K2 E-step with posteriors", "K3 model statistics"};
        for (int i = 0; i < 3; ++i)
            if (c->ph_n[i])
                fprintf(stderr, "rsem_b200 phase timing: %-28s %9.3f ms per launch over %llu launches (device %d)\n", names[i],
                        c->ph_ms[i] / (double)c->ph_n[i], (unsigned long long)c->ph_n[i], c->device);
        for (auto& e : c->ph_ev) cudaEventDestroy(e);
    }
    free_hits(c);
    free_reads(c);
    free_refs(c);
    free_gibbs(c);
    sim_free(c);
    ci_free(c);
    gbam_free(c);
    wig_free(c);
    if (c->model_buf) cudaFree(c->model_buf);
    if (c->stats_buf) cudaFree(c->stats_buf);
    if (c->d_stats) cudaFree(c->d_stats);
    cudaFree(c->done_flag);
    cudaFree(c->err_flag);
    for (auto& e : c->ev_pool) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    block_cache_flush(c);
    cudaStreamDestroy(c->copy_stream);
    cudaStreamDestroy(c->own_stream);
    delete c;
    return 0;
}

int rsem_b200_ctx_set_stream(rsem_b200_ctx* c, void* s) {
    RB_ARG(c, "ctx is NULL");
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    c->stream = s ? static_cast<cudaStream_t>(s) : c->own_stream;
    return 0;
}

int rsem_b200_ctx_sync(rsem_b200_ctx* c) {
    RB_ARG(c, "ctx is NULL");
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    harvest_events(c);
    return 0;
}

int rsem_b200_ctx_device_bytes(rsem_b200_ctx* c, uint64_t* bytes) {
    RB_ARG(c && bytes, "NULL argument");
    *bytes = c->dev_bytes;
    return 0;
}

int rsem_b200_comm_unique_id(void* id) {
    RB_ARG(id, "id is NULL");
    return nccl_unique_id(id);
}

int rsem_b200_comm_init(rsem_b200_ctx* c, const void* id, int n_ranks, int rank) {
    RB_ARG(c && id, "NULL argument");
    RB_ARG(n_ranks >= 1 && rank >= 0 && rank < n_ranks, "bad rank / n_ranks");
    RB_CUDA(cudaSetDevice(c->device));
    p2p_release(c);
    if (c->comm) { nccl_comm_destroy(c->comm); c->comm = nullptr; }
    c->n_ranks = n_ranks;
    c->rank = rank;
    if (n_ranks == 1) return 0;
    return nccl_comm_init(&c->comm, id, n_ranks, rank);
}

int rsem_b200_shard_reads(uint64_t N, const uint64_t* row_ptr, int32_t n_shards, uint64_t* bounds) {
    RB_ARG(row_ptr && bounds, "NULL argument");
    RB_ARG(n_shards >= 1, "n_shards must be >= 1");
    // EM.cpp:135-157: worker i takes reads until it holds >= nHits / nThreads hits, while one read is left for every
    // later worker; the last worker takes the rest.  More shards than reads: the surplus shards stay empty (the
    // reference clamps nThreads to N1 instead, EM.cpp:640).
    const uint64_t world = std::min<uint64_t>((uint64_t)n_shards, std::max<uint64_t>(N, 1));
    const uint64_t thr = row_ptr[N] / world;
    uint64_t cur = 0;
    bounds[0] = 0;
    for (uint64_t i = 0; i < world; ++i) {
        uint64_t end = N;
        if (i != world - 1) {
            const uint64_t left = world - i - 1, target = row_ptr[cur] + thr;
            end = (uint64_t)(std::lower_bound(row_ptr, row_ptr + N + 1, target) - row_ptr);
            if (end < cur) end = cur;
            if (end > N - left) end = N - left;
        }
        bounds[i + 1] = end;
        cur = end;
    }
    for (uint64_t i = world; i < (uint64_t)n_shards; ++i) bounds[i + 1] = N;
    return 0;
}

int rsem_b200_upload_hits(rsem_b200_ctx* c, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr,
                          const int32_t* sid, const int32_t* pos, const int32_t* insertL) {
    RB_ARG(c && row_ptr && (sid || H == 0), "NULL argument");
    RB_ARG(M >= 1, "M must be >= 1");
    RB_ARG(row_ptr[0] == 0 && row_ptr[N] == H, "row_ptr must start at 0 and end at H");
    RB_CUDA(cudaSetDevice(c->device));
    free_hits(c);
    c->M = M;
    if (int rc = upload(c, &c->row_ptr, row_ptr, (size_t)N + 1)) return rc;
    c->N = N;
    c->H = H;
    if (int rc = upload(c, &c->sid, sid, (size_t)H)) return rc;
    if (pos) if (int rc = upload(c, &c->pos, pos, (size_t)H)) return rc;
    if (insertL) if (int rc = upload(c, &c->insertL, insertL, (size_t)H)) return rc;
    if (int rc = dev_alloc(c, &c->conprb, (size_t)H)) return rc;
    if (int rc = dev_alloc(c, &c->ncpv, (size_t)N)) return rc;
    RB_CUDA(cudaMemsetAsync(c->conprb, 0, H * sizeof(double), c->stream));
    RB_CUDA(cudaMemsetAsync(c->ncpv, 0, N * sizeof(double), c->stream));
    if (int rc = finish_matrix_setup(c)) return rc;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_upload_conprb(rsem_b200_ctx* c, const double* conprb, const double* ncpv) {
    RB_ARG(c && (conprb || c->H == 0) && (ncpv || c->N == 0), "NULL argument");
    RB_ARG(c->row_ptr, "upload_hits must be called first");
    RB_CUDA(cudaSetDevice(c->device));
    // The copies (8 bytes per hit: the bulk of a job's PCIe traffic) go to the copy stream; while they are in flight the
    // directory of the equivalence-class layout - which depends on row_ptr / sid only - is built on the compute stream.
    RB_CUDA(cudaStreamSynchronize(c->stream));   // whatever still reads or clears conprb / ncpv
    RB_CUDA(cudaMemcpyAsync(c->conprb, conprb, c->H * sizeof(double), cudaMemcpyHostToDevice, c->copy_stream));
    RB_CUDA(cudaMemcpyAsync(c->ncpv, ncpv, c->N * sizeof(double), cudaMemcpyHostToDevice, c->copy_stream));
    int rc = em_prepare_frozen_layout(c);
    const cudaError_t e = cudaStreamSynchronize(c->copy_stream);
    if (rc) return rc;
    RB_CUDA(e);
    RB_CUDA(cudaStreamSynchronize(c->stream));
    c->conprb_valid = true;
    c->conprb_epoch++;
    return 0;
}

int rsem_b200_download_conprb(rsem_b200_ctx* c, double* conprb, double* ncpv) {
    RB_ARG(c && c->row_ptr, "no hit matrix");
    RB_CUDA(cudaSetDevice(c->device));
    if (conprb) RB_CUDA(cudaMemcpyAsync(conprb, c->conprb, c->H * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (ncpv) RB_CUDA(cudaMemcpyAsync(ncpv, c->ncpv, c->N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_adopt_device_matrix(rsem_b200_ctx* c, uint64_t N, uint64_t H, int32_t M, const uint64_t* d_row_ptr,
                                  const int32_t* d_sid, const double* d_conprb, const double* d_ncpv) {
    RB_ARG(c && d_row_ptr && d_sid && d_conprb && d_ncpv, "NULL argument");
    RB_ARG(M >= 1, "M must be >= 1");
    RB_CUDA(cudaSetDevice(c->device));
    free_hits(c);
    c->M = M;
    if (int rc = dev_alloc(c, &c->row_ptr, (size_t)N + 1)) return rc;
    c->N = N;
    c->H = H;
    if (int rc = dev_alloc(c, &c->sid, (size_t)H)) return rc;
    if (int rc = dev_alloc(c, &c->conprb, (size_t)H)) return rc;
    if (int rc = dev_alloc(c, &c->ncpv, (size_t)N)) return rc;
    RB_CUDA(cudaMemcpyAsync(c->row_ptr, d_row_ptr, (N + 1) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->sid, d_sid, H * sizeof(int32_t), cudaMemcpyDeviceToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->conprb, d_conprb, H * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->ncpv, d_ncpv, N * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    if (int rc = finish_matrix_setup(c)) return rc;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    c->conprb_valid = true;
    c->conprb_epoch++;
    return 0;
}

int rsem_b200_upload_reads(rsem_b200_ctx* c, int32_t n_mates, const uint64_t* off1, const uint8_t* base1,
                           const uint8_t* qual1, const uint64_t* off2, const uint8_t* base2, const uint8_t* qual2,
                           const uint8_t* low_quality) {
    RB_ARG(c && off1 && base1 && low_quality, "NULL argument");
    RB_ARG(n_mates == 1 || (n_mates == 2 && off2 && base2), "n_mates must be 1 or 2 (with mate-2 arrays)");
    RB_ARG(c->row_ptr, "upload_hits must be called first (defines N)");
    RB_ARG((qual1 != nullptr) == (n_mates == 1 || qual2 != nullptr) || n_mates == 1, "qualities must be given for both mates or none");
    RB_CUDA(cudaSetDevice(c->device));
    free_reads(c);
    const uint64_t N = c->N;
    const uint64_t* offs[2] = {off1, off2};
    const uint8_t* bases[2] = {base1, base2};
    const uint8_t* quals[2] = {qual1, qual2};
    int max_len = 0;
    for (int m = 0; m < n_mates; ++m) {
        const uint64_t total = offs[m][N];
        for (uint64_t i = 0; i < N; ++i) max_len = std::max<int>(max_len, (int)(offs[m][i + 1] - offs[m][i]));
        c->reads.total_bases[m] = total;
        RB_CUDA(cudaMalloc(&c->reads.off[m], (N + 1) * sizeof(uint64_t)));
        RB_CUDA(cudaMalloc(&c->reads.base[m], total + 16));
        RB_CUDA(cudaMemcpyAsync(c->reads.off[m], offs[m], (N + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
        RB_CUDA(cudaMemcpyAsync(c->reads.base[m], bases[m], total, cudaMemcpyHostToDevice, c->stream));
        if (quals[m]) {
            RB_CUDA(cudaMalloc(&c->reads.qual[m], total + 16));
            RB_CUDA(cudaMemcpyAsync(c->reads.qual[m], quals[m], total, cudaMemcpyHostToDevice, c->stream));
        }
    }
    RB_CUDA(cudaMalloc(&c->reads.lowq, N + 16));
    RB_CUDA(cudaMemcpyAsync(c->reads.lowq, low_quality, N, cudaMemcpyHostToDevice, c->stream));
    c->reads.n_mates = n_mates;
    c->reads.has_qual = qual1 != nullptr;
    c->reads.max_len = max_len;
    c->reads.qmax = -1;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_upload_refs(rsem_b200_ctx* c, int32_t M, const uint64_t* seq_off, const uint8_t* seq,
                          const int32_t* full_len, const int32_t* tot_len, const uint64_t* mask_off,
                          const uint32_t* mask_words) {
    RB_ARG(c && seq_off && seq && full_len && tot_len && mask_off && mask_words, "NULL argument");
    RB_ARG(M >= 1, "M must be >= 1");
    RB_CUDA(cudaSetDevice(c->device));
    free_refs(c);
    const uint64_t seq_total = seq_off[M] + (uint64_t)tot_len[M];
    const uint64_t mask_total = mask_off[M] + (uint64_t)((full_len[M] - 1) / 32 + 1);
    RB_CUDA(cudaMalloc(&c->refs.seq_off, (M + 1) * sizeof(uint64_t)));
    RB_CUDA(cudaMalloc(&c->refs.seq, seq_total + 16));
    RB_CUDA(cudaMalloc(&c->refs.full_len, (M + 1) * sizeof(int32_t)));
    RB_CUDA(cudaMalloc(&c->refs.tot_len, (M + 1) * sizeof(int32_t)));
    RB_CUDA(cudaMalloc(&c->refs.mask_off, (M + 1) * sizeof(uint64_t)));
    RB_CUDA(cudaMalloc(&c->refs.mask_words, (mask_total + 4) * sizeof(uint32_t)));
    RB_CUDA(cudaMemcpyAsync(c->refs.seq_off, seq_off, (M + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->refs.seq, seq, seq_total, cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->refs.full_len, full_len, (M + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->refs.tot_len, tot_len, (M + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->refs.mask_off, mask_off, (M + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->refs.mask_words, mask_words, mask_total * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    c->refs.M = M;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_set_model(rsem_b200_ctx* c, const rsem_b200_model* m) {
    RB_ARG(c && m, "NULL argument");
    RB_ARG(m->model_type >= 0 && m->model_type <= 3, "model_type must be 0..3");
    RB_ARG(m->gld.pdf && m->gld.cdf && m->rspd_pdf && m->rspd_cdf && m->profile && m->noise_profile && m->mw,
           "model table pointer is NULL");
    RB_ARG(!m->has_mld || (m->mld.pdf && m->mld.cdf), "has_mld set but mld tables are NULL");
    RB_ARG(m->model_type < 2 || m->has_mld, "paired-end models need the mate length distribution");
    const bool hasq = m->model_type & 1;
    RB_ARG(hasq || m->pro_len > 0, "pro_len must be > 0 for no-quality models");
    RB_CUDA(cudaSetDevice(c->device));

    // pack every table into one host staging vector, one device buffer
    const size_t n_gld = (size_t)m->gld.span + 1, n_mld = m->has_mld ? (size_t)m->mld.span + 1 : 0;
    const size_t n_rspd = (size_t)m->rspd_B + 2;
    const size_t n_prof = hasq ? 2500 : (size_t)m->pro_len * 25;
    const size_t n_noise = hasq ? 500 : 5;
    const size_t n_mw = (size_t)m->M + 1;
    const size_t total = 2 * n_gld + 2 * n_mld + 2 * n_rspd + n_prof + n_noise + n_mw;
    std::vector<double> h(total);
    size_t o = 0;
    auto put = [&](const double* src, size_t n) { size_t at = o; if (n) memcpy(h.data() + o, src, n * sizeof(double)); o += n; return at; };
    const size_t o_gp = put(m->gld.pdf, n_gld), o_gc = put(m->gld.cdf, n_gld);
    const size_t o_mp = put(m->mld.pdf, n_mld), o_mc = put(m->mld.cdf, n_mld);
    const size_t o_rp = put(m->rspd_pdf, n_rspd), o_rc = put(m->rspd_cdf, n_rspd);
    const size_t o_pr = put(m->profile, n_prof), o_np = put(m->noise_profile, n_noise), o_mw = put(m->mw, n_mw);
    if (c->model_buf_doubles < total) {
        if (c->model_buf) cudaFree(c->model_buf);
        RB_CUDA(cudaMalloc(&c->model_buf, total * sizeof(double)));
        c->model_buf_doubles = total;
    }
    RB_CUDA(cudaMemcpyAsync(c->model_buf, h.data(), total * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));  // h goes out of scope
    DevModel& d = c->model;
    d.model_type = m->model_type; d.M = m->M; d.seed_len = m->seed_len; d.est_rspd = m->est_rspd;
    d.rspd_B = m->rspd_B; d.has_mld = m->has_mld; d.pro_len = m->pro_len;
    d.ori[0] = m->ori[0]; d.ori[1] = m->ori[1];
    d.gld = DevLenDist{m->gld.lb, m->gld.ub, m->gld.span, c->model_buf + o_gp, c->model_buf + o_gc};
    d.mld = DevLenDist{m->mld.lb, m->mld.ub, m->mld.span, c->model_buf + o_mp, c->model_buf + o_mc};
    d.rspd_pdf = c->model_buf + o_rp; d.rspd_cdf = c->model_buf + o_rc;
    d.profile = c->model_buf + o_pr; d.noise_profile = c->model_buf + o_np; d.mw = c->model_buf + o_mw;
    c->model_set = true;
    c->conprb_valid = false;  // Model::finish() sets needCalcConPrb = true (e.g. SingleQModel.h:335-341)
    return 0;
}

int rsem_b200_calc_conprb(rsem_b200_ctx* c) {
    RB_ARG(c, "ctx is NULL");
    RB_ARG(c->row_ptr && c->pos, "hit matrix with positions required");
    RB_ARG(c->model_set && c->reads.n_mates > 0 && c->refs.M > 0, "model, reads and refs must be uploaded first");
    RB_ARG((c->model.model_type >= 2) == (c->reads.n_mates == 2), "model type does not match the number of mates");
    RB_ARG((c->model.model_type >= 2) == (c->insertL != nullptr), "paired-end models need insertL");
    RB_ARG(((c->model.model_type & 1) != 0) == c->reads.has_qual, "model type does not match quality availability");
    RB_CUDA(cudaSetDevice(c->device));
    if (int rc = model_launch_conprb(c)) return rc;
    if (int rc = check_err_flag(c)) return rc;
    c->conprb_valid = true;
    c->conprb_epoch++;
    return 0;
}

int rsem_b200_set_theta(rsem_b200_ctx* c, const double* theta) {
    RB_ARG(c && theta && c->theta, "no hit matrix / NULL theta");
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMemcpyAsync(c->theta, theta, ((size_t)c->M + 1) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemsetAsync(c->done_flag, 0, sizeof(int), c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_get_theta(rsem_b200_ctx* c, double* theta) {
    RB_ARG(c && theta && c->theta, "no hit matrix / NULL theta");
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMemcpyAsync(theta, c->theta, ((size_t)c->M + 1) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int rsem_b200_em_rounds(rsem_b200_ctx* c, int32_t first_round, int32_t max_rounds_this_call, int32_t min_round,
                        int32_t max_round, double n0, rsem_b200_round_stats* stats_out, int32_t* rounds_run,
                        int32_t* stopped) {
    RB_ARG(c && rounds_run && stopped, "NULL argument");
    RB_ARG(c->row_ptr && c->conprb_valid, "conprb not available: upload_conprb or calc_conprb first");
    RB_ARG(max_rounds_this_call >= 0, "max_rounds_this_call < 0");
    RB_CUDA(cudaSetDevice(c->device));
    const int n = max_rounds_this_call;
    *rounds_run = 0;
    *stopped = 0;
    if (n == 0) return 0;
    if (int rc = ensure_stats(c, n)) return rc;
    RB_CUDA(cudaMemsetAsync(c->d_stats, 0xff, sizeof(rsem_b200_round_stats) * n, c->stream));  // totnum = -1 marks "not run"
    for (int r = 0; r < n; ++r) {
        if (c->p2p.on) {   // counts summed over NVLink peer memory, folded into the round's kernels (p2p.cu)
            c->k2_target = p2p_k2_target(c);
            const int rc = em_launch_estep(c, false);
            c->k2_target = c->count;
            if (rc) return rc;
            if (int rc2 = p2p_reduce(c)) return rc2;
        } else {
            if (int rc = em_launch_estep(c, false)) return rc;
            if (c->comm) if (int rc = nccl_allreduce_sum_f64(c->comm, c->count, (size_t)c->M + 1, c->stream)) return rc;
        }
        if (int rc = em_launch_theta_update(c, n0, first_round + r, min_round, max_round, r)) return rc;
    }
    std::vector<rsem_b200_round_stats> h(n);
    int done = 0;
    RB_CUDA(cudaMemcpyAsync(h.data(), c->d_stats, sizeof(rsem_b200_round_stats) * n, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaMemcpyAsync(&done, c->done_flag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    harvest_events(c);
    if (int rc = check_err_flag(c)) return rc;
    int ran = 0;
    while (ran < n && h[ran].totnum >= 0) ++ran;
    if (stats_out) memcpy(stats_out, h.data(), sizeof(rsem_b200_round_stats) * ran);
    *rounds_run = ran;
    *stopped = done;
    return 0;
}

int rsem_b200_em_model_round(rsem_b200_ctx* c, double n0, rsem_b200_model_stats* stats,
                             rsem_b200_round_stats* round_stats) {
    RB_ARG(c && stats && round_stats, "NULL argument");
    RB_ARG(c->row_ptr && c->pos && c->model_set && c->reads.n_mates > 0 && c->refs.M > 0,
           "hits (with positions), model, reads and refs must be uploaded first");
    RB_CUDA(cudaSetDevice(c->device));
    const bool pt = c->phase_timing;
    bool ran_k1 = false;
    if (pt) RB_CUDA(cudaEventRecord(c->ph_ev[0], c->stream));
    if (!c->conprb_valid) {
        if (int rc = rsem_b200_calc_conprb(c)) return rc;
        ran_k1 = true;
    }
    if (int rc = ensure_post(c)) return rc;
    if (int rc = ensure_stats(c, 1)) return rc;
    RB_CUDA(cudaMemsetAsync(c->done_flag, 0, sizeof(int), c->stream));
    if (pt) RB_CUDA(cudaEventRecord(c->ph_ev[1], c->stream));
    if (int rc = em_launch_estep(c, true)) return rc;
    if (pt) RB_CUDA(cudaEventRecord(c->ph_ev[2], c->stream));
    // K3 needs the (local) posteriors; statistics buffer layout is set up by model_launch_update
    c->stats.gld_lb = stats->gld_lb;
    c->stats.gld_span = stats->gld_span;
    if (int rc = model_launch_update(c)) return rc;
    if (pt) RB_CUDA(cudaEventRecord(c->ph_ev[3], c->stream));
    if (c->comm) {
        if (int rc = nccl_allreduce_sum_f64(c->comm, c->count, (size_t)c->M + 1, c->stream)) return rc;
        if (int rc = nccl_allreduce_sum_f64(c->comm, c->stats_buf, c->stats.total_doubles, c->stream)) return rc;
    }
    // round / min / max chosen so that the stop test never fires here (the host drives rounds 1-10)
    if (int rc = em_launch_theta_update(c, n0, 0, 1, 1 << 30, 0)) return rc;
    RB_CUDA(cudaMemcpyAsync(round_stats, c->d_stats, sizeof(rsem_b200_round_stats), cudaMemcpyDeviceToHost, c->stream));
    const bool hasq = c->model.model_type & 1;
    const size_t n_prof = hasq ? 2500 : (size_t)c->model.pro_len * 25, n_noise = hasq ? 500 : 5;
    if (stats->profile)
        RB_CUDA(cudaMemcpyAsync(stats->profile, c->stats.profile, n_prof * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (stats->noise_profile)
        RB_CUDA(cudaMemcpyAsync(stats->noise_profile, c->stats.noise_profile, n_noise * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (stats->gld_pdf && c->model.model_type >= 2)
        RB_CUDA(cudaMemcpyAsync(stats->gld_pdf, c->stats.gld_pdf, ((size_t)stats->gld_span + 1) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (stats->rspd_pdf && c->model.est_rspd)
        RB_CUDA(cudaMemcpyAsync(stats->rspd_pdf, c->stats.rspd_pdf, ((size_t)c->model.rspd_B + 2) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    harvest_events(c);
    if (pt) {
        for (int i = 0; i < 3; ++i) {
            if (i == 0 && !ran_k1) continue;
            float ms = 0;
            if (cudaEventElapsedTime(&ms, c->ph_ev[i], c->ph_ev[i + 1]) == cudaSuccess) { c->ph_ms[i] += ms; c->ph_n[i]++; }
        }
    }
    return check_err_flag(c);
}

int rsem_b200_expected_weights(rsem_b200_ctx* c, double* counts_out) {
    RB_ARG(c && counts_out, "NULL argument");
    RB_ARG(c->row_ptr && c->conprb_valid, "conprb not available");
    RB_CUDA(cudaSetDevice(c->device));
    if (int rc = ensure_post(c)) return rc;
    RB_CUDA(cudaMemsetAsync(c->done_flag, 0, sizeof(int), c->stream));
    RB_CUDA(cudaMemsetAsync(c->count, 0, ((size_t)c->M + 1) * sizeof(double), c->stream));
    if (int rc = em_launch_estep(c, true)) return rc;
    if (c->comm) if (int rc = nccl_allreduce_sum_f64(c->comm, c->count, (size_t)c->M + 1, c->stream)) return rc;
    RB_CUDA(cudaMemcpyAsync(counts_out, c->count, ((size_t)c->M + 1) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    // the posteriors replace conprb / ncpv (hit.setConPrb(fracs[id]), EM.cpp:227,234)
    RB_CUDA(cudaMemcpyAsync(c->conprb, c->post, c->H * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->ncpv, c->post0, c->N * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    RB_CUDA(cudaMemsetAsync(c->count, 0, ((size_t)c->M + 1) * sizeof(double), c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    harvest_events(c);
    // conprb / ncpv now hold posteriors, not conditional probabilities: another E-step on them would be wrong
    c->conprb_valid = false;
    c->conprb_epoch++;
    return 0;
}

int rsem_b200_gibbs_upload(rsem_b200_ctx* c, uint64_t N1, uint64_t E, int32_t M, const uint64_t* row_ptr,
                           const int32_t* sid, const double* conprb) {
    RB_ARG(c && row_ptr && (E == 0 || (sid && conprb)), "NULL argument");
    RB_ARG(row_ptr[0] == 0 && row_ptr[N1] == E, "row_ptr must start at 0 and end at E");
    RB_CUDA(cudaSetDevice(c->device));
    free_gibbs(c);
    RB_CUDA(cudaMalloc(&c->gibbs.row_ptr, (N1 + 1) * sizeof(uint64_t)));
    RB_CUDA(cudaMalloc(&c->gibbs.sid, (E + 4) * sizeof(int32_t)));
    RB_CUDA(cudaMalloc(&c->gibbs.conprb, (E + 4) * sizeof(double)));
    RB_CUDA(cudaMemcpyAsync(c->gibbs.row_ptr, row_ptr, (N1 + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->gibbs.sid, sid, E * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(c->gibbs.conprb, conprb, E * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    c->gibbs.N1 = N1;
    c->gibbs.E = E;
    c->gibbs.M = M;
    if (int rc = gibbs_prepare(c, row_ptr, sid)) return rc;
    c->gibbs.ready = true;
    return 0;
}

int rsem_b200_gibbs_upload_from(rsem_b200_ctx* dst, const rsem_b200_ctx* src) {
    RB_ARG(dst && src, "NULL argument");
    RB_ARG(dst != src, "gibbs_upload_from: source and destination are the same context");
    RB_ARG(src->gibbs.ready, "gibbs_upload_from: the source context holds no completed gibbs_upload");
    RB_CUDA(cudaSetDevice(dst->device));
    free_gibbs(dst);
    if (dst->device != src->device) {   // copies go over NVLink when dst may map src's memory, else through the host
        int can = 0;
        RB_CUDA(cudaDeviceCanAccessPeer(&can, dst->device, src->device));
        if (can) {
            const cudaError_t e = cudaDeviceEnablePeerAccess(src->device, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else RB_CUDA(e);
        }
    }
    const DevGibbs& s = src->gibbs;
    DevGibbs& d = dst->gibbs;
    d.N1 = s.N1; d.E = s.E; d.M = s.M;
    d.n_comp_tids = s.n_comp_tids; d.n_segs = s.n_segs; d.max_len = s.max_len; d.empty_row = s.empty_row;
    // same allocation sizes as gibbs_upload / gibbs_prepare; the padding past the data is never copied there either
    auto copy = [&](auto** to, const auto* from, size_t alloc, size_t n) -> int {
        if (!from) return 0;
        RB_CUDA(cudaMalloc(to, alloc * sizeof(**to)));
        if (n) RB_CUDA(cudaMemcpyPeerAsync(*to, dst->device, from, src->device, n * sizeof(**to), dst->stream));
        return 0;
    };
    int rc = 0;
    const size_t n_segs = (size_t)s.n_segs;
    if (!rc) rc = copy(&d.row_ptr, s.row_ptr, s.N1 + 1, s.N1 + 1);
    if (!rc) rc = copy(&d.sid, s.sid, s.E + 4, s.E);
    if (!rc) rc = copy(&d.conprb, s.conprb, s.E + 4, s.E);
    if (!rc) rc = copy(&d.order, s.order, s.N1, s.N1);
    if (!rc) rc = copy(&d.p_off, s.p_off, s.N1 + 1, s.N1 + 1);
    if (!rc) rc = copy(&d.p_sid, s.p_sid, s.E + 16, s.E);
    if (!rc) rc = copy(&d.p_con, s.p_con, s.E + 16, s.E);
    if (!rc) rc = copy(&d.seg_start, s.seg_start, n_segs + 1, n_segs + 1);
    if (!rc) rc = copy(&d.seg_ntr, s.seg_ntr, std::max<size_t>(n_segs, 1), n_segs);
    if (!rc) rc = copy(&d.seg_tid_off, s.seg_tid_off, n_segs + 1, n_segs + 1);
    if (!rc) rc = copy(&d.comp_tids, s.comp_tids, s.n_comp_tids, s.n_comp_tids);
    if (!rc) {
        const cudaError_t e = cudaStreamSynchronize(dst->stream);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    }
    if (rc) { free_gibbs(dst); return rc; }
    d.ready = true;
    return 0;
}

static int check_gibbs_run(const rsem_b200_ctx* c, const rsem_b200_gibbs_params* p) {
    RB_ARG(c && p, "NULL argument");
    RB_ARG(c->gibbs.row_ptr, "gibbs_upload must be called first");
    RB_ARG(p->M == c->gibbs.M, "M mismatch");
    RB_ARG(p->n_chains >= 1 && p->chain_samples && p->chain_seeds, "bad chain parameters");
    return 0;
}

int rsem_b200_gibbs_run_chains(rsem_b200_ctx* c, const rsem_b200_gibbs_params* p, int32_t* count_vectors, double* chain_acc,
                               rsem_b200_gibbs_stats* stats) {
    if (int rc = check_gibbs_run(c, p)) return rc;
    RB_ARG(count_vectors && chain_acc, "NULL argument");
    RB_CUDA(cudaSetDevice(c->device));
    return gibbs_run(c, p, count_vectors, chain_acc, stats);
}

int rsem_b200_gibbs_sum_chains(const rsem_b200_gibbs_params* p, const double* chain_acc, rsem_b200_gibbs_out* out) {
    RB_ARG(p && chain_acc && out && out->sum_c && out->sum_c2 && out->sum_tpm && out->sum_fpkm &&
               (p->n_genes == 0 || out->sum_gene_c2), "NULL argument");
    RB_ARG(p->M >= 0 && p->n_genes >= 0 && p->n_chains >= 0, "bad sizes");
    const size_t M1 = (size_t)p->M + 1, acc_per = 4 * M1 + (size_t)p->n_genes;
    for (size_t i = 0; i < M1; ++i) out->sum_c[i] = out->sum_c2[i] = out->sum_tpm[i] = out->sum_fpkm[i] = 0.0;
    for (int gi = 0; gi < p->n_genes; ++gi) out->sum_gene_c2[gi] = 0.0;
    for (int t = 0; t < p->n_chains; ++t) {   // Gibbs.cpp:372-397: chain 0 first
        const double* b = chain_acc + (size_t)t * acc_per;
        for (size_t i = 0; i < M1; ++i) {
            out->sum_c[i] += b[i];
            out->sum_c2[i] += b[M1 + i];
            out->sum_tpm[i] += b[2 * M1 + i];
            out->sum_fpkm[i] += b[3 * M1 + i];
        }
        for (int gi = 0; gi < p->n_genes; ++gi) out->sum_gene_c2[gi] += b[4 * M1 + gi];
    }
    return 0;
}

int rsem_b200_gibbs_split_chains(int32_t n_chains, const int32_t* chain_samples, int32_t burnin, int32_t gap, int32_t n_parts,
                                 int32_t* bounds) {
    RB_ARG(bounds && (n_chains == 0 || chain_samples), "NULL argument");
    RB_ARG(n_chains >= 0 && n_parts >= 1 && burnin >= 0 && gap >= 1, "bad arguments");
    std::vector<int64_t> prefix((size_t)n_chains + 1, 0);   // sweeps of chains [0, t)
    for (int t = 0; t < n_chains; ++t) {
        RB_ARG(chain_samples[t] >= 1, "every chain keeps at least one sample");
        prefix[t + 1] = prefix[t] + burnin + 1 + (int64_t)(chain_samples[t] - 1) * gap;
    }
    const int used = std::min(n_parts, std::max(n_chains, 1));
    bounds[0] = 0;
    for (int i = 1; i < used; ++i) {
        // nearest to i / used of the total: |used prefix[t] - i total| smallest, the lower t on a tie
        const int lo = bounds[i - 1] + 1, hi = n_chains - (used - i);
        int best = lo;
        for (int t = lo + 1; t <= hi; ++t)
            if (std::llabs(used * prefix[t] - i * prefix[n_chains]) < std::llabs(used * prefix[best] - i * prefix[n_chains])) best = t;
        bounds[i] = best;
    }
    for (int i = used; i <= n_parts; ++i) bounds[i] = n_chains;
    return 0;
}

int rsem_b200_gibbs_run(rsem_b200_ctx* c, const rsem_b200_gibbs_params* p, rsem_b200_gibbs_out* out) {
    RB_ARG(out, "NULL argument");
    if (int rc = check_gibbs_run(c, p)) return rc;
    std::vector<double> acc((size_t)p->n_chains * (4 * ((size_t)p->M + 1) + (size_t)std::max(p->n_genes, 0)));
    if (int rc = rsem_b200_gibbs_run_chains(c, p, out->count_vectors, acc.data(), nullptr)) return rc;
    return rsem_b200_gibbs_sum_chains(p, acc.data(), out);
}

int rsem_b200_gibbs_batch_create(rsem_b200_ctx* c, uint64_t capacity_bytes, int32_t worker_ctas, rsem_b200_gibbs_batch** out) {
    RB_ARG(c && out, "NULL argument");
    return gibbs_batch_create(c, capacity_bytes, worker_ctas, out);
}

int rsem_b200_gibbs_batch_destroy(rsem_b200_gibbs_batch* b) {
    if (b) gibbs_batch_destroy(b);
    return 0;
}

int rsem_b200_gibbs_batch_sample_bytes(uint64_t N1, uint64_t E, int32_t M, int32_t n_genes, int32_t n_samples,
                                       int32_t n_chains, uint64_t* bytes) {
    RB_ARG(bytes, "NULL argument");
    RB_ARG(M >= 0 && n_genes >= 0 && n_samples >= 1 && n_chains >= 1, "bad sizes");
    return gibbs_batch_sample_bytes(N1, E, M, n_genes, n_samples, n_chains, bytes);
}

int rsem_b200_gibbs_batch_add(rsem_b200_gibbs_batch* b, uint64_t N1, uint64_t E, const uint64_t* row_ptr, const int32_t* sid,
                              const double* conprb, const rsem_b200_gibbs_params* p, int32_t* slot) {
    RB_ARG(b && p && slot && row_ptr && (E == 0 || (sid && conprb)), "NULL argument");
    RB_ARG(row_ptr[0] == 0 && row_ptr[N1] == E, "row_ptr must start at 0 and end at E");
    RB_ARG(p->M >= 0 && p->n_genes >= 0 && p->burnin >= 0 && p->gap >= 1, "bad parameters");
    RB_ARG(p->n_chains >= 1 && p->chain_samples && p->chain_seeds && p->init_counts && p->pseudo_counts && p->eel && p->mw &&
               p->gene_start, "bad chain parameters");
    return gibbs_batch_add(b, N1, E, row_ptr, sid, conprb, p, slot);
}

int rsem_b200_gibbs_batch_run(rsem_b200_gibbs_batch* b, rsem_b200_gibbs_batch_stats* stats) {
    RB_ARG(b, "NULL argument");
    return gibbs_batch_run(b, stats);
}

int rsem_b200_gibbs_batch_result(rsem_b200_gibbs_batch* b, int32_t slot, int32_t* count_vectors, double* chain_acc) {
    RB_ARG(b && count_vectors && chain_acc, "NULL argument");
    return gibbs_batch_result(b, slot, count_vectors, chain_acc);
}

int rsem_b200_gibbs_batch_clear(rsem_b200_gibbs_batch* b) {
    RB_ARG(b, "NULL argument");
    gibbs_batch_clear(b);
    return 0;
}

int rsem_b200_sim_begin(rsem_b200_ctx* c, const rsem_b200_sim_params* p) {
    RB_ARG(c && p, "NULL argument");
    RB_ARG(p->model_type >= 0 && p->model_type <= 3 && p->M >= 1, "bad model type or M");
    RB_ARG(p->theta_cdf && p->gld.cdf && p->profile_cdf && p->noise_cdf && p->seq_off && p->seq && p->tot_len &&
               p->full_len, "NULL table");
    RB_ARG(p->gld.span == p->gld.ub - p->gld.lb && p->gld.span >= 1, "bad gld");
    RB_ARG(p->model_type < 2 || p->has_mld, "paired-end models need mld");
    RB_ARG(!p->has_mld || (p->mld.cdf && p->mld.span == p->mld.ub - p->mld.lb && p->mld.span >= 1), "bad mld");
    RB_ARG(!p->est_rspd || (p->rspd_off && p->rspd_cdf), "estRSPD needs rspd_off / rspd_cdf");
    RB_ARG(!(p->model_type & 1) || (p->qd_init_cdf && p->qd_tran_cdf && p->pro_rows == 100), "Q models need QualDist");
    RB_CUDA(cudaSetDevice(c->device));
    return sim_begin(c, p);
}

int rsem_b200_sim_next(rsem_b200_ctx* c, const char* text[2], uint64_t bytes[2], uint64_t* n_reads) {
    RB_ARG(c && text && bytes && n_reads, "NULL argument");
    RB_CUDA(cudaSetDevice(c->device));
    return sim_next(c, text, bytes, n_reads);
}

int rsem_b200_sim_end(rsem_b200_ctx* c, double* counts, uint64_t* resim, rsem_b200_sim_stats* stats) {
    RB_ARG(c, "NULL argument");
    RB_CUDA(cudaSetDevice(c->device));
    return sim_end(c, counts, resim, stats);
}

int rsem_b200_ci_begin(rsem_b200_ctx* c, const rsem_b200_ci_params* p) {
    RB_ARG(c && p, "NULL argument");
    RB_ARG(p->M >= 1 && p->n_genes >= 1 && p->n_samples >= 1 && p->n_parts >= 1, "bad M, gene count, sample count or parts");
    RB_ARG(p->gene_start && p->part_gene_start && (p->n_isoforms == 0 || p->isoform_start), "NULL group array");
    RB_ARG(p->gene_start[0] == 1 && p->gene_start[p->n_genes] == p->M + 1, "gene_start must cover transcripts 1..M");
    for (int32_t g = 0; g < p->n_genes; ++g) RB_ARG(p->gene_start[g] < p->gene_start[g + 1], "empty gene");
    RB_ARG(p->part_gene_start[0] == 0 && p->part_gene_start[p->n_parts] == p->n_genes, "parts must cover the genes");
    for (int32_t i = 0; i < p->n_parts; ++i) RB_ARG(p->part_gene_start[i] <= p->part_gene_start[i + 1], "parts out of order");
    if (p->n_isoforms) {
        RB_ARG(p->isoform_start[0] == 1 && p->isoform_start[p->n_isoforms] == p->M + 1, "isoform_start must cover 1..M");
        for (int32_t i = 0; i < p->n_isoforms; ++i) RB_ARG(p->isoform_start[i] < p->isoform_start[i + 1], "empty isoform");
    }
    RB_ARG(p->n_samples <= INT32_MAX, "too many samples");
    RB_CUDA(cudaSetDevice(c->device));
    return ci_begin(c, p);
}

int rsem_b200_ci_push(rsem_b200_ctx* c, const float* rows, const float* l_bars, int64_t first, int64_t count) {
    RB_ARG(c && (count == 0 || (rows && l_bars)), "NULL argument");
    RB_CUDA(cudaSetDevice(c->device));
    return ci_push(c, rows, l_bars, first, count);
}

int rsem_b200_ci_end(rsem_b200_ctx* c, float* transcripts, float* genes, float* isoforms, rsem_b200_ci_stats* stats) {
    RB_ARG(c && transcripts && genes, "NULL argument");
    RB_ARG(c->ci, "ci_begin must be called first");
    RB_CUDA(cudaSetDevice(c->device));
    return ci_end(c, transcripts, genes, isoforms, stats);
}

int rsem_b200_kmer_shared(rsem_b200_ctx* c, const rsem_b200_kmer_params* p, uint64_t* shared_counts,
                          rsem_b200_kmer_stats* stats) {
    RB_ARG(c && p && p->offsets && (shared_counts || p->n_transcripts == 0), "NULL argument");
    RB_ARG(p->k >= 1, "k must be >= 1");
    RB_ARG(p->fingerprint_bits >= 0 && p->fingerprint_bits <= 24, "fingerprint_bits must be 0..24");
    RB_ARG(p->offsets[0] == 0, "offsets[0] must be 0");
    for (uint64_t t = 0; t < p->n_transcripts; ++t) RB_ARG(p->offsets[t] <= p->offsets[t + 1], "offsets must not decrease");
    RB_ARG(p->bases || p->offsets[p->n_transcripts] == 0, "NULL bases");
    RB_ARG(p->n_transcripts < 0xffffffffull, "too many transcripts");
    RB_CUDA(cudaSetDevice(c->device));
    return kmer_shared(c, p, shared_counts, stats);
}

int rsem_b200_gbam_convert(rsem_b200_ctx* c, const rsem_b200_gbam_tables* t, const rsem_b200_gbam_batch* b, uint8_t* out,
                           uint64_t out_cap, uint64_t* out_bytes, rsem_b200_gbam_stats* stats) {
    RB_ARG(c && t && b && out_bytes && (out || out_cap == 0), "NULL argument");
    RB_ARG(t->M >= 1 && t->out_tid && t->minus && t->length && t->exon_off && t->mapq_prb, "NULL or empty transcript table");
    RB_ARG(t->exon_off[0] == 0 && (t->exon_off[t->M + 1] == 0 || (t->exon_start && t->exon_end)), "bad exon table");
    RB_ARG(b->n_units == 0 || (b->data && b->rec_off && b->unit_rec && b->unit_group && b->unit_tr), "NULL batch array");
    RB_ARG(b->n_units < 0xffffffffull && b->n_records < 0xffffffffull, "batch too large");
    RB_ARG(b->n_units == 0 || (b->unit_rec[0] == 0 && b->unit_rec[b->n_units] == b->n_records), "unit_rec must cover the records");
    RB_CUDA(cudaSetDevice(c->device));
    return gbam_convert(c, t, b, out, out_cap, out_bytes, stats);
}

int rsem_b200_wig_depth(rsem_b200_ctx* c, const rsem_b200_wig_batch* b, double* out, uint64_t out_cap, uint64_t* out_len,
                        rsem_b200_wig_stats* stats) {
    if (stats) *stats = rsem_b200_wig_stats{0.0, 0, 0, -1, 0, 0};   // bad_record -1 on every other failure
    RB_ARG(c && b && out_len && (out || out_cap == 0), "NULL argument");
    RB_ARG(b->n_records == 0 || (b->data && b->rec_off && b->rec_run), "NULL batch array");
    RB_ARG(b->n_runs == 0 || b->run_len, "NULL run_len");
    RB_ARG(b->n_records == 0 || b->n_runs > 0, "records without runs");
    RB_ARG(b->n_records < 0xffffffffull, "batch too large");
    RB_CUDA(cudaSetDevice(c->device));
    return wig_depth(c, b, out, out_cap, out_len, stats);
}

int rsem_b200_batch_create(rsem_b200_ctx* c, uint64_t capacity_bytes, rsem_b200_batch** out) {
    RB_ARG(c && out, "NULL argument");
    return batch_create(c, capacity_bytes, out);
}

int rsem_b200_batch_destroy(rsem_b200_batch* b) {
    if (b) batch_destroy(b);
    return 0;
}

int rsem_b200_batch_sample_bytes(uint64_t N, uint64_t H, const uint64_t* row_ptr, int32_t m, uint64_t* bytes) {
    RB_ARG(row_ptr && bytes, "NULL argument");
    RB_ARG(m >= 0 && row_ptr[0] == 0 && row_ptr[N] == H, "row_ptr must start at 0 and end at H, m >= 0");
    return batch_sample_bytes(N, H, row_ptr, m, bytes);
}

int rsem_b200_batch_add(rsem_b200_batch* b, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr,
                        const int32_t* sid, const double* conprb, const double* ncpv, const double* theta, double n0,
                        int32_t first_round, int32_t min_round, int32_t max_round, int32_t* slot) {
    RB_ARG(b && row_ptr && (sid || H == 0) && (conprb || H == 0) && (ncpv || N == 0) && theta && slot, "NULL argument");
    RB_ARG(M >= 1 && N >= 1, "M and N must be >= 1");
    RB_ARG(row_ptr[0] == 0 && row_ptr[N] == H, "row_ptr must start at 0 and end at H");
    for (uint64_t i = 0; i < N; ++i) RB_ARG(row_ptr[i] <= row_ptr[i + 1], "row_ptr must not decrease");
    RB_ARG(first_round >= 2, "the batch starts after round 1 (first_round >= 2)");
    return batch_add(b, N, H, M, row_ptr, sid, conprb, ncpv, theta, n0, first_round, min_round, max_round, slot);
}

int rsem_b200_batch_run(rsem_b200_batch* b, int32_t max_rounds, rsem_b200_round_stats* stats, int32_t* rounds_run,
                        int32_t* stopped) {
    RB_ARG(b && rounds_run && stopped, "NULL argument");
    RB_ARG(max_rounds >= 0, "max_rounds < 0");
    return batch_run(b, max_rounds, stats, rounds_run, stopped);
}

int rsem_b200_batch_slots(rsem_b200_batch* b, int32_t* n_slots) {
    RB_ARG(b && n_slots, "NULL argument");
    *n_slots = batch_slots(b);
    return 0;
}

int rsem_b200_batch_final(rsem_b200_batch* b, int32_t slot, double* theta, double* counts, double* post, double* post0) {
    RB_ARG(b, "NULL argument");
    RB_ARG(batch_slot_live(b, slot), "no sample in this slot");
    return batch_final(b, slot, theta, counts, post, post0);
}

int rsem_b200_batch_remove(rsem_b200_batch* b, int32_t slot) {
    RB_ARG(b, "NULL argument");
    RB_ARG(batch_slot_live(b, slot), "no sample in this slot");
    batch_remove(b, slot);
    return 0;
}

int rsem_b200_batch_timing(rsem_b200_batch* b, double* total_ms, uint64_t* sample_rounds) {
    RB_ARG(b && total_ms && sample_rounds, "NULL argument");
    return batch_timing(b, total_ms, sample_rounds);
}

int rsem_b200_launch_count(rsem_b200_ctx* c, uint64_t* launches) {
    RB_ARG(c && launches, "NULL argument");
    *launches = c->launches;
    return 0;
}

int rsem_b200_estep_timing(rsem_b200_ctx* c, double* total_ms, uint64_t* launches, int32_t reset) {
    RB_ARG(c, "ctx is NULL");
    if (total_ms) *total_ms = c->estep_ms;
    if (launches) *launches = c->estep_launches;
    if (reset) { c->estep_ms = 0; c->estep_launches = 0; }
    return 0;
}

int rsem_b200_set_profiling(rsem_b200_ctx* c, int32_t enabled) {
    RB_ARG(c, "ctx is NULL");
    c->profiling = enabled != 0;
    return 0;
}

int rsem_b200_class_layout_info(rsem_b200_ctx* c, uint64_t* out) {
    RB_ARG(c && out, "NULL argument");
    const ClassLayout& L = c->cls;
    out[0] = L.built ? 1 : 0;
    out[1] = L.n_rows;
    out[2] = L.n_long;
    out[3] = L.n_segs;
    out[4] = L.n_batches;
    out[5] = L.n_tiles;
    out[6] = L.n_vals;
    out[7] = L.n_ids;
    out[8] = L.n_tiles_main;
    out[9] = L.n_run_hits;
    return 0;
}

int rsem_b200_estep_cta_times(rsem_b200_ctx* c, uint64_t* out_ns, int32_t cap, int32_t* n) {
    RB_ARG(c && out_ns && n, "NULL argument");
    *n = 0;
    const ClassLayout& L = c->cls;
    if (!L.cta_ns || L.last_grid == 0) return 0;
    RB_CUDA(cudaSetDevice(c->device));
    const int k = std::min<int>(cap, (int)L.last_grid);
    RB_CUDA(cudaMemcpyAsync(out_ns, L.cta_ns, (size_t)k * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    *n = k;
    return 0;
}

int rsem_b200_estep_wait_times(rsem_b200_ctx* c, uint64_t* out_ns, int32_t cap, int32_t* n) {
    RB_ARG(c && out_ns && n, "NULL argument");
    *n = 0;
    const ClassLayout& L = c->cls;
    if (!L.wait_ns || !L.last_profiled || L.last_grid == 0) return 0;
    RB_CUDA(cudaSetDevice(c->device));
    const int k = std::min<int>(cap, (int)L.last_grid);
    RB_CUDA(cudaMemcpyAsync(out_ns, L.wait_ns, (size_t)k * kWaitRecord * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    *n = k;
    return 0;
}

int rsem_b200_set_estep_variant(rsem_b200_ctx* c, int32_t v) {
    RB_ARG(c && (v == 0 || v == 2 || v == 4 || v == 5),
           "variant must be 0 (auto), 2 (direct), 4 (row groups on staged tiles) or 5 (class layout)");
    c->variant = v;
    return 0;
}

}  // extern "C"
