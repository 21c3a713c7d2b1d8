// K12: frozen-conprb EM rounds (EM.cpp:199-244 E_STEP + EM.cpp:385-416 M-step and stop test) for many samples at once.
//
// A sample's rounds from 11 on touch only the transcripts its hits name: every M-step sets theta_i = count_i / sum, so
// after round 1 theta_i is exactly 0 for a transcript without a hit (EM.cpp:394-398), the probv >= 1e-7 test
// (EM.cpp:406-413) leaves it out of bChange / totNum, and it stays 0.  batch_add therefore maps the sample's distinct
// transcript ids to 1..m (the noise entry stays 0), checks that theta is exactly 0 outside that set, and keeps the
// sample's matrix in that compact space.  batch_final scatters theta and the counts back to M + 1 entries.
//
// Layout per sample (one device block): compact ids i32 and conprb f64 per hit, row offsets u32 and ncpv f64 per read,
// theta and count f64 per compact transcript, tile bounds (rows, hits) u32.  Tiles hold at most kHitCap hits and
// kRowCap rows, so that a tile plus the lead-ins of its 16-byte aligned copies fits a Stage.
//
// Kernel: persistent CTAs of kThreads threads.  A CTA claims a sample from a device counter (the host orders the
// samples largest first), copies its theta into shared memory and runs up to `rounds` rounds back to back with no
// grid-wide synchronisation: the sample's tiles stream through a kStages-deep ring filled by 1-D bulk copies (tma.cuh),
// and because the staged data (ids, conprb, rows) do not change between rounds, the ring runs ahead across round
// boundaries.  The E-step gathers theta from shared memory and adds the normalised weights to the sample's count
// vector with red.global.add.f64 (L2-resident; a shared-memory fp64 atomic is a CAS loop on sm_90a); the noise entry is
// kept in registers.  The M-step reads the counts back through L2, writes theta to shared memory, zeroes the counts and
// records (sum, bChange, totNum) of the round.  Then the CTA claims the next sample.
#include <algorithm>
#include <cstring>

#include "common.cuh"
#include "tma.cuh"

namespace rsem_b200 {

namespace {

constexpr int kThreads = 512;
constexpr int kStages = 2;
constexpr unsigned kHitCap = 2048;
constexpr unsigned kRowCap = 512;
constexpr int kThetaCap = 12288;           // compact transcripts (incl. noise) whose theta fits shared memory
constexpr uint64_t kMaxHits = 1ull << 20;  // larger samples converge faster on the whole-GPU path (em_rounds)

struct __align__(16) Stage {
    double con[kHitCap + 4];
    double ncp[kRowCap + 4];
    int sid[kHitCap + 8];
    unsigned rp[kRowCap + 8];
};
static_assert(sizeof(Stage) % 16 == 0, "stage must keep 16 B alignment");

struct BatchSmem {
    Stage stage[kStages];
    unsigned long long bar[kStages];
    double red_d[kThreads / 32];
    long long red_l[kThreads / 32];
    int idx;
    int stop;
};
constexpr size_t kThetaOffset = (sizeof(BatchSmem) + 15) & ~size_t(15);

}  // namespace

// one sample as the kernel sees it; `round`, `done` and `err` are written back by the kernel
struct BatchDesc {
    const int* sid;
    const double* con;
    const unsigned* rp;
    const double* ncp;
    const unsigned* tile_row;
    const unsigned* tile_hit;
    double* theta;
    double* count;
    double* post;
    double* post0;
    rsem_b200_round_stats* stats;
    double n0;
    unsigned N, H, m1, n_tiles;
    int G;
    int round, min_round, max_round;
    int done, err;
};

}  // namespace rsem_b200

struct rsem_b200_batch {
    rsem_b200_ctx* ctx = nullptr;
    uint64_t capacity = 0, used = 0;
    struct Slot {
        bool live = false;
        void* block = nullptr;
        uint64_t bytes = 0;
        int32_t M = 0;
        std::vector<int32_t> ids;   // compact id -> transcript id (ids[0] = 0)
        rsem_b200::BatchDesc d{};
    };
    std::vector<Slot> slots;
    rsem_b200::BatchDesc* d_desc = nullptr;
    size_t desc_cap = 0;
    rsem_b200_round_stats* d_stats = nullptr;
    size_t stats_cap = 0;
    unsigned* d_claim = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    double k12_ms = 0.0;
    uint64_t k12_rounds = 0;
};

namespace rsem_b200 {

namespace {

template <int G>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void issue_tile(const BatchDesc& d, unsigned k, Stage& st, unsigned long long* bar) {
    const unsigned rs = d.tile_row[k], re = d.tile_row[k + 1];
    const unsigned hs = d.tile_hit[k], he = d.tile_hit[k + 1];
    const unsigned hs4 = hs & ~3u, hs2 = hs & ~1u, rs4 = rs & ~3u, rs2 = rs & ~1u;
    const unsigned b_sid = round16((he - hs4) * 4u);
    const unsigned b_con = round16((he - hs2) * 8u);
    const unsigned b_rp = round16((re + 1 - rs4) * 4u);
    const unsigned b_nc = round16((re - rs2) * 8u);
    fence_proxy_async();   // the generic-proxy reads of this stage (before the caller's barrier) precede the copy
    mbar_expect_tx(bar, b_sid + b_con + b_rp + b_nc);
    if (b_sid) bulk_load(st.sid, d.sid + hs4, b_sid, bar);
    if (b_con) bulk_load(st.con, d.con + hs2, b_con, bar);
    bulk_load(st.rp, d.rp + rs4, b_rp, bar);
    if (b_nc) bulk_load(st.ncp, d.ncp + rs2, b_nc, bar);
}

// The rows of one staged tile: G lanes per row, rows spread over the warps.  Returns the lane's share of count[0].
template <int G, bool POST>
__device__ __forceinline__ double tile_rows(const BatchDesc& d, unsigned k, const Stage& st, const double* th, double th0) {
    const unsigned rs = d.tile_row[k], re = d.tile_row[k + 1], hs = d.tile_hit[k];
    const unsigned nr = re - rs;
    const unsigned* rp = st.rp + (rs & 3u);
    const double* ncp = st.ncp + (rs & 1u);
    const int* sid = st.sid + (hs & 3u);   // sid[j - hs], con[j - hs] for the sample's hit j
    const double* con = st.con + (hs & 1u);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned g = lane % G;
    double acc0 = 0.0;
    for (unsigned base = (unsigned)warp * (32 / G); base < nr; base += (kThreads / 32) * (32 / G)) {
        const unsigned r = base + lane / G;
        const bool valid = r < nr;
        unsigned hb = 0, he = 0;
        if (valid) { hb = rp[r]; he = rp[r + 1]; }
        double part = 0.0, f0 = 0.0;
        for (unsigned j = hb + g; j < he; j += G) {
            double f = th[sid[j - hs]] * con[j - hs];
            if (f < kEpsilon) f = 0.0;
            part += f;
        }
        if (valid && g == 0) {
            f0 = th0 * ncp[r];
            if (f0 < kEpsilon) f0 = 0.0;
            part += f0;
        }
        const double sum = group_sum<G>(part);
        if (!valid) continue;
        const double inv = sum >= kEpsilon ? 1.0 / sum : 0.0;   // a row whose sum < 1e-300 contributes nothing
        if (g == 0) {
            acc0 += f0 * inv;
            if (POST) d.post0[rs + r] = f0 * inv;
        }
        for (unsigned j = hb + g; j < he; j += G) {
            const int t = sid[j - hs];
            double f = th[t] * con[j - hs];
            if (f < kEpsilon) f = 0.0;
            const double w = f * inv;
            if (w != 0.0) red_add_f64(d.count + t, w);
            if (POST) d.post[j] = w;
        }
    }
    return acc0;
}

template <bool POST>
__device__ __forceinline__ double tile_dispatch(const BatchDesc& d, unsigned k, const Stage& st, const double* th, double th0) {
    switch (d.G) {
        case 1: return tile_rows<1, POST>(d, k, st, th, th0);
        case 2: return tile_rows<2, POST>(d, k, st, th, th0);
        case 4: return tile_rows<4, POST>(d, k, st, th, th0);
        case 8: return tile_rows<8, POST>(d, k, st, th, th0);
        case 16: return tile_rows<16, POST>(d, k, st, th, th0);
        default: return tile_rows<32, POST>(d, k, st, th, th0);
    }
}

__device__ __forceinline__ double block_sum(double v, BatchSmem& sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) sm.red_d[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += sm.red_d[w];   // same order in every thread
    return s;
}

// mode 0: up to `rounds` frozen rounds per sample; mode 1: the final pass (counts + posteriors, theta unchanged)
template <bool FINAL>
__global__ void __launch_bounds__(kThreads, 1) k12_kernel(BatchDesc* descs, int n, unsigned* claim, int rounds) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BatchSmem& sm = *reinterpret_cast<BatchSmem*>(smem_raw);
    double* th = reinterpret_cast<double*>(smem_raw + kThetaOffset);
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&sm.bar[s], 1);
        fence_barrier_init();
    }
    unsigned issued = 0, consumed = 0;   // tiles through the ring over the CTA's lifetime (same in every thread)
    for (;;) {
        __syncthreads();
        if (tid == 0) sm.idx = (int)atomicAdd(claim, 1u);
        __syncthreads();
        const int idx = sm.idx;
        if (idx >= n) break;
        BatchDesc& dd = descs[idx];
        const BatchDesc d = dd;
        if (d.done || d.n_tiles == 0) continue;
        for (unsigned i = tid; i < d.m1; i += kThreads) th[i] = d.theta[i];
        // the sample's tile stream: q = round * n_tiles + tile, run ahead by kStages
        const unsigned long long Q = (unsigned long long)(FINAL ? 1 : rounds) * d.n_tiles;
        unsigned long long q_issue = 0;
#define K12_ISSUE_NEXT()                                                                                              \
    if (q_issue < Q) {                                                                                                \
        if (tid == 0) issue_tile(d, (unsigned)(q_issue % d.n_tiles), sm.stage[issued % kStages], &sm.bar[issued % kStages]); \
        ++q_issue;                                                                                                    \
        ++issued;                                                                                                     \
    }
        for (int s = 0; s < kStages; ++s) { K12_ISSUE_NEXT() }
        __syncthreads();
        int round = d.round, done = 0, err = 0;
        const int n_rounds = FINAL ? 1 : rounds;
        for (int r = 0; r < n_rounds && !done; ++r) {
            const double th0 = th[0];
            double acc0 = 0.0;
            for (unsigned k = 0; k < d.n_tiles; ++k) {
                const int s = consumed % kStages;
                mbar_wait(&sm.bar[s], (consumed / kStages) & 1u);
                acc0 += tile_dispatch<FINAL>(d, k, sm.stage[s], th, th0);
                ++consumed;
                __syncthreads();   // every thread is done with stage s
                K12_ISSUE_NEXT()
            }
            __threadfence();   // this thread's red.global adds are performed before the counts are read back
            const double c0 = block_sum(acc0, sm);
            if (FINAL) {
                if (tid == 0) d.count[0] = c0;
                break;
            }
            // M-step (EM.cpp:391-398) and the convergence statistics (EM.cpp:406-413)
            double part = 0.0;
            for (unsigned i = 1 + tid; i < d.m1; i += kThreads) part += __ldcg(d.count + i);
            const double sum = block_sum(part, sm) + c0 + d.n0;
            ++round;
            if (!(sum >= kEpsilon)) {   // reference: assert(sum >= EPSILON), EM.cpp:397
                err = 1;
                done = 1;
                break;
            }
            double bmax = 0.0;
            long long tot = 0;
            for (unsigned i = tid; i < d.m1; i += kThreads) {
                const double c = i == 0 ? c0 + d.n0 : __ldcg(d.count + i);
                const double tn = c / sum;
                const double old = th[i];
                if (old >= 1e-7) {
                    const double change = fabs(tn - old) / old;
                    if (change >= 0.001) ++tot;
                    if (bmax < change) bmax = change;
                }
                th[i] = tn;
                if (i > 0) __stcg(d.count + i, 0.0);
            }
            const int lane = tid & 31, warp = tid >> 5;
            for (int o = 16; o > 0; o >>= 1) {
                bmax = fmax(bmax, __shfl_xor_sync(0xffffffffu, bmax, o));
                tot += __shfl_xor_sync(0xffffffffu, tot, o);
            }
            __syncthreads();
            if (lane == 0) { sm.red_d[warp] = bmax; sm.red_l[warp] = tot; }
            __syncthreads();
            if (tid == 0) {
                double b = 0.0;
                long long t = 0;
                for (int w = 0; w < kThreads / 32; ++w) { b = fmax(b, sm.red_d[w]); t += sm.red_l[w]; }
                d.stats[r] = rsem_b200_round_stats{sum, b, (int64_t)t};
                // the reference's loop runs while ROUND < MIN_ROUND || (totNum > 0 && ROUND < MAX_ROUND) (EM.cpp:416)
                sm.stop = !(round < d.min_round || (t > 0 && round < d.max_round));
            }
            __syncthreads();
            done = sm.stop;
        }
        // drain the copies that ran ahead past the last round
        while (consumed < issued) {
            mbar_wait(&sm.bar[consumed % kStages], (consumed / kStages) & 1u);
            ++consumed;
        }
        __syncthreads();
        if (!FINAL) {
            for (unsigned i = tid; i < d.m1; i += kThreads) d.theta[i] = th[i];
            if (tid == 0) { dd.round = round; dd.done = done; dd.err = err; }
        }
    }
#undef K12_ISSUE_NEXT
}

int lanes_per_row(uint64_t N, uint64_t H) {   // kRowSlots-free version of em_build_tiles' rule
    const double mean_deg = (double)H / (double)std::max<uint64_t>(N, 1) + 1.0;
    return mean_deg <= 3.0 ? 1 : mean_deg <= 6.0 ? 2 : mean_deg <= 12.0 ? 4 : mean_deg <= 24.0 ? 8 : mean_deg <= 48.0 ? 16 : 32;
}

inline uint64_t al(uint64_t b) { return (b + 255) & ~uint64_t(255); }

struct Parts { uint64_t sid, con, rp, ncp, theta, count, trow, thit, total; };

Parts layout(uint64_t N, uint64_t H, uint64_t m1, uint64_t n_tiles) {
    Parts p{};
    uint64_t o = 0;
    p.sid = o; o += al(H * 4 + 64);
    p.con = o; o += al(H * 8 + 64);
    p.rp = o; o += al((N + 1) * 4 + 64);
    p.ncp = o; o += al(N * 8 + 64);
    p.theta = o; o += al(m1 * 8);
    p.count = o; o += al(m1 * 8);
    p.trow = o; o += al((n_tiles + 1) * 4);
    p.thit = o; o += al((n_tiles + 1) * 4);
    p.total = o;
    return p;
}

// tiles over the rows: at most kHitCap hits and kRowCap rows each; false when a row alone exceeds kHitCap
bool cut_tiles(uint64_t N, const uint64_t* row_ptr, std::vector<unsigned>& trow, std::vector<unsigned>& thit) {
    trow.assign(1, 0);
    thit.assign(1, 0);
    uint64_t r0 = 0;
    for (uint64_t r = 0; r < N; ++r) {
        const uint64_t d = row_ptr[r + 1] - row_ptr[r];
        if (d > kHitCap) return false;
        if (r - r0 + 1 > kRowCap || row_ptr[r + 1] - row_ptr[r0] > kHitCap) {
            trow.push_back((unsigned)r);
            thit.push_back((unsigned)row_ptr[r]);
            r0 = r;
        }
    }
    trow.push_back((unsigned)N);
    thit.push_back((unsigned)row_ptr[N]);
    return true;
}

int ensure_buffers(rsem_b200_batch* b, size_t n_desc, size_t n_stats) {
    if (b->desc_cap < n_desc) {
        if (b->d_desc) cudaFree(b->d_desc);
        RB_CUDA(cudaMalloc(&b->d_desc, n_desc * sizeof(BatchDesc)));
        b->desc_cap = n_desc;
    }
    if (b->stats_cap < n_stats) {
        if (b->d_stats) cudaFree(b->d_stats);
        RB_CUDA(cudaMalloc(&b->d_stats, n_stats * sizeof(rsem_b200_round_stats)));
        b->stats_cap = n_stats;
    }
    return 0;
}

template <bool FINAL>
int launch(rsem_b200_batch* b, const std::vector<BatchDesc>& descs, int rounds) {
    rsem_b200_ctx* c = b->ctx;
    unsigned max_m1 = 1;
    for (const auto& d : descs) max_m1 = std::max(max_m1, d.m1);
    const size_t smem = kThetaOffset + (size_t)max_m1 * sizeof(double);
    auto kern = k12_kernel<FINAL>;
    RB_CUDA(raise_dyn_smem((const void*)kern, smem));
    int per_sm = 0;
    RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
    const int grid = std::max(1, std::min<int>((int)descs.size(), std::max(per_sm, 1) * c->sm_count));
    RB_CUDA(cudaMemcpyAsync(b->d_desc, descs.data(), descs.size() * sizeof(BatchDesc), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemsetAsync(b->d_claim, 0, sizeof(unsigned), c->stream));
    RB_CUDA(cudaEventRecord(b->ev[0], c->stream));
    kern<<<grid, kThreads, smem, c->stream>>>(b->d_desc, (int)descs.size(), b->d_claim, rounds);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(cudaEventRecord(b->ev[1], c->stream));
    c->launches++;
    return 0;
}

}  // namespace

int batch_create(rsem_b200_ctx* c, uint64_t capacity, rsem_b200_batch** out) {
    RB_CUDA(cudaSetDevice(c->device));
    if (capacity == 0) {   // half of the device memory that is free now
        size_t free_b = 0, total_b = 0;
        RB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        capacity = free_b / 2;
    }
    auto* b = new rsem_b200_batch();
    b->ctx = c;
    b->capacity = capacity;
    cudaError_t e = cudaMalloc(&b->d_claim, sizeof(unsigned));
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev[0]);
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev[1]);
    if (e != cudaSuccess) {
        batch_destroy(b);
        return cuda_fail(e, "batch_create", __FILE__, __LINE__);
    }
    *out = b;
    return 0;
}

void batch_remove(rsem_b200_batch* b, int slot) {
    auto& s = b->slots[slot];
    if (!s.live) return;
    cudaFreeAsync(s.block, b->ctx->stream);
    b->used -= s.bytes;
    s = rsem_b200_batch::Slot{};
}

void batch_destroy(rsem_b200_batch* b) {
    cudaSetDevice(b->ctx->device);
    for (size_t i = 0; i < b->slots.size(); ++i) batch_remove(b, (int)i);
    cudaStreamSynchronize(b->ctx->stream);
    if (b->d_desc) cudaFree(b->d_desc);
    if (b->d_stats) cudaFree(b->d_stats);
    if (b->d_claim) cudaFree(b->d_claim);
    for (auto& e : b->ev) if (e) cudaEventDestroy(e);
    delete b;
}

int batch_sample_bytes(uint64_t N, uint64_t H, const uint64_t* row_ptr, int32_t m, uint64_t* bytes) {
    if (H > kMaxHits || m + 1 > kThetaCap) {
        set_error("the sample is outside the batch layout (more than 2^20 hits or 12287 distinct transcripts): "
                  "run it with rsem_b200_em_rounds");
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    std::vector<unsigned> trow, thit;
    if (!cut_tiles(N, row_ptr, trow, thit)) {
        set_error("the sample has a read with more than 2048 alignments, outside the batch layout: run it with rsem_b200_em_rounds");
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    *bytes = layout(N, H, (uint64_t)m + 1, trow.size() - 1).total;
    return 0;
}

int batch_add(rsem_b200_batch* b, uint64_t N, uint64_t H, int32_t M, const uint64_t* row_ptr, const int32_t* sid,
              const double* conprb, const double* ncpv, const double* theta, double n0, int32_t first_round,
              int32_t min_round, int32_t max_round, int32_t* slot_out) {
    rsem_b200_ctx* c = b->ctx;
    // the compact id space: distinct |sid| in increasing order
    std::vector<char> seen((size_t)M + 1, 0);
    for (uint64_t h = 0; h < H; ++h) {
        const int32_t t = std::abs(sid[h]);
        if (t < 1 || t > M) { set_error("a hit names a transcript outside 1..M"); return RSEM_B200_ERR_ARG; }
        seen[t] = 1;
    }
    std::vector<int32_t> ids(1, 0), to_compact((size_t)M + 1, 0);
    for (int32_t t = 1; t <= M; ++t)
        if (seen[t]) { to_compact[t] = (int32_t)ids.size(); ids.push_back(t); }
        else if (theta[t] != 0.0) {   // the condition the compaction rests on
            set_error("theta is not 0 for a transcript without hits: the batch starts after round 1 (EM.cpp:394-398)");
            return RSEM_B200_ERR_ARG;
        }
    const int32_t m = (int32_t)ids.size() - 1;
    uint64_t bytes = 0;
    if (int rc = batch_sample_bytes(N, H, row_ptr, m, &bytes)) return rc;
    if (b->used + bytes > b->capacity) {
        set_error("the batch arena is full");
        return RSEM_B200_ERR_FULL;
    }
    std::vector<unsigned> trow, thit;
    cut_tiles(N, row_ptr, trow, thit);
    const uint64_t n_tiles = trow.size() - 1;
    const Parts p = layout(N, H, (uint64_t)m + 1, n_tiles);
    // host image of the block, one copy
    std::vector<unsigned char> img(p.total, 0);
    int32_t* csid = reinterpret_cast<int32_t*>(img.data() + p.sid);
    for (uint64_t h = 0; h < H; ++h) csid[h] = to_compact[std::abs(sid[h])];
    if (H) memcpy(img.data() + p.con, conprb, H * 8);
    unsigned* rp = reinterpret_cast<unsigned*>(img.data() + p.rp);
    for (uint64_t i = 0; i <= N; ++i) rp[i] = (unsigned)row_ptr[i];
    if (N) memcpy(img.data() + p.ncp, ncpv, N * 8);
    double* th = reinterpret_cast<double*>(img.data() + p.theta);
    for (int32_t k = 0; k <= m; ++k) th[k] = theta[ids[k]];
    memcpy(img.data() + p.trow, trow.data(), trow.size() * 4);
    memcpy(img.data() + p.thit, thit.data(), thit.size() * 4);
    RB_CUDA(cudaSetDevice(c->device));
    void* block = nullptr;
    RB_CUDA(cudaMallocAsync(&block, p.total, c->stream));
    RB_CUDA(cudaMemcpyAsync(block, img.data(), p.total, cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));   // img goes out of scope

    int slot = -1;
    for (size_t i = 0; i < b->slots.size(); ++i) if (!b->slots[i].live) { slot = (int)i; break; }
    if (slot < 0) { slot = (int)b->slots.size(); b->slots.emplace_back(); }
    auto& s = b->slots[slot];
    s.live = true;
    s.block = block;
    s.bytes = bytes;
    s.M = M;
    s.ids = std::move(ids);
    unsigned char* base = static_cast<unsigned char*>(block);
    BatchDesc& d = s.d;
    d = BatchDesc{};
    d.sid = reinterpret_cast<const int*>(base + p.sid);
    d.con = reinterpret_cast<const double*>(base + p.con);
    d.rp = reinterpret_cast<const unsigned*>(base + p.rp);
    d.ncp = reinterpret_cast<const double*>(base + p.ncp);
    d.tile_row = reinterpret_cast<const unsigned*>(base + p.trow);
    d.tile_hit = reinterpret_cast<const unsigned*>(base + p.thit);
    d.theta = reinterpret_cast<double*>(base + p.theta);
    d.count = reinterpret_cast<double*>(base + p.count);
    d.n0 = n0;
    d.N = (unsigned)N;
    d.H = (unsigned)H;
    d.m1 = (unsigned)m + 1;
    d.n_tiles = (unsigned)n_tiles;
    d.G = lanes_per_row(N, H);
    d.round = first_round - 1;
    d.min_round = min_round;
    d.max_round = max_round;
    b->used += bytes;
    *slot_out = slot;
    return 0;
}

int batch_run(rsem_b200_batch* b, int32_t rounds, rsem_b200_round_stats* stats, int32_t* rounds_run, int32_t* stopped) {
    rsem_b200_ctx* c = b->ctx;
    const size_t n_slots = b->slots.size();
    std::fill(rounds_run, rounds_run + n_slots, 0);
    std::fill(stopped, stopped + n_slots, 0);
    std::vector<int> order;
    for (size_t i = 0; i < n_slots; ++i) {
        const auto& s = b->slots[i];
        if (s.live) stopped[i] = s.d.done;
        if (s.live && !s.d.done) order.push_back((int)i);
    }
    if (order.empty() || rounds <= 0) return 0;
    // largest first: the longest rounds start first and the small samples fill in behind them
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
        return (uint64_t)b->slots[x].d.H + b->slots[x].d.N > (uint64_t)b->slots[y].d.H + b->slots[y].d.N;
    });
    RB_CUDA(cudaSetDevice(c->device));
    if (int rc = ensure_buffers(b, order.size(), order.size() * (size_t)rounds)) return rc;
    std::vector<BatchDesc> descs;
    for (size_t k = 0; k < order.size(); ++k) {
        BatchDesc d = b->slots[order[k]].d;
        d.stats = b->d_stats + k * (size_t)rounds;
        descs.push_back(d);
    }
    if (int rc = launch<false>(b, descs, rounds)) return rc;
    std::vector<rsem_b200_round_stats> h(order.size() * (size_t)rounds);
    RB_CUDA(cudaMemcpyAsync(descs.data(), b->d_desc, descs.size() * sizeof(BatchDesc), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaMemcpyAsync(h.data(), b->d_stats, h.size() * sizeof(rsem_b200_round_stats), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    float ms = 0;
    if (cudaEventElapsedTime(&ms, b->ev[0], b->ev[1]) == cudaSuccess) b->k12_ms += ms;
    int err = 0;
    for (size_t k = 0; k < order.size(); ++k) {
        auto& s = b->slots[order[k]];
        const int ran = descs[k].round - s.d.round;
        b->k12_rounds += (uint64_t)std::max(ran, 0);
        if (stats)
            for (int r = 0; r < ran; ++r) stats[(size_t)order[k] * rounds + r] = h[k * (size_t)rounds + r];
        rounds_run[order[k]] = ran;
        stopped[order[k]] = descs[k].done;
        s.d.round = descs[k].round;
        s.d.done = descs[k].done;
        s.d.err = descs[k].err;
        if (descs[k].err) err = 1;
    }
    if (err) {
        set_error("sum of expected counts < 1e-300 (reference: assert(sum >= EPSILON), EM.cpp:397)");
        return RSEM_B200_ERR_ARG;
    }
    return 0;
}

int batch_final(rsem_b200_batch* b, int32_t slot, double* theta, double* counts, double* post, double* post0) {
    rsem_b200_ctx* c = b->ctx;
    auto& s = b->slots[slot];
    BatchDesc d = s.d;
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMallocAsync(&d.post, (size_t)d.H * 8 + 8, c->stream));   // the final mode always writes posteriors
    RB_CUDA(cudaMallocAsync(&d.post0, (size_t)d.N * 8 + 8, c->stream));
    d.done = 0;
    if (int rc = ensure_buffers(b, 1, 1)) return rc;
    d.stats = b->d_stats;
    std::vector<BatchDesc> descs{d};
    if (int rc = launch<true>(b, descs, 1)) return rc;
    std::vector<double> th(d.m1), cnt(d.m1);
    RB_CUDA(cudaMemcpyAsync(th.data(), d.theta, d.m1 * 8, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaMemcpyAsync(cnt.data(), d.count, d.m1 * 8, cudaMemcpyDeviceToHost, c->stream));
    if (post) RB_CUDA(cudaMemcpyAsync(post, d.post, (size_t)d.H * 8, cudaMemcpyDeviceToHost, c->stream));
    if (post0) RB_CUDA(cudaMemcpyAsync(post0, d.post0, (size_t)d.N * 8, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaMemsetAsync(d.count, 0, d.m1 * 8, c->stream));
    RB_CUDA(cudaFreeAsync(d.post, c->stream));
    RB_CUDA(cudaFreeAsync(d.post0, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (theta) {
        std::fill(theta, theta + s.M + 1, 0.0);
        for (unsigned k = 0; k < d.m1; ++k) theta[s.ids[k]] = th[k];
    }
    if (counts) {
        std::fill(counts, counts + s.M + 1, 0.0);
        for (unsigned k = 0; k < d.m1; ++k) counts[s.ids[k]] = cnt[k];
    }
    return 0;
}

int batch_slots(const rsem_b200_batch* b) { return (int)b->slots.size(); }
bool batch_slot_live(const rsem_b200_batch* b, int slot) { return slot >= 0 && slot < (int)b->slots.size() && b->slots[slot].live; }

int batch_timing(const rsem_b200_batch* b, double* ms, uint64_t* sample_rounds) {
    *ms = b->k12_ms;
    *sample_rounds = b->k12_rounds;
    return 0;
}

}  // namespace rsem_b200
