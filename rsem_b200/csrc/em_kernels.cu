// E-step / M-step kernels for frozen conditional probabilities (K2) and the theta update +
// convergence test (K4).
//
// What they compute is the reference's E_STEP inner loops (EM.cpp:199-244) and the M-step +
// relative-change statistics (EM.cpp:385-416).  How they compute it is specific to sm_90a:
//
//   * the hit matrix is SoA CSR in HBM (row_ptr u64, sid i32, conprb f64, ncpv f64); one pass
//     streams 12 B per hit + 16 B per read, nothing else comes from HBM (theta / count live in L2);
//   * estep_rows_kernel: rows are cut into byte-balanced tiles once per upload; one persistent CTA of 1024 threads
//     per SM walks a contiguous range of tiles through a 3-stage shared-memory ring filled by 1-D bulk-async copies
//     (TMA, cp.async.bulk + mbarrier complete_tx), so the bytes in flight per SM are set by the ring depth, not by
//     occupancy or by the dependent row_ptr -> hits -> theta load chain.  Warps claim batches of rows from a
//     shared-memory counter, G lanes own a row with its products in registers, row sums by xor-shuffles, normalised
//     weights go to the count vector with red.global.add.f64 (L2-resident); no CTA-wide barrier per tile, the warp
//     that finishes a tile last refills its stage.  The noise entry count[0] - which every row touches - is
//     privatised in a register and flushed once per CTA;
//   * estep_direct_kernel: the same row logic with loads straight from global memory.  It runs when the matrix has
//     no tiles (an empty row, or a row longer than a stage holds) and on request (variant 2);
//   * the M-step is one 8-CTA thread-block cluster exchanging partial sums through distributed shared memory.
//
// Clamp semantics are the reference's: a term < 1e-300 is 0, a row whose sum < 1e-300
// contributes nothing (EM.cpp:212,219,223).
#include <cooperative_groups.h>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/unique.h>

#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "tma.cuh"

namespace rsem_b200 {

namespace {

// ------------------------------------------------------------------------------------------------
// geometry of the TMA-staged row kernel: one CTA of kThreads threads per SM, tiles of <= kHitCap hits and
// <= kRowCap rows (em_build_tiles), kStages of them in flight
// ------------------------------------------------------------------------------------------------
constexpr int kStages = 3;
constexpr int kThreads = 1024;
constexpr int kHitCap = 4 * kThreads;
constexpr int kRowCap = kThreads;
constexpr int kRowUnroll = 2;  // row batches a warp works on at once (instruction-level parallelism)
constexpr int kRowSlots = 4;   // hits of a row a lane keeps in registers

// A stage holds a tile plus the lead-in of its 16-byte aligned copies.
struct __align__(16) Stage {
    double con[kHitCap + 4];
    unsigned long long rp[kRowCap + 4];
    double ncp[kRowCap + 4];
    int sid[kHitCap + 8];
};

struct TileDesc {  // written by the thread that issues the tile, read by everyone after the wait
    unsigned long long rs, hs;
    unsigned nr;
};

struct RowSmem {
    Stage stage[kStages];
    unsigned long long full_bar[kStages];
    TileDesc desc[kStages];
    unsigned int next_batch[kStages];
    unsigned int warps_done[kStages];
    double red[kThreads / 32];
};
static_assert(sizeof(Stage) % 16 == 0, "stage must keep 16 B alignment");
static_assert(sizeof(RowSmem) <= 227 * 1024, "shared memory per SM");

struct EstepArgs {
    const unsigned long long* row_ptr;
    const int* sid;
    const double* conprb;
    const double* ncpv;
    const double* theta;
    double* count;
    double* post;
    double* post0;
    const unsigned long long* tile_row;
    const unsigned long long* tile_hit;
    unsigned int n_tiles;
    unsigned long long N;
    const int* done_flag;
};

template <int G>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <>
__device__ __forceinline__ double group_sum<1>(double v) { return v; }

// One row handled by the G lanes of a group.  sp/cp point at the row's first hit (shared or
// global memory), `d` is its degree, `g` the lane's index inside the group.
// Returns the lane's contribution to count[0] (non-zero on g == 0 only).
template <int G, bool WRITE_POST>
__device__ __forceinline__ double process_row(bool valid, int g, unsigned d, const int* sp, const double* cp, double nc,
                                              const double* __restrict__ theta, double theta0, double* count,
                                              double* post_row, double* post0_row) {
    double fa = 0.0, fb = 0.0, part = 0.0, f0 = 0.0;
    int ta = 0, tb = 0;
    if (valid) {
        if (g < d) {
            ta = abs(sp[g]);
            fa = __ldg(theta + ta) * cp[g];
            if (fa < kEpsilon) fa = 0.0;
        }
        if (g + G < d) {
            tb = abs(sp[g + G]);
            fb = __ldg(theta + tb) * cp[g + G];
            if (fb < kEpsilon) fb = 0.0;
        }
        part = fa + fb;
        for (unsigned j = g + 2 * G; j < d; j += G) {
            double f = __ldg(theta + abs(sp[j])) * cp[j];
            if (f < kEpsilon) f = 0.0;
            part += f;
        }
        if (g == 0) {
            f0 = theta0 * nc;
            if (f0 < kEpsilon) f0 = 0.0;
            part += f0;
        }
    }
    const double sum = group_sum<G>(part);
    double acc0 = 0.0;
    if (!valid) return 0.0;
    if (sum >= kEpsilon) {
        const double inv = 1.0 / sum;
        if (g == 0) {
            acc0 = f0 * inv;
            if (WRITE_POST) *post0_row = acc0;
        }
        if (g < d) {
            const double w = fa * inv;
            if (fa != 0.0) red_add_f64(count + ta, w);
            if (WRITE_POST) post_row[g] = w;
        }
        if (g + G < d) {
            const double w = fb * inv;
            if (fb != 0.0) red_add_f64(count + tb, w);
            if (WRITE_POST) post_row[g + G] = w;
        }
        for (unsigned j = g + 2 * G; j < d; j += G) {
            const int t = abs(sp[j]);
            double f = __ldg(theta + t) * cp[j];
            if (f < kEpsilon) f = 0.0;
            const double w = f * inv;
            if (f != 0.0) red_add_f64(count + t, w);
            if (WRITE_POST) post_row[j] = w;
        }
    } else if (WRITE_POST) {
        if (g == 0) *post0_row = 0.0;
        for (unsigned j = g; j < d; j += G) post_row[j] = 0.0;
    }
    return acc0;
}

// flush the per-thread count[0] partials: warp shuffle -> shared -> one red per CTA
__device__ __forceinline__ void flush_count0(double acc0, double* red_smem, double* count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red_smem[warp] = acc0;
    __syncthreads();
    if (warp == 0) {
        double v = lane < (blockDim.x >> 5) ? red_smem[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && v != 0.0) red_add_f64(count, v);
    }
}

// ------------------------------------------------------------------------------------------------
// K2, row groups on TMA-staged tiles.  grid = min(#SMs, #tiles) persistent CTAs of kThreads threads, each walking a
// contiguous range of tiles through its kStages-deep ring.  A tile is consumed in ONE pass with no CTA-wide barrier:
// a warp claims batches of 32 / G rows from a shared-memory counter, G lanes own a row, lane g holds the row's hits
// g, g + G, ... (kRowSlots of them in registers): ids and conprb come from the stage (each byte of it is read once),
// theta is gathered, the row sum goes through log2(G) xor-shuffles and the normalised weights leave as
// red.global.add.f64 - a warp instruction covers 32 / G runs of G adjacent transcripts, which the L2 reduction unit
// handles as well as 32 consecutive ones.  kRowUnroll batches are in flight per warp for instruction-level
// parallelism.  The warp that finishes a tile last refills its stage.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void issue_tile(const EstepArgs& a, unsigned k, Stage& st, unsigned long long* bar,
                                           TileDesc& desc) {
    const unsigned long long rs = a.tile_row[k], re = a.tile_row[k + 1];
    const unsigned long long hs = a.tile_hit[k], he = a.tile_hit[k + 1];
    desc.rs = rs;
    desc.hs = hs;
    desc.nr = (unsigned)(re - rs);
    const unsigned long long hs4 = hs & ~3ull, hs2 = hs & ~1ull, rs2 = rs & ~1ull;
    const unsigned b_sid = round16((unsigned)(he - hs4) * 4u);
    const unsigned b_con = round16((unsigned)(he - hs2) * 8u);
    const unsigned b_rp = round16((unsigned)(re + 1 - rs2) * 8u);
    const unsigned b_nc = round16((unsigned)(re - rs2) * 8u);
    mbar_expect_tx(bar, b_sid + b_con + b_rp + b_nc);
    if (b_sid) bulk_load(st.sid, a.sid + hs4, b_sid, bar);
    if (b_con) bulk_load(st.con, a.conprb + hs2, b_con, bar);
    bulk_load(st.rp, a.row_ptr + rs2, b_rp, bar);
    bulk_load(st.ncp, a.ncpv + rs2, b_nc, bar);
}

template <int G, bool WRITE_POST>
__global__ void __launch_bounds__(kThreads, 1) estep_rows_kernel(const EstepArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RowSmem& sm = *reinterpret_cast<RowSmem*>(smem_raw);
    if (*a.done_flag) return;
    constexpr unsigned kWarps = kThreads / 32;
    constexpr unsigned kRowsPerBatch = 32 / G;

    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&sm.full_bar[s], 1);
            sm.next_batch[s] = 0;
            sm.warps_done[s] = 0;
        }
        fence_barrier_init();
    }
    __syncthreads();
    const unsigned per_cta = a.n_tiles / gridDim.x, extra = a.n_tiles % gridDim.x;  // the first `extra` CTAs take one more
    const unsigned k_first = blockIdx.x * per_cta + min(blockIdx.x, extra);
    const unsigned k_end = k_first + per_cta + (blockIdx.x < extra ? 1u : 0u);
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            const unsigned k = k_first + s;
            if (k < k_end) issue_tile(a, k, sm.stage[s], &sm.full_bar[s], sm.desc[s]);
        }
    }

    const unsigned g = lane % G;
    const unsigned row_in_batch = lane / G;
    const double theta0 = __ldg(a.theta);
    double acc0 = 0.0;

    for (unsigned it = 0; k_first + it < k_end; ++it) {
        const unsigned k = k_first + it;
        const int s = it % kStages;
        const unsigned parity = (it / kStages) & 1u;
        Stage& st = sm.stage[s];
        mbar_wait(&sm.full_bar[s], parity);

        const unsigned long long rs = sm.desc[s].rs, hs = sm.desc[s].hs;
        const unsigned nr = sm.desc[s].nr;
        const unsigned roff = (unsigned)(rs & 1ull);
        const int* s_sid = st.sid + (unsigned)(hs & 3ull);
        const double* s_con = st.con + (unsigned)(hs & 1ull);
        const unsigned n_batches = (nr + kRowsPerBatch - 1) / kRowsPerBatch;

        for (;;) {
            unsigned b0 = 0;
            if (lane == 0) b0 = atomicAdd(&sm.next_batch[s], (unsigned)kRowUnroll);
            b0 = __shfl_sync(0xffffffffu, b0, 0);
            if (b0 >= n_batches) break;

            unsigned row[kRowUnroll], hb[kRowUnroll], he[kRowUnroll];
            bool valid[kRowUnroll];
            int t[kRowUnroll][kRowSlots];
            double x[kRowUnroll][kRowSlots];
            double f0[kRowUnroll], part[kRowUnroll];
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
                row[u] = (b0 + u) * kRowsPerBatch + row_in_batch;
                valid[u] = row[u] < nr;
                hb[u] = he[u] = 0;
                if (valid[u]) {
                    hb[u] = (unsigned)(st.rp[roff + row[u]] - hs);
                    he[u] = (unsigned)(st.rp[roff + row[u] + 1] - hs);
                }
            }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u)
#pragma unroll
                for (int q = 0; q < kRowSlots; ++q) {
                    const unsigned j = hb[u] + g + q * G;
                    t[u][q] = j < he[u] ? s_sid[j] : 0;
                }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u)
#pragma unroll
                for (int q = 0; q < kRowSlots; ++q) x[u][q] = __ldg(a.theta + t[u][q]);
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
#pragma unroll
                for (int q = 0; q < kRowSlots; ++q) {
                    const unsigned j = hb[u] + g + q * G;
                    const double c = j < he[u] ? s_con[j] : 0.0;
                    x[u][q] *= c;
                    if (x[u][q] < kEpsilon) x[u][q] = 0.0;
                }
                part[u] = (x[u][0] + x[u][1]) + (x[u][2] + x[u][3]);
                for (unsigned j = hb[u] + g + kRowSlots * G; j < he[u]; j += G) {  // rows longer than kRowSlots * G
                    double f = __ldg(a.theta + s_sid[j]) * s_con[j];
                    if (f < kEpsilon) f = 0.0;
                    part[u] += f;
                }
                f0[u] = 0.0;
                if (valid[u] && g == 0) {
                    f0[u] = theta0 * st.ncp[roff + row[u]];
                    if (f0[u] < kEpsilon) f0[u] = 0.0;
                    part[u] += f0[u];
                }
            }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) part[u] = group_sum<G>(part[u]);
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
                const double inv = part[u] >= kEpsilon ? 1.0 / part[u] : 0.0;
                const double p0 = f0[u] * inv;
                acc0 += p0;
                if (WRITE_POST && valid[u] && g == 0) a.post0[rs + row[u]] = p0;
#pragma unroll
                for (int q = 0; q < kRowSlots; ++q) {
                    const unsigned j = hb[u] + g + q * G;
                    const double w = x[u][q] * inv;
                    if (w != 0.0) red_add_f64(a.count + t[u][q], w);
                    if (WRITE_POST && j < he[u]) a.post[hs + j] = w;
                }
                for (unsigned j = hb[u] + g + kRowSlots * G; j < he[u]; j += G) {
                    const int tt = s_sid[j];
                    double f = __ldg(a.theta + tt) * s_con[j];
                    if (f < kEpsilon) f = 0.0;
                    const double w = f * inv;
                    if (w != 0.0) red_add_f64(a.count + tt, w);
                    if (WRITE_POST) a.post[hs + j] = w;
                }
            }
        }
        // this warp has read everything it needs from stage s; the last warp to get here refills the stage
        __syncwarp();
        if (lane == 0) {
            const unsigned old = atomicAdd(&sm.warps_done[s], 1u);
            if (old == kWarps - 1) {
                sm.warps_done[s] = 0;
                sm.next_batch[s] = 0;
                const unsigned long long kn = (unsigned long long)k + kStages;
                if (kn < k_end) issue_tile(a, (unsigned)kn, st, &sm.full_bar[s], sm.desc[s]);
            }
        }
    }
    __syncthreads();
    flush_count0(acc0, sm.red, a.count);
}

// ------------------------------------------------------------------------------------------------
// K2, direct variant: same row logic, loads straight from global memory (no staging).  Used for
// matrices without tiles (an empty row, or a row longer than a stage holds) and for variant 2.
// ------------------------------------------------------------------------------------------------
template <int G, bool WRITE_POST>
__global__ void __launch_bounds__(256) estep_direct_kernel(const EstepArgs a) {
    __shared__ double red[8];
    if (*a.done_flag) return;
    constexpr int kGroupsPerWarp = 32 / G;
    const int lane = threadIdx.x & 31;
    const int g = lane % G;
    const int group_in_warp = lane / G;
    const unsigned long long warps_total = (unsigned long long)gridDim.x * (blockDim.x >> 5);
    const unsigned long long warp_id = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const double theta0 = __ldg(a.theta);
    double acc0 = 0.0;
    for (unsigned long long base = warp_id * kGroupsPerWarp; base < a.N; base += warps_total * kGroupsPerWarp) {
        const unsigned long long i = base + group_in_warp;
        const bool valid = i < a.N;
        unsigned long long rp0 = 0, rp1 = 0;
        double nc = 0.0;
        if (valid) {
            rp0 = a.row_ptr[i];
            rp1 = a.row_ptr[i + 1];
            nc = a.ncpv[i];
        }
        const unsigned d = (unsigned)(rp1 - rp0);
        acc0 += process_row<G, WRITE_POST>(valid, g, d, a.sid + rp0, a.conprb + rp0, nc, a.theta, theta0, a.count,
                                           WRITE_POST ? a.post + rp0 : nullptr, WRITE_POST ? a.post0 + i : nullptr);
    }
    flush_count0(acc0, red, a.count);
}

// ------------------------------------------------------------------------------------------------
// tile construction: tile k holds the rows r with  row_ptr[r] + C * r  in  [k W, (k + 1) W)
// => at most W / C + 1 rows and at most W + max_degree hits per tile.
// ------------------------------------------------------------------------------------------------
__global__ void tile_bounds_kernel(const unsigned long long* row_ptr, unsigned long long N, unsigned long long W,
                                   unsigned long long C, unsigned long long n_raw, unsigned long long* tile_row) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k > n_raw) return;
    if (k == n_raw) {
        tile_row[k] = N;
        return;
    }
    const unsigned long long target = k * W;
    unsigned long long lo = 0, hi = N;  // first r in [0, N] with row_ptr[r] + C r >= target
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (row_ptr[mid] + C * mid < target) lo = mid + 1;
        else hi = mid;
    }
    tile_row[k] = lo;
}

__global__ void max_diff_kernel(const unsigned long long* v, unsigned long long n, unsigned int* out) {
    unsigned int m = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x)
        m = max(m, (unsigned)(v[i + 1] - v[i]));
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void gather_u64_kernel(const unsigned long long* src, const unsigned long long* idx, unsigned long long n,
                                  unsigned long long* out) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = src[idx[k]];
}

__global__ void max_degree_kernel(const unsigned long long* row_ptr, unsigned long long N, unsigned int* out) {
    unsigned int m = 0, has_empty = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < N;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long d = row_ptr[i + 1] - row_ptr[i];
        m = max(m, d > 0xffffffffull ? 0xffffffffu : (unsigned)d);
        if (d == 0) has_empty = 1;
    }
    if (has_empty) out[1] = 1;
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// ------------------------------------------------------------------------------------------------
// K4: theta update + convergence statistics (EM.cpp:391-416).  The M-vector is tiny (<= 1.6 MB):
// one CTA, two passes, block reductions.
// ------------------------------------------------------------------------------------------------
constexpr int kThetaCluster = 8;  // CTAs of the M-step kernel: one thread-block cluster, partial results through DSMEM

__global__ void __cluster_dims__(kThetaCluster, 1, 1) __launch_bounds__(1024)
    theta_update_kernel(double* count, double* theta, int M1, double n0, int round, int min_round, int max_round,
                        rsem_b200_round_stats* stats_slot, int* done_flag, int* err_flag) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ double sh_d[32];
    __shared__ long long sh_l[32];
    __shared__ double cl_sum[kThetaCluster];     // every CTA receives every CTA's partial sum
    __shared__ double cl_b[kThetaCluster];       // rank 0 receives the partial statistics
    __shared__ long long cl_t[kThetaCluster];
    if (*done_flag) return;  // same value in every CTA of the cluster
    // distributed shared memory may only be written once the target CTA has started executing (racecheck: "block that
    // might not have entered yet"): every CTA of the cluster passes this barrier before the first remote store
    cluster.sync();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    const unsigned rank = cluster.block_rank();
    const int first = (int)rank * (int)blockDim.x + tid, step = kThetaCluster * (int)blockDim.x;

    double s = 0.0;
    for (int i = first; i < M1; i += step) s += count[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) sh_d[warp] = s;
    __syncthreads();
    if (warp == 0) {
        double v = lane < nwarp ? sh_d[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane < kThetaCluster) *cluster.map_shared_rank(&cl_sum[rank], lane) = v;
    }
    cluster.sync();
    double sum = n0;
    for (int r = 0; r < kThetaCluster; ++r) sum += cl_sum[r];  // same order in every CTA
    if (!(sum >= kEpsilon)) {  // reference: assert(sum >= EPSILON), EM.cpp:397
        if (rank == 0 && tid == 0) { *err_flag = 1; *done_flag = 1; }
        return;
    }

    double bmax = 0.0;
    long long tot = 0;
    for (int i = first; i < M1; i += step) {
        const double c = count[i] + (i == 0 ? n0 : 0.0);
        const double tn = c / sum;
        const double old = theta[i];
        if (old >= 1e-7) {
            const double change = fabs(tn - old) / old;
            if (change >= 0.001) ++tot;
            if (bmax < change) bmax = change;
        }
        theta[i] = tn;
        count[i] = 0.0;
    }
    for (int o = 16; o > 0; o >>= 1) {
        bmax = fmax(bmax, __shfl_xor_sync(0xffffffffu, bmax, o));
        tot += __shfl_xor_sync(0xffffffffu, tot, o);
    }
    __syncthreads();
    if (lane == 0) { sh_d[warp] = bmax; sh_l[warp] = tot; }
    __syncthreads();
    if (warp == 0) {
        double b = lane < nwarp ? sh_d[lane] : 0.0;
        long long t = lane < nwarp ? sh_l[lane] : 0;
        for (int o = 16; o > 0; o >>= 1) {
            b = fmax(b, __shfl_xor_sync(0xffffffffu, b, o));
            t += __shfl_xor_sync(0xffffffffu, t, o);
        }
        if (lane == 0) {
            *cluster.map_shared_rank(&cl_b[rank], 0) = b;
            *cluster.map_shared_rank(&cl_t[rank], 0) = t;
        }
    }
    cluster.sync();
    if (rank == 0 && tid == 0) {
        double b = 0.0;
        long long t = 0;
        for (int r = 0; r < kThetaCluster; ++r) { b = fmax(b, cl_b[r]); t += cl_t[r]; }
        stats_slot->sum = sum;
        stats_slot->bchange = b;
        stats_slot->totnum = t;
        // loop continues while ROUND < MIN_ROUND || (totNum > 0 && ROUND < MAX_ROUND)
        if (!(round < min_round || (t > 0 && round < max_round))) *done_flag = 1;
    }
}

template <int G, bool WP>
int launch_rows(rsem_b200_ctx* ctx, const EstepArgs& a) {
    auto kern = estep_rows_kernel<G, WP>;
    const size_t smem = sizeof(RowSmem);
    RB_CUDA(raise_dyn_smem((const void*)kern, smem));
    const unsigned grid = std::min<unsigned>((unsigned)ctx->sm_count, a.n_tiles);
    kern<<<grid, kThreads, smem, ctx->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

template <int G, bool WP>
int launch_direct(rsem_b200_ctx* ctx, const EstepArgs& a) {
    auto kern = estep_direct_kernel<G, WP>;
    unsigned long long rows_per_block = (256 / 32) * (32 / G);
    unsigned long long want = (a.N + rows_per_block - 1) / rows_per_block;
    unsigned grid = (unsigned)std::min<unsigned long long>(want ? want : 1, (unsigned long long)ctx->sm_count * 8);
    kern<<<grid, 256, 0, ctx->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

template <bool WP>
int launch_csr(rsem_b200_ctx* ctx, const EstepArgs& a, bool direct) {
    if (direct) {
        switch (ctx->group) {
            case 4: return launch_direct<4, WP>(ctx, a);
            case 8: return launch_direct<8, WP>(ctx, a);
            case 16: return launch_direct<16, WP>(ctx, a);
            default: return launch_direct<32, WP>(ctx, a);
        }
    }
    switch (ctx->rows_group) {
        case 1: return launch_rows<1, WP>(ctx, a);
        case 2: return launch_rows<2, WP>(ctx, a);
        case 4: return launch_rows<4, WP>(ctx, a);
        case 8: return launch_rows<8, WP>(ctx, a);
        case 16: return launch_rows<16, WP>(ctx, a);
        default: return launch_rows<32, WP>(ctx, a);
    }
}

}  // namespace

__global__ void abs_kernel(const int* in, int* out, unsigned long long n) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x)
        out[i] = abs(in[i]);
}

int em_make_abs_sid(rsem_b200_ctx* ctx) {
    if (ctx->H == 0) return 0;
    abs_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(ctx->sid, ctx->sid_abs, ctx->H);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

int em_max_degree(rsem_b200_ctx* ctx, uint32_t* max_deg) {  // max_deg[0] = longest row, max_deg[1] = 1 if some row is empty
    unsigned int* d = nullptr;
    RB_CUDA(cudaMalloc(&d, 2 * sizeof(unsigned int)));
    RB_CUDA(cudaMemsetAsync(d, 0, 2 * sizeof(unsigned int), ctx->stream));
    if (ctx->N > 0) {
        max_degree_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(
            reinterpret_cast<const unsigned long long*>(ctx->row_ptr), ctx->N, d);
        ctx->launches++;
    }
    RB_CUDA(cudaMemcpyAsync(max_deg, d, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(d);
    return 0;
}

// Cuts the rows into tiles of at most W + max_deg hits and at most row_cap rows: tile k holds the rows r with
// row_ptr[r] + C * r in [k W, (k + 1) W).  C starts at the byte-balanced weight 1 (a row costs about as much
// traffic as a hit) and doubles only for matrices whose rows are so short that row_cap would be exceeded.
static int build_tile_set(rsem_b200_ctx* ctx, unsigned long long W, unsigned row_cap, uint64_t** out_row,
                          uint64_t** out_hit, uint32_t* out_n) {
    unsigned long long C = 1, n_raw = 0;
    unsigned long long* raw = nullptr;
    for (;;) {
        const unsigned long long total = ctx->H + C * ctx->N;
        n_raw = total / W + 1;
        RB_CUDA(cudaMalloc(&raw, (n_raw + 1) * sizeof(unsigned long long)));
        tile_bounds_kernel<<<(unsigned)((n_raw + 1 + 255) / 256), 256, 0, ctx->stream>>>(
            reinterpret_cast<const unsigned long long*>(ctx->row_ptr), ctx->N, W, C, n_raw, raw);
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
        unsigned int* d_max = nullptr;
        unsigned int h_max = 0;
        RB_CUDA(cudaMalloc(&d_max, sizeof(unsigned int)));
        RB_CUDA(cudaMemsetAsync(d_max, 0, sizeof(unsigned int), ctx->stream));
        max_diff_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(raw, n_raw, d_max);
        ctx->launches++;
        RB_CUDA(cudaMemcpyAsync(&h_max, d_max, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        RB_CUDA(cudaStreamSynchronize(ctx->stream));
        cudaFree(d_max);
        if (h_max <= row_cap) break;
        cudaFree(raw);
        raw = nullptr;
        C *= 2;
    }
    ctx->tile_weight = C;
    // drop empty tiles: consecutive equal boundaries
    thrust::device_ptr<unsigned long long> p(raw);
    auto end = thrust::unique(thrust::cuda::par.on(ctx->stream), p, p + n_raw + 1);
    const unsigned long long n_bounds = (unsigned long long)(end - p);
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (n_bounds < 2) { cudaFree(raw); *out_n = 0; return 0; }
    *out_n = (uint32_t)(n_bounds - 1);
    RB_CUDA(cudaMalloc(out_row, n_bounds * sizeof(uint64_t)));
    RB_CUDA(cudaMalloc(out_hit, n_bounds * sizeof(uint64_t)));
    RB_CUDA(cudaMemcpyAsync(*out_row, raw, n_bounds * sizeof(uint64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    gather_u64_kernel<<<(unsigned)((n_bounds + 255) / 256), 256, 0, ctx->stream>>>(
        reinterpret_cast<const unsigned long long*>(ctx->row_ptr), reinterpret_cast<const unsigned long long*>(*out_row),
        n_bounds, reinterpret_cast<unsigned long long*>(*out_hit));
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(raw);
    return 0;
}

int em_build_tiles(rsem_b200_ctx* ctx) {
    if (ctx->tile_row) { cudaFree(ctx->tile_row); ctx->tile_row = nullptr; }
    if (ctx->tile_hit) { cudaFree(ctx->tile_hit); ctx->tile_hit = nullptr; }
    ctx->n_tiles = 0;
    ctx->tile_weight = 0;
    ctx->has_empty_row = false;
    if (ctx->N == 0) return 0;
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    uint32_t deg_info[2] = {0, 0};
    if (int rc = em_max_degree(ctx, deg_info)) return rc;
    ctx->max_deg = deg_info[0];
    ctx->has_empty_row = deg_info[1] != 0;

    // lanes per row from the mean degree (+1 for the noise entry)
    const double mean_deg = (double)ctx->H / (double)ctx->N + 1.0;
    ctx->group = mean_deg <= 5.0 ? 4 : mean_deg <= 11.0 ? 8 : mean_deg <= 26.0 ? 16 : 32;
    // lanes per row of the row kernel: kRowSlots hits per lane should cover about 1.5 mean rows
    ctx->rows_group = mean_deg <= 3.0 ? 1 : mean_deg <= 6.0 ? 2 : mean_deg <= 12.0 ? 4 : mean_deg <= 24.0 ? 8 : mean_deg <= 48.0 ? 16 : 32;
    // rows without hits are never produced by rsem-parse-alignments (HitContainer.h:67 asserts tot > 0): the
    // row kernel does not handle them, the direct kernel does
    if (deg_info[1]) return 0;

    // tiles of at most W + max_deg = kHitCap - 2 hits and kRowCap rows: with the lead-ins of the aligned copies
    // (<= 3 ids, <= 1 conprb, row_ptr and ncpv value) and the 16 B round-up of each copy, a tile fits a Stage
    if (ctx->max_deg <= (uint32_t)kThreads) {
        const unsigned long long W = (unsigned long long)kHitCap - 2 - ctx->max_deg;
        if (int rc = build_tile_set(ctx, W, kRowCap, &ctx->tile_row, &ctx->tile_hit, &ctx->n_tiles)) return rc;
    }
    return 0;
}

// frozen-conprb rounds run on the equivalence-class layout unless a CSR variant was selected
static bool wants_class_layout(const rsem_b200_ctx* ctx) {
    static const int no_class = getenv("RSEM_B200_NO_CLASS") ? atoi(getenv("RSEM_B200_NO_CLASS")) : 0;
    return ctx->variant == 5 || (ctx->variant == 0 && !no_class);
}

// Builds the class directory ahead of the first frozen round (it depends on row_ptr / sid only).  rsem_b200_upload_conprb
// calls this while the conprb copy is in flight; without it the first em_launch_estep builds the directory itself.
int em_prepare_frozen_layout(rsem_b200_ctx* ctx) {
    if (ctx->N == 0 || !wants_class_layout(ctx) || ctx->cls.built) return 0;
    return class_build(ctx);
}

// runs launch() between the two events of a K2 timing interval when profiling is on (rsem_b200_set_profiling)
template <class F>
static int profiled(rsem_b200_ctx* ctx, F&& launch) {
    if (!ctx->profiling) return launch();
    if (ctx->ev_used == ctx->ev_pool.size()) {
        cudaEvent_t x, y;
        RB_CUDA(cudaEventCreate(&x));
        RB_CUDA(cudaEventCreate(&y));
        ctx->ev_pool.emplace_back(x, y);
    }
    const auto ev = ctx->ev_pool[ctx->ev_used++];
    RB_CUDA(cudaEventRecord(ev.first, ctx->stream));
    if (int rc = launch()) return rc;
    RB_CUDA(cudaEventRecord(ev.second, ctx->stream));
    return 0;
}

int em_launch_estep(rsem_b200_ctx* ctx, bool write_post) {
    if (ctx->N == 0) return 0;
    // frozen-conprb rounds: equivalence-class layout (class_kernels.cu), built on first use after an upload and
    // re-gathered when conprb changed; posterior write-back stays on the CSR stream (hit order)
    if (!write_post && wants_class_layout(ctx)) {
        if (!ctx->cls.built) {
            if (int rc = class_build(ctx)) return rc;
        }
        if (ctx->cls.built) {
            if (ctx->cls.vals_epoch != ctx->conprb_epoch) {
                if (int rc = class_fill_vals(ctx)) return rc;
            }
            return profiled(ctx, [&] { return class_launch_estep(ctx); });
        }
        if (ctx->variant == 5) {
            set_error("class-layout E-step requested but the matrix is outside its limits (>= 2^32 reads or >= 2^40 hits)");
            return RSEM_B200_ERR_UNSUPPORTED;
        }
    }
    // CSR stream: the row kernel on the tiles, the direct kernel when there are none or on request (variant 2)
    if (ctx->variant == 4 && ctx->n_tiles == 0) {
        set_error("staged E-step requested but the matrix has rows that are empty or too long for a stage");
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    const bool direct = ctx->variant == 2 || ctx->n_tiles == 0;
    EstepArgs a;
    a.row_ptr = reinterpret_cast<const unsigned long long*>(ctx->row_ptr);
    a.sid = ctx->sid_abs;
    a.conprb = ctx->conprb;
    a.ncpv = ctx->ncpv;
    a.theta = ctx->theta;
    a.count = ctx->k2_target;
    a.post = ctx->post;
    a.post0 = ctx->post0;
    a.tile_row = reinterpret_cast<const unsigned long long*>(ctx->tile_row);
    a.tile_hit = reinterpret_cast<const unsigned long long*>(ctx->tile_hit);
    a.n_tiles = ctx->n_tiles;
    a.N = ctx->N;
    a.done_flag = ctx->done_flag;
    return profiled(ctx, [&] { return write_post ? launch_csr<true>(ctx, a, direct) : launch_csr<false>(ctx, a, direct); });
}

int em_launch_theta_update(rsem_b200_ctx* ctx, double n0, int round, int min_round, int max_round, int stats_slot) {
    theta_update_kernel<<<kThetaCluster, 1024, 0, ctx->stream>>>(ctx->count, ctx->theta, ctx->M + 1, n0, round, min_round,
                                                     max_round, ctx->d_stats + stats_slot, ctx->done_flag,
                                                     ctx->err_flag);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

}  // namespace rsem_b200
