// E-step / M-step kernels for frozen conditional probabilities (K2) and the theta update +
// convergence test (K4).
//
// What they compute is the reference's E_STEP inner loops (/root/reference/EM.cpp:199-244) and
// the M-step + relative-change statistics (/root/reference/EM.cpp:385-416).  How they compute
// it is specific to sm_90a:
//
//   * the hit matrix is SoA CSR in HBM (row_ptr u64, sid i32, conprb f64, ncpv f64); one pass
//     streams 12 B per hit + 16 B per read, nothing else comes from HBM (theta / count live in L2);
//   * rows are cut into byte-balanced tiles once per upload; a persistent CTA per SM walks its
//     tiles through a 3-stage shared-memory ring filled by 1-D bulk-async copies (TMA,
//     cp.async.bulk + mbarrier complete_tx), so the bytes in flight per SM are set by the ring
//     depth, not by occupancy or by the dependent row_ptr -> hits -> theta load chain;
//   * default kernel (estep_rows_kernel): warps claim batches of rows from a shared-memory counter, G lanes
//     own a row with its products in registers, row sums by xor-shuffles, normalised weights go to the
//     count vector with red.global.add.f64 (L2-resident); no CTA-wide barrier per tile, the warp that finishes a
//     tile last refills its stage.  The noise entry count[0] - which every row touches - is privatised in a
//     register and flushed once per CTA;
//   * alternatives kept for comparison and as fallbacks: three CTA-wide flat phases per tile (estep_tma_kernel),
//     warp-private tiles (estep_warp_kernel), no staging (estep_direct_kernel);
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

namespace rsem_b200 {

namespace {

// ------------------------------------------------------------------------------------------------
// tile geometry of the TMA-staged kernel
// ------------------------------------------------------------------------------------------------
constexpr int kStages = 3;
constexpr int kEnt = 4;  // hits per thread and tile in the flat phases (independent gathers in flight)

// A CTA of T threads works on tiles of <= 4 T - 2 hits and <= T rows; (T, CTAs per SM) = (512, 2), (256, 4) or
// (128, 8) keep 32 warps per SM and stay below 227 KB of shared memory per SM.
template <int T>
struct Geo {
    static constexpr int kThreads = T;
    static constexpr int kCtasPerSm = 1024 / T;
    static constexpr int kHitCap = kEnt * T;
    static constexpr int kRowCap = T;
    static constexpr int kSidElems = kHitCap + 8;
    static constexpr int kConElems = kHitCap + 4;
    static constexpr int kRowElems = kRowCap + 4;
    static constexpr int kMaskWords = kHitCap / 32 + 4;
};

// Static per-tile metadata, built once per upload and streamed with the tile.  Word w describes the elements
// q = 32 w .. 32 w + 31 of the tile (q = tile-local hit index + (first hit index & 1)): bit b of .x is set iff
// element 32 w + b starts a row, .y = number of row starts in the words before w, so that
// row(q) = w.y + popc(w.x & bits(0 .. q % 32)) - 1 with one 8-byte shared-memory load.
template <int T>
struct __align__(16) TileMeta {
    uint2 w[Geo<T>::kMaskWords];
};

template <int T>
struct __align__(16) Stage {
    double con[Geo<T>::kConElems];
    unsigned long long rp[Geo<T>::kRowElems];
    double ncp[Geo<T>::kRowElems];
    int sid[Geo<T>::kSidElems];
    TileMeta<T> meta;
};

struct TileDesc {  // written by the producer thread when it issues the tile, read by everyone after the wait
    unsigned long long rs, hs;
    unsigned nr, nh;
};

template <int T>
struct SmemLayout {
    Stage<T> stage[kStages];
    unsigned long long full_bar[kStages];
    TileDesc desc[kStages];
    double red[T / 32];
    double inv[Geo<T>::kRowCap];  // 1 / row sum of the tile being processed
};
static_assert(sizeof(Stage<512>) % 16 == 0 && sizeof(Stage<256>) % 16 == 0 && sizeof(Stage<128>) % 16 == 0,
              "stage must keep 16 B alignment");
static_assert(sizeof(TileMeta<512>) % 16 == 0 && sizeof(TileMeta<256>) % 16 == 0 && sizeof(TileMeta<128>) % 16 == 0,
              "tile metadata must keep 16 B alignment");
static_assert(sizeof(Stage<1024>) * kStages + 4096 <= 227 * 1024, "shared memory per SM");
static_assert(sizeof(SmemLayout<512>) * 2 <= 227 * 1024 && sizeof(SmemLayout<256>) * 4 <= 227 * 1024 &&
                  sizeof(SmemLayout<128>) * 8 <= 227 * 1024,
              "shared memory per SM");

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
    const void* tile_meta;
    unsigned int n_tiles;
    const unsigned long long* wtile_row;
    const unsigned long long* wtile_hit;
    unsigned int n_wtiles;
    unsigned long long N;
    const int* done_flag;
    cudaTextureObject_t theta_tex;  // theta as a 1-D int2 texture (row-group kernel, optional gather path)
    unsigned int contig;  // 1: a CTA walks a contiguous range of tiles, 0: tiles strided by the grid
};

// ---- PTX helpers -------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "RB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra RB_DONE;\n"
        "bra RB_WAIT;\n"
        "RB_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D bulk asynchronous copy global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP)
__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void red_add_f64(double* addr, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

// the same, skipped when v == 0 (no branch: the reduction is predicated)
__device__ __forceinline__ void red_add_f64_nz(double* addr, double v) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.neu.f64 p, %1, 0d0000000000000000;\n"
        "@p red.global.add.f64 [%0], %1;\n"
        "}\n" ::"l"(addr),
        "d"(v)
        : "memory");
}

template <int G>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <>
__device__ __forceinline__ double group_sum<1>(double v) { return v; }

__device__ __forceinline__ unsigned round16(unsigned bytes) { return (bytes + 15u) & ~15u; }

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
// K2, TMA-staged.  grid = #SMs (persistent), block = kThreads.
// ------------------------------------------------------------------------------------------------
template <int T, bool META = true>
__device__ __forceinline__ void issue_tile(const EstepArgs& a, unsigned k, Stage<T>& st, unsigned long long* bar,
                                           TileDesc& desc) {
    const unsigned long long rs = a.tile_row[k], re = a.tile_row[k + 1];
    const unsigned long long hs = a.tile_hit[k], he = a.tile_hit[k + 1];
    desc.rs = rs;
    desc.hs = hs;
    desc.nr = (unsigned)(re - rs);
    desc.nh = (unsigned)(he - hs);
    const unsigned long long hs4 = hs & ~3ull, hs2 = hs & ~1ull, rs2 = rs & ~1ull;
    const unsigned b_sid = round16((unsigned)(he - hs4) * 4u);
    const unsigned b_con = round16((unsigned)(he - hs2) * 8u);
    const unsigned b_rp = round16((unsigned)(re + 1 - rs2) * 8u);
    const unsigned b_nc = round16((unsigned)(re - rs2) * 8u);
    mbar_expect_tx(bar, b_sid + b_con + b_rp + b_nc + (META ? (unsigned)sizeof(TileMeta<T>) : 0u));
    if (b_sid) bulk_load(st.sid, a.sid + hs4, b_sid, bar);
    if (b_con) bulk_load(st.con, a.conprb + hs2, b_con, bar);
    bulk_load(st.rp, a.row_ptr + rs2, b_rp, bar);
    bulk_load(st.ncp, a.ncpv + rs2, b_nc, bar);
    if (META) bulk_load(&st.meta, static_cast<const TileMeta<T>*>(a.tile_meta) + k, (unsigned)sizeof(TileMeta<T>), bar);
}

// ------------------------------------------------------------------------------------------------
// K2, TMA-staged.  Persistent CTAs, two per SM (so one CTA's barrier bubbles are filled by the
// other), kThreads threads each.  A tile (<= kTileHitCap hits, <= kThreads / G rows) goes through
// three CTA-wide phases:
//   A  flat over hits (thread = hit, stride kThreads):  f = theta[|sid|] * conprb, clamped, written
//      over the conprb slot.  All loads are independent (4 gathers in flight per thread) and
//      consecutive threads touch consecutive transcript ids (isoforms of a gene are adjacent), so a
//      warp-wide gather needs only a few L2 sectors.
//   B  one row per group of G lanes (G ~ degree / 5, so every row of the tile is handled in ONE
//      pass with all lanes busy):  row sum incl. the noise term, reciprocal, f <- f / sum in place.
//   C  flat over hits again:  red.global.add.f64 of the normalised weight on the count vector -
//      consecutive threads -> consecutive addresses -> few sectors per request - and, for the
//      posterior variant, a coalesced store.
// ------------------------------------------------------------------------------------------------
template <int T, int G, bool WRITE_POST>
__global__ void __launch_bounds__(T, 1024 / T) estep_tma_kernel(const EstepArgs a) {
    constexpr int kThreads = T;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SmemLayout<T>& sm = *reinterpret_cast<SmemLayout<T>*>(smem_raw);
    if (*a.done_flag) return;

    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&sm.full_bar[s], 1);
        fence_barrier_init();
    }
    __syncthreads();
    unsigned k_first = blockIdx.x, k_end = a.n_tiles, k_step = gridDim.x;
    if (a.contig) {
        const unsigned q = a.n_tiles / gridDim.x, r = a.n_tiles % gridDim.x;
        k_first = blockIdx.x * q + min(blockIdx.x, r);
        k_end = k_first + q + (blockIdx.x < r ? 1u : 0u);
        k_step = 1;
    }
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            const unsigned k = k_first + s * k_step;
            if (k < k_end) issue_tile(a, k, sm.stage[s], &sm.full_bar[s], sm.desc[s]);
        }
    }

    constexpr int kSlots = 8;                     // hits a lane keeps in registers in phase B
    const int g = tid % G;
    const unsigned row_in_tile = tid / G;
    const double theta0 = __ldg(a.theta);
    double acc0 = 0.0;

    unsigned it = 0;
    for (unsigned k = k_first; k < k_end; k += k_step, ++it) {
        const int s = it % kStages;
        const unsigned parity = (it / kStages) & 1u;
        Stage<T>& st = sm.stage[s];
        mbar_wait(&sm.full_bar[s], parity);

        const unsigned long long rs = sm.desc[s].rs, hs = sm.desc[s].hs;
        const unsigned nr = sm.desc[s].nr, nh = sm.desc[s].nh;
        const unsigned roff = (unsigned)(rs & 1ull);
        // Flat phases: thread tid owns the tile-local hits tid, tid + kThreads, ... - a warp instruction touches 32
        // CONSECUTIVE hits, i.e. 1-3 runs of adjacent transcript ids.  That mapping is what the L2 reduction
        // unit wants (measured with tools/micro/red_bench.cu: 495 G red/s, against 279 G/s when a warp covers 64
        // hits with stride 2 and 201 G/s with stride 4) and it keeps the theta gathers to a few sectors too.
        // The stage arrays start at the aligned hit index below hs, hence the lead offsets.
        const unsigned con_lead = (unsigned)(hs & 1ull);
        const int* s_sid = st.sid + (unsigned)(hs & 3ull);
        double* s_con = st.con + con_lead;  // element 0 = first hit of the tile

        // ---- phase A: products; they stay in registers for phase C and are also written over the conprb
        //      slots for the row sums of phase B.  (A tile holds <= kThreads * kEnt hits, so one pass covers it.)
        int t[kEnt];
        double f[kEnt];
        {
            double th[kEnt], c[kEnt];
#pragma unroll
            for (int u = 0; u < kEnt; ++u) {
                const unsigned j = tid + kThreads * u;
                t[u] = j < nh ? s_sid[j] : 0;
            }
#pragma unroll
            for (int u = 0; u < kEnt; ++u) th[u] = __ldg(a.theta + t[u]);
#pragma unroll
            for (int u = 0; u < kEnt; ++u) {
                const unsigned j = tid + kThreads * u;
                c[u] = j < nh ? s_con[j] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < kEnt; ++u) {
                const unsigned j = tid + kThreads * u;
                f[u] = th[u] * c[u];
                if (f[u] < kEpsilon) f[u] = 0.0;
                if (j < nh) s_con[j] = f[u];
            }
        }
        __syncthreads();

        // ---- phase B: 1 / (noise term + row sum) per row (one pass when the tile has <= kThreads / G rows,
        //      which the tile builder aims for)
        for (unsigned rbase = 0; rbase < nr; rbase += kThreads / G) {
            const unsigned row = rbase + row_in_tile;
            const bool valid = row < nr;
            unsigned b = 0, e = 0;
            double x[kSlots];
            double part = 0.0, f0 = 0.0;
            if (valid) {
                b = (unsigned)(st.rp[roff + row] - hs);
                e = (unsigned)(st.rp[roff + row + 1] - hs);
            }
#pragma unroll
            for (int q = 0; q < kSlots; ++q) {
                const unsigned j = b + g + q * G;
                x[q] = j < e ? s_con[j] : 0.0;
            }
            part = ((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7]));
            for (unsigned j = b + g + kSlots * G; j < e; j += G) part += s_con[j];
            if (valid && g == 0) {
                f0 = theta0 * st.ncp[roff + row];
                if (f0 < kEpsilon) f0 = 0.0;
                part += f0;
            }
            const double sum = group_sum<G>(part);
            if (valid && g == 0) {
                const double inv = sum >= kEpsilon ? 1.0 / sum : 0.0;
                sm.inv[row] = inv;
                const double p0 = f0 * inv;
                acc0 += p0;
                if (WRITE_POST) a.post0[rs + row] = p0;
            }
        }
        __syncthreads();

        // ---- phase C: weight = product (register) * inv[row]; the row of a hit comes from the static head mask:
        //      q = hit index + lead, row(q) = w[q / 32].y + popc(w[q / 32].x & bits(0 .. q % 32)) - 1
#pragma unroll
        for (int u = 0; u < kEnt; ++u) {
            const unsigned j = tid + kThreads * u;
            if (j < nh) {
                const unsigned q = j + con_lead;
                const uint2 mw = st.meta.w[q >> 5];
                const unsigned row = mw.y + __popc(mw.x & (0xffffffffu >> (31u - (q & 31u)))) - 1u;
                const double w = f[u] * sm.inv[row];
                if (w != 0.0) red_add_f64(a.count + t[u], w);
                if (WRITE_POST) a.post[hs + j] = w;
            }
        }
        fence_proxy_async();  // generic-proxy writes to the stage precede its next bulk-async fill
        __syncthreads();      // every thread is done with stage s
        if (tid == 0) {
            const unsigned long long kn = (unsigned long long)k + (unsigned long long)kStages * k_step;
            if (kn < k_end) issue_tile(a, (unsigned)kn, st, &sm.full_bar[s], sm.desc[s]);
        }
    }
    flush_count0(acc0, sm.red, a.count);
}

// ------------------------------------------------------------------------------------------------
// K2, row groups on staged tiles (variant 4).  Same TMA ring as above, but a tile is consumed in ONE pass with
// no CTA-wide barrier: a warp claims batches of 32 / G rows from a shared-memory counter, G lanes own a row,
// lane g holds the row's hits g, g + G, ... (kRowSlots of them in registers): ids and conprb come from the stage
// (each byte of it is read once), theta is gathered, the row sum goes through log2(G) xor-shuffles and the
// normalised weights leave as red.global.add.f64 - a warp instruction covers 32 / G runs of G adjacent
// transcripts, which the L2 reduction unit handles as well as 32 consecutive ones.  Two batches are in flight
// per warp for instruction-level parallelism.  The warp that finishes a tile last refills its stage.
// ------------------------------------------------------------------------------------------------
constexpr int kRowSlots = 4;

template <int T>
struct RowSmem {
    Stage<T> stage[kStages];
    unsigned long long full_bar[kStages];
    TileDesc desc[kStages];
    unsigned int next_batch[kStages];
    unsigned int warps_done[kStages];
    double red[T / 32];
};

// theta[i] through the texture pipe instead of the LSU pipe (which is the busiest unit of this kernel)
__device__ __forceinline__ double theta_fetch(cudaTextureObject_t tex, unsigned i) {
    const int2 v = tex1Dfetch<int2>(tex, (int)i);
    return __hiloint2double(v.y, v.x);
}

template <int T, int G, bool WRITE_POST, int kRowUnroll, bool TEX>
__global__ void __launch_bounds__(T, 1024 / T) estep_rows_kernel(const EstepArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RowSmem<T>& sm = *reinterpret_cast<RowSmem<T>*>(smem_raw);
    if (*a.done_flag) return;
    constexpr unsigned kWarps = T / 32;
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
    unsigned k_first = blockIdx.x, k_end = a.n_tiles, k_step = gridDim.x;
    if (a.contig) {
        const unsigned q = a.n_tiles / gridDim.x, r = a.n_tiles % gridDim.x;
        k_first = blockIdx.x * q + min(blockIdx.x, r);
        k_end = k_first + q + (blockIdx.x < r ? 1u : 0u);
        k_step = 1;
    }
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            const unsigned k = k_first + s * k_step;
            if (k < k_end) issue_tile<T, false>(a, k, sm.stage[s], &sm.full_bar[s], sm.desc[s]);
        }
    }

    const unsigned g = lane % G;
    const unsigned row_in_batch = lane / G;
    const double theta0 = __ldg(a.theta);
    double acc0 = 0.0;

    unsigned it = 0;
    for (unsigned k = k_first; k < k_end; k += k_step, ++it) {
        const int s = it % kStages;
        const unsigned parity = (it / kStages) & 1u;
        Stage<T>& st = sm.stage[s];
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
                for (int q = 0; q < kRowSlots; ++q)
                    x[u][q] = TEX ? theta_fetch(a.theta_tex, (unsigned)t[u][q]) : __ldg(a.theta + t[u][q]);
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
                const unsigned long long kn = (unsigned long long)k + (unsigned long long)kStages * k_step;
                if (kn < k_end) issue_tile<T, false>(a, (unsigned)kn, st, &sm.full_bar[s], sm.desc[s]);
            }
        }
    }
    __syncthreads();
    flush_count0(acc0, sm.red, a.count);
}

// ------------------------------------------------------------------------------------------------
// K2, warp-pipelined.  Same three phases, but every WARP owns its own small tiles (<= kWHitCap hits,
// <= kWRowCap rows), its own 2-stage shared-memory ring and its own mbarriers: a warp's lane 0 issues the
// bulk-async copies of its next tile, the warp waits on its own barrier, phases are separated by
// __syncwarp only.  There is no CTA-wide barrier anywhere in the main loop, so the latency one warp spends
// waiting for its theta gathers or for the shared-memory chain of a row sum is filled by the other ~11
// warps of the SM instead of being multiplied by a __syncthreads.
// Phase B maps G = 32 / rows lanes to a row, chosen per tile at run time (lane = row for the typical 20-30
// rows per tile, more lanes per row when rows are long).
// ------------------------------------------------------------------------------------------------
constexpr int kWWarps = 4;        // warps per CTA
constexpr int kWStages = 2;
constexpr int kWHitCap = 576;     // hits per warp tile
constexpr int kWRowCap = 128;     // rows per warp tile

struct __align__(16) WStage {
    double con[kWHitCap + 4];
    unsigned long long rp[kWRowCap + 4];
    double ncp[kWRowCap + 4];
    int sid[kWHitCap + 8];
};
static_assert(sizeof(WStage) % 16 == 0, "stage must keep 16 B alignment");

struct WSmem {
    WStage stage[kWWarps][kWStages];
    unsigned long long full_bar[kWWarps][kWStages];
    TileDesc desc[kWWarps][kWStages];
    double red[kWWarps];
};

__device__ __forceinline__ void issue_wtile(const EstepArgs& a, unsigned k, WStage& st, unsigned long long* bar,
                                            TileDesc& desc) {
    const unsigned long long rs = a.wtile_row[k], re = a.wtile_row[k + 1];
    const unsigned long long hs = a.wtile_hit[k], he = a.wtile_hit[k + 1];
    desc.rs = rs;
    desc.hs = hs;
    desc.nr = (unsigned)(re - rs);
    desc.nh = (unsigned)(he - hs);
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

template <bool WRITE_POST>
__global__ void __launch_bounds__(kWWarps * 32, 3) estep_warp_kernel(const EstepArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    WSmem& sm = *reinterpret_cast<WSmem*>(smem_raw);
    if (*a.done_flag) return;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned n_streams = gridDim.x * kWWarps;          // one tile stream per warp
    const unsigned stream = blockIdx.x * kWWarps + warp;
    if (lane == 0) {
        for (int s = 0; s < kWStages; ++s) mbar_init(&sm.full_bar[warp][s], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (lane == 0) {
        for (int s = 0; s < kWStages; ++s) {
            const unsigned long long k = (unsigned long long)stream + (unsigned long long)s * n_streams;
            if (k < a.n_wtiles) issue_wtile(a, (unsigned)k, sm.stage[warp][s], &sm.full_bar[warp][s], sm.desc[warp][s]);
        }
    }
    __syncwarp();

    constexpr int kPairs = 2;
    const double theta0 = __ldg(a.theta);
    double acc0 = 0.0;
    unsigned it = 0;
    for (unsigned long long k = stream; k < a.n_wtiles; k += n_streams, ++it) {
        const int s = it % kWStages;
        const unsigned parity = (it / kWStages) & 1u;
        WStage& st = sm.stage[warp][s];
        mbar_wait(&sm.full_bar[warp][s], parity);

        const unsigned long long rs = sm.desc[warp][s].rs, hs = sm.desc[warp][s].hs;
        const unsigned nr = sm.desc[warp][s].nr, nh = sm.desc[warp][s].nh;
        const unsigned roff = (unsigned)(rs & 1ull);
        const unsigned con_lead = (unsigned)(hs & 1ull);
        const unsigned sid_shift = (unsigned)(hs & 2ull);
        const unsigned n_pairs = (con_lead + nh + 1) >> 1;
        double2* con2 = reinterpret_cast<double2*>(st.con);
        const uint2* sid2 = reinterpret_cast<const uint2*>(st.sid + sid_shift);
        double* s_con = st.con + con_lead;

        // ---- phase A: products, flat over pairs of hits
        for (unsigned p0 = lane; p0 < n_pairs; p0 += 32 * kPairs) {
            uint2 t[kPairs];
            double2 c[kPairs];
            double th[2 * kPairs];
#pragma unroll
            for (int u = 0; u < kPairs; ++u) {
                const unsigned p = p0 + 32 * u;
                t[u] = p < n_pairs ? sid2[p] : make_uint2(0u, 0u);
            }
#pragma unroll
            for (int u = 0; u < kPairs; ++u) {
                th[2 * u] = __ldg(a.theta + t[u].x);
                th[2 * u + 1] = __ldg(a.theta + t[u].y);
            }
#pragma unroll
            for (int u = 0; u < kPairs; ++u) {
                const unsigned p = p0 + 32 * u;
                c[u] = p < n_pairs ? con2[p] : make_double2(0.0, 0.0);
            }
#pragma unroll
            for (int u = 0; u < kPairs; ++u) {
                const unsigned p = p0 + 32 * u;
                double2 f;
                f.x = th[2 * u] * c[u].x;
                f.y = th[2 * u + 1] * c[u].y;
                if (f.x < kEpsilon) f.x = 0.0;
                if (f.y < kEpsilon) f.y = 0.0;
                if (p < n_pairs) con2[p] = f;
            }
        }
        __syncwarp();

        // ---- phase B: row sums; G lanes per row, G = largest power of two <= 32 / min(nr, 32)
        {
            const unsigned rows_now = nr < 32u ? nr : 32u;
            const unsigned shift = 31u - __clz(32u / rows_now);   // log2(G)
            const unsigned G = 1u << shift;
            const unsigned g = lane & (G - 1), row_in_pass = lane >> shift, rows_per_pass = 32u >> shift;
            for (unsigned rb = 0; rb < nr; rb += rows_per_pass) {
                const unsigned row = rb + row_in_pass;
                const bool valid = row < nr;
                unsigned b = 0, e = 0;
                if (valid) {
                    b = (unsigned)(st.rp[roff + row] - hs);
                    e = (unsigned)(st.rp[roff + row + 1] - hs);
                }
                double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, f0 = 0.0;
                unsigned j = b + g;
                const unsigned step = G;
                for (; j + 3 * step < e; j += 4 * step) {
                    s0 += s_con[j];
                    s1 += s_con[j + step];
                    s2 += s_con[j + 2 * step];
                    s3 += s_con[j + 3 * step];
                }
                for (; j < e; j += step) s0 += s_con[j];
                double part = (s0 + s1) + (s2 + s3);
                if (valid && g == 0) {
                    f0 = theta0 * st.ncp[roff + row];
                    if (f0 < kEpsilon) f0 = 0.0;
                    part += f0;
                }
                for (unsigned o = G >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                const double inv = part >= kEpsilon ? 1.0 / part : 0.0;
                for (j = b + g; j < e; j += step) s_con[j] *= inv;
                if (valid && g == 0) {
                    const double p0 = f0 * inv;
                    acc0 += p0;
                    if (WRITE_POST) a.post0[rs + row] = p0;
                }
            }
        }
        __syncwarp();

        // ---- phase C: count updates, flat over pairs of hits
        for (unsigned p = lane; p < n_pairs; p += 32) {
            const double2 w = con2[p];
            const uint2 t = sid2[p];
            const unsigned j0 = 2 * p - con_lead, j1 = j0 + 1;
            if (j0 < nh) {
                if (w.x != 0.0) red_add_f64(a.count + t.x, w.x);
                if (WRITE_POST) a.post[hs + j0] = w.x;
            }
            if (j1 < nh) {
                if (w.y != 0.0) red_add_f64(a.count + t.y, w.y);
                if (WRITE_POST) a.post[hs + j1] = w.y;
            }
        }
        fence_proxy_async();  // this warp's generic-proxy writes to the stage precede its next bulk-async fill
        __syncwarp();
        if (lane == 0) {
            const unsigned long long kn = k + (unsigned long long)kWStages * n_streams;
            if (kn < a.n_wtiles) issue_wtile(a, (unsigned)kn, st, &sm.full_bar[warp][s], sm.desc[warp][s]);
        }
        __syncwarp();
    }
    flush_count0(acc0, sm.red, a.count);
}

// ------------------------------------------------------------------------------------------------
// K2, direct variant: same row logic, loads straight from global memory (no staging).  Used as
// the fallback for rows longer than a stage and as the comparison point in the profiles.
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

// one block per tile: row-start bit mask over the tile's elements + prefix counts (TileMeta)
template <int T>
__global__ void tile_meta_kernel(const unsigned long long* row_ptr, const unsigned long long* tile_row,
                                 const unsigned long long* tile_hit, TileMeta<T>* out) {
    constexpr int kMaskWords = Geo<T>::kMaskWords;
    __shared__ unsigned m[kMaskWords];
    const unsigned k = blockIdx.x;
    for (int w = threadIdx.x; w < kMaskWords; w += blockDim.x) m[w] = 0u;
    __syncthreads();
    const unsigned long long rs = tile_row[k], re = tile_row[k + 1], hs = tile_hit[k];
    const unsigned lead = (unsigned)(hs & 1ull);
    for (unsigned long long r = rs + threadIdx.x; r < re; r += blockDim.x) {
        const unsigned q = (unsigned)(row_ptr[r] - hs) + lead;
        atomicOr(&m[q >> 5], 1u << (q & 31u));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned run = 0;
        for (int w = 0; w < kMaskWords; ++w) {
            out[k].w[w] = make_uint2(m[w], run);
            run += __popc(m[w]);
        }
    }
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

template <int T, int G, bool WP>
int launch_staged(rsem_b200_ctx* ctx, const EstepArgs& a) {
    auto kern = estep_tma_kernel<T, G, WP>;
    const size_t smem = sizeof(SmemLayout<T>);
    RB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    unsigned grid = ctx->sm_count * Geo<T>::kCtasPerSm;
    if (grid > a.n_tiles) grid = a.n_tiles ? a.n_tiles : 1;
    kern<<<grid, T, smem, ctx->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

template <int T, int G, bool WP, bool TEX>
int launch_rows_tex(rsem_b200_ctx* ctx, const EstepArgs& a) {
    auto kern = estep_rows_kernel<T, G, WP, 2, TEX>;
    const size_t smem = sizeof(RowSmem<T>);
    RB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    unsigned grid = ctx->sm_count * Geo<T>::kCtasPerSm;
    if (grid > a.n_tiles) grid = a.n_tiles ? a.n_tiles : 1;
    kern<<<grid, T, smem, ctx->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

template <int T, int G, bool WP>
int launch_rows(rsem_b200_ctx* ctx, const EstepArgs& a) {
    return a.theta_tex ? launch_rows_tex<T, G, WP, true>(ctx, a) : launch_rows_tex<T, G, WP, false>(ctx, a);
}

template <int G, bool WP>
int launch_variant(rsem_b200_ctx* ctx, const EstepArgs& a, bool tma) {
    if (tma && ctx->tiles_for_rows) {
        switch (ctx->cta_threads) {
            case 128: return launch_rows<128, G, WP>(ctx, a);
            case 256: return launch_rows<256, G, WP>(ctx, a);
            case 1024: return launch_rows<1024, G, WP>(ctx, a);
            default: return launch_rows<512, G, WP>(ctx, a);
        }
    }
    if (tma) {
        switch (ctx->cta_threads) {
            case 128: return launch_staged<128, G, WP>(ctx, a);
            case 256: return launch_staged<256, G, WP>(ctx, a);
            default: return launch_staged<512, G, WP>(ctx, a);
        }
    }
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
int launch_warp(rsem_b200_ctx* ctx, const EstepArgs& a) {
    auto kern = estep_warp_kernel<WP>;
    const size_t smem = sizeof(WSmem);
    RB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    unsigned long long want = ((unsigned long long)a.n_wtiles + kWWarps - 1) / kWWarps;
    unsigned grid = (unsigned)std::min<unsigned long long>(want ? want : 1, (unsigned long long)ctx->sm_count * 3);
    kern<<<grid, kWWarps * 32, smem, ctx->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    ctx->launches++;
    return 0;
}

template <bool WP>
int launch_group(rsem_b200_ctx* ctx, const EstepArgs& a, bool tma) {
    if (tma) {
        switch (ctx->tiles_for_rows ? ctx->rows_group : ctx->tma_group) {
            case 1: return launch_variant<1, WP>(ctx, a, true);
            case 2: return launch_variant<2, WP>(ctx, a, true);
            case 4: return launch_variant<4, WP>(ctx, a, true);
            case 8: return launch_variant<8, WP>(ctx, a, true);
            case 16: return launch_variant<16, WP>(ctx, a, true);
            default: return launch_variant<32, WP>(ctx, a, true);
        }
    }
    switch (ctx->group) {
        case 4: return launch_variant<4, WP>(ctx, a, tma);
        case 8: return launch_variant<8, WP>(ctx, a, tma);
        case 16: return launch_variant<16, WP>(ctx, a, tma);
        default: return launch_variant<32, WP>(ctx, a, tma);
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
    if (ctx->tile_meta) { cudaFree(ctx->tile_meta); ctx->tile_meta = nullptr; }
    if (ctx->wtile_row) { cudaFree(ctx->wtile_row); ctx->wtile_row = nullptr; }
    if (ctx->wtile_hit) { cudaFree(ctx->wtile_hit); ctx->wtile_hit = nullptr; }
    ctx->n_tiles = ctx->n_wtiles = 0;
    if (ctx->N == 0) return 0;
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    uint32_t deg_info[2] = {0, 0};
    if (int rc = em_max_degree(ctx, deg_info)) return rc;
    ctx->max_deg = deg_info[0];

    // lanes per row from the mean degree (+1 for the noise entry)
    const double mean_deg = (double)ctx->H / (double)ctx->N + 1.0;
    ctx->group = mean_deg <= 5.0 ? 4 : mean_deg <= 11.0 ? 8 : mean_deg <= 26.0 ? 16 : 32;
    // lanes per row in phase B of the CTA-staged kernel: about one lane per 5 hits
    ctx->tma_group = mean_deg <= 7.0 ? 1 : mean_deg <= 14.0 ? 2 : mean_deg <= 28.0 ? 4 : mean_deg <= 56.0 ? 8 : mean_deg <= 112.0 ? 16 : 32;
    // lanes per row of the row-group kernel: kRowSlots hits per lane should cover about 1.5 mean rows
    ctx->rows_group = mean_deg <= 3.0 ? 1 : mean_deg <= 6.0 ? 2 : mean_deg <= 12.0 ? 4 : mean_deg <= 24.0 ? 8 : mean_deg <= 48.0 ? 16 : 32;
    if (const char* e = getenv("RSEM_B200_GROUP")) {  // tuning knob (profiling only)
        const int v = atoi(e);
        if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16 || v == 32) ctx->tma_group = ctx->rows_group = v;
    }
    // rows without hits are never produced by rsem-parse-alignments (HitContainer.h:67 asserts tot > 0): the
    // staged kernels do not handle them, the direct kernel does
    if (deg_info[1]) return 0;

    // CTA tiles of the staged kernel: hits <= W + max_deg <= 4 T - 2, so that every thread owns at most kEnt hits
    // of a tile (one fully unrolled pass per flat phase) and a lead-in element still fits the mask.
    // Tile geometry follows the kernel that will consume the tiles.  Measured on C3 (ms per round):
    //   row-group kernel (variants 0 / 4): 3.40 with 1024 threads x 1 CTA per SM, 3.50 with 512 x 2, 3.75 with 256 x 4
    //   three-phase kernel (variant 1):    4.35 with 256 x 4, 4.39 with 128 x 8, 4.61 with 512 x 2
    ctx->tiles_for_rows = ctx->variant == 0 || ctx->variant == 4 || ctx->variant == 5;
    if (ctx->tiles_for_rows) ctx->cta_threads = 1024;
    else ctx->cta_threads = ctx->max_deg <= 256 ? 256 : 512;
    if (const char* e = getenv("RSEM_B200_CTA_THREADS")) {  // tuning knob
        const int v = atoi(e);
        if (v == 128 || v == 256 || v == 512 || (v == 1024 && ctx->tiles_for_rows)) ctx->cta_threads = v;
    }
    const unsigned T = (unsigned)ctx->cta_threads;
    if (ctx->max_deg <= T) {
        const unsigned long long W = (unsigned long long)kEnt * T - 2 - ctx->max_deg;
        if (int rc = build_tile_set(ctx, W, T, &ctx->tile_row, &ctx->tile_hit, &ctx->n_tiles)) return rc;
        if (ctx->n_tiles > 0) {
            const unsigned long long* rp = reinterpret_cast<const unsigned long long*>(ctx->row_ptr);
            const unsigned long long* tr = reinterpret_cast<const unsigned long long*>(ctx->tile_row);
            const unsigned long long* th = reinterpret_cast<const unsigned long long*>(ctx->tile_hit);
            if (ctx->tiles_for_rows) {
                // the row-group kernel needs no row-start masks
            } else if (T == 128) {
                RB_CUDA(cudaMalloc(&ctx->tile_meta, (size_t)ctx->n_tiles * sizeof(TileMeta<128>)));
                tile_meta_kernel<128><<<ctx->n_tiles, 64, 0, ctx->stream>>>(rp, tr, th, static_cast<TileMeta<128>*>(ctx->tile_meta));
            } else if (T == 256) {
                RB_CUDA(cudaMalloc(&ctx->tile_meta, (size_t)ctx->n_tiles * sizeof(TileMeta<256>)));
                tile_meta_kernel<256><<<ctx->n_tiles, 64, 0, ctx->stream>>>(rp, tr, th, static_cast<TileMeta<256>*>(ctx->tile_meta));
            } else {
                RB_CUDA(cudaMalloc(&ctx->tile_meta, (size_t)ctx->n_tiles * sizeof(TileMeta<512>)));
                tile_meta_kernel<512><<<ctx->n_tiles, 64, 0, ctx->stream>>>(rp, tr, th, static_cast<TileMeta<512>*>(ctx->tile_meta));
            }
            RB_CUDA(cudaGetLastError());
            ctx->launches++;
            RB_CUDA(cudaStreamSynchronize(ctx->stream));
        }
    }
    // warp tiles
    if (ctx->max_deg <= (uint32_t)kWHitCap / 2) {
        const unsigned long long W = (unsigned long long)kWHitCap - ctx->max_deg;
        if (int rc = build_tile_set(ctx, W, kWRowCap, &ctx->wtile_row, &ctx->wtile_hit, &ctx->n_wtiles)) return rc;
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

int em_launch_estep(rsem_b200_ctx* ctx, bool write_post) {
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
    a.tile_meta = ctx->tile_meta;
    a.n_tiles = ctx->n_tiles;
    a.wtile_row = reinterpret_cast<const unsigned long long*>(ctx->wtile_row);
    a.wtile_hit = reinterpret_cast<const unsigned long long*>(ctx->wtile_hit);
    a.n_wtiles = ctx->n_wtiles;
    a.N = ctx->N;
    a.done_flag = ctx->done_flag;
    // each CTA walks a contiguous range of tiles (4 % faster on C3 than striding by the grid); 0 = strided
    static const int tile_order = getenv("RSEM_B200_TILE_ORDER") ? atoi(getenv("RSEM_B200_TILE_ORDER")) : 1;
    a.contig = tile_order != 0;
    a.theta_tex = 0;
    static const int use_tex = getenv("RSEM_B200_THETA_TEX") ? atoi(getenv("RSEM_B200_THETA_TEX")) : 0;
    if (use_tex) {
        if (ctx->theta_tex && ctx->theta_tex_ptr != ctx->theta) {
            cudaDestroyTextureObject(ctx->theta_tex);
            ctx->theta_tex = 0;
        }
        if (!ctx->theta_tex) {
            cudaResourceDesc rd = {};
            rd.resType = cudaResourceTypeLinear;
            rd.res.linear.devPtr = ctx->theta;
            rd.res.linear.desc = cudaCreateChannelDesc<int2>();
            rd.res.linear.sizeInBytes = ((size_t)ctx->M + 1) * sizeof(double);
            cudaTextureDesc td = {};
            td.readMode = cudaReadModeElementType;
            RB_CUDA(cudaCreateTextureObject(&ctx->theta_tex, &rd, &td, nullptr));
            ctx->theta_tex_ptr = ctx->theta;
        }
        a.theta_tex = ctx->theta_tex;
    }
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
            cudaEvent_t c0 = nullptr, c1 = nullptr;
            if (ctx->profiling) {
                if (ctx->ev_used == ctx->ev_pool.size()) {
                    cudaEvent_t x, y;
                    RB_CUDA(cudaEventCreate(&x));
                    RB_CUDA(cudaEventCreate(&y));
                    ctx->ev_pool.emplace_back(x, y);
                }
                c0 = ctx->ev_pool[ctx->ev_used].first;
                c1 = ctx->ev_pool[ctx->ev_used].second;
                ctx->ev_used++;
                RB_CUDA(cudaEventRecord(c0, ctx->stream));
            }
            if (int rc = class_launch_estep(ctx)) return rc;
            if (ctx->profiling) RB_CUDA(cudaEventRecord(c1, ctx->stream));
            return 0;
        }
        if (ctx->variant == 5) {
            set_error("class-layout E-step requested but the matrix is outside its limits (>= 2^32 reads or >= 2^40 hits)");
            return RSEM_B200_ERR_UNSUPPORTED;
        }
    }
    if (ctx->tiles_for_rows != (ctx->variant == 0 || ctx->variant == 4 || ctx->variant == 5)) {  // variant changed after the upload
        if (int rc = em_build_tiles(ctx)) return rc;
        a.tile_row = reinterpret_cast<const unsigned long long*>(ctx->tile_row);
        a.tile_hit = reinterpret_cast<const unsigned long long*>(ctx->tile_hit);
        a.tile_meta = ctx->tile_meta;
        a.n_tiles = ctx->n_tiles;
        a.wtile_row = reinterpret_cast<const unsigned long long*>(ctx->wtile_row);
        a.wtile_hit = reinterpret_cast<const unsigned long long*>(ctx->wtile_hit);
        a.n_wtiles = ctx->n_wtiles;
    }
    // variant: 0 auto (row groups on staged tiles > warp-pipelined > direct), 1 three-phase CTA-staged, 2 direct,
    // 3 warp-pipelined, 4 row groups on staged tiles
    const bool use_warp = ctx->n_wtiles > 0 && (ctx->variant == 3 || (ctx->variant == 0 && ctx->n_tiles == 0));
    const bool tma = !use_warp && ctx->n_tiles > 0 && ctx->variant != 2 && ctx->variant != 3;
    if (((ctx->variant == 1 || ctx->variant == 4) && ctx->n_tiles == 0) || (ctx->variant == 3 && ctx->n_wtiles == 0)) {
        set_error("staged E-step requested but the matrix has rows that are empty or too long for a stage");
        return RSEM_B200_ERR_UNSUPPORTED;
    }

    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (ctx->profiling) {
        if (ctx->ev_used == ctx->ev_pool.size()) {
            cudaEvent_t x, y;
            RB_CUDA(cudaEventCreate(&x));
            RB_CUDA(cudaEventCreate(&y));
            ctx->ev_pool.emplace_back(x, y);
        }
        e0 = ctx->ev_pool[ctx->ev_used].first;
        e1 = ctx->ev_pool[ctx->ev_used].second;
        ctx->ev_used++;
        RB_CUDA(cudaEventRecord(e0, ctx->stream));
    }
    int rc;
    if (use_warp) rc = write_post ? launch_warp<true>(ctx, a) : launch_warp<false>(ctx, a);
    else rc = write_post ? launch_group<true>(ctx, a, tma) : launch_group<false>(ctx, a, tma);
    if (rc) return rc;
    if (ctx->profiling) RB_CUDA(cudaEventRecord(e1, ctx->stream));
    return 0;
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
