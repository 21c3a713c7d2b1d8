// K2 for the frozen-conprb rounds (ROUND >= 12 of /root/reference/EM.cpp:364-416) on an equivalence-class layout.
//
// What is computed is still E_STEP's inner loops (EM.cpp:199-244) + the count accumulation of EM.cpp:385-389.
// Why a second layout: on the CSR stream the row kernel (em_kernels.cu) is bound by the SM's load/store pipe, not by
// HBM - every hit costs one theta gather and one red.global on the count vector.  Reads that align to exactly the
// same transcript set (an "equivalence class": all fragments from the shared body of an isoform family) need the
// same theta values and add to the same counts, so
//
//   * at upload the rows are sorted by (degree, hash of the id list) and verified pairwise -> classes;
//   * a class is cut into SEGMENTS of <= R rows; a lane group owns a segment: it loads the ids and theta ONCE,
//     walks the segment's rows keeping the normalised weights in per-lane accumulators and issues ONE reduction per
//     transcript and segment (R x fewer gathers and reductions; singletons degrade to the row kernel's cost);
//   * 32 / G segments of equal (rows, degree) form a BATCH = the unit a warp claims; a batch's conprb / ncpv values
//     are stored interleaved (value (segment gi, row r, column c) at (r d + c) nsb + gi) so that every warp-wide
//     shared-memory load reads 32 consecutive doubles (no bank conflicts), with no padding in HBM;
//   * ids are stored once per segment (4 B per hit / rows per segment) and row pointers disappear (a batch
//     descriptor of 16 B replaces them); a segment over consecutive transcripts (a run, the common case) stores only
//     its first id: ~8.5 B per hit at C3 instead of 12.8;
//   * batches are staged by 1-D bulk-async copies (TMA) into a 3-stage shared-memory ring per persistent CTA, as in the
//     row kernel; each CTA claims tiles from a counter in global memory, no CTA-wide barrier per tile;
//   * rows longer than kLongDeg hits (never produced behind RSEM's aligner caps of 200) are left out of the
//     layout and handled by their own launch on the CSR stream - they no longer demote the whole matrix.
//
// The layout is derived data: the directory depends on (row_ptr, sid) only and is built once per upload; the value
// stream is re-gathered from conprb / ncpv whenever those change (once, after round 11).  Posterior write-back
// (rounds 1-10 and the final pass, EM.cpp:460-478) keeps using the CSR kernels, which preserve hit order.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <ctime>

#include "common.cuh"
#include "tma.cuh"

namespace rsem_b200 {

namespace {

constexpr int kStages = 3;
constexpr unsigned kStageBytes = 64 * 1024;
constexpr unsigned kLongDeg = 2047;       // rows with more hits are handled outside the class layout
constexpr unsigned kMaxBatchVals = 4096;  // values (conprb + ncpv) per batch, so that a batch is <= half a stage
constexpr unsigned long long kLongKey = 1ull << 59;
constexpr unsigned long long kOff48 = (1ull << 48) - 1, kOff40 = (1ull << 40) - 1;

// A row of degree d has d + 1 columns: its d hits and the noise entry (theta[0] * ncpv, EM.cpp:210-213), which is
// stored and processed as the last column.  Lanes per segment (G) and register slots per lane (S) from the column
// count w: S * G >= w up to w = 128.  Wider rows (G = 32, S = 4 plus a loop over the columns beyond 128) are
// configuration kTailCfg; they run in a launch of their own so that configurations 0-11 carry no code for them.
constexpr unsigned kTailCfg = 12;
__host__ __device__ __forceinline__ unsigned group_of_deg(unsigned d) {
    const unsigned w = d + 1u;
    return w <= 4 ? 1u : w <= 8 ? 2u : w <= 16 ? 4u : w <= 32 ? 8u : w <= 64 ? 16u : 32u;
}
__host__ __device__ __forceinline__ unsigned cfg_of_deg(unsigned d) {  // 2 * log2(G) + (S == 4), or kTailCfg
    if (d + 1u > 128u) return kTailCfg;
    const unsigned G = group_of_deg(d);
    const unsigned lg = G == 1 ? 0u : G == 2 ? 1u : G == 4 ? 2u : G == 8 ? 3u : G == 16 ? 4u : 5u;
    return 2u * lg + (d + 1u > 3u * G ? 1u : 0u);
}
__host__ __device__ __forceinline__ unsigned rows_cap(unsigned d, unsigned R) {
    const unsigned P = 32u / group_of_deg(d);
    const unsigned c = kMaxBatchVals / (P * (d + 1u));
    return c < 1u ? 1u : (c < R ? c : R);
}

// A segment is a RUN when its ids are first, first + 1, ..., first + d - 1 (a row over consecutive transcripts: the
// isoforms of a gene are numbered contiguously).  The ids of a run batch (all its segments runs) are stored as one
// first per segment, or one for the batch when all its segments belong to one class; other batches store every id.
// Rows of configuration kTailCfg are never marked runs: the tail launch reads their ids from the stage.
struct __align__(16) BatchDesc {
    unsigned long long w0;  // val_off (48 bits) | degree << 48
    unsigned long long w1;  // id_off (40 bits) | rows << 40 | segments << 48 | cfg << 56 | same_class << 60 | run << 61
};

// segment sort key: degree << 9 | run << 8 | (255 - rows), 20 bits (degree <= kLongDeg): segments ordered by degree,
// then non-runs before runs, then by decreasing row count
constexpr int kKey2Bits = 20;
__host__ __device__ __forceinline__ unsigned key2_deg(unsigned k) { return k >> 9; }
__host__ __device__ __forceinline__ unsigned key2_run(unsigned k) { return (k >> 8) & 1u; }
__host__ __device__ __forceinline__ unsigned key2_rows(unsigned k) { return 255u - (k & 255u); }

struct TileRec {
    unsigned long long val_begin, id_begin, batch_begin;
};

// ---- PTX helpers beyond tma.cuh ----------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// mbar_wait that adds the time it blocked to *acc when profiling (acc != nullptr); no timer read otherwise
__device__ __forceinline__ void mbar_wait_timed(unsigned long long* bar, unsigned parity, unsigned long long* acc) {
    if (acc) {
        const unsigned long long t0 = global_ns();
        mbar_wait(bar, parity);
        *acc += global_ns() - t0;
    } else {
        mbar_wait(bar, parity);
    }
}

// %clock64 reads of the profiling build (SM cycles; one clock per SM, so the warps of a CTA share it)
__device__ __forceinline__ long long clk() {
    long long t;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
    return t;
}
// the same read behind a branch on v, so that it cannot issue before v has arrived (v is never NaN here)
__device__ __forceinline__ long long clk_after(double v) {
    long long t = 0;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.nan.f64 p, %1, %1;\n"
        "@p bra RB_CLK;\n"
        "mov.u64 %0, %%clock64;\n"
        "RB_CLK:\n"
        "}\n"
        : "+l"(t)
        : "d"(v)
        : "memory");
    return t;
}
// Phases of a consumer warp's time, in SM cycles of lane 0 (profiling build only): front = a batch's descriptor, ids
// and theta gather until theta is usable, rows = the row walk, flush = fold + reductions on the count vector,
// hand-over = releasing a stage -> the next stage's data seen.
enum { kPhFront = 0, kPhRows, kPhFlush, kPhHandOver, kPhases };

// ------------------------------------------------------------------------------------------------------------------
// directory construction
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long mix_id(int id, unsigned c) {
    unsigned long long x = (unsigned long long)(unsigned)id * 0x9E3779B97F4A7C15ull + (unsigned long long)(c + 1u) * 0xC2B2AE3D27D4EB4Full;
    x ^= x >> 29;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 32;
    return x;
}

// 8 lanes per row: key = degree << 48 | 48-bit hash of the (position, id) pairs; long rows get kLongKey
__global__ void cls_row_key_kernel(const unsigned long long* __restrict__ rp, const int* __restrict__ sid_abs,
                                   unsigned long long N, unsigned long long* keys, unsigned* rows, unsigned* n_long) {
    const unsigned long long gid = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const unsigned g = threadIdx.x & 7u;
    if (gid >= N) return;  // whole groups leave together
    const unsigned long long b = rp[gid], e = rp[gid + 1];
    const unsigned long long d = e - b;
    unsigned long long h = 0;
    if (d <= kLongDeg)
        for (unsigned c = g; c < (unsigned)d; c += 8) h += mix_id(sid_abs[b + c], c);
    const unsigned mask = 0xffu << ((threadIdx.x & 31u) & ~7u);
    h += __shfl_xor_sync(mask, h, 1);
    h += __shfl_xor_sync(mask, h, 2);
    h += __shfl_xor_sync(mask, h, 4);
    if (g == 0) {
        rows[gid] = (unsigned)gid;
        if (d > kLongDeg) {
            keys[gid] = kLongKey;
            atomicAdd(n_long, 1u);
        } else {
            keys[gid] = (d << 48) | (h >> 16);
        }
    }
}

// 8 lanes per sorted position: does row p start a new class (different key, degree or id list than row p - 1)?
__global__ void cls_new_class_kernel(const unsigned long long* __restrict__ rp, const int* __restrict__ sid_abs,
                                     const unsigned long long* __restrict__ keys, const unsigned* __restrict__ rows,
                                     unsigned n_rows, unsigned* start_or_zero) {
    const unsigned long long gid = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const unsigned g = threadIdx.x & 7u;
    if (gid >= n_rows) return;
    const unsigned p = (unsigned)gid;
    bool same = p > 0 && keys[p] == keys[p - 1];
    if (same) {
        const unsigned long long a = rp[rows[p]], b = rp[rows[p - 1]];
        const unsigned d = (unsigned)(keys[p] >> 48);
        for (unsigned c = g; c < d; c += 8)
            if (sid_abs[a + c] != sid_abs[b + c]) same = false;
    }
    const unsigned mask = 0xffu << ((threadIdx.x & 31u) & ~7u);
    const unsigned all = __ballot_sync(mask, same);
    if (g == 0) start_or_zero[p] = ((all & mask) == mask) ? 0u : p;
}

struct MaxOp {
    __device__ __forceinline__ unsigned operator()(unsigned a, unsigned b) const { return a > b ? a : b; }
};

__global__ void cls_seg_flag_kernel(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cstart,
                                    unsigned n_rows, unsigned R, unsigned* flag) {
    const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_rows) return;
    const unsigned d = (unsigned)(keys[p] >> 48);
    flag[p] = ((p - cstart[p]) % rows_cap(d, R)) == 0u ? 1u : 0u;
}

__global__ void cls_seg_scatter_kernel(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cstart,
                                       const unsigned* __restrict__ flag, const unsigned* __restrict__ segidx1,
                                       unsigned n_rows, unsigned* seg_first, unsigned* seg_cls) {
    const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_rows || !flag[p]) return;
    const unsigned s = segidx1[p] - 1u;
    seg_first[s] = p;
    seg_cls[s] = cstart[p];
}

// key2 of every segment (see key2_deg); the rows of a segment share their id list, so its first row decides "run"
__global__ void cls_seg_key_kernel(const unsigned long long* __restrict__ rp, const int* __restrict__ sid_abs,
                                   const unsigned long long* __restrict__ keys, const unsigned* __restrict__ rows,
                                   const unsigned* __restrict__ seg_first, unsigned n_segs, unsigned n_rows, unsigned* key2,
                                   unsigned* segid) {
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_segs) return;
    const unsigned first = seg_first[s];
    const unsigned n = (s + 1 < n_segs ? seg_first[s + 1] : n_rows) - first;
    const unsigned d = (unsigned)(keys[first] >> 48);
    bool run = d >= 1u && cfg_of_deg(d) != kTailCfg;
    if (run) {
        const int* ids = sid_abs + rp[rows[first]];
        const unsigned id0 = (unsigned)ids[0];
        for (unsigned c = 1; c < d && run; ++c) run = (unsigned)ids[c] == id0 + c;
    }
    key2[s] = (d << 9) | (run ? 256u : 0u) | (255u - n);
    segid[s] = s;
}

__global__ void cls_run_start_kernel(const unsigned* __restrict__ key2s, unsigned n_segs, unsigned* start_or_zero) {
    const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_segs) return;
    start_or_zero[f] = (f > 0 && key2s[f] == key2s[f - 1]) ? 0u : f;
}

__global__ void cls_batch_flag_kernel(const unsigned* __restrict__ key2s, const unsigned* __restrict__ rstart,
                                      unsigned n_segs, unsigned* flag) {
    const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_segs) return;
    const unsigned P = 32u / group_of_deg(key2_deg(key2s[f]));
    flag[f] = ((f - rstart[f]) % P) == 0u ? 1u : 0u;
}

__global__ void cls_batch_scatter_kernel(const unsigned* __restrict__ flag, const unsigned* __restrict__ bidx1,
                                         unsigned n_segs, unsigned* batch_first) {
    const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_segs || !flag[f]) return;
    batch_first[bidx1[f] - 1u] = f;
}

// per batch: value / id counts (scanned into offsets afterwards) and the "all segments belong to one class" flag;
// *run_hits += the hits of run batches.  A batch's segments share key2, so they are all runs or all not.
__global__ void cls_batch_size_kernel(const unsigned* __restrict__ key2s, const unsigned* __restrict__ batch_first,
                                      const unsigned* __restrict__ segid_s, const unsigned* __restrict__ seg_cls,
                                      unsigned n_batches, unsigned n_segs, unsigned long long* n_vals,
                                      unsigned long long* n_ids, unsigned char* same_class, unsigned* max_bytes,
                                      unsigned long long* run_hits) {
    const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_batches) return;
    const unsigned f0 = batch_first[b];
    const unsigned nsb = (b + 1 < n_batches ? batch_first[b + 1] : n_segs) - f0;
    const unsigned k = key2s[f0], d = key2_deg(k), n = key2_rows(k);
    const unsigned per_seg = key2_run(k) ? 1u : d;  // ids stored per segment
    const unsigned long long nv = (unsigned long long)nsb * n * (d + 1u);
    bool same = true;
    const unsigned c0 = seg_cls[segid_s[f0]];
    for (unsigned i = 1; i < nsb; ++i) same = same && seg_cls[segid_s[f0 + i]] == c0;
    n_vals[b] = nv;
    same_class[b] = same ? 1 : 0;
    n_ids[b] = same ? per_seg : (unsigned long long)nsb * per_seg;
    atomicMax(max_bytes, (unsigned)(8u * nv + 4u * nsb * per_seg + 16u));
    if (key2_run(k)) atomicAdd(run_hits, (unsigned long long)nsb * n * d);
}

__global__ void cls_batch_desc_kernel(const unsigned* __restrict__ key2s, const unsigned* __restrict__ batch_first,
                                      const unsigned long long* __restrict__ val_off,
                                      const unsigned long long* __restrict__ id_off,
                                      const unsigned char* __restrict__ same_class, unsigned n_batches, unsigned n_segs,
                                      BatchDesc* desc) {
    const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_batches) return;
    const unsigned f0 = batch_first[b];
    const unsigned nsb = (b + 1 < n_batches ? batch_first[b + 1] : n_segs) - f0;
    const unsigned k = key2s[f0], d = key2_deg(k), n = key2_rows(k);
    BatchDesc o;
    o.w0 = val_off[b] | ((unsigned long long)d << 48);
    o.w1 = id_off[b] | ((unsigned long long)n << 40) | ((unsigned long long)nsb << 48) |
           ((unsigned long long)cfg_of_deg(d) << 56) | ((unsigned long long)same_class[b] << 60) |
           ((unsigned long long)key2_run(k) << 61);
    desc[b] = o;
}

__device__ __forceinline__ unsigned long long staged_before(const unsigned long long* __restrict__ val_off,
                                                            const unsigned long long* __restrict__ id_off, unsigned long long b) {
    return 8ull * val_off[b] + 4ull * id_off[b] + 16ull * b;  // bytes staged before batch b
}

// one thread: out = {first batch of configuration kTailCfg (n_batches if none), bytes staged before it}.  Batches are
// sorted by degree, so the kTailCfg batches are a suffix of the stream.
__global__ void cls_tail_start_kernel(const unsigned* __restrict__ key2s, const unsigned* __restrict__ batch_first,
                                      const unsigned long long* __restrict__ val_off, const unsigned long long* __restrict__ id_off,
                                      unsigned n_batches, unsigned long long* out) {
    unsigned lo = 0, hi = n_batches;
    while (lo < hi) {
        const unsigned mid = (lo + hi) >> 1;
        if (cfg_of_deg(key2_deg(key2s[batch_first[mid]])) != kTailCfg) lo = mid + 1;
        else hi = mid;
    }
    out[0] = lo;
    out[1] = staged_before(val_off, id_off, lo);
}

// tiles of the batch range [b_lo, b_hi): bound[k] = first batch b in it with staged_before(b) >= base + k W, where
// base = staged_before(b_lo); bound[n_raw] = b_hi
__global__ void cls_tile_bounds_kernel(const unsigned long long* __restrict__ val_off,
                                       const unsigned long long* __restrict__ id_off, unsigned b_lo, unsigned b_hi,
                                       unsigned long long base, unsigned long long W, unsigned long long n_raw,
                                       unsigned long long* bound) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k > n_raw) return;
    if (k == n_raw) { bound[k] = b_hi; return; }
    const unsigned long long target = base + k * W;
    unsigned long long lo = b_lo, hi = b_hi;  // val_off / id_off have n_batches + 1 entries
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (staged_before(val_off, id_off, mid) < target) lo = mid + 1;
        else hi = mid;
    }
    bound[k] = lo;
}

__global__ void cls_tile_rec_kernel(const unsigned long long* __restrict__ bound, const unsigned long long* __restrict__ val_off,
                                    const unsigned long long* __restrict__ id_off, unsigned long long n_bounds, TileRec* rec) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_bounds) return;
    const unsigned long long b = bound[k];
    rec[k].val_begin = val_off[b];
    rec[k].id_begin = id_off[b];
    rec[k].batch_begin = b;
}

// one warp per batch: ids of segment gi, column c at id_off + c nsb + gi (or id_off + c for a one-class batch); a run
// batch stores column 0 only (the segments' firsts)
__global__ void cls_fill_ids_kernel(const unsigned long long* __restrict__ rp, const int* __restrict__ sid_abs,
                                    const BatchDesc* __restrict__ desc, const unsigned* __restrict__ batch_first,
                                    const unsigned* __restrict__ fseg_first, const unsigned* __restrict__ rows,
                                    unsigned n_batches, int* ids) {
    const unsigned lane = threadIdx.x & 31u;
    for (unsigned long long b = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n_batches;
         b += ((unsigned long long)gridDim.x * blockDim.x) >> 5) {
        const BatchDesc bd = desc[b];
        const unsigned nsb = (unsigned)(bd.w1 >> 48) & 255u, same = (unsigned)(bd.w1 >> 60) & 1u;
        const unsigned d = (bd.w1 >> 61) & 1u ? 1u : (unsigned)(bd.w0 >> 48);  // ids stored per segment
        const unsigned long long ioff = bd.w1 & kOff40;
        const unsigned f0 = batch_first[b];
        const unsigned ns = same ? 1u : nsb;
        for (unsigned idx = lane; idx < ns * d; idx += 32) {
            const unsigned gi = idx % ns, c = idx / ns;
            const unsigned row = rows[fseg_first[f0 + gi]];
            ids[ioff + idx] = sid_abs[rp[row] + c];
        }
    }
}

// one warp per batch: value (segment gi, row r, column c) at val_off + (r (d + 1) + c) nsb + gi; column d is the row's ncpv
__global__ void cls_fill_vals_kernel(const unsigned long long* __restrict__ rp, const double* __restrict__ conprb,
                                     const double* __restrict__ ncpv, const BatchDesc* __restrict__ desc,
                                     const unsigned* __restrict__ batch_first, const unsigned* __restrict__ fseg_first,
                                     const unsigned* __restrict__ rows, unsigned n_batches, double* vals) {
    const unsigned lane = threadIdx.x & 31u;
    for (unsigned long long b = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n_batches;
         b += ((unsigned long long)gridDim.x * blockDim.x) >> 5) {
        const BatchDesc bd = desc[b];
        const unsigned d = (unsigned)(bd.w0 >> 48), n = (unsigned)(bd.w1 >> 40) & 255u, nsb = (unsigned)(bd.w1 >> 48) & 255u;
        double* out = vals + (bd.w0 & kOff48);
        const unsigned f0 = batch_first[b];
        // lane -> (gi, column): consecutive lanes write consecutive doubles, each lane walks its own source row
        const unsigned per_row = nsb * (d + 1u);  // elements of one row-step of the batch
        for (unsigned r = 0; r < n; ++r)
            for (unsigned idx = lane; idx < per_row; idx += 32) {
                const unsigned gi = idx % nsb, c = idx / nsb;
                const unsigned row = rows[fseg_first[f0 + gi] + r];
                out[(unsigned long long)r * per_row + idx] = c < d ? conprb[rp[row] + c] : ncpv[row];
            }
    }
}

__global__ void cls_gather_u32_kernel(const unsigned* __restrict__ src, const unsigned* __restrict__ idx, unsigned n, unsigned* out) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[idx[i]];
}

__global__ void cls_long_rows_kernel(const unsigned long long* __restrict__ keys_sorted, const unsigned* __restrict__ rows,
                                     unsigned n_rows, unsigned n_long, unsigned* out) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_long) out[i] = rows[n_rows + i];
}

// ------------------------------------------------------------------------------------------------------------------
// the E-step kernel
// ------------------------------------------------------------------------------------------------------------------
struct ClassArgs {
    const double* vals;
    const int* ids;
    const BatchDesc* desc;
    const TileRec* tile;
    unsigned n_tiles;
    const double* theta;
    double* count;
    const int* done_flag;
    unsigned* claim;             // {next tile to claim, CTAs done}: 0 between launches (the last CTA to finish resets it)
    unsigned long long* cta_ns;  // per-CTA busy time of this launch (globaltimer, ns): load-balance evidence; or nullptr
    unsigned long long* wait_ns;  // profiling only (else nullptr): kWaitRecord entries per CTA {consumer ns blocked on
                                  // data, producer ns blocked on a free stage, consumer warps, SM cycles of the consumer
                                  // warps in the phases front, rows, flush and hand-over, SM cycles the CTA was busy}
};

struct StageDesc {  // written by the producer when it issues a tile
    unsigned long long val_base;  // index of the first staged value (val_begin rounded down to 16 B)
    unsigned long long id_base;
    unsigned o_ids, o_desc;       // byte offsets of the id and descriptor slices inside the stage
    unsigned n_batches;           // kNoTile: no tile left, the consumers leave
    unsigned first_batch_mod;     // (global index of the tile's first batch) % consumer warps
};
constexpr unsigned kNoTile = 0xffffffffu;

template <int W>
struct ClassSmem {
    __align__(128) unsigned char stage[kStages][kStageBytes];
    unsigned long long full_bar[kStages];   // producer -> consumers: the stage's bytes have landed (complete_tx)
    unsigned long long empty_bar[kStages];  // consumers -> producer: every consumer warp is done with the stage
    StageDesc sd[kStages];
    double red[W + 1];
    unsigned long long wait[2];
    unsigned long long phase[4];  // profiling: cycles per phase, summed over the consumer warps
};

__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// t0, t1: the tile's records, loaded by the caller before it waits for the stage
__device__ __forceinline__ void issue_class_tile(const ClassArgs& a, const TileRec& t0, const TileRec& t1, unsigned char* st,
                                                 unsigned long long* bar, StageDesc& sd, unsigned n_consumers) {
    const unsigned long long vb = t0.val_begin & ~1ull, ib = t0.id_begin & ~3ull;
    const unsigned b_val = round16((unsigned)(t1.val_begin - vb) * 8u);
    const unsigned b_ids = round16((unsigned)(t1.id_begin - ib) * 4u);
    const unsigned nb = (unsigned)(t1.batch_begin - t0.batch_begin);
    const unsigned b_desc = nb * 16u;
    sd.val_base = vb;
    sd.id_base = ib;
    sd.o_ids = b_val;
    sd.o_desc = b_val + b_ids;
    sd.n_batches = nb;
    sd.first_batch_mod = (unsigned)(t0.batch_begin % n_consumers);
    mbar_expect_tx(bar, b_val + b_ids + b_desc);
    // The layout is read once per launch and is far larger than L2; theta and the count vector (a few MB) are read
    // and added to by every batch.  With the default priority the stream's lines push those out and the theta gather
    // and the reductions queue behind HBM; evict_first keeps them resident (C3: 3.39 -> 3.20 ms per round).
    const unsigned long long once = l2_evict_first();
    if (b_val) bulk_load_hint(st, a.vals + vb, b_val, bar, once);
    if (b_ids) bulk_load_hint(st + b_val, a.ids + ib, b_ids, bar, once);
    bulk_load_hint(st + b_val + b_ids, a.desc + t0.batch_begin, b_desc, bar, once);
}

#ifdef RB_CLASS_DEBUG
__device__ int g_dbg_flag = 0;
#endif

template <int G>
__device__ __forceinline__ double seg_sum(double v) {  // lanes of a segment are strided by P = 32 / G
#pragma unroll
    for (int o = 32 / G; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <>
__device__ __forceinline__ double seg_sum<1>(double v) { return v; }

// 1 / x for a normal, positive x: hardware seed (about 20 bits) + two Newton steps.  The row sums are >= 1e-300 and
// far below overflow, so none of the special cases of a full fp64 division can occur; the result is within one ulp
// of the correctly rounded reciprocal (the weights f / sum are formed as f * (1 / sum): EM.cpp:231 divides instead,
// parity is checked at 1e-9 relative on theta).
__device__ __forceinline__ double fast_rcp(double x) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    double e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    return r;
}

// U rows of a batch at once.  ROWS_OK: all U rows exist (main loop) - otherwise rows >= n_left are idle (remainder).
// TAIL: the rows have more than G * S = 128 columns (configuration kTailCfg); the rest are walked from shared memory.
template <int G, int S, int U, bool ROWS_OK, bool TAIL>
__device__ __forceinline__ void batch_rows(const double* __restrict__ cr, unsigned row_stride, unsigned n_left,
                                           const double (&th)[S], const bool (&col_ok)[S], const unsigned (&coff)[S],
                                           double (&acc)[S], unsigned g, unsigned w, unsigned nsb, unsigned d,
                                           const int* __restrict__ bi, unsigned ids_stride, unsigned ids_gi, bool seg_ok,
                                           const double* __restrict__ theta, double* count, double& acc0) {
    double x[U][S], part[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const bool row_ok = ROWS_OK || (unsigned)u < n_left;
#pragma unroll
        for (int q = 0; q < S; ++q) {
            double c = 0.0;  // idle lanes must not read: the bytes behind a batch are arbitrary (possibly NaN patterns)
            if (col_ok[q] && row_ok) c = cr[u * row_stride + coff[q]];
            x[u][q] = th[q] * c;
            if (x[u][q] < kEpsilon) x[u][q] = 0.0;
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        if (S == 4) part[u] = (x[u][0] + x[u][1]) + (x[u][2] + x[u][3]);
        else part[u] = (x[u][0] + x[u][1]) + x[u][2];
    }
    if (TAIL && seg_ok) {  // columns beyond G * S (rows with more than 127 hits): not kept in registers
        for (unsigned c = g + G * S; c < w; c += G) {
            const double thc = __ldg(theta + (c < d ? bi[c * ids_stride + ids_gi] : 0));
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (ROWS_OK || (unsigned)u < n_left) {
                    double f = thc * cr[u * row_stride + c * nsb];
                    if (f < kEpsilon) f = 0.0;
                    part[u] += f;
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) part[u] = seg_sum<G>(part[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const double inv = part[u] >= kEpsilon ? fast_rcp(part[u]) : 0.0;  // idle rows: part = 0 -> inv = 0
#pragma unroll
        for (int q = 0; q < S; ++q) acc[q] += x[u][q] * inv;
        if (TAIL && seg_ok && (ROWS_OK || (unsigned)u < n_left)) {
            for (unsigned c = g + G * S; c < w; c += G) {
                const int tt = c < d ? bi[c * ids_stride + ids_gi] : 0;
                double f = __ldg(theta + tt) * cr[u * row_stride + c * nsb];
                if (f < kEpsilon) f = 0.0;
                const double wgt = f * inv;
                if (tt == 0) acc0 += wgt;
                else if (wgt != 0.0) red_add_f64(count + tt, wgt);
            }
        }
    }
}

// One batch: P = 32 / G segments of n rows x (d + 1) columns; lane = g * P + gi owns columns g, g + G, ... of segment
// gi: ids and theta are loaded once, the rows are walked U at a time (instruction-level parallelism across the
// load -> product -> row sum -> reciprocal chain), the normalised weights are summed per lane and leave as ONE
// reduction per transcript and segment.  The noise column's sum stays in the thread (count[0] is flushed per CTA).
// run: the batch stores its segments' firsts, column c < d is transcript first + c.
// PROF: ph[] takes the cycles from t0 (read by the caller before it loaded the batch's descriptor) to theta usable,
// of the row walk and of the flush.
template <int G, int S, int U, bool TAIL, bool PROF>
__device__ __forceinline__ double process_batch(const double* __restrict__ bv, const int* __restrict__ bi, unsigned d,
                                                unsigned n, unsigned nsb, bool same, bool run, const double* __restrict__ theta,
                                                double* count, unsigned lane, long long t0, long long (&ph)[kPhases]) {
    constexpr unsigned P = 32 / G;
    const unsigned gi = lane % P, g = lane / P;
    const bool seg_ok = gi < nsb;
    const unsigned w = d + 1u;
    const unsigned ids_stride = same ? 1u : nsb, ids_gi = same ? 0u : gi;
    const int first = (run && seg_ok) ? bi[ids_gi] : 0;
    int t[S];
    double th[S], acc[S];
    bool col_ok[S];
    unsigned coff[S];
#pragma unroll
    for (int q = 0; q < S; ++q) {
        const unsigned c = g + G * q;
        col_ok[q] = seg_ok && c < w;
        coff[q] = c * nsb;
        // column d is the noise entry: transcript 0
        t[q] = (seg_ok && c < d) ? (run ? first + (int)c : bi[c * ids_stride + ids_gi]) : 0;
    }
#pragma unroll
    for (int q = 0; q < S; ++q) {
        th[q] = col_ok[q] ? __ldg(theta + t[q]) : 0.0;
        acc[q] = 0.0;
    }
    if (PROF) {
        const long long t1 = clk_after(S == 4 ? (th[0] + th[1]) + (th[2] + th[3]) : (th[0] + th[1]) + th[2]);
        ph[kPhFront] += t1 - t0;
        t0 = t1;
    }
    const double* con = bv + gi;  // value (r, c) of this lane's segment at con[(r w + c) nsb]
    const unsigned row_stride = w * nsb;
    double acc0 = 0.0;
    unsigned r = 0;
    for (; r + U <= n; r += U)
        batch_rows<G, S, U, true, TAIL>(con + (unsigned long long)r * row_stride, row_stride, U, th, col_ok, coff, acc, g, w, nsb, d,
                                        bi, ids_stride, ids_gi, seg_ok, theta, count, acc0);
    if (U > 1 && r < n)
        batch_rows<G, S, U, false, TAIL>(con + (unsigned long long)r * row_stride, row_stride, n - r, th, col_ok, coff, acc, g, w,
                                         nsb, d, bi, ids_stride, ids_gi, seg_ok, theta, count, acc0);
    if (PROF) {
        const long long t1 = clk_after(acc[0]);
        ph[kPhRows] += t1 - t0;
        t0 = t1;
    }
    if (same && P > 1) {  // every segment of the batch adds to the same transcripts: fold them first
#pragma unroll
        for (int q = 0; q < S; ++q) {
#pragma unroll
            for (int o = 1; o < (int)P; o <<= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
            if (gi != 0) acc[q] = 0.0;
        }
    }
#pragma unroll
    for (int q = 0; q < S; ++q) {
        if (t[q] == 0) acc0 += acc[q];  // noise column (or an idle slot, whose sum is 0)
        else if (acc[q] != 0.0) red_add_f64(count + t[q], acc[q]);
    }
    if (PROF) ph[kPhFlush] += clk() - t0;
    return acc0;
}

// W consumer warps + 1 producer warp per CTA (one CTA per SM).  The producer's lane 0 keeps the 3-stage ring full:
// it claims the next tile from a counter in global memory, waits on a stage's "empty" barrier (one arrival per
// consumer warp) and issues the tile's bulk copies on its "full" barrier; when no tile is left it hands the consumers
// a stage without tile instead.  Consumers wait for "full", take the batches whose global index is congruent to their
// warp index (batches of a tile have similar shape, so the static assignment is balanced and costs no atomics), arrive
// on "empty".
// PROF: wait and phase accounting into a.wait_ns (profiling on); the kernel without it has no timer reads.
// TAIL: the tiles hold only configuration-kTailCfg batches (rows with more than 127 hits), else none of them.
template <int W, int U, bool TAIL, bool PROF>
__global__ void __launch_bounds__((W + 1) * 32, 1) estep_class_kernel(const ClassArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ClassSmem<W>& sm = *reinterpret_cast<ClassSmem<W>*>(smem_raw);
    if (*a.done_flag) return;
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    unsigned long long t_start = 0;
    long long c_start = 0;
    if (tid == 0) {
        t_start = global_ns();
        if (PROF) c_start = clk();
        if (PROF)
            for (int i = 0; i < kPhases; ++i) sm.phase[i] = 0;
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&sm.full_bar[s], 1);
            mbar_init(&sm.empty_bar[s], W);
        }
        sm.wait[0] = sm.wait[1] = 0;
        fence_barrier_init();
    }
    __syncthreads();
    unsigned long long waited = 0;
    unsigned long long* const wacc = PROF ? &waited : nullptr;
    long long ph[kPhases] = {0, 0, 0, 0};
    // Tiles are claimed in stream order by whichever CTA has a stage to fill next.  Neighbouring tiles hold batches of
    // similar shape (the stream is sorted by degree), so every CTA sees the same mix, and a CTA whose tiles go slower
    // (SMs do not all see the same memory latency) takes fewer of them: the CTAs finish within about a tile of each
    // other, where a fixed stride over the grid left the launch waiting on the slowest CTA.
    double acc0 = 0.0;
    if (warp == W) {
        if (lane == 0) {
            unsigned k = atomicAdd(&a.claim[0], 1u);
            for (unsigned it = 0;; ++it) {
                const int s = it % kStages;
                const bool last = k >= a.n_tiles;
                TileRec t0{}, t1{};
                if (!last) {
                    t0 = a.tile[k];  // in flight while the stage is still in use
                    t1 = a.tile[k + 1];
                }
                const unsigned k_next = last ? k : atomicAdd(&a.claim[0], 1u);  // likewise
                if (it >= (unsigned)kStages) {
                    mbar_wait_timed(&sm.empty_bar[s], ((it / kStages) - 1u) & 1u, wacc);
                    fence_proxy_async();  // the consumers' generic-proxy reads precede the async-proxy refill
                }
                if (last) {
                    sm.sd[s].n_batches = kNoTile;
                    mbar_arrive(&sm.full_bar[s]);
                    break;
                }
                issue_class_tile(a, t0, t1, sm.stage[s], &sm.full_bar[s], sm.sd[s], W);
                k = k_next;
            }
        }
    } else {
        long long tc = PROF ? clk() : 0;
        for (unsigned it = 0;; ++it) {
            const int s = it % kStages;
            mbar_wait_timed(&sm.full_bar[s], (it / kStages) & 1u, wacc);
            if (PROF) ph[kPhHandOver] += clk() - tc;
            const unsigned char* st = sm.stage[s];
            const StageDesc sd = sm.sd[s];
            if (sd.n_batches == kNoTile) break;
            const double* s_val = reinterpret_cast<const double*>(st);
            const int* s_ids = reinterpret_cast<const int*>(st + sd.o_ids);
            const BatchDesc* s_desc = reinterpret_cast<const BatchDesc*>(st + sd.o_desc);
            for (unsigned b = (warp + W - sd.first_batch_mod) % W; b < sd.n_batches; b += W) {
                if (PROF) tc = clk();
                const BatchDesc bd = s_desc[b];
                const unsigned d = (unsigned)(bd.w0 >> 48), n = (unsigned)(bd.w1 >> 40) & 255u, nsb = (unsigned)(bd.w1 >> 48) & 255u;
                const unsigned cfg = (unsigned)(bd.w1 >> 56) & 15u;
                const bool same = (bd.w1 >> 60) & 1ull, run = (bd.w1 >> 61) & 1ull;
                const double* bv = s_val + ((bd.w0 & kOff48) - sd.val_base);
                const int* bi = s_ids + ((bd.w1 & kOff40) - sd.id_base);
#ifdef RB_CLASS_DEBUG
                {
                    const unsigned long long vo = (bd.w0 & kOff48) - sd.val_base;
                    const unsigned long long nv = (unsigned long long)nsb * n * (d + 1);
                    const bool bad = cfg != cfg_of_deg(d) || nsb == 0 || nsb > 32u / group_of_deg(d) || n == 0 ||
                                     (vo + nv) * 8ull > sd.o_ids || sd.n_batches > 4096;
                    bool nan = false;
                    if (!bad)
                        for (unsigned long long i = lane; i < nv; i += 32) nan = nan || (bv[i] != bv[i]) || bv[i] < 0.0 || bv[i] > 1.0;
                    if ((bad || __any_sync(0xffffffffu, nan)) && lane == 0 && atomicCAS(&g_dbg_flag, 0, 1) == 0)
                        printf("CLASSDBG cta %u warp %u it %u s %d b %u/%u bad %d | d %u n %u nsb %u cfg %u vo %llu nv %llu o_ids %u o_desc %u "
                               "val_base %llu id_base %llu fbm %u | w0 %llx w1 %llx\n",
                               blockIdx.x, warp, it, s, b, sd.n_batches, (int)bad, d, n, nsb, cfg, vo, nv, sd.o_ids, sd.o_desc, sd.val_base,
                               sd.id_base, sd.first_batch_mod, bd.w0, bd.w1);
                }
#endif
                if constexpr (TAIL) {
                    acc0 += process_batch<32, 4, U, true, PROF>(bv, bi, d, n, nsb, same, false, a.theta, a.count, lane, tc, ph);
                } else {
                    switch (cfg) {
                        case 0: acc0 += process_batch<1, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 1: acc0 += process_batch<1, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 2: acc0 += process_batch<2, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 3: acc0 += process_batch<2, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 4: acc0 += process_batch<4, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 5: acc0 += process_batch<4, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 6: acc0 += process_batch<8, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 7: acc0 += process_batch<8, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 8: acc0 += process_batch<16, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 9: acc0 += process_batch<16, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        case 10: acc0 += process_batch<32, 3, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                        default: acc0 += process_batch<32, 4, U, false, PROF>(bv, bi, d, n, nsb, same, run, a.theta, a.count, lane, tc, ph); break;
                    }
                }
            }
            if (PROF) tc = clk();
            __syncwarp();  // every lane's reads of the stage are done before lane 0 releases it
            if (lane == 0) mbar_arrive(&sm.empty_bar[s]);
        }
    }
    // count[0] partials: warp shuffle -> shared -> one reduction per CTA
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    if (lane == 0) sm.red[warp] = acc0;
    if (PROF && lane == 0) {
        atomicAdd(&sm.wait[warp == W ? 1 : 0], waited);
        if (warp < W)
            for (int i = 0; i < kPhases; ++i) atomicAdd(&sm.phase[i], (unsigned long long)ph[i]);
    }
    __syncthreads();
    if (warp == 0) {
        double v = 0.0;
        for (unsigned i = lane; i < (unsigned)W; i += 32) v += sm.red[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && v != 0.0) red_add_f64(a.count, v);
        if (lane == 0 && atomicAdd(&a.claim[1], 1u) == gridDim.x - 1u) {  // every CTA has made its last claim
            a.claim[0] = 0;
            a.claim[1] = 0;
        }
        if (lane == 0) {
            if (a.cta_ns) a.cta_ns[blockIdx.x] = global_ns() - t_start;
            if (PROF) {
                unsigned long long* o = a.wait_ns + (size_t)kWaitRecord * blockIdx.x;
                o[0] = sm.wait[0];
                o[1] = sm.wait[1];
                o[2] = W;
                for (int i = 0; i < kPhases; ++i) o[3 + i] = sm.phase[i];
                o[3 + kPhases] = (unsigned long long)(clk() - c_start);
            }
        }
    }
}

// rows with more than kLongDeg hits: one CTA per row on the CSR stream
__global__ void __launch_bounds__(256) estep_long_rows_kernel(const unsigned long long* __restrict__ rp, const int* __restrict__ sid_abs,
                                                              const double* __restrict__ conprb, const double* __restrict__ ncpv,
                                                              const unsigned* __restrict__ long_rows, unsigned n_long,
                                                              const double* __restrict__ theta, double* count,
                                                              const int* done_flag) {
    __shared__ double red[8];
    __shared__ double s_inv;
    if (*done_flag) return;
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const double theta0 = __ldg(theta);
    for (unsigned i = blockIdx.x; i < n_long; i += gridDim.x) {
        const unsigned row = long_rows[i];
        const unsigned long long b = rp[row], e = rp[row + 1];
        double part = 0.0;
        for (unsigned long long j = b + tid; j < e; j += blockDim.x) {
            double f = __ldg(theta + sid_abs[j]) * conprb[j];
            if (f < kEpsilon) f = 0.0;
            part += f;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if (lane == 0) red[warp] = part;
        __syncthreads();
        if (tid == 0) {
            double f0 = theta0 * ncpv[row];
            if (f0 < kEpsilon) f0 = 0.0;
            double sum = f0;
            for (int w = 0; w < 8; ++w) sum += red[w];
            const double inv = sum >= kEpsilon ? 1.0 / sum : 0.0;
            s_inv = inv;
            if (f0 * inv != 0.0) red_add_f64(count, f0 * inv);
        }
        __syncthreads();
        const double inv = s_inv;
        for (unsigned long long j = b + tid; j < e; j += blockDim.x) {
            const int t = sid_abs[j];
            double f = __ldg(theta + t) * conprb[j];
            if (f < kEpsilon) f = 0.0;
            if (f * inv != 0.0) red_add_f64(count + t, f * inv);
        }
        __syncthreads();
    }
}

// ---- host helpers --------------------------------------------------------------------------------------------------
struct Scratch {  // returns its buffers (to the context's block cache) on every exit path
    rsem_b200_ctx* ctx;
    std::vector<void*> p;
    explicit Scratch(rsem_b200_ctx* c) : ctx(c) {}
    ~Scratch() {
        for (void* q : p) block_free(ctx, q);
    }
    template <class T>
    cudaError_t alloc(T** out, size_t n) {
        void* q = nullptr;
        cudaError_t e = block_alloc(ctx, &q, (n ? n : 1) * sizeof(T));
        if (e == cudaSuccess) p.push_back(q);
        *out = static_cast<T*>(q);
        return e;
    }
    void release(void* q) {
        for (auto& x : p)
            if (x == q) { block_free(ctx, q); x = nullptr; }
    }
    void keep(void* q) {  // ownership moves to the context
        for (auto& x : p)
            if (x == q) x = nullptr;
    }
};

inline unsigned blocks_for(unsigned long long n, unsigned per_block) { return (unsigned)((n + per_block - 1) / per_block); }

struct PhaseTimer {  // RSEM_B200_CLASS_TIMING=1: wall-clock per build phase on stderr (syncs the stream; diagnostics only)
    cudaStream_t st;
    bool on;
    double t0;
    static double now() {
        timespec ts;
        clock_gettime(CLOCK_MONOTONIC, &ts);
        return ts.tv_sec + 1e-9 * ts.tv_nsec;
    }
    explicit PhaseTimer(cudaStream_t s) : st(s), on(getenv("RSEM_B200_CLASS_TIMING") != nullptr), t0(0) {
        if (on) { cudaStreamSynchronize(st); t0 = now(); }
    }
    void mark(const char* what) {
        if (!on) return;
        cudaStreamSynchronize(st);
        const double t = now();
        fprintf(stderr, "rsem_b200 class layout: %8.3f ms  %s\n", (t - t0) * 1e3, what);
        t0 = t;
    }
};

}  // namespace

void class_free(rsem_b200_ctx* ctx) {
    ClassLayout& L = ctx->cls;
    block_free(ctx, L.vals); block_free(ctx, L.ids); block_free(ctx, L.desc); block_free(ctx, L.tile); block_free(ctx, L.batch_first);
    block_free(ctx, L.fseg_first); block_free(ctx, L.rows); block_free(ctx, L.long_rows); block_free(ctx, L.cta_ns);
    block_free(ctx, L.wait_ns); block_free(ctx, L.claim);
    L = ClassLayout{};
}

// Builds the class directory of the context's hit matrix (row_ptr, sid_abs).  Returns 0 and leaves L.built == false
// when the matrix is outside what the layout supports (>= 2^32 rows); the caller then keeps the row kernel.
int class_build(rsem_b200_ctx* ctx) {
    ClassLayout& L = ctx->cls;
    class_free(ctx);
    const unsigned long long N = ctx->N;
    if (N == 0 || N >= 0xfffffff0ull || ctx->H >= (1ull << 40)) return 0;
    cudaStream_t st = ctx->stream;
    const unsigned long long* rp = reinterpret_cast<const unsigned long long*>(ctx->row_ptr);
    const int* sid_abs = ctx->sid_abs;
    unsigned R = 8;
    if (const char* e = getenv("RSEM_B200_CLASS_ROWS")) {  // tuning knob: rows per segment
        const int v = atoi(e);
        if (v >= 1 && v <= 255) R = (unsigned)v;
    }
    Scratch sc(ctx);
    PhaseTimer pt(st);
    // ---- 1. row keys, sorted
    unsigned long long *keys = nullptr, *keys_s = nullptr;
    unsigned *rows0 = nullptr, *rows_s = nullptr, *d_cnt = nullptr;
    RB_CUDA(sc.alloc(&keys, N));
    RB_CUDA(sc.alloc(&keys_s, N));
    RB_CUDA(sc.alloc(&rows0, N));
    RB_CUDA(sc.alloc(&rows_s, N));
    RB_CUDA(sc.alloc(&d_cnt, 4));
    RB_CUDA(cudaMemsetAsync(d_cnt, 0, 4 * sizeof(unsigned), st));
    cls_row_key_kernel<<<blocks_for(N * 8, 256), 256, 0, st>>>(rp, sid_abs, N, keys, rows0, d_cnt);
    RB_CUDA(cudaGetLastError());
    size_t tmp_bytes = 0, need = 0;
    void* tmp = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, need, keys, keys_s, rows0, rows_s, (long long)N, 0, 60, st);
    tmp_bytes = need;
    cub::DeviceScan::InclusiveScan(nullptr, need, (unsigned*)nullptr, (unsigned*)nullptr, MaxOp(), (long long)N, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::DeviceScan::InclusiveSum(nullptr, need, (unsigned*)nullptr, (unsigned*)nullptr, (long long)N, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::DeviceScan::ExclusiveSum(nullptr, need, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (long long)N + 1, st);
    tmp_bytes = std::max(tmp_bytes, need);
    RB_CUDA(sc.alloc(reinterpret_cast<unsigned char**>(&tmp), tmp_bytes));
    need = tmp_bytes;
    RB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, need, keys, keys_s, rows0, rows_s, (long long)N, 0, 60, st));
    unsigned h_cnt[4] = {0, 0, 0, 0};
    RB_CUDA(cudaMemcpyAsync(h_cnt, d_cnt, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    const unsigned n_long = h_cnt[0];
    const unsigned n_rows = (unsigned)(N - n_long);
    pt.mark("row keys + sort by (degree, hash)");
    sc.release(keys); keys = nullptr;
    sc.release(rows0); rows0 = nullptr;
    L.n_long = n_long;
    L.n_rows = n_rows;
    if (n_long) {
        RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.long_rows), (size_t)n_long * sizeof(unsigned)));
        cls_long_rows_kernel<<<blocks_for(n_long, 256), 256, 0, st>>>(keys_s, rows_s, n_rows, n_long, L.long_rows);
        RB_CUDA(cudaGetLastError());
    }
    if (n_rows == 0) {
        sc.keep(rows_s);
        L.rows = rows_s;
        L.built = true;
        RB_CUDA(cudaStreamSynchronize(st));
        return 0;
    }
    // ---- 2. classes -> segments
    unsigned *a32 = nullptr, *b32 = nullptr, *c32 = nullptr;  // n_rows-sized work arrays
    RB_CUDA(sc.alloc(&a32, n_rows));
    RB_CUDA(sc.alloc(&b32, n_rows));
    RB_CUDA(sc.alloc(&c32, n_rows));
    cls_new_class_kernel<<<blocks_for((unsigned long long)n_rows * 8, 256), 256, 0, st>>>(rp, sid_abs, keys_s, rows_s, n_rows, a32);
    RB_CUDA(cudaGetLastError());
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::InclusiveScan(tmp, need, a32, b32, MaxOp(), (long long)n_rows, st));  // b32 = class start
    cls_seg_flag_kernel<<<blocks_for(n_rows, 256), 256, 0, st>>>(keys_s, b32, n_rows, R, a32);    // a32 = segment flag
    RB_CUDA(cudaGetLastError());
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::InclusiveSum(tmp, need, a32, c32, (long long)n_rows, st));            // c32 = segment idx + 1
    unsigned n_segs = 0;
    RB_CUDA(cudaMemcpyAsync(&n_segs, c32 + (n_rows - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    unsigned *seg_first = nullptr, *seg_cls = nullptr, *key2 = nullptr, *key2_s = nullptr, *segid = nullptr, *segid_s = nullptr;
    RB_CUDA(sc.alloc(&seg_first, n_segs));
    RB_CUDA(sc.alloc(&seg_cls, n_segs));
    cls_seg_scatter_kernel<<<blocks_for(n_rows, 256), 256, 0, st>>>(keys_s, b32, a32, c32, n_rows, seg_first, seg_cls);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(cudaStreamSynchronize(st));
    sc.release(a32); sc.release(b32); sc.release(c32);
    a32 = b32 = c32 = nullptr;
    pt.mark("classes verified, segments cut");
    // ---- 3. segments ordered by (degree, rows), batches of 32 / G equal segments
    RB_CUDA(sc.alloc(&key2, n_segs));
    RB_CUDA(sc.alloc(&key2_s, n_segs));
    RB_CUDA(sc.alloc(&segid, n_segs));
    RB_CUDA(sc.alloc(&segid_s, n_segs));
    cls_seg_key_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(rp, sid_abs, keys_s, rows_s, seg_first, n_segs, n_rows, key2, segid);
    RB_CUDA(cudaGetLastError());
    {
        size_t need2 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, need2, key2, key2_s, segid, segid_s, (long long)n_segs, 0, kKey2Bits, st);
        if (need2 > tmp_bytes) {
            sc.release(tmp);
            RB_CUDA(sc.alloc(reinterpret_cast<unsigned char**>(&tmp), need2));
            tmp_bytes = need2;
        }
        need2 = tmp_bytes;
        RB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, need2, key2, key2_s, segid, segid_s, (long long)n_segs, 0, kKey2Bits, st));
    }
    RB_CUDA(cudaStreamSynchronize(st));
    sc.release(keys_s); keys_s = nullptr;
    unsigned *s_a = key2, *s_b = segid, *s_c = nullptr;  // reuse as work arrays (their contents are sorted copies now)
    RB_CUDA(sc.alloc(&s_c, n_segs));
    cls_run_start_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(key2_s, n_segs, s_a);
    RB_CUDA(cudaGetLastError());
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::InclusiveScan(tmp, need, s_a, s_b, MaxOp(), (long long)n_segs, st));  // s_b = run start
    cls_batch_flag_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(key2_s, s_b, n_segs, s_a);      // s_a = batch flag
    RB_CUDA(cudaGetLastError());
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::InclusiveSum(tmp, need, s_a, s_c, (long long)n_segs, st));            // s_c = batch idx + 1
    unsigned n_batches = 0;
    RB_CUDA(cudaMemcpyAsync(&n_batches, s_c + (n_segs - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.batch_first), (size_t)n_batches * sizeof(unsigned)));
    cls_batch_scatter_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(s_a, s_c, n_segs, L.batch_first);
    RB_CUDA(cudaGetLastError());
    unsigned long long *n_vals = nullptr, *n_ids = nullptr, *val_off = nullptr, *id_off = nullptr;
    unsigned long long* run_hits = nullptr;
    unsigned char* same_class = nullptr;
    RB_CUDA(sc.alloc(&run_hits, 1));
    RB_CUDA(cudaMemsetAsync(run_hits, 0, sizeof(unsigned long long), st));
    RB_CUDA(sc.alloc(&n_vals, (size_t)n_batches + 1));
    RB_CUDA(sc.alloc(&n_ids, (size_t)n_batches + 1));
    RB_CUDA(sc.alloc(&val_off, (size_t)n_batches + 1));
    RB_CUDA(sc.alloc(&id_off, (size_t)n_batches + 1));
    RB_CUDA(sc.alloc(&same_class, n_batches));
    RB_CUDA(cudaMemsetAsync(n_vals + n_batches, 0, sizeof(unsigned long long), st));
    RB_CUDA(cudaMemsetAsync(n_ids + n_batches, 0, sizeof(unsigned long long), st));
    cls_batch_size_kernel<<<blocks_for(n_batches, 256), 256, 0, st>>>(key2_s, L.batch_first, segid_s, seg_cls, n_batches, n_segs,
                                                                     n_vals, n_ids, same_class, d_cnt + 1, run_hits);
    RB_CUDA(cudaGetLastError());
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, need, n_vals, val_off, (long long)n_batches + 1, st));
    need = tmp_bytes;
    RB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, need, n_ids, id_off, (long long)n_batches + 1, st));
    unsigned long long totals[3] = {0, 0, 0};
    RB_CUDA(cudaMemcpyAsync(&totals[0], val_off + n_batches, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaMemcpyAsync(&totals[1], id_off + n_batches, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaMemcpyAsync(&totals[2], run_hits, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaMemcpyAsync(h_cnt, d_cnt, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    const unsigned max_batch_bytes = h_cnt[1];
    if (max_batch_bytes + 256u > kStageBytes) {
        set_error("class layout: a batch does not fit a shared-memory stage (internal limit)");
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    pt.mark("segments sorted, batches formed");
    L.n_vals = totals[0];
    L.n_ids = totals[1];
    L.n_run_hits = totals[2];
    L.n_segs = n_segs;
    L.n_batches = n_batches;
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.desc), ((size_t)n_batches + 1) * sizeof(BatchDesc)));
    cls_batch_desc_kernel<<<blocks_for(n_batches, 256), 256, 0, st>>>(key2_s, L.batch_first, val_off, id_off, same_class, n_batches,
                                                                     n_segs, static_cast<BatchDesc*>(L.desc));
    RB_CUDA(cudaGetLastError());
    // ---- 4. tiles: contiguous batch ranges of <= kStageBytes staged bytes.  The kTailCfg batches start a tile of
    // their own: tiles [0, n_tiles_main) have none of them, the rest nothing else.
    {
        unsigned long long* d_cut = nullptr;
        RB_CUDA(sc.alloc(&d_cut, 2));
        cls_tail_start_kernel<<<1, 1, 0, st>>>(key2_s, L.batch_first, val_off, id_off, n_batches, d_cut);
        RB_CUDA(cudaGetLastError());
        unsigned long long cut[2] = {0, 0};  // first kTailCfg batch, bytes staged before it
        RB_CUDA(cudaMemcpyAsync(cut, d_cut, sizeof(cut), cudaMemcpyDeviceToHost, st));
        RB_CUDA(cudaStreamSynchronize(st));
        const unsigned long long W = kStageBytes - max_batch_bytes - 128u;
        const unsigned long long total = 8ull * totals[0] + 4ull * totals[1] + 16ull * n_batches;
        const unsigned b_tail = (unsigned)cut[0];
        const unsigned piece_b[3] = {0u, b_tail, n_batches};
        const unsigned long long piece_bytes[3] = {0ull, cut[1], total};
        unsigned long long n_raw[2] = {0, 0};
        for (int p = 0; p < 2; ++p)
            if (piece_b[p] < piece_b[p + 1]) n_raw[p] = (piece_bytes[p + 1] - piece_bytes[p]) / W + 1;
        unsigned long long *bound = nullptr, *bound_u = nullptr;
        unsigned long long* d_n = nullptr;
        RB_CUDA(sc.alloc(&bound, n_raw[0] + n_raw[1] + 2));
        RB_CUDA(sc.alloc(&bound_u, n_raw[0] + n_raw[1] + 2));
        RB_CUDA(sc.alloc(&d_n, 1));
        size_t need3 = 0;
        cub::DeviceSelect::Unique(nullptr, need3, bound, bound_u, d_n, (long long)std::max(n_raw[0], n_raw[1]) + 1, st);
        if (need3 > tmp_bytes) {
            sc.release(tmp);
            RB_CUDA(sc.alloc(reinterpret_cast<unsigned char**>(&tmp), need3));
            tmp_bytes = need3;
        }
        // each piece's bounds run from its first batch to its last + 1; the main piece's last bound is the tail
        // piece's first, so the tail piece's bounds overwrite it
        unsigned long long n_bounds = 0;
        L.n_tiles_main = 0;
        for (int p = 0; p < 2; ++p) {
            if (!n_raw[p]) continue;
            cls_tile_bounds_kernel<<<blocks_for(n_raw[p] + 1, 256), 256, 0, st>>>(val_off, id_off, piece_b[p], piece_b[p + 1],
                                                                                  piece_bytes[p], W, n_raw[p], bound);
            RB_CUDA(cudaGetLastError());
            const unsigned long long at = n_bounds ? n_bounds - 1 : 0;
            need3 = tmp_bytes;
            RB_CUDA(cub::DeviceSelect::Unique(tmp, need3, bound, bound_u + at, d_n, (long long)n_raw[p] + 1, st));
            unsigned long long n = 0;
            RB_CUDA(cudaMemcpyAsync(&n, d_n, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            RB_CUDA(cudaStreamSynchronize(st));
            n_bounds = at + n;
            if (p == 0) L.n_tiles_main = (unsigned)(n_bounds - 1);
        }
        L.n_tiles = (unsigned)(n_bounds - 1);
        RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.tile), n_bounds * sizeof(TileRec)));
        cls_tile_rec_kernel<<<blocks_for(n_bounds, 256), 256, 0, st>>>(bound_u, val_off, id_off, n_bounds, static_cast<TileRec*>(L.tile));
        RB_CUDA(cudaGetLastError());
    }
    // ---- 5. what the value gather needs later: first sorted position of every segment in final order + the row order
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.fseg_first), (size_t)n_segs * sizeof(unsigned)));
    cls_gather_u32_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(seg_first, segid_s, n_segs, L.fseg_first);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.ids), ((size_t)L.n_ids + 64) * sizeof(int)));
    RB_CUDA(cudaMemsetAsync(L.ids + L.n_ids, 0, 64 * sizeof(int), st));
    cls_fill_ids_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(rp, sid_abs, static_cast<const BatchDesc*>(L.desc), L.batch_first,
                                                          L.fseg_first, rows_s, n_batches, L.ids);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.vals), ((size_t)L.n_vals + 32) * sizeof(double)));
    RB_CUDA(cudaMemsetAsync(L.vals + L.n_vals, 0, 32 * sizeof(double), st));
    RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.claim), 2 * sizeof(unsigned)));
    RB_CUDA(cudaMemsetAsync(L.claim, 0, 2 * sizeof(unsigned), st));
    RB_CUDA(cudaStreamSynchronize(st));
    pt.mark("tiles, descriptors, ids");
    sc.keep(rows_s);
    L.rows = rows_s;
    L.R = R;
    L.built = true;
    L.vals_epoch = 0;
    ctx->launches += 20;
    return 0;
}

int class_fill_vals(rsem_b200_ctx* ctx) {
    ClassLayout& L = ctx->cls;
    if (!L.built) return 0;
    PhaseTimer pt(ctx->stream);
    if (L.n_batches) {
        cls_fill_vals_kernel<<<ctx->sm_count * 16, 256, 0, ctx->stream>>>(
            reinterpret_cast<const unsigned long long*>(ctx->row_ptr), ctx->conprb, ctx->ncpv,
            static_cast<const BatchDesc*>(L.desc), L.batch_first, L.fseg_first, L.rows, L.n_batches, L.vals);
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    pt.mark("value stream gathered from conprb / ncpv");
    L.vals_epoch = ctx->conprb_epoch;
    return 0;
}

int class_launch_estep(rsem_b200_ctx* ctx) {
    ClassLayout& L = ctx->cls;
    ClassArgs a;
    a.vals = L.vals;
    a.ids = L.ids;
    a.desc = static_cast<const BatchDesc*>(L.desc);
    a.theta = ctx->theta;
    a.count = ctx->k2_target;
    a.done_flag = ctx->done_flag;
    a.claim = L.claim;
    L.last_grid = 0;
    if (L.n_tiles_main) {  // rows of <= 127 hits; the per-CTA busy and wait times come from this launch
        a.tile = static_cast<const TileRec*>(L.tile);
        a.n_tiles = L.n_tiles_main;
        if (!L.cta_ns) {
            RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.cta_ns), (size_t)ctx->sm_count * sizeof(unsigned long long)));
        }
        a.cta_ns = reinterpret_cast<unsigned long long*>(L.cta_ns);
        if (ctx->profiling && !L.wait_ns) {
            RB_CUDA(block_alloc(ctx, reinterpret_cast<void**>(&L.wait_ns), (size_t)ctx->sm_count * kWaitRecord * sizeof(unsigned long long)));
        }
        a.wait_ns = ctx->profiling ? reinterpret_cast<unsigned long long*>(L.wait_ns) : nullptr;
        L.last_profiled = ctx->profiling;
        const unsigned grid = std::min<unsigned>((unsigned)ctx->sm_count, a.n_tiles);
        L.last_grid = grid;
        // 15 consumer warps x 2 rows in flight per lane (98 registers, no spills).  Without the tail code more warps
        // fit and hide more of a batch's latency (ids -> theta gather -> values -> row sums); 18 warps are no faster.
        // Measured on H100 80GB HBM3 at 700 W, ms per round, median of 3 alternating runs in one process:
        //   consumer warps x rows:  11x2   11x3   11x4   14x2   14x3   14x4   15x2   15x3   15x4   18x2   18x3   18x4
        //   C3                      3.505  3.460  3.446  3.389  3.396  3.410  3.389  3.394  3.397  3.387  3.483  3.697
        //   C2                      0.373  0.373  0.376  0.371  0.372  0.374  0.372  0.372  0.374  0.370  0.371  0.405
        //   C5                      8.167  8.292  8.589  7.952  8.044  8.294  7.813  7.977  8.187  7.818  7.895  8.302
        // (18 x 3 and 18 x 4 spill; the sweep predates the evict_first priority of the copies, which took 15 x 2 at C3
        // from 3.39 to 3.20 ms.)  The previous kernel, with the tail code in every configuration (11 x 2, 167
        // registers), in a separate process on the same card: C3 3.519, C2 0.373, C5 8.579.
        // Re-swept with evict_first and run batches (same card, one process per run, 3 alternating runs, ms per round):
        //   consumer warps x rows:  14x2                 15x2                 18x2
        //   C3                      3.039 3.040 3.036    3.028 3.041 3.029    3.030 3.031 3.032
        //   C2                      0.357 0.356 0.352    0.353 0.360 0.351    0.356 0.353 0.354
        //   C5                      7.561 7.562 7.540    7.428 7.421 7.398    7.216 7.213 7.202
        // 18 warps tie at C3 and C2 and are 2.7 % faster at C5 (88 registers), but their profiling instantiation
        // spills (16 bytes), so 15 stays: the profiled launch (tools/k2_anatomy.py) has to run the configuration
        // that is timed, or its phase shares describe another kernel, and no instantiation may spill.
        constexpr int W = 15, U = 2;
        const size_t smem = sizeof(ClassSmem<W>);
        if (ctx->profiling) {
            RB_CUDA(cudaFuncSetAttribute(estep_class_kernel<W, U, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            estep_class_kernel<W, U, false, true><<<grid, (W + 1) * 32, smem, ctx->stream>>>(a);
        } else {
            RB_CUDA(cudaFuncSetAttribute(estep_class_kernel<W, U, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            estep_class_kernel<W, U, false, false><<<grid, (W + 1) * 32, smem, ctx->stream>>>(a);
        }
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    if (L.n_tiles > L.n_tiles_main) {  // rows of 128..kLongDeg hits (none at C2 / C3, a third of the hits at C5)
        a.tile = static_cast<const TileRec*>(L.tile) + L.n_tiles_main;
        a.n_tiles = L.n_tiles - L.n_tiles_main;
        a.cta_ns = nullptr;
        a.wait_ns = nullptr;
        const unsigned grid = std::min<unsigned>((unsigned)ctx->sm_count, a.n_tiles);
        constexpr int W = 11, U = 2;
        const size_t smem = sizeof(ClassSmem<W>);
        RB_CUDA(cudaFuncSetAttribute(estep_class_kernel<W, U, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        estep_class_kernel<W, U, true, false><<<grid, (W + 1) * 32, smem, ctx->stream>>>(a);
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    if (L.n_long) {
        estep_long_rows_kernel<<<std::min<unsigned>(L.n_long, (unsigned)ctx->sm_count * 4), 256, 0, ctx->stream>>>(
            reinterpret_cast<const unsigned long long*>(ctx->row_ptr), ctx->sid_abs, ctx->conprb, ctx->ncpv, L.long_rows, L.n_long,
            ctx->theta, ctx->k2_target, ctx->done_flag);
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    return 0;
}

}  // namespace rsem_b200
