// K5 / K6: collapsed Gibbs sampler over read -> transcript assignments (rsem-run-gibbs).
//
// Reference: /root/reference/Gibbs.cpp:265-353 (chain), sampling.h:50-65 (categorical draw by
// binary search on a cumulative array), boost mt19937 + uniform_01 (u = x * 2^-32, one draw per
// read per sweep).  "Same seed, same draws" is part of the contract, so everything that decides a
// draw keeps the reference's arithmetic exactly:
//   * the cumulative array is a LEFT-TO-RIGHT fp64 running sum of (count + alpha) * conprb;
//   * the drawn index is the number of entries <= u * total, which equals the reference's binary
//     search because the array is non-decreasing;
//   * MT19937 is regenerated 624 words at a time by the chain's warp (three dependent phases of the
//     standard recurrence), tempering is done at extraction.
//
// Two kernels: gibbs_chain_kernel (serial cross-check: one CTA per chain, warp 0 walks the reads in order - the loads,
// the (count + alpha) * conprb products and the index count are spread over its 32 lanes, only the running sum is
// serial) and gibbs_parallel_kernel (the product path: connected components of the read x transcript graph walked
// concurrently by 16-lane groups, exact through a fixed-point iteration over the reads that change their noise
// membership; see the block comment "Component-parallel EXACT sampler" below).  In both, the chain's CTA(s) also do the
// O(M) per-sample work (count vector dump, theta -> polish -> TPM/FPKM, accumulation).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {
namespace {

constexpr int kGibbsThreads = 256;
constexpr int kRowCap = 2048;  // cumulative-array slots in shared memory; longer rows use global scratch

struct GibbsArgs {
    unsigned long long N1;
    const unsigned long long* row_ptr;
    const int* sid;
    const double* conprb;
    int M, burnin, gap, n_genes;
    const int* chain_samples;
    const unsigned* chain_seeds;
    const long long* chain_cv_offset;  // first sample slot of each chain in count_vectors
    double n0, totc;
    const int* init_counts;
    const double* alpha;
    const double* eel;
    const double* mw;
    const int* gene_start;
    // per-chain state / outputs
    int* counts;          // n_chains * (M + 1)
    int* z;               // n_chains * N1
    double* scratch;      // n_chains * max_len (only when max_len > kRowCap)
    unsigned max_len;
    int* count_vectors;   // total_samples * (M + 1)
    double* acc;          // n_chains * (4 * (M + 1) + n_genes): sum_c, sum_c2, sum_tpm, sum_fpkm, sum_gene_c2
    double* theta_tmp;    // n_chains * 2 * (M + 1)  (theta / fpkm scratch)
    int* err_flag;
};

struct MtState {
    unsigned mt[624];
};

__device__ __forceinline__ unsigned mt_twist(unsigned a, unsigned b, unsigned c) {
    const unsigned y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

// regenerate all 624 words with the 32 lanes of the calling warp
__device__ void mt_regenerate(MtState& s, int lane) {
    // phase 1: k in [0, 227) needs old[k], old[k+1], old[k+397]
    // phase 2: k in [227, 454) needs old[k], old[k+1], new[k-227]
    // phase 3: k in [454, 623) needs old[k], old[k+1], new[k-227]
    // phase 4: k = 623 needs old[623], new[0], new[396]
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        const int lo = 227 * p, hi = p == 2 ? 623 : 227 * (p + 1);
        unsigned v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = lo + lane + 32 * j;
            const int k3 = k + 397 >= 624 ? k + 397 - 624 : k + 397;
            v[j] = k < hi ? mt_twist(s.mt[k], s.mt[k + 1], s.mt[k3]) : 0u;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = lo + lane + 32 * j;
            if (k < hi) s.mt[k] = v[j];
        }
        __syncwarp();
    }
    if (lane == 0) s.mt[623] = mt_twist(s.mt[623], s.mt[0], s.mt[396]);
    __syncwarp();
}

__device__ __forceinline__ unsigned mt_temper(unsigned y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// block-wide sum of doubles (all threads call)
__device__ double block_sum(double v, double* sh) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
    return t;
}

// one draw for read i by warp 0 (all 32 lanes call).  use_counts = false for the initial state.
__device__ __forceinline__ void draw_read(const GibbsArgs& a, unsigned long long i, bool use_counts, int* counts, int* z,
                                          double* s_arr, double* g_arr, MtState& mt, int& mt_idx, int lane) {
    const unsigned long long fr = a.row_ptr[i], to = a.row_ptr[i + 1];
    const unsigned len = (unsigned)(to - fr);
    double* arr = len <= kRowCap ? s_arr : g_arr;
    if (use_counts) {
        if (lane == 0) --counts[z[i]];
        __syncwarp();
    }
    for (unsigned k = lane; k < len; k += 32) {
        const int t = a.sid[fr + k];
        const double c = a.conprb[fr + k];
        arr[k] = use_counts ? ((double)counts[t] + a.alpha[t]) * c : c;
    }
    __syncwarp();
    if (lane == 0) {  // left-to-right running sum (Gibbs.cpp:286-288, 301-308)
        double run = 0.0;
        for (unsigned k = 0; k < len; ++k) {
            run = k ? arr[k] + run : arr[k];
            arr[k] = run;
        }
    }
    if (mt_idx >= 624) {
        mt_regenerate(mt, lane);
        mt_idx = 0;
    }
    __syncwarp();
    const double u = mt_temper(mt.mt[mt_idx]) * (1.0 / 4294967296.0);
    ++mt_idx;
    const double prb = u * arr[len - 1];
    int below = 0;
    for (unsigned k = lane; k < len; k += 32) below += arr[k] <= prb;
    for (int o = 16; o > 0; o >>= 1) below += __shfl_xor_sync(0xffffffffu, below, o);
    if (below >= (int)len) {  // reference: assert(l < len), sampling.h:62
        *a.err_flag = 3;
        below = (int)len - 1;
    }
    __syncwarp();
    if (lane == 0) {
        const int zn = a.sid[fr + below];
        z[i] = zn;
        ++counts[zn];
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kGibbsThreads) gibbs_chain_kernel(const GibbsArgs a) {
    __shared__ MtState mt;
    __shared__ double s_arr[kRowCap];
    __shared__ double sh_red[kGibbsThreads / 32];
    const int chain = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int M1 = a.M + 1;
    int* counts = a.counts + (size_t)chain * M1;
    int* z = a.z + (size_t)chain * a.N1;
    double* g_arr = a.scratch ? a.scratch + (size_t)chain * a.max_len : nullptr;
    double* acc = a.acc + (size_t)chain * (4 * (size_t)M1 + a.n_genes);
    double* theta = a.theta_tmp + (size_t)chain * 2 * M1;
    double* fpkm = theta + M1;
    const int n_samples = a.chain_samples[chain];
    int* cv = a.count_vectors + a.chain_cv_offset[chain] * M1;

    for (int i = tid; i < M1; i += blockDim.x) counts[i] = a.init_counts[i] + (i == 0 ? (int)a.n0 : 0);
    if (tid == 0) {  // init_genrand (boost mt19937 seeding)
        mt.mt[0] = a.chain_seeds[chain];
        for (int k = 1; k < 624; ++k) mt.mt[k] = 1812433253u * (mt.mt[k - 1] ^ (mt.mt[k - 1] >> 30)) + (unsigned)k;
    }
    __syncthreads();
    int mt_idx = 624;

    if (warp == 0)
        for (unsigned long long i = 0; i < a.N1; ++i) draw_read(a, i, false, counts, z, s_arr, g_arr, mt, mt_idx, lane);
    __syncthreads();

    const int chainlen = 1 + (n_samples - 1) * a.gap;
    int kept = 0;
    for (int round = 1; round <= a.burnin + chainlen; ++round) {
        if (warp == 0)
            for (unsigned long long i = 0; i < a.N1; ++i) draw_read(a, i, true, counts, z, s_arr, g_arr, mt, mt_idx, lane);
        __syncthreads();
        if (round > a.burnin && (round - a.burnin - 1) % a.gap == 0) {  // Gibbs.cpp:313-346
            // count vector + theta = (c + alpha) / totc, zero for omitted; polishTheta; TPM / FPKM
            double part = 0.0;
            for (int i = tid; i < M1; i += blockDim.x) {
                const int c = counts[i];
                cv[(size_t)kept * M1 + i] = c;
                double th = c < 0 ? 0.0 : ((double)c + a.alpha[i]) / a.totc;
                if (i > 0 && (a.mw[i] < kEpsilon || a.eel[i] < kEpsilon)) th = 0.0;
                else th = th / a.mw[i];
                theta[i] = th;
                part += th;
            }
            const double tsum = block_sum(part, sh_red);
            part = 0.0;
            for (int i = tid; i < M1; i += blockDim.x) {
                const double th = theta[i] / tsum;
                theta[i] = th;
                if (i > 0 && a.eel[i] >= kEpsilon) part += th;
            }
            double denom = block_sum(part, sh_red);
            if (denom < kEpsilon) denom = 1.0;
            part = 0.0;
            for (int i = tid; i < M1; i += blockDim.x) {
                const double f = (i > 0 && a.eel[i] >= kEpsilon) ? (theta[i] / denom) * 1e9 / a.eel[i] : 0.0;
                fpkm[i] = f;
                part += f;
            }
            double fsum = block_sum(part, sh_red);
            if (fsum < kEpsilon) fsum = 1.0;
            for (int i = tid; i < M1; i += blockDim.x) {
                const double c = (double)counts[i];
                acc[i] += c;
                acc[M1 + i] += c * c;
                acc[2 * (size_t)M1 + i] += i > 0 ? fpkm[i] / fsum * 1e6 : 0.0;
                acc[3 * (size_t)M1 + i] += fpkm[i];
            }
            for (int gi = tid; gi < a.n_genes; gi += blockDim.x) {
                double c = 0.0;
                for (int j = a.gene_start[gi]; j < a.gene_start[gi + 1]; ++j) c += counts[j];
                acc[4 * (size_t)M1 + gi] += c * c;
            }
            ++kept;
            __syncthreads();
        }
    }
}

// ================================================================================================
// Component-parallel EXACT sampler.
//
// Within a chain every draw reads the counts the previous reads wrote, so a sweep is sequential - but only
// between reads that share a candidate transcript.  Reads of different connected components of the
// read x transcript graph (noise transcript 0 excluded) touch disjoint counts and commute exactly.  The only
// global coupling is the noise count c0 = counts[0], which enters every row that has a noise entry.
//
//   * Static, once per upload (gibbs_prepare, host): connected components (union-find over transcripts); the reads
//     grouped by component in read order ("segments", longest first); rows re-laid in that slot order.
//   * A sweep of a chain: every segment is walked by ONE group of 16 lanes in read order with the live counts of its
//     component (component-private: registers for components of < 32 transcripts, L2 otherwise).  The noise count read i must see is c0(i) = c0 at the start of the
//     sweep + (#reads before i that joined the noise transcript) - (#reads before i that left it).  Those "flips" are
//     rare, so the sweep is a fixed-point iteration over the SET of flips:
//         pass k walks all segments with c0(i) taken from the flips recorded by pass k - 1 (none for k = 0) and
//         records its own flips (two bitmaps over read positions);
//         if pass k recorded exactly the flips it was given, every read saw the noise count the sequential sweep
//         would have shown it - by induction over the read positions the draws ARE the sequential draws - done;
//         otherwise the counts are restored from the copy taken at the start of the sweep and pass k + 1 runs.
//     A draw changes with c0 only when u * total falls into the sliver by which the noise entry moved, so the
//     iteration ends after two passes almost always (one when no read changed its noise membership).
//   * The i-th uniform of sweep s is output s * N1 + i of the chain's MT19937.  A dedicated generator CTA per chain
//     runs one sweep ahead of the workers (624-word regenerations, 227 threads wide, ping-pong state in shared memory).
//   * A chain is served by `ctas_per_chain` worker CTAs + 1 generator CTA, all co-resident (cooperative launch); the
//     workers meet at a per-chain barrier in global memory a handful of times per sweep (not once per block of reads);
//     chains never synchronise with each other.
// ================================================================================================
constexpr int kPThreads = 256;

struct ChainSync {
    unsigned count, gen;        // barrier among the chain's worker CTAs
    unsigned u_ready;           // generator -> workers: uniforms of sweeps < u_ready are complete
    unsigned sweeps_done;       // workers -> generator: sweeps < sweeps_done no longer need their uniform buffer
    unsigned changed;           // some flip word differs between the pass's input and output sets
    unsigned next_seg;          // next component to be claimed in the current pass
    int err;
    unsigned passes;            // diagnostics: passes run over all sweeps
    unsigned long long prof[4]; // clock64 totals of worker CTA 0: wait for uniforms, passes, barriers + bookkeeping, per-sample work
};

struct PArgs {
    unsigned long long N1;
    const int* order;                   // read id of slot q (component by component, read order inside)
    const unsigned long long* p_off;    // N1 + 1 entry offsets of the slots, rows stored in slot order
    const int* p_sid;
    const double* p_con;
    const int* seg_start;               // n_segs + 1 slot offsets
    const int* seg_ntr;                 // transcripts of the component (0: the segment is a read with only the noise entry)
    const int* seg_tid_off;             // offset of the component's sorted transcript ids in comp_tids
    const int* comp_tids;
    int n_segs;
    int fast_rows;                      // converged walk: lean code path for rows of register-resident components
    int M, burnin, gap, n_genes, n_chains, ctas_per_chain, chain_base;
    const int* chain_samples;
    const unsigned* chain_seeds;
    const long long* chain_cv_offset;
    double n0, totc;
    const int* init_counts;
    const double* alpha;
    const double* eel;
    const double* mw;
    const int* gene_start;
    int* counts;           // n_chains * (M + 1)
    int* counts_start;     // n_chains * (M + 1): copy taken at the start of a sweep
    int* z;                // n_chains * 2 * N1, indexed by SLOT; [sweep parity]
    unsigned* ubuf;        // n_chains * 2 * N1 raw MT outputs; [sweep parity]
    unsigned* flips;       // n_chains * 4 * W words: [set 0 / 1][joined / left]
    int* pre;              // n_chains * W: net flips in the words before w inside its CTA slice
    int* slice_tot;        // n_chains * ctas_per_chain: net flips of every CTA slice
    unsigned n_words;      // W = ceil(N1 / 32)
    ChainSync* sync;       // n_chains
    int* count_vectors;
    double* acc;
    double* theta_tmp;
};

__device__ __forceinline__ int ld_cg(const int* p) { return __ldcg(p); }
__device__ __forceinline__ void st_cg(int* p, int v) { __stcg(p, v); }

__device__ void chain_barrier(ChainSync* s, unsigned n_ctas) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned gen = *((volatile unsigned*)&s->gen);
        if (atomicAdd(&s->count, 1u) == n_ctas - 1) {
            s->count = 0;
            __threadfence();
            atomicAdd(&s->gen, 1u);
        } else {
            while (*((volatile unsigned*)&s->gen) == gen) {}
        }
        __threadfence();
    }
    __syncthreads();
}

// ---- generator CTA: the chain's MT19937, at most one sweep ahead of the workers ----------------------------------------
// The state ping-pongs between two shared-memory arrays: a phase reads only words that are already final, so one
// __syncthreads per phase (four per 624 outputs) is all the ordering it needs.  Output g of the stream belongs to
// sweep g / N1, position g % N1, and goes to that sweep's buffer ([sweep parity]).
__device__ void generator_loop(const PArgs& a, ChainSync* sy, unsigned* ubuf, unsigned n_sweeps, unsigned seed) {
    __shared__ unsigned st[2][624];
    const unsigned tid = threadIdx.x;
    if (tid == 0) {  // init_genrand (boost mt19937 seeding)
        st[0][0] = seed;
        for (int k = 1; k < 624; ++k) st[0][k] = 1812433253u * (st[0][k - 1] ^ (st[0][k - 1] >> 30)) + (unsigned)k;
    }
    __syncthreads();
    int cur = 0;
    const unsigned long long total = (unsigned long long)n_sweeps * a.N1;
    unsigned acquired = 1;   // sweeps 0 and 1 own fresh buffers
    unsigned published = 0;
    for (unsigned long long g0 = 0; g0 < total; g0 += 624) {
        const unsigned* o = st[cur];
        unsigned* n = st[cur ^ 1];
        if (tid < 227) n[tid] = mt_twist(o[tid], o[tid + 1], o[tid + 397]);                 // k in [0, 227)
        __syncthreads();
        if (tid < 227) n[227 + tid] = mt_twist(o[227 + tid], o[228 + tid], n[tid]);         // k in [227, 454)
        __syncthreads();
        if (tid < 169) n[454 + tid] = mt_twist(o[454 + tid], o[455 + tid], n[227 + tid]);   // k in [454, 623)
        __syncthreads();
        if (tid == 0) n[623] = mt_twist(o[623], n[0], n[396]);                              // k = 623
        __syncthreads();
        cur ^= 1;
        const unsigned take = (unsigned)min((unsigned long long)624, total - g0);
        const unsigned sweep_hi = (unsigned)((g0 + take - 1) / a.N1);
        if (sweep_hi > acquired) {   // first touch of a recycled buffer: the sweep two before must be finished
            if (tid == 0) {
                while (*((volatile unsigned*)&sy->sweeps_done) + 1 < sweep_hi) {}
                __threadfence();
            }
            __syncthreads();
            acquired = sweep_hi;
        }
        const unsigned sweep_lo = (unsigned)(g0 / a.N1);
        const unsigned long long pos_lo = g0 - (unsigned long long)sweep_lo * a.N1;
        for (unsigned k = tid; k < take; k += kPThreads) {
            unsigned long long pos = pos_lo + k;
            unsigned sw = sweep_lo;
            while (pos >= a.N1) { pos -= a.N1; ++sw; }   // at most one step unless N1 < 624
            __stcg(ubuf + (size_t)(sw & 1u) * a.N1 + pos, mt_temper(st[cur][k]));
        }
        const unsigned complete = (unsigned)((g0 + take) / a.N1);   // sweeps whose last output has been written
        if (complete > published) {
            __threadfence();
            __syncthreads();
            if (tid == 0) atomicExch(&sy->u_ready, complete);
            published = complete;
        }
    }
}

// A group of kGL = 16 lanes walks the reads of one component (segment) in order; the lanes hold the entries of the
// current row.  What is sequential in the reference stays sequential - reads in order, the left-to-right fp64 running
// sum of a row - everything else is spread over the lanes:
//   * the next row (header, ids, conprb) is loaded while the current one is drawn;
//   * REG components (<= 31 transcripts: a gene family) keep their counts in REGISTERS - lane j owns local ids j and
//     j + 16, a lookup is a 16-wide shuffle, an update a predicated add - so the dependent chain of a read contains no
//     memory round trip at all; their rows and assignments are stored as local ids (0 = noise);
//   * larger components read and write their counts in L2 (component-private, ld.cg / st.cg);
//   * the running sum is formed by every lane for its own prefix from the row's products in shared memory, in entry
//     order (bit-identical to arr[k] += arr[k - 1], Gibbs.cpp:286-288, 301-308); the drawn index is the number of
//     entries <= u * total (sampling.h:50-65 on a non-decreasing array).
constexpr int kGL = 16;

struct alignas(16) GroupSmem {
    double v[kGL];         // products of the current chunk (lanes past the chunk's end store 0.0)
    double w[2][2 * kGL];  // fast path of the converged walk: products of rows r, r + 1 (double-buffered: one __syncwarp per row)
    double al[2 * kGL];    // REG: alpha of the component's local ids
};

struct RowHead {
    int i;                 // read id (position in the sweep order)
    unsigned len;
    unsigned long long off;
    int zo;                // assignment left by the previous sweep
    unsigned raw;          // MT19937 output of this read in this sweep
    int t;                 // this lane's entry of the first chunk (id or local id)
    double c;
};

__device__ __forceinline__ void load_head(const PArgs& a, const int* z_prev, const unsigned* u, int q, bool use_counts, int gl, RowHead& r) {
    r.i = a.order[q];
    r.off = a.p_off[q];
    r.len = (unsigned)(a.p_off[q + 1] - r.off);
    r.zo = use_counts ? ld_cg(z_prev + q) : 0;
    r.raw = __ldcg(u + r.i);
    const bool in = (unsigned)gl < r.len;
    r.t = in ? a.p_sid[r.off + gl] : -1;
    r.c = in ? a.p_con[r.off + gl] : 0.0;
}

// prefix sums of the chunk's products in entry order; lane gl gets arr[base + gl]; returns the running sum after the chunk.
// The sum starts from `carry` (0.0 for the first chunk: 0.0 + x == x exactly, so arr[0] is the first product itself as in
// Gibbs.cpp:286-288) and lanes past the end of the chunk contribute +0.0, which leaves a non-negative sum unchanged: every
// lane can run the same unrolled sequence of 16-byte shared-memory loads and predicated adds.
__device__ __forceinline__ double chunk_running_sum(GroupSmem& sm, unsigned gmask, int gl, double v, unsigned base, unsigned n_valid,
                                                    double carry, double& arr) {
    (void)base;
    sm.v[gl] = v;
    __syncwarp(gmask);
    double run = carry;
    const double2* p = reinterpret_cast<const double2*>(sm.v);
#pragma unroll
    for (int j = 0; j < kGL; j += 4) {
        if (j < (int)n_valid) {   // group-uniform
            const double2 a = p[j / 2], b = p[j / 2 + 1];
            if (j <= gl) run = __dadd_rn(a.x, run);
            if (j + 1 <= gl) run = __dadd_rn(a.y, run);
            if (j + 2 <= gl) run = __dadd_rn(b.x, run);
            if (j + 3 <= gl) run = __dadd_rn(b.y, run);
        }
    }
    arr = run;
    const double last = __shfl_sync(gmask, run, (int)n_valid - 1, kGL);
    __syncwarp(gmask);
    return last;
}

// One draw: the sequential part of a row.  `cur` is the row (first chunk of entries in cur.t / cur.c), c0 the noise count it
// must see.  REG components keep their counts in cnt0 / cnt1 (local ids gl and gl + 16).
template <bool REG>
__device__ __forceinline__ void process_row(const PArgs& a, const RowHead& cur, int q, int c0, bool use_counts, int* counts, int* z_cur,
                                            unsigned* f_out, unsigned W, int* err, GroupSmem& sm, unsigned gmask, int gl, int& cnt0, int& cnt1) {
    const double uni = cur.raw * (1.0 / 4294967296.0);
    const int zo = cur.zo;
    // value of one entry: (count + alpha) * conprb with the read's own assignment taken out (Gibbs.cpp:298-306)
    auto entry_value = [&](int t, double c, bool valid, int& cnt_seen) -> double {
        int cnt = c0;
        double al;
        if (REG) {
            const int src = valid ? (t & (kGL - 1)) : 0;
            const int x0 = __shfl_sync(gmask, cnt0, src, kGL), x1 = __shfl_sync(gmask, cnt1, src, kGL);
            if (valid && t != 0) cnt = t < kGL ? x0 : x1;
            al = sm.al[valid ? t : 0];
        } else {
            if (valid && t != 0) cnt = ld_cg(counts + t);
            al = a.alpha[valid ? t : 0];
        }
        if (valid && t == zo) cnt -= 1;
        cnt_seen = cnt;
        if (!valid) return 0.0;
        return use_counts ? __dmul_rn(__dadd_rn((double)cnt, al), c) : c;
    };
    int znew;
    if (cur.len <= (unsigned)kGL) {
        const bool valid = (unsigned)gl < cur.len;
        int seen;
        const double v = entry_value(cur.t, cur.c, valid, seen);
        double arr;
        const double total = chunk_running_sum(sm, gmask, gl, v, 0u, cur.len, 0.0, arr);
        const double prb = __dmul_rn(uni, total);
        int l = __popc(__ballot_sync(gmask, valid && arr <= prb));
        if (l >= (int)cur.len) { *err = 3; l = (int)cur.len - 1; }   // reference: assert(l < len), sampling.h:62
        znew = __shfl_sync(gmask, cur.t, l, kGL);
        if (!REG && use_counts && znew != zo) {   // the lanes that hold the two entries know the counts they saw
            if (valid && zo != 0 && cur.t == zo) st_cg(counts + zo, seen);
            if (gl == l && znew != 0) st_cg(counts + znew, seen + 1);
        }
        if (!REG && !use_counts && gl == l && znew != 0) st_cg(counts + znew, ld_cg(counts + znew) + 1);
    } else {
        // rows longer than a group: one pass for the total, one for the index
        double carry = 0.0;
        for (unsigned base = 0; base < cur.len; base += kGL) {
            const unsigned k = base + gl, nv = min((unsigned)kGL, cur.len - base);
            const bool valid = k < cur.len;
            const int t = valid ? a.p_sid[cur.off + k] : -1;
            const double c = valid ? a.p_con[cur.off + k] : 0.0;
            int seen;
            double arr;
            carry = chunk_running_sum(sm, gmask, gl, entry_value(t, c, valid, seen), base, nv, carry, arr);
        }
        const double prb = __dmul_rn(uni, carry);
        int l = 0;
        carry = 0.0;
        znew = -1;
        for (unsigned base = 0; base < cur.len; base += kGL) {
            const unsigned k = base + gl, nv = min((unsigned)kGL, cur.len - base);
            const bool valid = k < cur.len;
            const int t = valid ? a.p_sid[cur.off + k] : -1;
            const double c = valid ? a.p_con[cur.off + k] : 0.0;
            int seen;
            double arr;
            carry = chunk_running_sum(sm, gmask, gl, entry_value(t, c, valid, seen), base, nv, carry, arr);
            const int below = __popc(__ballot_sync(gmask, valid && arr <= prb));
            l += below;
            if (znew < 0 && below < (int)nv) znew = __shfl_sync(gmask, t, below, kGL);   // first entry with arr > prb (group-uniform branch)
        }
        if (znew < 0) {   // reference: assert(l < len)
            *err = 3;
            znew = a.p_sid[cur.off + cur.len - 1];
        }
        if (!REG && gl == 0) {
            if (use_counts) {
                if (znew != zo) {
                    if (zo != 0) st_cg(counts + zo, ld_cg(counts + zo) - 1);
                    if (znew != 0) st_cg(counts + znew, ld_cg(counts + znew) + 1);
                }
            } else if (znew != 0) st_cg(counts + znew, ld_cg(counts + znew) + 1);
        }
    }
    if (REG && znew != zo) {   // owners of the two local ids adjust their registers
        if (use_counts && zo != 0 && (zo & (kGL - 1)) == gl) { if (zo < kGL) --cnt0; else --cnt1; }
        if (znew != 0 && (znew & (kGL - 1)) == gl) { if (znew < kGL) ++cnt0; else ++cnt1; }
    }
    if (gl == 0) {
        st_cg(z_cur + q, znew);
        if (use_counts) {
            if (zo != 0 && znew == 0) atomicOr(f_out + ((unsigned)cur.i >> 5), 1u << ((unsigned)cur.i & 31u));
            if (zo == 0 && znew != 0) atomicOr(f_out + W + ((unsigned)cur.i >> 5), 1u << ((unsigned)cur.i & 31u));
        } else if (znew == 0) atomicAdd(counts, 1);
    }
    if (!REG) __syncwarp(gmask);   // the count stores of this read precede the next read's loads (other lanes)
}

template <bool REG>
__device__ __forceinline__ void segment_counts_in(const PArgs& a, int seg, int* counts, GroupSmem& sm, unsigned gmask, int gl, int& cnt0, int& cnt1) {
    cnt0 = cnt1 = 0;
    if (REG) {
        const int K = a.seg_ntr[seg];
        const int* tids = a.comp_tids + a.seg_tid_off[seg];
        if (gl >= 1 && gl <= K) cnt0 = ld_cg(counts + tids[gl - 1]);
        if (gl + kGL <= K) cnt1 = ld_cg(counts + tids[gl + kGL - 1]);
        sm.al[gl] = a.alpha[(gl >= 1 && gl <= K) ? tids[gl - 1] : 0];
        sm.al[gl + kGL] = a.alpha[gl + kGL <= K ? tids[gl + kGL - 1] : 0];
        __syncwarp(gmask);
    }
}
template <bool REG>
__device__ __forceinline__ void segment_counts_out(const PArgs& a, int seg, int* counts, int gl, int cnt0, int cnt1) {
    if (REG) {
        const int K = a.seg_ntr[seg];
        const int* tids = a.comp_tids + a.seg_tid_off[seg];
        if (gl >= 1 && gl <= K) st_cg(counts + tids[gl - 1], cnt0);
        if (gl + kGL <= K) st_cg(counts + tids[gl + kGL - 1], cnt1);
    }
}

// Row-at-a-time walk: the next row's head is loaded while the current one is drawn (prefetch distance 1).  Kept as the
// cross-check of the pipelined walk below (RSEM_B200_GIBBS_PF=0).
template <bool REG>
__device__ __forceinline__ void walk_segment(const PArgs& a, int seg, bool use_counts, int* counts, const int* z_prev, int* z_cur,
                                             const unsigned* u, int c0_start, const unsigned* f_in, unsigned* f_out, const int* pre,
                                             const int* sh_base, unsigned w_per, unsigned W, int* err, GroupSmem& sm, unsigned gmask, int gl) {
    const int q0 = a.seg_start[seg], q_end = a.seg_start[seg + 1];
    int cnt0, cnt1;
    segment_counts_in<REG>(a, seg, counts, sm, gmask, gl, cnt0, cnt1);
    RowHead nxt;
    load_head(a, z_prev, u, q0, use_counts, gl, nxt);
    for (int q = q0; q < q_end; ++q) {
        const RowHead cur = nxt;
        if (q + 1 < q_end) load_head(a, z_prev, u, q + 1, use_counts, gl, nxt);   // in flight while `cur` is drawn
        int c0 = c0_start;
        if (use_counts) {   // noise count seen by read i: flips of the input set before position i
            const unsigned w = (unsigned)cur.i >> 5, m = (1u << ((unsigned)cur.i & 31u)) - 1u;
            c0 += sh_base[w / w_per] + ld_cg(pre + w) + __popc(__ldcg(f_in + w) & m) - __popc(__ldcg(f_in + W + w) & m);
        }
        process_row<REG>(a, cur, q, c0, use_counts, counts, z_cur, f_out, W, err, sm, gmask, gl, cnt0, cnt1);
    }
    segment_counts_out<REG>(a, seg, counts, gl, cnt0, cnt1);
}

// ---- pipelined walk -------------------------------------------------------------------------------------------------------
// A walk is one dependent chain per component, so its speed is the latency of one read.  With the row-at-a-time walk that
// latency is two DRAM round trips (slot -> read id / entry offset -> uniforms, flip words, entries): ~1.5 us per read at
// 10 M reads.  Here nothing on the chain waits for memory:
//   * slot metadata (read id, entry offset, length) is loaded 16 slots at a time, one slot per lane, two batches ahead;
//   * what depends on the read id and is rewritten inside the kernel (the previous assignment, the uniform, the flip words and
//     their prefix - read through L2, ld.cg) is loaded one batch ahead, again one slot per lane, and handed out by shuffles;
//   * the entries (ids, conprb: immutable) of the row kPD slots ahead are copied global -> shared with cp.async into a ring of
//     kPR rows per group; a row is drawn once its copy group has landed (cp.async.wait_group kPD).
constexpr int kPD = 2;    // rows of entries in flight
constexpr int kPR = 4;    // ring slots (>= kPD + 2: a slot is rewritten only after every lane has left its row)
constexpr int kPE = 2 * kGL;   // entries of a row kept in the ring (two per lane); longer rows read the rest from global memory

struct EntryRing {
    int t[kPR][kPE];
    double c[kPR][kPE];
};

__device__ __forceinline__ void cp_async_4(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_8(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct SlotMeta {   // lane gl: slot qb + gl of a batch
    int i;                    // read id
    unsigned len;
    unsigned long long off;
};
struct SlotMut {    // read through L2: rewritten by other CTAs between sweeps / passes
    int z;
    unsigned raw;
    int pre;
    unsigned f0, f1;
};

__device__ __forceinline__ void load_meta(const PArgs& a, int q, int q_end, SlotMeta& m) {
    m.i = 0; m.len = 0; m.off = 0;
    if (q < q_end) {
        m.i = __ldg(a.order + q);
        m.off = __ldg(a.p_off + q);
        m.len = (unsigned)(__ldg(a.p_off + q + 1) - m.off);
    }
}
__device__ __forceinline__ void load_mut(const SlotMeta& m, int q, int q_end, bool use_counts, const int* z_prev, const unsigned* u,
                                         const unsigned* f_in, const int* pre, unsigned W, SlotMut& x) {
    x.z = 0; x.raw = 0; x.pre = 0; x.f0 = 0; x.f1 = 0;
    if (q < q_end) {
        x.raw = __ldcg(u + m.i);
        if (use_counts) {
            const unsigned w = (unsigned)m.i >> 5;
            x.z = ld_cg(z_prev + q);
            x.pre = ld_cg(pre + w);
            x.f0 = __ldcg(f_in + w);
            x.f1 = __ldcg(f_in + W + w);
        }
    }
}
// net flips of the input set before read i (the noise count read i must see, minus c0 at the start of the sweep)
__device__ __forceinline__ int noise_adjust(const SlotMeta& m, const SlotMut& x, const int* sh_base, unsigned w_per) {
    const unsigned w = (unsigned)m.i >> 5, msk = (1u << ((unsigned)m.i & 31u)) - 1u;
    return sh_base[w / w_per] + x.pre + __popc(x.f0 & msk) - __popc(x.f1 & msk);
}

template <bool REG>
__device__ __forceinline__ void walk_segment_pf(const PArgs& a, int seg, bool use_counts, int* counts, const int* z_prev, int* z_cur,
                                                const unsigned* u, int c0_start, const unsigned* f_in, unsigned* f_out, const int* pre,
                                                const int* sh_base, unsigned w_per, unsigned W, int* err, GroupSmem& sm, EntryRing& ring,
                                                unsigned gmask, int gl) {
    const int q0 = a.seg_start[seg], q_end = a.seg_start[seg + 1];
    const int n = q_end - q0;
    int cnt0, cnt1;
    segment_counts_in<REG>(a, seg, counts, sm, gmask, gl, cnt0, cnt1);
    SlotMeta m0, m1, m2;   // batches b, b + 1, b + 2 of 16 slots
    load_meta(a, q0 + gl, q_end, m0);
    load_meta(a, q0 + kGL + gl, q_end, m1);
    load_meta(a, q0 + 2 * kGL + gl, q_end, m2);
    SlotMut x0, x1;        // batches b, b + 1
    load_mut(m0, q0 + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x0);
    load_mut(m1, q0 + kGL + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x1);
    int adj0 = use_counts ? noise_adjust(m0, x0, sh_base, w_per) : 0;
    // row r of the segment lives in batch r / 16; while row r0 of batch b is drawn, rows up to r0 + kPD are fetched: they are
    // in batch b (m0) or b + 1 (m1)
    auto fetch = [&](int r, bool next_batch) {
        const int lr = r & (kGL - 1);
        const unsigned long long off = __shfl_sync(gmask, next_batch ? m1.off : m0.off, lr, kGL);
        const unsigned len = __shfl_sync(gmask, next_batch ? m1.len : m0.len, lr, kGL);
        if (r < n && (unsigned)gl < len) {
            const int s = r & (kPR - 1);
            cp_async_4(&ring.t[s][gl], a.p_sid + off + gl);
            cp_async_8(&ring.c[s][gl], a.p_con + off + gl);
        }
        cp_async_commit();
    };
#pragma unroll
    for (int d = 0; d < kPD; ++d) fetch(d, false);
    for (int r = 0; r < n; ++r) {
        const int lr = r & (kGL - 1);
        if (lr == 0 && r > 0) {   // next batch: rotate, start the loads of the batches after it
            m0 = m1; m1 = m2;
            load_meta(a, q0 + r + 2 * kGL + gl, q_end, m2);
            x0 = x1;
            adj0 = use_counts ? noise_adjust(m0, x0, sh_base, w_per) : 0;
            load_mut(m1, q0 + r + kGL + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x1);
        }
        fetch(r + kPD, lr + kPD >= kGL);
        cp_async_wait<kPD>();
        __syncwarp(gmask);
        RowHead cur;
        cur.i = __shfl_sync(gmask, m0.i, lr, kGL);
        cur.len = __shfl_sync(gmask, m0.len, lr, kGL);
        cur.off = __shfl_sync(gmask, m0.off, lr, kGL);
        cur.zo = __shfl_sync(gmask, x0.z, lr, kGL);
        cur.raw = __shfl_sync(gmask, x0.raw, lr, kGL);
        const int c0 = c0_start + __shfl_sync(gmask, adj0, lr, kGL);
        const bool in = (unsigned)gl < cur.len;
        const int s = r & (kPR - 1);
        cur.t = in ? ring.t[s][gl] : -1;
        cur.c = in ? ring.c[s][gl] : 0.0;
        process_row<REG>(a, cur, q0 + r, c0, use_counts, counts, z_cur, f_out, W, err, sm, gmask, gl, cnt0, cnt1);
    }
    cp_async_wait<0>();
    __syncwarp(gmask);   // every lane has left the ring before the group's next segment refills it
    segment_counts_out<REG>(a, seg, counts, gl, cnt0, cnt1);
}

// The draw of a row of <= 16 entries of a register-resident component with live counts (every sweep but the first) - the
// case almost every read is - written for the shortest dependent chain: the running sum is a chain of DADDs only (terms past
// the lane's own index enter as +0.0, which leaves a non-negative sum unchanged), the product buffer is double-buffered so
// that a row needs one __syncwarp, and nothing that is only needed when the read changes its noise membership is computed
// up front.  Same arithmetic as process_row<true>: (count + alpha) * conprb, left-to-right fp64 sums, index = #{arr <= u * total}.
__device__ __forceinline__ double reg_entry_value(const GroupSmem& sm, unsigned gmask, bool valid, int t, double c, int zo, int c0,
                                                  int cnt0, int cnt1) {
    const int x0 = __shfl_sync(gmask, cnt0, t & (kGL - 1), kGL), x1 = __shfl_sync(gmask, cnt1, t & (kGL - 1), kGL);
    int cnt = (t & kGL) ? x1 : x0;
    if (t == 0) cnt = c0;
    if (t == zo) cnt -= 1;
    const double al = sm.al[valid ? t : 0];
    return valid ? __dmul_rn(__dadd_rn((double)cnt, al), c) : 0.0;
}

// Rows of up to 32 entries: lane gl owns entries gl and gl + 16.  The second half continues the first half's sum:
// arr[gl + 16] = ((x_0 + ... + x_15) + x_16 + ... + x_{gl+16}), all in entry order.
__device__ __forceinline__ int draw_reg_row(GroupSmem& sm, int buf, unsigned gmask, int gl, int len, int zo, unsigned raw, int c0, int t0,
                                            double c0v, int t1, double c1v, int& cnt0, int& cnt1, int* err) {
    const bool two = len > kGL;   // group-uniform
    const bool valid0 = gl < len, valid1 = gl + kGL < len;
    sm.w[buf][gl] = reg_entry_value(sm, gmask, valid0, t0, c0v, zo, c0, cnt0, cnt1);
    if (two) sm.w[buf][gl + kGL] = reg_entry_value(sm, gmask, valid1, t1, c1v, zo, c0, cnt0, cnt1);
    __syncwarp(gmask);
    const double2* p = reinterpret_cast<const double2*>(sm.w[buf]);
    double run0 = 0.0, run1 = 0.0;
#pragma unroll
    for (int j = 0; j < kGL; j += 4) {
        if (j < len) {   // group-uniform
            const double2 A = p[j / 2], B = p[j / 2 + 1];
            run0 = __dadd_rn(j <= gl ? A.x : 0.0, run0);
            run0 = __dadd_rn(j + 1 <= gl ? A.y : 0.0, run0);
            run0 = __dadd_rn(j + 2 <= gl ? B.x : 0.0, run0);
            run0 = __dadd_rn(j + 3 <= gl ? B.y : 0.0, run0);
            if (two) {       // the sum of the whole first half, the same in every lane
                run1 = __dadd_rn(A.x, run1);
                run1 = __dadd_rn(A.y, run1);
                run1 = __dadd_rn(B.x, run1);
                run1 = __dadd_rn(B.y, run1);
            }
        }
    }
    if (two) {
#pragma unroll
        for (int j = 0; j < kGL; j += 4) {
            if (j + kGL < len) {
                const double2 A = p[(j + kGL) / 2], B = p[(j + kGL) / 2 + 1];
                run1 = __dadd_rn(j <= gl ? A.x : 0.0, run1);
                run1 = __dadd_rn(j + 1 <= gl ? A.y : 0.0, run1);
                run1 = __dadd_rn(j + 2 <= gl ? B.x : 0.0, run1);
                run1 = __dadd_rn(j + 3 <= gl ? B.y : 0.0, run1);
            }
        }
    }
    const double total = two ? __shfl_sync(gmask, run1, len - 1 - kGL, kGL) : __shfl_sync(gmask, run0, len - 1, kGL);
    const double prb = __dmul_rn(raw * (1.0 / 4294967296.0), total);
    int l = __popc(__ballot_sync(gmask, valid0 && run0 <= prb));
    if (two) l += __popc(__ballot_sync(gmask, valid1 && run1 <= prb));
    if (l >= len) { *err = 3; l = len - 1; }   // reference: assert(l < len), sampling.h:62
    const int znew = l < kGL ? __shfl_sync(gmask, t0, l, kGL) : __shfl_sync(gmask, t1, l - kGL, kGL);
    if (znew != zo) {   // owners of the two local ids adjust their registers
        if (zo != 0 && (zo & (kGL - 1)) == gl) { if (zo < kGL) --cnt0; else --cnt1; }
        if (znew != 0 && (znew & (kGL - 1)) == gl) { if (znew < kGL) ++cnt0; else ++cnt1; }
    }
    return znew;
}

// ---- one pass, both lane groups of a warp in ONE loop ---------------------------------------------------------------------
// With a walk function per segment the two groups of a warp fall out of step at the first segment boundary and from then on
// every instruction is issued twice, once per half-warp, the two dependent chains taking turns on one instruction stream.
// Here a warp runs a single loop over "the current row of each group"; claiming the next component and priming its pipeline
// is a short divergent section, the draw itself is issued once for both groups.
__device__ __forceinline__ void walk_pass_converged(const PArgs& a, ChainSync* sy, bool use_counts, int* counts, const int* z_prev,
                                                    int* z_cur, const unsigned* u, int c0_start, const unsigned* f_in, unsigned* f_out,
                                                    const int* pre, const int* sh_base, unsigned w_per, unsigned W, GroupSmem& sm,
                                                    EntryRing& ring, unsigned gmask, int gl) {
    int seg = -1, q0 = 0, q_end = 0, n = 0, r = 0;
    bool active = true, reg = true;
    int cnt0 = 0, cnt1 = 0, adj0 = 0;
    SlotMeta m0, m1, m2;
    SlotMut x0, x1;
    m0.i = m1.i = m2.i = 0; m0.len = m1.len = m2.len = 0; m0.off = m1.off = m2.off = 0;
    x0.z = x1.z = 0; x0.raw = x1.raw = 0; x0.pre = x1.pre = 0; x0.f0 = x1.f0 = 0; x0.f1 = x1.f1 = 0;
    auto fetch = [&](int rr, bool next_batch) {
        const int lr = rr & (kGL - 1);
        const unsigned long long off = __shfl_sync(gmask, next_batch ? m1.off : m0.off, lr, kGL);
        const unsigned len = __shfl_sync(gmask, next_batch ? m1.len : m0.len, lr, kGL);
        if (rr < n) {
            const int sl = rr & (kPR - 1);
            if ((unsigned)gl < len) {
                cp_async_4(&ring.t[sl][gl], a.p_sid + off + gl);
                cp_async_8(&ring.c[sl][gl], a.p_con + off + gl);
            }
            if ((unsigned)gl + kGL < len) {
                cp_async_4(&ring.t[sl][gl + kGL], a.p_sid + off + gl + kGL);
                cp_async_8(&ring.c[sl][gl + kGL], a.p_con + off + gl + kGL);
            }
        }
        cp_async_commit();
    };
    for (;;) {
        if (active && r == n) {   // group-divergent: finish the component, claim the next one, prime its pipeline
            if (seg >= 0) {
                cp_async_wait<0>();
                __syncwarp(gmask);   // every lane has left the ring
                if (reg) segment_counts_out<true>(a, seg, counts, gl, cnt0, cnt1);
            }
            int sgm = 0;
            if (gl == 0) sgm = (int)atomicAdd(&sy->next_seg, 1u);
            sgm = __shfl_sync(gmask, sgm, 0, kGL);
            if (sgm >= a.n_segs) active = false;
            else {
                seg = sgm;
                q0 = a.seg_start[seg];
                q_end = a.seg_start[seg + 1];
                n = q_end - q0;
                r = 0;
                reg = a.seg_ntr[seg] < 2 * kGL;
                if (reg) segment_counts_in<true>(a, seg, counts, sm, gmask, gl, cnt0, cnt1);
                load_meta(a, q0 + gl, q_end, m0);
                load_meta(a, q0 + kGL + gl, q_end, m1);
                load_meta(a, q0 + 2 * kGL + gl, q_end, m2);
                load_mut(m0, q0 + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x0);
                load_mut(m1, q0 + kGL + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x1);
                adj0 = use_counts ? noise_adjust(m0, x0, sh_base, w_per) : 0;
#pragma unroll
                for (int d = 0; d < kPD; ++d) fetch(d, false);
            }
        }
        if (!__any_sync(0xffffffffu, active)) break;   // both groups of the warp are here in every iteration
        if (active) {
            const int lr = r & (kGL - 1);
            if (lr == 0 && r > 0) {   // next batch of 16 slots: rotate, start the loads of the batches after it
                m0 = m1; m1 = m2;
                load_meta(a, q0 + r + 2 * kGL + gl, q_end, m2);
                x0 = x1;
                adj0 = use_counts ? noise_adjust(m0, x0, sh_base, w_per) : 0;
                load_mut(m1, q0 + r + kGL + gl, q_end, use_counts, z_prev, u, f_in, pre, W, x1);
            }
            fetch(r + kPD, lr + kPD >= kGL);
            cp_async_wait<kPD>();
            __syncwarp(gmask);
            const int len = (int)__shfl_sync(gmask, m0.len, lr, kGL);
            const int zo = __shfl_sync(gmask, x0.z, lr, kGL);
            const unsigned raw = __shfl_sync(gmask, x0.raw, lr, kGL);
            const int c0 = c0_start + __shfl_sync(gmask, adj0, lr, kGL);
            const bool in = gl < len;
            const int sl = r & (kPR - 1);
            const int t = in ? ring.t[sl][gl] : -1;
            const double c = in ? ring.c[sl][gl] : 0.0;
            if (a.fast_rows && reg && use_counts && len <= kPE) {
                const bool in1 = gl + kGL < len;
                const int t1 = in1 ? ring.t[sl][gl + kGL] : -1;
                const double c1 = in1 ? ring.c[sl][gl + kGL] : 0.0;
                const int znew = draw_reg_row(sm, r & 1, gmask, gl, len, zo, raw, c0, t, c, t1, c1, cnt0, cnt1, &sy->err);
                if (gl == 0) st_cg(z_cur + q0 + r, znew);
                if ((zo == 0) != (znew == 0)) {   // the read joined or left the noise transcript (group-uniform, rare)
                    const unsigned i = (unsigned)__shfl_sync(gmask, m0.i, lr, kGL);
                    if (gl == 0) atomicOr(f_out + (znew == 0 ? 0u : W) + (i >> 5), 1u << (i & 31u));
                }
            } else {
                __syncwarp(gmask);   // a fast row may still be read from sm.w by a slower lane; sm.v is separate, but keep rows apart
                RowHead cur;
                cur.i = __shfl_sync(gmask, m0.i, lr, kGL);
                cur.len = (unsigned)len;
                cur.off = __shfl_sync(gmask, m0.off, lr, kGL);
                cur.zo = zo;
                cur.raw = raw;
                cur.t = t;
                cur.c = c;
                if (reg) process_row<true>(a, cur, q0 + r, c0, use_counts, counts, z_cur, f_out, W, &sy->err, sm, gmask, gl, cnt0, cnt1);
                else process_row<false>(a, cur, q0 + r, c0, use_counts, counts, z_cur, f_out, W, &sy->err, sm, gmask, gl, cnt0, cnt1);
            }
            ++r;
        }
    }
}

// One chain on the CTAs of its team: worker CTAs 0 .. ctas_per_chain - 1 and the generator CTA (cta == ctas_per_chain).
// `chain` indexes what belongs to the chain (chain_samples, chain_seeds, chain_cv_offset, sync, slice_tot, acc), `slot` the
// scratch it runs in (counts, counts_start, z, ubuf, flips, pre, theta_tmp).  gibbs_parallel_kernel runs chain c in slot c;
// gibbs_batch_kernel runs a job's chain of its sample in slot 0 of a PArgs whose scratch pointers are the team's.
template <int PF>   // 0: row-at-a-time walk, 1: pipelined walk per segment, 2: pipelined, both groups of a warp in one loop
__device__ __forceinline__ void chain_body(const PArgs& a, const int chain, const size_t slot, const unsigned cta) {
    __shared__ EntryRing sh_ring[PF ? kPThreads / kGL : 1];
    __shared__ double sh_red[kPThreads / 32];
    __shared__ int sh_scan[kPThreads];
    __shared__ int sh_base[512];     // exclusive prefix of the slice totals (<= 512 worker CTAs per chain)
    __shared__ GroupSmem sh_grp[kPThreads / kGL];
    const unsigned n_ctas = a.ctas_per_chain;
    const int tid = threadIdx.x;
    const int M1 = a.M + 1;
    const unsigned W = a.n_words;
    ChainSync* sy = a.sync + chain;
    const int n_samples = a.chain_samples[chain];
    const int chainlen = 1 + (n_samples - 1) * a.gap;
    const unsigned n_sweeps = 1u + (unsigned)(a.burnin + chainlen);   // sweep 0 = initial state from conprb alone
    unsigned* ubuf = a.ubuf + slot * 2 * a.N1;
    if (cta == n_ctas) {
        generator_loop(a, sy, ubuf, n_sweeps, a.chain_seeds[chain]);
        return;
    }
    const unsigned chain_threads = n_ctas * kPThreads, ctid = cta * kPThreads + tid;
    int* counts = a.counts + slot * M1;
    int* counts_start = a.counts_start + slot * M1;
    int* zbuf = a.z + slot * 2 * a.N1;
    unsigned* fl = a.flips + slot * 4 * W;
    int* pre = a.pre + slot * W;
    int* slice_tot = a.slice_tot + (size_t)chain * n_ctas;
    double* acc = a.acc + (size_t)chain * (4 * (size_t)M1 + a.n_genes);
    double* theta = a.theta_tmp + slot * 2 * M1;
    double* fpkm = theta + M1;
    int* cv = a.count_vectors + a.chain_cv_offset[chain] * M1;
    // this CTA's slice of flip words (prefix sums are formed per slice, the slice bases are added on the fly)
    const unsigned w_per = (W + n_ctas - 1) / n_ctas;
    const unsigned w_lo = min(W, cta * w_per), w_hi = min(W, w_lo + w_per);

    for (int i = ctid; i < M1; i += chain_threads) st_cg(counts + i, a.init_counts[i] + (i == 0 ? (int)a.n0 : 0));
    chain_barrier(sy, n_ctas);

    int kept = 0;
    for (unsigned sweep = 0; sweep < n_sweeps; ++sweep) {
        const bool use_counts = sweep > 0;
        const int round = (int)sweep;
        const unsigned* u = ubuf + (size_t)(sweep & 1u) * a.N1;
        const int* z_prev = zbuf + (size_t)((sweep + 1u) & 1u) * a.N1;
        int* z_cur = zbuf + (size_t)(sweep & 1u) * a.N1;
        long long t0 = clock64();
        if (tid == 0) {
            while (*((volatile unsigned*)&sy->u_ready) < sweep + 1) {}
            __threadfence();
        }
        __syncthreads();
        long long t1 = clock64();
        if (cta == 0 && tid == 0) sy->prof[0] += t1 - t0;
        const int c0_start = ld_cg(counts);
        // start of the sweep: copy of the counts for restarts; the input flip set (set 0) is empty
        if (use_counts) {
            for (int i = ctid; i < M1; i += chain_threads) st_cg(counts_start + i, ld_cg(counts + i));
            for (unsigned w = ctid; w < 2 * W; w += chain_threads) __stcg(fl + w, 0u);
            for (unsigned w = w_lo + tid; w < w_hi; w += kPThreads) st_cg(pre + w, 0);
            if (tid == 0) st_cg(slice_tot + cta, 0);
        }
        unsigned in_set = 0;   // flip set the pass reads; it writes the other one
        for (unsigned pass = 0;; ++pass) {
            unsigned* f_in = fl + (size_t)in_set * 2 * W;
            unsigned* f_out = fl + (size_t)(in_set ^ 1u) * 2 * W;
            if (use_counts) {
                for (unsigned w = ctid; w < 2 * W; w += chain_threads) __stcg(f_out + w, 0u);
                if (pass > 0)
                    for (int i = ctid + 1; i < M1; i += chain_threads) st_cg(counts + i, ld_cg(counts_start + i));
                if (cta == 0 && tid == 0) { sy->changed = 0; sy->passes++; }
                chain_barrier(sy, n_ctas);
                // exclusive prefix of the slice totals of the input set
                for (unsigned c = tid; c < n_ctas; c += kPThreads) sh_base[c] = ld_cg(slice_tot + c);
                __syncthreads();
                if (tid == 0) {
                    int run = 0;
                    for (unsigned c = 0; c < n_ctas; ++c) { const int v = sh_base[c]; sh_base[c] = run; run += v; }
                }
                __syncthreads();
            }
            const long long tp0 = clock64();
            {   // groups of kGL lanes claim components, longest first (a walk is sequential: the long ones must start early)
                const int gl = tid & (kGL - 1);
                const unsigned gmask = 0xffffu << ((tid & 31) & ~(kGL - 1));
                GroupSmem& gsm = sh_grp[tid / kGL];
                if (PF == 2) {
                    walk_pass_converged(a, sy, use_counts, counts, z_prev, z_cur, u, c0_start, f_in, f_out, pre, sh_base, w_per, W, gsm,
                                        sh_ring[PF ? tid / kGL : 0], gmask, gl);
                } else
                for (;;) {
                    int sgm = 0;
                    if (gl == 0) sgm = (int)atomicAdd(&sy->next_seg, 1u);
                    sgm = __shfl_sync(gmask, sgm, 0, kGL);
                    if (sgm >= a.n_segs) break;
                    if (PF) {
                        EntryRing& ring = sh_ring[PF ? tid / kGL : 0];
                        if (a.seg_ntr[sgm] < 2 * kGL)
                            walk_segment_pf<true>(a, sgm, use_counts, counts, z_prev, z_cur, u, c0_start, f_in, f_out, pre, sh_base, w_per, W,
                                                  &sy->err, gsm, ring, gmask, gl);
                        else
                            walk_segment_pf<false>(a, sgm, use_counts, counts, z_prev, z_cur, u, c0_start, f_in, f_out, pre, sh_base, w_per, W,
                                                   &sy->err, gsm, ring, gmask, gl);
                    } else if (a.seg_ntr[sgm] < 2 * kGL)
                        walk_segment<true>(a, sgm, use_counts, counts, z_prev, z_cur, u, c0_start, f_in, f_out, pre, sh_base, w_per, W, &sy->err,
                                           gsm, gmask, gl);
                    else
                        walk_segment<false>(a, sgm, use_counts, counts, z_prev, z_cur, u, c0_start, f_in, f_out, pre, sh_base, w_per, W,
                                            &sy->err, gsm, gmask, gl);
                }
            }
            const long long tp1 = clock64();
            if (cta == 0 && tid == 0) sy->prof[1] += tp1 - tp0;
            if (!use_counts) {
                chain_barrier(sy, n_ctas);
                if (cta == 0 && tid == 0) sy->next_seg = 0;   // the next pass starts behind another barrier
                break;
            }
            chain_barrier(sy, n_ctas);
            if (cta == 0 && tid == 0) sy->next_seg = 0;
            // compare the two sets on this CTA's slice and form the prefix sums of the output set
            bool diff = false;
            int part = 0;
            const unsigned per_thread = (w_hi - w_lo + kPThreads - 1) / kPThreads;
            const unsigned my_lo = min(w_hi, w_lo + tid * per_thread), my_hi = min(w_hi, my_lo + per_thread);
            for (unsigned w = my_lo; w < my_hi; ++w) {
                const unsigned pj = __ldcg(f_out + w), pl = __ldcg(f_out + W + w);
                diff = diff || pj != __ldcg(f_in + w) || pl != __ldcg(f_in + W + w);
                part += __popc(pj) - __popc(pl);
            }
            sh_scan[tid] = part;
            __syncthreads();
            if (tid == 0) {
                int run = 0;
                for (int t = 0; t < kPThreads; ++t) { const int v = sh_scan[t]; sh_scan[t] = run; run += v; }
                st_cg(slice_tot + cta, run);
            }
            __syncthreads();
            {
                int run = sh_scan[tid];
                for (unsigned w = my_lo; w < my_hi; ++w) {
                    st_cg(pre + w, run);
                    run += __popc(__ldcg(f_out + w)) - __popc(__ldcg(f_out + W + w));
                }
            }
            if (__syncthreads_or(diff) && tid == 0) atomicExch(&sy->changed, 1u);
            chain_barrier(sy, n_ctas);
            in_set ^= 1u;   // the output set (with its prefix sums) is the next pass's input - or the final flip set
            if (*((volatile unsigned*)&sy->changed) == 0) break;
            chain_barrier(sy, n_ctas);   // everyone has read `changed` before CTA 0 clears it
        }
        if (use_counts) {
            // net change of the noise count = all flips of the final set
            for (unsigned c = tid; c < n_ctas; c += kPThreads) sh_base[c] = ld_cg(slice_tot + c);
            __syncthreads();
            if (cta == 0 && tid == 0) {
                int run = 0;
                for (unsigned c = 0; c < n_ctas; ++c) run += sh_base[c];
                st_cg(counts, c0_start + run);
            }
        }
        const long long t2 = clock64();
        chain_barrier(sy, n_ctas);
        if (cta == 0 && tid == 0) {
            __threadfence();
            atomicExch(&sy->sweeps_done, sweep + 1);   // this sweep's uniforms (and the previous z) are no longer read
        }
        if (round > a.burnin && (round - a.burnin - 1) % a.gap == 0) {   // Gibbs.cpp:313-346, by CTA 0 of the chain
            if (cta == 0) {
                double part = 0.0;
                for (int i = tid; i < M1; i += kPThreads) {
                    const int c = ld_cg(counts + i);
                    cv[(size_t)kept * M1 + i] = c;
                    double th = c < 0 ? 0.0 : ((double)c + a.alpha[i]) / a.totc;
                    if (i > 0 && (a.mw[i] < kEpsilon || a.eel[i] < kEpsilon)) th = 0.0;
                    else th = th / a.mw[i];
                    theta[i] = th;
                    part += th;
                }
                const double tsum = block_sum(part, sh_red);
                part = 0.0;
                for (int i = tid; i < M1; i += kPThreads) {
                    const double th = theta[i] / tsum;
                    theta[i] = th;
                    if (i > 0 && a.eel[i] >= kEpsilon) part += th;
                }
                double denom = block_sum(part, sh_red);
                if (denom < kEpsilon) denom = 1.0;
                part = 0.0;
                for (int i = tid; i < M1; i += kPThreads) {
                    const double f = (i > 0 && a.eel[i] >= kEpsilon) ? (theta[i] / denom) * 1e9 / a.eel[i] : 0.0;
                    fpkm[i] = f;
                    part += f;
                }
                double fsum = block_sum(part, sh_red);
                if (fsum < kEpsilon) fsum = 1.0;
                for (int i = tid; i < M1; i += kPThreads) {
                    const double c = (double)ld_cg(counts + i);
                    acc[i] += c;
                    acc[M1 + i] += c * c;
                    acc[2 * (size_t)M1 + i] += i > 0 ? fpkm[i] / fsum * 1e6 : 0.0;
                    acc[3 * (size_t)M1 + i] += fpkm[i];
                }
                for (int gi = tid; gi < a.n_genes; gi += kPThreads) {
                    double c = 0.0;
                    for (int j = a.gene_start[gi]; j < a.gene_start[gi + 1]; ++j) c += ld_cg(counts + j);
                    acc[4 * (size_t)M1 + gi] += c * c;
                }
            }
            ++kept;
            chain_barrier(sy, n_ctas);
        }
        if (cta == 0 && tid == 0) { sy->prof[2] += t2 - t1; sy->prof[3] += clock64() - t2; }
    }
}

template <int PF>
__global__ void __launch_bounds__(kPThreads, PF ? 3 : 4) gibbs_parallel_kernel(const PArgs a) {
    const unsigned group = a.ctas_per_chain + 1;   // worker CTAs + the generator CTA
    const int chain = a.chain_base + blockIdx.x / group;
    chain_body<PF>(a, chain, (size_t)chain, blockIdx.x % group);
}

// ---- K13: the chains of many samples in one cooperative launch (rsem_b200_gibbs_batch_*) -----------------------------
// A job is one (sample, chain); a team is k worker CTAs + 1 generator CTA, the shape of one chain of gibbs_parallel_kernel.
// Worker CTA 0 of a team claims the next job from a device counter (jobs are numbered largest first) and hands its number
// to the team's other CTAs through the team's mailbox word (claim number << 32 | job).  Every CTA then copies the job's
// sample view into shared memory - the sample's PArgs with the team's scratch in slot 0 - and runs chain_body<2> on it.
// A job's ChainSync and slice totals belong to the job (zeroed before the launch): a team starts every job fresh.  The
// team's CTAs have all read claim r before worker CTA 0 can post claim r + 1: the workers passed the job's first barrier
// and the generator published the job's first uniforms, both of which worker CTA 0 waits for.
struct BArgs {
    const PArgs* samples;
    const int2* jobs;                 // (sample, chain of the sample), largest first
    unsigned n_jobs, k;
    unsigned* next_job;
    unsigned long long* mailbox;      // one word per team
    // per team scratch, sized for the largest sample of the launch
    int* counts;
    int* counts_start;
    int* z;
    unsigned* ubuf;
    unsigned* flips;
    int* pre;
    double* theta_tmp;
    unsigned long long n1_max;
    unsigned w_max;
    int M1;
};

__global__ void __launch_bounds__(kPThreads, 3) gibbs_batch_kernel(const BArgs b) {
    __shared__ PArgs sa;
    __shared__ unsigned sh_job;
    const unsigned group = b.k + 1;
    const unsigned team = blockIdx.x / group, cta = blockIdx.x % group;
    unsigned long long* box = b.mailbox + team;
    for (unsigned long long r = 1;; ++r) {
        if (threadIdx.x == 0) {
            unsigned job;
            if (cta == 0) {
                job = atomicAdd(b.next_job, 1u);
                atomicExch(box, (r << 32) | job);
            } else {
                unsigned long long v;
                while (((v = *((volatile unsigned long long*)box)) >> 32) != r) {}
                job = (unsigned)v;
            }
            sh_job = job;
            if (job < b.n_jobs) {
                const int2 jb = b.jobs[job];
                sa = b.samples[jb.x];
                sa.counts = b.counts + (size_t)team * b.M1;
                sa.counts_start = b.counts_start + (size_t)team * b.M1;
                sa.z = b.z + (size_t)team * 2 * b.n1_max;
                sa.ubuf = b.ubuf + (size_t)team * 2 * b.n1_max;
                sa.flips = b.flips + (size_t)team * 4 * b.w_max;
                sa.pre = b.pre + (size_t)team * b.w_max;
                sa.theta_tmp = b.theta_tmp + (size_t)team * 2 * b.M1;
                sa.chain_base = jb.y;
            }
        }
        __syncthreads();
        if (sh_job >= b.n_jobs) return;
        chain_body<2>(sa, sa.chain_base, 0, cta);
        __syncthreads();   // sa and sh_job are rewritten by the next claim
    }
}

template <class T>
int to_dev(T** d, const T* h, size_t n, cudaStream_t s) {
    RB_CUDA(cudaMalloc(d, std::max<size_t>(n, 1) * sizeof(T)));
    if (n) RB_CUDA(cudaMemcpyAsync(*d, h, n * sizeof(T), cudaMemcpyHostToDevice, s));
    return 0;
}

}  // namespace

static int gibbs_run_serial(rsem_b200_ctx* c, const rsem_b200_gibbs_params* p, int32_t* count_vectors, double* chain_acc,
                            rsem_b200_gibbs_stats* stats) {
    const DevGibbs& g = c->gibbs;
    const int M1 = p->M + 1, nc = p->n_chains;
    long long total_samples = 0;
    std::vector<long long> cv_off(nc);
    for (int t = 0; t < nc; ++t) { cv_off[t] = total_samples; total_samples += p->chain_samples[t]; }

    // longest row decides whether the cumulative array fits shared memory
    std::vector<uint64_t> h_rp(g.N1 + 1);
    RB_CUDA(cudaMemcpyAsync(h_rp.data(), g.row_ptr, (g.N1 + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    uint64_t max_len = 1;
    for (uint64_t i = 0; i < g.N1; ++i) max_len = std::max(max_len, h_rp[i + 1] - h_rp[i]);

    GibbsArgs a{};
    a.N1 = g.N1;
    a.row_ptr = reinterpret_cast<const unsigned long long*>(g.row_ptr);
    a.sid = g.sid;
    a.conprb = g.conprb;
    a.M = p->M; a.burnin = p->burnin; a.gap = p->gap; a.n_genes = p->n_genes;
    a.n0 = p->n0; a.totc = p->totc;
    a.max_len = (unsigned)max_len;
    a.err_flag = c->err_flag;

    int *d_samples = nullptr, *d_init = nullptr, *d_gene = nullptr, *d_counts = nullptr, *d_z = nullptr, *d_cv = nullptr;
    unsigned* d_seeds = nullptr;
    long long* d_off = nullptr;
    double *d_alpha = nullptr, *d_eel = nullptr, *d_mw = nullptr, *d_scratch = nullptr, *d_acc = nullptr, *d_tmp = nullptr;
    const size_t acc_per = 4 * (size_t)M1 + p->n_genes;
    int rc = 0;
    auto cleanup = [&]() {
        cudaFree(d_samples); cudaFree(d_init); cudaFree(d_gene); cudaFree(d_counts); cudaFree(d_z); cudaFree(d_cv);
        cudaFree(d_seeds); cudaFree(d_off); cudaFree(d_alpha); cudaFree(d_eel); cudaFree(d_mw); cudaFree(d_scratch);
        cudaFree(d_acc); cudaFree(d_tmp);
    };
#define RB_TRY(x) do { rc = (x); if (rc) { cleanup(); return rc; } } while (0)
#define RB_TRYC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cleanup(); return cuda_fail(e_, #x, __FILE__, __LINE__); } } while (0)
    RB_TRY(to_dev(&d_samples, p->chain_samples, nc, c->stream));
    RB_TRY(to_dev(&d_seeds, p->chain_seeds, nc, c->stream));
    RB_TRY(to_dev(&d_off, cv_off.data(), nc, c->stream));
    RB_TRY(to_dev(&d_init, p->init_counts, M1, c->stream));
    RB_TRY(to_dev(&d_alpha, p->pseudo_counts, M1, c->stream));
    RB_TRY(to_dev(&d_eel, p->eel, M1, c->stream));
    RB_TRY(to_dev(&d_mw, p->mw, M1, c->stream));
    RB_TRY(to_dev(&d_gene, p->gene_start, (size_t)p->n_genes + 1, c->stream));
    RB_TRYC(cudaMalloc(&d_counts, (size_t)nc * M1 * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_z, std::max<size_t>((size_t)nc * g.N1, 1) * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_cv, std::max<size_t>((size_t)total_samples * M1, 1) * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_acc, (size_t)nc * acc_per * sizeof(double)));
    RB_TRYC(cudaMalloc(&d_tmp, (size_t)nc * 2 * M1 * sizeof(double)));
    RB_TRYC(cudaMemsetAsync(d_acc, 0, (size_t)nc * acc_per * sizeof(double), c->stream));
    if (max_len > kRowCap) RB_TRYC(cudaMalloc(&d_scratch, (size_t)nc * max_len * sizeof(double)));
    a.chain_samples = d_samples; a.chain_seeds = d_seeds; a.chain_cv_offset = d_off; a.init_counts = d_init;
    a.alpha = d_alpha; a.eel = d_eel; a.mw = d_mw; a.gene_start = d_gene; a.counts = d_counts; a.z = d_z;
    a.scratch = d_scratch; a.count_vectors = d_cv; a.acc = d_acc; a.theta_tmp = d_tmp;

    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (stats) { cudaEventCreate(&ev0); cudaEventCreate(&ev1); cudaEventRecord(ev0, c->stream); }
    gibbs_chain_kernel<<<nc, kGibbsThreads, 0, c->stream>>>(a);
    RB_TRYC(cudaGetLastError());
    c->launches++;
    if (stats) cudaEventRecord(ev1, c->stream);

    RB_TRYC(cudaMemcpyAsync(chain_acc, d_acc, (size_t)nc * acc_per * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_TRYC(cudaMemcpyAsync(count_vectors, d_cv, (size_t)total_samples * M1 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    int err = 0;
    RB_TRYC(cudaMemcpyAsync(&err, c->err_flag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    RB_TRYC(cudaStreamSynchronize(c->stream));
    cleanup();
#undef RB_TRY
#undef RB_TRYC
    if (stats) {
        float ms = 0;
        cudaEventElapsedTime(&ms, ev0, ev1);
        cudaEventDestroy(ev0); cudaEventDestroy(ev1);
        *stats = rsem_b200_gibbs_stats{ms, 0, 1};
    }
    if (err) {
        cudaMemset(c->err_flag, 0, sizeof(int));
        set_error("gibbs: categorical draw fell off the cumulative array (reference: assert(l < len), sampling.h:62)");
        return RSEM_B200_ERR_ARG;
    }
    return 0;
}


__global__ void permute_rows_kernel(const unsigned long long* row_ptr, const double* conprb, const int* order,
                                    const unsigned long long* p_off, unsigned long long N1, double* p_con) {
    for (unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; q < N1;
         q += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long src = row_ptr[order[q]], dst = p_off[q], n = p_off[q + 1] - dst;
        for (unsigned long long k = 0; k < n; ++k) p_con[dst + k] = conprb[src + k];
    }
}

// ---- static preparation for the component-parallel sampler (host) ---------------------------------------------
int gibbs_layout(const uint64_t* row_ptr, const int32_t* sid, uint64_t N1, int M, GibbsLayout& L) {
    L = GibbsLayout{};
    L.N1 = N1;
    if (N1 == 0) return 0;
    if (N1 > 0x7fffffffull) { set_error("gibbs: more than 2^31 reads are not supported"); return RSEM_B200_ERR_UNSUPPORTED; }
    // connected components of the read x transcript graph, noise transcript excluded (union-find with path halving)
    std::vector<int32_t> parent((size_t)M + 1);
    for (int t = 0; t <= M; ++t) parent[t] = t;
    auto find = [&](int32_t x) {
        while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; }
        return x;
    };
    uint64_t max_len = 1;
    for (uint64_t i = 0; i < N1; ++i) {
        int32_t first = 0;
        max_len = std::max(max_len, row_ptr[i + 1] - row_ptr[i]);
        if (row_ptr[i + 1] == row_ptr[i]) L.empty_row = true;
        for (uint64_t j = row_ptr[i]; j < row_ptr[i + 1]; ++j) {
            const int32_t t = sid[j];
            if (t < 0 || t > M) { set_error("gibbs: transcript id out of range in the .ofg matrix"); return RSEM_B200_ERR_ARG; }
            if (t == 0) continue;
            if (first == 0) first = find(t);
            else {
                const int32_t r = find(t);
                if (r != first) parent[r] = first;
            }
        }
    }
    L.max_len = (uint32_t)max_len;
    // component of a read = root of its first non-noise transcript; 0 = the row holds only the noise entry (its own segment)
    std::vector<int32_t> comp(N1);
    std::vector<uint32_t> comp_reads((size_t)M + 1, 0);
    uint64_t n_lonely = 0;
    for (uint64_t i = 0; i < N1; ++i) {
        int32_t k = 0;
        for (uint64_t j = row_ptr[i]; j < row_ptr[i + 1]; ++j)
            if (sid[j] != 0) { k = find(sid[j]); break; }
        comp[i] = k;
        if (k) ++comp_reads[k]; else ++n_lonely;
    }
    // segments: one per component, longest first (a thread walks a whole segment: the long ones must start first),
    // then the noise-only reads one by one; reads keep their order inside a segment (counting sort)
    std::vector<int32_t> roots;
    for (int t = 1; t <= M; ++t) if (comp_reads[t]) roots.push_back(t);
    std::stable_sort(roots.begin(), roots.end(), [&](int32_t x, int32_t y) { return comp_reads[x] > comp_reads[y]; });
    std::vector<int32_t>& seg_start = L.seg_start;
    seg_start.reserve(roots.size() + n_lonely + 1);
    std::vector<uint64_t> fill((size_t)M + 1, 0);
    uint64_t at = 0;
    for (int32_t r : roots) { seg_start.push_back((int32_t)at); fill[r] = at; at += comp_reads[r]; }
    std::vector<int32_t>& order = L.order;
    order.resize(N1);
    for (uint64_t i = 0; i < N1; ++i) {
        if (comp[i]) order[fill[comp[i]]++] = (int32_t)i;
        else { seg_start.push_back((int32_t)at); order[at++] = (int32_t)i; }
    }
    seg_start.push_back((int32_t)N1);
    L.n_segs = (int32_t)seg_start.size() - 1;
    // transcripts of every component (sorted) and the local id of a transcript inside its component (1.., 0 = noise):
    // components of fewer than 32 transcripts are walked with their counts in registers, rows and assignments in local ids
    std::vector<int32_t> lid((size_t)M + 1, 0), ntr((size_t)M + 1, 0);
    for (int t = 1; t <= M; ++t) lid[t] = ++ntr[find(t)];
    L.seg_ntr.assign(L.n_segs, 0);
    L.seg_tid_off.assign(L.n_segs + 1, 0);
    {
        std::vector<int32_t> tid_at((size_t)M + 1, 0);   // offset of root r's list
        int32_t at_t = 0;
        for (size_t sgi = 0; sgi < roots.size(); ++sgi) {
            L.seg_ntr[sgi] = ntr[roots[sgi]];
            L.seg_tid_off[sgi] = at_t;
            tid_at[roots[sgi]] = at_t;
            at_t += ntr[roots[sgi]];
        }
        for (int sgi = (int)roots.size(); sgi <= L.n_segs; ++sgi) L.seg_tid_off[sgi] = at_t;
        L.comp_tids.assign((size_t)at_t + 1, 0);
        for (int t = 1; t <= M; ++t) {
            const int32_t r = find(t);
            if (comp_reads[r]) L.comp_tids[(size_t)tid_at[r] + lid[t] - 1] = t;
        }
    }
    // rows re-laid in slot order so that a segment is one contiguous stream
    const uint64_t E = row_ptr[N1];
    L.p_off.resize(N1 + 1);
    L.p_sid.resize(E);
    L.p_off[0] = 0;
    for (uint64_t q = 0; q < N1; ++q) L.p_off[q + 1] = L.p_off[q] + (row_ptr[order[q] + 1] - row_ptr[order[q]]);
    for (uint64_t q = 0; q < N1; ++q) {
        const uint64_t src = row_ptr[order[q]], n = row_ptr[order[q] + 1] - src;
        const int32_t k = comp[order[q]];
        if (k == 0 || ntr[k] < 32) {   // register-resident component: local ids
            for (uint64_t j = 0; j < n; ++j) L.p_sid[L.p_off[q] + j] = lid[sid[src + j]];
        } else memcpy(L.p_sid.data() + L.p_off[q], sid + src, n * sizeof(int32_t));
    }
    return 0;
}

int gibbs_prepare(rsem_b200_ctx* c, const uint64_t* row_ptr, const int32_t* sid) {
    DevGibbs& g = c->gibbs;
    const uint64_t N1 = g.N1;
    if (N1 == 0) return 0;
    GibbsLayout L;
    if (int rc = gibbs_layout(row_ptr, sid, N1, g.M, L)) return rc;
    g.max_len = L.max_len;
    g.empty_row = L.empty_row;
    g.n_segs = L.n_segs;
    {
        const uint64_t E = row_ptr[N1];
        RB_CUDA(cudaMalloc(&g.p_off, (N1 + 1) * sizeof(uint64_t)));
        RB_CUDA(cudaMalloc(&g.p_sid, (E + 16) * sizeof(int32_t)));
        RB_CUDA(cudaMalloc(&g.p_con, (E + 16) * sizeof(double)));
        RB_CUDA(cudaMemcpyAsync(g.p_off, L.p_off.data(), (N1 + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
        RB_CUDA(cudaMemcpyAsync(g.p_sid, L.p_sid.data(), E * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        // conprb is permuted on the device from the already uploaded copy
        RB_CUDA(cudaMalloc(&g.order, N1 * sizeof(int32_t)));
        RB_CUDA(cudaMemcpyAsync(g.order, L.order.data(), N1 * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        permute_rows_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(reinterpret_cast<const unsigned long long*>(g.row_ptr), g.conprb,
                                                                   g.order, reinterpret_cast<const unsigned long long*>(g.p_off), N1, g.p_con);
        RB_CUDA(cudaGetLastError());
        c->launches++;
        RB_CUDA(cudaStreamSynchronize(c->stream));
    }
    RB_CUDA(cudaMalloc(&g.seg_start, L.seg_start.size() * sizeof(int32_t)));
    RB_CUDA(cudaMemcpyAsync(g.seg_start, L.seg_start.data(), L.seg_start.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMalloc(&g.seg_ntr, std::max<size_t>(L.seg_ntr.size(), 1) * sizeof(int32_t)));
    RB_CUDA(cudaMalloc(&g.seg_tid_off, L.seg_tid_off.size() * sizeof(int32_t)));
    RB_CUDA(cudaMalloc(&g.comp_tids, L.comp_tids.size() * sizeof(int32_t)));
    g.n_comp_tids = L.comp_tids.size();
    RB_CUDA(cudaMemcpyAsync(g.seg_ntr, L.seg_ntr.data(), L.seg_ntr.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(g.seg_tid_off, L.seg_tid_off.data(), L.seg_tid_off.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemcpyAsync(g.comp_tids, L.comp_tids.data(), L.comp_tids.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

static int gibbs_run_parallel(rsem_b200_ctx* c, const rsem_b200_gibbs_params* p, int32_t* count_vectors, double* chain_acc,
                              rsem_b200_gibbs_stats* stats) {
    const DevGibbs& g = c->gibbs;
    const int M1 = p->M + 1, nc = p->n_chains;
    long long total_samples = 0;
    std::vector<long long> cv_off(nc);
    for (int t = 0; t < nc; ++t) { cv_off[t] = total_samples; total_samples += p->chain_samples[t]; }
    const size_t acc_per = 4 * (size_t)M1 + p->n_genes;
    const unsigned W = (unsigned)((g.N1 + 31) / 32);

    PArgs a{};
    a.N1 = g.N1;
    a.order = g.order; a.seg_start = g.seg_start; a.n_segs = g.n_segs;
    a.seg_ntr = g.seg_ntr; a.seg_tid_off = g.seg_tid_off; a.comp_tids = g.comp_tids;
    a.p_off = reinterpret_cast<const unsigned long long*>(g.p_off); a.p_sid = g.p_sid; a.p_con = g.p_con;
    a.M = p->M; a.burnin = p->burnin; a.gap = p->gap; a.n_genes = p->n_genes; a.n_chains = nc;
    a.n0 = p->n0; a.totc = p->totc;
    a.n_words = W;

    // co-resident CTAs: chains run in waves, every chain gets the same number of worker CTAs (one lane group per component
    // is all the parallelism a sweep has) + 1 generator CTA
    // RSEM_B200_GIBBS_PF: 2 (default) pipelined walk with both lane groups of a warp in one loop, 1 pipelined walk per
    // segment, 0 row-at-a-time walk (prefetch distance 1); 0 and 1 are kept as cross-checks
    const char* pf_env = getenv("RSEM_B200_GIBBS_PF");
    const int pf = pf_env ? std::max(0, std::min(2, atoi(pf_env))) : 2;
    void* kernel = pf == 2 ? (void*)gibbs_parallel_kernel<2> : pf == 1 ? (void*)gibbs_parallel_kernel<1> : (void*)gibbs_parallel_kernel<0>;
    int per_sm = 0;
    RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (void (*)(const PArgs))kernel, kPThreads, 0));
    const int resident = std::max(1, per_sm) * c->sm_count;
    int ctas = std::max(1, std::min(512, (g.n_segs * kGL + kPThreads - 1) / kPThreads));
    if (const char* e = getenv("RSEM_B200_GIBBS_CTAS")) { const int v = atoi(e); if (v >= 1 && v <= 512) ctas = v; }
    ctas = std::min(ctas, std::max(1, resident / std::min(nc, std::max(1, resident / 2)) - 1));
    const int chains_per_wave = std::max(1, std::min(nc, resident / (ctas + 1)));

    int *d_samples = nullptr, *d_init = nullptr, *d_gene = nullptr, *d_counts = nullptr, *d_counts0 = nullptr, *d_z = nullptr, *d_cv = nullptr,
        *d_pre = nullptr, *d_tot = nullptr;
    unsigned *d_seeds = nullptr, *d_u = nullptr, *d_flips = nullptr;
    long long* d_off = nullptr;
    ChainSync* d_sync = nullptr;
    double *d_alpha = nullptr, *d_eel = nullptr, *d_mw = nullptr, *d_acc = nullptr, *d_tmp = nullptr;
    int rc = 0;
    auto cleanup = [&]() {
        cudaFree(d_samples); cudaFree(d_init); cudaFree(d_gene); cudaFree(d_counts); cudaFree(d_counts0); cudaFree(d_z); cudaFree(d_cv);
        cudaFree(d_pre); cudaFree(d_tot); cudaFree(d_seeds); cudaFree(d_u); cudaFree(d_flips); cudaFree(d_off); cudaFree(d_sync);
        cudaFree(d_alpha); cudaFree(d_eel); cudaFree(d_mw); cudaFree(d_acc); cudaFree(d_tmp);
    };
#define RB_TRY(x) do { rc = (x); if (rc) { cleanup(); return rc; } } while (0)
#define RB_TRYC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cleanup(); return cuda_fail(e_, #x, __FILE__, __LINE__); } } while (0)
    RB_TRY(to_dev(&d_samples, p->chain_samples, nc, c->stream));
    RB_TRY(to_dev(&d_seeds, p->chain_seeds, nc, c->stream));
    RB_TRY(to_dev(&d_off, cv_off.data(), nc, c->stream));
    RB_TRY(to_dev(&d_init, p->init_counts, M1, c->stream));
    RB_TRY(to_dev(&d_alpha, p->pseudo_counts, M1, c->stream));
    RB_TRY(to_dev(&d_eel, p->eel, M1, c->stream));
    RB_TRY(to_dev(&d_mw, p->mw, M1, c->stream));
    RB_TRY(to_dev(&d_gene, p->gene_start, (size_t)p->n_genes + 1, c->stream));
    RB_TRYC(cudaMalloc(&d_counts, (size_t)nc * M1 * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_counts0, (size_t)nc * M1 * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_z, (size_t)nc * 2 * g.N1 * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_u, (size_t)nc * 2 * g.N1 * sizeof(unsigned)));
    RB_TRYC(cudaMalloc(&d_flips, (size_t)nc * 4 * W * sizeof(unsigned)));
    RB_TRYC(cudaMalloc(&d_pre, (size_t)nc * W * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_tot, (size_t)nc * ctas * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_sync, (size_t)nc * sizeof(ChainSync)));
    RB_TRYC(cudaMalloc(&d_cv, std::max<size_t>((size_t)total_samples * M1, 1) * sizeof(int)));
    RB_TRYC(cudaMalloc(&d_acc, (size_t)nc * acc_per * sizeof(double)));
    RB_TRYC(cudaMalloc(&d_tmp, (size_t)nc * 2 * M1 * sizeof(double)));
    RB_TRYC(cudaMemsetAsync(d_acc, 0, (size_t)nc * acc_per * sizeof(double), c->stream));
    RB_TRYC(cudaMemsetAsync(d_sync, 0, (size_t)nc * sizeof(ChainSync), c->stream));
    RB_TRYC(cudaMemsetAsync(d_tot, 0, (size_t)nc * ctas * sizeof(int), c->stream));
    a.chain_samples = d_samples; a.chain_seeds = d_seeds; a.chain_cv_offset = d_off; a.init_counts = d_init;
    a.alpha = d_alpha; a.eel = d_eel; a.mw = d_mw; a.gene_start = d_gene; a.counts = d_counts; a.counts_start = d_counts0; a.z = d_z;
    a.ubuf = d_u; a.flips = d_flips; a.pre = d_pre; a.slice_tot = d_tot; a.sync = d_sync; a.count_vectors = d_cv; a.acc = d_acc;
    a.theta_tmp = d_tmp;

    {
        const char* e = getenv("RSEM_B200_GIBBS_FAST");
        a.fast_rows = !(e && !strcmp(e, "0"));
    }
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    const bool timing = getenv("RSEM_B200_TIMING") != nullptr;
    if (timing || stats) { cudaEventCreate(&ev0); cudaEventCreate(&ev1); cudaEventRecord(ev0, c->stream); }
    int waves = 0;
    for (int base = 0; base < nc; base += chains_per_wave) {
        const int wave = std::min(nc - base, chains_per_wave);
        a.chain_base = base;
        a.ctas_per_chain = ctas;
        void* kargs[] = {(void*)&a};
        RB_TRYC(cudaLaunchCooperativeKernel(kernel, dim3(wave * (ctas + 1)), dim3(kPThreads), kargs, 0, c->stream));
        c->launches++;
        ++waves;
    }
    if (timing || stats) cudaEventRecord(ev1, c->stream);
    std::vector<ChainSync> h_sync(nc);
    RB_TRYC(cudaMemcpyAsync(chain_acc, d_acc, (size_t)nc * acc_per * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_TRYC(cudaMemcpyAsync(count_vectors, d_cv, (size_t)total_samples * M1 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    RB_TRYC(cudaMemcpyAsync(h_sync.data(), d_sync, (size_t)nc * sizeof(ChainSync), cudaMemcpyDeviceToHost, c->stream));
    RB_TRYC(cudaStreamSynchronize(c->stream));
    cleanup();
#undef RB_TRY
#undef RB_TRYC
    if (timing || stats) {
        float ms = 0;
        cudaEventElapsedTime(&ms, ev0, ev1);
        cudaEventDestroy(ev0); cudaEventDestroy(ev1);
        if (stats) *stats = rsem_b200_gibbs_stats{ms, ctas, waves};
        unsigned max_passes = 0;
        for (int t = 0; t < nc; ++t) max_passes = std::max(max_passes, h_sync[t].passes);
        if (timing)
            fprintf(stderr, "gibbs kernels: %.2f ms on the device (walk variant %d, fast rows %d), most passes of a chain %u\n", ms, pf,
                    a.fast_rows, max_passes);
    }
    if (timing)
        fprintf(stderr, "gibbs chain 0 (%d worker CTAs, %d segments): %u passes; worker CTA 0 thread 0 cycles: wait for uniforms %llu, passes %llu, "
                "barriers + bookkeeping %llu (incl. the passes), per-sample work %llu\n", ctas, g.n_segs, h_sync[0].passes, h_sync[0].prof[0],
                h_sync[0].prof[1], h_sync[0].prof[2], h_sync[0].prof[3]);
    for (int t = 0; t < nc; ++t)
        if (h_sync[t].err) {
            set_error("gibbs: categorical draw fell off the cumulative array (reference: assert(l < len), sampling.h:62)");
            return RSEM_B200_ERR_ARG;
        }
    return 0;
}

int gibbs_run(rsem_b200_ctx* c, const rsem_b200_gibbs_params* p, int32_t* count_vectors, double* chain_acc,
              rsem_b200_gibbs_stats* stats) {
    // a row without entries has nothing to draw from (both kernels would fall off its empty cumulative array)
    if (c->gibbs.empty_row) { set_error("gibbs: a read without any entry (the .ofg writer never emits one)"); return RSEM_B200_ERR_ARG; }
    const char* mode = getenv("RSEM_B200_GIBBS");   // "serial" = the one-warp-per-chain kernel (cross-check / debugging)
    if (mode && !strcmp(mode, "serial")) return gibbs_run_serial(c, p, count_vectors, chain_acc, stats);
    // tiny inputs: a 624-word regeneration would span more than two sweeps (the generator runs only one sweep ahead)
    if (c->gibbs.N1 < 1248 || !c->gibbs.order) return gibbs_run_serial(c, p, count_vectors, chain_acc, stats);
    return gibbs_run_parallel(c, p, count_vectors, chain_acc, stats);
}

// ---- K13 host side ------------------------------------------------------------------------------------------------------
namespace {
constexpr int kBatchMaxWorkers = 8;   // worker CTAs per team; slice totals are sized for it
constexpr int kBatchDefaultWorkers = 2;

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// byte offsets of a sample's parts in its block; n_segs <= N1 and comp_tids <= M + 1 bound the layout before it is built
struct GParts {
    size_t order, p_off, p_sid, p_con, seg_start, seg_ntr, seg_tid_off, comp_tids, init, alpha, eel, mw, gene, samples, seeds,
        cv_off, head, sync, slice_tot, acc, zero_end, cv, total;
};
GParts gparts(uint64_t N1, uint64_t E, int M, int n_genes, int n_samples, int n_chains) {
    const size_t M1 = (size_t)M + 1;
    GParts p{};
    size_t at = 0;
    auto put = [&](size_t& off, size_t bytes) { off = at; at = align_up(at + bytes); };
    put(p.order, N1 * 4);
    put(p.p_off, (N1 + 1) * 8);
    put(p.p_sid, (E + 16) * 4);
    put(p.p_con, (E + 16) * 8);
    put(p.seg_start, (N1 + 1) * 4);
    put(p.seg_ntr, std::max<uint64_t>(N1, 1) * 4);
    put(p.seg_tid_off, (N1 + 1) * 4);
    put(p.comp_tids, (M1 + 1) * 4);
    put(p.init, M1 * 4);
    put(p.alpha, M1 * 8);
    put(p.eel, M1 * 8);
    put(p.mw, M1 * 8);
    put(p.gene, ((size_t)n_genes + 1) * 4);
    put(p.samples, (size_t)n_chains * 4);
    put(p.seeds, (size_t)n_chains * 4);
    put(p.cv_off, (size_t)n_chains * 8);
    p.head = at;
    put(p.sync, (size_t)n_chains * sizeof(ChainSync));
    put(p.slice_tot, (size_t)n_chains * kBatchMaxWorkers * 4);
    put(p.acc, (size_t)n_chains * (4 * M1 + (size_t)n_genes) * 8);
    p.zero_end = at;
    put(p.cv, (size_t)n_samples * M1 * 4);
    p.total = at;
    return p;
}
}  // namespace

}  // namespace rsem_b200

struct rsem_b200_gibbs_batch {
    struct Slot {
        bool live = false, ran = false;
        void* block = nullptr;
        uint64_t bytes = 0;
        int n_chains = 0, n_samples = 0;
        uint64_t cost = 0;                 // reads x sweeps of its longest chain: the claim order
        std::vector<int32_t> chain_samples;
        rsem_b200::PArgs a{};              // device pointers into the block; scratch pointers are the team's
        size_t sync_off = 0, acc_off = 0, cv_off = 0;
    };
    rsem_b200_ctx* ctx = nullptr;
    uint64_t capacity = 0, used = 0;
    int k = 2;
    int M = -1, n_genes = -1;
    std::vector<Slot> slots;
};

namespace rsem_b200 {

int gibbs_batch_create(rsem_b200_ctx* c, uint64_t capacity, int worker_ctas, rsem_b200_gibbs_batch** out) {
    if (worker_ctas < 0 || worker_ctas > kBatchMaxWorkers) { set_error("gibbs_batch_create: worker_ctas must be 0..8"); return RSEM_B200_ERR_ARG; }
    RB_CUDA(cudaSetDevice(c->device));
    if (capacity == 0) {   // half of the device memory that is free now
        size_t free_b = 0, total_b = 0;
        RB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        capacity = free_b / 2;
    }
    auto* b = new rsem_b200_gibbs_batch();
    b->ctx = c;
    b->capacity = capacity;
    b->k = worker_ctas ? worker_ctas : kBatchDefaultWorkers;
    *out = b;
    return 0;
}

void gibbs_batch_clear(rsem_b200_gibbs_batch* b) {
    cudaSetDevice(b->ctx->device);
    for (auto& s : b->slots)
        if (s.live) cudaFreeAsync(s.block, b->ctx->stream);
    cudaStreamSynchronize(b->ctx->stream);
    b->slots.clear();
    b->used = 0;
    b->M = b->n_genes = -1;
}

void gibbs_batch_destroy(rsem_b200_gibbs_batch* b) {
    gibbs_batch_clear(b);
    delete b;
}

int gibbs_batch_sample_bytes(uint64_t N1, uint64_t E, int32_t M, int32_t n_genes, int32_t n_samples, int32_t n_chains,
                             uint64_t* bytes) {
    if (N1 < RSEM_B200_GIBBS_BATCH_MIN_READS || N1 > RSEM_B200_GIBBS_BATCH_MAX_READS) {
        set_error("the sample is outside the Gibbs batch's size rule (1248 <= N1 <= 2^19 reads): run it with "
                  "rsem_b200_gibbs_upload + rsem_b200_gibbs_run_chains");
        return RSEM_B200_ERR_UNSUPPORTED;
    }
    *bytes = gparts(N1, E, M, n_genes, n_samples, n_chains).total;
    return 0;
}

int gibbs_batch_add(rsem_b200_gibbs_batch* b, uint64_t N1, uint64_t E, const uint64_t* row_ptr, const int32_t* sid,
                    const double* conprb, const rsem_b200_gibbs_params* p, int32_t* slot_out) {
    rsem_b200_ctx* c = b->ctx;
    const int M = p->M, nc = p->n_chains;
    if (b->M >= 0 && (M != b->M || p->n_genes != b->n_genes)) {
        set_error("gibbs_batch_add: every sample of a batch has the M and n_genes of the first");
        return RSEM_B200_ERR_ARG;
    }
    int64_t n_samples = 0;
    uint64_t longest = 0;
    for (int t = 0; t < nc; ++t) {
        if (p->chain_samples[t] < 1) { set_error("gibbs_batch_add: every chain keeps at least one sample"); return RSEM_B200_ERR_ARG; }
        n_samples += p->chain_samples[t];
        longest = std::max<uint64_t>(longest, (uint64_t)p->burnin + 2 + (uint64_t)(p->chain_samples[t] - 1) * p->gap);
    }
    uint64_t bytes = 0;
    if (int rc = gibbs_batch_sample_bytes(N1, E, M, p->n_genes, (int32_t)n_samples, nc, &bytes)) return rc;
    if (b->used + bytes > b->capacity) {
        set_error("the Gibbs batch arena is full");
        return RSEM_B200_ERR_FULL;
    }
    GibbsLayout L;
    if (int rc = gibbs_layout(row_ptr, sid, N1, M, L)) return rc;
    // a row without entries has nothing to draw from (as gibbs_run refuses it)
    if (L.empty_row) { set_error("gibbs: a read without any entry (the .ofg writer never emits one)"); return RSEM_B200_ERR_ARG; }
    const GParts q = gparts(N1, E, M, p->n_genes, (int)n_samples, nc);
    const size_t M1 = (size_t)M + 1;
    std::vector<unsigned char> img(q.head, 0);
    auto put = [&](size_t off, const void* src, size_t n) { if (n) memcpy(img.data() + off, src, n); };
    put(q.order, L.order.data(), N1 * 4);
    put(q.p_off, L.p_off.data(), (N1 + 1) * 8);
    put(q.p_sid, L.p_sid.data(), E * 4);
    {
        double* pc = reinterpret_cast<double*>(img.data() + q.p_con);
        for (uint64_t r = 0; r < N1; ++r) {
            const uint64_t src = row_ptr[L.order[r]], n = row_ptr[L.order[r] + 1] - src;
            memcpy(pc + L.p_off[r], conprb + src, n * 8);
        }
    }
    put(q.seg_start, L.seg_start.data(), L.seg_start.size() * 4);
    put(q.seg_ntr, L.seg_ntr.data(), L.seg_ntr.size() * 4);
    put(q.seg_tid_off, L.seg_tid_off.data(), L.seg_tid_off.size() * 4);
    put(q.comp_tids, L.comp_tids.data(), L.comp_tids.size() * 4);
    put(q.init, p->init_counts, M1 * 4);
    put(q.alpha, p->pseudo_counts, M1 * 8);
    put(q.eel, p->eel, M1 * 8);
    put(q.mw, p->mw, M1 * 8);
    put(q.gene, p->gene_start, ((size_t)p->n_genes + 1) * 4);
    put(q.samples, p->chain_samples, (size_t)nc * 4);
    put(q.seeds, p->chain_seeds, (size_t)nc * 4);
    {
        long long* off = reinterpret_cast<long long*>(img.data() + q.cv_off);
        long long at = 0;
        for (int t = 0; t < nc; ++t) { off[t] = at; at += p->chain_samples[t]; }
    }
    RB_CUDA(cudaSetDevice(c->device));
    void* block = nullptr;
    RB_CUDA(cudaMallocAsync(&block, q.total, c->stream));
    RB_CUDA(cudaMemcpyAsync(block, img.data(), q.head, cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaMemsetAsync(static_cast<unsigned char*>(block) + q.head, 0, q.zero_end - q.head, c->stream));   // sync, slice totals, sums
    RB_CUDA(cudaStreamSynchronize(c->stream));   // img goes out of scope

    int slot = -1;
    for (size_t i = 0; i < b->slots.size(); ++i) if (!b->slots[i].live) { slot = (int)i; break; }
    if (slot < 0) { slot = (int)b->slots.size(); b->slots.emplace_back(); }
    auto& s = b->slots[slot];
    s = rsem_b200_gibbs_batch::Slot{};
    s.live = true;
    s.block = block;
    s.bytes = bytes;
    s.n_chains = nc;
    s.n_samples = (int)n_samples;
    s.cost = longest * N1;
    s.chain_samples.assign(p->chain_samples, p->chain_samples + nc);
    s.sync_off = q.sync; s.acc_off = q.acc; s.cv_off = q.cv;
    unsigned char* base = static_cast<unsigned char*>(block);
    PArgs& a = s.a;
    a.N1 = N1;
    a.order = reinterpret_cast<const int*>(base + q.order);
    a.p_off = reinterpret_cast<const unsigned long long*>(base + q.p_off);
    a.p_sid = reinterpret_cast<const int*>(base + q.p_sid);
    a.p_con = reinterpret_cast<const double*>(base + q.p_con);
    a.seg_start = reinterpret_cast<const int*>(base + q.seg_start);
    a.seg_ntr = reinterpret_cast<const int*>(base + q.seg_ntr);
    a.seg_tid_off = reinterpret_cast<const int*>(base + q.seg_tid_off);
    a.comp_tids = reinterpret_cast<const int*>(base + q.comp_tids);
    a.n_segs = L.n_segs;
    a.fast_rows = 1;
    a.M = M; a.burnin = p->burnin; a.gap = p->gap; a.n_genes = p->n_genes; a.n_chains = nc;
    a.ctas_per_chain = b->k;
    a.chain_samples = reinterpret_cast<const int*>(base + q.samples);
    a.chain_seeds = reinterpret_cast<const unsigned*>(base + q.seeds);
    a.chain_cv_offset = reinterpret_cast<const long long*>(base + q.cv_off);
    a.n0 = p->n0; a.totc = p->totc;
    a.init_counts = reinterpret_cast<const int*>(base + q.init);
    a.alpha = reinterpret_cast<const double*>(base + q.alpha);
    a.eel = reinterpret_cast<const double*>(base + q.eel);
    a.mw = reinterpret_cast<const double*>(base + q.mw);
    a.gene_start = reinterpret_cast<const int*>(base + q.gene);
    a.slice_tot = reinterpret_cast<int*>(base + q.slice_tot);
    a.n_words = (unsigned)((N1 + 31) / 32);
    a.sync = reinterpret_cast<ChainSync*>(base + q.sync);
    a.count_vectors = reinterpret_cast<int*>(base + q.cv);
    a.acc = reinterpret_cast<double*>(base + q.acc);
    b->used += bytes;
    b->M = M;
    b->n_genes = p->n_genes;
    *slot_out = slot;
    return 0;
}

int gibbs_batch_run(rsem_b200_gibbs_batch* b, rsem_b200_gibbs_batch_stats* stats) {
    rsem_b200_ctx* c = b->ctx;
    if (stats) *stats = rsem_b200_gibbs_batch_stats{0, b->k, 0, 0, 0, 0};
    std::vector<int> run;
    for (size_t i = 0; i < b->slots.size(); ++i)
        if (b->slots[i].live && !b->slots[i].ran) run.push_back((int)i);
    if (run.empty()) return 0;
    RB_CUDA(cudaSetDevice(c->device));
    std::vector<PArgs> args;
    std::vector<int2> jobs;
    uint64_t n1_max = 0;
    for (size_t r = 0; r < run.size(); ++r) {
        const auto& s = b->slots[run[r]];
        args.push_back(s.a);
        n1_max = std::max<uint64_t>(n1_max, s.a.N1);
        for (int t = 0; t < s.n_chains; ++t) jobs.push_back(make_int2((int)r, t));
    }
    // largest first: reads x sweeps of the chain, so that the long jobs start first and the short ones fill in behind them
    auto cost = [&](const int2& j) {
        const PArgs& a = args[j.x];
        return a.N1 * (uint64_t)(a.burnin + 2 + (uint64_t)(b->slots[run[j.x]].chain_samples[j.y] - 1) * a.gap);
    };
    std::stable_sort(jobs.begin(), jobs.end(), [&](const int2& x, const int2& y) { return cost(x) > cost(y); });
    int per_sm = 0;
    RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gibbs_batch_kernel, kPThreads, 0));
    const int resident = std::max(1, per_sm) * c->sm_count;
    if (resident < b->k + 1) { set_error("gibbs_batch_run: a team does not fit the device"); return RSEM_B200_ERR_UNSUPPORTED; }
    const int teams = std::min<int>((int)jobs.size(), resident / (b->k + 1));
    const int M1 = b->M + 1;
    const unsigned w_max = (unsigned)((n1_max + 31) / 32);

    BArgs ba{};
    ba.n_jobs = (unsigned)jobs.size();
    ba.k = (unsigned)b->k;
    ba.n1_max = n1_max;
    ba.w_max = w_max;
    ba.M1 = M1;
    void* scratch = nullptr;
    const size_t per_team[] = {(size_t)M1 * 4, (size_t)M1 * 4, 2 * n1_max * 4, 2 * n1_max * 4, 4 * (size_t)w_max * 4,
                               (size_t)w_max * 4, 2 * (size_t)M1 * 8};
    size_t off[8] = {0};
    for (int i = 0; i < 7; ++i) off[i + 1] = off[i] + align_up(per_team[i] * teams);
    const size_t head = align_up(args.size() * sizeof(PArgs)) + align_up(jobs.size() * sizeof(int2)) + 256 + align_up(teams * 8ull);
    RB_CUDA(cudaMallocAsync(&scratch, off[7] + head, c->stream));
    unsigned char* sb = static_cast<unsigned char*>(scratch);
    ba.counts = reinterpret_cast<int*>(sb + off[0]);
    ba.counts_start = reinterpret_cast<int*>(sb + off[1]);
    ba.z = reinterpret_cast<int*>(sb + off[2]);
    ba.ubuf = reinterpret_cast<unsigned*>(sb + off[3]);
    ba.flips = reinterpret_cast<unsigned*>(sb + off[4]);
    ba.pre = reinterpret_cast<int*>(sb + off[5]);
    ba.theta_tmp = reinterpret_cast<double*>(sb + off[6]);
    unsigned char* hp = sb + off[7];
    ba.samples = reinterpret_cast<const PArgs*>(hp);
    hp += align_up(args.size() * sizeof(PArgs));
    ba.jobs = reinterpret_cast<const int2*>(hp);
    hp += align_up(jobs.size() * sizeof(int2));
    ba.next_job = reinterpret_cast<unsigned*>(hp);
    ba.mailbox = reinterpret_cast<unsigned long long*>(hp + 256);
    int rc = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    auto fail = [&](cudaError_t e, const char* what) {
        if (!rc) rc = cuda_fail(e, what, __FILE__, __LINE__);
    };
    cudaError_t e = cudaMemcpyAsync((void*)ba.samples, args.data(), args.size() * sizeof(PArgs), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)ba.jobs, jobs.data(), jobs.size() * sizeof(int2), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(hp, 0, 256 + align_up(teams * 8ull), c->stream);
    if (e == cudaSuccess) e = cudaEventCreate(&ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&ev1);
    if (e == cudaSuccess) e = cudaEventRecord(ev0, c->stream);
    if (e == cudaSuccess) {
        void* kargs[] = {(void*)&ba};
        e = cudaLaunchCooperativeKernel((void*)gibbs_batch_kernel, dim3(teams * (b->k + 1)), dim3(kPThreads), kargs, 0, c->stream);
        c->launches++;
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev1, c->stream);
    if (e != cudaSuccess) fail(e, "gibbs_batch_kernel launch");
    cudaFreeAsync(scratch, c->stream);
    e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) fail(e, "cudaStreamSynchronize");
    float ms = 0;
    if (!rc && cudaEventElapsedTime(&ms, ev0, ev1) != cudaSuccess) ms = 0;
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (rc) return rc;
    bool err = false;
    uint64_t chain_cyc = 0, sample_cyc = 0;
    for (int i : run) {
        auto& s = b->slots[i];
        std::vector<ChainSync> sy(s.n_chains);
        RB_CUDA(cudaMemcpy(sy.data(), static_cast<unsigned char*>(s.block) + s.sync_off, s.n_chains * sizeof(ChainSync),
                           cudaMemcpyDeviceToHost));
        for (const ChainSync& y : sy) {
            err = err || y.err;
            chain_cyc += y.prof[0] + y.prof[2] + y.prof[3];
            sample_cyc += y.prof[3];
        }
        s.ran = true;
    }
    if (stats) *stats = rsem_b200_gibbs_batch_stats{ms, b->k, teams, (int64_t)jobs.size(), chain_cyc, sample_cyc};
    if (err) {
        set_error("gibbs: categorical draw fell off the cumulative array (reference: assert(l < len), sampling.h:62)");
        return RSEM_B200_ERR_ARG;
    }
    return 0;
}

int gibbs_batch_result(rsem_b200_gibbs_batch* b, int32_t slot, int32_t* count_vectors, double* chain_acc) {
    if (slot < 0 || slot >= (int)b->slots.size() || !b->slots[slot].live) { set_error("no sample in this slot"); return RSEM_B200_ERR_ARG; }
    const auto& s = b->slots[slot];
    if (!s.ran) { set_error("gibbs_batch_result: the sample has not run yet"); return RSEM_B200_ERR_ARG; }
    rsem_b200_ctx* c = b->ctx;
    const size_t M1 = (size_t)b->M + 1, acc_per = 4 * M1 + (size_t)b->n_genes;
    RB_CUDA(cudaSetDevice(c->device));
    const unsigned char* base = static_cast<const unsigned char*>(s.block);
    RB_CUDA(cudaMemcpyAsync(count_vectors, base + s.cv_off, (size_t)s.n_samples * M1 * 4, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaMemcpyAsync(chain_acc, base + s.acc_off, (size_t)s.n_chains * acc_per * 8, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

}  // namespace rsem_b200
