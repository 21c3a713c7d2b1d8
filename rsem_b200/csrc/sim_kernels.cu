// rsem-simulate-reads on the device (simulation.cpp:86-130 and the four Model::simulate functions).
//
// The reference draws every random decision from ONE boost::mt19937 stream: u = word * 2^-32, then either a compare
// (Orientation), a scaled truncation (RSPD without estRSPD, the zero-row fallback) or simul::sample, a binary search on
// a cumulative array (simul.h:17-36).  No libm function is involved, so the device reproduces the reference's reads
// exactly.  The stream is processed in windows of W words:
//
//   1. sim_mt_kernel       one CTA continues the mt19937 stream (state in shared memory; the 624-word twist in its four
//                          dependent phases, tempering in parallel) and writes the window's words.  It runs one window
//                          ahead on its own stream, into the other of two buffers;
//   2. sim_len_kernel      for every start position p of the window, a dry run of Model::simulate gives the number of
//                          words an attempt starting at p consumes and whether it succeeds.  Without a reachable
//                          all-zero table row (host decides) the body costs one word per quality value and per base,
//                          so the dry run stops after the mate lengths;
//   3. the chain p -> p + len[p] from the window's entry point, by pointer doubling: K levels of jump tables
//                          (sim_double_kernel), then K + 1 marking passes from the entry point (sim_mark_kernel); the
//                          marked starts are compacted in order, their successes counted by a scan, and the first
//                          N - done successes kept; the failures before them are the reference's resimulation count;
//   4. sim_head_kernel     per successful attempt: the read's name fields and byte sizes; an exclusive scan gives the
//                          offsets;
//   5. sim_write_kernel    per successful attempt: the FASTA / FASTQ text of its mate(s), and counts[sid] += 1.
//
// A window's words extend past its last start position by the longest possible attempt, so every attempt that starts
// inside the window is complete; the chain's first position past the window is the next window's entry point.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <memory>
#include <type_traits>
#include <vector>

#include "common.cuh"

// several contexts, each owning every G-th window (sim_begin_devices)
struct rsem_b200_sim_multi {
    std::vector<rsem_b200_ctx*> ctx;
    uint64_t N = 0, done = 0;
    uint64_t window = 0;   // the window sim_next_devices resolves next, on context window % G
    uint32_t entry = 0;    // its entry point
    double handoff_ms = 0;
};

namespace rsem_b200 {

namespace {

constexpr int kQ = 100;   // QualDist / QProfile SIZE
constexpr int kMtN = 624;

struct SimTables {
    int type, M;
    const double* theta_cdf;
    double ori0;
    int gld_lb, gld_ub;
    const double* gld_cdf;
    int has_mld, mld_lb, mld_ub;
    const double* mld_cdf;
    int est_rspd;
    const uint64_t* rspd_off;
    const double* rspd_cdf;
    const double* qd_init;
    const double* qd_tran;
    const double* pro;
    const double* noise;
    const uint64_t* seq_off;
    const uint8_t* seq;
    const int32_t* tot_len;
    const int32_t* full_len;
};

struct Cur {
    const uint32_t* w;
    uint64_t p;
    __device__ double u() { return __ldg(w + p++) * (1.0 / 4294967296.0); }  // boost uniform_01 on a 32-bit engine
};

// simul::sample (simul.h:17-36): first l with arr[l] > u * arr[len - 1]; an all-zero row draws a second word
__device__ int sample(const double* arr, int len, Cur& c) {
    const double prb = __dmul_rn(c.u(), __ldg(arr + len - 1));
    int l = 0, r = len - 1;
    while (l <= r) {
        const int mid = (l + r) / 2;
        if (__ldg(arr + mid) <= prb) l = mid + 1;
        else r = mid - 1;
    }
    if (l >= len) l = int(__dmul_rn(c.u(), (double)len));
    return l;
}

// LenDist::simulate (LenDist.h:255-262): -1 without a draw when refL <= lb or the cdf is 0
__device__ int lendist(const double* cdf, int lb, int ub, int refL, Cur& c) {
    if (refL == -1) refL = ub;
    if (refL <= lb) return -1;
    const int dlen = min(ub, refL) - lb;
    if (__ldg(cdf + dlen) <= 0.0) return -1;
    return lb + 1 + sample(cdf + 1, dlen, c);
}

enum Mode { kCount = 0, kWalk = 1, kWrite = 2 };

// RefSeq::get_id (RefSeq.h:84-87) on forward-strand codes 0..4
__device__ __forceinline__ int ref_id(const SimTables& t, int sid, int pos, int dir) {
    const int tot = t.tot_len[sid];
    if (dir == 0) return t.seq[t.seq_off[sid] + pos];
    const int b = t.seq[t.seq_off[sid] + tot - pos - 1];
    return b < 4 ? 3 - b : 4;
}

__device__ __forceinline__ char base_char(int id) { return "ACGTN"[id]; }

// one mate's qualities and bases: QualDist::simulate + (Noise)(Q)Profile::simulate.  sid 0 is noise.
// kCount adds the draws without looking at them (valid only without a reachable all-zero row).
// Q models: the quality chain is replayed by a second cursor while the bases are drawn, so nothing is stored.
template <int MODE>
__device__ void body(const SimTables& t, Cur& c, int len, int sid, int pos, int dir, char* seq_out, char* qual_out) {
    const bool q = t.type & 1;
    if (MODE == kCount) {
        c.p += (uint64_t)(q ? max(len, 1) : 0) + (uint64_t)max(len, 0);
        return;
    }
    if (q) {
        Cur cq = c;
        int qv = sample(t.qd_init, kQ, c);
        if (MODE == kWrite) qual_out[0] = (char)(qv + 33);
        for (int i = 1; i < len; ++i) {
            qv = sample(t.qd_tran + qv * kQ, kQ, c);
            if (MODE == kWrite) qual_out[i] = (char)(qv + 33);
        }
        qv = sample(t.qd_init, kQ, cq);
        for (int i = 0; i < len; ++i) {
            if (i > 0) qv = sample(t.qd_tran + qv * kQ, kQ, cq);
            const double* row = sid == 0 ? t.noise + qv * 5 : t.pro + (qv * 5 + ref_id(t, sid, i + pos, dir)) * 5;
            const int b = sample(row, 5, c);
            if (MODE == kWrite) seq_out[i] = base_char(b);
        }
    } else {
        for (int i = 0; i < len; ++i) {
            const double* row = sid == 0 ? t.noise : t.pro + (i * 5 + ref_id(t, sid, i + pos, dir)) * 5;
            const int b = sample(row, 5, c);
            if (MODE == kWrite) seq_out[i] = base_char(b);
        }
    }
}

struct Head {
    int sid, dir, pos, insertL, len[2];
};

// Model::simulate (SingleModel.h:413-452, SingleQModel.h:428-471, PairedEndModel.h:372-415, PairedEndQModel.h:386-433).
// Returns false for a failed attempt (the caller's while loop redraws).  kWrite fills the mates' seq / qual text.
template <int MODE>
__device__ bool attempt(const SimTables& t, Cur& c, Head& h, char* seq_out[2], char* qual_out[2]) {
    const bool paired = t.type >= 2;
    h.sid = sample(t.theta_cdf, t.M + 1, c);
    h.dir = h.pos = h.insertL = 0;
    h.len[1] = 0;
    if (h.sid == 0) {
        if (paired) {
            for (int m = 0; m < 2; ++m) {
                h.len[m] = lendist(t.mld_cdf, t.mld_lb, t.mld_ub, -1, c);
                body<MODE>(t, c, h.len[m], 0, 0, 0, seq_out[m], qual_out[m]);
            }
        } else {
            h.len[0] = t.has_mld ? lendist(t.mld_cdf, t.mld_lb, t.mld_ub, -1, c) : lendist(t.gld_cdf, t.gld_lb, t.gld_ub, -1, c);
            body<MODE>(t, c, h.len[0], 0, 0, 0, seq_out[0], qual_out[0]);
        }
        return true;
    }
    const int sid = h.sid, tot = t.tot_len[sid], full = t.full_len[sid];
    h.dir = c.u() < t.ori0 ? 0 : 1;  // Orientation::simulate
    const int frag = lendist(t.gld_cdf, t.gld_lb, t.gld_ub, tot, c);
    if (frag < 0) return false;
    const int effL = min(full, tot - frag + 1);
    int pos;
    if (t.est_rspd) {  // RSPD::simulate (RSPD.h:195-198)
        const double* arr = t.rspd_cdf + t.rspd_off[sid];
        pos = __ldg(arr + effL - 1) > 0.0 ? sample(arr, effL, c) : -1;
    } else {
        pos = int(__dmul_rn(c.u(), (double)effL));
    }
    if (pos < 0) return false;
    if (h.dir > 0) pos = tot - pos - frag;
    h.pos = pos;
    if (paired) {
        h.insertL = frag;
        h.len[0] = lendist(t.mld_cdf, t.mld_lb, t.mld_ub, frag, c);
        body<MODE>(t, c, h.len[0], sid, pos, h.dir, seq_out[0], qual_out[0]);
        h.len[1] = lendist(t.mld_cdf, t.mld_lb, t.mld_ub, frag, c);
        body<MODE>(t, c, h.len[1], sid, tot - pos - frag, !h.dir, seq_out[1], qual_out[1]);
    } else if (t.has_mld) {
        h.len[0] = lendist(t.mld_cdf, t.mld_lb, t.mld_ub, frag, c);
        if (h.len[0] < 0) return false;
        body<MODE>(t, c, h.len[0], sid, pos, h.dir, seq_out[0], qual_out[0]);
    } else {
        h.len[0] = frag;
        body<MODE>(t, c, frag, sid, pos, h.dir, seq_out[0], qual_out[0]);
    }
    return true;
}

// ---- 1. the mt19937 stream ------------------------------------------------------------------------------------------
// boost's twist of the 624 words in shared memory, thread k of 624 owning word k.  Phase i uses mt[i + 1] (old) and
// mt[i + 397 mod 624], new from phase i - 1 for i >= 227.  Ends with a barrier.
__device__ __forceinline__ void mt_twist(uint32_t* mt, int k) {
    auto twist = [&](int i, uint32_t next) {
        const uint32_t y = (mt[i] & 0x80000000u) | (next & 0x7fffffffu);
        return mt[(i + 397) % kMtN] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    };
    uint32_t v = 0;
    if (k < 227) v = twist(k, mt[k + 1]);
    __syncthreads();
    if (k < 227) mt[k] = v;
    __syncthreads();
    if (k >= 227 && k < 454) v = twist(k, mt[k + 1]);
    __syncthreads();
    if (k >= 227 && k < 454) mt[k] = v;
    __syncthreads();
    if (k >= 454 && k < 623) v = twist(k, mt[k + 1]);
    __syncthreads();
    if (k >= 454 && k < 623) mt[k] = v;
    __syncthreads();
    if (k == 623) mt[k] = twist(k, mt[0]);
    __syncthreads();
}

// state[0..623] = the engine's words, state[624] = its index (boost: i == n means "twist before the next draw")
__global__ void __launch_bounds__(kMtN) sim_mt_kernel(uint32_t* __restrict__ state, uint32_t* __restrict__ out, uint64_t n) {
    __shared__ uint32_t mt[kMtN];
    __shared__ int idx_s;
    const int k = threadIdx.x;
    mt[k] = state[k];
    if (k == 0) idx_s = (int)state[kMtN];
    __syncthreads();
    int idx = idx_s;
    uint64_t done = 0;
    while (done < n) {
        if (idx >= kMtN) {
            mt_twist(mt, k);
            idx = 0;
        }
        const uint64_t take = min((uint64_t)(kMtN - idx), n - done);
        if (k >= idx && (uint64_t)(k - idx) < take) {
            uint32_t y = mt[k];
            y ^= y >> 11;
            y ^= (y << 7) & 0x9d2c5680u;
            y ^= (y << 15) & 0xefc60000u;
            y ^= y >> 18;
            out[done + (k - idx)] = y;
        }
        done += take;
        idx += (int)take;
    }
    __syncthreads();
    state[k] = mt[k];
    if (k == 0) state[kMtN] = (uint32_t)idx;
}

// The jump of several devices' generators (mt_jump.cpp has the method and its host twin).  The state's array moves
// one twist, to S, then by g(T) S with g cut into blocks h_b of 624 coefficients:
// conv[b][j] = sum_i h_b,i s_{i + j} over the 1248 words s = (S, twist(S)), one CTA per block (they are independent);
__global__ void __launch_bounds__(kMtN) sim_mt_jump_conv_kernel(const uint32_t* __restrict__ state,
                                                                const uint32_t* __restrict__ poly,
                                                                uint32_t* __restrict__ conv) {
    __shared__ uint32_t s[2 * kMtN];
    __shared__ uint32_t h[kMtBlockWords];
    const int k = threadIdx.x, b = blockIdx.x;
    s[k] = state[k];
    if (k < kMtBlockWords) h[k] = poly[b * kMtBlockWords + k];
    __syncthreads();
    mt_twist(s, k);
    s[kMtN + k] = s[k];
    __syncthreads();
    mt_twist(s + kMtN, k);
    uint32_t acc = 0;
#pragma unroll 1
    for (int wi = 0; wi < kMtBlockWords; ++wi) {
        const uint32_t w = h[wi];
        const int base = wi * 32 + k;
#pragma unroll
        for (int i = 0; i < 32; ++i)
            if (wi * 32 + i < kMtN) acc ^= s[base + i] & (0u - ((w >> i) & 1u));
    }
    conv[b * kMtN + k] = acc;
}

// then Horner's rule over the blocks, acc = twist(acc) ^ conv[b] from the last block down, and the new index.
// nb == 0: the array stays, only the index moves.
__global__ void __launch_bounds__(kMtN) sim_mt_jump_horner_kernel(uint32_t* __restrict__ state,
                                                                  const uint32_t* __restrict__ conv, int nb,
                                                                  uint32_t idx) {
    __shared__ uint32_t mt[kMtN];
    const int k = threadIdx.x;
    if (nb > 0) {
        mt[k] = conv[(nb - 1) * kMtN + k];
        __syncthreads();
        for (int b = nb - 2; b >= 0; --b) {
            mt_twist(mt, k);
            mt[k] ^= conv[b * kMtN + k];
            __syncthreads();
        }
        state[k] = mt[k];
    }
    if (k == 0) state[kMtN] = idx;
}

// ---- 2. attempt lengths -----------------------------------------------------------------------------------------------
// len[p] = words consumed by an attempt starting at p, bit 31 set when it succeeds; jump[p] = the next attempt's start,
// clamped to the sink W.  Positions before the entry point `first` point at the sink.
template <int MODE>
__global__ void sim_len_kernel(SimTables t, const uint32_t* __restrict__ words, uint32_t first, uint32_t W,
                               uint32_t* __restrict__ len, uint32_t* __restrict__ jump) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > W) return;
    if (p < first || p == W) { jump[p] = W; return; }
    Cur c{words, p};
    Head h;
    char* none[2] = {nullptr, nullptr};
    const bool ok = attempt<MODE>(t, c, h, none, none);
    const uint32_t n = (uint32_t)(c.p - p);
    len[p] = n | (ok ? 0x80000000u : 0u);
    jump[p] = min(p + n, W);
}

// ---- 3. the chain of attempts, by pointer doubling -------------------------------------------------------------------
// level k: jump_k[p] = jump_{k-1}[jump_{k-1}[p]], the start 2^k attempts after p
__global__ void sim_double_kernel(const uint32_t* __restrict__ prev, uint32_t* __restrict__ next, uint32_t first, uint32_t W) {
    const uint32_t p = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (p <= W) next[p] = prev[prev[p]];
}

// From the entry point alone, levels K..0 mark the starts at distances 0 .. 2^(K+1) - 1 along the chain: after level k
// every marked node also marks the node 2^k attempts further.  A node marked earlier in the same pass only adds more
// nodes of the same chain, so the marked set is exactly the chain once 2^(K+1) exceeds its length.
__global__ void sim_mark_kernel(const uint32_t* __restrict__ jump, uint8_t* __restrict__ mark, uint32_t first, uint32_t W) {
    const uint32_t p = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (p < W && mark[p]) mark[jump[p]] = 1;
}

__global__ void sim_okflag_kernel(const uint32_t* __restrict__ chain, const uint32_t* __restrict__ n_chain,
                                  const uint32_t* __restrict__ len, uint32_t* __restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *n_chain) ok[i] = len[chain[i]] >> 31;
}

// cum = inclusive count of successes along the chain.  The first `need` successes are the reads of this window; the
// reference's loop stops at the N-th success, so failures after it are never drawn.
// io[0] = the next window's entry (absolute in this window's frame), io[1] = successes, io[2] = failures
__global__ void sim_cut_kernel(const uint32_t* __restrict__ chain, const uint32_t* __restrict__ n_chain_p,
                               const uint32_t* __restrict__ cum, const uint32_t* __restrict__ len, uint64_t need,
                               uint32_t* __restrict__ starts, uint64_t* __restrict__ io) {
    const uint32_t n_chain = *n_chain_p;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chain) return;
    const uint32_t p = chain[i];
    const bool ok = len[p] >> 31;
    if (ok && cum[i] <= need) starts[cum[i] - 1] = p;
    if (ok && cum[i] == need) {  // the N-th read of the run
        io[1] = need;
        io[2] = i + 1 - need;
        io[0] = (uint64_t)p + (len[p] & 0x7fffffffu);
    } else if (i == n_chain - 1 && cum[i] < need) {
        io[1] = cum[i];
        io[2] = n_chain - cum[i];
        io[0] = (uint64_t)p + (len[p] & 0x7fffffffu);
    }
}

// ---- 4. read heads and text sizes ---------------------------------------------------------------------------------------
__device__ __forceinline__ int dec_len(long long v) {
    int n = v < 0 ? 2 : 1;
    unsigned long long a = v < 0 ? (unsigned long long)(-v) : (unsigned long long)v;
    while (a >= 10) { a /= 10; ++n; }
    return n;
}
__device__ __forceinline__ char* put_dec(char* o, long long v) {
    if (v < 0) { *o++ = '-'; v = -v; }
    char tmp[24];
    int n = 0;
    unsigned long long a = (unsigned long long)v;
    do { tmp[n++] = (char)('0' + a % 10); a /= 10; } while (a);
    while (n) *o++ = tmp[--n];
    return o;
}

// name "rid_dir_sid_pos[_insertL]" (+ "/1" "/2" for paired reads); record ">name\nseq\n" or "@name\nseq\n+\nqual\n"
__device__ __forceinline__ uint32_t name_len(const Head& h, uint64_t rid, bool paired) {
    uint32_t n = dec_len((long long)rid) + 1 + dec_len(h.dir) + 1 + dec_len(h.sid) + 1 + dec_len(h.pos);
    if (paired) n += 1 + dec_len(h.insertL) + 2;
    return n;
}

template <int MODE>
__global__ void sim_head_kernel(SimTables t, const uint32_t* __restrict__ words, const uint32_t* __restrict__ starts,
                                uint32_t n, uint64_t rid0, Head* __restrict__ heads, uint64_t* __restrict__ bytes0,
                                uint64_t* __restrict__ bytes1) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    Cur c{words, starts[r]};
    Head h;
    char* none[2] = {nullptr, nullptr};
    attempt<MODE>(t, c, h, none, none);
    heads[r] = h;
    const bool q = t.type & 1, paired = t.type >= 2;
    const uint32_t nl = name_len(h, rid0 + r, paired);
    for (int m = 0; m < (paired ? 2 : 1); ++m) {
        const uint32_t sl = max(h.len[m], 0);
        const uint64_t b = q ? 1 + nl + 1 + sl + 1 + 2 + max(h.len[m], 1) + 1 : 1 + nl + 1 + sl + 1;
        (m ? bytes1 : bytes0)[r] = b;
    }
}

__global__ void sim_write_kernel(SimTables t, const uint32_t* __restrict__ words, const uint32_t* __restrict__ starts,
                                 uint32_t n, uint64_t rid0, const Head* __restrict__ heads, const uint64_t* __restrict__ off0,
                                 const uint64_t* __restrict__ off1, char* __restrict__ text0, char* __restrict__ text1,
                                 double* __restrict__ counts) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const Head h = heads[r];
    const bool q = t.type & 1, paired = t.type >= 2;
    char* seq_out[2] = {nullptr, nullptr};
    char* qual_out[2] = {nullptr, nullptr};
    for (int m = 0; m < (paired ? 2 : 1); ++m) {
        char* o = (m ? text1 + off1[r] : text0 + off0[r]);
        *o++ = q ? '@' : '>';
        o = put_dec(o, (long long)(rid0 + r));
        *o++ = '_';
        o = put_dec(o, h.dir);
        *o++ = '_';
        o = put_dec(o, h.sid);
        *o++ = '_';
        o = put_dec(o, h.pos);
        if (paired) {
            *o++ = '_';
            o = put_dec(o, h.insertL);
            *o++ = '/';
            *o++ = (char)('1' + m);
        }
        *o++ = '\n';
        seq_out[m] = o;
        const int sl = max(h.len[m], 0);
        o += sl;
        *o++ = '\n';
        if (q) {
            *o++ = '+';
            *o++ = '\n';
            qual_out[m] = o;
            o += max(h.len[m], 1);
            *o++ = '\n';
        }
    }
    Cur c{words, starts[r]};
    Head h2;
    attempt<kWrite>(t, c, h2, seq_out, qual_out);
    atomicAdd(counts + h.sid, 1.0);
}

}  // namespace

// The state of the context's runs.  A run (sim_begin .. sim_end) fills the fields from `t` to `jump_ms`; the device
// buffers, the generator stream, the events and the host text buffers are kept from run to run and freed by sim_free
// (rsem_b200_ctx_destroy), so that a context running sample after sample (rsem-simulate-reads-batch) makes no
// cudaMalloc / cudaFree call, each of which synchronises the whole device, unless a run needs more than the runs before.
struct SimState {
    bool running = false;          // between sim_begin and sim_end
    SimTables t{};
    bool exact_body = false;
    uint64_t N = 0, done = 0, resim = 0;
    uint32_t W = 0, L = 0, K = 0;
    uint32_t entry = 0;
    uint64_t window = 0;           // index of the window sim_next processes next
    cudaStream_t gen_stream = nullptr;  // the generator runs one window ahead on its own stream
    cudaEvent_t gen_ev[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // per buffer: generation start / end
    cudaEvent_t used_ev[2] = {nullptr, nullptr};                           // per buffer: its window is resolved and read
    cudaEvent_t ph_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // the run's buffers, carved out of `arena` (sim_layout)
    char* arena = nullptr;
    size_t arena_bytes = 0;
    uint32_t* mt = nullptr;          // 625 words
    uint32_t* words[2] = {nullptr, nullptr};  // W + L each
    uint32_t* len = nullptr;         // W
    std::vector<uint32_t*> jump;     // K + 1 levels of W + 1
    uint8_t* mark = nullptr;         // W + 1
    uint32_t* chain = nullptr;       // W
    uint32_t* n_chain = nullptr;
    uint32_t* cum = nullptr;         // W
    uint32_t* starts = nullptr;      // W
    uint64_t* io = nullptr;          // 3
    Head* heads = nullptr;           // R: the most successful attempts a window can hold
    uint32_t R = 0;
    uint64_t* bytes[2] = {nullptr, nullptr};  // R + 1 each: sizes, then offsets
    void* scan_tmp = nullptr;
    size_t scan_tmp_bytes = 0;
    char* text_d[2] = {nullptr, nullptr};
    size_t text_cap[2] = {0, 0};
    std::vector<char> text_h[2][2];  // [slot][mate]: a chunk stays valid until the second following sim_next
    int slot = 0;
    double* counts = nullptr;
    rsem_b200_sim_stats stats{};
    // the reference of rsem_b200_sim_upload_refs, used by runs whose params carry no sequences
    int ref_M = 0;
    void* ref_block = nullptr;
    const uint64_t* ref_seq_off = nullptr;
    const uint8_t* ref_seq = nullptr;
    const int32_t* ref_tot_len = nullptr;
    const int32_t* ref_full_len = nullptr;

    // one of G >= 2 contexts of sim_begin_devices: `window` counts this context's own windows, each W + L fresh words
    // followed by a jump to the start of its next one
    int G = 1;
    uint64_t gen_pos = 0;            // stream position of the generator's state once the enqueued work has run
    uint64_t step_blocks = 0;        // the jump between windows moves the array step_blocks or step_blocks + 1 twists
    uint32_t* step_poly[2] = {nullptr, nullptr};  // kMtJumpBlocks x kMtBlockWords each, for those two
    int step_nb[2] = {0, 0};
    uint32_t* jump_conv = nullptr;   // kMtJumpBlocks x 624
    cudaEvent_t jump_ev[2] = {nullptr, nullptr};       // per buffer: generation done, jump starts
    cudaEvent_t prep_ev[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // per buffer: attempt lengths + tables
    double jump_ms = 0;
};

void sim_free(rsem_b200_ctx* ctx) {
    SimState* s = ctx->sim;
    if (!s) return;
    cudaStreamSynchronize(ctx->stream);
    if (s->gen_stream) cudaStreamSynchronize(s->gen_stream);
    cudaFree(s->arena);
    cudaFree(s->ref_block);
    cudaFree(s->text_d[0]);
    cudaFree(s->text_d[1]);
    for (auto& e : s->gen_ev) for (cudaEvent_t x : e) if (x) cudaEventDestroy(x);
    for (cudaEvent_t x : s->used_ev) if (x) cudaEventDestroy(x);
    for (cudaEvent_t x : s->ph_ev) if (x) cudaEventDestroy(x);
    for (cudaEvent_t x : s->jump_ev) if (x) cudaEventDestroy(x);
    for (auto& e : s->prep_ev) for (cudaEvent_t x : e) if (x) cudaEventDestroy(x);
    if (s->gen_stream) cudaStreamDestroy(s->gen_stream);
    delete s;
    ctx->sim = nullptr;
}

namespace {

// the context's SimState with its generator stream and events, created on first use
int sim_state(rsem_b200_ctx* ctx, SimState** out) {
    if (!ctx->sim) {
        SimState* s = new SimState();
        ctx->sim = s;
        auto make = [&]() -> int {
            RB_CUDA(cudaStreamCreateWithFlags(&s->gen_stream, cudaStreamNonBlocking));
            for (auto& e : s->gen_ev) for (cudaEvent_t& x : e) RB_CUDA(cudaEventCreate(&x));
            for (cudaEvent_t& x : s->used_ev) RB_CUDA(cudaEventCreate(&x));
            for (cudaEvent_t& x : s->ph_ev) RB_CUDA(cudaEventCreate(&x));
            for (cudaEvent_t& x : s->jump_ev) RB_CUDA(cudaEventCreate(&x));
            for (auto& e : s->prep_ev) for (cudaEvent_t& x : e) RB_CUDA(cudaEventCreate(&x));
            return 0;
        };
        if (int rc = make()) { sim_free(ctx); return rc; }
    }
    *out = ctx->sim;
    return 0;
}

// a run's end: nothing of it is left on either stream, its buffers stay for the next run
void sim_stop(rsem_b200_ctx* ctx) {
    SimState* s = ctx->sim;
    if (!s || !s->running) return;
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(s->gen_stream);
    s->running = false;
}

}  // namespace

int sim_upload_refs(rsem_b200_ctx* ctx, int M, const uint64_t* seq_off, const uint8_t* seq, const int32_t* tot_len,
                    const int32_t* full_len) {
    SimState* s = nullptr;
    if (int rc = sim_state(ctx, &s)) return rc;
    RB_ARG(!s->running, "sim_upload_refs: a simulation is running on this context (rsem_b200_sim_end first)");
    cudaFree(s->ref_block);
    s->ref_block = nullptr;
    s->ref_M = 0;
    const size_t n_off = ((size_t)M + 2) * sizeof(uint64_t), n_len = ((size_t)M + 1) * sizeof(int32_t);
    const size_t n_seq = seq_off[M + 1];
    char* b = nullptr;
    RB_CUDA(cudaMalloc(&b, n_off + 2 * n_len + n_seq + 1));
    s->ref_block = b;
    RB_CUDA(cudaMemcpyAsync(b, seq_off, n_off, cudaMemcpyHostToDevice, ctx->stream));
    RB_CUDA(cudaMemcpyAsync(b + n_off, tot_len, n_len, cudaMemcpyHostToDevice, ctx->stream));
    RB_CUDA(cudaMemcpyAsync(b + n_off + n_len, full_len, n_len, cudaMemcpyHostToDevice, ctx->stream));
    if (n_seq) RB_CUDA(cudaMemcpyAsync(b + n_off + 2 * n_len, seq, n_seq, cudaMemcpyHostToDevice, ctx->stream));
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    s->ref_seq_off = reinterpret_cast<const uint64_t*>(b);
    s->ref_tot_len = reinterpret_cast<const int32_t*>(b + n_off);
    s->ref_full_len = reinterpret_cast<const int32_t*>(b + n_off + n_len);
    s->ref_seq = reinterpret_cast<const uint8_t*>(b + n_off + 2 * n_len);
    s->ref_M = M;
    return 0;
}

namespace {

// enqueue the stream words of window w into buffer w % 2 on the generator stream: window 0 takes W + L fresh words;
// later windows start with the last L words of the previous buffer and add W fresh ones
int sim_enqueue_gen(SimState* s, uint64_t w) {
    const int b = (int)(w & 1);
    cudaStream_t gs = s->gen_stream;
    RB_CUDA(cudaStreamWaitEvent(gs, s->used_ev[b], 0));  // window w - 2 is done with this buffer
    RB_CUDA(cudaEventRecord(s->gen_ev[b][0], gs));
    if (w == 0) {
        sim_mt_kernel<<<1, kMtN, 0, gs>>>(s->mt, s->words[0], (uint64_t)s->W + s->L);
    } else {
        RB_CUDA(cudaMemcpyAsync(s->words[b], s->words[1 - b] + s->W, (size_t)s->L * sizeof(uint32_t),
                                cudaMemcpyDeviceToDevice, gs));
        sim_mt_kernel<<<1, kMtN, 0, gs>>>(s->mt, s->words[b] + s->L, (uint64_t)s->W);
    }
    RB_CUDA(cudaEventRecord(s->gen_ev[b][1], gs));
    return 0;
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

}  // namespace

namespace {

// the tables and buffers of a run on the context's kept state; the generator's state is boost::mt19937(seed), or `state`
// (625 words) when given.  G > 1: the run is one of G contexts of sim_begin_devices, which also needs the jump scratch.
int sim_setup(rsem_b200_ctx* ctx, const rsem_b200_sim_params* p, const uint32_t* state, int G) {
    SimState* s = nullptr;
    if (int rc = sim_state(ctx, &s)) return rc;
    sim_stop(ctx);
    const int M = p->M;
    const bool q = p->model_type & 1, paired = p->model_type >= 2;
    const bool own_refs = p->seq != nullptr;
    RB_ARG(own_refs || (s->ref_block && s->ref_M == M),
           "sim_begin: params->seq is NULL and no reference with this M was uploaded (rsem_b200_sim_upload_refs)");
    SimTables& t = s->t;
    t = SimTables{};
    t.type = p->model_type;
    t.M = M;
    t.ori0 = p->ori_prob0;
    t.gld_lb = p->gld.lb;
    t.gld_ub = p->gld.ub;
    t.has_mld = p->has_mld;
    t.mld_lb = p->has_mld ? p->mld.lb : 0;
    t.mld_ub = p->has_mld ? p->mld.ub : 0;
    t.est_rspd = p->est_rspd;
    s->exact_body = p->exact_body != 0;
    s->N = p->N;
    s->done = s->resim = 0;
    s->entry = 0;
    s->window = 0;
    s->slot = 0;
    s->stats = rsem_b200_sim_stats{};
    s->G = G;
    s->gen_pos = s->step_blocks = 0;
    s->step_nb[0] = s->step_nb[1] = 0;
    s->jump_ms = 0;

    // longest attempt: every draw takes at most 2 words; draws = sid, dir, length, position, 2 mate lengths, and per
    // mate max(len, 1) qualities + len bases
    const int maxlen = std::max(p->gld.ub, p->has_mld ? p->mld.ub : 0);
    const uint64_t draws = 6 + (uint64_t)(paired ? 2 : 1) * (2 * (uint64_t)maxlen + 1);
    s->L = (uint32_t)(2 * draws + 8);
    uint64_t W = p->window_words ? p->window_words : (uint64_t)1 << 22;
    W = std::max<uint64_t>(W, s->L);
    RB_ARG(W < 0x7fffffffu - s->L, "window too large");
    s->W = (uint32_t)W;
    s->K = 0;
    while (((uint64_t)1 << (s->K + 1)) <= W) ++s->K;  // 2^(K+1) > W >= any chain length
    // a successful attempt takes at least 2 words (the sid draw and one more), and a window holds at most N reads
    s->R = (uint32_t)std::min<uint64_t>(W / 2 + 1, std::max<uint64_t>(s->N, 1));
    s->jump.assign(s->K + 1, nullptr);
    size_t need = 0, tmp = 0;
    RB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, (uint64_t*)nullptr, (uint64_t*)nullptr, (int)s->R + 1, ctx->stream));
    need = std::max(need, tmp);
    RB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)s->W, ctx->stream));
    need = std::max(need, tmp);
    RB_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, thrust::counting_iterator<uint32_t>(0), (uint8_t*)nullptr,
                                       (uint32_t*)nullptr, (uint32_t*)nullptr, (int)s->W, ctx->stream));
    need = std::max(need, tmp);
    s->scan_tmp_bytes = need;

    // every table and buffer of the run in one arena: the first pass (base nullptr) sizes it, the second points into it
    const uint64_t total_seq = own_refs ? p->seq_off[M + 1] : 0;
    struct Upload { void* dst; const void* src; size_t bytes; };
    std::vector<Upload> up;
    auto layout = [&](char* base) {
        size_t off = 0;
        auto carve = [&](auto*& ptr, size_t n, const void* src = nullptr) {
            using T = std::remove_cv_t<std::remove_reference_t<decltype(*ptr)>>;
            off = (off + 255) & ~(size_t)255;
            T* at = base ? reinterpret_cast<T*>(base + off) : nullptr;
            ptr = at;
            if (base && src && n) up.push_back({at, src, n * sizeof(T)});
            off += std::max<size_t>(n, 1) * sizeof(T);
        };
        carve(t.theta_cdf, (size_t)M + 1, p->theta_cdf);
        carve(t.gld_cdf, (size_t)p->gld.span + 1, p->gld.cdf);
        if (p->has_mld) carve(t.mld_cdf, (size_t)p->mld.span + 1, p->mld.cdf);
        if (p->est_rspd) {
            carve(t.rspd_off, (size_t)M + 2, p->rspd_off);
            carve(t.rspd_cdf, (size_t)p->rspd_off[M + 1], p->rspd_cdf);
        }
        if (q) {
            carve(t.qd_init, kQ, p->qd_init_cdf);
            carve(t.qd_tran, (size_t)kQ * kQ, p->qd_tran_cdf);
        }
        carve(t.pro, (size_t)p->pro_rows * 25, p->profile_cdf);
        carve(t.noise, q ? (size_t)kQ * 5 : 5, p->noise_cdf);
        if (own_refs) {
            carve(t.seq_off, (size_t)M + 2, p->seq_off);
            carve(t.seq, (size_t)total_seq, p->seq);
            carve(t.tot_len, (size_t)M + 1, p->tot_len);
            carve(t.full_len, (size_t)M + 1, p->full_len);
        }
        carve(s->mt, (size_t)kMtN + 1);
        carve(s->words[0], (size_t)s->W + s->L);
        carve(s->words[1], (size_t)s->W + s->L);
        carve(s->len, s->W);
        for (auto& j : s->jump) carve(j, (size_t)s->W + 1);
        carve(s->mark, (size_t)s->W + 1);
        carve(s->chain, s->W);
        carve(s->n_chain, 1);
        carve(s->cum, s->W);
        carve(s->starts, s->R);
        carve(s->io, 3);
        carve(s->heads, s->R);
        carve(s->bytes[0], (size_t)s->R + 1);
        carve(s->bytes[1], (size_t)s->R + 1);
        carve(s->counts, (size_t)M + 1);
        char* scan = nullptr;
        carve(scan, s->scan_tmp_bytes);
        s->scan_tmp = scan;
        if (G > 1) {
            for (auto& sp : s->step_poly) carve(sp, (size_t)kMtJumpBlocks * kMtBlockWords);
            carve(s->jump_conv, (size_t)kMtJumpBlocks * kMtN);
        }
        return off;
    };
    const size_t bytes = layout(nullptr);
    if (bytes > s->arena_bytes) {  // the only allocation of a run, when it needs more than every run before it
        cudaFree(s->arena);
        s->arena = nullptr;
        s->arena_bytes = 0;
        RB_CUDA(cudaMalloc(&s->arena, bytes));
        s->arena_bytes = bytes;
    }
    layout(s->arena);
    if (!own_refs) {
        t.seq_off = s->ref_seq_off;
        t.seq = s->ref_seq;
        t.tot_len = s->ref_tot_len;
        t.full_len = s->ref_full_len;
    }

    std::vector<uint32_t> mt(kMtN + 1);  // boost::mt19937(seed) (mersenne_twister.hpp seed())
    mt[0] = p->seed;
    for (int i = 1; i < kMtN; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    mt[kMtN] = kMtN;
    if (state) mt.assign(state, state + kMtN + 1);
    up.push_back({s->mt, mt.data(), mt.size() * sizeof(uint32_t)});
    for (const Upload& u : up) RB_CUDA(cudaMemcpyAsync(u.dst, u.src, u.bytes, cudaMemcpyHostToDevice, ctx->stream));
    RB_CUDA(cudaMemsetAsync(s->counts, 0, ((size_t)M + 1) * sizeof(double), ctx->stream));
    RB_CUDA(cudaEventRecord(s->used_ev[0], ctx->stream));  // the buffers are free; counts are zeroed first
    RB_CUDA(cudaEventRecord(s->used_ev[1], ctx->stream));
    RB_CUDA(cudaStreamSynchronize(ctx->stream));  // the tables are on the device before the host's copies go away
    s->running = true;
    return 0;
}

}  // namespace

int sim_begin(rsem_b200_ctx* ctx, const rsem_b200_sim_params* p) {
    if (int rc = sim_setup(ctx, p, nullptr, 1)) return rc;
    if (int rc = sim_enqueue_gen(ctx->sim, 0)) return rc;
    ctx->launches += 1;
    return 0;
}

namespace {

constexpr int kTb = 256;

// 2. + the doubling tables of step 3 for the window in `words`, from start position `first` on
void sim_lengths(SimState* s, cudaStream_t st, const uint32_t* words, uint32_t first) {
    const uint32_t W = s->W, span = W - first;
    const unsigned gw = (W + 1 + kTb - 1) / kTb, gs_ = (span + 1 + kTb - 1) / kTb;
    if (s->exact_body) sim_len_kernel<kWalk><<<gw, kTb, 0, st>>>(s->t, words, first, W, s->len, s->jump[0]);
    else sim_len_kernel<kCount><<<gw, kTb, 0, st>>>(s->t, words, first, W, s->len, s->jump[0]);
    for (uint32_t k = 1; k <= s->K; ++k) sim_double_kernel<<<gs_, kTb, 0, st>>>(s->jump[k - 1], s->jump[k], first, W);
}

// 3. the chain of attempts from the entry point `first`, keeping at most `need` successes: io = the exit (in this
// window's frame), the successes and the failures.  Records ph_ev[1] and waits for the stream.
int sim_resolve(SimState* s, cudaStream_t st, uint32_t first, uint64_t need, uint64_t io[3]) {
    const uint32_t W = s->W, span = W - first;
    const unsigned gs_ = (span + 1 + kTb - 1) / kTb;
    RB_CUDA(cudaMemsetAsync(s->mark, 0, (size_t)W + 1, st));
    RB_CUDA(cudaMemsetAsync(s->mark + first, 1, 1, st));
    for (int k = (int)s->K; k >= 0; --k) sim_mark_kernel<<<gs_, kTb, 0, st>>>(s->jump[k], s->mark, first, W);
    RB_CUDA(cub::DeviceSelect::Flagged(s->scan_tmp, s->scan_tmp_bytes, thrust::counting_iterator<uint32_t>(0),
                                       s->mark, s->chain, s->n_chain, (int)W, st));
    sim_okflag_kernel<<<gs_, kTb, 0, st>>>(s->chain, s->n_chain, s->len, s->cum);
    RB_CUDA(cub::DeviceScan::InclusiveSum(s->scan_tmp, s->scan_tmp_bytes, s->cum, s->cum, (int)span, st));
    sim_cut_kernel<<<gs_, kTb, 0, st>>>(s->chain, s->n_chain, s->cum, s->len, need, s->starts, s->io);
    RB_CUDA(cudaMemcpyAsync(io, s->io, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaEventRecord(s->ph_ev[1], st));
    RB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// 4. + 5. the n reads resolved in buffer b, numbered from rid0, as text in the host buffers of the next slot
int sim_emit(rsem_b200_ctx* ctx, SimState* s, int b, uint32_t n, uint64_t rid0, const char* text[2], uint64_t bytes[2]) {
    cudaStream_t st = ctx->stream;
    const uint32_t* words = s->words[b];
    const bool paired = s->t.type >= 2;
    const int nm = paired ? 2 : 1;
    const unsigned gb = (n + kTb - 1) / kTb;
    RB_CUDA(cudaEventRecord(s->ph_ev[0], st));
    if (s->exact_body)
        sim_head_kernel<kWalk><<<gb, kTb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1]);
    else
        sim_head_kernel<kCount><<<gb, kTb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1]);
    uint64_t tot[2] = {0, 0};
    for (int m = 0; m < nm; ++m) {
        RB_CUDA(cudaMemsetAsync(s->bytes[m] + n, 0, sizeof(uint64_t), st));
        RB_CUDA(cub::DeviceScan::ExclusiveSum(s->scan_tmp, s->scan_tmp_bytes, s->bytes[m], s->bytes[m], (int)n + 1, st));
        RB_CUDA(cudaMemcpyAsync(&tot[m], s->bytes[m] + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    }
    RB_CUDA(cudaStreamSynchronize(st));
    // each mate's buffer grows on its own: the context's runs may alternate single-end and paired-end models
    for (int m = 0; m < nm; ++m)
        if (tot[m] > s->text_cap[m]) {
            cudaFree(s->text_d[m]);
            s->text_d[m] = nullptr;
            s->text_cap[m] = 0;
            RB_CUDA(cudaMalloc(&s->text_d[m], tot[m] + tot[m] / 4));
            s->text_cap[m] = tot[m] + tot[m] / 4;
        }
    sim_write_kernel<<<gb, kTb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1],
                                         s->text_d[0], s->text_d[1], s->counts);
    RB_CUDA(cudaEventRecord(s->ph_ev[2], st));
    RB_CUDA(cudaEventRecord(s->used_ev[b], st));
    ctx->launches += 2 + nm;
    auto& th = s->text_h[s->slot];
    s->slot ^= 1;
    for (int m = 0; m < nm; ++m) {
        th[m].resize(tot[m]);
        RB_CUDA(cudaMemcpyAsync(th[m].data(), s->text_d[m], tot[m], cudaMemcpyDeviceToHost, st));
        text[m] = th[m].data();
        bytes[m] = tot[m];
    }
    RB_CUDA(cudaEventRecord(s->ph_ev[3], st));
    RB_CUDA(cudaStreamSynchronize(st));
    RB_CUDA(cudaGetLastError());
    s->stats.reads_ms += elapsed(s->ph_ev[0], s->ph_ev[2]);
    s->stats.copy_ms += elapsed(s->ph_ev[2], s->ph_ev[3]);
    return 0;
}

}  // namespace

int sim_next(rsem_b200_ctx* ctx, const char* text[2], uint64_t bytes[2], uint64_t* n_reads) {
    SimState* s = ctx->sim;
    RB_ARG(s && s->running, "sim_begin must be called first");
    cudaStream_t st = ctx->stream;
    *n_reads = 0;
    bytes[0] = bytes[1] = 0;
    text[0] = text[1] = nullptr;
    while (*n_reads == 0 && s->done < s->N) {
        const uint32_t W = s->W;
        const int b = (int)(s->window & 1);
        // the next window's words are generated while this one is resolved and read
        if (int rc = sim_enqueue_gen(s, s->window + 1)) return rc;
        RB_CUDA(cudaStreamWaitEvent(st, s->gen_ev[b][1], 0));

        RB_CUDA(cudaEventRecord(s->ph_ev[0], st));
        const uint32_t first = s->entry;
        sim_lengths(s, st, s->words[b], first);
        uint64_t io[3];
        if (int rc = sim_resolve(s, st, first, s->N - s->done, io)) return rc;
        ctx->launches += 5 + 2 * s->K + 2;
        s->entry = (uint32_t)(io[0] - W);  // < L: an attempt starting inside the window ends before W + L
        s->resim += io[2];
        const uint32_t n = (uint32_t)io[1];
        s->stats.generate_ms += elapsed(s->gen_ev[b][0], s->gen_ev[b][1]);
        s->stats.resolve_ms += elapsed(s->ph_ev[0], s->ph_ev[1]);
        s->stats.words += s->window == 0 ? (uint64_t)W + s->L : W;
        ++s->window;
        if (n == 0) {
            RB_CUDA(cudaEventRecord(s->used_ev[b], st));
            continue;
        }
        if (int rc = sim_emit(ctx, s, b, n, s->done, text, bytes)) return rc;
        s->stats.windows = s->window;
        s->done += n;
        *n_reads = n;
    }
    return 0;
}

int sim_end(rsem_b200_ctx* ctx, double* counts, uint64_t* resim, rsem_b200_sim_stats* stats) {
    SimState* s = ctx->sim;
    RB_ARG(s && s->running, "sim_begin must be called first");
    if (counts) {
        RB_CUDA(cudaMemcpyAsync(counts, s->counts, ((size_t)s->t.M + 1) * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        RB_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (resim) *resim = s->resim;
    if (stats) { s->stats.windows = s->window; *stats = s->stats; }
    sim_stop(ctx);
    return 0;
}

// ---- several contexts ------------------------------------------------------------------------------------------------
// Window w (words [w W, (w + 1) W + L)) belongs to context w mod G.  A context generates its window's W + L words with
// sim_mt_kernel and then jumps its generator by (G - 1) W - L to the start of its next window (>= 0 as W >= L), on its
// generator stream.  The attempt lengths and doubling tables do not depend on the entry point, so every context works
// them out for its window as soon as the words are there (from start position 0); only the chain from the entry point
// (sim_resolve) runs window after window, the exit of one window handed by the host to the context of the next.
namespace {

// boost's index after pos draws from the seeded state
uint32_t mt_index_at(uint64_t pos) { return pos == 0 ? kMtN : (uint32_t)(pos - (uint64_t)kMtN * ((pos - 1) / kMtN)); }

int sim_enqueue_gen_jump(rsem_b200_ctx* ctx, SimState* s, uint64_t lw) {
    const int b = (int)(lw & 1);
    cudaStream_t gs = s->gen_stream;
    const uint64_t n = (uint64_t)s->W + s->L, J = (uint64_t)(s->G - 1) * s->W - s->L;
    RB_CUDA(cudaStreamWaitEvent(gs, s->used_ev[b], 0));  // window lw - 2 of this context is done with this buffer
    RB_CUDA(cudaEventRecord(s->gen_ev[b][0], gs));
    sim_mt_kernel<<<1, kMtN, 0, gs>>>(s->mt, s->words[b], n);
    RB_CUDA(cudaEventRecord(s->jump_ev[b], gs));
    const MtJumpPlan plan = mt_jump_plan(mt_index_at(s->gen_pos + n), J);
    if (plan.blocks) {
        const int v = (int)(plan.blocks - s->step_blocks);  // 0 or 1: the index before the jump lies in [1, 624]
        sim_mt_jump_conv_kernel<<<s->step_nb[v], kMtN, 0, gs>>>(s->mt, s->step_poly[v], s->jump_conv);
        sim_mt_jump_horner_kernel<<<1, kMtN, 0, gs>>>(s->mt, s->jump_conv, s->step_nb[v], plan.idx);
        ctx->launches += 3;
    } else {
        sim_mt_jump_horner_kernel<<<1, kMtN, 0, gs>>>(s->mt, nullptr, 0, plan.idx);
        ctx->launches += 2;
    }
    s->gen_pos += n + J;
    RB_CUDA(cudaEventRecord(s->gen_ev[b][1], gs));
    return 0;
}

int sim_enqueue_prep(rsem_b200_ctx* ctx, SimState* s, uint64_t lw) {
    const int b = (int)(lw & 1);
    RB_CUDA(cudaStreamWaitEvent(ctx->stream, s->gen_ev[b][1], 0));
    RB_CUDA(cudaEventRecord(s->prep_ev[b][0], ctx->stream));
    sim_lengths(s, ctx->stream, s->words[b], 0);
    RB_CUDA(cudaEventRecord(s->prep_ev[b][1], ctx->stream));
    ctx->launches += 1 + s->K;
    return 0;
}

void stop_all(const std::vector<rsem_b200_ctx*>& ctxs) {
    for (rsem_b200_ctx* c : ctxs) {
        cudaSetDevice(c->device);
        sim_stop(c);
    }
}

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

}  // namespace

int sim_begin_devices(rsem_b200_ctx* const* ctxs, int n, const rsem_b200_sim_params* p, rsem_b200_sim_multi** out) {
    auto m = std::make_unique<rsem_b200_sim_multi>();
    m->ctx.assign(ctxs, ctxs + n);
    m->N = p->N;
    std::vector<uint32_t> seeded(kMtN + 1), state(kMtN + 1);  // boost::mt19937(seed)
    seeded[0] = p->seed;
    for (int i = 1; i < kMtN; ++i) seeded[i] = 1812433253u * (seeded[i - 1] ^ (seeded[i - 1] >> 30)) + (uint32_t)i;
    seeded[kMtN] = kMtN;
    // the jump between a context's windows moves its array step_blocks or step_blocks + 1 twists; g = x^(624 (k - 1))
    uint64_t step_blocks = 0;
    std::vector<uint32_t> step_h[2];
    int step_nb[2] = {0, 0};
    for (int g = 0; g < n; ++g) {
        rsem_b200_ctx* ctx = ctxs[g];
        auto fail = [&](int rc) { stop_all(m->ctx); return rc; };
        if (cudaSetDevice(ctx->device) != cudaSuccess) return fail(cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__));
        if (int rc = sim_setup(ctx, p, nullptr, n)) return fail(rc);
        SimState* s = ctx->sim;
        if (g == 0) {
            const uint64_t J = (uint64_t)(n - 1) * s->W - s->L;
            step_blocks = J / kMtN;
            for (int v = 0; v < 2; ++v) {
                if (step_blocks + v == 0) continue;
                std::vector<uint64_t> poly(kMtPolyWords);
                if (!mt_jump_poly((step_blocks + v - 1) * kMtN, poly.data())) {
                    set_error("sim_begin_devices: mt19937 characteristic polynomial not found");
                    return fail(RSEM_B200_ERR_CUDA);
                }
                step_h[v].resize(kMtJumpBlocks * kMtBlockWords);
                step_nb[v] = mt_jump_blocks(poly.data(), step_h[v].data());
            }
        }
        s->G = n;
        s->gen_pos = (uint64_t)g * s->W;
        s->step_blocks = step_blocks;
        auto setup = [&]() -> int {
            if (g > 0) {
                if (int rc = rsem_b200_mt19937_jump(seeded.data(), s->gen_pos, state.data())) return rc;
                RB_CUDA(cudaMemcpyAsync(s->mt, state.data(), state.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
            }
            for (int v = 0; v < 2; ++v) {
                s->step_nb[v] = step_nb[v];
                if (!step_h[v].empty())
                    RB_CUDA(cudaMemcpyAsync(s->step_poly[v], step_h[v].data(), step_h[v].size() * sizeof(uint32_t),
                                            cudaMemcpyHostToDevice, ctx->stream));
            }
            // the generator stream waits for these copies (the buffers' events were recorded before them)
            RB_CUDA(cudaEventRecord(s->used_ev[0], ctx->stream));
            RB_CUDA(cudaEventRecord(s->used_ev[1], ctx->stream));
            RB_CUDA(cudaStreamSynchronize(ctx->stream));
            if (int rc = sim_enqueue_gen_jump(ctx, s, 0)) return rc;
            return sim_enqueue_prep(ctx, s, 0);
        };
        if (int rc = setup()) return fail(rc);
    }
    *out = m.release();
    return 0;
}

int sim_next_devices(rsem_b200_sim_multi* m, const char* text[2], uint64_t bytes[2], uint64_t* n_reads) {
    *n_reads = 0;
    bytes[0] = bytes[1] = 0;
    text[0] = text[1] = nullptr;
    const size_t G = m->ctx.size();
    while (*n_reads == 0 && m->done < m->N) {
        rsem_b200_ctx* ctx = m->ctx[m->window % G];
        RB_CUDA(cudaSetDevice(ctx->device));
        SimState* s = ctx->sim;
        RB_ARG(s && s->running, "sim_begin_devices must be called first");
        cudaStream_t st = ctx->stream;
        const uint64_t lw = s->window;
        const int b = (int)(lw & 1);
        // this context's next window is generated while this one is resolved and read
        if (int rc = sim_enqueue_gen_jump(ctx, s, lw + 1)) return rc;
        RB_CUDA(cudaEventRecord(s->ph_ev[0], st));
        const double t0 = now_ms();
        uint64_t io[3];
        if (int rc = sim_resolve(s, st, m->entry, m->N - m->done, io)) return rc;
        m->handoff_ms += now_ms() - t0;
        ctx->launches += 5 + s->K;
        m->entry = (uint32_t)(io[0] - s->W);
        s->resim += io[2];
        const uint32_t n = (uint32_t)io[1];
        s->stats.generate_ms += elapsed(s->gen_ev[b][0], s->jump_ev[b]);
        s->jump_ms += elapsed(s->jump_ev[b], s->gen_ev[b][1]);
        s->stats.resolve_ms += elapsed(s->prep_ev[b][0], s->prep_ev[b][1]) + elapsed(s->ph_ev[0], s->ph_ev[1]);
        s->stats.words += (uint64_t)s->W + s->L;
        s->stats.windows = ++s->window;
        ++m->window;
        if (n == 0) {
            RB_CUDA(cudaEventRecord(s->used_ev[b], st));
        } else {
            if (int rc = sim_emit(ctx, s, b, n, m->done, text, bytes)) return rc;
            m->done += n;
            *n_reads = n;
        }
        if (int rc = sim_enqueue_prep(ctx, s, lw + 1)) return rc;
    }
    return 0;
}

int sim_end_devices(rsem_b200_sim_multi* m, double* counts, uint64_t* resim, rsem_b200_sim_devices_stats* stats,
                    rsem_b200_sim_stats* per_device) {
    std::unique_ptr<rsem_b200_sim_multi> own(m);
    rsem_b200_sim_devices_stats sum{};
    sum.handoff_ms = m->handoff_ms;
    uint64_t r_sum = 0;
    std::vector<double> c;
    for (size_t g = 0; g < m->ctx.size(); ++g) {
        rsem_b200_ctx* ctx = m->ctx[g];
        RB_CUDA(cudaSetDevice(ctx->device));
        SimState* s = ctx->sim;
        if (!s || !s->running) {
            stop_all(m->ctx);
            RB_ARG(false, "sim_begin_devices must be called first");
        }
        if (counts && c.empty()) c.assign((size_t)s->t.M + 1, 0.0);
        const double jump_ms = s->jump_ms;
        std::vector<double> cg(c.size());
        uint64_t r = 0;
        rsem_b200_sim_stats st{};
        if (int rc = sim_end(ctx, counts ? cg.data() : nullptr, &r, &st)) {
            stop_all(m->ctx);
            return rc;
        }
        for (size_t i = 0; i < c.size(); ++i) c[i] += cg[i];  // integers: any order gives the same sums
        r_sum += r;
        sum.jump_ms += jump_ms;
        sum.sum.generate_ms += st.generate_ms;
        sum.sum.resolve_ms += st.resolve_ms;
        sum.sum.reads_ms += st.reads_ms;
        sum.sum.copy_ms += st.copy_ms;
        sum.sum.words += st.words;
        sum.sum.windows += st.windows;
        if (per_device) per_device[g] = st;
    }
    if (counts) std::copy(c.begin(), c.end(), counts);
    if (resim) *resim = r_sum;
    if (stats) *stats = sum;
    return 0;
}

}  // namespace rsem_b200
