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
#include <cstring>
#include <vector>

#include "common.cuh"

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
    auto twist = [&](int i, uint32_t next) {
        const uint32_t y = (mt[i] & 0x80000000u) | (next & 0x7fffffffu);
        return mt[(i + 397) % kMtN] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    };
    while (done < n) {
        if (idx >= kMtN) {
            // phase i uses mt[i + 1] (old) and mt[i + 397 mod 624], new from phase i - 1 for i >= 227
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

template <class T>
T* dev_copy(const T* src, size_t n, std::vector<void*>& owned) {
    T* d = nullptr;
    if (cudaMalloc(&d, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
    owned.push_back(d);
    if (n && cudaMemcpy(d, src, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
    return d;
}

}  // namespace

struct SimState {
    SimTables t{};
    bool exact_body = false;
    uint64_t N = 0, done = 0, resim = 0;
    uint32_t W = 0, L = 0, K = 0;
    uint32_t entry = 0;
    uint64_t window = 0;           // index of the window sim_next processes next
    std::vector<void*> owned;
    cudaStream_t gen_stream = nullptr;  // the generator runs one window ahead on its own stream
    cudaEvent_t gen_ev[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // per buffer: generation start / end
    cudaEvent_t used_ev[2] = {nullptr, nullptr};                           // per buffer: its window is resolved and read
    cudaEvent_t ph_ev[4] = {nullptr, nullptr, nullptr, nullptr};
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
    size_t text_cap = 0;
    std::vector<char> text_h[2][2];  // [slot][mate]: a chunk stays valid until the second following sim_next
    int slot = 0;
    double* counts = nullptr;
    rsem_b200_sim_stats stats{};
};

void sim_free(rsem_b200_ctx* ctx) {
    SimState* s = ctx->sim;
    if (!s) return;
    cudaStreamSynchronize(ctx->stream);
    if (s->gen_stream) cudaStreamSynchronize(s->gen_stream);
    for (void* p : s->owned) cudaFree(p);
    cudaFree(s->text_d[0]);
    cudaFree(s->text_d[1]);
    for (auto& e : s->gen_ev) for (cudaEvent_t x : e) if (x) cudaEventDestroy(x);
    for (cudaEvent_t x : s->used_ev) if (x) cudaEventDestroy(x);
    for (cudaEvent_t x : s->ph_ev) if (x) cudaEventDestroy(x);
    if (s->gen_stream) cudaStreamDestroy(s->gen_stream);
    delete s;
    ctx->sim = nullptr;
}

#define SIM_ALLOC(ptr, n)                                                       \
    do {                                                                        \
        RB_CUDA(cudaMalloc(&(ptr), std::max<size_t>((n), 1) * sizeof(*(ptr)))); \
        s->owned.push_back((void*)(ptr));                                       \
    } while (0)

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

int sim_begin(rsem_b200_ctx* ctx, const rsem_b200_sim_params* p) {
    sim_free(ctx);
    SimState* s = new SimState();
    ctx->sim = s;
    const int M = p->M;
    const bool q = p->model_type & 1, paired = p->model_type >= 2;
    auto fail = [&]() { set_error("sim_begin: cudaMalloc / cudaMemcpy failed"); sim_free(ctx); return RSEM_B200_ERR_CUDA; };
    SimTables& t = s->t;
    t.type = p->model_type;
    t.M = M;
    t.ori0 = p->ori_prob0;
    t.gld_lb = p->gld.lb;
    t.gld_ub = p->gld.ub;
    t.has_mld = p->has_mld;
    t.mld_lb = p->has_mld ? p->mld.lb : 0;
    t.mld_ub = p->has_mld ? p->mld.ub : 0;
    t.est_rspd = p->est_rspd;
    const uint64_t total_seq = p->seq_off[M + 1];
    if (!(t.theta_cdf = dev_copy(p->theta_cdf, (size_t)M + 1, s->owned))) return fail();
    if (!(t.gld_cdf = dev_copy(p->gld.cdf, (size_t)p->gld.span + 1, s->owned))) return fail();
    if (p->has_mld && !(t.mld_cdf = dev_copy(p->mld.cdf, (size_t)p->mld.span + 1, s->owned))) return fail();
    if (p->est_rspd) {
        if (!(t.rspd_off = dev_copy(p->rspd_off, (size_t)M + 2, s->owned))) return fail();
        if (!(t.rspd_cdf = dev_copy(p->rspd_cdf, (size_t)p->rspd_off[M + 1], s->owned))) return fail();
    }
    if (q) {
        if (!(t.qd_init = dev_copy(p->qd_init_cdf, kQ, s->owned))) return fail();
        if (!(t.qd_tran = dev_copy(p->qd_tran_cdf, (size_t)kQ * kQ, s->owned))) return fail();
    }
    if (!(t.pro = dev_copy(p->profile_cdf, (size_t)p->pro_rows * 25, s->owned))) return fail();
    if (!(t.noise = dev_copy(p->noise_cdf, q ? (size_t)kQ * 5 : 5, s->owned))) return fail();
    if (!(t.seq_off = dev_copy(p->seq_off, (size_t)M + 2, s->owned))) return fail();
    if (!(t.seq = dev_copy(p->seq, (size_t)total_seq, s->owned))) return fail();
    if (!(t.tot_len = dev_copy(p->tot_len, (size_t)M + 1, s->owned))) return fail();
    if (!(t.full_len = dev_copy(p->full_len, (size_t)M + 1, s->owned))) return fail();
    s->exact_body = p->exact_body != 0;
    s->N = p->N;

    // longest attempt: every draw takes at most 2 words; draws = sid, dir, length, position, 2 mate lengths, and per
    // mate max(len, 1) qualities + len bases
    const int maxlen = std::max(p->gld.ub, p->has_mld ? p->mld.ub : 0);
    const uint64_t draws = 6 + (uint64_t)(paired ? 2 : 1) * (2 * (uint64_t)maxlen + 1);
    s->L = (uint32_t)(2 * draws + 8);
    uint64_t W = p->window_words ? p->window_words : (uint64_t)1 << 22;
    W = std::max<uint64_t>(W, s->L);
    RB_ARG(W < 0x7fffffffu - s->L, "window too large");
    s->W = (uint32_t)W;
    while (((uint64_t)1 << (s->K + 1)) <= W) ++s->K;  // 2^(K+1) > W >= any chain length
    // a successful attempt takes at least 2 words (the sid draw and one more), and a window holds at most N reads
    s->R = (uint32_t)std::min<uint64_t>(W / 2 + 1, std::max<uint64_t>(s->N, 1));

    std::vector<uint32_t> mt(kMtN + 1);  // boost::mt19937(seed) (mersenne_twister.hpp seed())
    mt[0] = p->seed;
    for (int i = 1; i < kMtN; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    mt[kMtN] = kMtN;
    if (!(s->mt = dev_copy(mt.data(), mt.size(), s->owned))) return fail();
    SIM_ALLOC(s->words[0], (size_t)s->W + s->L);
    SIM_ALLOC(s->words[1], (size_t)s->W + s->L);
    SIM_ALLOC(s->len, s->W);
    s->jump.resize(s->K + 1);
    for (auto& j : s->jump) SIM_ALLOC(j, (size_t)s->W + 1);
    SIM_ALLOC(s->mark, (size_t)s->W + 1);
    SIM_ALLOC(s->chain, s->W);
    SIM_ALLOC(s->n_chain, 1);
    SIM_ALLOC(s->cum, s->W);
    SIM_ALLOC(s->starts, s->R);
    SIM_ALLOC(s->io, 3);
    SIM_ALLOC(s->heads, s->R);
    SIM_ALLOC(s->bytes[0], (size_t)s->R + 1);
    SIM_ALLOC(s->bytes[1], (size_t)s->R + 1);
    SIM_ALLOC(s->counts, (size_t)M + 1);
    RB_CUDA(cudaMemsetAsync(s->counts, 0, ((size_t)M + 1) * sizeof(double), ctx->stream));
    size_t need = 0, tmp = 0;
    RB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, s->bytes[0], s->bytes[0], (int)s->R + 1, ctx->stream));
    need = std::max(need, tmp);
    RB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp, s->cum, s->cum, (int)s->W, ctx->stream));
    need = std::max(need, tmp);
    RB_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, thrust::counting_iterator<uint32_t>(0), s->mark, s->chain,
                                       s->n_chain, (int)s->W, ctx->stream));
    need = std::max(need, tmp);
    s->scan_tmp_bytes = need;
    RB_CUDA(cudaMalloc(&s->scan_tmp, std::max<size_t>(need, 1)));
    s->owned.push_back(s->scan_tmp);

    RB_CUDA(cudaStreamCreateWithFlags(&s->gen_stream, cudaStreamNonBlocking));
    for (auto& e : s->gen_ev) for (cudaEvent_t& x : e) RB_CUDA(cudaEventCreate(&x));
    for (cudaEvent_t& x : s->used_ev) RB_CUDA(cudaEventCreate(&x));
    for (cudaEvent_t& x : s->ph_ev) RB_CUDA(cudaEventCreate(&x));
    RB_CUDA(cudaEventRecord(s->used_ev[0], ctx->stream));  // the buffers are free; counts are zeroed first
    RB_CUDA(cudaEventRecord(s->used_ev[1], ctx->stream));
    if (int rc = sim_enqueue_gen(s, 0)) return rc;
    ctx->launches += 1;
    return 0;
}

int sim_next(rsem_b200_ctx* ctx, const char* text[2], uint64_t bytes[2], uint64_t* n_reads) {
    SimState* s = ctx->sim;
    RB_ARG(s, "sim_begin must be called first");
    cudaStream_t st = ctx->stream;
    *n_reads = 0;
    bytes[0] = bytes[1] = 0;
    text[0] = text[1] = nullptr;
    const bool paired = s->t.type >= 2;
    const int nm = paired ? 2 : 1;
    const int tb = 256;
    while (*n_reads == 0 && s->done < s->N) {
        const uint32_t W = s->W;
        const int b = (int)(s->window & 1);
        // the next window's words are generated while this one is resolved and read
        if (int rc = sim_enqueue_gen(s, s->window + 1)) return rc;
        RB_CUDA(cudaStreamWaitEvent(st, s->gen_ev[b][1], 0));
        const uint32_t* words = s->words[b];

        RB_CUDA(cudaEventRecord(s->ph_ev[0], st));
        const uint32_t first = s->entry, span = W - first;
        const unsigned gw = (W + 1 + tb - 1) / tb, gs_ = (span + 1 + tb - 1) / tb;
        if (s->exact_body) sim_len_kernel<kWalk><<<gw, tb, 0, st>>>(s->t, words, first, W, s->len, s->jump[0]);
        else sim_len_kernel<kCount><<<gw, tb, 0, st>>>(s->t, words, first, W, s->len, s->jump[0]);
        for (uint32_t k = 1; k <= s->K; ++k) sim_double_kernel<<<gs_, tb, 0, st>>>(s->jump[k - 1], s->jump[k], first, W);
        RB_CUDA(cudaMemsetAsync(s->mark, 0, (size_t)W + 1, st));
        RB_CUDA(cudaMemsetAsync(s->mark + first, 1, 1, st));
        for (int k = (int)s->K; k >= 0; --k) sim_mark_kernel<<<gs_, tb, 0, st>>>(s->jump[k], s->mark, first, W);
        RB_CUDA(cub::DeviceSelect::Flagged(s->scan_tmp, s->scan_tmp_bytes, thrust::counting_iterator<uint32_t>(0),
                                           s->mark, s->chain, s->n_chain, (int)W, st));
        sim_okflag_kernel<<<gs_, tb, 0, st>>>(s->chain, s->n_chain, s->len, s->cum);
        RB_CUDA(cub::DeviceScan::InclusiveSum(s->scan_tmp, s->scan_tmp_bytes, s->cum, s->cum, (int)span, st));
        sim_cut_kernel<<<gs_, tb, 0, st>>>(s->chain, s->n_chain, s->cum, s->len, s->N - s->done, s->starts, s->io);
        uint64_t io[3];
        RB_CUDA(cudaMemcpyAsync(io, s->io, sizeof io, cudaMemcpyDeviceToHost, st));
        RB_CUDA(cudaEventRecord(s->ph_ev[1], st));
        RB_CUDA(cudaStreamSynchronize(st));
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
        const uint64_t rid0 = s->done;
        const unsigned gb = (n + tb - 1) / tb;
        RB_CUDA(cudaEventRecord(s->ph_ev[0], st));
        if (s->exact_body)
            sim_head_kernel<kWalk><<<gb, tb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1]);
        else
            sim_head_kernel<kCount><<<gb, tb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1]);
        uint64_t tot[2] = {0, 0};
        for (int m = 0; m < nm; ++m) {
            RB_CUDA(cudaMemsetAsync(s->bytes[m] + n, 0, sizeof(uint64_t), st));
            RB_CUDA(cub::DeviceScan::ExclusiveSum(s->scan_tmp, s->scan_tmp_bytes, s->bytes[m], s->bytes[m], (int)n + 1, st));
            RB_CUDA(cudaMemcpyAsync(&tot[m], s->bytes[m] + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        }
        RB_CUDA(cudaStreamSynchronize(st));
        const size_t need = std::max(tot[0], tot[1]);
        if (need > s->text_cap) {
            RB_CUDA(cudaStreamSynchronize(st));
            cudaFree(s->text_d[0]);
            cudaFree(s->text_d[1]);
            s->text_d[0] = s->text_d[1] = nullptr;
            s->text_cap = need + need / 4;
            RB_CUDA(cudaMalloc(&s->text_d[0], s->text_cap));
            if (paired) RB_CUDA(cudaMalloc(&s->text_d[1], s->text_cap));
        }
        sim_write_kernel<<<gb, tb, 0, st>>>(s->t, words, s->starts, n, rid0, s->heads, s->bytes[0], s->bytes[1],
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
        s->stats.windows = s->window;
        s->done += n;
        *n_reads = n;
    }
    return 0;
}

int sim_end(rsem_b200_ctx* ctx, double* counts, uint64_t* resim, rsem_b200_sim_stats* stats) {
    SimState* s = ctx->sim;
    RB_ARG(s, "sim_begin must be called first");
    if (counts) RB_CUDA(cudaMemcpy(counts, s->counts, ((size_t)s->t.M + 1) * sizeof(double), cudaMemcpyDeviceToHost));
    if (resim) *resim = s->resim;
    if (stats) { s->stats.windows = s->window; *stats = s->stats; }
    sim_free(ctx);
    return 0;
}

}  // namespace rsem_b200
