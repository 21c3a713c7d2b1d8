// K1: per-hit conditional probabilities (getConPrb / getNoiseConPrb) and
// K3: model sufficient statistics (update / updateNoise) for the four RSEM read models.
//
// Reference semantics (paths relative to /root/reference):
//   getConPrb        SingleModel.h:95-146, SingleQModel.h:101-151, PairedEndModel.h:90-134,
//                    PairedEndQModel.h:94-138
//   getNoiseConPrb   SingleModel.h:148-157, SingleQModel.h:153-162, PairedEndModel.h:136-151,
//                    PairedEndQModel.h:140-155
//   update/updateNoise  SingleModel.h:163-215, SingleQModel.h:168-221, PairedEndModel.h:156-183,
//                    PairedEndQModel.h:161-188  (+ Profile.h:91-96, QProfile.h:88-93,
//                    NoiseProfile.h:71-76, NoiseQProfile.h:74-79, LenDist.h:46-49, RSPD.h:43-59)
//
// H100 mapping: reads (base codes + qualities) and transcripts are resident in HBM, parsed once
// (the reference re-parses the FASTA/FASTQ text every round).  A read is handled by a group of G
// lanes (the same grouping as the E-step); each lane walks the bases of its own hits.  The
// (Q)Profile table is staged in shared memory.  K3 accumulates with red.global.add.f64 into
// kReplicas copies of the statistics block (the ~20 hot (quality, base, base) cells would
// otherwise serialise in one L2 slice) which a second kernel folds into copy 0.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace rsem_b200 {
namespace {

constexpr int kReplicas = 64;
constexpr int kBlock = 256;

struct ModelArgs {
    DevModel m;
    // reads
    int n_mates;
    const unsigned long long* roff[2];
    const unsigned char* rbase[2];
    const unsigned char* rqual[2];
    const unsigned char* lowq;
    // refs
    const unsigned long long* seq_off;
    const unsigned char* seq;
    const int* full_len;
    const int* tot_len;
    const unsigned long long* mask_off;
    const unsigned int* mask_words;
    // hits
    unsigned long long N;
    const unsigned long long* row_ptr;
    const int* sid;
    const int* pos;
    const int* insertL;
    double* conprb;
    double* ncpv;
    const double* post;
    const double* post0;
    // K3 targets
    double* stats;          // kReplicas blocks of `stats_block` doubles
    size_t stats_block;
    size_t o_noise, o_gld, o_rspd;  // offsets inside a block (profile at 0)
    int gld_lb, gld_span;
    int prof_rows_smem;     // rows of the profile table staged in shared memory (0 = use global)
    int q_rows;             // quality models: (largest quality value in the read set) + 1
    int* err_flag;
    const unsigned char* uni;   // per read: 1 = every hit sees the same bases in read direction (window_uniform_kernel)
    int mode;                   // 0: every read on the per-hit path, 1: only uniform reads (cooperative path), 2: only the others
};

__device__ __forceinline__ double ld_adj(const DevLenDist& d, int len, int refL) {
    if (len <= d.lb || len > d.ub || refL <= d.lb) return 0.0;
    const int top = min(d.ub, refL) - d.lb;
    return d.pdf[len - d.lb] / d.cdf[top];
}
__device__ __forceinline__ double ld_prob(const DevLenDist& d, int len) {
    if (len <= d.lb || len > d.ub) return 0.0;  // the reference asserts this range (LenDist.h:58)
    return d.pdf[len - d.lb];
}
__device__ __forceinline__ double rspd_cdf_at(const DevModel& m, int fpos, int fullLen) {
    const int i = (int)(((long long)fpos) * m.rspd_B / fullLen);
    const double val = __dmul_rn(__ddiv_rn(fpos * 1.0, (double)fullLen), (double)m.rspd_B);
    return __dadd_rn(m.rspd_cdf[i], __dmul_rn(val - i, m.rspd_pdf[i + 1]));
}
__device__ __forceinline__ double rspd_adj(const DevModel& m, int fpos, int effL, int fullLen) {
    if (!m.est_rspd) return 1.0 / effL;
    const double denom = rspd_cdf_at(m, effL, fullLen);
    return denom >= kEpsilon ? (rspd_cdf_at(m, fpos + 1, fullLen) - rspd_cdf_at(m, fpos, fullLen)) / denom : 0.0;
}
__device__ __forceinline__ bool ref_mask(const ModelArgs& a, int sid, int p) {
    return (a.mask_words[a.mask_off[sid] + (p >> 5)] >> (p & 31)) & 1u;
}

// Byte streams through aligned 8-byte loads: a lane walks 50-150 consecutive bytes of a read, its qualities and a
// transcript; LDG.U8 per base made the LSU pipe the limiter (3 scattered byte loads per lane and base), one LDG.64
// per 8 bases and stream does not.  The arrays carry >= 16 bytes of tail padding (capi.cu).
struct FwdBytes {  // bytes p[0], p[1], ... 8 at a time
    const unsigned long long* q;
    unsigned long long cur, nxt;
    unsigned sh;
    __device__ __forceinline__ explicit FwdBytes(const unsigned char* p, bool active = true) {
        q = reinterpret_cast<const unsigned long long*>(reinterpret_cast<unsigned long long>(p) & ~7ull);
        sh = (unsigned)(reinterpret_cast<unsigned long long>(p) & 7ull) * 8u;
        cur = nxt = 0ull;
        if (active) {
            cur = __ldg(q);
            nxt = __ldg(q + 1);
        }
    }
    // the next 8 bytes (byte k of the stream chunk in bits 8k..8k+7); `more` = another chunk will be asked for
    __device__ __forceinline__ unsigned long long next(bool more) {
        const unsigned long long v = sh ? (cur >> sh) | (nxt << (64u - sh)) : cur;
        ++q;
        cur = nxt;
        if (more) nxt = __ldg(q + 1);
        return v;
    }
};
struct RevBytes {  // bytes p[0], p[-1], p[-2], ... 8 at a time; never loads below `floor`
    const unsigned long long* q;
    const unsigned long long* floor;
    unsigned long long lo, hi;
    unsigned sh;
    __device__ __forceinline__ RevBytes(const unsigned char* p, const unsigned char* base) {
        const unsigned long long a = reinterpret_cast<unsigned long long>(p) - 7ull;
        q = reinterpret_cast<const unsigned long long*>(a & ~7ull);
        floor = reinterpret_cast<const unsigned long long*>(base);
        sh = (unsigned)(a & 7ull) * 8u;
        lo = q >= floor ? __ldg(q) : 0ull;
        hi = __ldg(q + 1);
    }
    // 8 bytes p[-8c-7 .. -8c]: byte p[-8c-k] sits in bits 8(7-k)..8(7-k)+7
    __device__ __forceinline__ unsigned long long next(bool more) {
        const unsigned long long v = sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
        --q;
        hi = lo;
        if (more) lo = q >= floor ? __ldg(q) : 0ull;
        return v;
    }
};
__device__ __forceinline__ unsigned byte_of(unsigned long long w, int k) { return (unsigned)(w >> (8 * k)) & 0xffu; }

struct RefStream {  // bases of a transcript in read direction: forward strand as stored, reverse strand complemented
    const unsigned long long* q;
    const unsigned long long* floor;
    unsigned long long lo, hi;
    unsigned sh;
    bool rev;
    __device__ __forceinline__ RefStream(const unsigned char* s, bool rev_, const unsigned char* base, bool active) {
        const unsigned long long a = reinterpret_cast<unsigned long long>(s) - (rev_ ? 7ull : 0ull);
        q = reinterpret_cast<const unsigned long long*>(a & ~7ull);
        floor = reinterpret_cast<const unsigned long long*>(base);
        sh = (unsigned)(a & 7ull) * 8u;
        rev = rev_;
        lo = hi = 0ull;
        if (active) {
            lo = q >= floor ? __ldg(q) : 0ull;
            hi = __ldg(q + 1);
        }
    }
    __device__ __forceinline__ unsigned long long next(bool fetch) {
        const unsigned long long v = sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
        if (rev) {
            --q;
            hi = lo;
            if (fetch) lo = q >= floor ? __ldg(q) : 0ull;
        } else {
            ++q;
            lo = hi;
            if (fetch) hi = __ldg(q + 1);
        }
        return v;
    }
    __device__ __forceinline__ int base_at(unsigned long long v, int k) const {
        if (!rev) return (int)byte_of(v, k);
        const int c = (int)byte_of(v, 7 - k);
        return c < 4 ? 3 - c : 4;
    }
};


// product over the bases of one mate of p[row][ref][read]; row = quality (Q models) or position.
// Multiplication order = base order, as in the reference.
template <bool HASQ>
__device__ __forceinline__ double seq_prob(const ModelArgs& a, const double* prof, int mate, unsigned long long i,
                                           int sid, int pos, int dir) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    const int totLen = a.tot_len[sid];
    if (pos < 0 || pos + len > totLen) {  // reference: general_assert -> exit(-1) (e.g. SingleQModel.h:116-121)
        *a.err_flag = 2;
        return 0.0;
    }
    if (len <= 0) return 1.0;
    FwdBytes rb(a.rbase[mate] + o);
    FwdBytes rq(HASQ ? a.rqual[mate] + o : a.rbase[mate] + o, HASQ);
    // one loop for both strands (the lanes of a warp hold hits of either orientation; two loops would both be executed)
    RefStream sb(a.seq + a.seq_off[sid] + (dir == 0 ? pos : totLen - 1 - pos), dir != 0, a.seq, true);
    double prob = 1.0;
    for (int k0 = 0; k0 < len; k0 += 8) {
        const bool more = k0 + 8 < len;
        const unsigned long long ws = sb.next(more), wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
        const int n = min(8, len - k0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (k < n) {
                const int row = HASQ ? (int)byte_of(wq, k) : k0 + k;
                prob *= prof[(row * 5 + sb.base_at(ws, k)) * 5 + (int)byte_of(wr, k)];
            }
        }
    }
    return prob;
}

template <bool HASQ>
__device__ __forceinline__ double noise_prob(const ModelArgs& a, const double* nprof, int mate, unsigned long long i) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    if (len <= 0) return 1.0;
    FwdBytes rb(a.rbase[mate] + o);
    FwdBytes rq(HASQ ? a.rqual[mate] + o : a.rbase[mate] + o, HASQ);
    double prob = 1.0;
    for (int k0 = 0; k0 < len; k0 += 8) {
        const bool more = k0 + 8 < len;
        const unsigned long long wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
        const int n = min(8, len - k0);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < n) prob *= HASQ ? nprof[byte_of(wq, k) * 5 + byte_of(wr, k)] : nprof[byte_of(wr, k)];
    }
    return prob;
}

// ---- cooperative products for "uniform" reads ------------------------------------------------------------------------
// When all hits of a read show it the same bases (reads inside exons shared by the isoforms of a gene - the common case),
// the product over its bases is the same for every hit: the G lanes of the read's group each take a contiguous range of
// 8-base chunks and the partial products are multiplied in a butterfly (every lane ends with the same bits: fp
// multiplication is commutative and the tree is symmetric).  The product is therefore associated differently from the
// reference's left-to-right loop (SingleQModel.h:127-137): relative difference <= a few 1e-14, far inside the 1e-6 the
// outputs are compared at; non-uniform reads keep the reference's order.
template <int G>
__device__ __forceinline__ double group_product(double v) {
#pragma unroll
    for (int o = 1; o < G; o <<= 1) v *= __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int G, bool HASQ>
__device__ __forceinline__ double seq_prob_coop(const ModelArgs& a, const double* prof, int mate, unsigned long long i, int sid,
                                                int pos, int dir, int g, bool active) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    const int totLen = a.tot_len[sid];
    const int n_chunks = (len + 7) >> 3;
    const int c0 = g * n_chunks / G, c1 = (g + 1) * n_chunks / G;
    double prob = 1.0;
    if (active && c1 > c0) {
        FwdBytes rb(a.rbase[mate] + o + 8 * c0);
        FwdBytes rq(HASQ ? a.rqual[mate] + o + 8 * c0 : a.rbase[mate] + o, HASQ);
        const unsigned char* s0 = a.seq + a.seq_off[sid] + (dir == 0 ? pos + 8 * c0 : totLen - 1 - pos - 8 * c0);
        RefStream sb(s0, dir != 0, a.seq, true);
        for (int c = c0; c < c1; ++c) {
            const bool more = c + 1 < c1;
            const unsigned long long ws = sb.next(more), wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
            const int k0 = 8 * c, n = min(8, len - k0);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < n) {
                    const int row = HASQ ? (int)byte_of(wq, k) : k0 + k;
                    prob *= prof[(row * 5 + sb.base_at(ws, k)) * 5 + (int)byte_of(wr, k)];
                }
            }
        }
    }
    return group_product<G>(prob);
}

template <int G, bool HASQ>
__device__ __forceinline__ double noise_prob_coop(const ModelArgs& a, const double* nprof, int mate, unsigned long long i, int g,
                                                  bool active) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    const int n_chunks = (len + 7) >> 3;
    const int c0 = g * n_chunks / G, c1 = (g + 1) * n_chunks / G;
    double prob = 1.0;
    if (active && c1 > c0) {
        FwdBytes rb(a.rbase[mate] + o + 8 * c0);
        FwdBytes rq(HASQ ? a.rqual[mate] + o + 8 * c0 : a.rbase[mate] + o, HASQ);
        for (int c = c0; c < c1; ++c) {
            const bool more = c + 1 < c1;
            const unsigned long long wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
            const int n = min(8, len - 8 * c);
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (k < n) prob *= HASQ ? nprof[byte_of(wq, k) * 5 + byte_of(wr, k)] : nprof[byte_of(wr, k)];
        }
    }
    return group_product<G>(prob);
}

// COOP: the products over the bases (S1, S2) were formed cooperatively and are passed in
template <bool HASQ, bool COOP = false>
__device__ double conprb_single(const ModelArgs& a, const double* prof, unsigned long long i, int s, int pos, double S1 = 1.0) {
    const DevModel& m = a.m;
    const int sid = abs(s), dir = s < 0;
    const int fullLen = a.full_len[sid], totLen = a.tot_len[sid];
    const int readLen = (int)(a.roff[0][i + 1] - a.roff[0][i]);
    const int fpos = dir == 0 ? pos : totLen - pos - readLen;
    const int seedPos = dir == 0 ? pos : totLen - pos - m.seed_len;
    if (pos < 0 || fpos < 0 || seedPos < 0) { *a.err_flag = 2; return 0.0; }
    if (seedPos >= fullLen || ref_mask(a, sid, seedPos)) return 0.0;
    double value;
    if (m.has_mld) {
        const int minL = max(readLen, m.gld.lb + 1), maxL = min(totLen - pos, m.gld.ub);
        value = 0.0;
        for (int fragLen = minL; fragLen <= maxL; ++fragLen) {
            const int pfpos = dir == 0 ? pos : totLen - pos - fragLen;
            const int effL = min(fullLen, totLen - fragLen + 1);
            // __dadd_rn: a separate rounded add, as in the reference's loop (nvcc would otherwise contract it into an FMA)
            value = __dadd_rn(value, ld_adj(m.gld, fragLen, totLen) * rspd_adj(m, pfpos, effL, fullLen) * ld_adj(m.mld, readLen, fragLen));
        }
    } else {
        const int effL = min(fullLen, totLen - readLen + 1);
        value = ld_adj(m.gld, readLen, totLen) * rspd_adj(m, fpos, effL, fullLen);
    }
    double prob = m.ori[dir] * value * (COOP ? S1 : seq_prob<HASQ>(a, prof, 0, i, sid, pos, dir));
    if (prob < kEpsilon) prob = 0.0;
    const double w = m.mw[sid];
    return w < kEpsilon ? 0.0 : prob / w;
}

template <bool HASQ, bool COOP = false>
__device__ double conprb_paired(const ModelArgs& a, const double* prof, unsigned long long i, int s, int pos,
                                int insertLen, double S1 = 1.0, double S2 = 1.0) {
    const DevModel& m = a.m;
    const int sid = abs(s), dir = s < 0;
    const int fullLen = a.full_len[sid], totLen = a.tot_len[sid];
    const int fpos = dir == 0 ? pos : totLen - pos - insertLen;
    const int effL = min(fullLen, totLen - insertLen + 1);
    if (pos < 0 || fpos < 0 || insertLen > totLen) { *a.err_flag = 2; return 0.0; }
    if (fpos >= fullLen || ref_mask(a, sid, fpos)) return 0.0;
    double prob = m.ori[dir] * ld_adj(m.gld, insertLen, totLen) * rspd_adj(m, fpos, effL, fullLen);
    const int len1 = (int)(a.roff[0][i + 1] - a.roff[0][i]), len2 = (int)(a.roff[1][i + 1] - a.roff[1][i]);
    prob *= ld_adj(m.mld, len1, insertLen) * (COOP ? S1 : seq_prob<HASQ>(a, prof, 0, i, sid, pos, dir));
    prob *= ld_adj(m.mld, len2, insertLen) * (COOP ? S2 : seq_prob<HASQ>(a, prof, 1, i, sid, totLen - pos - insertLen, !dir));
    if (prob < kEpsilon) prob = 0.0;
    const double w = m.mw[sid];
    return w < kEpsilon ? 0.0 : prob / w;
}

template <bool HASQ, bool COOP = false>
__device__ double noise_conprb(const ModelArgs& a, const double* nprof, unsigned long long i, double P1 = 1.0, double P2 = 1.0) {
    const DevModel& m = a.m;
    double prob;
    if (m.model_type < 2) {
        const int readLen = (int)(a.roff[0][i + 1] - a.roff[0][i]);
        prob = m.has_mld ? ld_prob(m.mld, readLen) : ld_prob(m.gld, readLen);
        prob *= COOP ? P1 : noise_prob<HASQ>(a, nprof, 0, i);
    } else {
        const int len1 = (int)(a.roff[0][i + 1] - a.roff[0][i]), len2 = (int)(a.roff[1][i + 1] - a.roff[1][i]);
        prob = ld_prob(m.mld, len1) * (COOP ? P1 : noise_prob<HASQ>(a, nprof, 0, i));
        prob *= ld_prob(m.mld, len2) * (COOP ? P2 : noise_prob<HASQ>(a, nprof, 1, i));
    }
    if (prob < kEpsilon) prob = 0.0;
    const double w = m.mw[0];
    return w < kEpsilon ? 0.0 : prob / w;
}

// ---- K1 ---------------------------------------------------------------------------------------
// STAGED: the first prof_rows_smem rows (25 doubles each) of the profile + the noise table are copied to shared memory
// and read from there.  It is a template parameter so that the table pointer is known to be a shared-memory address
// (LDS instead of generic LD.E, which the per-base lookups are bound by).
template <int G, bool HASQ, bool PAIRED, bool STAGED>
__global__ void __launch_bounds__(kBlock) conprb_kernel(const ModelArgs a) {
    extern __shared__ double smem_tab[];
    const double* prof = a.m.profile;
    const double* nprof = a.m.noise_profile;
    if (STAGED) {
        const int n = a.prof_rows_smem * 25;
        for (int k = threadIdx.x; k < n; k += blockDim.x) smem_tab[k] = a.m.profile[k];
        const int nn = HASQ ? 500 : 5;
        for (int k = threadIdx.x; k < nn; k += blockDim.x) smem_tab[n + k] = a.m.noise_profile[k];
        __syncthreads();
        prof = smem_tab;
        nprof = smem_tab + n;
    }
    const int lane = threadIdx.x & 31, g = lane % G;
    const unsigned long long groups_total = (unsigned long long)gridDim.x * (kBlock / G);
    if (a.mode == 1) {
        // cooperative path: reads whose hits all show them the same bases (a.uni); whole warps stay convergent
        const unsigned long long base0 = (unsigned long long)blockIdx.x * (kBlock / G) + threadIdx.x / G;
        const unsigned long long n_iter = (a.N + groups_total - 1) / groups_total;
        for (unsigned long long it = 0; it < n_iter; ++it) {
            const unsigned long long i = base0 + it * groups_total;
            const bool in = i < a.N;
            const bool lq = in && a.lowq[i] != 0;
            const bool act = in && a.uni[i] != 0;
            unsigned long long fr = 0, to = 0;
            if (act) { fr = a.row_ptr[i]; to = a.row_ptr[i + 1]; }
            if (__ballot_sync(0xffffffffu, act) == 0u) continue;
            const bool work = act && !lq;
            // hit 0 defines the window
            int s0 = 1, p0 = 0, il0 = 0;
            if (work && to > fr) { s0 = a.sid[fr]; p0 = a.pos[fr]; if (PAIRED) il0 = a.insertL[fr]; }
            const int t0 = abs(s0), d0 = s0 < 0;
            const bool has_hit = work && to > fr;
            const double S1 = seq_prob_coop<G, HASQ>(a, prof, 0, in ? i : 0, t0, p0, d0, g, has_hit);
            double S2 = 1.0;
            if (PAIRED) S2 = seq_prob_coop<G, HASQ>(a, prof, 1, in ? i : 0, t0, a.tot_len[t0] - p0 - il0, !d0, g, has_hit);
            const double P1 = noise_prob_coop<G, HASQ>(a, nprof, 0, in ? i : 0, g, work);
            double P2 = 1.0;
            if (PAIRED) P2 = noise_prob_coop<G, HASQ>(a, nprof, 1, in ? i : 0, g, work);
            if (act && g == 0) a.ncpv[i] = lq ? 0.0 : noise_conprb<HASQ, true>(a, nprof, i, P1, P2);
            if (act)
                for (unsigned long long j = fr + g; j < to; j += G) {
                    double v = 0.0;
                    if (!lq)
                        v = PAIRED ? conprb_paired<HASQ, true>(a, prof, i, a.sid[j], a.pos[j], a.insertL[j], S1, S2)
                                   : conprb_single<HASQ, true>(a, prof, i, a.sid[j], a.pos[j], S1);
                    a.conprb[j] = v;
                }
        }
        return;
    }
    for (unsigned long long i = (unsigned long long)blockIdx.x * (kBlock / G) + threadIdx.x / G; i < a.N; i += groups_total) {
        if (a.mode == 2 && a.uni[i]) continue;
        const unsigned long long fr = a.row_ptr[i], to = a.row_ptr[i + 1];
        const bool lq = a.lowq[i] != 0;
        if (g == 0) a.ncpv[i] = lq ? 0.0 : noise_conprb<HASQ>(a, nprof, i);
        for (unsigned long long j = fr + g; j < to; j += G) {
            double v = 0.0;
            if (!lq)
                v = PAIRED ? conprb_paired<HASQ>(a, prof, i, a.sid[j], a.pos[j], a.insertL[j])
                           : conprb_single<HASQ>(a, prof, i, a.sid[j], a.pos[j]);
            a.conprb[j] = v;
        }
    }
}

// ---- which reads are "uniform" (once per upload: depends on the hits, the reads' lengths and the transcripts only) --------
// 8 bases of a transcript in read direction, one per byte, from a RefStream word
__device__ __forceinline__ unsigned long long read_dir_bases(unsigned long long w, bool rev) {
    if (!rev) return w;
    const unsigned long long is4 = (w >> 2) & 0x0101010101010101ull;         // code 4 (N) stays 4
    const unsigned long long x = 0x0303030303030303ull & ~(is4 | (is4 << 1));
    w ^= x;                                                                   // complement: c -> 3 - c for c < 4
    const unsigned lo = (unsigned)w, hi = (unsigned)(w >> 32);
    return ((unsigned long long)__byte_perm(lo, 0, 0x0123) << 32) | (unsigned long long)__byte_perm(hi, 0, 0x0123);
}

template <int G, bool PAIRED>
__global__ void __launch_bounds__(kBlock) window_uniform_kernel(const ModelArgs a, unsigned char* uni) {
    const int lane = threadIdx.x & 31, g = lane % G, grp = lane / G;
    const unsigned group_mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    const unsigned long long groups_total = (unsigned long long)gridDim.x * (kBlock / G);
    const unsigned long long base0 = (unsigned long long)blockIdx.x * (kBlock / G) + threadIdx.x / G;
    const unsigned long long n_iter = (a.N + groups_total - 1) / groups_total;
    for (unsigned long long it = 0; it < n_iter; ++it) {
        const unsigned long long i = base0 + it * groups_total;
        const bool in = i < a.N;
        unsigned long long fr = 0, to = 0;
        if (in) { fr = a.row_ptr[i]; to = a.row_ptr[i + 1]; }
        bool same = in && to > fr;
        int s0 = 1, p0 = 0, il0 = 0;
        if (same) { s0 = a.sid[fr]; p0 = a.pos[fr]; if (PAIRED) il0 = a.insertL[fr]; }
        for (unsigned long long j = fr + g; j < to; j += G) {   // lanes diverge only in the trip count
            const int sj = a.sid[j], pj = a.pos[j], ilj = PAIRED ? a.insertL[j] : 0;
            for (int mt = 0; mt < (PAIRED ? 2 : 1) && same; ++mt) {
                const int len = (int)(a.roff[mt][i + 1] - a.roff[mt][i]);
                int t[2], p[2], d[2];
                t[0] = abs(s0); t[1] = abs(sj);
                d[0] = (s0 < 0) ^ (mt == 1); d[1] = (sj < 0) ^ (mt == 1);
                p[0] = mt == 0 ? p0 : a.tot_len[t[0]] - p0 - il0;
                p[1] = mt == 0 ? pj : a.tot_len[t[1]] - pj - ilj;
                if (p[0] < 0 || p[0] + len > a.tot_len[t[0]] || p[1] < 0 || p[1] + len > a.tot_len[t[1]]) { same = false; break; }
                if (len <= 0) continue;
                RefStream r0(a.seq + a.seq_off[t[0]] + (d[0] == 0 ? p[0] : a.tot_len[t[0]] - 1 - p[0]), d[0] != 0, a.seq, true);
                RefStream r1(a.seq + a.seq_off[t[1]] + (d[1] == 0 ? p[1] : a.tot_len[t[1]] - 1 - p[1]), d[1] != 0, a.seq, true);
                for (int k0 = 0; k0 < len && same; k0 += 8) {
                    const bool more = k0 + 8 < len;
                    unsigned long long w0 = read_dir_bases(r0.next(more), d[0] != 0), w1 = read_dir_bases(r1.next(more), d[1] != 0);
                    const int n = min(8, len - k0);
                    if (n < 8) { const unsigned long long msk = (1ull << (8 * n)) - 1ull; w0 &= msk; w1 &= msk; }
                    if (w0 != w1) same = false;
                }
            }
        }
        const unsigned bad = __ballot_sync(0xffffffffu, in && !same) & group_mask;
        if (in && g == 0) uni[i] = bad == 0u ? 1 : 0;
    }
}

// ---- K3 ---------------------------------------------------------------------------------------
__device__ __forceinline__ void red_add(double* p, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

template <bool HASQ>
__device__ __forceinline__ void prof_update(const ModelArgs& a, double* tab, int mate, unsigned long long i, int sid,
                                            int pos, int dir, double frac) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    const int totLen = a.tot_len[sid];
    if (pos < 0 || pos + len > totLen || len <= 0) return;
    FwdBytes rb(a.rbase[mate] + o);
    FwdBytes rq(HASQ ? a.rqual[mate] + o : a.rbase[mate] + o, HASQ);
    const unsigned char* s = a.seq + a.seq_off[sid] + (dir == 0 ? pos : totLen - 1 - pos);
    if (dir == 0) {
        FwdBytes sb(s);
        for (int k0 = 0; k0 < len; k0 += 8) {
            const bool more = k0 + 8 < len;
            const unsigned long long ws = sb.next(more), wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
            const int n = min(8, len - k0);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < n) {
                    const int row = HASQ ? (int)byte_of(wq, k) : k0 + k;
                    red_add(tab + (row * 5 + (int)byte_of(ws, k)) * 5 + (int)byte_of(wr, k), frac);
                }
            }
        }
    } else {
        RevBytes sb(s, a.seq);
        for (int k0 = 0; k0 < len; k0 += 8) {
            const bool more = k0 + 8 < len;
            const unsigned long long ws = sb.next(more), wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
            const int n = min(8, len - k0);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < n) {
                    const int c = (int)byte_of(ws, 7 - k);
                    const int row = HASQ ? (int)byte_of(wq, k) : k0 + k;
                    red_add(tab + (row * 5 + (c < 4 ? 3 - c : 4)) * 5 + (int)byte_of(wr, k), frac);
                }
            }
        }
    }
}

template <bool HASQ>
__device__ __forceinline__ void noise_update(const ModelArgs& a, double* tab, int mate, unsigned long long i, double frac) {
    const unsigned long long o = a.roff[mate][i];
    const int len = (int)(a.roff[mate][i + 1] - o);
    if (len <= 0) return;
    FwdBytes rb(a.rbase[mate] + o);
    FwdBytes rq(HASQ ? a.rqual[mate] + o : a.rbase[mate] + o, HASQ);
    for (int k0 = 0; k0 < len; k0 += 8) {
        const bool more = k0 + 8 < len;
        const unsigned long long wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
        const int n = min(8, len - k0);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < n) red_add(tab + (HASQ ? byte_of(wq, k) * 5 + byte_of(wr, k) : byte_of(wr, k)), frac);
    }
}

// RSPD::update, RSPD.h:43-59
__device__ __forceinline__ void rspd_update(const ModelArgs& a, double* pdf, int fpos, int fullLen, double frac) {
    if (fpos >= fullLen || fpos < 0) return;
    const int B = a.m.rspd_B;
    int i;
    double x = fpos * 1.0 / fullLen, b;
    for (i = (int)(((long long)fpos) * B / fullLen + 1); i < (((long long)fpos + 1) * B - 1) / fullLen + 1; ++i) {
        b = i * 1.0 / B;
        red_add(pdf + i, (b - x) * fullLen * frac);
        x = b;
    }
    b = (fpos + 1.0) / fullLen;
    red_add(pdf + i, (b - x) * fullLen * frac);
}

template <int G, bool HASQ, bool PAIRED>
__global__ void __launch_bounds__(kBlock) update_kernel(const ModelArgs a) {
    const int lane = threadIdx.x & 31, g = lane % G;
    const unsigned warp_global = blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
    double* blk = a.stats + (size_t)(warp_global % kReplicas) * a.stats_block;
    double* t_prof = blk;
    double* t_noise = blk + a.o_noise;
    double* t_gld = blk + a.o_gld;
    double* t_rspd = blk + a.o_rspd;
    const DevModel& m = a.m;
    const unsigned long long groups_total = (unsigned long long)gridDim.x * (kBlock / G);
    for (unsigned long long i = (unsigned long long)blockIdx.x * (kBlock / G) + threadIdx.x / G; i < a.N; i += groups_total) {
        if (a.lowq[i]) continue;
        if (a.mode == 2 && a.uni[i]) continue;   // handled by update_coop_kernel
        const unsigned long long fr = a.row_ptr[i], to = a.row_ptr[i + 1];
        if (g == 0) {
            const double f0 = a.post0[i];
            if (f0 >= kEpsilon) {
                noise_update<HASQ>(a, t_noise, 0, i, f0);
                if (PAIRED) noise_update<HASQ>(a, t_noise, 1, i, f0);
            }
        }
        for (unsigned long long j = fr + g; j < to; j += G) {
            const double frac = a.post[j];
            if (frac < kEpsilon) continue;
            const int s = a.sid[j], t = abs(s), dir = s < 0, p = a.pos[j];
            const int fullLen = a.full_len[t], totLen = a.tot_len[t];
            if (!PAIRED) {
                if (m.est_rspd) {  // one strand only (SingleQModel.h:180-184; helper models have mld == NULL)
                    const int readLen = (int)(a.roff[0][i + 1] - a.roff[0][i]);
                    if (m.ori[0] >= 0.1 && dir == 0) rspd_update(a, t_rspd, p, fullLen, frac);
                    if (m.ori[0] < 0.1 && dir == 1) rspd_update(a, t_rspd, totLen - p - readLen, fullLen, frac);
                }
                prof_update<HASQ>(a, t_prof, 0, i, t, p, dir, frac);
            } else {
                const int il = a.insertL[j];
                if (il > a.gld_lb && il <= a.gld_lb + a.gld_span) red_add(t_gld + (il - a.gld_lb), frac);
                if (m.est_rspd) rspd_update(a, t_rspd, dir == 0 ? p : totLen - p - il, fullLen, frac);
                prof_update<HASQ>(a, t_prof, 0, i, t, p, dir, frac);
                prof_update<HASQ>(a, t_prof, 1, i, t, totLen - p - il, !dir, frac);
            }
        }
    }
}

// ---- K3 for the quality models (SingleQModel / PairedEndQModel) -----------------------------------
// The QProfile / NoiseQProfile statistics are 2500 + 500 cells of which ~20 ((frequent quality) x (matching base
// pair)) receive almost every update: one red.global per base and hit (update_kernel above) serialises in L2 -
// 1.8e9 reductions took 33 ms for 1 M paired reads.  Here every WARP owns a private copy of the two tables in
// shared memory and no atomics are needed:
//   * G lanes share a read (its bases and qualities are the same for all of them), each lane walks the transcript of
//     one hit; at a base position the lanes' cells differ only where the transcripts differ, so normally the whole
//     group agrees on the cell and ONE lane adds the group's summed weight;
//   * the 32 / G groups of the warp take turns (their cells often coincide), ordered by __syncwarp;
//   * positions where a group disagrees (isoform / allele differences) fall back to one lane at a time.
// At the end the CTA adds its warps' tables and sends one reduction per non-zero cell to a replica of the global block.
constexpr int kQMaxWarps = 16;   // warps per CTA; each owns (max quality + 1) * 30 doubles of shared memory

template <int G>
__device__ __forceinline__ double lane_group_sum(double v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int G, bool PAIRED>
__global__ void __launch_bounds__(kQMaxWarps * 32, 1) update_q_kernel(const ModelArgs a) {
    extern __shared__ double q_tabs[];
    const int kQWarps = blockDim.x >> 5;
    const int n_prof = a.q_rows * 25, kQTab = a.q_rows * 30;
    constexpr int R = 32 / G;
    constexpr int NM = PAIRED ? 2 : 1;   // mates
    constexpr int NI = 2 * NM;           // (position, mate) items a group's doer lane handles per turn
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane % G, grp = lane / G;
    double* tprof = q_tabs + warp * kQTab;
    double* tnoise = tprof + n_prof;
    for (int k = lane; k < kQTab; k += 32) tprof[k] = 0.0;
    __syncwarp();
    const unsigned group_mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    double* blk = a.stats + (size_t)((blockIdx.x * kQWarps + warp) % kReplicas) * a.stats_block;
    double* t_gld = blk + a.o_gld;
    double* t_rspd = blk + a.o_rspd;
    const DevModel& m = a.m;

    const unsigned long long warps_total = (unsigned long long)gridDim.x * kQWarps;
    for (unsigned long long base = ((unsigned long long)blockIdx.x * kQWarps + warp) * R; base < a.N; base += warps_total * R) {
        const unsigned long long i = base + grp;
        const bool valid = i < a.N && !a.lowq[i] && !(a.mode == 2 && a.uni[i]);   // uniform reads: update_coop_kernel
        unsigned long long fr = 0, to = 0;
        double f0 = 0.0;
        if (valid) {
            fr = a.row_ptr[i];
            to = a.row_ptr[i + 1];
            f0 = a.post0[i];
            if (f0 < kEpsilon) f0 = 0.0;  // updateNoise only if frac >= EPSILON
        }
        int len[NM];
        unsigned long long ro[NM];
#pragma unroll
        for (int mt = 0; mt < NM; ++mt) {
            ro[mt] = valid ? a.roff[mt][i] : 0ull;
            len[mt] = valid ? (int)(a.roff[mt][i + 1] - ro[mt]) : 0;
        }
        // a read without hits still updates the noise statistics: at least one pass
        const int n_pass = __reduce_max_sync(0xffffffffu, valid ? max(1, (int)((to - fr + G - 1) / G)) : 0);
        for (int pass = 0; pass < n_pass; ++pass) {
            const unsigned long long j = fr + (unsigned long long)pass * G + g;
            bool act = valid && j < to;
            double frac = act ? a.post[j] : 0.0;
            if (frac < kEpsilon) { act = false; frac = 0.0; }
            int t = 0, dir = 0, p = 0, il = 0, fullLen = 1, totLen = 0;
            if (act) {
                const int sgn = a.sid[j];
                t = abs(sgn);
                dir = sgn < 0;
                p = a.pos[j];
                fullLen = a.full_len[t];
                totLen = a.tot_len[t];
                if (!PAIRED) {
                    if (m.est_rspd) {  // one strand only (SingleQModel.h:180-184; helper models have mld == NULL)
                        if (m.ori[0] >= 0.1 && dir == 0) rspd_update(a, t_rspd, p, fullLen, frac);
                        if (m.ori[0] < 0.1 && dir == 1) rspd_update(a, t_rspd, totLen - p - len[0], fullLen, frac);
                    }
                } else {
                    il = a.insertL[j];
                    if (il > a.gld_lb && il <= a.gld_lb + a.gld_span) red_add(t_gld + (il - a.gld_lb), frac);
                    if (m.est_rspd) rspd_update(a, t_rspd, dir == 0 ? p : totLen - p - il, fullLen, frac);
                }
            }
            const bool noise_on = pass == 0 && valid && f0 != 0.0;  // the read's noise update rides on its first pass

            bool on[NM], has[NM];
            int leader[NM];
            double wg[NM];
            int lmax = 0;
#pragma unroll
            for (int mt = 0; mt < NM; ++mt) {
                const int mpos = mt == 0 ? p : totLen - p - il;
                on[mt] = act && len[mt] > 0 && mpos >= 0 && mpos + len[mt] <= totLen;  // QProfile::update guard
                const unsigned bm = __ballot_sync(0xffffffffu, on[mt]) & group_mask;
                has[mt] = bm != 0;
                leader[mt] = bm ? __ffs(bm) - 1 : lane;
                wg[mt] = lane_group_sum<G>(on[mt] ? frac : 0.0);
                lmax = max(lmax, (on[mt] || noise_on) ? len[mt] : 0);
            }
            lmax = __reduce_max_sync(0xffffffffu, lmax);
            const int mpos1 = PAIRED ? totLen - p - il : 0;
            RefStream ref0(a.seq + (on[0] ? a.seq_off[t] + (dir == 0 ? p : totLen - 1 - p) : 0), dir != 0, a.seq, on[0]);
            RefStream ref1(a.seq + (on[NM - 1] && PAIRED ? a.seq_off[t] + (dir != 0 ? mpos1 : totLen - 1 - mpos1) : 0),
                           dir == 0, a.seq, PAIRED && on[NM - 1]);
            const bool rd0 = valid && (has[0] || noise_on) && len[0] > 0;
            const bool rd1 = PAIRED && valid && (has[NM - 1] || noise_on) && len[NM - 1] > 0;
            FwdBytes rb0(a.rbase[0] + ro[0], rd0), rq0(a.rqual[0] + ro[0], rd0);
            FwdBytes rb1(a.rbase[NM - 1] + ro[NM - 1], rd1), rq1(a.rqual[NM - 1] + ro[NM - 1], rd1);

            for (int k0 = 0; k0 < lmax; k0 += 8) {
                unsigned long long ws[NM], wr[NM], wq[NM];
                ws[0] = ref0.next(on[0] && k0 + 8 < len[0]);
                wr[0] = rb0.next(rd0 && k0 + 8 < len[0]);
                wq[0] = rq0.next(rd0 && k0 + 8 < len[0]);
                if (PAIRED) {
                    ws[NM - 1] = ref1.next(on[NM - 1] && k0 + 8 < len[NM - 1]);
                    wr[NM - 1] = rb1.next(rd1 && k0 + 8 < len[NM - 1]);
                    wq[NM - 1] = rq1.next(rd1 && k0 + 8 < len[NM - 1]);
                }
#pragma unroll
                for (int k = 0; k < 8; k += 2) {
                    if (k0 + k >= lmax) break;  // warp-uniform
                    // items x = 2 * mate + (position parity)
                    int c[NI], c_lead[NI], qv[NI], rv[NI];
                    bool inb[NI];
#pragma unroll
                    for (int x = 0; x < NI; ++x) {
                        const int mt = x >> 1, kk = k + (x & 1);
                        inb[x] = k0 + kk < len[mt];
                        c[x] = mt == 0 ? ref0.base_at(ws[0], kk) : ref1.base_at(ws[NM - 1], kk);
                        qv[x] = (int)byte_of(wq[mt], kk);
                        rv[x] = (int)byte_of(wr[mt], kk);
                        c_lead[x] = __shfl_sync(0xffffffffu, c[x], leader[mt]);
                    }
                    // Items on which a group agrees are added to the warp's shared-memory tables with its summed
                    // weight; the 2 NI (profile, noise) items of a group are spread over its lanes so that the whole
                    // warp issues ONE shared-memory atomic (a compare-and-swap loop in SASS; lanes of different groups
                    // often name the same hot cell).  Where the transcripts of a group disagree (exon junctions,
                    // alleles, spurious alignments) every lane sends its own weight to the global block instead -
                    // those are the cold cells, so the L2 reductions do not pile up on one address.
                    bool agree[NI];
#pragma unroll
                    for (int x = 0; x < NI; ++x) {
                        const int mt = x >> 1;
                        const unsigned dis = __ballot_sync(0xffffffffu, on[mt] && inb[x] && c[x] != c_lead[x]) & group_mask;
                        agree[x] = dis == 0;
                        if (!agree[x] && on[mt] && inb[x]) red_add(blk + (qv[x] * 5 + c[x]) * 5 + rv[x], frac);
                    }
#pragma unroll
                    for (int x0 = 0; x0 < 2 * NI; x0 += G) {
                        const int it = x0 + g;  // this lane's item: 0 .. NI-1 profile, NI .. 2 NI - 1 noise
                        double* tab = tprof;
                        int cell = 0;
                        double w = 0.0;
                        bool ok = false;
#pragma unroll
                        for (int x = 0; x < NI; ++x) {
                            const int mt = x >> 1;
                            if (it == x) {
                                ok = has[mt] && inb[x] && agree[x];
                                cell = (qv[x] * 5 + c_lead[x]) * 5 + rv[x];
                                w = wg[mt];
                            }
                            if (it == NI + x) {
                                ok = noise_on && inb[x];
                                cell = qv[x] * 5 + rv[x];
                                w = f0;
                                tab = tnoise;
                            }
                        }
                        if (ok) atomicAdd(tab + cell, w);
                    }
                }
            }
        }
    }
    __syncthreads();
    double* out = a.stats + (size_t)(blockIdx.x % kReplicas) * a.stats_block;
    for (int cidx = threadIdx.x; cidx < kQTab; cidx += blockDim.x) {
        double v = 0.0;
        for (int w = 0; w < kQWarps; ++w) v += q_tabs[w * kQTab + cidx];
        if (v != 0.0) red_add(out + (cidx < n_prof ? (size_t)cidx : a.o_noise + (size_t)(cidx - n_prof)), v);
    }
}

// ---- K3 for "uniform" reads (all hits show the read the same bases) ---------------------------------------------------
// The profile statistics of such a read are W = sum of its hits' posteriors added once per base, whatever the number of
// hits: the G lanes of the read's group each take a contiguous range of 8-base chunks of the window of hit 0 and add W
// (and the noise posterior) per base - to the warp's private shared-memory tables for the quality models (QProfile:
// ~20 hot cells), to a replica of the global block for the position-indexed Profile.  Per-hit statistics (fragment
// length histogram, RSPD bins) are added by the lanes that own the hits.  Posteriors below 1e-300 are skipped
// (SingleQModel.h:172, 204).
template <int G, bool HASQ, bool PAIRED>
__global__ void __launch_bounds__(kQMaxWarps * 32, 1) update_coop_kernel(const ModelArgs a) {
    extern __shared__ double q_tabs[];
    const int n_warps = blockDim.x >> 5;
    const int n_prof = a.q_rows * 25, kQTab = a.q_rows * 30;
    constexpr int R = 32 / G;
    constexpr int NM = PAIRED ? 2 : 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane % G, grp = lane / G;
    double* blk = a.stats + (size_t)((blockIdx.x * n_warps + warp) % kReplicas) * a.stats_block;
    double* tprof = HASQ ? q_tabs + warp * kQTab : blk;
    double* tnoise = HASQ ? tprof + n_prof : blk + a.o_noise;
    if (HASQ) {
        for (int k = lane; k < kQTab; k += 32) tprof[k] = 0.0;
        __syncwarp();
    }
    double* t_gld = blk + a.o_gld;
    double* t_rspd = blk + a.o_rspd;
    const DevModel& m = a.m;
    const unsigned long long warps_total = (unsigned long long)gridDim.x * n_warps;
    for (unsigned long long base = ((unsigned long long)blockIdx.x * n_warps + warp) * R; base < a.N; base += warps_total * R) {
        const unsigned long long i = base + grp;
        const bool valid = i < a.N && !a.lowq[i] && a.uni[i];
        if (__ballot_sync(0xffffffffu, valid) == 0u) continue;
        unsigned long long fr = 0, to = 0;
        double f0 = 0.0;
        if (valid) {
            fr = a.row_ptr[i];
            to = a.row_ptr[i + 1];
            f0 = a.post0[i];
            if (f0 < kEpsilon) f0 = 0.0;
        }
        int len[NM];
        unsigned long long ro[NM];
#pragma unroll
        for (int mt = 0; mt < NM; ++mt) {
            ro[mt] = valid ? a.roff[mt][i] : 0ull;
            len[mt] = valid ? (int)(a.roff[mt][i + 1] - ro[mt]) : 0;
        }
        // per-hit statistics and the summed posterior
        double wsum = 0.0;
        for (unsigned long long j = fr + g; j < to; j += G) {
            const double frac = a.post[j];
            if (frac < kEpsilon) continue;
            wsum += frac;
            const int sgn = a.sid[j], t = abs(sgn), dir = sgn < 0, p = a.pos[j];
            const int fullLen = a.full_len[t], totLen = a.tot_len[t];
            if (!PAIRED) {
                if (m.est_rspd) {  // one strand only (SingleQModel.h:180-184; helper models have mld == NULL)
                    if (m.ori[0] >= 0.1 && dir == 0) rspd_update(a, t_rspd, p, fullLen, frac);
                    if (m.ori[0] < 0.1 && dir == 1) rspd_update(a, t_rspd, totLen - p - len[0], fullLen, frac);
                }
            } else {
                const int il = a.insertL[j];
                if (il > a.gld_lb && il <= a.gld_lb + a.gld_span) red_add(t_gld + (il - a.gld_lb), frac);
                if (m.est_rspd) rspd_update(a, t_rspd, dir == 0 ? p : totLen - p - il, fullLen, frac);
            }
        }
        const double W = lane_group_sum<G>(wsum);
        // the window: hit 0
        int s0 = 1, p0 = 0, il0 = 0;
        if (valid && to > fr) { s0 = a.sid[fr]; p0 = a.pos[fr]; if (PAIRED) il0 = a.insertL[fr]; }
        const int t0 = abs(s0), d0 = s0 < 0, totLen0 = a.tot_len[t0];
#pragma unroll
        for (int mt = 0; mt < NM; ++mt) {
            if (!valid || len[mt] <= 0 || (W == 0.0 && f0 == 0.0)) continue;
            const int n_chunks = (len[mt] + 7) >> 3;
            const int c0 = g * n_chunks / G, c1 = (g + 1) * n_chunks / G;
            if (c1 <= c0) continue;
            const int mpos = mt == 0 ? p0 : totLen0 - p0 - il0, mdir = mt == 0 ? d0 : !d0;
            const bool prof_on = W != 0.0 && to > fr;
            FwdBytes rb(a.rbase[mt] + ro[mt] + 8 * c0);
            FwdBytes rq(HASQ ? a.rqual[mt] + ro[mt] + 8 * c0 : a.rbase[mt] + ro[mt], HASQ);
            RefStream sb(a.seq + (prof_on ? a.seq_off[t0] + (mdir == 0 ? mpos + 8 * c0 : totLen0 - 1 - mpos - 8 * c0) : 0), mdir != 0,
                         a.seq, prof_on);
            for (int c = c0; c < c1; ++c) {
                const bool more = c + 1 < c1;
                const unsigned long long ws = sb.next(prof_on && more), wr = rb.next(more), wq = HASQ ? rq.next(more) : 0ull;
                const int k0 = 8 * c, n = min(8, len[mt] - k0);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (k < n) {
                        const int rv = (int)byte_of(wr, k);
                        const int row = HASQ ? (int)byte_of(wq, k) : k0 + k;
                        if (prof_on) {
                            double* cell = tprof + (row * 5 + sb.base_at(ws, k)) * 5 + rv;
                            if (HASQ) atomicAdd(cell, W); else red_add(cell, W);
                        }
                        if (f0 != 0.0) {
                            double* cell = tnoise + (HASQ ? row * 5 + rv : rv);
                            if (HASQ) atomicAdd(cell, f0); else red_add(cell, f0);
                        }
                    }
                }
            }
        }
    }
    if (HASQ) {
        __syncthreads();
        double* out = a.stats + (size_t)(blockIdx.x % kReplicas) * a.stats_block;
        for (int cidx = threadIdx.x; cidx < kQTab; cidx += blockDim.x) {
            double v = 0.0;
            for (int w = 0; w < n_warps; ++w) v += q_tabs[w * kQTab + cidx];
            if (v != 0.0) red_add(out + (cidx < n_prof ? (size_t)cidx : a.o_noise + (size_t)(cidx - n_prof)), v);
        }
    }
}

__global__ void max_u8_kernel(const unsigned char* v, unsigned long long n, unsigned int* out) {
    unsigned int m = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x)
        m = max(m, (unsigned int)v[i]);
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void fold_replicas_kernel(double* stats, size_t block) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= block) return;
    double s = 0.0;
    for (int r = 0; r < kReplicas; ++r) s += stats[(size_t)r * block + k];
    stats[k] = s;
}

void fill_args(rsem_b200_ctx* c, ModelArgs& a) {
    a.m = c->model;
    a.n_mates = c->reads.n_mates;
    for (int k = 0; k < 2; ++k) {
        a.roff[k] = reinterpret_cast<const unsigned long long*>(c->reads.off[k]);
        a.rbase[k] = c->reads.base[k];
        a.rqual[k] = c->reads.qual[k];
    }
    a.lowq = c->reads.lowq;
    a.seq_off = reinterpret_cast<const unsigned long long*>(c->refs.seq_off);
    a.seq = c->refs.seq;
    a.full_len = c->refs.full_len;
    a.tot_len = c->refs.tot_len;
    a.mask_off = reinterpret_cast<const unsigned long long*>(c->refs.mask_off);
    a.mask_words = c->refs.mask_words;
    a.N = c->N;
    a.row_ptr = reinterpret_cast<const unsigned long long*>(c->row_ptr);
    a.sid = c->sid;
    a.pos = c->pos;
    a.insertL = c->insertL;
    a.conprb = c->conprb;
    a.ncpv = c->ncpv;
    a.post = c->post;
    a.post0 = c->post0;
    a.err_flag = c->err_flag;
    a.uni = c->reads.uni;
    a.mode = 0;
    const bool hasq = c->model.model_type & 1;
    int rows = hasq ? 100 : std::min(c->model.pro_len, std::max(c->reads.max_len, 1));
    if ((size_t)rows * 200 + 4096 > 200 * 1024) rows = 0;
    a.prof_rows_smem = rows;
    a.q_rows = c->reads.qmax >= 0 ? std::min(c->reads.qmax + 1, 100) : 100;
    a.stats = c->stats_buf;
    a.stats_block = c->stats.total_doubles;
    a.o_noise = c->stats.noise_profile ? (size_t)(c->stats.noise_profile - c->stats_buf) : 0;
    a.o_gld = c->stats.gld_pdf ? (size_t)(c->stats.gld_pdf - c->stats_buf) : 0;
    a.o_rspd = c->stats.rspd_pdf ? (size_t)(c->stats.rspd_pdf - c->stats_buf) : 0;
    a.gld_lb = c->stats.gld_lb;
    a.gld_span = c->stats.gld_span;
}

template <int G>
int launch_conprb_g(rsem_b200_ctx* c, const ModelArgs& a, unsigned grid, size_t smem) {
    const bool hasq = c->model.model_type & 1, paired = c->model.model_type >= 2;
#define RB_LAUNCH(Q, P)                                                                                      \
    do {                                                                                                     \
        if (smem) {                                                                                          \
            auto k = conprb_kernel<G, Q, P, true>;                                                           \
            if (smem > 48 * 1024) RB_CUDA(raise_dyn_smem((const void*)k, smem));                             \
            k<<<grid, kBlock, smem, c->stream>>>(a);                                                         \
        } else {                                                                                             \
            conprb_kernel<G, Q, P, false><<<grid, kBlock, 0, c->stream>>>(a);                                \
        }                                                                                                    \
    } while (0)
    if (hasq && paired) RB_LAUNCH(true, true);
    else if (hasq) RB_LAUNCH(true, false);
    else if (paired) RB_LAUNCH(false, true);
    else RB_LAUNCH(false, false);
#undef RB_LAUNCH
    RB_CUDA(cudaGetLastError());
    c->launches++;
    return 0;
}

template <int G, bool PAIRED>
int launch_update_q(rsem_b200_ctx* c, const ModelArgs& a) {
    auto k = update_q_kernel<G, PAIRED>;
    const size_t per_warp = (size_t)a.q_rows * 30 * sizeof(double);
    const int warps = (int)std::max<size_t>(1, std::min<size_t>(kQMaxWarps, (size_t)(200 * 1024) / per_warp));
    const size_t smem = per_warp * warps;
    RB_CUDA(raise_dyn_smem((const void*)k, smem));
    k<<<c->sm_count, warps * 32, smem, c->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    c->launches++;
    return 0;
}

template <int G, bool HASQ, bool PAIRED>
int launch_update_coop(rsem_b200_ctx* c, const ModelArgs& a) {
    auto k = update_coop_kernel<G, HASQ, PAIRED>;
    const size_t per_warp = HASQ ? (size_t)a.q_rows * 30 * sizeof(double) : 0;
    const int warps = HASQ ? (int)std::max<size_t>(1, std::min<size_t>(kQMaxWarps, (size_t)(200 * 1024) / per_warp)) : kQMaxWarps;
    const size_t smem = per_warp * warps;
    if (smem > 48 * 1024) RB_CUDA(raise_dyn_smem((const void*)k, smem));
    k<<<c->sm_count * (HASQ ? 1 : 2), warps * 32, smem, c->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    c->launches++;
    return 0;
}

template <int G>
int launch_update_g(rsem_b200_ctx* c, ModelArgs& a, unsigned grid) {
    const bool hasq = c->model.model_type & 1, paired = c->model.model_type >= 2;
    a.mode = 0;
    if (c->reads.uni_valid && !getenv("RSEM_B200_NO_COOP")) {   // uniform reads first, the per-hit kernels skip them (mode 2)
        a.mode = 1;
        int rc;
        if (hasq && paired) rc = launch_update_coop<G, true, true>(c, a);
        else if (hasq) rc = launch_update_coop<G, true, false>(c, a);
        else if (paired) rc = launch_update_coop<G, false, true>(c, a);
        else rc = launch_update_coop<G, false, false>(c, a);
        if (rc) return rc;
        a.mode = 2;
    }
    const bool global_reds = getenv("RSEM_B200_K3") && !strcmp(getenv("RSEM_B200_K3"), "global");
    if (hasq && !global_reds) return paired ? launch_update_q<G, true>(c, a) : launch_update_q<G, false>(c, a);
    if (hasq && paired) update_kernel<G, true, true><<<grid, kBlock, 0, c->stream>>>(a);
    else if (hasq) update_kernel<G, true, false><<<grid, kBlock, 0, c->stream>>>(a);
    else if (paired) update_kernel<G, false, true><<<grid, kBlock, 0, c->stream>>>(a);
    else update_kernel<G, false, false><<<grid, kBlock, 0, c->stream>>>(a);
    RB_CUDA(cudaGetLastError());
    c->launches++;
    return 0;
}

unsigned grid_for(rsem_b200_ctx* c, int G) {
    const unsigned long long per_block = kBlock / G;
    unsigned long long want = (c->N + per_block - 1) / per_block;
    if (want < 1) want = 1;
    return (unsigned)std::min<unsigned long long>(want, (unsigned long long)c->sm_count * 8);
}

}  // namespace

// per read: do all its hits show it the same bases?  Depends on hits, read lengths and transcripts only: once per upload.
static int ensure_uniform_flags(rsem_b200_ctx* c) {
    if (c->reads.uni_valid) return 0;
    if (!c->reads.uni) RB_CUDA(cudaMalloc(&c->reads.uni, c->N + 16));
    ModelArgs a;
    fill_args(c, a);
    const int G = c->group;
    const unsigned grid = grid_for(c, G);
    const bool paired = c->model.model_type >= 2;
#define RB_UNI(GG)                                                                                         \
    do {                                                                                                   \
        if (paired) window_uniform_kernel<GG, true><<<grid, kBlock, 0, c->stream>>>(a, c->reads.uni);      \
        else window_uniform_kernel<GG, false><<<grid, kBlock, 0, c->stream>>>(a, c->reads.uni);            \
    } while (0)
    switch (G) {
        case 4: RB_UNI(4); break;
        case 8: RB_UNI(8); break;
        case 16: RB_UNI(16); break;
        default: RB_UNI(32); break;
    }
#undef RB_UNI
    RB_CUDA(cudaGetLastError());
    c->launches++;
    c->reads.uni_valid = true;
    return 0;
}

template <int G>
static int launch_conprb_modes(rsem_b200_ctx* c, ModelArgs& a, unsigned grid, size_t smem, bool coop) {
    if (!coop) { a.mode = 0; return launch_conprb_g<G>(c, a, grid, smem); }
    a.mode = 1;
    if (int rc = launch_conprb_g<G>(c, a, grid, smem)) return rc;
    a.mode = 2;
    return launch_conprb_g<G>(c, a, grid, smem);
}

int model_launch_conprb(rsem_b200_ctx* c) {
    if (c->N == 0) return 0;
    // reads whose hits all show them the same bases take the cooperative path (one pass over the bases per READ instead
    // of per hit); RSEM_B200_NO_COOP=1 keeps every read on the per-hit path (the reference's multiplication order)
    const bool no_coop = getenv("RSEM_B200_NO_COOP") != nullptr;
    if (!no_coop) if (int rc = ensure_uniform_flags(c)) return rc;
    ModelArgs a;
    fill_args(c, a);
    const bool hasq = c->model.model_type & 1;
    const size_t smem = a.prof_rows_smem ? ((size_t)a.prof_rows_smem * 25 + (hasq ? 500 : 5)) * sizeof(double) : 0;
    const int G = c->group;
    const unsigned grid = grid_for(c, G);
    switch (G) {
        case 4: return launch_conprb_modes<4>(c, a, grid, smem, !no_coop);
        case 8: return launch_conprb_modes<8>(c, a, grid, smem, !no_coop);
        case 16: return launch_conprb_modes<16>(c, a, grid, smem, !no_coop);
        default: return launch_conprb_modes<32>(c, a, grid, smem, !no_coop);
    }
}

int model_launch_update(rsem_b200_ctx* c) {
    // (re)build the statistics block layout: [profile][noise][gld][rspd], kReplicas copies
    const bool hasq = c->model.model_type & 1, paired = c->model.model_type >= 2;
    const size_t n_prof = hasq ? 2500 : (size_t)c->model.pro_len * 25, n_noise = hasq ? 500 : 5;
    const size_t n_gld = paired ? (size_t)c->stats.gld_span + 1 : 0;
    const size_t n_rspd = c->model.est_rspd ? (size_t)c->model.rspd_B + 2 : 0;
    const size_t block = n_prof + n_noise + n_gld + n_rspd;
    if (c->stats_buf_doubles < block * kReplicas) {
        if (c->stats_buf) cudaFree(c->stats_buf);
        RB_CUDA(cudaMalloc(&c->stats_buf, block * kReplicas * sizeof(double)));
        c->stats_buf_doubles = block * kReplicas;
    }
    c->stats.total_doubles = block;
    c->stats.profile = c->stats_buf;
    c->stats.noise_profile = c->stats_buf + n_prof;
    c->stats.gld_pdf = c->stats_buf + n_prof + n_noise;
    c->stats.rspd_pdf = c->stats_buf + n_prof + n_noise + n_gld;
    RB_CUDA(cudaMemsetAsync(c->stats_buf, 0, block * kReplicas * sizeof(double), c->stream));
    if (c->N == 0) return 0;
    if (hasq && c->reads.qmax < 0) {  // largest quality value of the resident read set, once per upload
        unsigned int* d_max = nullptr;
        unsigned int h_max = 0;
        RB_CUDA(cudaMalloc(&d_max, sizeof(unsigned int)));
        RB_CUDA(cudaMemsetAsync(d_max, 0, sizeof(unsigned int), c->stream));
        for (int mt = 0; mt < c->reads.n_mates; ++mt) {
            const unsigned long long nb = c->reads.total_bases[mt];
            if (nb) max_u8_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(c->reads.qual[mt], nb, d_max);
        }
        RB_CUDA(cudaMemcpyAsync(&h_max, d_max, sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
        RB_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(d_max);
        c->reads.qmax = (int)h_max;
        c->launches += c->reads.n_mates;
    }
    ModelArgs a;
    fill_args(c, a);
    const int G = c->group;
    const unsigned grid = grid_for(c, G);
    int rc;
    switch (G) {
        case 4: rc = launch_update_g<4>(c, a, grid); break;
        case 8: rc = launch_update_g<8>(c, a, grid); break;
        case 16: rc = launch_update_g<16>(c, a, grid); break;
        default: rc = launch_update_g<32>(c, a, grid); break;
    }
    if (rc) return rc;
    fold_replicas_kernel<<<(unsigned)((block + 255) / 256), 256, 0, c->stream>>>(c->stats_buf, block);
    RB_CUDA(cudaGetLastError());
    c->launches++;
    return 0;
}

}  // namespace rsem_b200
