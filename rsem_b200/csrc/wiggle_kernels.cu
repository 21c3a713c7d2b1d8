// K11: the per-alignment work of rsem-bam2wig and rsem-bam2readdepth (build_wiggles, wiggle.cpp:16-83).
//
// The reference walks every aligned base of every record on one thread and adds the record's weight into one
// std::vector<double> per target, so each position's value is a left-to-right double sum in file order.  Here one batch
// of mapped records (runs of one target, see include/rsem_b200.h) goes through:
//   parse       one thread per record: the first ZW with htslib 1.3's skip_aux rules (or 1.0), the CIGAR walk, the
//               number of M blocks and of (tile, block) entries, the error code of the first bad record
//   scan        exclusive sums of both counts -> where each record's blocks and entries go
//   emit        the same walk, writing blocks (start, end, w) in record order and one entry (tile key, block) for every
//               tile of kTile positions a block touches
//   sort        cub's stable radix sort of the entries by tile key: each tile's list stays in record order
//   accumulate  one CTA per tile, one thread per position: the position's current value (non-zero when the run
//               continues from an earlier call), then every block of the tile's list in order, staged through shared
//               memory, added where it covers the position; one store at the end
// The adds restate x86 SSE's addsd for NaN and infinities (sse_add) and are __dadd_rn, so nothing is contracted or
// reassociated.  A tile under a deep pileup is one serial chain per position: that is the order the reference adds in.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {

namespace {
constexpr int kThreads = 256;
constexpr int kTile = 256;   // positions per accumulate CTA, one per thread
}  // namespace

struct WigBlock {
    double w;
    uint32_t start, end;     // positions [start, end) of the run
};

struct WigState {
    double* depth[2] = {nullptr, nullptr};   // the batch's runs back to back, run 0 at offset 0; ping-pong for keep_last
    size_t sz_depth[2] = {0, 0};
    int cur = 0;
    bool resident = false;                   // depth[cur][0, resident_len) is the run the last call kept
    uint64_t resident_len = 0;
    // per record (one capacity)
    uint8_t* data = nullptr;
    uint64_t *rec_off = nullptr, *blk_off = nullptr, *ent_off = nullptr;
    uint32_t* rec_run = nullptr;
    double* w = nullptr;
    // per run
    uint32_t* run_len = nullptr;
    uint64_t *run_off = nullptr, *run_tile = nullptr;
    // per entry (one capacity)
    WigBlock* blk = nullptr;
    uint32_t *key[2] = {nullptr, nullptr}, *val[2] = {nullptr, nullptr};
    void* temp = nullptr;
    unsigned long long* err = nullptr;
    size_t sz_data = 0, sz_rec = 0, sz_run = 0, sz_ent = 0, sz_temp = 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};
};

namespace {

enum Bad : unsigned { kBadM = 1, kBadAux = 2, kBadTrunc = 3 };

// operand order of the reference's `read_depth[pos] += w` (wiggle.cpp:32): both the scalar and the vectorised loop of
// the -O3 build keep the NaN of the depth operand when both are NaN (objdump of the reference build; DESIGN §3 K11)
constexpr bool kKeepDepthNaN = true;

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }

// bam_cigar_type (htslib 1.3 sam.h:104): bit 2 = consumes the reference
__device__ __forceinline__ bool consumes_ref(uint32_t op) { return (0x3C1A7u >> (op << 1)) & 2u; }

// cvtss2sd: a float NaN keeps its sign and payload and comes out quiet; everything else widens exactly
__device__ __forceinline__ double widen(uint32_t f) {
    if ((f & 0x7f800000u) == 0x7f800000u && (f & 0x7fffffu))
        return __longlong_as_double((long long)(((uint64_t)(f >> 31) << 63) | 0x7ff8000000000000ull | ((uint64_t)(f & 0x7fffffu) << 29)));
    return (double)__uint_as_float(f);
}

// addsd with the depth as the destination operand: a NaN operand comes out quiet with its sign and payload (the
// destination's when both are NaN); inf + -inf is the default NaN, sign bit set
__device__ __forceinline__ double sse_add(double d, double w) {
    const uint64_t ud = (uint64_t)__double_as_longlong(d), uw = (uint64_t)__double_as_longlong(w);
    const bool nd = (ud & 0x7fffffffffffffffull) > 0x7ff0000000000000ull;
    const bool nw = (uw & 0x7fffffffffffffffull) > 0x7ff0000000000000ull;
    if (nd || nw) {
        const uint64_t r = (nd && (kKeepDepthNaN || !nw)) ? ud : uw;
        return __longlong_as_double((long long)(r | 0x0008000000000000ull));
    }
    if ((ud & 0x7fffffffffffffffull) == 0x7ff0000000000000ull && (uw ^ ud) == 0x8000000000000000ull)
        return __longlong_as_double((long long)0xfff8000000000000ull);
    return __dadd_rn(d, w);
}

__device__ __forceinline__ void flag_bad(unsigned long long* err, uint32_t r, unsigned why) {
    atomicMin(err, ((unsigned long long)r << 8) | why);
}

// aux_type2size of htslib 1.3 (sam.c:344-360)
__device__ __forceinline__ uint64_t aux_type2size(uint8_t t) {
    switch (t) {
        case 'A': case 'c': case 'C': return 1;
        case 's': case 'S': return 2;
        case 'i': case 'I': case 'f': return 4;
        case 'd': return 8;
        case 'Z': case 'H': case 'B': return t;
    }
    return 0;
}

// bytes skip_aux (htslib 1.3 sam.c:1233-1252) steps over for the field whose type byte is at s, type byte included; 0 =
// unknown type (skip_aux aborts).  A 'B' array advances by aux_type2size(subtype) * count whatever the subtype, as
// skip_aux does; the other types are the shared aux_len.  The result may run past `end`: the caller checks.
__device__ __forceinline__ uint64_t skip_aux_len(const uint8_t* s, const uint8_t* end) {
    if (*s != 'B') {
        const int len = aux_len(s, end);
        return len > 0 ? (uint64_t)len : 0;
    }
    if (end - s < 6) return 6;   // the subtype and count run past the end
    return 6 + aux_type2size(s[1]) * (uint64_t)rd32(s + 2);
}

struct Rec {
    const uint8_t* cigar;
    uint32_t n_cig;
    int64_t pos;
    double w;
    bool adds;       // false: no ZW, the record adds nothing
    unsigned bad;
};

// the record after its block_size: the weight as add_bam_record_to_wiggle takes it (bam_aux_get + bam_aux2f, which scan
// only up to the first ZW), and the CIGAR
__device__ Rec read_rec(const uint8_t* rec, bool no_frac) {
    Rec r{nullptr, 0, 0, 1.0, true, 0};
    const uint32_t bs = rd32(rec);
    const uint8_t* in = rec + 4;
    const uint8_t* end = in + bs;
    if (bs < 32) { r.bad = kBadTrunc; return r; }
    r.pos = (int32_t)rd32(in + 4);
    r.n_cig = rd16(in + 12);
    const uint32_t l_seq = rd32(in + 16);
    r.cigar = in + 32 + in[8];
    if ((uint64_t)(end - r.cigar) < 4ull * r.n_cig) { r.bad = kBadTrunc; return r; }
    if (no_frac) return r;
    const uint64_t skip = 4ull * r.n_cig + (l_seq + 1ull) / 2 + l_seq;
    if ((uint64_t)(end - r.cigar) < skip) { r.bad = kBadTrunc; return r; }
    for (const uint8_t* a = r.cigar + skip; a < end;) {
        if (a + 3 > end) { r.bad = kBadTrunc; return r; }
        if (a[0] == 'Z' && a[1] == 'W') {
            const uint8_t t = a[2];
            if (t == 'f') {
                if (a + 7 > end) { r.bad = kBadTrunc; return r; }
                r.w = widen(rd32(a + 3));
            } else if (t == 'd') {
                if (a + 11 > end) { r.bad = kBadTrunc; return r; }
                r.w = __longlong_as_double((long long)((uint64_t)rd32(a + 3) | (uint64_t)rd32(a + 7) << 32));
            } else {
                r.w = 0.0;
            }
            return r;
        }
        const uint64_t len = skip_aux_len(a + 2, end);
        if (len == 0) { r.bad = kBadAux; return r; }
        if ((uint64_t)(end - a) < 2 + len) { r.bad = kBadTrunc; return r; }
        a += 2 + len;
    }
    r.adds = false;
    return r;
}

struct Batch {
    const uint8_t* data;
    const uint64_t* rec_off;
    const uint32_t* rec_run;
    const uint32_t* run_len;
    const uint64_t* run_tile;
    uint32_t n;
    bool no_frac;
};

__global__ void wig_parse_kernel(Batch B, uint64_t* __restrict__ n_blk, uint64_t* __restrict__ n_ent,
                                 double* __restrict__ w, unsigned long long* err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n) return;
    n_blk[i] = 0;
    n_ent[i] = 0;
    const Rec r = read_rec(B.data + B.rec_off[i], B.no_frac);
    if (r.bad) { flag_bad(err, i, r.bad); return; }
    if (!r.adds) return;
    const int64_t len_t = B.run_len[B.rec_run[i]];
    int64_t p = r.pos;
    uint64_t nb = 0, ne = 0;
    for (uint32_t k = 0; k < r.n_cig; ++k) {
        const uint32_t c = rd32(r.cigar + 4 * k), op = c & 15u, l = c >> 4;
        if (op == 0) {
            if (l == 0) continue;
            if (p + l > len_t) { flag_bad(err, i, kBadM); return; }
            ++nb;
            ne += (uint64_t)((p + l - 1) / kTile - p / kTile + 1);
            p += l;
        } else if (consumes_ref(op)) {
            p += l;
        }
    }
    n_blk[i] = nb;
    n_ent[i] = ne;
    w[i] = r.w;
}

__global__ void wig_emit_kernel(Batch B, const uint64_t* __restrict__ blk_off, const uint64_t* __restrict__ ent_off,
                                const double* __restrict__ w, WigBlock* __restrict__ blk, uint32_t* __restrict__ key,
                                uint32_t* __restrict__ val) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n) return;
    uint64_t b = blk_off[i], e = ent_off[i];
    if (blk_off[i + 1] == b) return;
    const Rec r = read_rec(B.data + B.rec_off[i], true);   // the CIGAR only: w comes from the parse pass
    const double wi = w[i];
    const uint64_t tile0 = B.run_tile[B.rec_run[i]];
    int64_t p = r.pos;
    for (uint32_t k = 0; k < r.n_cig; ++k) {
        const uint32_t c = rd32(r.cigar + 4 * k), op = c & 15u, l = c >> 4;
        if (op == 0) {
            if (l == 0) continue;
            blk[b] = WigBlock{wi, (uint32_t)p, (uint32_t)(p + l)};
            for (int64_t t = p / kTile; t <= (p + l - 1) / kTile; ++t) {
                key[e] = (uint32_t)(tile0 + t);
                val[e] = (uint32_t)b;
                ++e;
            }
            ++b;
            p += l;
        } else if (consumes_ref(op)) {
            p += l;
        }
    }
}

// one CTA per tile of the batch: [lo, hi) of the sorted entries with its key, then the ordered sum per position
__global__ void __launch_bounds__(kTile) wig_accumulate_kernel(const uint32_t* __restrict__ key, const uint32_t* __restrict__ val,
                                                               uint64_t n_ent, const WigBlock* __restrict__ blk,
                                                               const uint32_t* __restrict__ run_len,
                                                               const uint64_t* __restrict__ run_off,
                                                               const uint64_t* __restrict__ run_tile, uint32_t n_runs,
                                                               double* __restrict__ depth) {
    __shared__ uint32_t s_start[kTile], s_end[kTile];
    __shared__ double s_w[kTile];
    const uint32_t tile = blockIdx.x;
    uint64_t lo = 0, hi = n_ent;
    while (lo < hi) {   // first entry with key >= tile
        const uint64_t m = (lo + hi) / 2;
        if (key[m] < tile) lo = m + 1; else hi = m;
    }
    uint64_t end = lo, top = n_ent;
    while (end < top) {   // first entry with key > tile
        const uint64_t m = (end + top) / 2;
        if (key[m] <= tile) end = m + 1; else top = m;
    }
    if (lo == end) return;
    uint32_t a = 0, b = n_runs;   // the run: last with run_tile <= tile
    while (b - a > 1) {
        const uint32_t m = (a + b) / 2;
        if (run_tile[m] <= tile) a = m; else b = m;
    }
    const uint64_t p = (uint64_t)(tile - run_tile[a]) * kTile + threadIdx.x;
    const bool mine = p < run_len[a];
    double v = mine ? depth[run_off[a] + p] : 0.0;
    for (uint64_t c = lo; c < end; c += kTile) {
        __syncthreads();
        if (c + threadIdx.x < end) {
            const WigBlock k = blk[val[c + threadIdx.x]];
            s_start[threadIdx.x] = k.start;
            s_end[threadIdx.x] = k.end;
            s_w[threadIdx.x] = k.w;
        }
        __syncthreads();
        const int n = end - c < (uint64_t)kTile ? (int)(end - c) : kTile;
        for (int j = 0; j < n; ++j)
            if (p >= s_start[j] && p < s_end[j]) v = sse_add(v, s_w[j]);
    }
    if (mine) depth[run_off[a] + p] = v;
}

template <class T>
int realloc_n(T** p, size_t n) {
    if (*p) cudaFree(*p);
    *p = nullptr;
    RB_CUDA(cudaMalloc((void**)p, std::max<size_t>(n, 1) * sizeof(T)));
    return 0;
}

// capacity for n: grown by a quarter beyond the request so that slowly growing batches do not reallocate every call
size_t grown(size_t n) { return std::max<size_t>(n + n / 4, 1024); }

const char* bad_text(unsigned why) {
    switch (why) {
        case kBadM: return "an M operation that ends past the end of its target (reference: writes past its depth vector)";
        case kBadAux: return "an optional field of unknown type before the first ZW (reference: abort() in bam_aux_get)";
        default: return "a record cut short: its CIGAR or an optional field before the first ZW runs past its end";
    }
}

// grow depth[k] to hold n doubles, keeping its first `keep` values
int grow_depth(WigState& S, int k, uint64_t n, uint64_t keep, cudaStream_t s) {
    if (n <= S.sz_depth[k] && S.depth[k]) return 0;
    const size_t cap = grown(n);
    double* q = nullptr;
    const cudaError_t e = cudaMalloc((void**)&q, cap * sizeof(double));
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("wig_depth: cannot allocate the depth of " + std::to_string(n) + " positions on the device (" +
                  cudaGetErrorString(e) + ")");
        return RSEM_B200_ERR_CUDA;
    }
    if (keep) RB_CUDA(cudaMemcpyAsync(q, S.depth[k], keep * sizeof(double), cudaMemcpyDeviceToDevice, s));
    RB_CUDA(cudaStreamSynchronize(s));
    if (S.depth[k]) cudaFree(S.depth[k]);
    S.depth[k] = q;
    S.sz_depth[k] = cap;
    return 0;
}

}  // namespace

void wig_free(rsem_b200_ctx* ctx) {
    WigState* S = ctx->wig;
    if (!S) return;
    void* ptrs[] = {S->depth[0], S->depth[1], S->data, S->rec_off, S->blk_off, S->ent_off, S->rec_run, S->w, S->run_len,
                    S->run_off, S->run_tile, S->blk, S->key[0], S->key[1], S->val[0], S->val[1], S->temp, S->err};
    for (void* p : ptrs) if (p) cudaFree(p);
    for (auto& e : S->ev) if (e) cudaEventDestroy(e);
    delete S;
    ctx->wig = nullptr;
}

int wig_depth(rsem_b200_ctx* ctx, const rsem_b200_wig_batch* b, double* out, uint64_t out_cap, uint64_t* out_len,
              rsem_b200_wig_stats* stats) {
    if (!ctx->wig) {
        ctx->wig = new WigState;
        RB_CUDA(cudaEventCreate(&ctx->wig->ev[0]));
        RB_CUDA(cudaEventCreate(&ctx->wig->ev[1]));
        RB_CUDA(cudaMalloc((void**)&ctx->wig->err, sizeof(unsigned long long)));
    }
    WigState& S = *ctx->wig;
    const cudaStream_t s = ctx->stream;
    rsem_b200_wig_stats st{0.0, 0, 0, -1, 0, 0};
    if (stats) *stats = st;   // every early return leaves bad_record = -1
    *out_len = 0;
    const uint32_t R = b->n_runs;
    const uint32_t n = (uint32_t)b->n_records;
    RB_ARG(!b->continues || (S.resident && R > 0 && b->run_len[0] == S.resident_len), "continues without a matching resident run");
    for (uint64_t i = 1; i < b->n_records; ++i)
        RB_ARG(b->rec_run[i - 1] <= b->rec_run[i], "rec_run must not decrease");
    RB_ARG(n == 0 || b->rec_run[n - 1] < R, "rec_run out of range");

    // where the runs go, and what this call hands back
    std::vector<uint64_t> run_off(R + 1, 0), run_tile(R + 1, 0);
    for (uint32_t i = 0; i < R; ++i) {
        run_off[i + 1] = run_off[i] + b->run_len[i];
        run_tile[i + 1] = run_tile[i] + (b->run_len[i] + kTile - 1) / kTile;
    }
    RB_ARG(run_tile[R] < 0xffffffffull, "batch spans too many positions");
    const bool flush_resident = S.resident && !b->continues;
    const uint32_t done_runs = R - (R > 0 && b->keep_last ? 1 : 0);
    const uint64_t want = (flush_resident ? S.resident_len : 0) + run_off[done_runs];
    RB_ARG(want <= out_cap, "wig_depth: the output buffer is too small");
    RB_CUDA(cudaEventRecord(S.ev[0], s));
    uint64_t at = 0;
    if (flush_resident) {
        if (S.resident_len) RB_CUDA(cudaMemcpyAsync(out, S.depth[S.cur], S.resident_len * 8, cudaMemcpyDeviceToHost, s));
        at = S.resident_len;
        S.resident = false;
    }
    auto finish = [&]() -> int {
        RB_CUDA(cudaEventRecord(S.ev[1], s));
        RB_CUDA(cudaStreamSynchronize(s));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, S.ev[0], S.ev[1]);
        st.device_ms = ms;
        *out_len = want;
        if (stats) *stats = st;
        return 0;
    };
    if (R == 0) return finish();
    const uint64_t keep = b->continues ? b->run_len[0] : 0;
    S.resident = false;   // until this call ends well
    int rc;
    if ((rc = grow_depth(S, S.cur, run_off[R], keep, s))) return rc;
    double* D = S.depth[S.cur];
    if (run_off[R] > keep) RB_CUDA(cudaMemsetAsync(D + keep, 0, (run_off[R] - keep) * 8, s));

    // per-run and per-record arrays
    if (R + 1 > S.sz_run) {
        const size_t cap = grown(R + 1);
        S.sz_run = 0;   // until every array of the group is reallocated
        if ((rc = realloc_n(&S.run_len, cap)) || (rc = realloc_n(&S.run_off, cap)) || (rc = realloc_n(&S.run_tile, cap))) return rc;
        S.sz_run = cap;
    }
    if (n + 1 > S.sz_rec) {   // every per-record array holds sz_rec entries
        const size_t cap = grown(n + 1);
        S.sz_rec = 0;
        if ((rc = realloc_n(&S.rec_off, cap)) || (rc = realloc_n(&S.rec_run, cap)) || (rc = realloc_n(&S.blk_off, cap)) ||
            (rc = realloc_n(&S.ent_off, cap)) || (rc = realloc_n(&S.w, cap)))
            return rc;
        S.sz_rec = cap;
    }
    if (b->n_bytes > S.sz_data) {
        S.sz_data = 0;
        if ((rc = realloc_n(&S.data, grown(b->n_bytes)))) return rc;
        S.sz_data = grown(b->n_bytes);
    }
    RB_CUDA(cudaMemcpyAsync(S.run_len, b->run_len, (size_t)R * 4, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.run_off, run_off.data(), (size_t)(R + 1) * 8, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.run_tile, run_tile.data(), (size_t)(R + 1) * 8, cudaMemcpyHostToDevice, s));
    if (n) {
        RB_CUDA(cudaMemcpyAsync(S.data, b->data, b->n_bytes, cudaMemcpyHostToDevice, s));
        RB_CUDA(cudaMemcpyAsync(S.rec_off, b->rec_off, (size_t)n * 8, cudaMemcpyHostToDevice, s));
        RB_CUDA(cudaMemcpyAsync(S.rec_run, b->rec_run, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    }
    RB_CUDA(cudaMemsetAsync(S.err, 0xff, sizeof(unsigned long long), s));
    Batch B{S.data, S.rec_off, S.rec_run, S.run_len, S.run_tile, n, b->no_fractional_weight != 0};
    const unsigned grid = (n + kThreads - 1) / kThreads;
    uint64_t tot[2] = {0, 0};
    if (n) {
        wig_parse_kernel<<<grid, kThreads, 0, s>>>(B, S.blk_off, S.ent_off, S.w, S.err);
        RB_CUDA(cudaGetLastError());
        size_t tb = 0;
        RB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, S.blk_off, S.blk_off, n + 1, s));
        if (tb > S.sz_temp) {
            S.sz_temp = 0;
            if ((rc = realloc_n((uint8_t**)&S.temp, grown(tb)))) return rc;
            S.sz_temp = grown(tb);
        }
        // the parse pass does not write entry n: the totals land there after the scans
        RB_CUDA(cudaMemsetAsync(S.blk_off + n, 0, 8, s));
        RB_CUDA(cudaMemsetAsync(S.ent_off + n, 0, 8, s));
        RB_CUDA(cub::DeviceScan::ExclusiveSum(S.temp, tb, S.blk_off, S.blk_off, n + 1, s));
        RB_CUDA(cub::DeviceScan::ExclusiveSum(S.temp, tb, S.ent_off, S.ent_off, n + 1, s));
        RB_CUDA(cudaMemcpyAsync(&tot[0], S.blk_off + n, 8, cudaMemcpyDeviceToHost, s));
        RB_CUDA(cudaMemcpyAsync(&tot[1], S.ent_off + n, 8, cudaMemcpyDeviceToHost, s));
        unsigned long long err = 0;
        RB_CUDA(cudaMemcpyAsync(&err, S.err, sizeof err, cudaMemcpyDeviceToHost, s));
        RB_CUDA(cudaStreamSynchronize(s));
        ctx->launches += 3;
        if (err != ~0ull) {
            st.bad_record = (int64_t)(err >> 8);
            st.bad_code = (int32_t)(err & 255);
            if (stats) *stats = st;
            set_error(std::string("wig_depth: ") + bad_text((unsigned)(err & 255)));
            return RSEM_B200_ERR_ARG;
        }
    }
    st.blocks = tot[0];
    st.entries = tot[1];
    if (tot[1]) {
        RB_ARG(tot[1] < 0x7fffffffull, "wig_depth: more than 2^31 - 1 (tile, block) entries in one batch; use smaller batches");
        const int n_ent = (int)tot[1];
        if (tot[1] > S.sz_ent) {   // every per-entry array holds sz_ent entries
            const size_t cap = grown(tot[1]);
            S.sz_ent = 0;
            if ((rc = realloc_n(&S.blk, cap)) || (rc = realloc_n(&S.key[0], cap)) || (rc = realloc_n(&S.key[1], cap)) ||
                (rc = realloc_n(&S.val[0], cap)) || (rc = realloc_n(&S.val[1], cap)))
                return rc;
            S.sz_ent = cap;
        }
        wig_emit_kernel<<<grid, kThreads, 0, s>>>(B, S.blk_off, S.ent_off, S.w, S.blk, S.key[0], S.val[0]);
        RB_CUDA(cudaGetLastError());
        int end_bit = 1;
        while (end_bit < 32 && (run_tile[R] >> end_bit)) ++end_bit;
        size_t tb = 0;
        RB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, S.key[0], S.key[1], S.val[0], S.val[1], n_ent, 0, end_bit, s));
        if (tb > S.sz_temp) {
            S.sz_temp = 0;
            if ((rc = realloc_n((uint8_t**)&S.temp, grown(tb)))) return rc;
            S.sz_temp = grown(tb);
        }
        RB_CUDA(cub::DeviceRadixSort::SortPairs(S.temp, tb, S.key[0], S.key[1], S.val[0], S.val[1], n_ent, 0, end_bit, s));
        wig_accumulate_kernel<<<(unsigned)run_tile[R], kTile, 0, s>>>(S.key[1], S.val[1], tot[1], S.blk, S.run_len, S.run_off,
                                                                     S.run_tile, R, D);
        RB_CUDA(cudaGetLastError());
        ctx->launches += 3;
    }
    if (run_off[done_runs]) RB_CUDA(cudaMemcpyAsync(out + at, D, run_off[done_runs] * 8, cudaMemcpyDeviceToHost, s));
    if (b->keep_last) {
        const uint64_t L = b->run_len[R - 1];
        if (run_off[R - 1]) {   // the kept run moves to offset 0 of the other buffer
            const int o = 1 - S.cur;
            if ((rc = grow_depth(S, o, L, 0, s))) return rc;
            if (L) RB_CUDA(cudaMemcpyAsync(S.depth[o], D + run_off[R - 1], L * 8, cudaMemcpyDeviceToDevice, s));
            S.cur = o;
        }
        S.resident = true;
        S.resident_len = L;
    }
    return finish();
}

}  // namespace rsem_b200
