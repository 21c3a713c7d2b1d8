// K8: Phase II of rsem-calculate-credibility-intervals (calcCI.cpp:218-385) on the device.
//
// The host pushes sample rows (M TPMs + l_bar per sample, sample-major) as its threads produce them.  They are kept in
// one sample-major matrix S: on the device when it fits next to the working set of a block (the default), otherwise in
// pinned host memory.  ci_end then walks gene-aligned blocks of transcripts:
//   transpose   the block's columns of S into transcript-major rows of nSamples (from host memory: a strided copy of the
//               columns first)
//   sums        FPKM rows 1e3 / l_bar * tpm (double quotient and product, stored as float, calcCI.cpp:338) and the gene
//               sums of multi-transcript genes as float sums in transcript order (calcCI.cpp:343-344)
//   isoforms    allele-specific references: the running isoform sums of calcCI.cpp:307-373, kept in
//               transcript order across blocks by ci_end
//   sort        every row, one segmented CUB sort
//   interval    calcCI() per row: the shortest interval holding the confidence mass with ties kept together, Tukey's
//               hinges and the coefficient of quartile variation, in the reference's float / double mix
// Results go back as (lb, ub, cqv) per row.  Every float operation uses explicit round-to-nearest intrinsics, so no
// contraction into an FMA changes a bit.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {

namespace {

constexpr int kTile = 32;
constexpr size_t kStageBytes = 32u << 20;  // pinned staging for one push copy

// dst[c][k] = src[k * pitch + col0 + c] for c < w, k < n
__global__ void ci_transpose_kernel(const float* __restrict__ src, int64_t pitch, int64_t col0, int w, int64_t n,
                                    float* __restrict__ dst) {
    __shared__ float tile[kTile][kTile + 1];
    const int64_t k0 = (int64_t)blockIdx.x * kTile;
    for (int64_t c0 = (int64_t)blockIdx.y * kTile; c0 < w; c0 += (int64_t)gridDim.y * kTile) {  // gridDim.y <= 65535
        for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
            const int64_t k = k0 + i, c = c0 + threadIdx.x;
            if (k < n && c < w) tile[i][threadIdx.x] = src[k * pitch + col0 + c];
        }
        __syncthreads();
        for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
            const int64_t c = c0 + i, k = k0 + threadIdx.x;
            if (k < n && c < w) dst[c * n + k] = tile[threadIdx.x][i];
        }
        __syncthreads();
    }
}

// F = 1e3 / l_bar * T: double quotient, double product, rounded to float (calcCI.cpp:338)
__global__ void ci_fpkm_kernel(const float* __restrict__ T, const float* __restrict__ lbar, float* __restrict__ F,
                               int64_t total, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = i % n;
        F[i] = __double2float_rn(__dmul_rn(__ddiv_rn(1e3, (double)lbar[k]), (double)T[i]));
    }
}

// gene g < gm of the block: GT[g] = sum of the rows T[gb[g] .. ge[g]), GF likewise from F, float adds in transcript
// order.  Genes stride over grid.y (at most 65535 CTAs on that axis; a block may hold more multi-transcript genes).
__global__ void ci_gene_sums_kernel(const float* __restrict__ T, const float* __restrict__ F, const int* __restrict__ gb,
                                    const int* __restrict__ ge, int gm, int64_t n, float* __restrict__ GT,
                                    float* __restrict__ GF) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    for (int g = blockIdx.y; g < gm; g += gridDim.y) {
        float st = 0.0f, sf = 0.0f;
        for (int j = gb[g]; j < ge[g]; ++j) {
            st = __fadd_rn(st, T[(int64_t)j * n + k]);
            sf = __fadd_rn(sf, F[(int64_t)j * n + k]);
        }
        GT[(int64_t)g * n + k] = st;
        GF[(int64_t)g * n + k] = sf;
    }
}

__global__ void ci_add_kernel(float* __restrict__ at, float* __restrict__ af, const float* __restrict__ t,
                              const float* __restrict__ f, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        at[k] = __fadd_rn(at[k], t[k]);
        af[k] = __fadd_rn(af[k], f[k]);
    }
}

// calcCI() (calcCI.cpp:218-284) on a sorted row
__device__ void ci_row(const float* s, int n, int threshold, float* out) {
    int p = 0, q = n - 1, newp, newq = n - 1;
    do {
        q = newq;
        while (newq > 0 && s[newq - 1] == s[newq]) newq--;
        newq--;
    } while (newq >= 0 && n - (newq + 1) <= threshold);
    int nOutside = n - (q + 1);
    float lb = -1e30f, ub = 1e30f;
    do {
        if (__fsub_rn(s[q], s[p]) < __fsub_rn(ub, lb)) {
            lb = s[p];
            ub = s[q];
        }
        newp = p;
        while (newp < n - 1 && s[newp] == s[newp + 1]) newp++;
        newp++;
        if (newp <= threshold) {
            nOutside += newp - p;
            p = newp;
            while (nOutside > threshold && q < n - 1) {
                newq = q + 1;
                while (newq < n - 1 && s[newq] == s[newq + 1]) newq++;
                nOutside -= newq - q;
                q = newq;
            }
        } else {
            p = newp;
        }
    } while (p <= threshold);

    // Tukey's hinges; (a + b) / 2.0 is a float sum halved (exact)
    const int quotient = n / 4, residue = n % 4;
    float Q1, Q3;
    if (residue == 0) {
        Q1 = __fmul_rn(__fadd_rn(s[quotient - 1], s[quotient]), 0.5f);
        Q3 = __fmul_rn(__fadd_rn(s[3 * quotient - 1], s[3 * quotient]), 0.5f);
    } else if (residue == 3) {
        Q1 = __fmul_rn(__fadd_rn(s[quotient], s[quotient + 1]), 0.5f);
        Q3 = __fmul_rn(__fadd_rn(s[quotient * 3 + 1], s[quotient * 3 + 2]), 0.5f);
    } else {
        Q1 = s[quotient];
        Q3 = s[3 * quotient];
    }
    const float d = __fsub_rn(Q3, Q1);
    out[0] = lb;
    out[1] = ub;
    out[2] = d > 0.0f ? __fdiv_rn(d, __fadd_rn(Q3, Q1)) : 0.0f;
}

__global__ void ci_interval_kernel(const float* __restrict__ X, int rows, int64_t n, int threshold, float* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) ci_row(X + (int64_t)r * n, (int)n, threshold, out + 3 * (int64_t)r);
}

__global__ void ci_offsets_kernel(int64_t* off, int rows, int64_t n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= rows) off[r] = (int64_t)r * n;
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

// grid-stride launches of 256 threads: 16 CTAs per SM at most
int blocks_for(const rsem_b200_ctx* ctx, int64_t total) {
    return (int)std::max<int64_t>(1, std::min<int64_t>((total + 255) / 256, (int64_t)ctx->sm_count * 16));
}

}  // namespace

struct CiState {
    int M = 0, m = 0, threshold = 0;
    int64_t n = 0;
    std::vector<int> gene_start, iso_start, part_gene;  // 1-based transcript ids as GroupInfo holds them
    bool resident = true;
    float* S = nullptr;       // n x M, device (resident) or pinned host
    std::vector<float> lbar_h;
    float* lbar = nullptr;    // n, device
    char* stage[2] = {nullptr, nullptr};
    cudaEvent_t stage_ev[2] = {nullptr, nullptr};
    int next_stage = 0;
    uint64_t budget = 0;
    std::mutex mu;
    rsem_b200_ci_stats stats{};
};

void ci_free(rsem_b200_ctx* ctx) {
    CiState* s = ctx->ci;
    if (!s) return;
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamSynchronize(ctx->stream);
    if (s->resident) cudaFree(s->S); else cudaFreeHost(s->S);
    cudaFree(s->lbar);
    for (int b = 0; b < 2; ++b) {
        if (s->stage[b]) cudaFreeHost(s->stage[b]);
        if (s->stage_ev[b]) cudaEventDestroy(s->stage_ev[b]);
    }
    delete s;
    ctx->ci = nullptr;
}

namespace {

// rows of gene g in a block: tpm + fpkm per transcript, + a gene tpm / fpkm pair when it has more than one transcript
int64_t gene_rows(const CiState* s, int g) {
    const int w = s->gene_start[g + 1] - s->gene_start[g];
    return 2 * (int64_t)w + (w > 1 ? 2 : 0);
}

// bytes a block of `rows` rows needs besides S: the rows, CUB's alternate buffer, column staging for a host-resident S
int64_t block_bytes_per_row(const CiState* s) { return s->n * 4 * (s->resident ? 2 : 3); }

}  // namespace

int ci_begin(rsem_b200_ctx* ctx, const rsem_b200_ci_params* p) {
    ci_free(ctx);
    CiState* s = new CiState();
    ctx->ci = s;
    s->M = p->M;
    s->m = p->n_genes;
    s->n = p->n_samples;
    s->threshold = p->threshold;
    s->gene_start.assign(p->gene_start, p->gene_start + p->n_genes + 1);
    if (p->n_isoforms > 0) s->iso_start.assign(p->isoform_start, p->isoform_start + p->n_isoforms + 1);
    s->part_gene.assign(p->part_gene_start, p->part_gene_start + p->n_parts + 1);
    s->lbar_h.assign(s->n, 0.0f);
    size_t free_b = 0, total_b = 0;
    RB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t reserve = 512ull << 20;
    s->budget = p->device_budget ? p->device_budget : (free_b > reserve ? free_b - reserve : 0);
    int64_t max_rows = 0;
    for (int g = 0; g < s->m; ++g) max_rows = std::max(max_rows, gene_rows(s, g));
    const int64_t s_bytes = s->n * (int64_t)s->M * 4;
    const int64_t fixed = s->n * 4 * (1 + 4) + (1 << 20);  // l_bars, isoform sums and their sort buffers, small arrays
    s->resident = (int64_t)s->budget >= s_bytes + fixed + max_rows * s->n * 8;
    if (!s->resident && (int64_t)s->budget < fixed + max_rows * s->n * 12) {
        set_error("ci_begin: the device budget cannot hold the rows of the largest gene");
        ci_free(ctx);
        return RSEM_B200_ERR_ARG;
    }
    if (s->resident) {
        RB_CUDA(cudaMalloc(&s->S, (size_t)s_bytes));
        for (int b = 0; b < 2; ++b) {
            RB_CUDA(cudaHostAlloc(&s->stage[b], kStageBytes, cudaHostAllocDefault));
            RB_CUDA(cudaEventCreateWithFlags(&s->stage_ev[b], cudaEventDisableTiming));
        }
    } else {
        RB_CUDA(cudaHostAlloc(&s->S, (size_t)s_bytes, cudaHostAllocDefault));
    }
    RB_CUDA(cudaMalloc(&s->lbar, (size_t)s->n * 4));
    s->stats.resident = s->resident;
    return 0;
}

int ci_push(rsem_b200_ctx* ctx, const float* rows, const float* l_bars, int64_t first, int64_t count) {
    CiState* s = ctx->ci;
    RB_ARG(s, "ci_begin must be called first");
    RB_ARG(first >= 0 && count >= 0 && first + count <= s->n, "samples out of range");
    std::lock_guard<std::mutex> lock(s->mu);
    memcpy(&s->lbar_h[first], l_bars, (size_t)count * 4);
    const size_t row_bytes = (size_t)s->M * 4;
    if (!s->resident) {
        memcpy(s->S + first * s->M, rows, (size_t)count * row_bytes);
        return 0;
    }
    // pageable rows -> one of two pinned stages -> device, on the copy stream; the caller may reuse `rows` on return
    const int64_t per = std::max<int64_t>(1, (int64_t)(kStageBytes / row_bytes));
    for (int64_t done = 0; done < count;) {
        const int64_t k = std::min(per, count - done);
        const int b = s->next_stage;
        s->next_stage ^= 1;
        RB_CUDA(cudaEventSynchronize(s->stage_ev[b]));
        char* src = (char*)rows + done * row_bytes;
        float* dst = s->S + (first + done) * s->M;
        if ((size_t)k * row_bytes <= kStageBytes) {
            memcpy(s->stage[b], src, (size_t)k * row_bytes);
            RB_CUDA(cudaMemcpyAsync(dst, s->stage[b], (size_t)k * row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        } else {  // a single row larger than a stage
            RB_CUDA(cudaMemcpyAsync(dst, src, row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
            RB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
        }
        RB_CUDA(cudaEventRecord(s->stage_ev[b], ctx->copy_stream));
        done += k;
    }
    return 0;
}

namespace {

// Device buffers of the blocked walk.
struct Work {
    float* X = nullptr;    // rows x n
    float* Y = nullptr;    // CUB's alternate buffer
    float* col = nullptr;  // n x w staging for a host-resident S
    int64_t* off = nullptr;
    int* gb = nullptr;
    int* ge = nullptr;
    float* res = nullptr;  // rows x 3
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    float* iso[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // running isoform tpm / fpkm sums and alternates
    float* iso_res = nullptr;  // 6
};

// sort the two running isoform sums in place and compute their intervals into out[6]
int ci_finish_isoform(rsem_b200_ctx* ctx, Work& wk, float* out_h) {
    CiState* s = ctx->ci;
    cudaStream_t st = ctx->stream;
    for (int a = 0; a < 2; ++a) {
        cub::DoubleBuffer<float> keys(wk.iso[a][0], wk.iso[a][1]);
        size_t need = wk.tmp_bytes;
        RB_CUDA(cub::DeviceRadixSort::SortKeys(wk.tmp, need, keys, (int)s->n, 0, 32, st));
        if (keys.Current() != wk.iso[a][0]) std::swap(wk.iso[a][0], wk.iso[a][1]);
        ci_interval_kernel<<<1, 1, 0, st>>>(wk.iso[a][0], 1, s->n, s->threshold, wk.iso_res + 3 * a);
        RB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    RB_CUDA(cudaMemcpyAsync(out_h, wk.iso_res, 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace

int ci_end(rsem_b200_ctx* ctx, float* tr_out, float* gene_out, float* iso_out, rsem_b200_ci_stats* stats) {
    CiState* s = ctx->ci;
    RB_ARG(s, "ci_begin must be called first");
    RB_ARG(s->iso_start.empty() || iso_out, "isoforms is NULL for an allele-specific reference");
    cudaStream_t st = ctx->stream;
    const int64_t n = s->n;
    const int M = s->M;
    RB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    RB_CUDA(cudaMemcpyAsync(s->lbar, s->lbar_h.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));

    // block capacity from what the budget leaves next to S
    const int64_t s_bytes = s->resident ? n * (int64_t)M * 4 : 0;
    const int64_t fixed = n * 4 * (1 + 4) + (1 << 20);
    int64_t rows_cap = ((int64_t)s->budget - s_bytes - fixed) / block_bytes_per_row(s);
    rows_cap = std::min<int64_t>(rows_cap, (int64_t)INT32_MAX / n);
    int64_t max_rows = 0, all_rows = 0;
    for (int g = 0; g < s->m; ++g) {
        max_rows = std::max(max_rows, gene_rows(s, g));
        all_rows += gene_rows(s, g);
    }
    rows_cap = std::min(rows_cap, all_rows);
    RB_ARG(rows_cap >= max_rows, "ci_end: the device budget cannot hold the rows of the largest gene");

    Work wk;
    std::vector<void*> owned;
    auto alloc = [&](auto** p, size_t bytes) {
        cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(bytes, 16));
        if (e == cudaSuccess) owned.push_back((void*)*p);
        return e;
    };
    auto release = [&]() { for (void* q : owned) cudaFree(q); };
    cudaEvent_t ev[6];
    for (auto& e : ev) cudaEventCreate(&e);
    auto cleanup = [&]() {
        cudaStreamSynchronize(st);
        release();
        for (auto& e : ev) cudaEventDestroy(e);
    };
#define CI_CUDA(call)                                                                 \
    do {                                                                              \
        cudaError_t _e = (call);                                                      \
        if (_e != cudaSuccess) {                                                      \
            cleanup();                                                                \
            return ::rsem_b200::cuda_fail(_e, #call, __FILE__, __LINE__);             \
        }                                                                             \
    } while (0)
    const size_t row_b = (size_t)n * 4;
    CI_CUDA(alloc(&wk.X, rows_cap * row_b));
    CI_CUDA(alloc(&wk.Y, rows_cap * row_b));
    if (!s->resident) CI_CUDA(alloc(&wk.col, rows_cap * row_b));
    CI_CUDA(alloc(&wk.off, (rows_cap + 1) * sizeof(int64_t)));
    CI_CUDA(alloc(&wk.gb, rows_cap * sizeof(int)));
    CI_CUDA(alloc(&wk.ge, rows_cap * sizeof(int)));
    CI_CUDA(alloc(&wk.res, rows_cap * 3 * sizeof(float)));
    CI_CUDA(alloc(&wk.iso_res, 6 * sizeof(float)));
    const bool alleles = !s->iso_start.empty();
    if (alleles)
        for (auto& a : wk.iso)
            for (auto& b : a) CI_CUDA(alloc(&b, row_b));
    {
        size_t seg = 0, one = 0;
        cub::DoubleBuffer<float> keys(wk.X, wk.Y);
        CI_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, seg, keys, (int)(rows_cap * n), (int)rows_cap, wk.off,
                                                   wk.off + 1, st));
        CI_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, one, keys, (int)n, 0, 32, st));
        wk.tmp_bytes = std::max(seg, one);
        CI_CUDA(alloc(&wk.tmp, wk.tmp_bytes));
    }

    // isoform chain state (calcCI.cpp:307-373): allele id -> isoform id, and every isoform result in the order the
    // reference assigns it (an isoform may be assigned twice when it straddles two Phase II thread ranges)
    std::vector<int> iso_of;
    if (alleles) {
        iso_of.assign(M + 1, -1);
        for (int i = 0; i + 1 < (int)s->iso_start.size(); ++i)
            for (int j = s->iso_start[i]; j < s->iso_start[i + 1]; ++j) iso_of[j] = i;
    }
    struct IsoEvent { int tid, copy_from; float v[6]; };
    std::vector<IsoEvent> iso_events;
    int curtid = -1, curaid = -1, part = 0;
    auto finish_iso = [&](int end_j) -> int {  // the isoform curtid ends before transcript end_j
        IsoEvent e{curtid, -1, {0, 0, 0, 0, 0, 0}};
        if (end_j - curaid > 1) {
            if (int rc = ci_finish_isoform(ctx, wk, e.v)) return rc;
        } else {
            e.copy_from = curaid;
        }
        iso_events.push_back(e);
        return 0;
    };

    std::vector<float> res_h;
    std::vector<int> gb_h, ge_h, gene_row;
    for (int g0 = 0; g0 < s->m;) {
        int g1 = g0;
        int64_t rows = 0;
        while (g1 < s->m && rows + gene_rows(s, g1) <= rows_cap) rows += gene_rows(s, g1++);
        const int b = s->gene_start[g0], e = s->gene_start[g1];  // transcripts [b, e), 1-based
        const int w = e - b;
        gb_h.clear(); ge_h.clear(); gene_row.clear();
        for (int g = g0; g < g1; ++g)
            if (s->gene_start[g + 1] - s->gene_start[g] > 1) {
                gb_h.push_back(s->gene_start[g] - b);
                ge_h.push_back(s->gene_start[g + 1] - b);
                gene_row.push_back(g);
            }
        const int gm = (int)gb_h.size();
        float* T = wk.X;
        float* F = wk.X + (int64_t)w * n;
        float* GT = wk.X + (int64_t)2 * w * n;
        float* GF = GT + (int64_t)gm * n;

        CI_CUDA(cudaEventRecord(ev[0], st));
        if (s->resident) {
            dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)std::min<int64_t>((w + kTile - 1) / kTile, 65535));
            ci_transpose_kernel<<<grid, dim3(kTile, 8), 0, st>>>(s->S, M, b - 1, w, n, T);
        } else {  // gather the block's columns from pinned host memory, then transpose on the device
            CI_CUDA(cudaMemcpy2DAsync(wk.col, (size_t)w * 4, s->S + (b - 1), (size_t)M * 4, (size_t)w * 4, (size_t)n,
                                      cudaMemcpyHostToDevice, st));
            dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)std::min<int64_t>((w + kTile - 1) / kTile, 65535));
            ci_transpose_kernel<<<grid, dim3(kTile, 8), 0, st>>>(wk.col, w, 0, w, n, T);
        }
        CI_CUDA(cudaGetLastError());
        ctx->launches++;
        CI_CUDA(cudaEventRecord(ev[1], st));
        ci_fpkm_kernel<<<blocks_for(ctx, (int64_t)w * n), 256, 0, st>>>(T, s->lbar, F, (int64_t)w * n, n);
        CI_CUDA(cudaGetLastError());
        ctx->launches++;
        if (gm) {
            CI_CUDA(cudaMemcpyAsync(wk.gb, gb_h.data(), gm * sizeof(int), cudaMemcpyHostToDevice, st));
            CI_CUDA(cudaMemcpyAsync(wk.ge, ge_h.data(), gm * sizeof(int), cudaMemcpyHostToDevice, st));
            dim3 grid((unsigned)((n + 255) / 256), (unsigned)std::min(gm, 65535));
            ci_gene_sums_kernel<<<grid, 256, 0, st>>>(T, F, wk.gb, wk.ge, gm, n, GT, GF);
            CI_CUDA(cudaGetLastError());
            ctx->launches++;
        }
        CI_CUDA(cudaEventRecord(ev[2], st));
        if (alleles) {  // calcCI.cpp:313-345, transcript by transcript, before the rows are sorted
            for (int g = g0; g < g1; ++g) {
                while (g == s->part_gene[part + 1]) {  // a new Phase II thread range starts from zeroed sums
                    if (curtid >= 0)
                        if (int rc = finish_iso(s->gene_start[g])) { cleanup(); return rc; }
                    curtid = curaid = -1;
                    ++part;
                }
                if (curtid < 0)
                    for (auto& a : wk.iso) CI_CUDA(cudaMemsetAsync(a[0], 0, row_b, st));
                for (int j = s->gene_start[g]; j < s->gene_start[g + 1]; ++j) {
                    const int tid = iso_of[j];
                    if (curtid != tid) {
                        if (curtid >= 0)
                            if (int rc = finish_iso(j)) { cleanup(); return rc; }
                        curtid = tid;
                        curaid = j;
                    }
                    ci_add_kernel<<<blocks_for(ctx, n), 256, 0, st>>>(wk.iso[0][0], wk.iso[1][0], T + (int64_t)(j - b) * n,
                                                                 F + (int64_t)(j - b) * n, n);
                    CI_CUDA(cudaGetLastError());
                    ctx->launches++;
                }
            }
        }
        CI_CUDA(cudaEventRecord(ev[3], st));
        const int nrows = 2 * w + 2 * gm;
        ci_offsets_kernel<<<(nrows + 256) / 256, 256, 0, st>>>(wk.off, nrows, n);
        CI_CUDA(cudaGetLastError());
        cub::DoubleBuffer<float> keys(wk.X, wk.Y);
        size_t need = wk.tmp_bytes;
        CI_CUDA(cub::DeviceSegmentedSort::SortKeys(wk.tmp, need, keys, (int)(nrows * n), nrows, wk.off, wk.off + 1, st));
        ctx->launches += 2;
        CI_CUDA(cudaEventRecord(ev[4], st));
        ci_interval_kernel<<<(nrows + 127) / 128, 128, 0, st>>>(keys.Current(), nrows, n, s->threshold, wk.res);
        CI_CUDA(cudaGetLastError());
        ctx->launches++;
        CI_CUDA(cudaEventRecord(ev[5], st));
        res_h.resize((size_t)nrows * 3);
        CI_CUDA(cudaMemcpyAsync(res_h.data(), wk.res, res_h.size() * 4, cudaMemcpyDeviceToHost, st));
        CI_CUDA(cudaStreamSynchronize(st));
        s->stats.transpose_ms += elapsed(ev[0], ev[1]);
        s->stats.sums_ms += elapsed(ev[1], ev[2]) + elapsed(ev[2], ev[3]);
        s->stats.sort_ms += elapsed(ev[3], ev[4]);
        s->stats.interval_ms += elapsed(ev[4], ev[5]);
        s->stats.blocks++;

        // transcript rows: (tpm lb ub cqv, fpkm lb ub cqv) per transcript; genes likewise
        for (int c = 0; c < w; ++c) {
            float* o = tr_out + (size_t)(b - 1 + c) * 6;
            memcpy(o, &res_h[(size_t)c * 3], 12);
            memcpy(o + 3, &res_h[(size_t)(w + c) * 3], 12);
        }
        for (int i = 0; i < gm; ++i) {
            float* o = gene_out + (size_t)gene_row[i] * 6;
            memcpy(o, &res_h[(size_t)(2 * w + i) * 3], 12);
            memcpy(o + 3, &res_h[(size_t)(2 * w + gm + i) * 3], 12);
        }
        for (int g = g0; g < g1; ++g)  // single-transcript genes take their transcript's intervals (calcCI.cpp:354-357)
            if (s->gene_start[g + 1] - s->gene_start[g] == 1)
                memcpy(gene_out + (size_t)g * 6, tr_out + (size_t)(s->gene_start[g] - 1) * 6, 24);
        g0 = g1;
    }
    if (alleles) {
        if (curtid >= 0)
            if (int rc = finish_iso(s->gene_start[s->m])) { cleanup(); return rc; }
        for (const IsoEvent& e : iso_events) {
            if (e.copy_from >= 0) memcpy(iso_out + (size_t)e.tid * 6, tr_out + (size_t)(e.copy_from - 1) * 6, 24);
            else memcpy(iso_out + (size_t)e.tid * 6, e.v, 24);
        }
    }
#undef CI_CUDA
    cleanup();
    if (stats) *stats = s->stats;
    ci_free(ctx);
    return 0;
}

}  // namespace rsem_b200
