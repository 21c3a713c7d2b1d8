// Micro-benchmark: the HBM read rate a streaming kernel can reach, and with which copy geometry.  Every variant reads the
// same >= 8 GB buffer once per launch with a trivial consume step; 20 timed launches (CUDA events) per variant.
//   a  grid-stride 16-byte ld.global.nc loads, xor-summed so that they are not eliminated
//   b  one CTA per SM: one issuing thread, 3 x 64 KB cp.async.bulk stages, 15 consumer warps that only arrive
//   c  two CTAs per SM, 3 x 32 KB stages each (otherwise as b)
//   d  per-warp rings: W warps per CTA, each warp's lane 0 keeps S bulk copies of B bytes in flight into its own slots
// Prints one JSON line.  build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o hbm_read hbm_read.cu
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <cuda_runtime.h>

#define CK(x)                                                                                     \
    do {                                                                                          \
        cudaError_t e_ = (x);                                                                     \
        if (e_ != cudaSuccess) {                                                                  \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));   \
            exit(1);                                                                              \
        }                                                                                         \
    } while (0)

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "HW_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra HW_DONE;\n"
        "bra HW_WAIT;\n"
        "HW_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint4 ld_nc(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// (a) ---------------------------------------------------------------------------------------------------------------
__global__ void ldg_kernel(const uint4* __restrict__ p, size_t n16, unsigned* sink) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned acc = 0;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 v0 = ld_nc(p + i), v1 = ld_nc(p + i + stride), v2 = ld_nc(p + i + 2 * stride), v3 = ld_nc(p + i + 3 * stride);
        acc ^= v0.x ^ v0.y ^ v0.z ^ v0.w ^ v1.x ^ v1.y ^ v1.z ^ v1.w ^ v2.x ^ v2.y ^ v2.z ^ v2.w ^ v3.x ^ v3.y ^ v3.z ^ v3.w;
    }
    for (; i < n16; i += stride) {
        const uint4 v = ld_nc(p + i);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x9e3779b9u) sink[0] = acc;
}

// (b), (c): shared ring of 3 stages per CTA, one issuing thread, W consumer warps ------------------------------------
__global__ void staged_kernel(const unsigned char* __restrict__ buf, unsigned long long n_tiles, unsigned stage_bytes, int W,
                              unsigned* sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned long long* full = reinterpret_cast<unsigned long long*>(smem + 3ull * stage_bytes);
    unsigned long long* empty = full + 3;
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < 3; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], W);
        }
        fence_barrier_init();
    }
    __syncthreads();
    unsigned acc = 0;
    if ((int)warp == W) {
        if (lane == 0) {
            unsigned it = 0;
            for (unsigned long long k = blockIdx.x; k < n_tiles; k += gridDim.x, ++it) {
                const int s = it % 3;
                if (it >= 3) {
                    mbar_wait(&empty[s], ((it / 3) - 1u) & 1u);
                    fence_proxy_async();
                }
                mbar_expect_tx(&full[s], stage_bytes);
                bulk_load(smem + (size_t)s * stage_bytes, buf + k * stage_bytes, stage_bytes, &full[s]);
            }
        }
    } else {
        unsigned it = 0;
        for (unsigned long long k = blockIdx.x; k < n_tiles; k += gridDim.x, ++it) {
            const int s = it % 3;
            mbar_wait(&full[s], (it / 3) & 1u);
            acc ^= reinterpret_cast<const unsigned*>(smem + (size_t)s * stage_bytes)[warp * 32 + lane];
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    }
    if (acc == 0x9e3779b9u) sink[0] = acc;
}

// (d): per-warp rings -----------------------------------------------------------------------------------------------
__global__ void warp_ring_kernel(const unsigned char* __restrict__ buf, unsigned long long n_chunks, unsigned B, int S,
                                 unsigned* sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    unsigned char* ring = smem + (size_t)warp * S * B;
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(smem + (size_t)W * S * B) + warp * S;
    const unsigned long long gw = (unsigned long long)blockIdx.x * W + warp, GW = (unsigned long long)gridDim.x * W;
    if (lane == 0) {
        for (int s = 0; s < S; ++s) mbar_init(&bar[s], 1);
        fence_barrier_init();
        for (int s = 0; s < S; ++s) {
            const unsigned long long k = gw + (unsigned long long)s * GW;
            if (k < n_chunks) {
                mbar_expect_tx(&bar[s], B);
                bulk_load(ring + (size_t)s * B, buf + k * B, B, &bar[s]);
            }
        }
    }
    __syncwarp();
    unsigned acc = 0;
    unsigned it = 0;
    for (unsigned long long k = gw; k < n_chunks; k += GW, ++it) {
        const int s = it % S;
        mbar_wait(&bar[s], (it / S) & 1u);
        acc ^= reinterpret_cast<const unsigned*>(ring + (size_t)s * B)[lane];
        __syncwarp();
        const unsigned long long kn = k + (unsigned long long)S * GW;
        if (lane == 0 && kn < n_chunks) {
            fence_proxy_async();
            mbar_expect_tx(&bar[s], B);
            bulk_load(ring + (size_t)s * B, buf + kn * B, B, &bar[s]);
        }
    }
    if (acc == 0x9e3779b9u) sink[0] = acc;
}

// ------------------------------------------------------------------------------------------------------------------
static const int kLaunches = 20;

template <class F>
static double time_gbs(F launch, double bytes) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    launch();  // warm-up
    launch();
    CK(cudaGetLastError());
    CK(cudaEventRecord(e0));
    for (int i = 0; i < kLaunches; ++i) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return bytes * kLaunches / (ms * 1e-3) / 1e9;
}

int main(int argc, char** argv) {
    const size_t total = (argc > 1 ? strtoull(argv[1], nullptr, 10) : 8ull) << 30;
    int dev = 0, sms = 0, smem_optin = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    unsigned char* buf = nullptr;
    unsigned* sink = nullptr;
    CK(cudaMalloc(&buf, total));
    CK(cudaMalloc(&sink, 16));
    CK(cudaMemset(buf, 1, total));
    CK(cudaDeviceSynchronize());
    std::string js = "{\"tool\": \"hbm_read\", \"gpu\": \"" + std::string(prop.name) + "\", \"sms\": " + std::to_string(sms) +
                     ", \"bytes_per_launch\": " + std::to_string(total) + ", \"launches\": " + std::to_string(kLaunches);
    char tmp[256];
    double best_a = 0, best_d = 0;
    std::string best_d_cfg;

    js += ", \"a_ldg_nc\": {";
    {
        const int cfg[][2] = {{256, 4}, {256, 8}, {512, 4}, {1024, 2}};
        bool first = true;
        for (auto& c : cfg) {
            const size_t n16 = total / 16;
            const double g = time_gbs([&] { ldg_kernel<<<sms * c[1], c[0]>>>(reinterpret_cast<const uint4*>(buf), n16, sink); },
                                      (double)n16 * 16);
            best_a = g > best_a ? g : best_a;
            snprintf(tmp, sizeof tmp, "%s\"%dx%d_per_sm\": %.1f", first ? "" : ", ", c[0], c[1], g);
            js += tmp;
            first = false;
        }
    }
    js += "}";

    auto staged = [&](unsigned stage_bytes, int ctas_per_sm, const char* key) {
        const int W = 15;
        const size_t smem = 3ull * stage_bytes + 6 * 8;
        CK(cudaFuncSetAttribute(staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const unsigned long long n_tiles = total / stage_bytes;
        const double g = time_gbs([&] { staged_kernel<<<sms * ctas_per_sm, (W + 1) * 32, smem>>>(buf, n_tiles, stage_bytes, W, sink); },
                                  (double)n_tiles * stage_bytes);
        snprintf(tmp, sizeof tmp, ", \"%s\": %.1f", key, g);
        js += tmp;
    };
    staged(64 * 1024, 1, "b_1cta_3x64KB");
    staged(32 * 1024, 2, "c_2cta_3x32KB");

    js += ", \"d_warp_rings\": {";
    {
        const int Ws[] = {8, 12, 16, 24}, Ss[] = {2, 3, 4};
        const unsigned Bs[] = {4096, 8192, 12288, 16384};
        bool first = true;
        for (int W : Ws)
            for (int S : Ss)
                for (unsigned B : Bs) {
                    const size_t smem = (size_t)W * S * B + (size_t)W * S * 8;
                    if (smem > (size_t)smem_optin) continue;
                    CK(cudaFuncSetAttribute(warp_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                    const unsigned long long n_chunks = total / B;
                    const double g = time_gbs([&] { warp_ring_kernel<<<sms, W * 32, smem>>>(buf, n_chunks, B, S, sink); },
                                              (double)n_chunks * B);
                    snprintf(tmp, sizeof tmp, "%s\"W%d_S%d_B%u\": %.1f", first ? "" : ", ", W, S, B / 1024, g);
                    js += tmp;
                    if (g > best_d) {
                        best_d = g;
                        snprintf(tmp, sizeof tmp, "W%d_S%d_B%u", W, S, B / 1024);
                        best_d_cfg = tmp;
                    }
                    first = false;
                }
    }
    js += "}";
    snprintf(tmp, sizeof tmp, ", \"best_a_gbs\": %.1f, \"best_d_gbs\": %.1f, \"best_d\": \"%s\", \"unit\": \"GB/s\"}", best_a, best_d,
             best_d_cfg.c_str());
    js += tmp;
    printf("%s\n", js.c_str());
    CK(cudaFree(buf));
    CK(cudaFree(sink));
    return 0;
}
