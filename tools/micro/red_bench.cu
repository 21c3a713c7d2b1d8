// Micro-benchmark: throughput of red.global.add.f64 / __ldg gathers on a 1.6 MB table for the lane -> entry mappings
// the E-step kernel can use.  Rows are runs of `deg` consecutive table entries at random starts (like the hits of a read).
//   mapping 0: natural   entry = 32 * i + lane            (i = 0..3)
//   mapping 1: pairs     entry = 64 * (i / 2) + 2 * lane + (i & 1)
//   mapping 2: blocked4  entry = 4 * lane + i
//   mapping 3: random    every lane its own random address (no locality at all)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o red_bench red_bench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

__device__ __forceinline__ void red_add_f64(double* addr, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

template <int MAP, bool RED>
__global__ void __launch_bounds__(512, 2) bench_kernel(double* table, const unsigned* start, unsigned n_chunks, int deg,
                                                        double* sink) {
    const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const unsigned n_warps = (gridDim.x * blockDim.x) >> 5;
    double acc = 0.0;
    for (unsigned c = warp; c < n_chunks; c += n_warps) {
        // chunk c = 128 entries = rows c * 8 .. (8 start slots reserved per chunk)
        const unsigned* st = start + (size_t)c * 8;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            unsigned e;
            if (MAP == 0) e = 32 * i + lane;
            else if (MAP == 1) e = 64 * (i >> 1) + 2 * lane + (i & 1);
            else e = 4 * lane + i;
            unsigned addr;
            if (MAP == 3) {
                addr = (st[i] * 2654435761u + lane * 40503u * (c + 1)) % 200000u;
            } else {
                const unsigned r = e / deg, col = e - r * deg;
                addr = __ldg(st + r) + col;
            }
            if (RED) red_add_f64(table + addr, 1.0);
            else acc += __ldg(table + addr);
        }
    }
    if (!RED && acc == 123.456) *sink = acc;
}

template <int MAP, bool RED>
float run(double* table, const unsigned* start, unsigned n_chunks, int deg, double* sink) {
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    bench_kernel<MAP, RED><<<296, 512>>>(table, start, n_chunks, deg, sink);
    cudaEventRecord(a);
    for (int it = 0; it < 3; ++it) bench_kernel<MAP, RED><<<296, 512>>>(table, start, n_chunks, deg, sink);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    return ms / 3;
}

int main(int argc, char** argv) {
    const int deg = argc > 1 ? atoi(argv[1]) : 21;
    const unsigned M = 200000, n_chunks = 2000000;  // 256 M entries per launch
    std::vector<unsigned> h((size_t)n_chunks * 8);
    unsigned long long s = 88172645463325252ull;
    for (auto& x : h) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        x = (unsigned)(s % (M - 64));
    }
    unsigned* start;
    double *table, *sink;
    cudaMalloc(&start, h.size() * 4);
    cudaMemcpy(start, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    cudaMalloc(&table, (M + 64) * 8);
    cudaMemset(table, 0, (M + 64) * 8);
    cudaMalloc(&sink, 8);
    const double n = (double)n_chunks * 128;
    printf("deg %d, %.0f M entries per launch\n", deg, n / 1e6);
    float t;
    t = run<0, true>(table, start, n_chunks, deg, sink);  printf("RED natural   %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<1, true>(table, start, n_chunks, deg, sink);  printf("RED pairs     %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<2, true>(table, start, n_chunks, deg, sink);  printf("RED blocked4  %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<3, true>(table, start, n_chunks, deg, sink);  printf("RED random    %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<0, false>(table, start, n_chunks, deg, sink); printf("LDG natural   %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<1, false>(table, start, n_chunks, deg, sink); printf("LDG pairs     %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<2, false>(table, start, n_chunks, deg, sink); printf("LDG blocked4  %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    t = run<3, false>(table, start, n_chunks, deg, sink); printf("LDG random    %.3f ms  %.1f G/s\n", t, n / t / 1e6);
    cudaError_t e = cudaDeviceSynchronize();
    printf("status %s\n", cudaGetErrorString(e));
    return 0;
}
