// PTX helpers for the E-step kernels (em_kernels.cu, class_kernels.cu): shared-memory stages filled by 1-D bulk
// asynchronous copies (TMA) whose completion is counted in bytes on an mbarrier, and the fp64 reduction on the count
// vector.
#pragma once

namespace rsem_b200 {

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
// L2 eviction priority for bytes that are read once (a stream much larger than L2): their lines go first, so that
// they do not push out the few lines every CTA reads and adds to over and over
__device__ __forceinline__ unsigned long long l2_evict_first() {
    unsigned long long p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// bulk_load with an L2 eviction priority for the lines it reads
__device__ __forceinline__ void bulk_load_hint(void* dst, const void* src, unsigned bytes, unsigned long long* bar,
                                               unsigned long long policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void red_add_f64(double* addr, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

// bulk copies move multiples of 16 B
__device__ __forceinline__ unsigned round16(unsigned bytes) { return (bytes + 15u) & ~15u; }

}  // namespace rsem_b200
