// ptx_helpers.cuh -- inline-PTX wrappers shared by the kernels (included by kernels.cu inside smr::dev): mbarrier / TMA,
// volatile shared-memory loads of TMA stages, and FP32 pair helpers.
#pragma once

namespace tma {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void *tmap, int x, int y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(tmap), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// loads from the TMA stage: volatile, the compiler does not see the asynchronous writer
__device__ __forceinline__ void lds64v(uint32_t a, uint32_t &x, uint32_t &y) {
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(x), "=r"(y) : "r"(a) : "memory");
}
__device__ __forceinline__ uint32_t lds32v(uint32_t a) {
    uint32_t x;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(a) : "memory");
    return x;
}
__device__ __forceinline__ uint32_t lds16v(uint32_t a) {
    uint32_t x;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(x) : "r"(a) : "memory");
    return x;
}
__device__ __forceinline__ uint32_t lds8v(uint32_t a) {
    uint32_t x;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(x) : "r"(a) : "memory");
    return x;
}
// read-only table in shared memory, 32-bit address arithmetic (the table never changes after set-up)
__device__ __forceinline__ float lds_tab(uint32_t a) {
    float x;
    asm("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(a));
    return x;
}

// ---- FP32 pairs, IEEE round-to-nearest per component ------------------------------------------------------------
// sm_90 has no packed FP32 arithmetic: a pair is two scalar FFMA / FMUL / FADD.  The _rn intrinsics are never contracted,
// so every component is rounded exactly where the expression says, as in the oracle.
__device__ __forceinline__ unsigned long long pk(float2 a) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a.x), "f"(a.y));
    return r;
}
__device__ __forceinline__ float2 upk(unsigned long long r) {
    float2 a;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a.x), "=f"(a.y) : "l"(r));
    return a;
}
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 splat(float a) { return make_float2(a, a); }
// a pair held as one 64-bit register pair (the layout of the weight pairs and of the shared-memory loads below)
__device__ __forceinline__ unsigned long long fma2q(unsigned long long a, unsigned long long b, unsigned long long c) {
    return pk(fma2(upk(a), upk(b), upk(c)));
}
__device__ __forceinline__ void lds128q(uint32_t addr, unsigned long long &lo, unsigned long long &hi) {
    asm volatile("ld.shared.v2.b64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(addr));
}
// a + c for an `a` that is the result of mul2(): the product is rounded on its own, then the sum
__device__ __forceinline__ float2 add2_after_mul(float2 a, float2 c) { return add2(a, c); }


}  // namespace tma
