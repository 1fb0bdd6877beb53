// sm_90a device primitives shared by the vilbert_b200 kernels: mbarrier, TMA, programmatic dependent launch and small math
// (the warpgroup MMA wrappers are in wgmma.cuh).  Raw PTX only (no CUTLASS dependency).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>

namespace vb {

// ---------------------------------------------------------------------------------------------
// Bounded spin: a protocol bug must trap (error surfaces through cudaGetLastError on the host)
// instead of hanging the GPU.
// ---------------------------------------------------------------------------------------------
#ifndef VB_SPIN_LIMIT
#define VB_SPIN_LIMIT (1u << 26)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    // make mbarrier.init visible to the async proxy (TMA) and to the cluster
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t tx_bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(tx_bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > VB_SPIN_LIMIT) {
            printf("vb: mbarrier timeout block(%d,%d) thread %d parity %u\n", blockIdx.x, blockIdx.y, threadIdx.x,
                   parity);
            __trap();
        }
    }
}

// The same wait without the diagnostic printf, for code that waits while a wgmma group is in flight: a function call (vprintf)
// inside that window makes ptxas serialise every wgmma of the kernel (C7510).
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > VB_SPIN_LIMIT) __trap();
    }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
// 2-D tiled load global -> shared (this CTA), completes tx bytes on `bar`.  c0 = inner (contiguous) coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* desc, uint64_t* bar, int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// 2-D tiled store shared (this CTA) -> global through the TMA; completion tracked with bulk groups.
__device__ __forceinline__ void tma_store_2d(const void* desc, const void* smem_src, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit_and_wait_read() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");     // shared memory may be reused / the CTA may exit
}
// generic-proxy writes to shared memory -> visible to the async proxy (TMA) that is about to read them
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ programmatic dependent launch
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// L2 prefetch of one 128-byte line (no data returned, no register)
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ------------------------------------------------------------------ math
// erf to 1.5e-7 absolute (Abramowitz & Stegun 7.1.26): branch-free, 2 MUFU + ~10 FMA-class instructions per value.
// The libdevice erff costs several times more (two range-dependent paths, both executed by a divergent warp), and the
// GELU epilogue evaluates it 16K times per 128x128 tile on only four warps.
__device__ __forceinline__ float erf_fast(float x) {
    const float ax = fabsf(x);
    const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    poly *= t;
    const float e = exp2f(-1.4426950408889634f * ax * ax);
    return copysignf(fmaf(-poly, e, 1.0f), x);
}
// GELU, erf form: x * 0.5 * (1 + erf(x / sqrt(2)))   ([UPSTREAM] vilbert.py `gelu`)
__device__ __forceinline__ float gelu_erf_as(float x) { return x * 0.5f * (1.0f + erf_fast(x * 0.70710678118654752440f)); }
// Same function, 11 issue slots and no MUFU: gelu(x) = x * Phi(x) with Phi(x) ~ sat(0.5 + x * Q(x^2)), Q of degree 8 in x^2 fitted on
// |x| <= 4.25 with weight |x| (scripts/fit_gelu.py), sat = the FFMA's free saturation to [0, 1].  Q's leading coefficient is positive, so
// beyond the fitted range x * Q(x^2) runs monotonically to +-inf and the saturation returns Phi = 1 / 0 EXACTLY: a strongly negative
// pre-activation gives -0 and a strongly positive one x itself, with no range clamp.  |gelu error| <= 4.3e-5 over the whole fp32 range,
// < 5 % of half an fp16 ulp at the magnitude where it occurs; the A&S form above is 30x more accurate but costs ~27 slots incl. 2 MUFU,
// and the FFN-in epilogue evaluates it 16 K times per 128x128 tile.
__device__ __forceinline__ float gelu_erf(float x) {
    const float u = x * x;
    float q = 4.547042257e-11f;
    q = fmaf(q, u, -4.515281038e-09f);
    q = fmaf(q, u, 1.986152114e-07f);
    q = fmaf(q, u, -5.147503089e-06f);
    q = fmaf(q, u, 8.848903963e-05f);
    q = fmaf(q, u, -1.079077483e-03f);
    q = fmaf(q, u, 9.718777612e-03f);
    q = fmaf(q, u, -6.619028002e-02f);
    q = fmaf(q, u, 3.988192081e-01f);
    return x * __saturatef(fmaf(x, q, 0.5f));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
}
// 16-bit activation format selected at run time (warp-uniform): fp16 (11-bit significand) or bf16 (8-bit).
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t u) {
    __half2 v = *reinterpret_cast<__half2*>(&u);
    return __half22float2(v);
}
template <bool F16>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
    if constexpr (F16) return pack_h2(lo, hi);
    else return pack_bf16x2(lo, hi);
}
template <bool F16>
__device__ __forceinline__ float2 unpack16x2(uint32_t u) {
    if constexpr (F16) return unpack_h2(u);
    else return unpack_bf16x2(u);
}
__device__ __forceinline__ uint32_t pack16x2_rt(float lo, float hi, int f16) {
    // fp16 saturates instead of overflowing to inf (activations are LayerNorm-bounded; this is a guard rail)
    if (f16) return pack_h2(fminf(fmaxf(lo, -65504.0f), 65504.0f), fminf(fmaxf(hi, -65504.0f), 65504.0f));
    return pack_bf16x2(lo, hi);
}
__device__ __forceinline__ uint16_t cvt16_rt(float v, int f16) { return static_cast<uint16_t>(pack16x2_rt(v, 0.0f, f16) & 0xffffu); }

// ---- fp32-parity mode ("fp32x"): a value x travels as TWO fp16 numbers hi = fp16(x), lo = fp16(x - hi).  hi + lo is x to about
// |x| 2^-22 relative, with an absolute floor of 2^-25 (half the fp16 subnormal step, where lo is a subnormal, which the tensor cores
// handle): 22 significand bits for |x| >= 2^-3, 25 + log2|x| below that, about 19.4 for a weight of 0.02.  16-bit operand
// buffers then hold, per 64 logical columns, 192 physical ones: hi | lo | hi for activations, hi | hi | lo for weights, so that an
// ordinary K' = 3K GEMM computes hi.hi + lo.hi + hi.lo (the dropped lo.lo term is 2^-22 relative) with fp32 accumulation.
__host__ __device__ __forceinline__ int split_col(int c) { return (c >> 6) * 192 + (c & 63); }   // column of the first hi
__device__ __forceinline__ float split_hi(float x) {
    return __half2float(__float2half_rn(fminf(fmaxf(x, -65504.0f), 65504.0f)));
}
__device__ __forceinline__ float split_lo(float x) { return x - split_hi(x); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace vb
