// Residual-add + LayerNorm row kernel: x = y + res; out = (x - mean) / sqrt(var + eps) * gamma + beta, written as the
// fp32 residual stream AND the 16-bit operand of the next GEMM.
//
// Every LayerNorm after a GEMM runs here: the GEMM writes fp32, and this L2-resident row kernel (one warp per row, 16-byte
// coalesced accesses, two-pass fp32 statistics in registers) normalises it.  A row of N columns spans N / BLOCK_N GEMM tiles, so
// normalising inside the GEMM epilogue would need an exchange of statistics across CTAs; keeping it here keeps the GEMM epilogue
// light.  Replaces BertSelfOutput / BertOutput / BertBiOutput `LayerNorm(dense(x) + residual)` and the
// LayerNorm inside SimpleClassifier ([UPSTREAM] vilbert/vilbert.py; anchor worker.py:286-289).
#include <cstdlib>
#include "kernels.h"

namespace vb {

constexpr int kLnMaxVec = 16;   // N <= 2048: float4 per lane per 128 columns

// NV = float4 vectors per lane (N / 128): 6 for the 768-wide text stream, 8 for 1024; kLnMaxVec covers everything up to 2048
// with run-time predication (the specialised forms carry a third of the instructions and registers).
// SPLIT: fp32-parity mode, the 16-bit output is written as fp16 hi | lo | hi per 64 columns (common.cuh split_col).
template <bool F16, bool SPLIT, int NV>
__global__ void __launch_bounds__(256)
ln_residual_kernel(const float* __restrict__ y, int ld_y, const float* __restrict__ res, int ld_res,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   float* __restrict__ out_f32, int ld_f32, uint16_t* __restrict__ out16, int ld16, int M, int N, int pdl,
                   const int* __restrict__ m_rows) {
    if (pdl) pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M || (m_rows != nullptr && row >= *m_rows)) return;      // packed batches: rows past the device row count
    const int nvec = NV < kLnMaxVec ? NV : (N >> 7);
    const float4* yp = reinterpret_cast<const float4*>(y + static_cast<size_t>(row) * ld_y);
    const float4* rp = res ? reinterpret_cast<const float4*>(res + static_cast<size_t>(row) * ld_res) : nullptr;
    float4 x[NV];
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        if (k < nvec) {
            float4 a = yp[lane + 32 * k];
            if (rp) {
                const float4 r = rp[lane + 32 * k];
                a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
            }
            x[k] = a;
            s += a.x + a.y + a.z + a.w;
        }
    }
    if (pdl) pdl_launch_dependents();       // inputs are in registers: the next kernel's prologue may overlap the rest
    const float mean = warp_sum(s) / static_cast<float>(N);
    float sq = 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        if (k < nvec) {
            const float a = x[k].x - mean, b = x[k].y - mean, c = x[k].z - mean, d = x[k].w - mean;
            sq += a * a + b * b + c * c + d * d;
        }
    }
    const float rstd = 1.0f / sqrtf(warp_sum(sq) / static_cast<float>(N) + eps);
    const float4* gp = reinterpret_cast<const float4*>(gamma);
    const float4* bp = reinterpret_cast<const float4*>(beta);
    float4* of = out_f32 ? reinterpret_cast<float4*>(out_f32 + static_cast<size_t>(row) * ld_f32) : nullptr;
    uint2* oh = out16 ? reinterpret_cast<uint2*>(out16 + static_cast<size_t>(row) * ld16) : nullptr;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        if (k < nvec) {
            const float4 g = gp[lane + 32 * k], b = bp[lane + 32 * k];
            float4 o;
            o.x = (x[k].x - mean) * rstd * g.x + b.x;
            o.y = (x[k].y - mean) * rstd * g.y + b.y;
            o.z = (x[k].z - mean) * rstd * g.z + b.z;
            o.w = (x[k].w - mean) * rstd * g.w + b.w;
            if (of) of[lane + 32 * k] = o;
            if constexpr (SPLIT) {
                if (oh) {
                    const int c = 4 * (lane + 32 * k);                 // logical column of o.x; 4 columns stay inside one 64-group
                    uint2* o3 = reinterpret_cast<uint2*>(out16 + static_cast<size_t>(row) * ld16 + split_col(c));
                    const uint2 hi = make_uint2(pack16x2_rt(o.x, o.y, 1), pack16x2_rt(o.z, o.w, 1));
                    o3[0] = hi;
                    o3[16] = make_uint2(pack16x2_rt(split_lo(o.x), split_lo(o.y), 1), pack16x2_rt(split_lo(o.z), split_lo(o.w), 1));
                    o3[32] = hi;
                }
            } else {
                if (oh) oh[lane + 32 * k] = make_uint2(pack16x2<F16>(o.x, o.y), pack16x2<F16>(o.z, o.w));
            }
        }
    }
}

cudaError_t launch_ln_residual(const float* y, int ld_y, const float* res, int ld_res, const float* gamma, const float* beta,
                               float eps, float* out_f32, int ld_f32, __nv_bfloat16* out16, int ld16, int M, int N, int f16,
                               int split16, int pdl, cudaStream_t st, const int* m_rows) {
    if (N % 128 != 0 || N / 128 > kLnMaxVec || (ld_y & 3) || (res && (ld_res & 3)) || (out_f32 && (ld_f32 & 3)) ||
        (out16 && (ld16 & 3)) || M < 1 || (split16 && !f16))
        return cudaErrorInvalidValue;
    // one warp per row; 2 rows per CTA by default (VB200_LN_ROWS: 1..8)
    static const int rows_per_cta = [] { const char* e = getenv("VB200_LN_ROWS"); const int v = e ? atoi(e) : 2; return (v >= 1 && v <= 8) ? v : 2; }();
    const dim3 grid((M + rows_per_cta - 1) / rows_per_cta), block(32 * rows_per_cta);
    uint16_t* o16 = reinterpret_cast<uint16_t*>(out16);
#define VB_LN(F, S, V) launch_ex(ln_residual_kernel<F, S, V>, grid, block, 0, pdl, st, y, ld_y, res, ld_res, gamma, beta, eps, \
                               out_f32, ld_f32, o16, ld16, M, N, pdl, m_rows)
    if (split16) return VB_LN(true, true, kLnMaxVec);
    if (N == 768) return f16 ? VB_LN(true, false, 6) : VB_LN(false, false, 6);
    if (N == 1024) return f16 ? VB_LN(true, false, 8) : VB_LN(false, false, 8);
    return f16 ? VB_LN(true, false, kLnMaxVec) : VB_LN(false, false, kLnMaxVec);
#undef VB_LN
}

}  // namespace vb
