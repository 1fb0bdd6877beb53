// fp32 attention on CUDA cores: softmax(Q K^T / sqrt(d) + mask) V with every product, the softmax and the P V sum in fp32.
//
// Two users, both off the throughput path (attention is 0.9 % of the FLOPs; the default path is the mma.sync kernel of
// attention.cu):
//   * the fp32-parity mode (compute_dtype = "fp32x"): Q/K/V arrive as fp32 from the split-operand QKV GEMM and the context
//     leaves as the fp16 hi | lo | hi operand of the next GEMM (common.cuh split_col);
//   * `attn_data_list`, element 9 of the reference's 10-tuple (worker.py:287-288, returned because the worker
//     sets config.visualization, worker.py:522): the attention probabilities [B, heads, Lq, Lk] in fp32, written by this
//     kernel from the same 16-bit Q/K the tensor-core kernel consumed (context output off).
//
// One CTA = (head, sample, 8 query rows), one warp per query row.  Keys are staged 32 at a time in shared memory with an odd
// row stride, lane j owns key j of the chunk (no shuffle reductions); P V reads V rows straight from global memory (32
// consecutive columns per warp instruction; the rows stay in L1/L2 for the other seven warps).
//
// Packed batches (VB200_OUT_ATTENTION_PACKED, kernels.h PackedProbs): the same kernel with PACKED = true.  Each CTA takes its
// sample's query / key row offsets from the plan's d_meta, runs every loop, the key chunking and the softmax at the sample's own
// Lq_b / Lk_b (the grid and shared memory are sized for the capacities; CTAs past Lq_b exit at once) and writes its probability
// rows straight into the caller's buffer.  The arithmetic is this one code path, so each sample's probabilities are bit-identical
// to a dense forward of that sample alone.  No context output: the tensor-core kernel writes it.
//
// Head mean (vb200_set_option "attention_heads" = 1): attention_f32_mean_kernel, dense and packed, one CTA per (sample, 8 query
// rows) looping over the heads; each head's row comes from the same score_row / softmax_row code as the per-head kernel's.
#include "kernels.h"

namespace vb {

namespace {

constexpr int kQRows = 8;          // query rows (= warps) per CTA
constexpr int kKeyChunk = 32;      // keys staged per pass

template <int IN> struct InT;
template <> struct InT<0> { using type = float; };
template <> struct InT<1> { using type = uint16_t; };     // fp16 bits
template <> struct InT<2> { using type = uint16_t; };     // bf16 bits

template <int IN>
__device__ __forceinline__ float ld_as_f32(const typename InT<IN>::type* p) {
    if constexpr (IN == 0) return *p;
    else if constexpr (IN == 1) return __half2float(__ushort_as_half(*p));
    else return __uint_as_float(static_cast<uint32_t>(*p) << 16);
}

// Scores of head h for this warp's query row i = i0 + warp (row_ok: i < Lq) over keys [0, Lk) of sample rows q0 / k0: Q row to qs,
// keys staged kKeyChunk at a time in ks, score j (scaled, plus the additive key mask; -inf past Lk) to pr[j] by lane j % 32.  Every
// thread of the CTA calls it: the key staging holds block-wide barriers.
template <int IN>
__device__ __forceinline__ void score_row(const typename InT<IN>::type* __restrict__ q, int ld_q,
                                          const typename InT<IN>::type* __restrict__ k, int ld_kv,
                                          const float* __restrict__ key_mask_add, int q0, int k0, int i, bool row_ok, int Lk, int D,
                                          int h, float scale, float* qs, float* ks, float* pr) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (row_ok) {
        const auto* qp = q + static_cast<size_t>(q0 + i) * ld_q + h * D;
        for (int d = lane; d < D; d += 32) qs[warp * D + d] = ld_as_f32<IN>(qp + d);
    }
    // a chunk is at most kKeyChunk x 128 elements, kStage per thread: every load of a chunk is issued before the first store, so their
    // latencies overlap instead of adding up (the head-mean kernel runs its heads' chunks one after another)
    constexpr int kStage = kKeyChunk * 128 / (32 * kQRows);
    for (int j0 = 0; j0 < Lk; j0 += kKeyChunk) {
        float kv[kStage];
#pragma unroll
        for (int t = 0; t < kStage; ++t) {
            const int e = threadIdx.x + t * 32 * kQRows, j = e / D, d = e - j * D;
            kv[t] = (e < kKeyChunk * D && j0 + j < Lk) ? ld_as_f32<IN>(k + static_cast<size_t>(k0 + j0 + j) * ld_kv + h * D + d) : 0.0f;
        }
        __syncthreads();                               // previous chunk consumed (and qs written, first pass)
#pragma unroll
        for (int t = 0; t < kStage; ++t) {
            const int e = threadIdx.x + t * 32 * kQRows, j = e / D, d = e - j * D;
            if (e < kKeyChunk * D) ks[j * (D + 1) + d] = kv[t];
        }
        __syncthreads();
        if (row_ok) {
            float acc = 0.0f;
            const float* kr = ks + lane * (D + 1);
            const float* qr = qs + warp * D;
#pragma unroll 8
            for (int d = 0; d < D; ++d) acc = fmaf(qr[d], kr[d], acc);
            const int j = j0 + lane;
            pr[j] = j < Lk ? acc * scale + key_mask_add[k0 + j] : -INFINITY;
        }
    }
}

// Softmax of one warp's score row pr[0, Lk) in place, unnormalised: pr[j] = exp(s_j - max); returns 1 / sum.  The probability is
// pr[j] * inv.
__device__ __forceinline__ float softmax_row(float* pr, int Lk) {
    const int lane = threadIdx.x & 31;
    float m = -INFINITY;
    for (int j = lane; j < Lk; j += 32) m = fmaxf(m, pr[j]);
    m = warp_max(m);
    float sum = 0.0f;
    for (int j = lane; j < Lk; j += 32) { const float e = expf(pr[j] - m); pr[j] = e; sum += e; }
    sum = warp_sum(sum);
    return 1.0f / sum;
}

// q / k / v point at column 0 of head 0 of sample 0; row (b, i) of Q is q + (b * Lq + i) * ld_q, K/V rows use ld_kv.
// ctx_mode: 0 no context output, 1 fp16, 2 bf16, 3 fp16 hi | lo | hi (ld_ctx is then the 3x wider physical stride).
// PACKED: Lq / Lk are the capacities; sample b's rows and lengths come from pk (probs and ctx are unused).
// __launch_bounds__(.., 4): at most 64 registers, four CTAs per SM, no spills with the 16 staged key values per thread
template <int IN, bool PACKED>
__global__ void __launch_bounds__(32 * kQRows, 4)
attention_f32_kernel(const typename InT<IN>::type* __restrict__ q, int ld_q, const typename InT<IN>::type* __restrict__ k,
                     const typename InT<IN>::type* __restrict__ v, int ld_kv, const float* __restrict__ key_mask_add, int Lq,
                     int Lk, int D, float scale, uint16_t* __restrict__ ctx, int ld_ctx, int ctx_mode, float* __restrict__ probs,
                     int pdl, PackedProbs pk) {
    extern __shared__ __align__(16) float smem_f32[];
    const int h = blockIdx.x, b = blockIdx.y, i0 = blockIdx.z * kQRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Lkp = (Lk + 31) & ~31;                   // PACKED: the capacity's, an upper bound of every sample's
    float* qs = smem_f32;                              // [kQRows][D]
    float* ks = qs + kQRows * D;                       // [kKeyChunk][D + 1]
    float* ps = ks + kKeyChunk * (D + 1);              // [kQRows][Lkp]
    if (pdl) pdl_wait();
    // sample b: query rows [q0, q0 + Lq), key rows [k0, k0 + Lk)
    int q0 = b * Lq, k0 = b * Lk;
    if constexpr (PACKED) {
        q0 = pk.offs_q[b]; Lq = pk.offs_q[b + 1] - q0;
        k0 = pk.offs_k[b]; Lk = pk.offs_k[b + 1] - k0;
        if (i0 >= Lq) return;                          // the whole CTA is past this sample's rows (no barrier reached yet)
    }
    const int i = i0 + warp;                           // this warp's query row
    const bool row_ok = i < Lq;
    float* pr = ps + warp * Lkp;
    score_row<IN>(q, ld_q, k, ld_kv, key_mask_add, q0, k0, i, row_ok, Lk, D, h, scale, qs, ks, pr);
    if (pdl) pdl_launch_dependents();
    if (!row_ok) return;                               // no block-wide barrier below this line
    __syncwarp();
    const float inv = softmax_row(pr, Lk);
    float* gp = nullptr;
    float g = 1.0f;
    if constexpr (PACKED) {
        g = pk.gate.at(b, h);                          // gated plans report g * p
        // entry offset + heads * sum_{b' < b} Lq_b' Lk_b' + (h, i) inside the sample's [heads, Lq, Lk] block, in int64: one call's
        // entries hold more than 2^31 floats at large batches
        float* dst = reinterpret_cast<float*>(pk.dst[0]);
        if (dst) gp = dst + pk.entry[0] + static_cast<int64_t>(gridDim.x) * pk.prefix[b] + (static_cast<int64_t>(h) * Lq + i) * Lk;
    } else {
        gp = probs ? probs + ((static_cast<size_t>(b) * gridDim.x + h) * Lq + i) * Lk : nullptr;
    }
    for (int j = lane; j < Lk; j += 32) {
        const float pj = pr[j] * inv;
        pr[j] = pj;
        if (gp) gp[j] = pj * g;
    }
    __syncwarp();
    if (PACKED || ctx_mode == 0) return;
    // ---- context row: lane owns columns lane, lane + 32, ...
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};           // D <= 128
    const auto* vb = v + static_cast<size_t>(b) * Lk * ld_kv + h * D;
    for (int j = 0; j < Lk; ++j) {
        const float pj = pr[j];
        const auto* vr = vb + static_cast<size_t>(j) * ld_kv;
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (lane + 32 * t < D) acc[t] = fmaf(pj, ld_as_f32<IN>(vr + lane + 32 * t), acc[t]);
    }
    uint16_t* orow = ctx + static_cast<size_t>(q0 + i) * ld_ctx;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int c = h * D + lane + 32 * t;
        if (lane + 32 * t < D) {
            if (ctx_mode == 3) {
                const int c3 = split_col(c);
                const uint16_t hi = cvt16_rt(acc[t], 1);
                orow[c3] = hi;
                orow[c3 + 64] = cvt16_rt(split_lo(acc[t]), 1);
                orow[c3 + 128] = hi;
            } else {
                orow[c] = cvt16_rt(acc[t], ctx_mode == 1 ? 1 : 0);
            }
        }
    }
}

// Head mean of the probabilities: one CTA = (sample, 8 query rows) loops over the heads in increasing order, computes each head's row
// with the per-head kernel's code (score_row, softmax_row, p = pr[j] * inv) and adds it into an fp32 accumulator row in shared
// memory; the row written is (sum_{h = 0..H-1} p_h, summed left to right in fp32) / H -- reproducible bit for bit from the per-head
// maps.  The add and the product are kept apart (__fadd_rn / __fmul_rn): a contracted fma would not be that sum.  Maps only, no
// context.  probs [B, Lq, Lk]; PACKED: sample b's [Lq_b, Lk_b] block at the entry's offset + prefix[b] (the heads factor is 1).
template <int IN, bool PACKED>
__global__ void __launch_bounds__(32 * kQRows, 4)
attention_f32_mean_kernel(const typename InT<IN>::type* __restrict__ q, int ld_q, const typename InT<IN>::type* __restrict__ k, int ld_kv,
                          const float* __restrict__ key_mask_add, int Lq, int Lk, int heads, int D, float scale, float* __restrict__ probs,
                          int pdl, PackedProbs pk) {
    extern __shared__ __align__(16) float smem_f32[];
    const int b = blockIdx.y, i0 = blockIdx.z * kQRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Lkp = (Lk + 31) & ~31;
    float* qs = smem_f32;                              // [kQRows][D]
    float* ks = qs + kQRows * D;                       // [kKeyChunk][D + 1]
    float* ps = ks + kKeyChunk * (D + 1);              // [kQRows][Lkp]
    float* as = ps + kQRows * Lkp;                     // [kQRows][Lkp]: the running sum over heads
    if (pdl) pdl_wait();
    int q0 = b * Lq, k0 = b * Lk;
    if constexpr (PACKED) {
        q0 = pk.offs_q[b]; Lq = pk.offs_q[b + 1] - q0;
        k0 = pk.offs_k[b]; Lk = pk.offs_k[b + 1] - k0;
        if (i0 >= Lq) return;                          // the whole CTA is past this sample's rows (no barrier reached yet)
    }
    const int i = i0 + warp;
    const bool row_ok = i < Lq;
    float* pr = ps + warp * Lkp;
    float* ar = as + warp * Lkp;
    for (int j = lane; j < Lk; j += 32) ar[j] = 0.0f;  // lane j % 32 owns column j of pr and ar throughout
    for (int h = 0; h < heads; ++h) {
        score_row<IN>(q, ld_q, k, ld_kv, key_mask_add, q0, k0, i, row_ok, Lk, D, h, scale, qs, ks, pr);
        if (row_ok) {                                  // rows past Lq keep staging keys with the CTA: no return before the last head
            __syncwarp();
            const float inv = softmax_row(pr, Lk);
            const float g = PACKED ? pk.gate.at(b, h) : 1.0f;     // gated plans average g * p (x * 1.0f is exact)
            for (int j = lane; j < Lk; j += 32) ar[j] = __fadd_rn(ar[j], __fmul_rn(__fmul_rn(pr[j], inv), g));
        }
    }
    if (pdl) pdl_launch_dependents();
    if (!row_ok) return;
    float* gp;
    if constexpr (PACKED) {
        float* dst = reinterpret_cast<float*>(pk.dst[0]);
        if (!dst) return;
        gp = dst + pk.entry[0] + pk.prefix[b] + static_cast<int64_t>(i) * Lk;
    } else {
        gp = probs + (static_cast<size_t>(b) * Lq + i) * Lk;
    }
    const float hf = static_cast<float>(heads);
    for (int j = lane; j < Lk; j += 32) gp[j] = __fdiv_rn(ar[j], hf);
}

}  // namespace

cudaError_t launch_attention_f32(const void* q, int ld_q, const void* k, const void* v, int ld_kv, int in_kind,
                                 const float* key_mask_add, int B, int Lq, int Lk, int heads, int D, __nv_bfloat16* ctx, int ld_ctx,
                                 int ctx_mode, float* probs, int pdl, cudaStream_t st, const PackedProbs* packed) {
    if (B < 1 || Lq < 1 || Lk < 1 || heads < 1 || D < 32 || D > 128 || (D & 31) || in_kind < 0 || in_kind > 2 || ctx_mode < 0 ||
        ctx_mode > 3 || (ctx_mode != 0 && ctx == nullptr) || (ctx_mode == 0 && probs == nullptr && packed == nullptr))
        return cudaErrorInvalidValue;
    if (packed && (ctx_mode != 0 || probs != nullptr || in_kind == 0 || !packed->offs_q || !packed->offs_k || !packed->dst ||
                   !packed->entry || !packed->prefix))
        return cudaErrorInvalidValue;
    const PackedProbs pk = packed ? *packed : PackedProbs{};
    const int Lkp = (Lk + 31) & ~31;
    const size_t smem = sizeof(float) * (static_cast<size_t>(kQRows) * D + kKeyChunk * (D + 1) + static_cast<size_t>(kQRows) * Lkp);
    const dim3 grid(heads, B, (Lq + kQRows - 1) / kQRows), block(32 * kQRows);
    const float scale = 1.0f / sqrtf(static_cast<float>(D));
    uint16_t* c16 = reinterpret_cast<uint16_t*>(ctx);
#define VB_AF(IN, P)                                                                                                     \
    do {                                                                                                                 \
        cudaError_t e = set_smem(attention_f32_kernel<IN, P>, smem);                                                     \
        if (e != cudaSuccess) return e;                                                                                  \
        using T = typename InT<IN>::type;                                                                                \
        return launch_ex(attention_f32_kernel<IN, P>, grid, block, smem, pdl, st, static_cast<const T*>(q), ld_q,        \
                         static_cast<const T*>(k), static_cast<const T*>(v), ld_kv, key_mask_add, Lq, Lk, D, scale, c16, \
                         ld_ctx, ctx_mode, probs, pdl, pk);                                                              \
    } while (0)
    if (packed) {
        if (in_kind == 1) VB_AF(1, true);
        VB_AF(2, true);
    }
    if (in_kind == 0) VB_AF(0, false);
    if (in_kind == 1) VB_AF(1, false);
    VB_AF(2, false);
#undef VB_AF
}

cudaError_t launch_attention_f32_mean(const void* q, int ld_q, const void* k, int ld_kv, int in_kind, const float* key_mask_add, int B,
                                      int Lq, int Lk, int heads, int D, float* probs, int pdl, cudaStream_t st, const PackedProbs* packed) {
    if (B < 1 || Lq < 1 || Lk < 1 || heads < 1 || D < 32 || D > 128 || (D & 31) || in_kind < 0 || in_kind > 2 ||
        (probs == nullptr) == (packed == nullptr))
        return cudaErrorInvalidValue;
    if (packed && (in_kind == 0 || !packed->offs_q || !packed->offs_k || !packed->dst || !packed->entry || !packed->prefix))
        return cudaErrorInvalidValue;
    const PackedProbs pk = packed ? *packed : PackedProbs{};
    const int Lkp = (Lk + 31) & ~31;
    const size_t smem = sizeof(float) * (static_cast<size_t>(kQRows) * D + kKeyChunk * (D + 1) + 2 * static_cast<size_t>(kQRows) * Lkp);
    const dim3 grid(1, B, (Lq + kQRows - 1) / kQRows), block(32 * kQRows);
    const float scale = 1.0f / sqrtf(static_cast<float>(D));
#define VB_AM(IN, P)                                                                                                     \
    do {                                                                                                                 \
        cudaError_t e = set_smem(attention_f32_mean_kernel<IN, P>, smem);                                                \
        if (e != cudaSuccess) return e;                                                                                  \
        using T = typename InT<IN>::type;                                                                                \
        return launch_ex(attention_f32_mean_kernel<IN, P>, grid, block, smem, pdl, st, static_cast<const T*>(q), ld_q,   \
                         static_cast<const T*>(k), ld_kv, key_mask_add, Lq, Lk, heads, D, scale, probs, pdl, pk);        \
    } while (0)
    if (packed) {
        if (in_kind == 1) VB_AM(1, true);
        VB_AM(2, true);
    }
    if (in_kind == 0) VB_AM(0, false);
    if (in_kind == 1) VB_AM(1, false);
    VB_AM(2, false);
#undef VB_AM
}

}  // namespace vb
