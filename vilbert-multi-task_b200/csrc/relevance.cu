// Attention relevance (vb200_attention_relevance): the residual-weighted attention rollout (Abnar & Zuidema 2020) of one forward's
// maps, carried through both ViLBERT streams, for the two rows the answer heads read -- the text CLS row (t_pooler) and the image
// global row (v_pooler).  For a sample with T text and V image rows, positions 0..T-1 are text and T..T+V-1 image.  A step (one text
// layer, one image layer, or both directions of one connection layer) defines W = I on the rows it does not write and
// 0.5 (e_i + M[i, :]) on the rows it writes, M its head-mean map in its block; the output rows are rows 0 and T of W_n ... W_1.
//
// Evaluation order, fixed so that a float32 restatement gives the same bits: r starts at e_0 / e_T and is multiplied by W from the
// last step to the first.  For each column j the step's map covers, acc_j = sum over the step's query rows i in increasing order of
// r_i * Abar[i, j] (separate fp32 products and adds from 0, no fma), then r_j = 0.5f * (r_j + acc_j); other columns keep r_j.  A
// connection step reads the old r for both directions.  Abar = (sum_h p_h, left to right in fp32) / heads: the engine's head mean,
// so maps written with every head and maps written as the mean give the same bits.
//
// One CTA per sample.  Shared memory: r and acc, 2 rows x (T + V) floats each, and a tile of the head-mean map of up to kTile
// floats.  Every thread fills the tile (consecutive threads read consecutive floats of a map row); then the thread owning column j
// adds the tile's rows into acc_j in increasing row order, so the sum over i runs in one order whatever the tile height.
#include "kernels.h"

namespace vb {

namespace {

constexpr int kRelThreads = 512;
constexpr int kTile = 4096;            // floats of head-mean map staged per pass (16 KB)

// The map block of one entry: sample b's [heads, Lq, Lk] at `p`, query rows at positions q0.., key columns at k0..
__device__ __forceinline__ void rollout_block(const float* __restrict__ p, int heads, int Lq, int Lk, int q0, int k0, int N, const float* r, float* acc,
                              float* tile) {
    const int rows = max(1, kTile / Lk);
    const float hf = static_cast<float>(heads);
    const int64_t hs = static_cast<int64_t>(Lq) * Lk;
    for (int i0 = 0; i0 < Lq; i0 += rows) {
        const int n = min(rows, Lq - i0) * Lk;
        const float* src = p + static_cast<int64_t>(i0) * Lk;
        for (int e = threadIdx.x; e < n; e += kRelThreads) {
            float s = 0.0f;
#pragma unroll 4
            for (int h = 0; h < heads; ++h) s = __fadd_rn(s, src[h * hs + e]);
            tile[e] = __fdiv_rn(s, hf);
        }
        __syncthreads();
        const int m = n / Lk;
        for (int j = threadIdx.x; j < Lk; j += kRelThreads) {
            float a0 = acc[k0 + j], a1 = acc[N + k0 + j];
            for (int i = 0; i < m; ++i) {
                const float a = tile[i * Lk + j];
                a0 = __fadd_rn(a0, __fmul_rn(r[q0 + i0 + i], a));
                a1 = __fadd_rn(a1, __fmul_rn(r[N + q0 + i0 + i], a));
            }
            acc[k0 + j] = a0;
            acc[N + k0 + j] = a1;
        }
        __syncthreads();                               // tile consumed
    }
}

__global__ void __launch_bounds__(kRelThreads, 1)
attention_relevance_kernel(const float* __restrict__ maps, const RelevanceEntry* __restrict__ entries, int n_entries,
                           const RelevanceSample* __restrict__ samples, float* __restrict__ relevance) {
    extern __shared__ __align__(16) float smem_rel[];
    const RelevanceSample s = samples[blockIdx.x];
    const int T = s.T, V = s.V, N = T + V;
    float* r = smem_rel;                               // [2][N]: the rows of CLS (0) and of the image global row (T)
    float* acc = r + 2 * N;                            // [2][N]
    float* tile = acc + 2 * N;                         // [kTile]
    for (int c = threadIdx.x; c < 2 * N; c += kRelThreads) r[c] = (c == 0 || c == N + T) ? 1.0f : 0.0f;
    for (int e = n_entries - 1; e >= 0; --e) {
        const RelevanceEntry d = entries[e];
        // kind 3: a connection layer, entries e - 1 (kind 2, checked on the host) and e, one step
        const int c0 = d.kind == 1 ? T : 0, c1 = d.kind == 0 ? T : N;      // the columns the step covers
        for (int c = c0 + threadIdx.x; c < c1; c += kRelThreads) acc[c] = acc[N + c] = 0.0f;
        __syncthreads();
        if (d.kind == 0) {
            rollout_block(maps + d.offset + d.heads * s.prefix[0], d.heads, T, T, 0, 0, N, r, acc, tile);
        } else if (d.kind == 1) {
            rollout_block(maps + d.offset + d.heads * s.prefix[1], d.heads, V, V, T, T, N, r, acc, tile);
        } else {
            const RelevanceEntry tv = entries[e - 1];  // kind 2: text queries over image keys [T, V]
            rollout_block(maps + tv.offset + tv.heads * s.prefix[2], tv.heads, T, V, 0, T, N, r, acc, tile);
            rollout_block(maps + d.offset + d.heads * s.prefix[2], d.heads, V, T, T, 0, N, r, acc, tile);
            --e;
        }
        for (int c = c0 + threadIdx.x; c < c1; c += kRelThreads) {
            r[c] = __fmul_rn(0.5f, __fadd_rn(r[c], acc[c]));
            r[N + c] = __fmul_rn(0.5f, __fadd_rn(r[N + c], acc[N + c]));
        }
        __syncthreads();
    }
    float* out = relevance + s.out;
    for (int c = threadIdx.x; c < 2 * N; c += kRelThreads) out[c] = r[c];
}

}  // namespace

cudaError_t launch_attention_relevance(const float* maps, const RelevanceEntry* entries, int n_entries, const RelevanceSample* samples,
                                       int B, int max_cols, float* relevance, cudaStream_t st) {
    if (B < 1 || n_entries < 1 || max_cols < 2 || maps == nullptr || relevance == nullptr) return cudaErrorInvalidValue;
    const size_t smem = sizeof(float) * (4 * static_cast<size_t>(max_cols) + kTile);
    cudaError_t e = set_smem(attention_relevance_kernel, smem);
    if (e != cudaSuccess) return e;
    return launch_ex(attention_relevance_kernel, dim3(B), dim3(kRelThreads), smem, 0, st, maps, entries, n_entries, samples, relevance);
}

}  // namespace vb
