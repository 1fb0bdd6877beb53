// Answer decode: logits of a forward -> each message's top-N probabilities, indices and (grounding) pixel boxes, one CTA per
// message.  Replaces prediction()'s per-message decode (worker.py:295-386): torch.softmax over the message's flattened logits,
// topk, and for grounding spatials[0][idx] scaled back to pixels (worker.py:374-385).
//
// Softmax as torch.softmax(x.view(-1), 0) computes it, in fp32: max, expf(x - max) (the accurate expf, not __expf), block sum,
// then a division by the sum.  Only the summation order differs from torch, so probabilities agree to rounding of the sum.
// Ranking is by probability, descending; equal probabilities rank the lower index first (torch.topk leaves that order open).
// Boxes: int((double)spatial * (double)image_size), truncated toward zero, as the reference's int(b[1] * image_h) on Python
// floats -- an fp32 product rounds some values across an integer boundary.
#include "kernels.h"

namespace vb {

constexpr int kDecodeThreads = 256;
constexpr int kDecodeWarps = kDecodeThreads / 32;

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

// Ranking key of element i with probability p >= 0: the bits of a non-negative float order as the float does, and the low word
// 0xffffffff - i puts the lower index first among equal probabilities.  Every element has its own key.
__device__ __forceinline__ unsigned long long rank_key(float p, int i) {
    return (static_cast<unsigned long long>(__float_as_uint(p)) << 32) | (0xffffffffu - static_cast<unsigned>(i));
}

// The softmax's max and sum of the `len` logits at x (every thread gets both), as torch.softmax computes them up to the order of the sum.
__device__ __forceinline__ float2 softmax_stats(const float* __restrict__ x, int len, float* s_f) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float m = -INFINITY;
    for (int i = tid; i < len; i += kDecodeThreads) m = fmaxf(m, x[i]);
    m = warp_max(m);
    if (lane == 0) s_f[warp] = m;
    __syncthreads();
    m = warp_max(lane < kDecodeWarps ? s_f[lane] : -INFINITY);
    __syncthreads();

    float s = 0.f;
    for (int i = tid; i < len; i += kDecodeThreads) s += expf(x[i] - m);
    s = warp_sum(s);
    if (lane == 0) s_f[warp] = s;
    __syncthreads();
    s = warp_sum(lane < kDecodeWarps ? s_f[lane] : 0.f);
    __syncthreads();                                  // s_f is reused by the next row's statistics
    return make_float2(m, s);
}

// s_pick[k] for k < top_n: the rank key of pick k, the largest key below pick k - 1's -- top_n passes over the row, each recomputing
// the same probabilities
__device__ __forceinline__ void pick_top(const float* __restrict__ x, int len, float2 ms, int top_n, unsigned long long* s_k,
                                         unsigned long long* s_pick) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long prev = ~0ull;
    for (int k = 0; k < top_n; ++k) {
        unsigned long long best = 0;
        for (int i = tid; i < len; i += kDecodeThreads) {
            const unsigned long long key = rank_key(expf(x[i] - ms.x) / ms.y, i);
            if (key < prev && key > best) best = key;
        }
        best = warp_max_u64(best);
        if (lane == 0) s_k[warp] = best;
        __syncthreads();
        best = warp_max_u64(lane < kDecodeWarps ? s_k[lane] : 0ull);
        if (tid == 0) s_pick[k] = best;
        __syncthreads();
        prev = best;
    }
}

__device__ __forceinline__ int key_index(unsigned long long key) { return static_cast<int>(0xffffffffu - static_cast<unsigned>(key & 0xffffffffu)); }

__global__ void __launch_bounds__(kDecodeThreads)
answer_decode_kernel(const DecodeDesc* __restrict__ descs, vb200_answer* __restrict__ answers) {
    __shared__ float s_f[kDecodeWarps];
    __shared__ unsigned long long s_k[kDecodeWarps];
    __shared__ unsigned long long s_pick[VB200_DECODE_MAX_TOP];
    const DecodeDesc d = descs[blockIdx.x];
    const float* __restrict__ x = d.src;
    const int tid = threadIdx.x;

    const float2 ms = softmax_stats(x, d.len, s_f);
    pick_top(x, d.len, ms, d.top_n, s_k, s_pick);

    if (d.score != nullptr) {                         // answer ablation: one score, no answer
        const unsigned long long top1 = s_pick[0];
        int col = d.column;
        if (col < 0) {                                // the unablated segment's top-1, as its own decode ranks it
            const int ref_len = d.len + (d.drop >= 0 ? 1 : 0);
            const float2 ref = softmax_stats(d.ref, ref_len, s_f);
            pick_top(d.ref, ref_len, ref, 1, s_k, s_pick);
            col = key_index(s_pick[0]);
        }
        if (tid == 0) {
            // a dropped row: the attributed row of the unablated numbering maps into src, or is gone
            const bool gone = d.drop >= 0 && col == d.drop;
            const int at = d.drop >= 0 && col > d.drop ? col - 1 : col;
            const int t = key_index(top1);
            vb200_ablation_score sc;
            sc.answer = gone ? -1 : col;
            sc.prob = gone ? 0.f : expf(x[at] - ms.x) / ms.y;
            sc.top1 = d.drop >= 0 && t >= d.drop ? t + 1 : t;
            sc.top1_prob = __uint_as_float(static_cast<unsigned>(top1 >> 32));
            *d.score = sc;
        }
        return;
    }

    vb200_answer* a = answers + blockIdx.x;
    if (tid == 0) a->n = d.top_n;
    if (tid < VB200_DECODE_MAX_TOP) {
        const bool on = tid < d.top_n;
        a->index[tid] = on ? key_index(s_pick[tid]) : -1;
        a->prob[tid] = on ? __uint_as_float(static_cast<unsigned>(s_pick[tid] >> 32)) : 0.f;
    }
    if (tid < 4 * VB200_DECODE_MAX_TOP) {
        const int k = tid >> 2, c = tid & 3;       // box k, coordinate c of x1, y1, x2, y2 (spatials columns 0-3)
        int v = 0;
        if (d.spatials != nullptr && k < d.top_n) {
            const int row = key_index(s_pick[k]);
            const double size = (c & 1) ? d.image_h : d.image_w;
            v = __double2int_rz(static_cast<double>(d.spatials[static_cast<size_t>(row) * 5 + c]) * size);
        }
        a->box[k][c] = v;
    }
}

cudaError_t launch_answer_decode(const DecodeDesc* descs, int n, vb200_answer* answers, cudaStream_t st) {
    return launch_ex(answer_decode_kernel, dim3(n), dim3(kDecodeThreads), 0, 0, st, descs, answers);
}

__global__ void __launch_bounds__(128)
segment_gather_kernel(const SegmentDesc* __restrict__ descs, const __grid_constant__ SegmentHeads heads, float* __restrict__ out) {
    const SegmentDesc d = descs[blockIdx.x];
    const float* __restrict__ p = heads.p[d.head];
    const int64_t ld = heads.ld[d.head];
    const bool run = heads.cols[d.head] == 1;         // a one-column head: the segment is a run of rows
    float* __restrict__ dst = out + d.dst;
    for (int i = threadIdx.x; i < d.len; i += blockDim.x) {
        const int64_t at = i == d.sub ? d.sub_row * ld : run ? (d.row + i) * ld : d.row * ld + i;
        dst[i] = p[at];
    }
}

cudaError_t launch_segment_gather(const SegmentDesc* descs, int n, const SegmentHeads& heads, float* out, cudaStream_t st) {
    if (n < 1) return cudaErrorInvalidValue;
    return launch_ex(segment_gather_kernel, dim3(n), dim3(128), 0, 0, st, descs, heads, out);
}

// Permutation-sampled Shapley values: one CTA per message, thread u owns unit u.  For each permutation p the CTA inverts row p into
// shared memory (inv[perm[p][j]] = j), so unit u finds its position j and its marginal c[p][j+1] - c[p][j] in float64.  Pass 1 sums
// the marginals over p in order; pass 2 recomputes them group by group for the two-pass standard error.  Every float64 operation is
// an explicitly rounded intrinsic, so no multiply-add is contracted and numpy's sequential float64 arithmetic gives the same bits.  A
// row that is not a permutation of 0 .. n-1 (some unit has no position) gives NaN for every unit of the message.
__global__ void __launch_bounds__(kShapleyMaxUnits)
shapley_values_kernel(const ShapleyDesc* __restrict__ descs) {
    __shared__ int inv[kShapleyMaxUnits];
    const ShapleyDesc d = descs[blockIdx.x];
    const int n = d.n_units, P = d.n_perm, g = d.group, u = threadIdx.x;
    const float* __restrict__ v = d.values;
    auto chain = [&](int p, int j) -> double {                 // c[p][j]: v(empty) at 0, v(all) at n, the chain in between
        return static_cast<double>(j == 0 ? v[0] : j == n ? v[1] : v[2 + static_cast<int64_t>(p) * (n - 1) + (j - 1)]);
    };
    bool bad = false;
    auto marginal = [&](int p) -> double {                     // unit u's marginal in permutation p (every thread must call)
        const int32_t* __restrict__ row = d.perm + static_cast<int64_t>(p) * n;
        __syncthreads();                                       // the previous permutation's reads of inv are done
        if (u < n) inv[u] = -1;
        __syncthreads();
        if (u < n) {
            const int w = row[u];
            if (w >= 0 && w < n) inv[w] = u;
        }
        __syncthreads();
        if (u >= n) return 0.0;
        const int j = inv[u];
        if (j < 0 || row[j] != u) { bad = true; return 0.0; }
        return __dsub_rn(chain(p, j + 1), chain(p, j));
    };
    double sum = 0.0;
    for (int p = 0; p < P; ++p) sum = __dadd_rn(sum, marginal(p));
    const double phi = __ddiv_rn(sum, static_cast<double>(P));
    const int G = P / g;
    double ss = 0.0;
    for (int q = 0; q < G; ++q) {
        double m = 0.0;
        for (int i = 0; i < g; ++i) m = __dadd_rn(m, marginal(q * g + i));
        m = __ddiv_rn(m, static_cast<double>(g));
        const double t = __dsub_rn(m, phi);
        ss = __dadd_rn(ss, __dmul_rn(t, t));
    }
    bad = __syncthreads_or(bad) != 0;
    if (u >= n) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const double se = G < 2 ? nan : __dsqrt_rn(__ddiv_rn(__ddiv_rn(ss, static_cast<double>(G - 1)), static_cast<double>(G)));
    d.phi[u] = static_cast<float>(bad ? nan : phi);
    d.stderr_out[u] = static_cast<float>(bad ? nan : se);
}

cudaError_t launch_shapley_values(const ShapleyDesc* descs, int n, cudaStream_t st) {
    if (n < 1) return cudaErrorInvalidValue;
    return launch_ex(shapley_values_kernel, dim3(n), dim3(kShapleyMaxUnits), 0, 0, st, descs);
}

// Shapley-Taylor pair indices: CTA (m, k) takes pairs [k * 1024, k * 1024 + 1024) of message m, thread t owns pair k * 1024 + t.
// For each permutation p the CTA inverts row p into shared memory as shapley_values_kernel does; each thread then reads its pair's
// two ranks, the chain values c[p][r] and c[p][r + 1] and its x1, x2, and forms the second difference in float64.  Pass 1 sums the
// differences over p in order; pass 2 recomputes them group by group for the two-pass standard error.  Each thread's sums are
// serial in p, so numpy's sequential float64 arithmetic gives the same bits.  Thread t < n also checks that unit t has a position in
// row p; every CTA of a message checks every row in full, so a row that is not a permutation gives NaN for every pair of the message.
__global__ void __launch_bounds__(kInteractionPairs)
interaction_values_kernel(const InteractionDesc* __restrict__ descs) {
    __shared__ int inv[kShapleyMaxUnits];
    const InteractionDesc d = descs[blockIdx.x];
    const int q = blockIdx.y * kInteractionPairs + threadIdx.x;
    if (blockIdx.y * kInteractionPairs >= d.n_pairs) return;         // the whole CTA: this message has fewer pairs
    const int n = d.n_units, P = d.n_perm, g = d.group, Q = d.n_pairs, t = threadIdx.x;
    const bool on = q < Q;
    const int a = on ? d.pairs[2 * q] : 0, b = on ? d.pairs[2 * q + 1] : 0;
    const float* __restrict__ v = d.values;
    const float* __restrict__ x = v + 2 + static_cast<int64_t>(P) * (n - 1);    // x1, x2 of (p, q) at 2 (p Q + q)
    auto chain = [&](int p, int j) -> double {                 // c[p][j]: v(empty) at 0, the chain in between (j < n here)
        return static_cast<double>(j == 0 ? v[0] : v[2 + static_cast<int64_t>(p) * (n - 1) + (j - 1)]);
    };
    bool bad = false;
    auto delta = [&](int p) -> double {                        // the pair's second difference in permutation p (every thread calls)
        const int32_t* __restrict__ row = d.perm + static_cast<int64_t>(p) * n;
        __syncthreads();                                       // the previous permutation's reads of inv are done
        if (t < n) inv[t] = -1;
        __syncthreads();
        if (t < n) {
            const int w = row[t];
            if (w >= 0 && w < n) inv[w] = t;
        }
        __syncthreads();
        if (t < n && inv[t] < 0) bad = true;                   // unit t has no position: row p is not a permutation
        if (!on) return 0.0;
        const int ra = inv[a], rb = inv[b];
        if (ra < 0 || rb < 0) return 0.0;                      // flagged by the threads of units a and b
        const int r = min(ra, rb);
        const int64_t at = 2 * (static_cast<int64_t>(p) * Q + q);
        const double x1 = static_cast<double>(x[at]), x2 = static_cast<double>(x[at + 1]);
        return __dadd_rn(__dsub_rn(__dsub_rn(x2, chain(p, r + 1)), x1), chain(p, r));
    };
    double sum = 0.0;
    for (int p = 0; p < P; ++p) sum = __dadd_rn(sum, delta(p));
    const double inter = __ddiv_rn(sum, static_cast<double>(P));
    const int G = P / g;
    double ss = 0.0;
    for (int k = 0; k < G; ++k) {
        double m = 0.0;
        for (int i = 0; i < g; ++i) m = __dadd_rn(m, delta(k * g + i));
        m = __ddiv_rn(m, static_cast<double>(g));
        const double dm = __dsub_rn(m, inter);
        ss = __dadd_rn(ss, __dmul_rn(dm, dm));
    }
    bad = __syncthreads_or(bad) != 0;
    if (!on) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const double se = G < 2 ? nan : __dsqrt_rn(__ddiv_rn(__ddiv_rn(ss, static_cast<double>(G - 1)), static_cast<double>(G)));
    d.inter[q] = static_cast<float>(bad ? nan : inter);
    d.stderr_out[q] = static_cast<float>(bad ? nan : se);
}

// messages along x (any count), pair blocks along y (at most VB200_INTERACTION_MAX_PAIRS / 1024 = 64)
cudaError_t launch_interaction_values(const InteractionDesc* descs, int n, int max_pairs, cudaStream_t st) {
    if (n < 1 || max_pairs < 1) return cudaErrorInvalidValue;
    const dim3 grid(n, (max_pairs + kInteractionPairs - 1) / kInteractionPairs);
    return launch_ex(interaction_values_kernel, grid, dim3(kInteractionPairs), 0, 0, st, descs);
}

}  // namespace vb
