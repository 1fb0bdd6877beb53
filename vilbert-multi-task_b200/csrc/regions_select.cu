// Detector-region selection (vb200_select_regions): the detector's raw heads -> each image's top boxes, written straight into the
// packed box_features / boxes that vb200_forward_regions_packed reads.  Restates the feature extraction step of the reference worker
// (worker.py:123-176): per-proposal softmax, per-class greedy NMS on the original-pixel boxes, the per-box maximum confidence over the
// classes that keep it, a descending rank and the gather of the first K rows.
//
//   select_row_stats_kernel   per proposal: softmax max and sum over the C logits, the divided box proposals / (float)im_scale
//   select_iou_mask_kernel    per image: the n x n suppression bitmask (legacy "+1" IoU > nms_iou), shared by every class
//   select_class_nms_kernel   per (image, 8 classes): one warp per class sorts its probabilities and walks the bitmask greedily
//   select_rank_kernel        per image: rank max_conf, write keep_index / max_conf / boxes / num_boxes
//   select_gather_kernel      per output row: the feature row, and optionally the probability row and its argmax
//
// Every probability is expf(x - max) / sum from the row's two stats floats, so no [n, C] matrix is materialised and every kernel sees
// the same bits for the same (box, class).  Ranks order (probability desc, index asc): the key (float bits << 32) | (0xffffffff - i)
// is unique per element.  The only atomics are unsigned atomicMax on the bits of non-negative floats, which order as the floats do,
// so results do not depend on the order the classes finish in.
#include "kernels.h"

namespace vb {

constexpr int kSelWarps = 8;                   // classes per NMS block; rows per stats / mask block
constexpr int kSelThreads = kSelWarps * 32;
constexpr int kRankThreads = 512;

__device__ __forceinline__ unsigned long long sel_key(float p, int i) {
    return (static_cast<unsigned long long>(__float_as_uint(p)) << 32) | (0xffffffffu - static_cast<unsigned>(i));
}
__device__ __forceinline__ int key_index(unsigned long long k) {
    return static_cast<int>(0xffffffffu - static_cast<unsigned>(k & 0xffffffffu));
}

__global__ void __launch_bounds__(kSelThreads)
select_row_stats_kernel(const SelectDesc* __restrict__ descs, SelectArgs a) {
    const SelectDesc d = descs[blockIdx.y];
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kSelWarps + (threadIdx.x >> 5);
    if (r >= d.n) return;
    const float* __restrict__ x = d.scores + static_cast<size_t>(r) * a.C;
    float m = -INFINITY;
    for (int c = lane; c < a.C; c += 32) m = fmaxf(m, x[c]);
    m = warp_max(m);
    float s = 0.f;
    for (int c = lane; c < a.C; c += 32) s += expf(x[c] - m);
    s = warp_sum(s);
    const size_t row = d.row0 + r;
    if (lane == 0) a.stats[row] = make_float2(m, s);
    if (lane < 4) a.dbox[row * 4 + lane] = __fdiv_rn(d.proposals[static_cast<size_t>(r) * 4 + lane], d.im_scale);
}

// IoU of the maskrcnn_benchmark legacy NMS, every operation rounded on its own (no contraction into FMAs) so the host restatement
// in numpy fp32 gives the same bits.
__device__ __forceinline__ float legacy_iou(float4 a, float4 b) {
    const float w = fmaxf(__fadd_rn(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 1.f), 0.f);
    const float h = fmaxf(__fadd_rn(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 1.f), 0.f);
    const float inter = __fmul_rn(w, h);
    const float sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
    const float sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
}

// bit j of word w of row i: box 32 w + j overlaps box i by more than nms_iou
__global__ void __launch_bounds__(kSelThreads)
select_iou_mask_kernel(const SelectDesc* __restrict__ descs, SelectArgs a) {
    const SelectDesc d = descs[blockIdx.y];
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * kSelWarps + (threadIdx.x >> 5);
    if (i >= d.n) return;
    const float4* __restrict__ box = reinterpret_cast<const float4*>(a.dbox) + d.row0;
    const float4 bi = box[i];
    for (int w = lane; w < d.nw; w += 32) {
        unsigned bits = 0;
        for (int b = 0; b < 32; ++b) {
            const int j = w * 32 + b;
            if (j < d.n && legacy_iou(bi, box[j]) > a.nms_iou) bits |= 1u << b;
        }
        a.mask[d.mask0 + static_cast<size_t>(i) * d.nw + w] = bits;
    }
}

// Greedy NMS of classes c0 .. c0 + 7 of one image.  The block stages the classes' probabilities with row-contiguous reads (8
// adjacent logits of a row per 8 threads), then warp q sorts class c0 + q's keys (bitonic, descending) and walks them: a box not yet
// suppressed is kept, raises max_conf, and ORs its bitmask row into the suppressed set (lane l holds words l and l + 32).  Boxes
// with p <= thr (thr = max(conf_thresh, 0)) get key 0 and end the walk: they cannot raise max_conf, and the boxes they could
// suppress come after them and cannot either, so stopping there is exact.
__global__ void __launch_bounds__(kSelThreads)
select_class_nms_kernel(const SelectDesc* __restrict__ descs, SelectArgs a) {
    extern __shared__ unsigned long long s_keys[];
    const SelectDesc d = descs[blockIdx.y];
    const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
    const int c0 = a.start + blockIdx.x * kSelWarps;
    const float2* __restrict__ stats = a.stats + d.row0;
    for (int e = threadIdx.x; e < d.npad * kSelWarps; e += kSelThreads) {
        const int r = e / kSelWarps, cq = e % kSelWarps, c = c0 + cq;
        unsigned long long key = 0;
        if (r < d.n && c < a.C) {
            const float2 st = stats[r];
            const float p = expf(d.scores[static_cast<size_t>(r) * a.C + c] - st.x) / st.y;
            if (p > a.thr) key = sel_key(p, r);
        }
        s_keys[cq * d.npad + r] = key;
    }
    __syncthreads();
    if (c0 + q >= a.C) return;
    unsigned long long* keys = s_keys + q * d.npad;
    for (int k = 2; k <= d.npad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < d.npad; i += 32) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = keys[i], y = keys[ixj];
                    if (((i & k) == 0) ? (x < y) : (x > y)) { keys[i] = y; keys[ixj] = x; }
                }
            }
            __syncwarp();
        }
    }
    unsigned sup0 = 0, sup1 = 0;
    unsigned* __restrict__ max_conf = a.max_conf + d.row0;
    const unsigned* __restrict__ mask = a.mask + d.mask0;
    for (int base = 0; base < d.n; base += 32) {
        const unsigned long long mine = keys[base + lane];
        bool done = false;
        for (int t = 0; t < 32; ++t) {
            const unsigned long long kk = __shfl_sync(0xffffffffu, mine, t);
            if ((kk >> 32) == 0) { done = true; break; }
            const int j = key_index(kk), w = j >> 5;
            const unsigned word = __shfl_sync(0xffffffffu, (w >> 5) ? sup1 : sup0, w & 31);
            if ((word >> (j & 31)) & 1u) continue;
            if (lane == 0) atomicMax(max_conf + j, static_cast<unsigned>(kk >> 32));
            const unsigned* mrow = mask + static_cast<size_t>(j) * d.nw;
            if (lane < d.nw) sup0 |= mrow[lane];
            if (lane + 32 < d.nw) sup1 |= mrow[lane + 32];
        }
        if (done) break;
    }
}

// One CTA per image: rank the n max_conf values (desc, index asc; zeros rank by index too), keep the first k.
__global__ void __launch_bounds__(kRankThreads)
select_rank_kernel(const SelectDesc* __restrict__ descs, SelectArgs a) {
    __shared__ unsigned long long keys[kSelectMaxProposals];
    const SelectDesc d = descs[blockIdx.x];
    const int tid = threadIdx.x;
    for (int r = tid; r < d.npad; r += kRankThreads)
        keys[r] = r < d.n ? ((static_cast<unsigned long long>(a.max_conf[d.row0 + r]) << 32) | (0xffffffffu - static_cast<unsigned>(r)))
                          : 0ull;
    __syncthreads();
    for (int k = 2; k <= d.npad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < d.npad; i += kRankThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = keys[i], y = keys[ixj];
                    if (((i & k) == 0) ? (x < y) : (x > y)) { keys[i] = y; keys[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
    // kept rank r = r0 + tid, kRankThreads at a time (k may exceed the block: up to 1023 boxes)
    int nonzero = 0;
    for (int r0 = 0; r0 < d.k; r0 += kRankThreads) {
        const int r = r0 + tid;
        const bool on = r < d.k;
        const unsigned long long kk = on ? keys[r] : 0ull;
        nonzero += __syncthreads_count(on && (kk >> 32) != 0);
        if (!on) continue;
        const int j = key_index(kk);
        const size_t o = static_cast<size_t>(d.dst_row) + r;
        a.keep[static_cast<size_t>(blockIdx.x) * a.K + r] = j;
        if (a.keep_index) a.keep_index[o] = j;
        if (a.max_conf_out) a.max_conf_out[o] = __uint_as_float(static_cast<unsigned>(kk >> 32));
        reinterpret_cast<float4*>(a.boxes)[o] = reinterpret_cast<const float4*>(a.dbox)[d.row0 + j];
    }
    if (tid == 0) a.num_boxes[blockIdx.x] = nonzero;
}

// One CTA per output row: the kept proposal's feature row (16-byte copies), and with cls_prob / objects its probability row and
// the first column of its maximum.
__global__ void __launch_bounds__(kSelThreads)
select_gather_kernel(const SelectDesc* __restrict__ descs, SelectArgs a) {
    __shared__ unsigned long long s_best[kSelWarps];
    const SelectDesc d = descs[blockIdx.y];
    const int r = blockIdx.x;
    if (r >= d.k) return;
    const int j = a.keep[static_cast<size_t>(blockIdx.y) * a.K + r];
    const size_t o = static_cast<size_t>(d.dst_row) + r;
    const float4* __restrict__ src = reinterpret_cast<const float4*>(d.features + static_cast<size_t>(j) * a.F);
    float4* __restrict__ dst = reinterpret_cast<float4*>(a.box_features + o * a.F);
    for (int v = threadIdx.x; v < a.F / 4; v += kSelThreads) dst[v] = src[v];
    if (a.cls_prob == nullptr && a.objects == nullptr) return;
    const float2 st = a.stats[d.row0 + j];
    const float* __restrict__ x = d.scores + static_cast<size_t>(j) * a.C;
    float* prow = a.cls_prob ? a.cls_prob + o * a.C : nullptr;
    unsigned long long best = 0;
    for (int c = threadIdx.x; c < a.C; c += kSelThreads) {
        const float p = expf(x[c] - st.x) / st.y;
        if (prow) prow[c] = p;
        const unsigned long long key = sel_key(p, c);
        best = key > best ? key : best;
    }
    if (a.objects == nullptr) return;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, s);
        best = w > best ? w : best;
    }
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kSelWarps; ++w) best = s_best[w] > best ? s_best[w] : best;
        a.objects[o] = key_index(best);
    }
}

size_t select_nms_smem(int npad) { return static_cast<size_t>(kSelWarps) * npad * sizeof(unsigned long long); }

cudaError_t launch_select_regions(const SelectDesc* descs, int n, int max_n, int max_npad, const SelectArgs& a, cudaStream_t st) {
    const int row_blocks = (max_n + kSelWarps - 1) / kSelWarps;
    cudaError_t e = launch_ex(select_row_stats_kernel, dim3(row_blocks, n), dim3(kSelThreads), 0, 0, st, descs, a);
    if (e != cudaSuccess) return e;
    e = launch_ex(select_iou_mask_kernel, dim3(row_blocks, n), dim3(kSelThreads), 0, 0, st, descs, a);
    if (e != cudaSuccess) return e;
    const size_t smem = select_nms_smem(max_npad);
    e = set_smem(select_class_nms_kernel, smem);
    if (e != cudaSuccess) return e;
    const int class_blocks = (a.C - a.start + kSelWarps - 1) / kSelWarps;
    e = launch_ex(select_class_nms_kernel, dim3(class_blocks, n), dim3(kSelThreads), smem, 0, st, descs, a);
    if (e != cudaSuccess) return e;
    e = launch_ex(select_rank_kernel, dim3(n), dim3(kRankThreads), 0, 0, st, descs, a);
    if (e != cudaSuccess) return e;
    return launch_ex(select_gather_kernel, dim3(a.K, n), dim3(kSelThreads), 0, 0, st, descs, a);
}

}  // namespace vb
