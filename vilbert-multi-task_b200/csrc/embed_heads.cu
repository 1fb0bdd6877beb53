// K2 text embeddings, K1 image-operand pack, K8 narrow heads.  HBM / latency bound CUDA-core kernels:
// coalesced 16-byte accesses, one warp per output row, fp32 statistics.
//
// Replaces BertEmbeddings (3 gathers + cat + LayerNorm), the input side of BertImageEmbeddings and the
// 1-/3-wide nn.Linear heads (vil_logit, vil_tri_prediction, vision_logit, linguisic_logit, the last layer of
// vil_binary_prediction) of [UPSTREAM] vilbert/vilbert.py; anchors worker.py:286-289, 416-419, 452-455.
#include "kernels.h"

namespace vb {

constexpr int kMaxVec = 8;   // hidden <= 1024 (float4 per lane per 128 columns)

__global__ void __launch_bounds__(128)
text_embed_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ seg,
                  const int64_t* __restrict__ input_mask, const int64_t* __restrict__ task,
                  const float* __restrict__ word, const float* __restrict__ pos, const float* __restrict__ type,
                  const float* __restrict__ task_tab, const float* __restrict__ gamma, const float* __restrict__ beta,
                  float eps, float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16,
                  float* __restrict__ mask_add, int B, int Tin, int H, int vocab, int max_pos, int n_type, int n_task,
                  int task_tokens, int f16, int split16, const int* __restrict__ offs, int rows) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    int b, t, in0;                                                // sample, position in it, first input token of the sample
    if (offs == nullptr) {
        const int T = Tin + (task_tokens ? 1 : 0);
        b = row / T; t = row % T; in0 = b * Tin;
    } else {                                                      // packed batch: the sample whose rows [offs[b], offs[b+1]) hold `row`
        int lo = 0, hi = B - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (offs[mid] <= row) lo = mid; else hi = mid - 1; }
        b = lo; t = row - offs[b]; in0 = offs[b] - (task_tokens ? b : 0);
    }
    const int nvec = H / 128;

    // which source token does output position t carry?  [CLS], <task>, tok1, tok2, ...
    const bool is_task = task_tokens && t == 1;
    const int src = (task_tokens && t >= 2) ? t - 1 : t;          // index into the Tin-long inputs
    float4 x[kMaxVec];
    if (is_task) {
        long long tid = task[b];
        tid = tid < 0 ? 0 : (tid >= n_task ? n_task - 1 : tid);
        const float4* tp = reinterpret_cast<const float4*>(task_tab + tid * H);
#pragma unroll
        for (int k = 0; k < kMaxVec; ++k) if (k < nvec) x[k] = tp[lane + 32 * k];
    } else {
        long long id = ids[in0 + src];
        long long sg = seg[in0 + src];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        sg = sg < 0 ? 0 : (sg >= n_type ? n_type - 1 : sg);
        const int ps = src < max_pos ? src : max_pos - 1;
        const float4* wp = reinterpret_cast<const float4*>(word + id * H);
        const float4* pp = reinterpret_cast<const float4*>(pos + static_cast<size_t>(ps) * H);
        const float4* sp = reinterpret_cast<const float4*>(type + sg * H);
#pragma unroll
        for (int k = 0; k < kMaxVec; ++k) {
            if (k < nvec) {
                const float4 a = wp[lane + 32 * k], c = pp[lane + 32 * k], d = sp[lane + 32 * k];
                x[k] = make_float4(a.x + c.x + d.x, a.y + c.y + d.y, a.z + c.z + d.z, a.w + c.w + d.w);
            }
        }
    }
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < kMaxVec; ++k) if (k < nvec) s += x[k].x + x[k].y + x[k].z + x[k].w;
    const float mean = warp_sum(s) / static_cast<float>(H);
    float sq = 0.0f;
#pragma unroll
    for (int k = 0; k < kMaxVec; ++k) {
        if (k < nvec) {
            const float a = x[k].x - mean, c = x[k].y - mean, d = x[k].z - mean, e = x[k].w - mean;
            sq += a * a + c * c + d * d + e * e;
        }
    }
    const float rstd = 1.0f / sqrtf(warp_sum(sq) / static_cast<float>(H) + eps);
    float4* of = reinterpret_cast<float4*>(out_f32 + static_cast<size_t>(row) * H);
    uint2* ob = reinterpret_cast<uint2*>(out_bf16 + static_cast<size_t>(row) * (split16 ? 3 * H : H));
    const float4* gp = reinterpret_cast<const float4*>(gamma);
    const float4* bp = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int k = 0; k < kMaxVec; ++k) {
        if (k < nvec) {
            const float4 g = gp[lane + 32 * k], be = bp[lane + 32 * k];
            float4 y;
            y.x = (x[k].x - mean) * rstd * g.x + be.x;
            y.y = (x[k].y - mean) * rstd * g.y + be.y;
            y.z = (x[k].z - mean) * rstd * g.z + be.z;
            y.w = (x[k].w - mean) * rstd * g.w + be.w;
            of[lane + 32 * k] = y;
            if (split16) {             // fp32-parity mode: fp16 hi | lo | hi per 64 columns (common.cuh split_col)
                uint2* o3 = ob + split_col(4 * (lane + 32 * k)) / 4;
                const uint2 hi = make_uint2(pack16x2_rt(y.x, y.y, 1), pack16x2_rt(y.z, y.w, 1));
                o3[0] = hi;
                o3[16] = make_uint2(pack16x2_rt(split_lo(y.x), split_lo(y.y), 1), pack16x2_rt(split_lo(y.z), split_lo(y.w), 1));
                o3[32] = hi;
            } else {
                ob[lane + 32 * k] = make_uint2(pack16x2_rt(y.x, y.y, f16), pack16x2_rt(y.z, y.w, f16));
            }
        }
    }
    if (lane == 0) {
        // [UPSTREAM] BertModel.forward prepends a 1 to the mask when task tokens are on:
        //   ext_mask[0] = 1, ext_mask[t] = input_mask[t - 1] for t >= 1
        // (position 1, the task row, therefore carries input_mask[0], the [CLS] flag).
        // packed batches have no padding: every row's flag is 1
        const float m = offs != nullptr ? 1.0f
                                        : task_tokens ? (t == 0 ? 1.0f : static_cast<float>(input_mask[in0 + (t - 1)]))
                                                      : static_cast<float>(input_mask[in0 + t]);
        mask_add[row] = (1.0f - m) * -10000.0f;
    }
}

// one block per (sample, region) row; F % 8 == 0, Kp % 8 == 0, Kp >= F + 8
__global__ void __launch_bounds__(256)
image_pack_kernel(const float* __restrict__ feats, const float* __restrict__ loc, const uint8_t* __restrict__ image_mask,
                  __nv_bfloat16* __restrict__ a_out, float* __restrict__ mask_add, int F, int Kp, int f16, int split16) {
    const int row = blockIdx.x;
    const float4* src = reinterpret_cast<const float4*>(feats + static_cast<size_t>(row) * F);
    uint4* dst = reinterpret_cast<uint4*>(a_out + static_cast<size_t>(row) * (split16 ? 3 * Kp : Kp));
    const int nvec = F / 8;
    // 8 columns [8i, 8i+8) -> one 16-byte store; fp32-parity mode: fp16 hi | lo | hi per 64 columns (split_col), three stores
    auto put = [&](int i, float a0, float a1, float a2, float a3, float b0, float b1, float b2, float b3) {
        uint4 u;
        u.x = pack16x2_rt(a0, a1, f16); u.y = pack16x2_rt(a2, a3, f16);
        u.z = pack16x2_rt(b0, b1, f16); u.w = pack16x2_rt(b2, b3, f16);
        if (!split16) { dst[i] = u; return; }
        uint4* d3 = dst + split_col(8 * i) / 8;
        uint4 l;
        l.x = pack16x2_rt(split_lo(a0), split_lo(a1), 1); l.y = pack16x2_rt(split_lo(a2), split_lo(a3), 1);
        l.z = pack16x2_rt(split_lo(b0), split_lo(b1), 1); l.w = pack16x2_rt(split_lo(b2), split_lo(b3), 1);
        d3[0] = u; d3[8] = l; d3[16] = u;
    };
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const float4 a = __ldg(src + 2 * i), b = __ldg(src + 2 * i + 1);   // streamed once
        put(i, a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
    }
    const int tail_vec = (Kp - F) / 8;
    if (threadIdx.x < tail_vec) {
        if (threadIdx.x == 0) {
            const float* l = loc + static_cast<size_t>(row) * 5;
            put(nvec, l[0], l[1], l[2], l[3], l[4], 0.0f, 0.0f, 0.0f);
        } else {
            put(nvec + threadIdx.x, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f);
        }
    }
    if (threadIdx.x == 0) mask_add[row] = (1.0f - (image_mask ? static_cast<float>(image_mask[row]) : 1.0f)) * -10000.0f;
}

// custom_prediction()'s input builder on the device (worker.py:422-455): per image, the detector's n box features [n, F] become the
// GEMM operand rows [global mean row | box rows] (fp32 -> 16-bit, straight into the image-embedding GEMM's A buffer -- the fp32
// [n+1, F] tensor the reference builds with cat/stack is never materialised), pixel boxes become the 5-d normalised locations
// (x1/w, y1/h, x2/w, y2/h, area/(w h); global row 0,0,1,1,1), masks are set.  num_boxes (optional) marks padded boxes per image:
// they are excluded from the mean, written as zeros and masked.
// grid (B, ceil(F / 1024) + 1): the last grid row writes the location columns, the masks and the optional spatials copy.
// Packed batch (offs = the plan's image row offsets [B + 1]): image b owns regions [offs[b], offs[b+1]) -- its mean row, then its
// offs[b+1] - offs[b] - 1 boxes, which start at detector row offs[b] - b (one global row per image) -- every row is real, and
// spatials_out is packed [sum V_i, 5].  With src (the ablation calls), output image b is instead source image src[b].image's boxes
// named by its kept list (kept + src[b].kept, detector rows relative to src[b].box0, in order; src[b].kept = -1: every box): the
// mean sums the kept boxes in the order any image's boxes are summed, so the rows are those of the reduced image packed alone.
// No kept box gives the global row alone (zero features, location [0, 0, 1, 1, 1]).
__global__ void __launch_bounds__(128)
region_pack_kernel(const float* __restrict__ box_feats, const float* __restrict__ boxes, const float* __restrict__ image_wh,
                   const int32_t* __restrict__ num_boxes, __nv_bfloat16* __restrict__ a_out, float* __restrict__ mask_add,
                   float* __restrict__ spatials_out, int n, int F, int Kp, int f16, int split16, const int* __restrict__ offs,
                   const RegionSrc* __restrict__ src_img, const int32_t* __restrict__ kept) {
    const int b = blockIdx.x;
    int row0, box0, nb, img = b;                                     // first operand row, first detector row, valid boxes, source image
    const int32_t* rows = nullptr;                                   // kept detector rows (relative to box0), null: every box in order
    if (offs == nullptr) {
        row0 = b * (n + 1); box0 = b * n;
        nb = num_boxes ? num_boxes[b] : n;
        nb = nb < 0 ? 0 : (nb > n ? n : nb);
    } else {
        row0 = offs[b]; box0 = row0 - b;
        n = nb = offs[b + 1] - row0 - 1;
        if (src_img != nullptr) {
            const RegionSrc s = src_img[b];
            img = s.image; box0 = s.box0;
            if (s.kept >= 0) rows = kept + s.kept;
        }
    }
    // detector row of output box r
    auto det_row = [&](int r) { return static_cast<size_t>(box0) + (rows != nullptr ? rows[r] : r); };
    const int V = n + 1;
    const size_t ld = static_cast<size_t>(split16 ? 3 * Kp : Kp);
    auto put = [&](int row, int i, const float (&x)[8]) {           // 8 columns [8i, 8i+8) of operand row `row`
        uint4* dst = reinterpret_cast<uint4*>(a_out + static_cast<size_t>(row) * ld);
        uint4 u;
        u.x = pack16x2_rt(x[0], x[1], f16); u.y = pack16x2_rt(x[2], x[3], f16);
        u.z = pack16x2_rt(x[4], x[5], f16); u.w = pack16x2_rt(x[6], x[7], f16);
        if (!split16) { dst[i] = u; return; }
        uint4* d3 = dst + split_col(8 * i) / 8;
        uint4 l;
        l.x = pack16x2_rt(split_lo(x[0]), split_lo(x[1]), 1); l.y = pack16x2_rt(split_lo(x[2]), split_lo(x[3]), 1);
        l.z = pack16x2_rt(split_lo(x[4]), split_lo(x[5]), 1); l.w = pack16x2_rt(split_lo(x[6]), split_lo(x[7]), 1);
        d3[0] = u; d3[8] = l; d3[16] = u;
    };
    if (blockIdx.y + 1 < gridDim.y) {
        const int i = blockIdx.y * blockDim.x + threadIdx.x;           // 8-column group
        if (i * 8 >= F) return;
        float sum[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        for (int r = 0; r < n; ++r) {
            float x[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
            if (r < nb) {
                const float* src = box_feats + det_row(r) * F + i * 8;
                const float4 a = __ldg(reinterpret_cast<const float4*>(src));
                const float4 c = __ldg(reinterpret_cast<const float4*>(src) + 1);
                x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = c.x; x[5] = c.y; x[6] = c.z; x[7] = c.w;
#pragma unroll
                for (int j = 0; j < 8; ++j) sum[j] += x[j];
            }
            put(row0 + r + 1, i, x);
        }
        const float cnt = static_cast<float>(nb > 0 ? nb : 1);
#pragma unroll
        for (int j = 0; j < 8; ++j) sum[j] = sum[j] / cnt;              // torch.sum(feature, dim=0) / num_boxes (worker.py:432)
        put(row0, i, sum);
        return;
    }
    const float w = image_wh[2 * img], h = image_wh[2 * img + 1];
    const float wh = static_cast<float>(static_cast<double>(w) * static_cast<double>(h));     // float(image_w) * float(image_h)
    const int tail_groups = (Kp - F) / 8;
    for (int r = threadIdx.x; r < V; r += blockDim.x) {
        float loc[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        const bool real = r == 0 || r - 1 < nb;
        if (r == 0) { loc[2] = loc[3] = loc[4] = 1.0f; }               // g_location = [0, 0, 1, 1, 1] (worker.py:443)
        else if (real) {
            const float* bx = boxes + det_row(r - 1) * 4;
            const float x1 = bx[0], y1 = bx[1], x2 = bx[2], y2 = bx[3];
            loc[4] = (y2 - y1) * (x2 - x1) / wh;                       // computed before the coordinates are normalised (worker.py:438)
            loc[0] = x1 / w; loc[1] = y1 / h; loc[2] = x2 / w; loc[3] = y2 / h;
        }
        const float zero[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        for (int g = 0; g < tail_groups; ++g) {
            if (g == 0) put(row0 + r, F / 8, loc); else put(row0 + r, F / 8 + g, zero);
        }
        mask_add[row0 + r] = real ? 0.0f : -10000.0f;
        if (spatials_out)
            for (int j = 0; j < 5; ++j) spatials_out[(static_cast<size_t>(row0) + r) * 5 + j] = loc[j];
    }
}

// Retrieval reuse: row block `idx[b]` of a cached per-caption / per-image encoder state -> sample b of the pair plan's buffers
// (fp32 residual stream, 16-bit GEMM operand, additive mask).  One CTA per destination sample; 16-byte copies.
__global__ void __launch_bounds__(256)
gather_state_kernel(const int32_t* __restrict__ idx, int n_src, const float* __restrict__ src_f32, const uint16_t* __restrict__ src_16,
                    const float* __restrict__ src_mask, float* __restrict__ dst_f32, uint16_t* __restrict__ dst_16,
                    float* __restrict__ dst_mask, int L, int n32 /* uint4 per sample, fp32 */, int n16 /* uint4 per sample, 16-bit */) {
    const int b = blockIdx.x;
    int s = idx[b];
    s = s < 0 ? 0 : (s >= n_src ? n_src - 1 : s);
    if (src_f32 != nullptr) {
        const uint4* a = reinterpret_cast<const uint4*>(src_f32) + static_cast<size_t>(s) * n32;
        uint4* d = reinterpret_cast<uint4*>(dst_f32) + static_cast<size_t>(b) * n32;
        for (int i = threadIdx.x; i < n32; i += blockDim.x) d[i] = a[i];
    }
    const uint4* a2 = reinterpret_cast<const uint4*>(src_16) + static_cast<size_t>(s) * n16;
    uint4* d2 = reinterpret_cast<uint4*>(dst_16) + static_cast<size_t>(b) * n16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) d2[i] = a2[i];
    if (src_mask != nullptr)
        for (int i = threadIdx.x; i < L; i += blockDim.x) dst_mask[static_cast<size_t>(b) * L + i] = src_mask[static_cast<size_t>(s) * L + i];
}

// Packed retrieval: pair b's cached rows [src[b], src[b] + dst[b+1] - dst[b]) of a packed caption / image state -> rows
// [dst[b], dst[b+1]) of the pair plan's buffers (fp32 residual stream and 16-bit GEMM operand).  grid (B, 2): y = 0 text, 1 image;
// one contiguous range per CTA, 16-byte copies.
__device__ __forceinline__ void copy_packed_rows(const PackedStateCopy& c, int b) {
    const int d0 = c.dst_offs[b], rows = c.dst_offs[b + 1] - d0, s0 = c.src_offs[b];
    const size_t n32 = static_cast<size_t>(rows) * c.n32, n16 = static_cast<size_t>(rows) * c.n16;
    const uint4* a = reinterpret_cast<const uint4*>(c.src_f32) + static_cast<size_t>(s0) * c.n32;
    uint4* d = reinterpret_cast<uint4*>(c.dst_f32) + static_cast<size_t>(d0) * c.n32;
    for (size_t i = threadIdx.x; i < n32; i += blockDim.x) d[i] = a[i];
    const uint4* a2 = static_cast<const uint4*>(c.src_16) + static_cast<size_t>(s0) * c.n16;
    uint4* d2 = static_cast<uint4*>(c.dst_16) + static_cast<size_t>(d0) * c.n16;
    for (size_t i = threadIdx.x; i < n16; i += blockDim.x) d2[i] = a2[i];
}
__global__ void __launch_bounds__(256)
gather_packed_state_kernel(PackedStateCopy text, PackedStateCopy image) {
    if (blockIdx.y == 0) copy_packed_rows(text, blockIdx.x);
    else copy_packed_rows(image, blockIdx.x);
}

// Pre-training heads at chosen rows (vb200_pretraining_heads): row rows[i] of a forward's fp32 final state -> row i of the heads'
// compact operand.  The 16-bit forms are what ln_residual_kernel writes as the final LayerNorm's operand from the same fp32 value
// (pack16x2<F16>, or in fp32-parity mode the hi | lo | hi split through pack16x2_rt and split_lo), so every head row sees the bits the
// forward's full-row heads see.  MODE 0 bf16, 1 fp16, 2 fp16 hi | lo | hi, 3 fp32 copy (the pooled rows of the alignment head).
// Rows [n, rows_out) -- the rest of the last 128-row GEMM tile -- are zeroed.  One thread per 8 columns: two 16-byte loads, one
// 16-byte store per copy.
template <int MODE>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ rows, int n, int rows_out, int H, void* __restrict__ dst,
                   int ld_dst) {
    const int per_row = H >> 3;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = t / per_row, c = (t - r * per_row) * 8;
    if (r >= rows_out) return;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (r < n) {
        const float4* s = reinterpret_cast<const float4*>(src + static_cast<size_t>(rows[r]) * H + c);
        a = s[0];
        b = s[1];
    }
    if constexpr (MODE == 3) {
        float4* d = reinterpret_cast<float4*>(static_cast<float*>(dst) + static_cast<size_t>(r) * ld_dst + c);
        d[0] = a;
        d[1] = b;
    } else if constexpr (MODE == 2) {
        uint4* d = reinterpret_cast<uint4*>(static_cast<uint16_t*>(dst) + static_cast<size_t>(r) * ld_dst + split_col(c));
        const uint4 hi = make_uint4(pack16x2_rt(a.x, a.y, 1), pack16x2_rt(a.z, a.w, 1), pack16x2_rt(b.x, b.y, 1), pack16x2_rt(b.z, b.w, 1));
        d[0] = hi;
        d[8] = make_uint4(pack16x2_rt(split_lo(a.x), split_lo(a.y), 1), pack16x2_rt(split_lo(a.z), split_lo(a.w), 1),
                          pack16x2_rt(split_lo(b.x), split_lo(b.y), 1), pack16x2_rt(split_lo(b.z), split_lo(b.w), 1));
        d[16] = hi;
    } else {
        constexpr bool F16 = MODE == 1;
        uint4* d = reinterpret_cast<uint4*>(static_cast<uint16_t*>(dst) + static_cast<size_t>(r) * ld_dst + c);
        d[0] = make_uint4(pack16x2<F16>(a.x, a.y), pack16x2<F16>(a.z, a.w), pack16x2<F16>(b.x, b.y), pack16x2<F16>(b.z, b.w));
    }
}

// Pre-training objectives (vb200_pretraining_objectives): one CTA per listed row of the three heads' compact logits, in list order
// text | image | pair.  With z the row's logits, m = max z and s = sum exp(z - m), log_softmax(z)_c = (z_c - m) - log s:
//   token / pair row: cross-entropy log s - (z_label - m);
//   image row: KL(t || softmax z) = sum_c xlogy(t_c, t_c) - t_c log_softmax(z)_c (0 log 0 = 0), as torch.nn.functional.kl_div.
// Each thread takes the columns tid, tid + 256, ... and the partial sums meet in a fixed shuffle tree, so a row's loss has the same
// bits on every call.
constexpr int kLossThreads = 256, kLossWarps = kLossThreads / 32;
template <bool MAX>
__device__ __forceinline__ float loss_block_reduce(float v, float* s_f) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = MAX ? warp_max(v) : warp_sum(v);
    if (lane == 0) s_f[warp] = v;
    __syncthreads();
    const float w = lane < kLossWarps ? s_f[lane] : (MAX ? -INFINITY : 0.f);
    v = MAX ? warp_max(w) : warp_sum(w);
    __syncthreads();                                      // s_f is reused by the next reduction
    return v;
}

// row r of list g (inlined once per list, so every field is read from the kernel parameters directly)
__device__ __forceinline__ void loss_row(const LossRows& g, int r, float* s_f) {
    const float* __restrict__ z = g.logits + static_cast<size_t>(r) * g.ld;
    const int tid = threadIdx.x;
    float m = -INFINITY;
    for (int c = tid; c < g.N; c += kLossThreads) m = fmaxf(m, z[c]);
    m = loss_block_reduce<true>(m, s_f);
    float s = 0.f;
    for (int c = tid; c < g.N; c += kLossThreads) s += expf(z[c] - m);
    const float log_s = logf(loss_block_reduce<false>(s, s_f));
    float loss;
    if (g.targets != nullptr) {
        const float* __restrict__ tr = g.targets + static_cast<size_t>(r) * g.N;
        float k = 0.f;
        for (int c = tid; c < g.N; c += kLossThreads) {
            const float tc = tr[c];
            k += (tc == 0.f ? 0.f : tc * logf(tc)) - tc * ((z[c] - m) - log_s);
        }
        loss = loss_block_reduce<false>(k, s_f);
    } else {
        loss = log_s - (z[g.labels[r]] - m);
    }
    if (tid == 0) g.loss[r] = loss;
}

__global__ void __launch_bounds__(kLossThreads)
pretrain_loss_rows_kernel(LossRows t, LossRows v, LossRows p) {
    __shared__ float s_f[kLossWarps];
    const int r = blockIdx.x;
    if (r < t.n) loss_row(t, r, s_f);
    else if (r < t.n + v.n) loss_row(v, r - t.n, s_f);
    else loss_row(p, r - t.n - v.n, s_f);
}

// The reduced objectives: reduced[k] = (sum of list k's row losses) / n_k, summed in double in a fixed order by one CTA; an empty list
// gives 0 / 0 = NaN.
__device__ __forceinline__ void loss_mean(const LossRows& g, float* out, double* s_d) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double a = 0.0;
    for (int i = tid; i < g.n; i += 1024) a += static_cast<double>(g.loss[i]);
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) s_d[warp] = a;
    __syncthreads();
    if (warp == 0) {
        a = s_d[lane];
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) *out = static_cast<float>(a / static_cast<double>(g.n));
    }
    __syncthreads();
}

__global__ void __launch_bounds__(1024)
pretrain_loss_reduce_kernel(LossRows t, LossRows v, LossRows p, float* __restrict__ reduced) {
    __shared__ double s_d[32];
    loss_mean(t, reduced, s_d);
    loss_mean(v, reduced + 1, s_d);
    loss_mean(p, reduced + 2, s_d);
}

// one warp per row; n_out <= 4
__global__ void __launch_bounds__(128)
rowdot_kernel(const float* __restrict__ x, int ld_x, const float* __restrict__ W, const float* __restrict__ bias,
              const float* __restrict__ add, float* __restrict__ out, int ld_out, int M, int K, int n_out, int pdl,
              const int* __restrict__ m_rows) {
    if (pdl) { pdl_wait(); pdl_launch_dependents(); }
    const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (m >= M || (m_rows != nullptr && m >= *m_rows)) return;       // packed batches: rows past the device row count
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    const float4* xp = reinterpret_cast<const float4*>(x + static_cast<size_t>(m) * ld_x);
    for (int k = lane; k < K / 4; k += 32) {
        const float4 a = xp[k];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (j < n_out) {
                const float4 w = __ldg(reinterpret_cast<const float4*>(W + static_cast<size_t>(j) * K) + k);
                acc[j] += a.x * w.x + a.y * w.y + a.z * w.z + a.w * w.w;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = warp_sum(acc[j]);
    if (lane == 0) {
        const float extra = add ? add[m] : 0.0f;
        for (int j = 0; j < n_out; ++j) out[static_cast<size_t>(m) * ld_out + j] = acc[j] + (bias ? bias[j] : 0.0f) + extra;
    }
}

// Layer states: REDUCE 0 copies rows with a grid-stride loop of 16-byte accesses, 1 one CTA per sample copies its first row, 2 one
// CTA per (sample, 128 columns) where each thread owns one column and walks the sample's rows in order.  Every launch waits for the
// op that wrote src before looking at the destination, so the dependents of a launch that writes nothing still see that op's rows.
constexpr int kStateThreads = 128;
template <int REDUCE>
__global__ void __launch_bounds__(kStateThreads)
layer_state_kernel(StateArgs a, int pdl) {
    if (pdl) { pdl_wait(); pdl_launch_dependents(); }
    float* dst = reinterpret_cast<float*>(static_cast<uintptr_t>(a.dst[0]));
    if (dst == nullptr) return;
    const int b = blockIdx.x;
    if constexpr (REDUCE == 0) {
        const int rows = a.offs != nullptr ? *a.m_rows : a.B * a.L;
        const int64_t n4 = static_cast<int64_t>(rows) * (a.H / 4);
        const float4* src = reinterpret_cast<const float4*>(a.src);
        float4* out = reinterpret_cast<float4*>(dst);
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
            out[i] = src[i];
    } else if constexpr (REDUCE == 1) {
        const int64_t row = a.offs != nullptr ? a.offs[b] : static_cast<int64_t>(b) * a.L;
        const float4* src = reinterpret_cast<const float4*>(a.src + row * a.H);
        float4* out = reinterpret_cast<float4*>(dst + static_cast<int64_t>(b) * a.H);
        for (int c = threadIdx.x; c < a.H / 4; c += blockDim.x) out[c] = src[c];
    } else {
        const int col = blockIdx.y * kStateThreads + threadIdx.x;
        if (col >= a.H) return;
        const int r0 = a.offs != nullptr ? a.offs[b] : b * a.L;
        const int r1 = a.offs != nullptr ? a.offs[b + 1] : r0 + a.L;
        float sum = 0.0f;
        int count = 0;
        for (int r = r0; r < r1; ++r) {
            if (a.mask != nullptr && a.mask[r] != 0.0f) continue;
            sum = __fadd_rn(sum, a.src[static_cast<int64_t>(r) * a.H + col]);
            ++count;
        }
        dst[static_cast<int64_t>(b) * a.H + col] = count > 0 ? __fdiv_rn(sum, static_cast<float>(count)) : __int_as_float(0x7fc00000);
    }
}

cudaError_t launch_layer_state(const StateArgs& a, int pdl, cudaStream_t st) {
    if (a.B < 1 || a.L < 1 || a.H < 4 || a.H % 4 != 0 || a.dst == nullptr || (a.offs != nullptr) != (a.m_rows != nullptr) ||
        (reinterpret_cast<uintptr_t>(a.src) & 15) || a.reduce < 0 || a.reduce > 2)
        return cudaErrorInvalidValue;
    const dim3 block(kStateThreads);
    if (a.reduce == 0) {
        const int64_t n4 = static_cast<int64_t>(a.B) * a.L * (a.H / 4);
        const dim3 grid(static_cast<unsigned>(std::min<int64_t>((n4 + kStateThreads - 1) / kStateThreads, 2048)));
        return launch_ex(layer_state_kernel<0>, grid, block, 0, pdl, st, a, pdl);
    }
    if (a.reduce == 1) return launch_ex(layer_state_kernel<1>, dim3(a.B), block, 0, pdl, st, a, pdl);
    return launch_ex(layer_state_kernel<2>, dim3(a.B, (a.H + kStateThreads - 1) / kStateThreads), block, 0, pdl, st, a, pdl);
}

cudaError_t launch_text_embed(const int64_t* ids, const int64_t* seg, const int64_t* input_mask, const int64_t* task,
                              const float* word, const float* pos, const float* type, const float* task_tab,
                              const float* gamma, const float* beta, float eps, float* out_f32,
                              __nv_bfloat16* out_bf16, float* mask_add, int B, int Tin, int H, int vocab, int max_pos,
                              int n_type, int n_task, int task_tokens, int f16, int split16, cudaStream_t st,
                              const int* offs, int rows) {
    if (H % 128 != 0 || H / 128 > kMaxVec || (split16 && !f16) || (offs != nullptr && (B < 1 || rows < 1))) return cudaErrorInvalidValue;
    if (offs == nullptr) rows = B * (Tin + (task_tokens ? 1 : 0));
    text_embed_kernel<<<(rows + 3) / 4, 128, 0, st>>>(ids, seg, input_mask, task, word, pos, type, task_tab, gamma, beta,
                                                      eps, out_f32, out_bf16, mask_add, B, Tin, H, vocab, max_pos,
                                                      n_type, n_task, task_tokens, f16, split16, offs, rows);
    return cudaGetLastError();
}

cudaError_t launch_image_pack(const float* feats, const float* loc, const uint8_t* image_mask, __nv_bfloat16* a_out,
                              float* mask_add, int rows, int F, int Kp, int f16, int split16, cudaStream_t st) {
    if (F % 8 != 0 || Kp % 8 != 0 || Kp < F + 8 || (Kp - F) / 8 > 256 || (split16 && (!f16 || (Kp & 63)))) return cudaErrorInvalidValue;
    image_pack_kernel<<<rows, 256, 0, st>>>(feats, loc, image_mask, a_out, mask_add, F, Kp, f16, split16);
    return cudaGetLastError();
}

cudaError_t launch_region_pack(const float* box_feats, const float* boxes, const float* image_wh, const int32_t* num_boxes,
                               __nv_bfloat16* a_out, float* mask_add, float* spatials_out, int B, int n, int F, int Kp, int f16,
                               int split16, cudaStream_t st, const int* offs, const RegionSrc* src, const int32_t* kept) {
    if (B < 1 || (offs == nullptr && n < 1) || F % 8 != 0 || Kp % 8 != 0 || Kp < F + 8 || (split16 && (!f16 || (Kp & 63))) ||
        (offs != nullptr && (num_boxes != nullptr || split16)) || (src != nullptr && offs == nullptr) || (kept != nullptr && src == nullptr))
        return cudaErrorInvalidValue;
    const dim3 grid(B, (F / 8 + 127) / 128 + 1);
    region_pack_kernel<<<grid, 128, 0, st>>>(box_feats, boxes, image_wh, num_boxes, a_out, mask_add, spatials_out, n, F, Kp, f16, split16,
                                             offs, src, kept);
    return cudaGetLastError();
}

// The ablation calls' text inputs: variant k's token ids, segment ids and task id copied from its sample's single copy, every
// position whose bit is set in the call's bitmap (words from mask + masked, masked >= 0) replaced by mask_token, written where the
// packed text embedding reads variant k (offs[k] - k task_tokens).
__global__ void __launch_bounds__(128)
variant_text_kernel(const TextSrc* __restrict__ v, const int* __restrict__ offs, int task_tokens, const int64_t* __restrict__ q,
                    const int64_t* __restrict__ seg, const int64_t* __restrict__ task, int64_t mask_token, int64_t* __restrict__ q_out,
                    int64_t* __restrict__ seg_out, int64_t* __restrict__ task_out, const uint32_t* __restrict__ mask) {
    const int k = blockIdx.x;
    const TextSrc d = v[k];
    const int out0 = offs[k] - k * task_tokens;
    const uint32_t* bits = d.masked >= 0 ? mask + d.masked : nullptr;
    for (int t = threadIdx.x; t < d.len; t += blockDim.x) {
        const bool masked = bits != nullptr && ((bits[t >> 5] >> (t & 31)) & 1u);
        q_out[out0 + t] = masked ? mask_token : q[d.first + t];
        seg_out[out0 + t] = seg[d.first + t];
    }
    if (threadIdx.x == 0 && task_tokens) task_out[k] = task[d.sample];
}

cudaError_t launch_variant_text(const TextSrc* v, int n, const int* offs, int task_tokens, const int64_t* q, const int64_t* seg,
                                const int64_t* task, int64_t mask_token, int64_t* q_out, int64_t* seg_out, int64_t* task_out,
                                cudaStream_t st, const uint32_t* mask) {
    if (n < 1 || (task_tokens && (task == nullptr || task_out == nullptr))) return cudaErrorInvalidValue;
    variant_text_kernel<<<n, 128, 0, st>>>(v, offs, task_tokens, q, seg, task, mask_token, q_out, seg_out, task_out, mask);
    return cudaGetLastError();
}

// Head ablation's gate rows: row b of the [n, stride] gate table is all ones, with element zero[b] set to 0 (-1: none).  One CTA per
// row; every float of the row is written, so the table holds nothing from an earlier call.
__global__ void gate_rows_kernel(const int32_t* __restrict__ zero, int stride, float* __restrict__ gate) {
    const int b = blockIdx.x, z = zero[b];
    float* row = gate + static_cast<size_t>(b) * stride;
    for (int i = threadIdx.x; i < stride; i += blockDim.x) row[i] = i == z ? 0.0f : 1.0f;
}

cudaError_t launch_gate_rows(const int32_t* zero, int n, int stride, float* gate, cudaStream_t st) {
    if (n < 1 || stride < 1 || zero == nullptr || gate == nullptr) return cudaErrorInvalidValue;
    gate_rows_kernel<<<n, 128, 0, st>>>(zero, stride, gate);
    return cudaGetLastError();
}

cudaError_t launch_gather_state(const int32_t* idx, int n_src, const float* src_f32, const void* src_16, const float* src_mask,
                                float* dst_f32, void* dst_16, float* dst_mask, int B, int L, int H, int H16, cudaStream_t st) {
    if (B < 1 || n_src < 1 || (static_cast<long long>(L) * H) % 4 != 0 || (static_cast<long long>(L) * H16) % 8 != 0) return cudaErrorInvalidValue;
    gather_state_kernel<<<B, 256, 0, st>>>(idx, n_src, src_f32, static_cast<const uint16_t*>(src_16), src_mask, dst_f32,
                                           static_cast<uint16_t*>(dst_16), dst_mask, L, L * H / 4, L * H16 / 8);
    return cudaGetLastError();
}

cudaError_t launch_gather_packed_state(const PackedStateCopy& text, const PackedStateCopy& image, int B, cudaStream_t st) {
    if (B < 1) return cudaErrorInvalidValue;
    for (const PackedStateCopy* c : {&text, &image})
        if (c->n32 < 1 || c->n16 < 1 || (reinterpret_cast<uintptr_t>(c->src_f32) | reinterpret_cast<uintptr_t>(c->src_16) |
                                         reinterpret_cast<uintptr_t>(c->dst_f32) | reinterpret_cast<uintptr_t>(c->dst_16)) & 15)
            return cudaErrorInvalidValue;
    gather_packed_state_kernel<<<dim3(B, 2), 256, 0, st>>>(text, image);
    return cudaGetLastError();
}

cudaError_t launch_gather_rows(const float* src, const int32_t* rows, int n, int rows_out, int H, void* dst, int ld_dst, int mode,
                                cudaStream_t st) {
    if (n < 0 || rows_out < n || rows_out < 1 || H < 8 || H % 8 != 0 || mode < 0 || mode > 3 || (mode == 2 && H % 64 != 0) ||
        ld_dst % 8 != 0 || ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15))
        return cudaErrorInvalidValue;
    const int64_t threads = static_cast<int64_t>(rows_out) * (H / 8);
    const dim3 grid(static_cast<unsigned>((threads + 255) / 256)), block(256);
    switch (mode) {
        case 0: gather_rows_kernel<0><<<grid, block, 0, st>>>(src, rows, n, rows_out, H, dst, ld_dst); break;
        case 1: gather_rows_kernel<1><<<grid, block, 0, st>>>(src, rows, n, rows_out, H, dst, ld_dst); break;
        case 2: gather_rows_kernel<2><<<grid, block, 0, st>>>(src, rows, n, rows_out, H, dst, ld_dst); break;
        default: gather_rows_kernel<3><<<grid, block, 0, st>>>(src, rows, n, rows_out, H, dst, ld_dst); break;
    }
    return cudaGetLastError();
}

cudaError_t launch_pretrain_losses(const LossRows* g, float* reduced, cudaStream_t st) {
    int64_t blocks = 0;
    for (int k = 0; k < 3; ++k) {
        const LossRows& x = g[k];
        if (x.n < 0 || (x.n > 0 && (x.logits == nullptr || x.loss == nullptr || x.N < 1 || x.ld < x.N ||
                                    ((k == 1) != (x.targets != nullptr)) || ((k != 1) != (x.labels != nullptr)))))
            return cudaErrorInvalidValue;
        blocks += x.n;
    }
    if (blocks > 0x7fffffff) return cudaErrorInvalidValue;
    if (blocks > 0) pretrain_loss_rows_kernel<<<static_cast<unsigned>(blocks), kLossThreads, 0, st>>>(g[0], g[1], g[2]);
    if (reduced != nullptr) pretrain_loss_reduce_kernel<<<1, 1024, 0, st>>>(g[0], g[1], g[2], reduced);
    return cudaGetLastError();
}

cudaError_t launch_rowdot(const float* x, int ld_x, const float* W, const float* b, const float* add, float* out,
                          int ld_out, int M, int K, int n_out, int pdl, cudaStream_t st, const int* m_rows) {
    if (n_out < 1 || n_out > 4 || K % 4 != 0 || ld_x % 4 != 0) return cudaErrorInvalidValue;
    return launch_ex(rowdot_kernel, dim3((M + 3) / 4), dim3(128), 0, pdl, st, x, ld_x, W, b, add, out, ld_out, M, K,
                     n_out, pdl, m_rows);
}

}  // namespace vb
