// Internal launch interface of the vilbert_b200 sm_90a kernels (not part of the C ABI; see include/vilbert_b200.h).
#pragma once
#include "common.cuh"
#include "../../include/vilbert_b200.h"

namespace vb {

enum Act : int { kActNone = 0, kActGelu = 1, kActRelu = 2, kActGeluExact = 3 };   // 3: erf to 1.5e-7 (fp32-parity mode)

// Epilogue of the wgmma GEMM:  y = act(acc + bias) * mul.
struct GemmEpilogue {
    int M, N, K;
    const float* bias;            // [N] or null
    const float* mul;             // fp32 [M, ld_mul] multiplicand (pooled_t * pooled_v fusion) or null
    int ld_mul;
    __nv_bfloat16* out_bf16;      // optional
    int ld_bf16;
    float* out_f32;               // optional
    int ld_f32;
    int act;
    int pdl;                      // 0 = no programmatic dependent launch; 1 = LAUNCHED with programmatic stream serialization
                                  // (in-kernel griddepcontrol.wait / launch_dependents); 5 = as 1, and the producer puts the
                                  // first ring pass of WEIGHT tiles in flight before griddepcontrol.wait (weights do not depend
                                  // on the previous kernel)
    int a_f16;                    // both GEMM operands (activations A, weights W) are fp16 instead of bf16
    int out_f16;                  // 16-bit output is fp16 instead of bf16
    int split16;                  // fp32-parity mode: the 16-bit output is written as fp16 hi | lo | hi per 64 columns
                                  // (common.cuh split_col; ld_bf16 is the stride of that 3x wider buffer); plain kernel only
    long long* timing;            // optional (profiling): 8 clock64 stamps per CTA, see gemm_persistent.cu; null in production
    int tma_store;                // 0: register/LSU stores only; 1: 16-bit output, 2: fp32 output may leave through a TMA store
                                  // (plain persistent kernel: the LAST tile of every CTA is staged in the idle operand ring)
    int debug;                    // timing decomposition only (VB200_DEBUG through vb200_linear): 1 = issue no MMA, 2 = no epilogue
                                  // stores, 4 = no operand loads (the ring is "filled" by plain arrives); results are garbage
    const int* m_rows;            // optional device row count (packed batches): rows >= min(*m_rows, M) are neither loaded nor
                                  // computed -- the tile list ends at the last 128-row tile holding a row below it.  Written
                                  // before the launch's graph starts, so it is read ahead of griddepcontrol.wait.  Honoured by
                                  // the persistent kernel (PCfg MODE 6 in place of MODE 0); the fp32-parity kernel
                                  // computes every row.
    int split_acc;                // fp32-parity mode: A and W are hi / lo split operands over K' = 3K.  The kernel (PCfg MODE 7,
                                  // 64-wide tiles) sums each 64-wide k-block's wgmma result into a separate fp32 accumulator with
                                  // round-to-nearest adds: the tensor cores' own fp32 accumulation over K' drifts with K.
};

// persistent CTAs, wgmma consumer warpgroups (gemm_persistent.cuh)
int gemm_p_pick_block_n(int N);
int num_sms_host();          // SM count of the current device (132 on H100 SXM)
// tmap_c: the output map of the TMA store (ep.tma_store != 0), or null.  grid_pct (all GEMM launchers): 0 the default persistent
// grid (persistent_grid), 10..100 this percentage of the SMs.
cudaError_t launch_gemm_persistent_plain(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap* tmap_c,
                                         const GemmEpilogue& ep, int block_n, int grid_pct, cudaStream_t st);
// ping-pong consumer warpgroups (gemm_pingpong.cuh): plain bias / activation GEMMs with N a multiple of block_n (64 or 128), no
// pooled product or fp32-parity output; every output leaves through its TMA map (tmap_c16 for out_bf16, tmap_c32 for out_f32,
// SWIZZLE_128B boxes of 128 rows x 128 bytes).  Same bits as launch_gemm_persistent_plain.
bool gemm_pingpong_supports(const GemmEpilogue& ep, int block_n);
cudaError_t launch_gemm_pingpong(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap* tmap_c16,
                                 const CUtensorMap* tmap_c32, const GemmEpilogue& ep, int block_n, int grid_pct, cudaStream_t st);

// Head gate of the gated packed forwards (vb200_forward_packed_gated): sample b's head h context rows -- or its probabilities -- are
// scaled in fp32 by p[b * ld + h], p being one attention entry's column of the plan's [B, n_entries, max_heads] gate table.  A
// co-attention launch runs two entries: its image-query direction reads the column at p + next.  p null: no gate, today's bits
// (a gate of 1.0f gives them too).
struct HeadGate {
    const float* p; int ld, next;
    __device__ __forceinline__ float at(int b, int h, int dir = 0) const {
        return p ? p[static_cast<size_t>(b) * ld + dir * next + h] : 1.0f;
    }
};
// 16-bit activation buffers are typed __nv_bfloat16* throughout; `f16` says the bits are IEEE fp16 instead.
// K4: softmax(Q K^T / sqrt(d) + mask) V per (sample, head); qkv row = [Q | K | V], each `hidden` wide.  Every attention launcher takes
// an optional HeadGate (default: none).
cudaError_t launch_self_attention(const __nv_bfloat16* qkv, int ld_qkv, int hidden, const float* key_mask_add,
                                  __nv_bfloat16* ctx, int ld_ctx, int B, int L, int heads, int head_dim, int pdl,
                                  int f16, cudaStream_t st, const int* offs = nullptr, HeadGate gate = {});
// offs (packed batches, optional): device [B + 1] row offsets; sample b is rows [offs[b], offs[b+1]) of qkv / mask / ctx, and
// L is the shared-memory capacity (>= every sample's length).  nullptr: sample b is rows [b L, b L + L).
// K5: both co-attention directions in one kernel.  qkv_img rows = [Q1|K1|V1], qkv_txt rows = [Q2|K2|V2].
//   ctx_txt[b,t] = softmax(Q2 K1^T / sqrt(d) + img_mask) V1      ctx_img[b,v] = softmax(Q1 K2^T / sqrt(d) + txt_mask) V2
cudaError_t launch_co_attention(const __nv_bfloat16* qkv_img, int ld_img, const __nv_bfloat16* qkv_txt, int ld_txt,
                                int hidden, const float* img_mask_add, const float* txt_mask_add,
                                __nv_bfloat16* ctx_txt, int ld_ctx_txt, __nv_bfloat16* ctx_img, int ld_ctx_img, int B,
                                int T, int V, int heads, int head_dim, int pdl, int f16, cudaStream_t st,
                                const int* offs_t = nullptr, const int* offs_v = nullptr,   // as launch_self_attention, per stream
                                HeadGate gate = {});                                         // dir 0 ctx_txt, 1 ctx_img
// Streaming K4 / K5 (any length): same arguments and the same bits as the two above wherever those accept the length, but K and V
// stream through shared memory in 64-key blocks, one CTA per 64 query rows.  The engine uses them for plans with more than 256 rows
// per sample in a stream the op reads.
cudaError_t launch_self_attention_stream(const __nv_bfloat16* qkv, int ld_qkv, int hidden, const float* key_mask_add,
                                         __nv_bfloat16* ctx, int ld_ctx, int B, int L, int heads, int head_dim, int pdl,
                                         int f16, cudaStream_t st, const int* offs = nullptr, HeadGate gate = {});
cudaError_t launch_co_attention_stream(const __nv_bfloat16* qkv_img, int ld_img, const __nv_bfloat16* qkv_txt, int ld_txt,
                                       int hidden, const float* img_mask_add, const float* txt_mask_add,
                                       __nv_bfloat16* ctx_txt, int ld_ctx_txt, __nv_bfloat16* ctx_img, int ld_ctx_img, int B,
                                       int T, int V, int heads, int head_dim, int pdl, int f16, cudaStream_t st,
                                       const int* offs_t = nullptr, const int* offs_v = nullptr, HeadGate gate = {});

// LayerNorm(y + res) of a GEMM's fp32 output: fp32 stream out + 16-bit operand out (layernorm.cu); split16: hi | lo | hi operand (fp32-parity mode)
cudaError_t launch_ln_residual(const float* y, int ld_y, const float* res, int ld_res, const float* gamma, const float* beta,
                               float eps, float* out_f32, int ld_f32, __nv_bfloat16* out16, int ld16, int M, int N, int f16,
                               int split16, int pdl, cudaStream_t st,
                               const int* m_rows = nullptr);   // optional device row count: rows >= *m_rows are skipped
// K2: word + position + token-type gather, task-token row at index 1, LayerNorm; also builds the additive text mask.
cudaError_t launch_text_embed(const int64_t* ids, const int64_t* seg, const int64_t* input_mask, const int64_t* task,
                              const float* word, const float* pos, const float* type, const float* task_tab,
                              const float* gamma, const float* beta, float eps, float* out_f32,
                              __nv_bfloat16* out_bf16, float* mask_add, int B, int Tin, int H, int vocab, int max_pos,
                              int n_type, int n_task, int task_tokens, int f16, int split16, cudaStream_t st,
                              const int* offs = nullptr, int rows = 0);
// Packed batches (offs != nullptr): offs = device [B + 1] OUTPUT row offsets (T_b = Tin_b + task_tokens rows per sample), ids / seg
// hold sample b's Tin_b tokens at offs[b] - b * task_tokens, positions restart at 0 per sample, input_mask is unused (every row is
// real), `rows` = offs[B] and Tin is ignored.
// K1 (input half): fp32 region features + 5-d boxes -> bf16 GEMM operand [B*V, Kp] = [feat | loc | 0], additive image mask
// (image_mask nullptr: every row is real -- packed batches).
cudaError_t launch_image_pack(const float* feats, const float* loc, const uint8_t* image_mask, __nv_bfloat16* a_out,
                              float* mask_add, int rows, int F, int Kp, int f16, int split16, cudaStream_t st);
// custom_prediction()'s tensor construction on the device (worker.py:422-455): box features [B, n, F] + pixel boxes [B, n, 4] +
// image sizes [B, 2] (+ optional valid-box counts) -> operand rows [B * (n + 1), Kp] with the global mean row first, masks, spatials.
// Packed batches (offs != nullptr): offs = device [B + 1] image row offsets (V_b = boxes_b + 1 regions per image), box_features /
// boxes hold image b's V_b - 1 boxes from detector row offs[b] - b, every row is real, n and num_boxes are unused (num_boxes must be
// null, and split16 0), spatials_out is [offs[B], 5].
// src (packed only, the ablation calls): output image b holds nb = offs[b+1] - offs[b] - 1 detector boxes of source image
// src[b].image, box r being detector row src[b].box0 + kept[src[b].kept + r] (src[b].kept = -1: box0 + r, every box in order).  A kept
// list names any subset of the image's boxes in their original order; nb = 0 is the "no boxes" input: the global row alone, with
// zero features (the mean divides by max(nb, 1)) and location [0, 0, 1, 1, 1].
struct RegionSrc { int32_t image, box0, kept; };
cudaError_t launch_region_pack(const float* box_feats, const float* boxes, const float* image_wh, const int32_t* num_boxes,
                               __nv_bfloat16* a_out, float* mask_add, float* spatials_out, int B, int n, int F, int Kp, int f16,
                               int split16, cudaStream_t st, const int* offs = nullptr, const RegionSrc* src = nullptr,
                               const int32_t* kept = nullptr);
// The ablation calls' text ids: variant k (one CTA each, n of them) = tokens [first, first + len) of the packed question / segment
// ids, every position t whose bit is set in the call's bitmap replaced by mask_token, and task id task[sample] -> the packed layout
// of the plan's text offsets offs (device [n + 1]) in q_out / seg_out / task_out.  Position t's bit is bit t % 32 of word
// mask[masked + t / 32]; masked = -1: no position is replaced.
struct TextSrc { int32_t first, len, masked, sample; };
cudaError_t launch_variant_text(const TextSrc* v, int n, const int* offs, int task_tokens, const int64_t* q, const int64_t* seg,
                                const int64_t* task, int64_t mask_token, int64_t* q_out, int64_t* seg_out, int64_t* task_out,
                                cudaStream_t st, const uint32_t* mask = nullptr);
// Head ablation: row b of the [n, stride] gate table = ones with element zero[b] at 0 (zero[b] = -1: all ones), every float written.
cudaError_t launch_gate_rows(const int32_t* zero, int n, int stride, float* gate, cudaStream_t st);
// retrieval reuse: cached encoder state rows idx[b] -> sample b of a pair plan (fp32 stream [L, H], 16-bit operand [L, H16], mask [L]);
// the fp32 and mask copies are skipped when their pointers are null (packed poolers: the first 16-bit row of every sample)
cudaError_t launch_gather_state(const int32_t* idx, int n_src, const float* src_f32, const void* src_16, const float* src_mask,
                                float* dst_f32, void* dst_16, float* dst_mask, int B, int L, int H, int H16, cudaStream_t st);
// packed retrieval: one stream's copy from a packed caption / image state into a packed pair plan.  Pair b's rows
// [dst_offs[b], dst_offs[b+1]) come from rows starting at src_offs[b] (both device int32, [B + 1] and [B]); n32 / n16 = 16-byte
// vectors per row of the fp32 / 16-bit buffer.  Every pointer 16-byte aligned.
struct PackedStateCopy {
    const int* dst_offs;
    const int* src_offs;
    const float* src_f32;
    const void* src_16;
    float* dst_f32;
    void* dst_16;
    int n32, n16;
};
cudaError_t launch_gather_packed_state(const PackedStateCopy& text, const PackedStateCopy& image, int B, cudaStream_t st);
// Packed probabilities of the fp32 attention kernel (VB200_OUT_ATTENTION_PACKED).  Sample b's query rows are [offs_q[b],
// offs_q[b + 1]) of Q, its key rows [offs_k[b], offs_k[b + 1]) of K and of the key mask; its [heads, Lq_b, Lk_b] block goes to
// float dst[0] + entry[0] + heads * prefix[b], where dst[0] is the destination pointer (0: no write), entry[0] the entry's float
// offset and prefix[b] = sum over b' < b of Lq_b' * Lk_b'.  All of it lives in the plan's d_meta, filled per call.  gate: the
// entry's head gate (gated plans); the maps are then g * p, and the head mean averages the gated maps.
struct PackedProbs {
    const int* offs_q;
    const int* offs_k;
    const int64_t* dst;
    const int64_t* entry;
    const int64_t* prefix;
    HeadGate gate;
};
// fp32 CUDA-core attention (attention_f32.cu): in_kind 0 fp32 / 1 fp16 / 2 bf16 Q, K, V; ctx_mode 0 none / 1 fp16 / 2 bf16 /
// 3 fp16 hi | lo | hi; probs: optional [B, heads, Lq, Lk] fp32 attention probabilities.  packed (optional): a packed batch --
// Lq / Lk are then the per-sample capacities, the probabilities go where *packed says (probs must be null, ctx_mode 0, in_kind 1 or 2).
cudaError_t launch_attention_f32(const void* q, int ld_q, const void* k, const void* v, int ld_kv, int in_kind,
                                 const float* key_mask_add, int B, int Lq, int Lk, int heads, int D, __nv_bfloat16* ctx, int ld_ctx,
                                 int ctx_mode, float* probs, int pdl, cudaStream_t st, const PackedProbs* packed = nullptr);
// Head mean of the same probabilities (attention_f32.cu): probs [B, Lq, Lk] = (sum over heads in increasing order, in fp32) / heads,
// each head's row computed as launch_attention_f32 computes it; no context.  packed: a PackedProbs entry whose per-sample blocks
// are [Lq_b, Lk_b] (heads factor 1), probs NULL.
cudaError_t launch_attention_f32_mean(const void* q, int ld_q, const void* k, int ld_kv, int in_kind, const float* key_mask_add, int B,
                                      int Lq, int Lk, int heads, int D, float* probs, int pdl, cudaStream_t st,
                                      const PackedProbs* packed = nullptr);
// Pre-training heads at chosen rows: row rows[i] (device int32, i < n) of an fp32 state [*, H] -> row i of dst, in the 16-bit operand
// form the final LayerNorm writes (mode 0 bf16, 1 fp16, 2 fp16 hi | lo | hi with ld_dst the 3x wide stride) or as fp32 (mode 3); rows
// [n, rows_out) are zeroed.  H a multiple of 8 (64 in mode 2), 16-byte aligned src / dst; rows are bounds-checked on the host.
cudaError_t launch_gather_rows(const float* src, const int32_t* rows, int n, int rows_out, int H, void* dst, int ld_dst, int mode,
                               cudaStream_t st);
// Pre-training objectives: per listed row i < n of a head's fp32 logits [n, N] (row stride ld), loss[i] = the cross-entropy
// logsumexp(z) - z[labels[i]] (labels: device int32, token and pair heads) or KL(targets[i] || softmax z) (targets: device fp32 [n, N],
// image head); g = {token, image, pair}.  With `reduced` (device fp32 [3]) reduced[k] = mean of list k's losses (NaN for n_k = 0),
// in a fixed order.  Labels are range-checked on the host.
struct LossRows { const float* logits; int ld, N, n; const int32_t* labels; const float* targets; float* loss; };
cudaError_t launch_pretrain_losses(const LossRows* g, float* reduced, cudaStream_t st);
// Layer states (VB200_OUT_LAYER_STATES): one entry of an fp32 residual stream src [B x L rows, H] (dense: sample b's rows
// [b L, b L + L), mask the additive key mask, 0 on real rows; packed: rows [offs[b], offs[b + 1]), m_rows the device row count) into
// the float buffer whose address is *dst (0: no write; dst lives in the plan's staged meta).  reduce 0: every row (dense: B x L
// rows, padding included; packed: *m_rows rows); 1: each sample's first row, [B, H]; 2: [B, H], the mean over each sample's real
// rows, summed in increasing row order in fp32 and divided once by the count (NaN for a sample without one).  H a multiple of 4;
// src and *dst 16-byte aligned (the host checks the caller's buffer).
struct StateArgs { const float* src; const int* offs; const int* m_rows; const float* mask; const int64_t* dst; int B, L, H, reduce; };
cudaError_t launch_layer_state(const StateArgs& a, int pdl, cudaStream_t st);
// K8 (narrow heads): out[m, j] = dot(x[m, :K], W[j, :K]) + b[j] + (add ? add[m] : 0), j < n_out <= 4.
cudaError_t launch_rowdot(const float* x, int ld_x, const float* W, const float* b, const float* add, float* out,
                          int ld_out, int M, int K, int n_out, int pdl, cudaStream_t st, const int* m_rows = nullptr);
// Answer decode (decode.cu, vb200_decode_answers): message b's softmax over the `len` logits at src, its top_n (<= 10)
// probabilities and indices, and for grounding (spatials != null: the segment's first [len, 5] spatials row) the pixel boxes of
// the picked rows.  One CTA per message; the descriptors are resolved and bounds-checked on the host.
// Answer ablation (score != null, top_n 1): the CTA writes *score instead of an answer -- column `column` of src, or for column -1
// the top-1 of the logits at ref (the message's unablated segment, recomputed by every CTA), with its probability in src, and src's
// own top-1; answers may then be null.  drop >= 0 (a grounding box variant): src is ref without row `drop`, ref has len + 1 logits,
// and column and top-1 are reported in ref's numbering -- the attributed row maps into src, a dropped one reports column -1 with
// probability 0, and src's top-1 maps back by +1 from row `drop` on.
struct DecodeDesc {
    const float* src;
    const float* spatials;
    double image_w, image_h;
    int len, top_n;
    const float* ref;
    vb200_ablation_score* score;
    int column, drop;
};
cudaError_t launch_answer_decode(const DecodeDesc* descs, int n, vb200_answer* answers, cudaStream_t st);
// Message ablation's segments (decode.cu): variant k (one CTA each) copies `len` floats of head `head` into out + dst -- element i
// is heads.p[head][row * ld + i] for a head of several columns (one row), heads.p[head][(row + i) * ld] for a one-column head (a
// run of rows) -- with element `sub` (>= 0) read from row sub_row instead.  Heads are indexed as the engine's output slots.
constexpr int kSegmentHeads = 7;
struct SegmentHeads { const float* p[kSegmentHeads]; int ld[kSegmentHeads], cols[kSegmentHeads]; };
struct SegmentDesc { int32_t head, row, len, sub, sub_row; int64_t dst; };
cudaError_t launch_segment_gather(const SegmentDesc* descs, int n, const SegmentHeads& heads, float* out, cudaStream_t st);
// Shapley estimates (decode.cu, vb200_shapley_values): one CTA per message, the arithmetic documented at vb200_shapley_values.
// perm: [n_perm, n_units] int32, values: 2 + n_perm * (n_units - 1) floats, phi / stderr: n_units floats each.
struct ShapleyDesc { const int32_t* perm; const float* values; float* phi; float* stderr_out; int32_t n_units, n_perm, group; };
constexpr int kShapleyMaxUnits = 1024;
cudaError_t launch_shapley_values(const ShapleyDesc* descs, int n, cudaStream_t st);
// Shapley-Taylor pair indices (decode.cu, vb200_interaction_values): the arithmetic documented at vb200_interaction_values.  CTA
// (m, k) takes pairs [k * kInteractionPairs, (k + 1) * kInteractionPairs) of message m, one thread per pair; max_pairs is the
// largest n_pairs of the call.  pairs: [n_pairs, 2] int32 on the device, values: 2 + P (n - 1) + 2 P Q floats, inter / stderr: Q.
struct InteractionDesc {
    const int32_t* perm; const float* values; const int32_t* pairs; float* inter; float* stderr_out; int32_t n_units, n_perm, group, n_pairs;
};
constexpr int kInteractionPairs = 1024;
cudaError_t launch_interaction_values(const InteractionDesc* descs, int n, int max_pairs, cudaStream_t st);
// Attention relevance (relevance.cu, vb200_attention_relevance): per sample b (one CTA) the rollout rows of the text CLS row and the
// image global row, [2, T_b + V_b] at relevance + out.  Entry e of the maps starts at float `offset` and holds sample b's
// [heads, Lq_b, Lk_b] block at heads * prefix[k] (k 0 text layers, 1 image layers, 2 both directions of a connection layer); kinds
// follow the full list's execution order, every kind 3 right after a kind 2.  max_cols: the largest T_b + V_b (<= 2048).
struct RelevanceEntry { int64_t offset; int32_t kind, heads; };
struct RelevanceSample { int64_t prefix[3]; int64_t out; int32_t T, V; };
cudaError_t launch_attention_relevance(const float* maps, const RelevanceEntry* entries, int n_entries, const RelevanceSample* samples,
                                       int B, int max_cols, float* relevance, cudaStream_t st);
// Detector-region selection (regions_select.cu, vb200_select_regions).  Image i's n proposals are workspace rows [row0, row0 + n)
// of stats / dbox / max_conf and words [mask0, mask0 + n * nw) of the bitmask; its k = min(K, n) selected rows go to output rows
// [dst_row, dst_row + k).  npad: n rounded up to a power of two >= 32.  Descriptors are validated on the host.
constexpr int kSelectMaxProposals = 2048;
struct SelectDesc {
    const float* proposals;       // [n, 4]
    const float* scores;          // [n, C] logits
    const float* features;        // [n, F], 16-byte aligned
    size_t row0, mask0;
    float im_scale;
    int n, npad, nw, dst_row, k;
};
struct SelectArgs {
    int C, F, K, start;           // classes, feature width, max boxes, first class of the NMS (0 with background, else 1)
    float thr, nms_iou;           // thr = max(conf_thresh, 0)
    float2* stats;                // workspace [rows]: softmax max, sum
    float* dbox;                  // workspace [rows, 4]: proposals / im_scale
    unsigned* mask;               // workspace: per-image suppression bitmasks
    unsigned* max_conf;           // workspace [rows], zeroed before the NMS: bits of the per-box maximum confidence
    int* keep;                    // workspace [n_images, K]
    float* box_features;          // outputs: see vb200_selected
    float* boxes;
    int32_t* num_boxes;
    int32_t* keep_index;
    float* max_conf_out;
    float* cls_prob;
    int64_t* objects;
};
size_t select_nms_smem(int npad);
cudaError_t launch_select_regions(const SelectDesc* descs, int n, int max_n, int max_npad, const SelectArgs& a, cudaStream_t st);

// ---- shared host-side launch helpers
template <typename K>
inline cudaError_t set_smem(K kern, size_t bytes) {
    // opt in to > 48 KB dynamic shared memory (host-side attribute; launches are replayed from a CUDA graph,
    // so this runs at capture time only)
    if (bytes <= 48 * 1024) return cudaSuccess;
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, int pdl, cudaStream_t st,
                             Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    if (pdl) {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace vb
