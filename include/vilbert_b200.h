/* vilbert_b200 -- C ABI of the H100-native (sm_90a) ViLBERT multi-task forward.
 *
 * The reference has no FFI for this path: its boundary is the Python object protocol that
 * the reference worker.py fixes (SURVEY.md section 8b):
 *     config = BertConfig.from_json_file(...)                          worker.py:495, 506-522
 *     model  = VILBertForVLTasks.from_pretrained(ckpt, config=config,
 *                                                num_labels=3129, ...) worker.py:530-532
 *     model.eval(); model.cuda(0)                                      worker.py:534-536
 *     out10  = model(question, features, spatials, segment_ids, input_mask, image_mask,
 *                    co_attention_mask, task_tokens, output_all_attention_masks=True)
 *                                                                      worker.py:286-289
 * The entry points below are exactly what a binding for that protocol needs, and nothing else:
 * vb200_create <- from_pretrained + cuda(i); vb200_forward <- __call__; vb200_destroy <- del.
 * Beyond the protocol: packed variable-length batches (vb200_packed_inputs: samples with their own text lengths and region counts
 * in one forward, plans keyed on capacity buckets, GEMM tiles past the call's row totals skipped), detector output in, dense or
 * packed (vb200_region_inputs, vb200_packed_region_inputs: every image at its own box count), caption-image retrieval with reuse, dense or packed (vb200_packed_pairs: captions and images encoded once
 * at their own lengths, pairs scored without padding; vb200_encode_regions_packed: image states from detector output), the answer decode of every message of a batch in one kernel (vb200_decode_answers:
 * softmax, top N and grounding boxes, so a C host answers a message without re-implementing prediction()'s decode), the detector's
 * region selection (vb200_select_regions: per-class NMS, confidence ranking and the top boxes of every image, written into the packed
 * region inputs), the pre-training heads at the rows a caller lists (vb200_pretraining_heads: masked-token and masked-region logits and
 * the image-text alignment score from a forward's final states, ranked on the device), upstream's pre-training model
 * (vb200_create_pretraining: a checkpoint with the encoder and the `cls` heads but no task heads; vb200_pretraining_objectives: the
 * masked-token, masked-region and alignment losses from labels, on the device), and kernel-level entry points for the tests.
 * The Python shim in vilbert-multi-task_b200/ (ctypes) implements the protocol on top of them; see
 * INTEGRATION.md for the stub a maintainer of the reference would add.
 *
 * Conventions: plain pointers and sizes, no C++/torch types; every function returns 0 on success or a
 * negative vb200_status; no exception crosses the boundary; vb200_last_error() returns the message of the
 * last failure on that handle (or of the last failed vb200_create when handle == NULL).
 * vb200_forward is asynchronous on the caller's stream (no hidden synchronisation); input and output
 * buffers are owned by the caller; one handle serves one stream at a time (workspaces are per handle).
 */
#ifndef VILBERT_B200_H
#define VILBERT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB200_ABI_VERSION 2

typedef struct vb200_engine* vb200_handle;

typedef enum {
    VB200_OK = 0,
    VB200_ERR_INVALID = -1,      /* bad argument / unsupported shape */
    VB200_ERR_CONFIG = -2,       /* config JSON could not be parsed or is unsupported */
    VB200_ERR_CHECKPOINT = -3,   /* missing / unexpected / mis-shaped state_dict entry */
    VB200_ERR_CUDA = -4,         /* CUDA runtime or driver error (message has the detail) */
    VB200_ERR_NO_DEVICE = -5     /* no sm_90 device: there is deliberately no CPU fallback */
} vb200_status;

typedef enum { VB200_F32 = 0, VB200_F16 = 1, VB200_BF16 = 2 } vb200_dtype;

/* One entry of the flat checkpoint state_dict (worker.py:470, 530-532): upstream key name, host pointer. */
typedef struct {
    const char* name;        /* e.g. "bert.encoder.c_layer.3.biattention.query1.weight" ("module." prefix accepted) */
    int32_t dtype;           /* vb200_dtype */
    int32_t ndim;            /* 1 or 2 */
    int64_t shape[2];        /* nn.Linear weights are [out, in] row-major */
    const void* data;        /* host memory, contiguous */
} vb200_tensor;

/* Which elements of the reference's 10-tuple (worker.py:287) to compute. */
enum {
    VB200_OUT_VIL_PREDICTION = 1 << 0,         /* [B, num_labels]  VQA / VG-QA            worker.py:296 */
    VB200_OUT_VIL_PREDICTION_GQA = 1 << 1,     /* [B, 1533]        GQA                    worker.py:313 */
    VB200_OUT_VIL_LOGIT = 1 << 2,              /* [B, 1]           retrieval              worker.py:359 */
    VB200_OUT_VIL_BINARY_PREDICTION = 1 << 3,  /* [B/2, 2] (B even) / [B, 2] (B odd)  NLVR2  worker.py:329 */
    VB200_OUT_VIL_TRI_PREDICTION = 1 << 4,     /* [B, 3]           SNLI-VE                worker.py:345 */
    VB200_OUT_VISION_PREDICTION = 1 << 5,      /* [B, V, v_target_size]  pre-training head, unused by the worker */
    VB200_OUT_VISION_LOGIT = 1 << 6,           /* [B, V, 1]        grounding              worker.py:374 */
    VB200_OUT_LINGUISIC_PREDICTION = 1 << 7,   /* [B, T, vocab]    pre-training head, unused by the worker */
    VB200_OUT_LINGUISIC_LOGIT = 1 << 8,        /* [B, T, 1]        never read by the worker */
    VB200_OUT_TASK_HEADS = 0x15F,              /* the seven task heads (everything but the two pre-training heads) */
    VB200_OUT_ALL = 0x1FF,
    VB200_OUT_ATTENTION = 1 << 9,              /* element 9 of the tuple, attn_data_list: the attention probabilities of all 24 layers
                                                  (worker.py:287-288; the reference returns them because config.visualization is set,
                                                  worker.py:522, and never reads them).  Off unless requested: see
                                                  vb200_attention_layout and vb200_outputs.attention_probs. */
    VB200_OUT_ATTENTION_PACKED = 1 << 10,      /* the same probabilities for a packed batch, every sample at its own lengths: accepted by
                                                  vb200_forward_packed and vb200_forward_regions_packed only (see there and
                                                  vb200_attention_layout_packed); VB200_ERR_INVALID on every other forward */
    VB200_OUT_LAYER_STATES = 1 << 11           /* the fp32 state after every step that writes a stream, by selection ("state_entries",
                                                  "state_rows": see vb200_set_option), written by the forward's kernels into
                                                  vb200_outputs.layer_states at the offsets of vb200_state_layout (dense forwards) or
                                                  vb200_state_layout_packed (packed forwards).  Accepted by vb200_forward[_slot],
                                                  vb200_forward_regions, vb200_forward_packed and vb200_forward_regions_packed;
                                                  VB200_ERR_INVALID on every other entry point */
};

/* Inputs of one forward, in the dtypes the worker builds them (worker.py:416-419, 452-455).
 * T = Tin + 1 when config.task_specific_tokens (worker.py:516-517).  co_attention_mask is accepted for
 * signature compatibility and ignored, as upstream ignores it (worker passes zeros, worker.py:455). */
typedef struct {
    int32_t batch;                 /* B  */
    int32_t n_tokens;              /* Tin */
    int32_t n_regions;             /* V  */
    const int64_t* question;       /* [B, Tin] token ids */
    const float* features;         /* [B, V, v_feature_size] */
    const float* spatials;         /* [B, V, 5] */
    const int64_t* segment_ids;    /* [B, Tin] */
    const int64_t* input_mask;     /* [B, Tin] */
    const uint8_t* image_mask;     /* [B, V] */
    const float* co_attention_mask;/* [B, V, Tin] or NULL; ignored */
    const int64_t* task_tokens;    /* [B, 1] */
} vb200_inputs;

/* Caller-allocated fp32 outputs; a NULL pointer (or a cleared select bit) skips that output. */
typedef struct {
    float* vil_prediction;         /* [B, num_labels] */
    float* vil_prediction_gqa;     /* [B, gqa_labels] */
    float* vil_logit;              /* [B, 1] */
    float* vil_binary_prediction;  /* [B/2, 2] if B even else [B, 2] */
    float* vil_tri_prediction;     /* [B, 3] */
    float* vision_prediction;      /* [B, V, v_target_size] */
    float* vision_logit;           /* [B, V, 1] */
    float* linguisic_prediction;   /* [B, T, vocab] */
    float* linguisic_logit;        /* [B, T, 1] */
    float* sequence_output_t;      /* optional debug tap: final text stream  [B, T, hidden]   (fp32) */
    float* sequence_output_v;      /* optional debug tap: final image stream [B, V, v_hidden] (fp32) */
    float* pooled_output;          /* optional debug tap: pooled_t * pooled_v [B, bi_hidden] */
    float* attention_probs;        /* VB200_OUT_ATTENTION: one flat fp32 buffer holding every layer's softmax probabilities
                                      [B, heads, Lq, Lk] back to back in execution order (vb200_attention_layout gives the
                                      offsets); NULL skips the copy.  VB200_OUT_ATTENTION_PACKED: required, device memory of
                                      vb200_attention_layout_packed's total_floats, written in place by the forward's kernels */
    float* layer_states;           /* VB200_OUT_LAYER_STATES: required, 16-byte aligned (VB200_ERR_INVALID if NULL or not),
                                      device memory of vb200_state_layout's / vb200_state_layout_packed's total_floats, written in
                                      place by the forward's kernels with 16-byte stores.  Read only when the bit is set, so a host built against a header without
                                      this field stays correct as long as it never sets the bit. */
} vb200_outputs;

/* Engine options (all optional; zero-initialise for defaults).  Flags are tri-state: 0 default, 1 on, -1 off. */
typedef struct {
    int32_t device;                /* CUDA ordinal */
    int32_t num_labels;            /* vil_prediction width; 0 -> taken from the checkpoint (worker.py:523: 3129) */
    int32_t use_cuda_graph;        /* default on: each (B,Tin,V,select) plan is captured once and replayed */
    int32_t use_pdl;               /* programmatic dependent launch: 0 default (= every kernel), > 0 every kernel, < 0 none */
    int32_t strict;                /* default on: unexpected checkpoint keys are an error */
    int32_t act_fp16;              /* 16-bit format of the tensor-core operands (weights AND activations; wgmma needs
                                      matching A/B formats).  default on: IEEE fp16 (11-bit significand; activations
                                      are LayerNorm-bounded, converts saturate); -1: bf16.  Accumulation, residual stream,
                                      LayerNorm, softmax and logits are fp32 either way. */
    int32_t fused_layernorm;       /* reserved, must be 0 or negative (was the cluster-LayerNorm GEMM epilogue, which is removed;
                                      vb200_create returns VB200_ERR_INVALID for a positive value).  LayerNorm(dense(x) +
                                      residual) always runs as GEMM (fp32 out) + an L2-resident row kernel. */
    int32_t split_fp32;            /* 1: fp32-parity mode ("fp32x").  Every GEMM operand travels as TWO fp16 numbers (hi = fp16(x),
                                      lo = fp16(x - hi), 22 significand bits); operand buffers hold hi | lo | hi (weights hi | hi |
                                      lo) per 64 columns, so an ordinary wgmma GEMM over K' = 3K adds hi.hi + lo.hi + hi.lo in its
                                      fp32 accumulator; attention runs in fp32 on CUDA cores; GELU uses the 1.5e-7 erf.  3x the
                                      tensor work of the default mode -- for logit parity with the reference's fp32 forward
                                      (<= 1e-3 per logit, BASELINE.json north_star), not for throughput.  Implies act_fp16. */
    int32_t ln_fold;               /* reserved, must be 0 (was the LayerNorm fold, which is removed; vb200_create returns
                                      VB200_ERR_INVALID for any other value) */
    int32_t max_plans;             /* plan-cache bound: plans (workspace + CUDA graph per (batch, tokens, regions, select, slot))
                                      beyond this are evicted least-recently-used; 0 -> 24 */
} vb200_options;

int vb200_abi_version(void);

/* from_pretrained + cuda(device): parse the BertConfig JSON, audit the state_dict against the upstream key list,
 * repack weights to device (16-bit GEMM operands in the format vb200_options::act_fp16 selects -- fp16 by default, bf16, or the
 * fp16 hi/lo pairs of split_fp32 -- and fp32 LayerNorm / bias / embedding tables).  VB200_ERR_CONFIG, naming the field and the
 * entry, for a t_biattention_id / v_biattention_id entry outside [0, num_hidden_layers] / [0, v_num_hidden_layers] or below the
 * entry before it (equal entries are connection layers back to back; empty lists are a model without connection layers). */
int vb200_create(const char* config_json, int64_t n_tensors, const vb200_tensor* tensors, const vb200_options* opt,
                 vb200_handle* out);
/* BertForMultiModalPreTraining.from_pretrained + cuda(device): the same arguments, options and audit rules as vb200_create (`module.`
 * prefixes, gamma / beta, the ignored keys, strict vs strict = -1 for extra keys), against upstream's pre-training key set: `bert.*`
 * plus cls.predictions.*, cls.imagePredictions.* and cls.bi_seq_relationship.*.  Task-head keys are extra keys.  The audit runs
 * before any device is touched.  task_specific_tokens may be off (the pre-training config carries no task embeddings).
 * VB200_ERR_CONFIG for visual_target != 0 or predict_feature (feature regression / NCE are not implemented: the masked-region head is
 * the KL objective over v_target_size classes); VB200_ERR_INVALID for num_labels != 0.
 * The engine has no task head: every forward, encode and cached entry point accepts a `select` of the pre-training heads
 * (VB200_OUT_LINGUISIC_PREDICTION, VB200_OUT_VISION_PREDICTION), the taps and the attention maps, and returns VB200_ERR_INVALID, naming
 * the head, for any bit of VB200_OUT_TASK_HEADS; so does vb200_decode_answers for every family.  vb200_model_dim("num_labels") and
 * ("gqa_labels") are 0.  vb200_pretraining_heads and vb200_pretraining_objectives work as on any engine. */
int vb200_create_pretraining(const char* config_json, int64_t n_tensors, const vb200_tensor* tensors, const vb200_options* opt,
                             vb200_handle* out);
int vb200_destroy(vb200_handle h);
const char* vb200_last_error(vb200_handle h);

/* Device-pointer forward (what worker.py:286-289 does): all vb200_inputs / vb200_outputs pointers are device
 * memory on the engine's device; enqueued on `cuda_stream` (a cudaStream_t passed as void*).
 * Synchronisation: a call whose (batch, n_tokens, n_regions, select, slot) plan already exists only enqueues work and returns.
 * The FIRST call of a shape builds its plan: cudaMalloc of the workspace, one eager validation pass with a stream
 * synchronisation, and the CUDA-graph capture -- it blocks the host for some milliseconds and may synchronise the device (also
 * when the plan cache evicts an old plan, vb200_options::max_plans).  Warm a server's shapes up before taking traffic. */
int vb200_forward(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, void* cuda_stream);

/* Same with an explicit workspace slot (0..15): forwards on DIFFERENT slots may run concurrently on different streams (each
 * slot owns its workspace, TMA descriptors and captured graph; weights are shared) -- how a server keeps more than one batch in
 * flight so kernels of one batch fill the SMs another leaves idle.  vb200_forward is slot 0. */
int vb200_forward_slot(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                       void* cuda_stream);

/* Host-pointer forward: same, but every pointer is HOST memory (pinned for full speed); copies in, runs, copies
 * the selected outputs back and synchronises the stream before returning. */
int vb200_forward_host(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select,
                       void* cuda_stream);

/* Same on workspace slot `slot`; synchronize = 0 returns right after enqueueing (H2D copies, kernels and D2H copies are
 * ordered on `cuda_stream`; the host buffers must stay valid and the outputs are complete once the caller has synchronised
 * that stream).  Two slots on two streams overlap one batch's copies with the other's kernels. */
int vb200_forward_host_slot(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                            int32_t synchronize, void* cuda_stream);

/* Introspection used by the tests / bench: number of kernels one forward of this shape launches (with VB200_OUT_ATTENTION: one with
 * the current map selection), algorithmic FLOPs of it, model dimensions ("max_rows_per_sample": the engine's current bound;
 * "attention_entries" (-1 above 63 entries) and "attention_heads": the map selection; "state_entries" and "state_rows": the
 * layer-state selection; see vb200_set_option).  With VB200_OUT_LAYER_STATES the count includes one launch per selected entry. */
int vb200_plan_info(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select,
                    int64_t* n_launches, double* flops);
int vb200_model_dim(vb200_handle h, const char* key, int64_t* value);
/* Run-time knobs: "max_plans" (plan-cache bound); "profile_grid_pct" (0 or 10..100): the NEXT vb200_profile_ops call launches every
 * GEMM with this percentage of the resident CTA slots as its persistent grid --
 * for reporting what a launch does when it has the GPU to itself; forwards are never affected.  "gemm_kernel": 1 (default, or 0
 * under VB200_GEMM=coop) runs the plain GEMMs the ping-pong kernel supports on it, 0 runs every GEMM on the cooperative persistent
 * kernel; a change drops the cached plans.  Both give the same bits.  "max_rows_per_sample" (256..1024, default 256): the longest text
 * (T = n_tokens + task token) or image (V = regions, boxes + 1) sequence any call of this engine accepts; text is bounded by
 * max_position_embeddings as well, and vb200_select_regions keeps at most this - 1 boxes per image.  Up to 256 rows per sample a
 * plan's attention stages each (sample, head) whole in shared memory; a plan with more rows in a stream runs that stream's
 * attention on the streaming kernels (vb200_self_attention_stream), which give the same bits wherever both run.  The choice
 * follows from the plan's shape alone, so the bound only changes validation and no cached plan is dropped.
 * Attention maps by selection (VB200_OUT_ATTENTION and VB200_OUT_ATTENTION_PACKED): "attention_entries" is a bitmask over the entries
 * of the full list in execution order (bit e: entry e of vb200_attention_selection; default every entry) and "attention_heads" 0
 * (default) writes every head, 1 each selected entry averaged over its heads: (sum over h = 0..heads-1 of p_h, added left to right in
 * fp32) / heads, each p_h bit-identical to the per-head map.  A zero mask, a bit at or past the entry count, a configuration with more
 * than 63 entries (the default then stays every entry) or attention_heads outside {0, 1} is VB200_ERR_INVALID.  Both stay in force
 * until changed and both are readable through vb200_model_dim.  The selection is part of the plan key of a forward with maps: the first
 * call after a change builds (or finds) the plan of the new selection, and a plan without maps is unaffected.  Every other output is
 * bit-identical whatever the selection.
 * Layer states by selection (VB200_OUT_LAYER_STATES): "state_entries" is a bitmask over the full state list in execution order (bit e:
 * entry e of vb200_state_selection; default every entry) and "state_rows" 0 (default) writes every row of each selected entry, 1 each
 * sample's first row, 2 each sample's mean over its real rows.  A zero mask, a bit at or past the entry count, a configuration with
 * more than 63 entries or state_rows outside {0, 1, 2} is VB200_ERR_INVALID.  Both are engine-wide, readable through vb200_model_dim,
 * and part of the plan key of a forward with states only.  A selection with a stream's last entry reads that stream's final rows, so
 * that stream's last layer runs on every row, as with a sequence_output tap. */
int vb200_set_option(vb200_handle h, const char* key, int64_t value);
/* Profiling: after vb200_set_option(h, "timeline", 1) every persistent GEMM launch of a forward records 16 stamps per CTA (0: clock64 at
 * entry, 1: setup done, 2: first k-block landed [-DVB200_STAMPS builds], 8 / 9: %globaltimer ns at entry / exit, 10: last tile accumulated,
 * 11: tiles walked, 12: SM id).  Copies the stamps of the LAST forward run on (shape, select, slot): stamps[n_ops][304][16],
 * dims[n_ops][4] = M, N, K, graph branch.  Synchronises the device.  scripts/step_timeline.py turns two slots' worth into per-SM
 * occupancy figures. */
int vb200_timeline(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select, int32_t slot, int32_t max_ops,
                   int32_t* n_ops, int32_t* dims, int64_t* stamps);
/* Per-launch device time of one forward of this shape (after at least one vb200_forward of it): every kernel of the plan is
 * captured 8x into its own CUDA graph and replayed `iters` times between two CUDA events (no host launch gaps).  kinds: 0 GEMM, 1 self-attention,
 * 2 co-attention, 3 narrow head, 4 LayerNorm; dims[4*i..] = {M, N, K, act} for GEMMs.  Profiling aid for bench.py. */
int vb200_profile_ops(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select, int32_t iters,
                      int32_t max_ops, int32_t* n_ops, int32_t* kinds, double* ms, double* flops, int32_t* dims);

/* Layout of vb200_outputs.attention_probs for a shape: entry i is a [batch, dims[4i], dims[4i+1], dims[4i+2]] fp32 tensor
 * (heads, query length, key length) at float offset offsets[i]; dims[4i+3] is the layer kind: 0 text layer, 1 image layer,
 * 2 connection layer, text queries over image keys, 3 connection layer, image queries over text keys (kinds 2 and 3 of one layer
 * are adjacent: the reference's per-layer tuple).  *n_entries receives the entry count (30 for the 12/6/6 configuration: 24
 * layers, two tensors per connection layer), total_floats the buffer size.  Arrays may be NULL to query the count only.
 * Under a map selection (vb200_set_option "attention_entries" / "attention_heads") the layout holds the selected entries only, in
 * execution order: *n_entries is the mask's popcount, heads is 1 under the head mean, the kind is unchanged; each entry's index in
 * the full list is vb200_attention_selection's. */
int vb200_attention_layout(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, int32_t max_entries,
                           int32_t* n_entries, int32_t* dims, int64_t* offsets, int64_t* total_floats);
/* The full list of attention-map entries in execution order and the engine's current selection of it: *n_entries receives the full
 * count (30 for the 12/6/6 configuration), kinds[e] entry e's kind (as dims[4i+3] above) and layout_entry[e] its index in the
 * layouts of vb200_attention_layout / vb200_attention_layout_packed, or -1 when "attention_entries" leaves it out.  Arrays (up to
 * max_entries) may be NULL to query the count only. */
int vb200_attention_selection(vb200_handle h, int32_t max_entries, int32_t* n_entries, int32_t* kinds, int32_t* layout_entry);
/* Attention relevance: the residual-weighted attention rollout (Abnar & Zuidema 2020) of one forward's maps through both streams,
 * for the two rows the answer heads read, the text CLS row (t_pooler) and the image global row (v_pooler).  For a sample with T text
 * rows (task token included) and V image rows, a step -- one text layer, one image layer, or both directions of one connection
 * layer, which read the same pre-layer streams -- maps each row i it writes to 0.5 (e_i + Abar[i, :]), Abar its map averaged over
 * heads (fp32, heads summed left to right, then divided once: the engine's head mean, so maps kept with every head and maps written
 * as the mean give the same bits) in its block of the T + V positions, and leaves the other rows e_i.  The output per sample is
 * rows 0 and T of W_n ... W_1, each T + V floats (text columns first) summing to 1; padded positions of a dense forward are 0.
 * Evaluated from the last step to the first on the two row vectors, each column's sum over the step's query rows in increasing order
 * with separate fp32 products and adds (relevance.cu states the order).
 * attention_probs: DEVICE, the maps one forward wrote under the engine's CURRENT map selection, which must hold every entry (heads
 * kept or averaged).  packed = 0: the layout of vb200_attention_layout for n_tokens = &Tin, n_regions = &V (one HOST value each);
 * relevance is DEVICE [batch, 2, T + V].  packed = 1: the layout of vb200_attention_layout_packed for the HOST arrays n_tokens /
 * n_regions [batch] (V_b = n_boxes_b + 1 for region forwards), validated as it validates them; sample b's [2, T_b + V_b] block
 * starts at float 2 sum_{b' < b} (T_b' + V_b').  VB200_ERR_INVALID, before anything is enqueued and with relevance untouched, for a
 * NULL pointer, batch < 1, bad lengths, packed not 0 / 1, and a selection that leaves out an entry (the message names the first).
 * Asynchronous on cuda_stream; builds no plan; the descriptors reach the device through engine-owned pinned staging in stream order,
 * so back-to-back calls need no synchronisation.  One CTA per sample. */
int vb200_attention_relevance(vb200_handle h, const float* attention_probs, int32_t batch, const int32_t* n_tokens,
                              const int32_t* n_regions, int32_t packed, float* relevance, void* cuda_stream);

/* ---- Layer states (VB200_OUT_LAYER_STATES).  The full list holds the fp32 residual-stream state after every step that writes a
 * stream, in execution order: the text embedding, the image embedding, then per schedule step one text entry (text layer), one
 * image entry (image layer) or two, text then image (connection layer): 32 entries for the 12/6/6 configuration, 19 text and 13
 * image.  An entry's value is the row the step's last LayerNorm writes; the last text / image entries equal sequence_output_t / _v.
 * Layout of vb200_outputs.layer_states for a dense forward of this shape: selected entry i is kinds[i] (0 text, 1 image),
 * dims[2i] rows of dims[2i + 1] floats at float offset offsets[i]: rows B x L (state_rows 0, L = T or V, padding rows included)
 * or B (state_rows 1 and 2; a sample without a real row has NaN means).  Arrays may be NULL to query the count only.  Builds no
 * plan and never blocks. */
int vb200_state_layout(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, int32_t max_entries, int32_t* n_entries,
                       int32_t* kinds, int32_t* dims, int64_t* offsets, int64_t* total_floats);
/* The same for a packed forward with these Tin_b / V_b (HOST arrays, validated as vb200_attention_layout_packed validates them;
 * V_b = n_boxes_b + 1 for vb200_forward_regions_packed): under state_rows 0 an entry holds sum T_b (T_b = Tin_b + task token) or
 * sum V_b rows, sample b's rows after sample b - 1's, the layout of the packed sequence_output taps; under 1 and 2 B rows. */
int vb200_state_layout_packed(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_regions, int32_t max_entries,
                              int32_t* n_entries, int32_t* kinds, int32_t* dims, int64_t* offsets, int64_t* total_floats);
/* The full state list and the current selection: *n_entries receives the full count, kinds[e] entry e's kind (0 text, 1 image) and
 * layout_entry[e] its index in the layouts above, or -1 when "state_entries" leaves it out.  Arrays may be NULL. */
int vb200_state_selection(vb200_handle h, int32_t max_entries, int32_t* n_entries, int32_t* kinds, int32_t* layout_entry);

/* custom_prediction()'s tensor construction fused into the forward (worker.py:422-455): instead of features [B, V, F] /
 * spatials [B, V, 5] / image_mask the caller passes what the detector produced -- box features, pixel boxes, image sizes -- and one
 * kernel writes the image-embedding GEMM's 16-bit operand rows directly: global mean row first, 5-d normalised locations
 * ([0,0,1,1,1] for the global row), masks.  n_regions of the forward is n_boxes + 1. */
typedef struct {
    int32_t batch;                 /* images (= rows of the forward) */
    int32_t n_tokens;              /* Tin */
    int32_t n_boxes;               /* detector boxes per image (rows of box_features per image); n_regions = n_boxes + 1 */
    const int64_t* question;       /* [B, Tin]   (text already repeated per image for pair / retrieval tasks, worker.py:266-284) */
    const int64_t* segment_ids;    /* [B, Tin] */
    const int64_t* input_mask;     /* [B, Tin] */
    const int64_t* task_tokens;    /* [B, 1] */
    const float* box_features;     /* [B, n_boxes, v_feature_size] fp32, as the detector returns them (worker.py:213) */
    const float* boxes;            /* [B, n_boxes, 4] pixel x1, y1, x2, y2 (infos[i]['bbox'], worker.py:434) */
    const float* image_wh;         /* [B, 2] image_width, image_height */
    const int32_t* num_boxes;      /* [B] valid boxes per image or NULL (= n_boxes); padded boxes are zeroed, masked and left out
                                      of the mean */
    float* spatials_out;           /* optional [B, n_boxes + 1, 5]: the spatials tensor the reference would have built (the
                                      grounding decode reads spatials[0], worker.py:379) */
} vb200_region_inputs;
int vb200_forward_regions(vb200_handle h, const vb200_region_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                          void* cuda_stream);

/* ---- Packed variable-length batches: one forward for samples with different text lengths and region counts.  Sample i's
 * Tin_i tokens and V_i regions are stored back to back with no padding and no masks: every row is a real token or region.  The
 * result is the forward of the same samples padded to a common shape with input_mask / image_mask = 1 on the real rows,
 * restricted to the real rows -- and bit-identical to a forward of each sample alone at its own (Tin_i, V_i).
 * Per-sample outputs keep their shapes ([B, num_labels], [B/2, 2], pooled_output, ...); per-row outputs are packed: vision_logit
 * [sum V_i, 1], vision_prediction [sum V_i, v_target], linguisic_logit [sum T_i, 1], linguisic_prediction [sum T_i, vocab] and the
 * sequence_output_t / _v taps, with T_i = Tin_i + 1 (task token).
 * Plans are keyed on (B, round16(max_tokens + 1), round16(max_regions), select, slot): a capacity costs workspace only (GEMM tiles
 * past the call's row totals are skipped, attention runs each sample at its own length), so a server that passes fixed capacities
 * keeps one plan and one CUDA graph per batch size whatever the lengths.  The lengths are host arrays (the plan is chosen on the
 * host); the per-sample offsets and row totals are copied to the plan's workspace on cuda_stream through a pinned staging buffer.
 * Attention maps: VB200_OUT_ATTENTION_PACKED, see vb200_attention_layout_packed.
 * VB200_ERR_INVALID for VB200_OUT_ATTENTION, split_fp32 engines, a length < 1 or above a non-zero capacity, T_i or V_i above
 * max_rows_per_sample (see vb200_set_option) and Tin_i > max_position_embeddings. */
typedef struct {
    int32_t batch;                  /* B */
    int32_t max_tokens;             /* plan capacity: 0 -> max Tin_i of this call; else >= every Tin_i */
    int32_t max_regions;            /* plan capacity: 0 -> max V_i of this call;   else >= every V_i */
    const int32_t* n_tokens;        /* HOST [B]: Tin_i >= 1 (T_i = Tin_i + 1 with task tokens) */
    const int32_t* n_regions;       /* HOST [B]: V_i >= 1 */
    const int64_t* question;        /* DEVICE [sum Tin_i]      sample i's tokens back to back, no padding */
    const int64_t* segment_ids;     /* DEVICE [sum Tin_i] */
    const float*   features;        /* DEVICE [sum V_i, v_feature_size] */
    const float*   spatials;        /* DEVICE [sum V_i, 5] */
    const int64_t* task_tokens;     /* DEVICE [B, 1] */
} vb200_packed_inputs;
int vb200_forward_packed(vb200_handle h, const vb200_packed_inputs* in, const vb200_outputs* out, uint32_t select,
                         int32_t slot, void* cuda_stream);

/* ---- Packed detector output: vb200_forward_regions with every image at its own box count and every text at its own length, stored
 * back to back as in vb200_packed_inputs, with no padding and no masks.  Image i has V_i = n_boxes_i + 1 regions (its global mean row
 * first); one kernel writes each image's operand rows at its packed offset.  Each image's outputs, taps and spatials_out rows are
 * bit-identical to vb200_forward_regions of that image alone (batch 1, n_boxes = n_boxes_i, n_tokens = Tin_i).  Plans are the
 * PACKED plans of vb200_forward_packed, keyed on (B, round16(max_tokens + 1), round16(max_boxes + 1), select, slot): the same plan and
 * CUDA graph serve both calls at equal capacities.  Outputs follow vb200_forward_packed (per-image outputs [B, ...], per-row outputs
 * packed over sum V_i / sum T_i rows).  Attention maps: VB200_OUT_ATTENTION_PACKED, see vb200_attention_layout_packed (V_i = n_boxes_i + 1).
 * VB200_ERR_INVALID for VB200_OUT_ATTENTION, split_fp32 engines, NULL required pointers,
 * n_boxes_i < 1 or above a non-zero max_boxes, V_i or T_i above max_rows_per_sample, Tin_i > max_position_embeddings and negative capacities. */
typedef struct {
    int32_t batch;                  /* B images (rows of the forward); text already repeated per image as for vb200_region_inputs */
    int32_t max_tokens;             /* plan capacity in Tin units: 0 -> this call's maximum */
    int32_t max_boxes;              /* plan capacity in detector boxes (regions = boxes + 1): 0 -> this call's maximum */
    const int32_t* n_tokens;        /* HOST [B] Tin_i >= 1 */
    const int32_t* n_boxes;         /* HOST [B] boxes of image i >= 1; V_i = n_boxes_i + 1 */
    const int64_t* question;        /* DEVICE [sum Tin_i] */
    const int64_t* segment_ids;     /* DEVICE [sum Tin_i] */
    const int64_t* task_tokens;     /* DEVICE [B, 1] */
    const float*   box_features;    /* DEVICE [sum n_boxes_i, v_feature_size] */
    const float*   boxes;           /* DEVICE [sum n_boxes_i, 4] pixel x1, y1, x2, y2 */
    const float*   image_wh;        /* DEVICE [B, 2] */
    float*         spatials_out;    /* optional DEVICE [sum V_i, 5] */
} vb200_packed_region_inputs;
int vb200_forward_regions_packed(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_outputs* out,
                                 uint32_t select, int32_t slot, void* cuda_stream);

/* ---- Attention maps of a packed batch (VB200_OUT_ATTENTION_PACKED, both packed forwards above).  VB200_OUT_ATTENTION keeps
 * meaning the dense [B, heads, Lq, Lk] layout and stays VB200_ERR_INVALID on packed calls; the packed bit selects this layout instead:
 * entry e (execution order, the kinds of vb200_attention_layout: 30 entries for the 12/6/6 configuration) starts at float
 * offsets[e] and holds, for sample b in batch order, a contiguous [heads, Lq_b, Lk_b] block at heads * sum_{b' < b} Lq_b' * Lk_b'
 * inside the entry, with (Lq_b, Lk_b) = (T_b, T_b), (V_b, V_b), (T_b, V_b) or (V_b, T_b) for kinds 0-3 and T_b = Tin_b + 1 (task token).
 * dims[2e] = heads, dims[2e + 1] = kind; total_floats is the buffer size (every float of it is written); arrays may be NULL to query
 * the count only.  Under a map selection (vb200_set_option "attention_entries" / "attention_heads") the entries are the selected ones
 * only, in execution order, with heads 1 under the head mean (sample b's block is then [Lq_b, Lk_b] at prefix[b]); each entry's index
 * in the full list is vb200_attention_selection's.
 * Builds no plan and never blocks.  n_tokens / n_regions are HOST arrays of Tin_b and V_b, validated as the
 * packed forwards validate them (a length < 1, T_b or V_b above max_rows_per_sample, Tin_b > max_position_embeddings: VB200_ERR_INVALID); for
 * vb200_forward_regions_packed pass V_b = n_boxes_b + 1.
 * A forward with the bit needs vb200_outputs.attention_probs (VB200_ERR_INVALID if NULL): the probability kernels write into it
 * directly, each sample bit-identical to the probabilities of a dense forward of that sample alone, and every other output is
 * bit-identical to the same call without the bit.  The destination pointer is staged with the call's offsets, so a call returns as
 * soon as its work is enqueued, as without maps, and back-to-back calls may pass different buffers.  A packed plan with maps is a
 * plan of its own (built, with its blocking first call, once per batch size and capacities), shared by every call at those
 * capacities whatever the lengths. */
int vb200_attention_layout_packed(vb200_handle h, int32_t batch, const int32_t* n_tokens /* HOST [batch] Tin_b */,
                                  const int32_t* n_regions /* HOST [batch] V_b */, int32_t max_entries, int32_t* n_entries,
                                  int32_t* dims, int64_t* offsets, int64_t* total_floats);

/* ---- Head masks: the two packed forwards with a per-sample, per-head gate on every attention head (pytorch_transformers'
 * head_mask).  head_mask is DEVICE fp32 [batch, E, H] with E = vb200_model_dim "head_mask_entries" (the full list of
 * vb200_attention_selection in execution order, each connection layer's text-query then image-query direction: 30 for 12/6/6) and
 * H = "head_mask_heads" (the configuration's largest head count, 12); slots past an entry's own head count are ignored.  Sample b's
 * head h context rows at entry e are multiplied in fp32 by head_mask[b][e][h] before the 16-bit store -- attention_probs * head_mask
 * applied after the P V product -- so 1.0 gives the ungated bits exactly and 0 an exact zero context.  Packed attention maps
 * (VB200_OUT_ATTENTION_PACKED) report g * p, and under the head mean the mean of the gated maps.  The gate also holds in the pruned
 * last layers.  The mask is copied into the plan's gate table with one device-to-device copy on cuda_stream ahead of the forward, so
 * back-to-back calls may pass different masks without synchronising.  Gate values are device memory and are not checked.
 * A gated call runs a plan of its own (the PACKED plan's key plus gating), which launches the same kernels as the ungated plan and no
 * more; ungated calls keep their plans.  Everything else -- arguments, outputs, rejections -- follows vb200_forward_packed /
 * vb200_forward_regions_packed; a NULL head_mask is VB200_ERR_INVALID as well, and split_fp32 engines reject both calls as they
 * reject every packed call.  Dense, cached and retrieval forwards have no head mask. */
int vb200_forward_packed_gated(vb200_handle h, const vb200_packed_inputs* in, const float* head_mask /* DEVICE [batch, E, H] */,
                               const vb200_outputs* out, uint32_t select, int32_t slot, void* cuda_stream);
int vb200_forward_regions_packed_gated(vb200_handle h, const vb200_packed_region_inputs* in,
                                       const float* head_mask /* DEVICE [batch, E, H] */, const vb200_outputs* out, uint32_t select,
                                       int32_t slot, void* cuda_stream);

/* ---- Caption-image retrieval with reuse (SURVEY.md section 8e; reference semantics worker.py:278-284, 359).  Everything ahead of
 * the first connection layer depends on the caption alone or on the image alone: encode each caption / image ONCE, then score
 * pairs from the cached states.  Same kernels on the same rows as the full forward: scores are bit-identical to vb200_forward.
 * State buffers are caller-allocated device memory: fp32 [n, L, hidden], 16-bit [n, L, hidden * operand_width_factor] (2 bytes per
 * element; vb200_model_dim "operand_width_factor" is 1, or 3 in split_fp32 mode) and the additive mask fp32 [n, L], with
 * L = n_tokens + 1 (task token) for text and L = n_regions for images. */
int vb200_encode_text(vb200_handle h, int32_t n, int32_t n_tokens, const int64_t* question, const int64_t* segment_ids,
                      const int64_t* input_mask, const int64_t* task_tokens, float* state_f32, void* state_16, float* state_mask,
                      void* cuda_stream);
int vb200_encode_image(vb200_handle h, int32_t n, int32_t n_regions, const float* features, const float* spatials,
                       const uint8_t* image_mask, float* state_f32, void* state_16, float* state_mask, void* cuda_stream);
/* Pair b = (caption text_index[b], image image_index[b]); index arrays are device int32. */
int vb200_forward_cached(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, const int32_t* text_index,
                         int32_t n_text, const float* text_f32, const void* text_16, const float* text_mask,
                         const int32_t* image_index, int32_t n_image, const float* image_f32, const void* image_16,
                         const float* image_mask, const vb200_outputs* out, uint32_t select, int32_t slot, void* cuda_stream);

/* ---- Packed caption-image retrieval: the reuse above with every caption and image at its own length, stored back to back as in
 * vb200_packed_inputs, with no padding and no masks: every row is real.  Caption c's state is rows [sum_{c' < c} T_c', ... + T_c) with
 * T_c = Tin_c + 1 (task token); image i's state is rows [sum_{i' < i} V_i', ... + V_i).  State buffers are caller-allocated device
 * memory: fp32 [sum rows, hidden] and 16-bit [sum rows, hidden] (2 bytes per element).  Each caption's / image's rows are bit-identical
 * to vb200_encode_text / vb200_encode_image of that item alone at its own length.  Capacities follow vb200_forward_packed: 0 means
 * this call's maximum, and plans are keyed on round16 of the capacity.  VB200_ERR_INVALID for split_fp32 engines, NULL pointers, a
 * length < 1 or above a non-zero capacity, T or V above max_rows_per_sample and Tin > max_position_embeddings. */
int vb200_encode_text_packed(vb200_handle h, int32_t n, int32_t max_tokens, const int32_t* n_tokens /* HOST [n] Tin_c */,
                             const int64_t* question /* DEVICE [sum Tin_c] */, const int64_t* segment_ids /* DEVICE [sum Tin_c] */,
                             const int64_t* task_tokens /* DEVICE [n, 1] */, float* state_f32, void* state_16, void* cuda_stream);
int vb200_encode_image_packed(vb200_handle h, int32_t n, int32_t max_regions, const int32_t* n_regions /* HOST [n] V_i */,
                              const float* features /* DEVICE [sum V_i, v_feature_size] */, const float* spatials /* DEVICE [sum V_i, 5] */,
                              float* state_f32, void* state_16, void* cuda_stream);
/* vb200_encode_image_packed from detector output, as vb200_forward_regions_packed takes it: image i has n_boxes_i box feature rows and
 * pixel boxes, back to back, and its size in image_wh.  Its state is V_i = n_boxes_i + 1 rows, the global mean row first, in the layout
 * above (vb200_forward_cached_packed reads it unchanged).  The same region-pack kernel as vb200_forward_regions_packed writes the rows,
 * in front of the plan of vb200_encode_image_packed at max_regions = max_boxes + 1 (one plan serves both calls), so scores from these
 * states are bit-identical to vb200_forward_regions_packed of the same (caption, image) pairs.  max_boxes: plan capacity in boxes,
 * 0 -> this call's maximum.  VB200_ERR_INVALID, with nothing enqueued, for split_fp32 engines, NULL pointers, n_boxes_i < 1 or above
 * a non-zero max_boxes, a negative max_boxes and V_i above max_rows_per_sample. */
int vb200_encode_regions_packed(vb200_handle h, int32_t n, int32_t max_boxes, const int32_t* n_boxes /* HOST [n] */,
                                const float* box_features /* DEVICE [sum n_boxes_i, v_feature_size] */,
                                const float* boxes /* DEVICE [sum n_boxes_i, 4] pixels */, const float* image_wh /* DEVICE [n, 2] */,
                                float* state_f32, void* state_16, void* cuda_stream);
/* Pair b = (caption text_index[b], image image_index[b]) from packed states.  The index arrays and state offsets are HOST arrays (the
 * engine validates them and builds the plan's offsets on the host); the per-call offsets reach the plan's workspace on cuda_stream
 * through a pinned staging buffer, and one kernel gathers every pair's rows from the states.  Outputs follow vb200_forward_packed:
 * per-pair outputs keep their shapes, per-row outputs come back packed.  Scores are bit-identical to vb200_forward_packed of the same
 * pairs, which is bit-identical to a dense forward of each pair alone at its own (Tin_c, V_i).  VB200_ERR_INVALID for
 * VB200_OUT_ATTENTION, split_fp32 engines, NULL pointers, an index outside [0, n_text) / [0, n_image), offsets that do not increase
 * (a state of 0 rows included), a length above a non-zero capacity, T or V above max_rows_per_sample and Tin > max_position_embeddings. */
typedef struct {
    int32_t batch;                  /* B pairs */
    int32_t max_tokens, max_regions;   /* plan capacities (Tin and V units, as vb200_packed_inputs); 0 -> this call's maxima */
    const int32_t* text_index;      /* HOST [B] caption of pair b */
    const int32_t* image_index;     /* HOST [B] image of pair b */
    int32_t n_text;  const int32_t* text_offsets;   /* HOST [n_text + 1] state row offsets (rows T_c = Tin_c + 1) */
    const float* text_f32;  const void* text_16;    /* DEVICE packed text states from vb200_encode_text_packed */
    int32_t n_image; const int32_t* image_offsets;  /* HOST [n_image + 1] */
    const float* image_f32; const void* image_16;   /* DEVICE packed image states from vb200_encode_image_packed */
} vb200_packed_pairs;
int vb200_forward_cached_packed(vb200_handle h, const vb200_packed_pairs* in, const vb200_outputs* out, uint32_t select,
                                int32_t slot, void* cuda_stream);

/* ---- Answer decode: the step of prediction() that turns logits into answers (worker.py:295-386), for every message of a batch in
 * one kernel (one CTA per message).  Message i's segment is rows [first, first + count) of its family's source, flattened; the kernel
 * computes the softmax over the segment in fp32 as torch.softmax(x.view(-1), 0) does (max, expf(x - max), sum, division by the sum)
 * and writes the top_n probabilities and their indices in the segment.  Ties: equal probabilities rank the lower index first.
 *
 *   family                    source (vb200_outputs)   rows of the source                          segment width  reference
 *   VB200_DECODE_VQA          vil_prediction           batch                                       num_labels     worker.py:296
 *   VB200_DECODE_GQA          vil_prediction_gqa       batch                                       gqa_labels     worker.py:313
 *   VB200_DECODE_NLVR2        vil_binary_prediction    batch / 2 (batch even), else batch (pairs)  2              worker.py:329
 *   VB200_DECODE_SNLI_VE      vil_tri_prediction       batch                                       3              worker.py:345
 *   VB200_DECODE_RETRIEVAL    vil_logit                batch                                       1              worker.py:359
 *   VB200_DECODE_GROUNDING    vision_logit + spatials  vision_rows                                 1              worker.py:374-385
 *
 * The per-image families take one row (count 1) in the reference's decode, retrieval the request's count images (top_n = count), an
 * NLVR2 pair its pair row (image row lo of the pair -> pair row lo / 2).  Grounding reads vision_logit and spatials as flat [rows, 1]
 * and [rows, 5], which serves dense outputs (image b is rows b * V ... b * V + V - 1) and packed ones (image b is its packed rows)
 * alike; the segment is the image's rows, the global box included.  For each of the top_n rows the kernel writes box = x1, y1, x2, y2:
 * spatials columns 0-3 converted to double, times the double image_w / image_h, truncated toward zero -- the reference's
 * int(b[1] * image_h) on Python floats (worker.py:381-384).  Labels (worker.py:299-300, 311-315) and the confidence * 100 /
 * round(..., 2) of callback() (worker.py:571, 599, 617, 637) stay with the caller. */
#define VB200_DECODE_MAX_TOP 10
typedef enum {
    VB200_DECODE_VQA = 1,          /* task ids 1, 2 */
    VB200_DECODE_GQA = 2,          /* task id 15 */
    VB200_DECODE_NLVR2 = 3,        /* task id 12 */
    VB200_DECODE_SNLI_VE = 4,      /* task id 13 */
    VB200_DECODE_RETRIEVAL = 5,    /* task id 7 */
    VB200_DECODE_GROUNDING = 6     /* task ids 4, 16, 11 */
} vb200_decode_family;

typedef struct {
    int32_t family;                /* vb200_decode_family */
    int32_t first;                 /* first row of the source */
    int32_t count;                 /* rows of the segment (>= 1) */
    int32_t top_n;                 /* 1 .. min(VB200_DECODE_MAX_TOP, count * segment width) */
    double image_w, image_h;       /* grounding only: the image size in pixels */
} vb200_decode_msg;

typedef struct vb200_answer {
    int32_t n;                                  /* top_n */
    int32_t index[VB200_DECODE_MAX_TOP];        /* position in the flattened segment, best first; -1 past n */
    float prob[VB200_DECODE_MAX_TOP];           /* softmax probability; 0 past n */
    int32_t box[VB200_DECODE_MAX_TOP][4];       /* grounding: pixel x1, y1, x2, y2 of row `index`; 0 otherwise */
} vb200_answer;

/* Decodes n messages of one forward's outputs: `out` holds the device pointers that forward wrote (only the sources of the families
 * used are read), `batch` its per-sample row count, `vision_rows` the rows of vision_logit and of `spatials` (DEVICE fp32 [vision_rows, 5],
 * required for grounding).  Every descriptor is checked on the host before anything is enqueued: VB200_ERR_INVALID, with a message
 * naming the message index, for n < 1, an unknown family, count < 1, a row range outside its source, top_n < 1, above
 * VB200_DECODE_MAX_TOP or above the segment length, and a NULL source for a family that is used.  The descriptors reach the device
 * through a pinned staging buffer, asynchronously on cuda_stream: the call blocks only while the previous call's copy out of that
 * buffer is still in flight (and when a batch larger than any before grows that buffer), so back-to-back calls need no synchronisation
 * in between.  `answers` is DEVICE memory [n], complete once cuda_stream reaches the point of the call. */
int vb200_decode_answers(vb200_handle h, const vb200_decode_msg* msgs /* HOST [n] */, int32_t n, const vb200_outputs* out, int32_t batch,
                         int32_t vision_rows, const float* spatials, vb200_answer* answers /* DEVICE [n] */, void* cuda_stream);
/* The same with `answers` in HOST memory: the answers are copied back and cuda_stream is synchronised before the call returns.  The
 * form a C worker uses: forward, then this call, then the label lookup. */
int vb200_decode_answers_host(vb200_handle h, const vb200_decode_msg* msgs /* HOST [n] */, int32_t n, const vb200_outputs* out,
                              int32_t batch, int32_t vision_rows, const float* spatials, vb200_answer* answers /* HOST [n] */,
                              void* cuda_stream);

/* ---- Answer ablation: how much each question token and each detector box holds up one answer, from forwards alone.  For every
 * sample of a packed detector-output batch (laid out exactly as for vb200_forward_regions_packed), the engine builds on the device the
 * variants below, runs them all as one packed forward and scores each variant's head row against the attributed answer.
 *   Variants of sample i, in this order: the unablated input; then for each question position p in [token_begin, token_end) the
 *   input with question[p] replaced by mask_token (segment and task ids unchanged); then for each box j in [box_begin, box_end) the
 *   detector output without box j: n_boxes_i - 1 boxes, the ones after j moved up, the global mean row the mean of the remaining
 *   boxes summed in the order the region pack sums them.  Samples follow each other in batch order; the variant count is
 *   sum_i (1 + (token_end - token_begin) + (box_end - box_begin)) <= VB200_ABLATION_MAX_VARIANTS.
 *   Bit-identity: every variant's logits equal those of vb200_forward_regions_packed run on that variant's input alone.
 *   family: VB200_DECODE_VQA, _GQA or _SNLI_VE (one row of one image per answer).  NLVR2 (two images per answer), retrieval (many
 *   images per answer) and grounding (the answer is a box a variant may remove) are rejected.
 *   variant_logits (DEVICE, required): fp32 [n_variants, width], each variant's row of the family's head (width num_labels,
 *   gqa_labels or 3).  scores (DEVICE, optional, NULL skips them): one vb200_ablation_score per variant.  The softmax follows
 *   vb200_decode_answers (max, expf(x - max), the sum, a division; equal probabilities rank the lower index first), so every
 *   probability equals what vb200_decode_answers reports for that index of the same logits.  answer = -1 resolves to the
 *   unablated variant's top-1, and every variant of the sample reports against that column.
 * The variants run on the PACKED plan of vb200_forward_packed: the count is rounded up to a multiple of 64 with filler variants
 * (sample 0's first token and first box, outputs discarded), so a server keeps one plan per bucket and capacities.  max_tokens /
 * max_boxes are the plan's capacities as for vb200_forward_regions_packed (0: this call's maxima); spatials_out is not used.  The
 * plan's workspace grows with the bucket times the capacities: at 1024 variants and the default 256-row bound, some GB.  A caller
 * with more variants splits the ranges across calls.
 * VB200_ERR_INVALID, with nothing enqueued, no output written and a message naming the sample, for: split_fp32 and pre-training
 * engines; an excluded or unknown family; a range outside [0, Tin_i] / [0, n_boxes_i] or reversed; box ablation on an image with
 * fewer than 2 boxes; mask_token outside [0, vocab); answer outside [-1, width); more than VB200_ABLATION_MAX_VARIANTS variants;
 * NULL required pointers; box_features not 16-byte aligned; variant_logits or scores not 4-byte aligned; and every length rule of
 * vb200_forward_regions_packed.
 * Asynchronous on cuda_stream: the variant descriptors reach the device through engine-owned pinned staging and the variants' ids
 * live in an engine-owned workspace, both stream-ordered, so back-to-back calls need no synchronisation. */
#define VB200_ABLATION_MAX_VARIANTS 1024
typedef struct {
    int32_t answer;                   /* column of the family's head to attribute; -1: the unablated forward's top-1 */
    int32_t token_begin, token_end;   /* mask question positions [token_begin, token_end) of the sample's Tin ids, one at a time */
    int32_t box_begin, box_end;       /* drop boxes [box_begin, box_end) of the sample's n_boxes, one at a time */
} vb200_ablation_msg;

typedef struct {
    int32_t answer;                   /* the attributed column (answer -1 resolved) */
    float prob;                       /* its softmax probability in this variant */
    int32_t top1;                     /* this variant's own top-1 column */
    float top1_prob;                  /* and its probability */
} vb200_ablation_score;

int vb200_answer_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_ablation_msg* msgs /* HOST [batch] */,
                          int32_t family, int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot,
                          void* cuda_stream);

/* ---- Message ablation: answer ablation for every decode family, the answers of several images included.  The batch is a packed
 * detector-output batch laid out as the worker lays it out for vb200_forward_regions_packed (the text repeated per image, an NLVR2
 * pair on an even sample); each message names one answer by its images and is ablated one unit at a time.
 *   Message m reads samples [image_begin, image_begin + n_images) of the batch: VQA / GQA / SNLI-VE and grounding 1 image, NLVR2 2,
 *   retrieval K >= 1.  Its question, segment ids and task id are image_begin's (the other samples' text is not read).  Its segment
 *   is what vb200_decode_answers reads for it: the head row (width num_labels / gqa_labels / 3), the pair's vil_binary_prediction row
 *   (2), the K vil_logit values (K), or the image's vision_logit rows, the global row first (n_boxes + 1).  answer: an index in the
 *   segment (-1: the unablated top-1).  Boxes are numbered across the message's images in order.
 *   Variants of message m, in this order: the unablated input; each masked question position of [token_begin, token_end) (every
 *   image of the message with the masked question); each dropped box of [box_begin, box_end).  A dropped box runs both images for
 *   NLVR2 (the pair head reads adjacent pooled rows) and only the changed image otherwise: a retrieval box variant's segment is the
 *   unablated segment with element k (the changed image) replaced by that sample's vil_logit, exact because a packed sample's outputs
 *   do not depend on its neighbours; a grounding box variant's segment has n_boxes rows.
 *   vb200_message_ablation_layout owns the variant order: it writes one vb200_ablation_variant per variant (variants HOST, or NULL
 *   for the counts alone) and the totals: variants, floats of variant_logits and forward samples.  It checks the messages against
 *   the lengths as vb200_message_ablation does, without the sample cap.
 *   variant_logits (DEVICE, required): the segments back to back in layout order.  Bit-identity: every segment equals the same
 *   floats of vb200_forward_regions_packed run on that variant's input in the worker's layout (a retrieval box variant: all K images).
 *   scores (DEVICE, optional): one vb200_ablation_score per variant, with the arithmetic of vb200_answer_ablation.  Grounding reports
 *   answer and top1 in the unablated image's row numbering (a row after the dropped box maps back by +1); a variant that drops the
 *   attributed box reports answer -1 and prob 0.
 * The forward samples (at most VB200_ABLATION_MAX_VARIANTS per call; NLVR2 variants first, so each pair starts on an even sample) run
 * as one forward of the PACKED plan, rounded up to a multiple of 64 with fillers.  The plan selects the five pooled task heads, and
 * vision_logit as well when a message is a grounding message, so a server keeps at most two plans per bucket and capacities.
 * VB200_ERR_INVALID, with nothing enqueued, no output written and a message naming the message, for: split_fp32 and pre-training
 * engines; n_msgs < 1; an unknown family; n_images wrong for the family; an image range outside the batch; answer outside [-1,
 * segment length); a token range outside [0, Tin] or a box range outside [0, the message's boxes], or reversed; dropping a box of an
 * image with fewer than 2 boxes; mask_token outside [0, vocab); more than VB200_ABLATION_MAX_VARIANTS samples; NULL required pointers;
 * box_features not 16-byte aligned; and every length rule of vb200_forward_regions_packed.
 * Asynchronous and stream-ordered as vb200_answer_ablation. */
typedef struct {
    int32_t family;                   /* VB200_DECODE_* */
    int32_t image_begin, n_images;    /* the message's images: samples [image_begin, image_begin + n_images) of the batch */
    int32_t answer;                   /* attributed index in the message's segment; -1: the unablated top-1 */
    int32_t token_begin, token_end;   /* mask question positions [token_begin, token_end) of image_begin's Tin ids, one at a time */
    int32_t box_begin, box_end;       /* drop boxes [box_begin, box_end), numbered across the message's images in order, one at a time */
} vb200_ablation_message;

typedef struct {
    int32_t message, kind, unit;      /* kind 0: the unablated input (unit -1); 1: masked position `unit`; 2: dropped box `unit`;
                                         3 (head ablation): gate `unit` = entry * head_mask_heads + head at 0;
                                         4 (coalition ablation): coalition `unit` of the message */
    int32_t samples;                  /* forward samples this variant runs */
    int64_t offset;                   /* its segment: floats [offset, offset + length) of variant_logits */
    int32_t length;
} vb200_ablation_variant;

int vb200_message_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens /* HOST [batch] */,
                                  const int32_t* n_boxes /* HOST [batch] */, const vb200_ablation_message* msgs /* HOST [n_msgs] */,
                                  int32_t n_msgs, vb200_ablation_variant* variants /* HOST, NULL: counts only */, int64_t* n_variants,
                                  int64_t* n_floats, int64_t* n_samples);
int vb200_message_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_ablation_message* msgs /* HOST [n_msgs] */,
                           int32_t n_msgs, int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot,
                           void* cuda_stream);

/* ---- Head ablation (Michel et al. 2019): which attention heads an answer depends on.  Messages follow vb200_message_ablation (every
 * decode family, the same images per message and answer rule) with an entry range instead of token and box ranges.  A message's
 * variants, in order: the unablated input (kind 0, unit -1), then for each entry e in [entry_begin, entry_end) (the head mask's entry
 * order, see vb200_forward_packed_gated) and each of that entry's heads h, the message's samples unablated with gate (e, h) at 0 and
 * every other gate at 1 (kind 3, unit e * head_mask_heads + h).  Every sample of the message runs in each variant: an NLVR2 variant is
 * a pair on an even sample, a retrieval variant all K images.  The variants are built on the device (text and regions as message
 * ablation builds its unablated input, one kernel writing each sample's gate row) and run as one forward of the gated PACKED plan,
 * rounded up to a multiple of 64 samples with fillers (gate 1), at most VB200_ABLATION_MAX_VARIANTS samples per call.  Segments and
 * scores follow vb200_message_ablation: every segment is bit-identical to the same floats of vb200_forward_regions_packed_gated run on
 * the variant's input and gate row alone.  vb200_head_ablation_layout owns the variant order, as vb200_message_ablation_layout does.
 * Every head of one message: 1 + 288 = 289 forward samples for 12/6/6 (578 for NLVR2).
 * VB200_ERR_INVALID, with nothing enqueued, for every rejection of vb200_message_ablation that applies (mask_token aside) and an
 * entry range reversed or outside [0, head_mask_entries]. */
typedef struct {
    int32_t family;                   /* VB200_DECODE_* */
    int32_t image_begin, n_images;    /* the message's images in the batch, as vb200_ablation_message */
    int32_t answer;                   /* attributed index, -1: the unablated top-1 */
    int32_t entry_begin, entry_end;   /* remove each head of entries [entry_begin, entry_end), one at a time */
} vb200_head_ablation_message;

int vb200_head_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens /* HOST [batch] */,
                               const int32_t* n_boxes /* HOST [batch] */, const vb200_head_ablation_message* msgs /* HOST [n_msgs] */,
                               int32_t n_msgs, vb200_ablation_variant* variants /* HOST, NULL: counts only */, int64_t* n_variants,
                               int64_t* n_floats, int64_t* n_samples);
int vb200_head_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_head_ablation_message* msgs /* HOST [n_msgs] */,
                        int32_t n_msgs, float* variant_logits, vb200_ablation_score* scores, int32_t slot, void* cuda_stream);

/* ---- Coalition ablation: the answer with any set of units removed at once, the inputs of Shapley values and of any other
 * coalition-based attribution.  Messages follow vb200_message_ablation (family, images, answer) for VQA, GQA, SNLI-VE, NLVR2 and
 * retrieval; grounding is rejected (its answer is a box, which a coalition would renumber).
 *   Units: unit u of a message is a non-empty set of question positions of image_begin's Tin ids (positions[position_offsets[u] ..
 *   position_offsets[u + 1])) plus a set of boxes numbered across the message's images in order (boxes[box_offsets[u] ..
 *   box_offsets[u + 1])).  No position or box belongs to two units, or twice to one; 1 <= n_units <= VB200_COALITION_MAX_UNITS.
 *   Positions and boxes in no unit are never removed.
 *   Coalitions: coalition c is words [c * W, c * W + W) of `coalitions`, W = ceil(n_units / 64): bit u % 64 of word u / 64 set marks
 *   unit u PRESENT.  A coalition input removes every absent unit: its positions are replaced by mask_token in every image's question
 *   (segment and task ids unchanged), and each of its boxes is dropped from its own image -- the kept boxes stay in their order, and
 *   the global mean row is their mean summed in the order the region pack sums any image.  An image left with no box is the global
 *   row alone: zero features and location [0, 0, 1, 1, 1] (the mean divides by max(boxes, 1)).
 *   Variants of message m, in order: the full input (kind 0, unit -1), then its coalitions in the caller's order (kind 4, unit = the
 *   coalition's index).  Every variant runs every sample of the message (an NLVR2 pair on an even sample, all K retrieval images),
 *   and its segment is the message's segment as vb200_message_ablation gathers it.  Bit-identity: every segment equals the same
 *   floats of vb200_forward_regions_packed run on that coalition's input in the worker's layout.
 *   scores (DEVICE, optional): one vb200_ablation_score per variant with the arithmetic of vb200_answer_ablation; answer -1 resolves
 *   to the full input's top-1, and a coalition's prob is its value v(S).
 * vb200_coalition_ablation_layout writes the records and totals as vb200_message_ablation_layout does.  The samples (at most
 * VB200_ABLATION_MAX_VARIANTS per call, NLVR2 messages first) run as one forward of the PACKED plan message ablation uses, rounded up
 * to a multiple of 64 with fillers; the masked-position bitmaps and kept-box lists are staged with the other descriptors.
 * VB200_ERR_INVALID, with nothing enqueued and a message naming the message or unit, for every rejection of vb200_message_ablation
 * that applies (split_fp32 and pre-training engines included), grounding, n_units outside [1, VB200_COALITION_MAX_UNITS], n_coalitions
 * < 0, an empty unit, a position outside [0, Tin) or a box outside [0, the message's boxes), a position or box in two units, a
 * coalition bit at or past n_units, and NULL unit or coalition arrays.  Asynchronous and stream-ordered as vb200_answer_ablation. */
#define VB200_COALITION_MAX_UNITS 1024
typedef struct {
    int32_t family;                   /* VB200_DECODE_* except grounding */
    int32_t image_begin, n_images;    /* the message's images in the batch, as vb200_ablation_message */
    int32_t answer;                   /* attributed index in the message's segment; -1: the full input's top-1 */
    int32_t n_units;
    const int32_t* position_offsets;  /* HOST [n_units + 1], from 0 */
    const int32_t* positions;         /* HOST: each unit's question positions */
    const int32_t* box_offsets;       /* HOST [n_units + 1], from 0 */
    const int32_t* boxes;             /* HOST: each unit's boxes, numbered across the message's images */
    int32_t n_coalitions;
    const uint64_t* coalitions;       /* HOST [n_coalitions, ceil(n_units / 64)] presence bitmaps */
} vb200_coalition_message;

int vb200_coalition_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens /* HOST [batch] */,
                                    const int32_t* n_boxes /* HOST [batch] */, const vb200_coalition_message* msgs /* HOST [n_msgs] */,
                                    int32_t n_msgs, vb200_ablation_variant* variants /* HOST, NULL: counts only */, int64_t* n_variants,
                                    int64_t* n_floats, int64_t* n_samples);
int vb200_coalition_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_coalition_message* msgs /* HOST [n_msgs] */,
                             int32_t n_msgs, int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot,
                             void* cuda_stream);

/* ---- Shapley values from permutation-sampled coalition values, on the device (one CTA per message, float64 throughout).
 * Message i has n = n_units units, P = n_perm permutations and groups of g = group consecutive permutations (1, or 2 for antithetic
 * pairs; g divides P).  perm + perm_offset: DEVICE int32 [P, n], each row a permutation of 0 .. n-1.  values + value_offset: DEVICE
 * fp32 [2 + P (n - 1)]: v(empty), v(all), then for p = 0 .. P-1 the chain v(S^p_1) .. v(S^p_{n-1}), S^p_j the first j units of row p.
 * With c[p][0] = v(empty), c[p][n] = v(all), c[p][j] = chain value j of row p, every value widened to double:
 *   d[p][u] = c[p][j + 1] - c[p][j] for u = perm[p][j];
 *   s = 0; for p = 0 .. P-1: s = s + d[p][u];              phi_u = s / P;
 *   G = P / g; for q = 0 .. G-1: m = 0; for i = 0 .. g-1: m = m + d[q g + i][u];  m = m / g;  t = m - phi_u;  ss = ss + t * t
 *     (ss from 0);
 *   stderr_u = sqrt((ss / (G - 1)) / G), NaN when G < 2.
 * Each step is one correctly rounded float64 operation in that order (no fused multiply-add), so a numpy restatement in float64
 * reproduces it bit for bit.  phi + out_offset and stderr + out_offset: DEVICE fp32 [n], the float64 results rounded to nearest.  A
 * permutation row that is not a permutation gives NaN in both outputs for every unit of its message.
 * VB200_ERR_INVALID, with nothing enqueued, for n_msgs < 1, n_units outside [1, VB200_COALITION_MAX_UNITS], n_perm < 1, group not 1
 * or 2, n_perm not a multiple of group, a negative offset, NULL pointers, or phi / stderr / values not 4-byte aligned.  The
 * descriptors are staged as vb200_decode_answers stages its messages; asynchronous on cuda_stream. */
typedef struct {
    int32_t n_units, n_perm, group;
    int64_t perm_offset;              /* int32 elements of perm where the message's [n_perm, n_units] table starts */
    int64_t value_offset;             /* floats of values where its 2 + n_perm * (n_units - 1) values start */
    int64_t out_offset;               /* floats of phi and of stderr where its n_units outputs start */
} vb200_shapley_message;

int vb200_shapley_values(vb200_handle h, const vb200_shapley_message* msgs /* HOST [n_msgs] */, int32_t n_msgs, const int32_t* perm,
                         const float* values, float* phi, float* stderr_out, void* cuda_stream);

/* ---- Shapley-Taylor interaction indices of order 2 (Sundararajan, Dhamdhere & Agarwal 2020) from the same permutation chains, on
 * the device (float64 throughout): which pairs of units an answer needs together (> 0) or either of (< 0).  For a pair {a, b} the
 * index is the mean over permutations of v(S + {a, b}) - v(S + {a}) - v(S + {b}) + v(S), S the units before the first of a and b.
 * Message i has n = n_units >= 2 units, P = n_perm permutations in groups of g = group (as vb200_shapley_values) and Q = n_pairs
 * pairs (a, b), a != b, both in [0, n).  perm + perm_offset as vb200_shapley_values.  values + value_offset: DEVICE fp32
 * [2 + P (n - 1) + 2 P Q]: the 2 + P (n - 1) values vb200_shapley_values reads (so the same value_offset serves both calls), then for
 * p = 0 .. P-1 and q = 0 .. Q-1 the pair x1[p][q] at 2 + P (n - 1) + 2 (p Q + q) and x2[p][q] right after it.  With r the smaller of
 * pair q's two ranks in row p (rank: the unit's position in the row), S the first r units of row p and "second" whichever of a, b has
 * the larger rank: x1[p][q] = v(S + {second}), x2[p][q] = v(S + {a, b}).  With c[p][j] as in vb200_shapley_values and every value
 * widened to double:
 *   d[p][q] = ((x2[p][q] - c[p][r + 1]) - x1[p][q]) + c[p][r];
 *   s = 0; for p = 0 .. P-1: s = s + d[p][q];              I_q = s / P;
 *   G = P / g; for k = 0 .. G-1: m = 0; for i = 0 .. g-1: m = m + d[k g + i][q];  m = m / g;  t = m - I_q;  ss = ss + t * t
 *     (ss from 0);
 *   stderr_q = sqrt((ss / (G - 1)) / G), NaN when G < 2.
 * Each step is one correctly rounded float64 operation in that order (no fused multiply-add), so a numpy restatement in float64
 * reproduces it bit for bit; (a, b) and (b, a) give the same bits, since r and "second" follow the ranks.  inter + out_offset and
 * stderr + out_offset: DEVICE fp32 [Q], the float64 results rounded to nearest.  A permutation row that is not a permutation gives
 * NaN in both outputs for every pair of its message.  Pair q's first and second differences come from four values:
 * c[p][r] = v(S), c[p][r + 1] = v(S + {first}) from the chain, x1 and x2 from two more coalitions per permutation and pair.
 * VB200_ERR_INVALID, with nothing enqueued and a message naming the message or pair, for every rejection of vb200_shapley_values,
 * n_units < 2, n_pairs < 1, more than VB200_INTERACTION_MAX_PAIRS pairs over all messages, NULL pairs, and a pair with a == b or an
 * index outside [0, n).  The pairs are staged with the descriptors; asynchronous on cuda_stream. */
#define VB200_INTERACTION_MAX_PAIRS 65536     /* pairs per call, all messages together */
typedef struct {
    int32_t n_units, n_perm, group, n_pairs;
    int64_t perm_offset;              /* int32 elements of perm where the message's [n_perm, n_units] table starts */
    int64_t value_offset;             /* floats of values where its 2 + P (n - 1) + 2 P Q values start (layout above) */
    int64_t out_offset;               /* floats of inter and of stderr_out where its n_pairs outputs start */
    const int32_t* pairs;             /* HOST [n_pairs, 2] unit indices (a, b) */
} vb200_interaction_message;

int vb200_interaction_values(vb200_handle h, const vb200_interaction_message* msgs /* HOST [n_msgs] */, int32_t n_msgs,
                             const int32_t* perm, const float* values, float* inter, float* stderr_out, void* cuda_stream);

/* ---- Detector-region selection: the feature extraction step of the reference worker (worker.py:123-176) on the detector's raw heads,
 * for every image of a batch in one call, written straight into the packed box_features / boxes that vb200_forward_regions_packed reads.
 * For image i with n_i proposals, C score columns (column 0 is background) and features [n_i, F]:
 *   p = softmax(scores_i) per proposal row (fp32: max, expf(x - max), sum, division by the sum);
 *   dets = proposals_i / (float)im_scale_i (fp32 division: the original-pixel boxes);
 *   max_conf[b] = the largest p[b, c] over the classes c >= start (start = 0 with background, else 1) whose NMS keeps b and with
 *     p[b, c] > conf_thresh, else 0.  NMS: greedy in descending score order; IoU with the legacy "+1": w = max(min(x2) - max(x1) + 1, 0),
 *     the same for h, areas (x2 - x1 + 1)(y2 - y1 + 1), IoU = inter / (Sa + Sb - inter), each step rounded in fp32; suppression when
 *     IoU > nms_iou;
 *   keep = the first k_i = min(max_boxes, n_i) indices of max_conf in descending order.
 * Ties: equal scores rank the lower proposal index first, in every class's NMS order and in the final ranking.
 * Outputs of image i are rows [dst_row, dst_row + k_i) of each per-row output: box_features = features_i[keep], boxes = dets[keep],
 * and optionally keep_index, the sorted max_conf, cls_prob = p[keep] (full rows) and objects = argmax over all C columns of each
 * cls_prob row (ties: lower column).  num_boxes[i] = the count of nonzero max_conf among the k_i.  (The reference's objects is the
 * argmax of rows start .. k_i - 1 of p[keep]: objects[start:] of this output.)  Rows outside those ranges are not written, so a caller
 * can leave rows free for the filler images of a packed batch.
 * Limits: 1 <= n_i <= 2048, 2 <= C <= 2048, F a positive multiple of 4, 1 <= max_boxes <= max_rows_per_sample - 1 (255 by default), 0 < nms_iou <= 1, background 0 or 1,
 * 1 <= n <= 65535, im_scale > 0.  VB200_ERR_INVALID, with a message naming the image where there is one, for a limit broken, a NULL
 * required pointer, a features or box_features pointer not 16-byte aligned, and destination ranges that overlap or fall outside
 * [0, out_rows); nothing is enqueued then.
 * Asynchronous on cuda_stream.  The descriptors reach the device through a pinned staging buffer, and the workspace (row stats, IoU
 * bitmasks, max_conf) is owned by the engine and grows on demand, in stream order.  The call blocks only while the previous call's copy
 * out of the staging buffer is still in flight (and when a batch larger than any before grows that buffer); a call's kernels wait on
 * the device for the previous call's, so back-to-back calls need no synchronisation in between. */
typedef struct {
    int32_t n_proposals;           /* n_i */
    int32_t dst_row;               /* first output row of image i */
    double im_scale;               /* detector input scale: boxes are proposals / (float)im_scale */
    const float* proposals;        /* DEVICE [n_i, 4] x1, y1, x2, y2 at the detector's input scale */
    const float* scores;           /* DEVICE [n_i, n_classes] class logits, as the detector returns them */
    const float* features;         /* DEVICE [n_i, feature_size] (fc6), 16-byte aligned */
} vb200_detections;

typedef struct {
    int32_t n_classes;             /* C, background column included (1601) */
    int32_t feature_size;          /* F (2048) */
    int32_t max_boxes;             /* K (the worker's num_features, 100) */
    float conf_thresh;             /* 0 in the worker */
    float nms_iou;                 /* 0.5 in the worker */
    int32_t background;            /* 1: class 0 takes part in the NMS (the worker's default is 0) */
    int32_t out_rows;              /* rows of the per-row outputs */
} vb200_select_params;

typedef struct {
    float* box_features;           /* required DEVICE [out_rows, F], 16-byte aligned */
    float* boxes;                  /* required DEVICE [out_rows, 4] original-pixel x1, y1, x2, y2 */
    int32_t* num_boxes;            /* required DEVICE [n] */
    int32_t* keep_index;           /* optional DEVICE [out_rows]: proposal index within its image */
    float* max_conf;               /* optional DEVICE [out_rows]: the sorted scores */
    float* cls_prob;               /* optional DEVICE [out_rows, C] */
    int64_t* objects;              /* optional DEVICE [out_rows] */
} vb200_selected;

int vb200_select_regions(vb200_handle h, const vb200_detections* imgs /* HOST [n] */, int32_t n, const vb200_select_params* p,
                         const vb200_selected* out, void* cuda_stream);

/* ---- Pre-training heads at chosen rows: the three ViLBERT objectives of the checkpoint's `cls` heads on the rows a caller lists, from
 * the fp32 final states a forward returns as taps (vb200_outputs.sequence_output_t / _v and pooled_output, dense B x T / B x V rows
 * or packed sum T_i / sum V_i rows; any forward that writes them).
 *   token_logits[i]  = cls.predictions (768 -> 768 GELU + LayerNorm, tied 768 -> vocab decoder + bias) of text row text_rows[i];
 *   region_logits[i] = cls.imagePredictions (1024 -> 1024 GELU + LayerNorm, 1024 -> v_target_size) of image row image_rows[i];
 *   alignment[i]     = cls.bi_seq_relationship (bi_hidden -> 2) of pooled row pair_rows[i] (pooled_output = pooled_t * pooled_v).
 * Each logits row is bit-identical to that row of the same forward run with VB200_OUT_LINGUISIC_PREDICTION / VB200_OUT_VISION_PREDICTION,
 * and each alignment row to element 3 (vil_binary_prediction) of a batch-1 forward of that pair: one kernel gathers the listed rows into
 * the 16-bit operand the forward's final LayerNorm writes, and the forward's GEMMs, LayerNorm and narrow-head kernels run on them at the
 * bucket of the listed rows (128 rows times a power of two; tiles past the call's count are skipped).  Which alignment column means
 * "matched" is upstream's convention; the engine returns both logits in the head's order.
 * token_top / region_top: per listed row, the softmax over its logits and the top_k indices (columns) and probabilities, in the
 * vb200_answer convention of vb200_decode_answers (equal probabilities: lower index first; box unused, 0).
 * Every group is optional: a list of 0 rows, or NULL outputs, skips it.  Duplicate rows are allowed.  Everything is checked on the
 * host before anything is enqueued: VB200_ERR_INVALID, with a message naming the list and the index, for a negative count, a row outside
 * its state's rows, a NULL state for a non-empty list, top_k < 0, above VB200_DECODE_MAX_TOP or above the width of a head whose top
 * output is requested, and a top output with top_k = 0.
 * Asynchronous on cuda_stream; no forward plan is built, used or evicted.  The row lists reach the device through a pinned staging
 * buffer: a call blocks only while the previous call's copy out of it is in flight, and when a larger bucket of rows appears for the
 * first time (its workspace and TMA descriptors are built once and kept), so back-to-back calls need no synchronisation in between. */
typedef struct {
    const float* text_state;       /* DEVICE fp32 [t_rows, hidden]: a forward's sequence_output_t */
    const float* image_state;      /* DEVICE fp32 [v_rows, v_hidden]: sequence_output_v */
    const float* pooled_state;     /* DEVICE fp32 [p_rows, bi_hidden]: pooled_output */
    int32_t t_rows, v_rows, p_rows;
    int32_t n_t, n_v, n_p;         /* entries of the three row lists */
    const int32_t* text_rows;      /* HOST [n_t] rows of text_state */
    const int32_t* image_rows;     /* HOST [n_v] rows of image_state */
    const int32_t* pair_rows;      /* HOST [n_p] rows of pooled_state */
    int32_t top_k;                 /* 0: no ranking; else 1 .. VB200_DECODE_MAX_TOP */
} vb200_pretrain_rows;

typedef struct {                   /* DEVICE outputs, each optional (NULL skips it) */
    float* token_logits;           /* [n_t, vocab] */
    float* region_logits;          /* [n_v, v_target_size] */
    float* alignment;              /* [n_p, 2] */
    vb200_answer* token_top;       /* [n_t] */
    vb200_answer* region_top;      /* [n_v] */
} vb200_pretrain_out;

int vb200_pretraining_heads(vb200_handle h, const vb200_pretrain_rows* in, const vb200_pretrain_out* out, void* cuda_stream);

/* ---- The three pre-training objectives at the rows a caller lists (upstream BertForMultiModalPreTraining's losses, visual_target 0),
 * from the same row lists and the same head launches as vb200_pretraining_heads (in->top_k must be 0).  With z the listed row's
 * logits, bit-identical to that row of vb200_pretraining_heads:
 *   token_loss[i]  = logsumexp(z) - z[token_labels[i]]                 (masked-token cross-entropy, text_rows[i])
 *   region_loss[i] = sum_c t_c (log t_c - log_softmax(z)_c), 0 log 0 = 0, t = image_targets row i   (KL divergence as
 *                    torch.nn.functional.kl_div computes it: a negative target gives NaN)
 *   pair_loss[i]   = logsumexp(z) - z[pair_labels[i]]                  (alignment cross-entropy, pair_rows[i])
 *   reduced[0..2]  = the mean of token_loss, region_loss and pair_loss: upstream's masked_lm_loss and next_sentence_loss
 *                    (CrossEntropyLoss over the rows whose label is not -1) and masked_img_loss (the KL summed over the classes of the
 *                    rows whose image_label is 1, divided by their count).  An empty list gives NaN (0 / 0, as upstream).
 * One CTA per listed row reads that row's logits; one CTA sums each list in a fixed order, so repeated calls give the same bits.
 * Every output is optional.  Everything is checked on the host before anything is enqueued: VB200_ERR_INVALID, naming the list or
 * the label and the index, for the row-list faults of vb200_pretraining_heads, top_k != 0, a token label outside [0, vocab), a pair
 * label other than 0 / 1, a NULL label list or target pointer for a non-empty list, a target or reduced pointer that is not 4-byte
 * aligned.  Asynchronous on cuda_stream; rows and labels are staged as vb200_pretraining_heads stages its rows, so back-to-back calls
 * need no synchronisation; no forward plan is built, used or evicted. */
typedef struct {
    const int32_t* token_labels;   /* HOST [n_t]: the vocabulary id of each text row */
    const float* image_targets;    /* DEVICE fp32 [n_v, v_target_size]: the target distribution of each image row */
    const int32_t* pair_labels;    /* HOST [n_p]: 0 / 1, the cross-entropy class of each pair row */
} vb200_pretrain_targets;

typedef struct {                   /* DEVICE fp32 outputs, each optional (NULL skips it) */
    float* token_loss;             /* [n_t] */
    float* region_loss;            /* [n_v] */
    float* pair_loss;              /* [n_p] */
    float* reduced;                /* [3]: masked_lm_loss, masked_img_loss, next_sentence_loss */
} vb200_pretrain_losses;

int vb200_pretraining_objectives(vb200_handle h, const vb200_pretrain_rows* in, const vb200_pretrain_targets* targets,
                                 const vb200_pretrain_losses* out, void* cuda_stream);

/* ---- Kernel-level entry points (device pointers), used by the parity tests and the roofline bench.  ---- */
/* y = act(x[M,K] (16-bit) . w[N,K]^T (16-bit) + bias); act: 0 none, 1 GELU(erf), 2 ReLU.  residual, gamma and beta are reserved
 * and must be NULL (VB200_ERR_INVALID otherwise; LayerNorm is vb200_layernorm on the fp32 output); ld_res and eps are ignored.
 * act_fp16 != 0: x, w and the 16-bit output y are fp16, else bf16 (parameter names keep the historical _bf16 suffix).
 * act 3 = GELU with the 1.5e-7 erf (fp32-parity mode).  variant 0: persistent kernel (gemm_persistent.cuh, what the engine
 * uses); 2, 3 and 4 (names of Blackwell kernel configurations) select the persistent kernel: 2 and 3 with the plain 128-wide tile,
 * 4 with the plain 128- or 64-wide one.  variant 5: the ping-pong kernel (gemm_pingpong.cuh, what the engine uses for the plain
 * GEMMs it supports): act 0-2, N a multiple of block_n 64 or 128, outputs the TMA can store (16-byte aligned
 * base and row stride); VB200_ERR_INVALID otherwise.  Tiles are 64, 128 or 192 columns wide; block_n 256 runs
 * as 128-wide tiles.  Every variant and every width gives the same bits.
 * timing: NULL, or a device buffer of 16 int64 per CTA that receives clock64() / %globaltimer stamps (profiling aid). */
int vb200_linear(const void* x_bf16, int64_t ld_x, const void* w_bf16, int64_t ld_w, const float* bias,
                 const float* residual, int64_t ld_res, const float* gamma, const float* beta, float eps, int32_t act,
                 void* y_bf16, int64_t ld_y_bf16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K,
                 int32_t block_n, int32_t use_pdl, int32_t act_fp16, int32_t variant, long long* timing, void* cuda_stream);
/* The GEMM of vb200_linear with a device row count: rows >= min(*m_rows, M) are neither loaded nor computed -- the
 * 128-row tiles that start at or past it are skipped, what packed plans rely on (m_rows: device int32).  Runs on the kernel the
 * engine would pick: ping-pong (variant 5) where it applies unless VB200_GEMM=coop, else variant 0. */
int vb200_linear_rows(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, void* y16,
                      int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K, int32_t block_n, int32_t act_fp16,
                      const int32_t* m_rows, void* cuda_stream);
/* The same GEMM on fp32-parity-mode operands (fp16 only): x16 holds hi | lo | hi and w16 hi | hi | lo per 64 logical columns, K3 is
 * the PHYSICAL contraction length (3x the logical one), y16 (optional) is written in the activation split layout (stride ld_y16 of
 * the 3x wider buffer), y_f32 (optional) as usual. */
int vb200_linear_split(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, void* y16,
                       int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K3, void* cuda_stream);
/* ctx = softmax(Q K^T / sqrt(d) + mask) V, qkv rows = [Q | K | V] (bf16), mask_add fp32 [B, L]. */
/* out = LayerNorm(y + residual) * gamma + beta over rows of N (N % 128 == 0, N <= 2048); fp32 and/or 16-bit outputs. */
int vb200_layernorm(const float* y, int64_t ld_y, const float* residual, int64_t ld_res, const float* gamma, const float* beta,
                    float eps, float* out_f32, int64_t ld_f32, void* out_16, int64_t ld_16, int64_t M, int64_t N,
                    int32_t act_fp16, void* cuda_stream);
/* split16 != 0: out_16 is the fp16 hi | lo | hi operand (stride ld_16 of the 3x wider buffer). */
int vb200_layernorm_split(const float* y, int64_t ld_y, const float* residual, int64_t ld_res, const float* gamma, const float* beta,
                          float eps, float* out_f32, int64_t ld_f32, void* out_16, int64_t ld_16, int64_t M, int64_t N, void* cuda_stream);
/* fp32 CUDA-core attention (attention_f32.cu): q / k / v point at head 0 of sample 0 (row strides ld_q, ld_kv; the three may alias
 * one QKV buffer), in_kind 0 fp32 / 1 fp16 / 2 bf16; ctx_mode 0 no context / 1 fp16 / 2 bf16 / 3 fp16 hi | lo | hi;
 * probs optional [B, heads, Lq, Lk]. */
int vb200_attention_f32(const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv, int32_t in_kind,
                        const float* key_mask_add, int32_t B, int32_t Lq, int32_t Lk, int32_t heads, int32_t head_dim, void* ctx,
                        int64_t ld_ctx, int32_t ctx_mode, float* probs, void* cuda_stream);
int vb200_self_attention(const void* qkv_bf16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx_bf16,
                         int64_t ld_ctx, int32_t B, int32_t L, int32_t heads, int32_t head_dim, int32_t act_fp16,
                         void* cuda_stream);
int vb200_co_attention(const void* qkv_img_bf16, int64_t ld_img, const void* qkv_txt_bf16, int64_t ld_txt,
                       int32_t hidden, const float* img_mask_add, const float* txt_mask_add, void* ctx_txt_bf16,
                       int64_t ld_ctx_txt, void* ctx_img_bf16, int64_t ld_ctx_img, int32_t B, int32_t T, int32_t V,
                       int32_t heads, int32_t head_dim, int32_t act_fp16, void* cuda_stream);
/* Packed self-attention: sample b is rows [offs[b], offs[b+1]) of qkv / mask_add / ctx (offs: device int32 [B + 1]); L_cap >= every
 * sample's length.  Each sample's rows are bit-identical to vb200_self_attention of that sample alone. */
int vb200_self_attention_packed(const void* qkv16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx16, int64_t ld_ctx,
                                int32_t B, int32_t L_cap, int32_t heads, int32_t head_dim, int32_t act_fp16, const int32_t* offs,
                                void* cuda_stream);
/* Packed co-attention: per stream as vb200_self_attention_packed (offs_t text rows, offs_v image rows; T_cap / V_cap capacities). */
int vb200_co_attention_packed(const void* qkv_img16, int64_t ld_img, const void* qkv_txt16, int64_t ld_txt, int32_t hidden,
                              const float* img_mask_add, const float* txt_mask_add, void* ctx_txt16, int64_t ld_ctx_txt, void* ctx_img16,
                              int64_t ld_ctx_img, int32_t B, int32_t T_cap, int32_t V_cap, int32_t heads, int32_t head_dim,
                              int32_t act_fp16, const int32_t* offs_t, const int32_t* offs_v, void* cuda_stream);
/* Streaming self- / co-attention, the kernels forwards use when a stream has more than 256 rows per sample: one CTA per 64 query
 * rows, K and V streamed through shared memory in 64-key blocks, so any length runs.  Arguments as the packed calls above; NULL
 * offsets mean a dense batch (sample b is rows [b L, b L + L) of its stream; for co-attention offs_t and offs_v are both NULL or
 * both set).  Wherever vb200_self_attention / vb200_co_attention (or their packed forms) accept the lengths, the context rows are
 * bit-identical to theirs. */
int vb200_self_attention_stream(const void* qkv16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx16, int64_t ld_ctx,
                                int32_t B, int32_t L_cap, int32_t heads, int32_t head_dim, int32_t act_fp16, const int32_t* offs,
                                void* cuda_stream);
int vb200_co_attention_stream(const void* qkv_img16, int64_t ld_img, const void* qkv_txt16, int64_t ld_txt, int32_t hidden,
                              const float* img_mask_add, const float* txt_mask_add, void* ctx_txt16, int64_t ld_ctx_txt, void* ctx_img16,
                              int64_t ld_ctx_img, int32_t B, int32_t T_cap, int32_t V_cap, int32_t heads, int32_t head_dim,
                              int32_t act_fp16, const int32_t* offs_t, const int32_t* offs_v, void* cuda_stream);
/* Pooled-product GEMM: y = act(x . w^T + bias) * mul (mul fp32 [M, ld_mul]) on the cooperative persistent kernel, as the engine's
 * pooler builds it; act 0-2, 16-bit and / or fp32 outputs. */
int vb200_linear_product(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, const float* mul,
                         int64_t ld_mul, void* y16, int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K,
                         int32_t block_n, int32_t act_fp16, void* cuda_stream);
/* Text embeddings: LayerNorm(word[id] + position + token_type[seg]), the task row at index 1 when task_tokens != 0, the additive text
 * mask; ids / segments / task ids are clamped into their tables and positions to max_pos - 1.  offs NULL: dense [B, Tin] inputs;
 * else packed (device int32 [B + 1] output row offsets, `rows` = offs[B], every row real).  split16: fp16 hi | lo | hi output. */
int vb200_text_embed(const int64_t* ids, const int64_t* seg, const int64_t* input_mask, const int64_t* task, const float* word,
                     const float* pos, const float* type, const float* task_tab, const float* gamma, const float* beta, float eps,
                     float* out_f32, void* out16, float* mask_add, int32_t B, int32_t Tin, int32_t H, int32_t vocab, int32_t max_pos,
                     int32_t n_type, int32_t n_task, int32_t task_tokens, int32_t act_fp16, int32_t split16, const int32_t* offs,
                     int32_t rows, void* cuda_stream);
/* Image operand: rows of [feats (F) | loc (5) | 0 ...] (Kp wide) in 16 bits, additive mask from image_mask (NULL: every row real). */
int vb200_image_pack(const float* feats, const float* loc, const uint8_t* image_mask, void* a_out, float* mask_add, int32_t rows,
                     int32_t F, int32_t Kp, int32_t act_fp16, int32_t split16, void* cuda_stream);
/* Detector output -> image operand rows [mean row | box rows], masks and optional spatials (vb200_forward_regions' input builder);
 * offs NULL: dense [B, n] boxes with optional num_boxes, else packed (device int32 [B + 1] image row offsets). */
int vb200_region_pack(const float* box_feats, const float* boxes, const float* image_wh, const int32_t* num_boxes, void* a_out,
                      float* mask_add, float* spatials_out, int32_t B, int32_t n, int32_t F, int32_t Kp, int32_t act_fp16, int32_t split16,
                      const int32_t* offs, void* cuda_stream);
/* Narrow heads: out[m, j] = x[m] . w[j] + bias[j] + add[m] for j < n_out <= 4 (bias, add optional); rows >= *m_rows skipped if given. */
int vb200_rowdot(const float* x, int64_t ld_x, const float* w, const float* bias, const float* add, float* out, int64_t ld_out,
                 int64_t M, int64_t K, int32_t n_out, const int32_t* m_rows, void* cuda_stream);
/* Row-block gather: sample b of dst = block clamp(idx[b], 0, n_src - 1) of src (fp32 [L, H], 16-bit [L, H16], mask [L]; the fp32 and
 * mask copies are skipped when NULL). */
int vb200_gather_state(const int32_t* idx, int32_t n_src, const float* src_f32, const void* src16, const float* src_mask, float* dst_f32,
                       void* dst16, float* dst_mask, int32_t B, int32_t L, int32_t H, int32_t H16, void* cuda_stream);
/* Packed row-range gather, text (t_) and image (i_) streams in one launch: pair b's rows [dst_offs[b], dst_offs[b+1]) come from rows
 * starting at src_offs[b]; n32 / n16 = 16-byte vectors per row of the fp32 / 16-bit buffers; every pointer 16-byte aligned. */
int vb200_gather_packed_state(int32_t B, const int32_t* t_dst_offs, const int32_t* t_src_offs, const float* t_src_f32, const void* t_src16,
                              float* t_dst_f32, void* t_dst16, int32_t t_n32, int32_t t_n16, const int32_t* i_dst_offs,
                              const int32_t* i_src_offs, const float* i_src_f32, const void* i_src16, float* i_dst_f32, void* i_dst16,
                              int32_t i_n32, int32_t i_n16, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* VILBERT_B200_H */
