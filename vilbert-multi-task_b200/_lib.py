"""ctypes binding of libvilbert_b200.so (the C ABI declared in include/vilbert_b200.h).

The shared library is built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile``.  There is
deliberately NO fallback: if the library is missing, or no sm_90 GPU is visible when an engine is
created, the call raises -- the reference-facing API never silently runs on CPU or through PyTorch ops.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvilbert_b200.so")

VB200_ABI_VERSION = 2
F32, F16, BF16 = 0, 1, 2

OUT_VIL_PREDICTION = 1 << 0
OUT_VIL_PREDICTION_GQA = 1 << 1
OUT_VIL_LOGIT = 1 << 2
OUT_VIL_BINARY_PREDICTION = 1 << 3
OUT_VIL_TRI_PREDICTION = 1 << 4
OUT_VISION_PREDICTION = 1 << 5
OUT_VISION_LOGIT = 1 << 6
OUT_LINGUISIC_PREDICTION = 1 << 7
OUT_LINGUISIC_LOGIT = 1 << 8
OUT_TASK_HEADS = 0x15F
OUT_ALL = 0x1FF
OUT_ATTENTION = 1 << 9
OUT_ATTENTION_PACKED = 1 << 10
OUT_LAYER_STATES = 1 << 11


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dtype", C.c_int32), ("ndim", C.c_int32),
                ("shape", C.c_int64 * 2), ("data", C.c_void_p)]


class Inputs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("n_tokens", C.c_int32), ("n_regions", C.c_int32),
                ("question", C.c_void_p), ("features", C.c_void_p), ("spatials", C.c_void_p),
                ("segment_ids", C.c_void_p), ("input_mask", C.c_void_p), ("image_mask", C.c_void_p),
                ("co_attention_mask", C.c_void_p), ("task_tokens", C.c_void_p)]


OUTPUT_FIELDS = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction",
                 "vil_tri_prediction", "vision_prediction", "vision_logit", "linguisic_prediction",
                 "linguisic_logit", "sequence_output_t", "sequence_output_v", "pooled_output", "attention_probs"]


class RegionInputs(C.Structure):
    """vb200_region_inputs: custom_prediction()'s detector output (worker.py:422-455) instead of built tensors."""
    _fields_ = [("batch", C.c_int32), ("n_tokens", C.c_int32), ("n_boxes", C.c_int32),
                ("question", C.c_void_p), ("segment_ids", C.c_void_p), ("input_mask", C.c_void_p),
                ("task_tokens", C.c_void_p), ("box_features", C.c_void_p), ("boxes", C.c_void_p),
                ("image_wh", C.c_void_p), ("num_boxes", C.c_void_p), ("spatials_out", C.c_void_p)]


class PackedInputs(C.Structure):
    """vb200_packed_inputs: a packed variable-length batch (n_tokens / n_regions are HOST int32 arrays, the rest device memory)."""
    _fields_ = [("batch", C.c_int32), ("max_tokens", C.c_int32), ("max_regions", C.c_int32),
                ("n_tokens", C.c_void_p), ("n_regions", C.c_void_p), ("question", C.c_void_p), ("segment_ids", C.c_void_p),
                ("features", C.c_void_p), ("spatials", C.c_void_p), ("task_tokens", C.c_void_p)]


class PackedRegionInputs(C.Structure):
    """vb200_packed_region_inputs: packed detector output (n_tokens / n_boxes HOST int32 arrays, the rest device memory)."""
    _fields_ = [("batch", C.c_int32), ("max_tokens", C.c_int32), ("max_boxes", C.c_int32),
                ("n_tokens", C.c_void_p), ("n_boxes", C.c_void_p), ("question", C.c_void_p), ("segment_ids", C.c_void_p),
                ("task_tokens", C.c_void_p), ("box_features", C.c_void_p), ("boxes", C.c_void_p), ("image_wh", C.c_void_p),
                ("spatials_out", C.c_void_p)]


class PackedPairs(C.Structure):
    """vb200_packed_pairs: pairs scored from packed caption / image states (index and offset arrays HOST int32, states device)."""
    _fields_ = [("batch", C.c_int32), ("max_tokens", C.c_int32), ("max_regions", C.c_int32),
                ("text_index", C.c_void_p), ("image_index", C.c_void_p),
                ("n_text", C.c_int32), ("text_offsets", C.c_void_p), ("text_f32", C.c_void_p), ("text_16", C.c_void_p),
                ("n_image", C.c_int32), ("image_offsets", C.c_void_p), ("image_f32", C.c_void_p), ("image_16", C.c_void_p)]


class Outputs(C.Structure):
    """vb200_outputs up to attention_probs: the struct of hosts built before the layer_states field, which the engine accepts for
    every call without VB200_OUT_LAYER_STATES."""
    _fields_ = [(n, C.c_void_p) for n in OUTPUT_FIELDS]


class StateOutputs(Outputs):
    """The full vb200_outputs: Outputs and the last field, layer_states (VB200_OUT_LAYER_STATES)."""
    _fields_ = [("layer_states", C.c_void_p)]


# vb200_decode_family: which output a decode message reads (include/vilbert_b200.h, vb200_decode_answers)
DECODE_VQA, DECODE_GQA, DECODE_NLVR2, DECODE_SNLI_VE, DECODE_RETRIEVAL, DECODE_GROUNDING = 1, 2, 3, 4, 5, 6
DECODE_MAX_TOP = 10
# the worker's task ids -> decode family (worker.py:295-374)
TASK_DECODE_FAMILY = {"1": DECODE_VQA, "2": DECODE_VQA, "15": DECODE_GQA, "12": DECODE_NLVR2, "13": DECODE_SNLI_VE,
                      "7": DECODE_RETRIEVAL, "4": DECODE_GROUNDING, "16": DECODE_GROUNDING, "11": DECODE_GROUNDING}


class DecodeMsg(C.Structure):
    """vb200_decode_msg: one message's segment (rows [first, first + count) of its family's source) and top_n."""
    _fields_ = [("family", C.c_int32), ("first", C.c_int32), ("count", C.c_int32), ("top_n", C.c_int32),
                ("image_w", C.c_double), ("image_h", C.c_double)]


class Answer(C.Structure):
    """vb200_answer: top_n indices (best first) and probabilities, and grounding boxes x1, y1, x2, y2 in pixels."""
    _fields_ = [("n", C.c_int32), ("index", C.c_int32 * DECODE_MAX_TOP), ("prob", C.c_float * DECODE_MAX_TOP),
                ("box", (C.c_int32 * 4) * DECODE_MAX_TOP)]


ABLATION_MAX_VARIANTS = 1024


class AblationMsg(C.Structure):
    """vb200_ablation_msg: the attributed column (-1: the unablated top-1) and the token and box ranges ablated one unit at a time."""
    _fields_ = [("answer", C.c_int32), ("token_begin", C.c_int32), ("token_end", C.c_int32), ("box_begin", C.c_int32),
                ("box_end", C.c_int32)]


class AblationScore(C.Structure):
    """vb200_ablation_score: per variant the attributed column and its probability, and the variant's own top-1 and probability."""
    _fields_ = [("answer", C.c_int32), ("prob", C.c_float), ("top1", C.c_int32), ("top1_prob", C.c_float)]


class HeadAblationMessage(C.Structure):
    """vb200_head_ablation_message: one answer of any decode family by its images, the attributed index (-1: the unablated top-1)
    and the attention entries whose heads are removed one at a time."""
    _fields_ = [("family", C.c_int32), ("image_begin", C.c_int32), ("n_images", C.c_int32), ("answer", C.c_int32),
                ("entry_begin", C.c_int32), ("entry_end", C.c_int32)]


class AblationMessage(C.Structure):
    """vb200_ablation_message: one answer of any decode family by its images, the attributed index in its segment (-1: the
    unablated top-1) and the token and box ranges ablated one unit at a time (boxes numbered across the message's images)."""
    _fields_ = [("family", C.c_int32), ("image_begin", C.c_int32), ("n_images", C.c_int32), ("answer", C.c_int32),
                ("token_begin", C.c_int32), ("token_end", C.c_int32), ("box_begin", C.c_int32), ("box_end", C.c_int32)]


class AblationVariant(C.Structure):
    """vb200_ablation_variant: one variant in the engine's order -- its message, kind (0 unablated, 1 masked position, 2 dropped
    box, 3 removed head, 4 coalition) and unit, the forward samples it runs and its segment [offset, offset + length) of variant_logits."""
    _fields_ = [("message", C.c_int32), ("kind", C.c_int32), ("unit", C.c_int32), ("samples", C.c_int32), ("offset", C.c_int64),
                ("length", C.c_int32)]


COALITION_MAX_UNITS = 1024


class CoalitionMessage(C.Structure):
    """vb200_coalition_message: one answer by its images and attributed index (-1: the full input's top-1), its units (HOST int32
    offset / item arrays of question positions and boxes) and its coalitions (HOST uint64 presence bitmaps, ceil(n_units / 64) words
    each)."""
    _fields_ = [("family", C.c_int32), ("image_begin", C.c_int32), ("n_images", C.c_int32), ("answer", C.c_int32),
                ("n_units", C.c_int32), ("position_offsets", C.c_void_p), ("positions", C.c_void_p), ("box_offsets", C.c_void_p),
                ("boxes", C.c_void_p), ("n_coalitions", C.c_int32), ("coalitions", C.c_void_p)]


class ShapleyMessage(C.Structure):
    """vb200_shapley_message: units, permutations and group size of one message, and where its permutation table, values and
    outputs start in the call's device arrays."""
    _fields_ = [("n_units", C.c_int32), ("n_perm", C.c_int32), ("group", C.c_int32), ("perm_offset", C.c_int64),
                ("value_offset", C.c_int64), ("out_offset", C.c_int64)]


INTERACTION_MAX_PAIRS = 65536


class InteractionMessage(C.Structure):
    """vb200_interaction_message: units, permutations, group size and pair count of one message, where its permutation table,
    values and outputs start in the call's device arrays, and its HOST int32 [n_pairs, 2] pairs."""
    _fields_ = [("n_units", C.c_int32), ("n_perm", C.c_int32), ("group", C.c_int32), ("n_pairs", C.c_int32),
                ("perm_offset", C.c_int64), ("value_offset", C.c_int64), ("out_offset", C.c_int64), ("pairs", C.c_void_p)]


class Detections(C.Structure):
    """vb200_detections: one image's raw detector heads (device pointers) and its first output row."""
    _fields_ = [("n_proposals", C.c_int32), ("dst_row", C.c_int32), ("im_scale", C.c_double), ("proposals", C.c_void_p),
                ("scores", C.c_void_p), ("features", C.c_void_p)]


class SelectParams(C.Structure):
    """vb200_select_params: what vb200_select_regions selects, and the rows of its per-row outputs."""
    _fields_ = [("n_classes", C.c_int32), ("feature_size", C.c_int32), ("max_boxes", C.c_int32), ("conf_thresh", C.c_float),
                ("nms_iou", C.c_float), ("background", C.c_int32), ("out_rows", C.c_int32)]


class Selected(C.Structure):
    """vb200_selected: device outputs of vb200_select_regions (the last four may be NULL)."""
    _fields_ = [(n, C.c_void_p) for n in ("box_features", "boxes", "num_boxes", "keep_index", "max_conf", "cls_prob", "objects")]


class PretrainRows(C.Structure):
    """vb200_pretrain_rows: fp32 final states (device) and the HOST int32 row lists of vb200_pretraining_heads."""
    _fields_ = [("text_state", C.c_void_p), ("image_state", C.c_void_p), ("pooled_state", C.c_void_p),
                ("t_rows", C.c_int32), ("v_rows", C.c_int32), ("p_rows", C.c_int32),
                ("n_t", C.c_int32), ("n_v", C.c_int32), ("n_p", C.c_int32),
                ("text_rows", C.c_void_p), ("image_rows", C.c_void_p), ("pair_rows", C.c_void_p), ("top_k", C.c_int32)]


class PretrainOut(C.Structure):
    """vb200_pretrain_out: optional device outputs of vb200_pretraining_heads (logits fp32, top-k as vb200_answer)."""
    _fields_ = [(n, C.c_void_p) for n in ("token_logits", "region_logits", "alignment", "token_top", "region_top")]


class PretrainTargets(C.Structure):
    """vb200_pretrain_targets: HOST int32 token / pair labels, DEVICE fp32 image target rows of vb200_pretraining_objectives."""
    _fields_ = [(n, C.c_void_p) for n in ("token_labels", "image_targets", "pair_labels")]


class PretrainLosses(C.Structure):
    """vb200_pretrain_losses: optional device fp32 outputs of vb200_pretraining_objectives."""
    _fields_ = [(n, C.c_void_p) for n in ("token_loss", "region_loss", "pair_loss", "reduced")]


class Options(C.Structure):
    _fields_ = [("device", C.c_int32), ("num_labels", C.c_int32), ("use_cuda_graph", C.c_int32),
                ("use_pdl", C.c_int32), ("strict", C.c_int32), ("act_fp16", C.c_int32),
                ("fused_layernorm", C.c_int32), ("split_fp32", C.c_int32), ("ln_fold", C.c_int32), ("max_plans", C.c_int32)]


# every symbol include/vilbert_b200.h declares (tests/test_cabi.py checks the list against the header)
EXPORTS = ["vb200_abi_version", "vb200_create", "vb200_destroy", "vb200_last_error", "vb200_forward", "vb200_forward_slot",
           "vb200_forward_host", "vb200_forward_host_slot", "vb200_plan_info", "vb200_model_dim", "vb200_set_option", "vb200_timeline", "vb200_profile_ops",
           "vb200_attention_layout", "vb200_attention_layout_packed", "vb200_attention_selection", "vb200_attention_relevance", "vb200_state_layout", "vb200_state_layout_packed", "vb200_state_selection",
           "vb200_forward_regions", "vb200_forward_packed", "vb200_forward_regions_packed", "vb200_encode_text", "vb200_encode_image", "vb200_forward_cached",
           "vb200_encode_text_packed", "vb200_encode_image_packed", "vb200_encode_regions_packed", "vb200_forward_cached_packed", "vb200_linear", "vb200_linear_rows", "vb200_linear_split", "vb200_layernorm", "vb200_layernorm_split", "vb200_attention_f32",
           "vb200_self_attention", "vb200_co_attention", "vb200_self_attention_packed", "vb200_co_attention_packed",
           "vb200_self_attention_stream", "vb200_co_attention_stream",
           "vb200_linear_product", "vb200_text_embed", "vb200_image_pack", "vb200_region_pack", "vb200_rowdot", "vb200_gather_state",
           "vb200_gather_packed_state", "vb200_decode_answers", "vb200_decode_answers_host", "vb200_select_regions",
           "vb200_pretraining_heads", "vb200_create_pretraining", "vb200_pretraining_objectives", "vb200_answer_ablation",
           "vb200_message_ablation_layout", "vb200_message_ablation", "vb200_forward_packed_gated", "vb200_forward_regions_packed_gated",
           "vb200_head_ablation_layout", "vb200_head_ablation", "vb200_coalition_ablation_layout", "vb200_coalition_ablation",
           "vb200_shapley_values", "vb200_interaction_values"]

_lib = None


class VilbertB200Error(RuntimeError):
    pass


def load():
    """Load the shared library once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VilbertB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C vilbert-multi-task_b200/csrc`).  There is no CPU/PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise VilbertB200Error(f"{LIB_PATH} does not export {name}")
    vp, i32, i64, u32, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_float
    lib.vb200_abi_version.restype = C.c_int
    lib.vb200_create.argtypes = [C.c_char_p, i64, C.POINTER(Tensor), C.POINTER(Options), C.POINTER(vp)]
    lib.vb200_destroy.argtypes = [vp]
    lib.vb200_last_error.argtypes = [vp]
    lib.vb200_last_error.restype = C.c_char_p
    lib.vb200_forward.argtypes = [vp, C.POINTER(Inputs), C.POINTER(Outputs), u32, vp]
    lib.vb200_forward_slot.argtypes = [vp, C.POINTER(Inputs), C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_forward_host.argtypes = [vp, C.POINTER(Inputs), C.POINTER(Outputs), u32, vp]
    lib.vb200_forward_host_slot.argtypes = [vp, C.POINTER(Inputs), C.POINTER(Outputs), u32, i32, i32, vp]
    lib.vb200_plan_info.argtypes = [vp, i32, i32, i32, u32, C.POINTER(i64), C.POINTER(C.c_double)]
    lib.vb200_model_dim.argtypes = [vp, C.c_char_p, C.POINTER(i64)]
    lib.vb200_set_option.argtypes = [vp, C.c_char_p, i64]
    lib.vb200_timeline.argtypes = [vp, i32, i32, i32, u32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
    lib.vb200_profile_ops.argtypes = [vp, i32, i32, i32, u32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(C.c_double),
                                      C.POINTER(C.c_double), C.POINTER(i32)]
    lib.vb200_attention_layout.argtypes = [vp, i32, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    lib.vb200_attention_layout_packed.argtypes = [vp, i32, vp, vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    lib.vb200_attention_selection.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    lib.vb200_attention_relevance.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp]
    lib.vb200_state_layout.argtypes = [vp, i32, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i64),
                                       C.POINTER(i64)]
    lib.vb200_state_layout_packed.argtypes = [vp, i32, vp, vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i64),
                                              C.POINTER(i64)]
    lib.vb200_state_selection.argtypes = lib.vb200_attention_selection.argtypes
    lib.vb200_forward_regions.argtypes = [vp, C.POINTER(RegionInputs), C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_forward_packed.argtypes = [vp, C.POINTER(PackedInputs), C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_forward_regions_packed.argtypes = [vp, C.POINTER(PackedRegionInputs), C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_forward_packed_gated.argtypes = [vp, C.POINTER(PackedInputs), vp, C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_forward_regions_packed_gated.argtypes = [vp, C.POINTER(PackedRegionInputs), vp, C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_linear_rows.argtypes = [vp, i64, vp, i64, vp, i32, vp, i64, vp, i64, i64, i64, i64, i32, i32, vp, vp]
    lib.vb200_encode_text.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vb200_encode_image.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.vb200_forward_cached.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, vp, vp, i32, vp, vp, vp, C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_encode_text_packed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.vb200_encode_image_packed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.vb200_encode_regions_packed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.vb200_forward_cached_packed.argtypes = [vp, C.POINTER(PackedPairs), C.POINTER(Outputs), u32, i32, vp]
    lib.vb200_linear_split.argtypes = [vp, i64, vp, i64, vp, i32, vp, i64, vp, i64, i64, i64, i64, vp]
    lib.vb200_layernorm_split.argtypes = [vp, i64, vp, i64, vp, vp, f32, vp, i64, vp, i64, i64, i64, vp]
    lib.vb200_attention_f32.argtypes = [vp, i64, vp, vp, i64, i32, vp, i32, i32, i32, i32, i32, vp, i64, i32, vp, vp]
    lib.vb200_linear.argtypes = [vp, i64, vp, i64, vp, vp, i64, vp, vp, f32, i32, vp, i64, vp, i64,
                                 i64, i64, i64, i32, i32, i32, i32, vp, vp]
    lib.vb200_layernorm.argtypes = [vp, i64, vp, i64, vp, vp, f32, vp, i64, vp, i64, i64, i64, i32, vp]
    lib.vb200_self_attention.argtypes = [vp, i64, i32, vp, vp, i64, i32, i32, i32, i32, i32, vp]
    lib.vb200_co_attention.argtypes = [vp, i64, vp, i64, i32, vp, vp, vp, i64, vp, i64, i32, i32, i32, i32, i32, i32, vp]
    lib.vb200_self_attention_packed.argtypes = [vp, i64, i32, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp]
    lib.vb200_co_attention_packed.argtypes = [vp, i64, vp, i64, i32, vp, vp, vp, i64, vp, i64, i32, i32, i32, i32, i32, i32, vp, vp, vp]
    lib.vb200_self_attention_stream.argtypes = lib.vb200_self_attention_packed.argtypes
    lib.vb200_co_attention_stream.argtypes = lib.vb200_co_attention_packed.argtypes
    lib.vb200_linear_product.argtypes = [vp, i64, vp, i64, vp, i32, vp, i64, vp, i64, vp, i64, i64, i64, i64, i32, i32, vp]
    lib.vb200_text_embed.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32,
                                     i32, i32, vp, i32, vp]
    lib.vb200_image_pack.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.vb200_region_pack.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp]
    lib.vb200_rowdot.argtypes = [vp, i64, vp, vp, vp, vp, i64, i64, i64, i32, vp, vp]
    lib.vb200_gather_state.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.vb200_gather_packed_state.argtypes = [i32, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp]
    lib.vb200_decode_answers.argtypes = [vp, C.POINTER(DecodeMsg), i32, C.POINTER(Outputs), i32, i32, vp, vp, vp]
    lib.vb200_decode_answers_host.argtypes = [vp, C.POINTER(DecodeMsg), i32, C.POINTER(Outputs), i32, i32, vp, C.POINTER(Answer), vp]
    lib.vb200_select_regions.argtypes = [vp, C.POINTER(Detections), i32, C.POINTER(SelectParams), C.POINTER(Selected), vp]
    lib.vb200_pretraining_heads.argtypes = [vp, C.POINTER(PretrainRows), C.POINTER(PretrainOut), vp]
    lib.vb200_create_pretraining.argtypes = lib.vb200_create.argtypes
    lib.vb200_pretraining_objectives.argtypes = [vp, C.POINTER(PretrainRows), C.POINTER(PretrainTargets), C.POINTER(PretrainLosses), vp]
    lib.vb200_answer_ablation.argtypes = [vp, C.POINTER(PackedRegionInputs), C.POINTER(AblationMsg), i32, i64, vp, vp, i32, vp]
    lib.vb200_message_ablation_layout.argtypes = [vp, i32, vp, vp, C.POINTER(AblationMessage), i32, vp, C.POINTER(C.c_int64),
                                                  C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.vb200_message_ablation.argtypes = [vp, C.POINTER(PackedRegionInputs), C.POINTER(AblationMessage), i32, i64, vp, vp, i32, vp]
    lib.vb200_head_ablation_layout.argtypes = [vp, i32, vp, vp, C.POINTER(HeadAblationMessage), i32, vp, C.POINTER(C.c_int64),
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.vb200_head_ablation.argtypes = [vp, C.POINTER(PackedRegionInputs), C.POINTER(HeadAblationMessage), i32, vp, vp, i32, vp]
    lib.vb200_coalition_ablation_layout.argtypes = [vp, i32, vp, vp, C.POINTER(CoalitionMessage), i32, vp, C.POINTER(C.c_int64),
                                                    C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.vb200_coalition_ablation.argtypes = [vp, C.POINTER(PackedRegionInputs), C.POINTER(CoalitionMessage), i32, i64, vp, vp, i32, vp]
    lib.vb200_shapley_values.argtypes = [vp, C.POINTER(ShapleyMessage), i32, vp, vp, vp, vp, vp]
    lib.vb200_interaction_values.argtypes = [vp, C.POINTER(InteractionMessage), i32, vp, vp, vp, vp, vp]
    for name in EXPORTS:
        if name not in ("vb200_last_error",):
            getattr(lib, name).restype = C.c_int
    if lib.vb200_abi_version() != VB200_ABI_VERSION:
        raise VilbertB200Error("libvilbert_b200.so ABI version mismatch: rebuild the extension")
    _lib = lib
    return lib


def check(rc: int, handle=None):
    if rc != 0:
        msg = load().vb200_last_error(handle)
        raise VilbertB200Error(f"vilbert_b200 error {rc}: {msg.decode() if msg else '?'}")
