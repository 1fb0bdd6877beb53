"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  One schedule step of the 16-bit engine (compute_dtype "fp16" / "bf16") in fp64, rounded
where the engine rounds, to be fed the engine's own input state (teacher forcing).

End to end, a 16-bit forward can only be held to the format floor against the fp32 oracle (tests/test_gpu_model.py): two runs that
round at the same places decorrelate after a few layers.  The layer states (``output_layer_states``) are the fp32 residual stream
after every step, and the 16-bit operand the next step reads is ``sat_rn`` of that state bit for bit.  So ``StepRef`` restarts every
step from exactly the engine's input, and engine and reference then differ by one step's worth of last-bit disagreements only
(tests/test_gpu_step_parity.py).  The arithmetic is fp64, except inside the attention, where the kernel's fp32 registers (scores,
running max, p, the running sum and the context accumulator) are kept fp32 so that P is rounded from the value the kernel rounds.

Rounding points, r = kernel_refs.sat_rn to the mode's format, each where engine.cu writes a 16-bit buffer:

  load_linear               every tensor-core weight r(W); biases, LayerNorm, embedding tables and the rowdot heads stay fp32
  (LayerNorm row kernel)    a state is written fp32 and as its 16-bit copy: the next GEMM reads x16 = r(state)
  PlanBuilder::qkv          qkv = r(x16 W^T + b), Q | K | V for the tensor-core attention
  attention.cu attend_tile  per 64-key block over pad16(L) keys (keys at or past L at -inf): s = fma(q.k, log2e/sqrt(d), mask log2e),
                            running max m, c = exp2(m_old - m_new), p = exp2(s - m), l = l c + sum p, o = o c + r(p) V;
                            ctx = r(o (1 / l))  (attend_tile_short is the one-block case, same order per element)
  PlanBuilder::row_local    a = LN(ctx Wo^T + b + state_in) (fp32 GEMM output into the LayerNorm kernel);
                            inter = r(gelu_poly(r(a) Wi^T + b)) (act kActGelu: the epilogue polynomial kernel_refs.GELU_Q);
                            state_out = LN(inter Wf^T + b + a)
  PlanBuilder::connection   both streams' QKV, text queries over image keys with the image key mask and image queries over
                            text keys with the text key mask, then row_local per stream (dense1 / dense2 + LayerNorm, the FFNs)
  get_plan (embeddings)     text: fp32 gather + LayerNorm, no 16-bit rounding before the state (launch_text_embed); image:
                            LN(r([feat | loc | 0]) [r(W_img) | r(W_loc)]^T + (b_img + b_loc)), the bias sum in fp32
  PlanBuilder::heads        poolers: relu(r(first row) Wp^T + b) fp32, the image pooler's epilogue multiplies by the text one;
                            r(pooled) feeds the classifiers
  PlanBuilder::predict      SimpleClassifier and the pre-training heads: r(LN(gelu_poly(x16 W0^T + b0))) W3^T + b3, fp32 out;
                            the LM decoder is the rounded word table
  binary head (even B)      LN(gelu_poly(r(pooled pairs) W0^T + b0)) stays fp32 and meets the fp32 rowdot weights
  rowdot                    vil_logit, vil_tri_prediction, bi_seq_relationship on the fp32 pooled product; vision_logit (+ key
                            mask) and linguisic_logit on the fp32 final states; fp32 weights

With ``mode=None`` every r() is the identity, the GELU is erf and the attention runs in fp64: ``StepRef`` is then a restatement of
the fp64 oracle's own modules (tests/test_step_ref.py holds it there to 1e-12).  ``defects`` switches on one-line mistakes of the
engine (``DEFECTS``), the catalog tests/test_step_ref.py checks the bounds against.
"""
from __future__ import annotations

import copy
import math

import torch

from oracle import kernel_refs as K

LOG2E = 1.4426950408889634
KEY_BLOCK = 64                  # attention.cu kKeyBlock: keys per online-softmax block

# Engine step vs StepRef fed the engine's previous entries.  states / pooled / logits: oracle.fp64.rel_err, max |o - r| / max(1, |r|);
# maps: max |o - r|.  Each bound is ~4x the worst value of scripts/step_parity_sweep.py (20 seeds of every reduced-width case, 3 of
# the long-sequence and 268 M model cases) on an H100 80GB HBM3 at a 700 W power limit, 1980 MHz maximum SM clock (worst value in
# brackets; every one of them on the 268 M model), and under half the smallest movement of its family in the defect catalog
# (tests/test_step_ref.py enforces the latter).  bf16 states: 3.2x, since 4x would pass scale_without_log2e (2.3e-2).
STEP_BOUNDS = {
    "fp16": {"states": 2e-3,      # [5.0e-4]
             "maps": 1.2e-4,      # [3.0e-5]
             "pooled": 1.4e-5,    # [3.5e-6]
             "logits": 1.4e-3},   # [3.6e-4] linguisic_prediction
    "bf16": {"states": 1.1e-2,    # [3.5e-3]
             "maps": 6.5e-4,      # [1.6e-4]
             "pooled": 1.2e-5,    # [3.0e-6]
             "logits": 6e-3},     # [1.5e-3] linguisic_prediction
}
# The same checks at checkpoint-like weights (oracle/trained_like.py, seed trained_like.SEED; tests/test_gpu_trained_like.py): ~4x the
# worst value of scripts/step_parity_sweep.py --weights trained (20 seeds of every reduced-width case, 3 of the long-sequence and
# 268 M model cases) on an H100 80GB HBM3 at a 700 W power limit, 1980 MHz maximum SM clock.  In brackets: the worst value, its case
# and its step.
STEP_BOUNDS_TRAINED = {
    "fp16": {"states": 4.8e-3,    # [1.20e-3 full_B64, C2 image]
             "maps": 1.6e-2,      # [3.89e-3 full_B64, T10]
             "pooled": 2e-5,      # [4.90e-6 full_B64]
             "logits": 1.3e-3},   # [3.13e-4 full_B64, vision_prediction]
    "bf16": {"states": 3.5e-2,    # [8.68e-3 full_B64, V4 image]
             "maps": 7.2e-2,      # [1.81e-2 tiny_B2_T30_V36_pad0, C2 text->image]
             "pooled": 1.7e-5,    # [4.22e-6 full_B64]
             "logits": 1e-2},     # [2.44e-3 full_B64, linguisic_prediction]
}
FAMILIES = ("states", "maps", "pooled", "logits")

# One-line mistakes of the 16-bit engine, restated on StepRef (switched on by name), and which check family must see each:
# name -> (what the engine would do, the families, the modes whose bounds it clears twice).  tests/test_step_ref.py runs them on
# the 268 M model's steps fed the fp64 oracle's own states.
DEFECTS = {
    "sum_not_rescaled": ("the online-softmax sum not rescaled: l += sum p without * c", ("states",), ("fp16", "bf16")),
    "pad_keys_unmasked": ("keys between L and pad16(L) left unmasked (zero keys at mask 0)", ("states",), ("fp16", "bf16")),
    "ln2_residual_layer_input": ("the second LayerNorm taking the layer input as residual instead of a", ("states",), ("fp16", "bf16")),
    "coattention_masks_swapped": ("the co-attention directions given each other's key masks", ("states",), ("fp16", "bf16")),
    "scale_without_log2e": ("scores scaled by 1/sqrt(d) without log2e while the softmax uses exp2", ("states",), ("fp16", "bf16")),
    "pooled_t_rounded": ("the pooled product taken from the 16-bit text pooler output", ("pooled",), ("fp16", "bf16")),
    # the two online-softmax rescales past one key block; even at near-uniform attention the running max moves enough between
    # blocks (fp16 / bf16 states at these weights: 2.5e-1 / 2.5e-1 and 3.1e-2 / 3.3e-2)
    "ctx_not_rescaled": ("the online-softmax context not rescaled: o += r(p) V without * c (the sum rescaled)", ("states",),
                         ("fp16", "bf16")),
    "block_max_only": ("each key block's own max, no running max carried across blocks (nothing rescaled)", ("states",),
                       ("fp16", "bf16")),
}
# Restated too, but not separable from the step bounds: each is one extra or different 16-bit rounding, and moves a step's state
# by about what one rounding point moves it (on the 268 M model every rounding point alone moves T0's worst element by 4e-4 in
# fp16), which is also the size of the engine's own last-bit disagreements, the measured worst values behind STEP_BOUNDS.
NOT_SEPARABLE = {
    "p_normalised_before_rounding": "P normalised before its 16-bit rounding: r(p / l) V instead of r(p) V / l",
    "tanh_gelu": "tanh GELU in the GEMM GELU epilogue (FFNs and heads)",
    "p_other_format": "P stored in the other 16-bit format",
    "ctx_other_format": "the attention context stored in the other 16-bit format",
    "attn_out_rounded": "the attention-output GEMM's fp32 output rounded to 16 bits before its LayerNorm",
    "qkv_bias_after_rounding": "the QKV bias added after the 16-bit rounding: r(r(x16 W^T) + b)",
}

# The catalog at checkpoint-like weights, held to STEP_BOUNDS_TRAINED by tests/test_trained_like.py: every defect above, and the QKV
# bias added after rounding, which sharp heads turn from one more rounding into a move of the states (2.4x / 2.6x the bound).  Unmasked pad keys
# clear the bf16 states bound 0.9x only (3.2e-2 against 3.5e-2; fp16 6.8x): at these weights the pad keys' zero scores fall among
# the centred real scores and take a few percent of a mild head's mass, which bf16's own step noise (8.7e-3) comes within 4x of.
DEFECTS_TRAINED = dict(DEFECTS, **{
    "pad_keys_unmasked": DEFECTS["pad_keys_unmasked"][:2] + (("fp16",),),
    "qkv_bias_after_rounding": (NOT_SEPARABLE["qkv_bias_after_rounding"], ("states",), ("fp16", "bf16")),
})


def pad16(n: int) -> int:
    return (n + 15) // 16 * 16


def _split(x, heads):
    B, L, H = x.shape
    return x.double().reshape(B, L, heads, H // heads).transpose(1, 2)


def _merge(x):
    B, h, L, d = x.shape
    return x.transpose(1, 2).reshape(B, L, h * d)


def attention_blockwise(q, k, v, mask_add, heads, f16=None, defects=frozenset()):
    """The tensor-core attention (attend_tile) restated block by block: q [B, Lq, H], k / v [B, Lk, H] (16-bit values), mask_add
    [B, Lk] (0 / -10000) -> the context [B, Lq, H] fp64.  ``f16`` True / False: the kernel's rounding points in fp16 / bf16, fp32
    registers where the kernel keeps fp32; None: every step in fp64 with no rounding (softmax(q k^T / sqrt(d) + mask) v).  Keys past
    Lk contribute exactly 0 (their scores are -inf), so the blocks run over the Lk real keys at the kernel's block boundaries."""
    emu = f16 is not None
    acc = torch.float32 if emu else torch.float64
    dev = q.device
    d = q.shape[-1] // heads

    def r(x, other=False):
        return K.sat_rn(x, f16 != other).double() if emu else x

    qh, kh, vh = _split(q, heads), _split(k, heads), _split(v, heads)
    if emu:
        l2e = torch.tensor(LOG2E, dtype=torch.float32, device=dev)
        scale = l2e / torch.sqrt(torch.tensor(float(d), dtype=torch.float32, device=dev))          # kLog2e / sqrtf(D)
        if "scale_without_log2e" in defects:
            scale = 1.0 / torch.sqrt(torch.tensor(float(d), dtype=torch.float32, device=dev))
        ml2 = mask_add.float() * l2e                                                                  # mask_s[j] = mask * kLog2e
    else:
        scale = torch.tensor(LOG2E / math.sqrt(d), dtype=torch.float64, device=dev)
        ml2 = mask_add.double() * LOG2E
    if "pad_keys_unmasked" in defects:
        B, h, Lk, _ = kh.shape
        n = pad16(Lk) - Lk
        kh = torch.cat([kh, kh.new_zeros(B, h, n, d)], 2)
        vh = torch.cat([vh, vh.new_zeros(B, h, n, d)], 2)
        ml2 = torch.cat([ml2, ml2.new_zeros(B, n)], 1)
    n_keys = kh.shape[2]
    raw = (qh @ kh.transpose(-1, -2)).to(acc)                                  # fp32-accumulated Q K^T
    s = (raw.double() * scale.double() + ml2.double()[:, None, None, :]).to(acc)   # fmaf: one rounding
    m = torch.full(s.shape[:-1] + (1,), float("-inf"), dtype=acc, device=dev)
    l = torch.zeros_like(m)
    o = torch.zeros(s.shape[:-1] + (d,), dtype=acc, device=dev)
    for kb in range(0, n_keys, KEY_BLOCK):
        sb = s[..., kb:kb + KEY_BLOCK]
        nm = torch.maximum(m, sb.amax(-1, keepdim=True))
        c = torch.exp2(m - nm)                                                 # 0 on the first block
        if "block_max_only" in defects:                                        # no running max: each block against its own
            nm, c = sb.amax(-1, keepdim=True), torch.ones_like(c)
        p = torch.exp2(sb - nm)
        l = (l if "sum_not_rescaled" in defects else l * c) + p.sum(-1, keepdim=True)
        o = (o if "ctx_not_rescaled" in defects else o * c) + (r(p, "p_other_format" in defects) @ vh[..., kb:kb + KEY_BLOCK, :]).to(acc)
        m = nm
    if "p_normalised_before_rounding" in defects:
        o, l = (r(torch.exp2(s - m) * (1.0 / l)) @ vh).to(acc), torch.ones_like(l)
    return _merge(r(o * (1.0 / l), "ctx_other_format" in defects))


def softmax_probs(q, k, mask_add, heads):
    """softmax(q k^T / sqrt(d) + mask) in fp64, [B, heads, Lq, Lk]: the attention maps of the 16-bit Q and K."""
    qh, kh = _split(q, heads), _split(k, heads)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(qh.shape[-1]) + mask_add.double()[:, None, None, :]
    return torch.softmax(s, dim=-1)


def gelu_poly(x):
    """The GEMM epilogue's GELU (common.cuh gelu_erf) in fp64: x * sat(0.5 + x Q(x^2)), Q of kernel_refs.GELU_Q in Horner order."""
    u = x * x
    q = torch.full_like(x, K.GELU_Q[0])
    for c in K.GELU_Q[1:]:
        q = q * u + c
    return x * (0.5 + x * q).clamp(0.0, 1.0)


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def _layernorm(x, g, b, eps=1e-12):
    u = x.mean(-1, keepdim=True)
    s = (x - u).pow(2).mean(-1, keepdim=True)
    return g * ((x - u) / torch.sqrt(s + eps)) + b


class StepRef:
    """One step of the 16-bit engine's forward on ``oracle``'s weights (an fp32 oracle of oracle/vilbert_ref.py), in fp64 on
    ``device``.  ``mode``: "fp16", "bf16" or None (no rounding, erf GELU: the fp64 oracle).  Inputs are the engine's fp32 states."""

    def __init__(self, oracle, mode=None, defects=(), device="cpu"):
        assert mode in (None, "fp16", "bf16"), mode
        unknown = set(defects) - set(DEFECTS_TRAINED) - set(NOT_SEPARABLE)
        assert not unknown, unknown
        self.oracle, self.mode, self.defects = oracle, mode, frozenset(defects)
        self.f16 = mode == "fp16"
        self.dev = torch.device(device)
        self.cfg = oracle.config
        self.schedule = oracle.bert.encoder.schedule()
        self._p = dict(oracle.named_parameters(remove_duplicate=False))
        self._cache = {}
        self._emb = copy.deepcopy(oracle.bert.embeddings).double().to(self.dev).eval()

    # ---------------------------------------------------------------------------------------------------------- primitives
    def r(self, x, other=False):
        """The mode's 16-bit store of x (as fp64); the identity without a mode."""
        return x.double() if self.mode is None else K.sat_rn(x, self.f16 != other).double()

    def _param(self, name, rounded):
        key = (name, rounded)
        if key not in self._cache:
            p = self._p[name].detach().float().to(self.dev)
            self._cache[key] = self.r(p) if rounded else p.double()
        return self._cache[key]

    def w(self, prefix, rounded=True):
        """(weight, bias) of the nn.Linear ``prefix``: the weight as the engine stores it (16-bit for the tensor cores, fp32 for a
        rowdot head with ``rounded=False``), the bias fp32, both as fp64."""
        return self._param(prefix + ".weight", rounded), self._param(prefix + ".bias", False)

    def linear(self, x, prefix, rounded=True):
        W, b = self.w(prefix, rounded)
        return x @ W.t() + b

    def ln(self, x, prefix):
        return _layernorm(x, self._param(prefix + ".weight", False), self._param(prefix + ".bias", False))

    def gelu(self, x):
        if "tanh_gelu" in self.defects:
            return gelu_tanh(x)
        return gelu_poly(x) if self.mode is not None else K.gelu_fp64(x)

    def proj(self, x16, prefix):
        """Q, K or V: r(x16 W^T + b)."""
        W, b = self.w(prefix)
        if "qkv_bias_after_rounding" in self.defects:
            return self.r(self.r(x16 @ W.t()) + b)
        return self.r(x16 @ W.t() + b)

    def attention(self, q, k, v, mask, heads):
        return attention_blockwise(q, k, v, mask, heads, None if self.mode is None else self.f16, self.defects)

    def attn_out(self, ctx, x, dense, ln):
        y = self.linear(ctx, dense)
        if "attn_out_rounded" in self.defects:
            y = self.r(y)
        return self.ln(y + x, ln)

    def ffn(self, a, inter, out, ln, layer_in):
        h = self.r(self.gelu(self.linear(self.r(a), inter)))
        return self.ln(self.linear(h, out) + (layer_in if "ln2_residual_layer_input" in self.defects else a), ln)

    # ---------------------------------------------------------------------------------------------------------- steps
    def text_embed(self, input_ids, token_type_ids, task_ids):
        """Entry 0: the fp32 gather + LayerNorm (no 16-bit rounding), [B, Tin + 1, H]."""
        dv = self.dev
        with torch.no_grad():
            return self._emb(input_ids.to(dv), token_type_ids.to(dv), task_ids.to(dv))

    def image_embed(self, feat, loc):
        """Entry 1 from the fp32 operand rows: LN(r([feat | loc]) [r(W_img) | r(W_loc)]^T + (b_img + b_loc))."""
        p = "bert.v_embeddings."
        x = torch.cat([feat.float(), loc.float()], -1).to(self.dev)
        W = torch.cat([self.w(p + "image_embeddings")[0], self.w(p + "image_location_embeddings")[0]], 1)
        b1, b2 = self._p[p + "image_embeddings.bias"], self._p[p + "image_location_embeddings.bias"]
        b = (b1.detach().float() + b2.detach().float()) if self.mode is not None else b1.detach().double() + b2.detach().double()
        return self.ln(self.r(x) @ W.t() + b.double().to(self.dev), p + "LayerNorm")

    def layer(self, step, x, mask):
        """A text ("T3") or image ("V0") layer on its input state x [B, L, H] with the additive key mask [B, L]: (state, maps of the
        16-bit Q and K)."""
        text = step[0] == "T"
        pre = f"bert.encoder.{'layer' if text else 'v_layer'}.{int(step[1:])}."
        heads = self.cfg.num_attention_heads if text else self.cfg.v_num_attention_heads
        x = x.double().to(self.dev)
        mask = mask.to(self.dev)
        x16 = self.r(x)
        q, k, v = (self.proj(x16, pre + "attention.self." + n) for n in ("query", "key", "value"))
        ctx = self.attention(q, k, v, mask, heads)
        a = self.attn_out(ctx, x, pre + "attention.output.dense", pre + "attention.output.LayerNorm")
        out = self.ffn(a, pre + "intermediate.dense", pre + "output.dense", pre + "output.LayerNorm", x)
        return out, softmax_probs(q, k, mask, heads)

    def connection(self, idx, t, v, t_mask, v_mask):
        """Connection layer ``idx`` on the text and image states: (text state, image state, (text->image maps, image->text maps))."""
        pre = f"bert.encoder.c_layer.{idx}."
        ba = pre + "biattention."
        heads = self.cfg.bi_num_attention_heads
        t, v = t.double().to(self.dev), v.double().to(self.dev)
        t_mask, v_mask = t_mask.to(self.dev), v_mask.to(self.dev)
        t16, v16 = self.r(t), self.r(v)
        q1, k1, v1 = (self.proj(v16, ba + n) for n in ("query1", "key1", "value1"))
        q2, k2, v2 = (self.proj(t16, ba + n) for n in ("query2", "key2", "value2"))
        img_keys, txt_keys = v_mask, t_mask
        if "coattention_masks_swapped" in self.defects:
            img_keys, txt_keys = _read_as(t_mask, v_mask.shape), _read_as(v_mask, t_mask.shape)
        ctx_t = self.attention(q2, k1, v1, img_keys, heads)        # text queries over image keys -> the text stream's context
        ctx_v = self.attention(q1, k2, v2, txt_keys, heads)
        v_att = self.attn_out(ctx_v, v, pre + "biOutput.dense1", pre + "biOutput.LayerNorm1")
        t_att = self.attn_out(ctx_t, t, pre + "biOutput.dense2", pre + "biOutput.LayerNorm2")
        v_out = self.ffn(v_att, pre + "v_intermediate.dense", pre + "v_output.dense", pre + "v_output.LayerNorm", v)
        t_out = self.ffn(t_att, pre + "t_intermediate.dense", pre + "t_output.dense", pre + "t_output.LayerNorm", t)
        return t_out, v_out, (softmax_probs(q2, k1, v_mask, heads), softmax_probs(q1, k2, t_mask, heads))

    # ---------------------------------------------------------------------------------------------------------- heads
    def pooled(self, t_first, v_first):
        """The pooled product from each sample's first row of the final fp32 states [B, H] / [B, Hv] -> [B, Hb]."""
        pt = torch.relu(self.linear(self.r(t_first.double().to(self.dev)), "bert.t_pooler.dense"))
        pv = torch.relu(self.linear(self.r(v_first.double().to(self.dev)), "bert.v_pooler.dense"))
        if "pooled_t_rounded" in self.defects:
            pt = self.r(pt)
        return pt * pv

    def _predict(self, x16, transform, ln, decoder_w, decoder_b):
        h = self.r(self.ln(self.gelu(self.linear(x16, transform)), ln))
        return h @ decoder_w.t() + decoder_b

    def _cls(self, x16, name):
        W, b = self.w(name + ".logit_fc.3")
        return self._predict(x16, name + ".logit_fc.0", name + ".logit_fc.2", W, b)

    def outputs(self, pooled, t_rows, v_rows, v_mask_rows):
        """The nine outputs from the pooled product [B, Hb] and the final fp32 states (any leading shape; ``v_mask_rows`` the additive
        image mask of the same leading shape): a tuple in the order of oracle.fp64.OUTPUT_NAMES, each fp64 with the oracle's shape
        for those leading dimensions."""
        pooled = pooled.double().to(self.dev)
        t_rows, v_rows = t_rows.double().to(self.dev), v_rows.double().to(self.dev)
        B = pooled.shape[0]
        p16 = self.r(pooled)
        vqa, gqa = self._cls(p16, "vil_prediction"), self._cls(p16, "vil_prediction_gqa")
        if B % 2 == 0:
            h = self.ln(self.gelu(self.linear(p16.reshape(B // 2, -1), "vil_binary_prediction.logit_fc.0")),
                        "vil_binary_prediction.logit_fc.2")
            binary = self.linear(h, "vil_binary_prediction.logit_fc.3", rounded=False)
        else:
            binary = self.linear(pooled, "cls.bi_seq_relationship", rounded=False)
        vil_logit = self.linear(pooled, "vil_logit", rounded=False)
        tri = self.linear(pooled, "vil_tri_prediction", rounded=False)
        ip = "cls.imagePredictions."
        W, b = self.w(ip + "decoder")
        vision_pred = self._predict(self.r(v_rows), ip + "transform.dense", ip + "transform.LayerNorm", W, b)
        vision_logit = self.linear(v_rows, "vision_logit", rounded=False) + v_mask_rows.double().to(self.dev)[..., None]
        lp = "cls.predictions."
        word = self._param("bert.embeddings.word_embeddings.weight", True)
        ling_pred = self._predict(self.r(t_rows), lp + "transform.dense", lp + "transform.LayerNorm", word,
                                  self._param(lp + "bias", False))
        ling_logit = self.linear(t_rows, "linguisic_logit", rounded=False)
        return vqa, gqa, vil_logit, binary, tri, vision_pred, vision_logit, ling_pred, ling_logit


def _read_as(mask, shape):
    """The co-attention kernel handed the other stream's mask reads it at its own stream's row offsets: sample b's key j reads the
    flat mask at b * L_own + j (zero past its end)."""
    B, L = shape
    flat = mask.reshape(-1)
    idx = torch.arange(B, device=mask.device)[:, None] * L + torch.arange(L, device=mask.device)[None, :]
    out = torch.zeros(B, L, dtype=mask.dtype, device=mask.device)
    ok = idx < flat.numel()
    out[ok] = flat[idx[ok]]
    return out


def key_masks(input_mask, image_mask, task_tokens=True, dtype=torch.float64):
    """The additive key masks the engine builds: text [B, Tin + 1] (the task token's row always real), image [B, V]."""
    m = input_mask.long()
    if task_tokens:
        m = torch.cat([torch.ones_like(m[:, :1]), m], 1)
    return (1.0 - m.to(dtype)) * -10000.0, (1.0 - image_mask.to(dtype)) * -10000.0


# ---------------------------------------------------------------------------------------------------------------- teacher forcing
def row_err(out, ref):
    """(oracle.fp64.rel_err, where): the worst element's sample and row of [B, L, H] (or [B, H]) tensors."""
    o, r = out.detach().double().to(ref.device), ref.detach().double()
    assert tuple(o.shape) == tuple(r.shape), (tuple(o.shape), tuple(r.shape))
    if r.numel() == 0:
        return 0.0, ""
    e = (o - r).abs() / r.abs().clamp(min=1.0)
    e = e.reshape(e.shape[0], -1, e.shape[-1]).amax(-1)
    i = int(e.argmax())
    b, row = divmod(i, e.shape[1])
    return float(e.max()), f"sample {b} row {row}"


def map_err(out, ref):
    """(max |o - r|, where) of [B, heads, Lq, Lk] maps: sample, head and query row of the worst element."""
    o, r = out.detach().double().to(ref.device), ref.detach().double()
    assert tuple(o.shape) == tuple(r.shape), (tuple(o.shape), tuple(r.shape))
    if r.numel() == 0:
        return 0.0, ""
    e = (o - r).abs().amax(-1)
    i = int(e.argmax())
    b, rest = divmod(i, e.shape[1] * e.shape[2])
    h, row = divmod(rest, e.shape[2])
    return float(e.max()), f"sample {b} head {h} row {row}"


def entry_labels(schedule):
    """Labels of the full layer-state list: the embeddings, then per step its text state before its image state."""
    out = ["emb text", "emb image"]
    for step in schedule:
        out += ([f"{step} text"] if step[0] != "V" else []) + ([f"{step} image"] if step[0] != "T" else [])
    return out


def map_labels(schedule):
    """Labels of the attention maps flattened in execution order (both directions of a connection layer)."""
    return [x for step in schedule for x in ((f"{step} text->image", f"{step} image->text") if step[0] == "C" else (step,))]


def flat_maps(maps):
    """The engine's attention list (a tuple of two per connection layer) as one list in execution order."""
    return [x for m in maps for x in (m if isinstance(m, tuple) else (m,))]


def forced_steps(ref: StepRef, states, t_mask, v_mask, only=None):
    """The reference for entries 2.. of the full layer-state list, each step run on the given previous entries ``states``
    (teacher forcing), and the reference maps of every step (flattened): (entries, maps).  ``only``: run just these steps."""
    t, v = states[0], states[1]
    outs, maps = [], []
    e = 2
    for step in ref.schedule:
        if only is not None and step not in only:
            n = 2 if step[0] == "C" else 1
            t = states[e] if step[0] == "T" else states[e] if step[0] == "C" else t
            v = states[e + 1] if step[0] == "C" else states[e] if step[0] == "V" else v
            e += n
            continue
        if step[0] == "C":
            t_ref, v_ref, pair = ref.connection(int(step[1:]), t, v, t_mask, v_mask)
            outs += [t_ref, v_ref]
            maps += list(pair)
            t, v = states[e], states[e + 1]
            e += 2
            continue
        text = step[0] == "T"
        out, p = ref.layer(step, t if text else v, t_mask if text else v_mask)
        outs.append(out)
        maps.append(p)
        if text:
            t = states[e]
        else:
            v = states[e]
        e += 1
    assert e == len(states), (e, len(states))
    return outs, maps


def teacher_forced(ref: StepRef, states, emb_t, emb_v, t_mask, v_mask, maps=None):
    """Every entry of the engine's full layer-state list against ``ref`` run on the engine's previous entries.  ``states``: the
    entries [B, L, H] (embeddings, then per step its text state before its image state); ``emb_t`` / ``emb_v``: the reference
    embeddings; ``maps``: the engine's attention maps in execution order (as ``forward`` returns them) or None.  Returns
    {"states": [(label, err, where)], "maps": [...]}, each in execution order."""
    outs, ref_maps = forced_steps(ref, states, t_mask, v_mask)
    res = {"states": [(lab,) + row_err(s, r) for lab, s, r in zip(entry_labels(ref.schedule), states, [emb_t, emb_v] + outs)],
           "maps": []}
    if maps is not None:
        res["maps"] = [(lab,) + map_err(m, r) for lab, m, r in zip(map_labels(ref.schedule), flat_maps(maps), ref_maps)]
    return res


def worst(errs):
    """The (label, err, where) of a list with the largest err."""
    return max(errs, key=lambda x: x[1])


def first_over(errs, bound):
    """The first (label, err, where) of a list in execution order that is not below ``bound``, or None."""
    return next((x for x in errs if not x[1] < bound), None)
