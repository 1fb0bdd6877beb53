"""BertForMultiModalPreTraining: upstream's pre-training model (``vilbert.vilbert.BertForMultiModalPreTraining``) on the engine.

    model = BertForMultiModalPreTraining.from_pretrained(ckpt, config=config).eval().cuda(0)
    t, v, align, attn = model(input_ids, image_feat, image_loc, token_type_ids, attention_mask, image_attention_mask)
    lm, img, nsp = model(..., masked_lm_labels=..., image_label=..., image_target=..., next_sentence_label=...)

The checkpoint (Conceptual Captions pre-training, the one every ViLBERT task model is fine-tuned from) holds the encoder and the
``cls`` heads but no task heads; vb200_create_pretraining audits it against that key set.  Everything else -- packed and cached
forwards, retrieval, ``pretraining_heads`` and ``pretraining_objectives`` -- is ``VILBertForVLTasks``'s, with ``select`` limited to the
pre-training heads, the taps and the attention maps.  Inference only: ``train()`` raises.
"""
from __future__ import annotations

import torch

from . import _lib as L
from .model import VILBertForVLTasks


class BertForMultiModalPreTraining(VILBertForVLTasks):
    """Drop-in for ``vilbert.vilbert.BertForMultiModalPreTraining`` (visual_target 0) on the inference path."""

    _create_fn = "vb200_create_pretraining"

    def __init__(self, config, state_dict=None, **kwargs):
        kwargs.pop("num_labels", None)                 # a pre-training checkpoint has no answer head
        super().__init__(config, num_labels=0, state_dict=state_dict, **kwargs)

    @torch.no_grad()
    def forward(self, input_ids, image_feat, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                masked_lm_labels=None, image_label=None, image_target=None, next_sentence_label=None, output_all_attention_masks=False):
        """Upstream's pre-training forward.  Without labels: ``(prediction_scores_t [B, T, vocab], prediction_scores_v [B, V,
        v_target_size], seq_relationship_score [B, 2], all_attention_mask)`` -- the full-row heads of one forward, and the alignment
        head on each sample's pooled state (which column means "matched" is upstream's convention; both logits are returned).
        ``all_attention_mask`` follows ``VILBertForVLTasks.forward``'s element 9.

        With labels (all four together): ``(masked_lm_loss [1], masked_img_loss [1], next_sentence_loss [1])``, computed on the
        device by ``pretraining_objectives`` at the rows the labels pick (the labels are read on the host):
        ``masked_lm_labels`` [B, Tin] (-1: not masked) -> cross-entropy over the masked tokens; ``image_label`` [B, V - 1] and
        ``image_target`` [B, V - 1, v_target_size] for the regions after the global row -> the KL divergence summed over the
        classes of the regions with ``image_label == 1``, divided by their count; ``next_sentence_label`` [B] (-1: ignored) ->
        cross-entropy of the alignment head.  A batch with nothing to score in a list gives NaN for it, as upstream's 0 / 0."""
        labels = (masked_lm_labels, image_label, image_target, next_sentence_label)
        if any(x is not None for x in labels) and any(x is None for x in labels):
            raise ValueError("pass masked_lm_labels, image_label, image_target and next_sentence_label together")
        with_labels = masked_lm_labels is not None
        select = 0 if with_labels else L.OUT_LINGUISIC_PREDICTION | L.OUT_VISION_PREDICTION
        out, taps = super().forward(input_ids, image_feat, image_loc, token_type_ids, attention_mask, image_attention_mask, None, None,
                                    output_all_attention_masks=output_all_attention_masks, select=select, debug_taps=True)
        B, Tin = input_ids.shape
        V = image_feat.shape[1]
        if not with_labels:
            align = self.pretraining_heads(taps, pair_rows=range(B))["alignment"]
            return out[7], out[5], align, out[9]
        task = 1 if self._dims["task_specific_tokens"] else 0
        lm = torch.as_tensor(masked_lm_labels).to("cpu", torch.int64)
        il = torch.as_tensor(image_label).to("cpu", torch.int64)
        ns = torch.as_tensor(next_sentence_label).to("cpu", torch.int64).reshape(-1)
        if tuple(lm.shape) != (B, Tin) or tuple(il.shape) != (B, V - 1) or ns.numel() != B:
            raise ValueError(f"labels: masked_lm_labels [{B}, {Tin}], image_label [{B}, {V - 1}] and next_sentence_label [{B}] expected")
        tb, tt = (lm != -1).nonzero(as_tuple=True)
        vb_, vj = (il == 1).nonzero(as_tuple=True)
        pb = (ns != -1).nonzero(as_tuple=True)[0]
        target = torch.as_tensor(image_target)
        vt = self._dims["v_target_size"]
        if tuple(target.shape) != (B, V - 1, vt):
            raise ValueError(f"image_target must be [{B}, {V - 1}, {vt}]")
        targets = target.to(taps["sequence_output_v"].device, torch.float32)[vb_, vj]
        res = self.pretraining_objectives(taps, text_rows=tb * (Tin + task) + task + tt, token_labels=lm[tb, tt],
                                          image_rows=vb_ * V + 1 + vj, image_targets=targets, pair_rows=pb, pair_labels=ns[pb])
        return res["masked_lm_loss"], res["masked_img_loss"], res["next_sentence_loss"]
