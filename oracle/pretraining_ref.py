"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  Upstream's BertForMultiModalPreTraining (visual_target 0), restated.

Upstream's ``vilbert`` package is absent here, so the pre-training forward and its three losses are a restatement on top of
``vilbert_ref``'s ``BertModel`` and ``BertPreTrainingHeads`` (whose behaviour and ``UPSTREAM_ASSUMPTIONS`` this module leaves as
they are).  Every convention only upstream could confirm is a named flag in ``PRETRAINING_ASSUMPTIONS``.  The product path never
imports this module.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from oracle import vilbert_ref as R

PRETRAINING_ASSUMPTIONS = {
    "image_loss_skips_global_row": True,   # prediction_scores_v[:, 1:]: image_label / image_target cover the regions after row 0
    "image_loss_normalisation": "sum(KL over classes and masked regions) / count(image_label == 1)",   # 0 / 0 = NaN when none
    "image_loss": "KLDivLoss(reduction='none')(log_softmax(prediction_scores_v), image_target)",     # visual_target 0
    "ignore_index": -1,                    # masked_lm_labels and next_sentence_label: CrossEntropyLoss(ignore_index=-1), mean
    "forward_without_task_ids": True,      # the pre-training config has task_specific_tokens off; no task ids reach the embeddings
    "matched_alignment_column": None,      # which bi_seq_relationship column means "matched": unfixed (the losses do not need it)
    "loss_shapes": "[1]",                  # each loss is returned unsqueezed to [1]
}


def pretraining_config(**kw) -> R.RefConfig:
    """``vilbert_ref``'s config with the pre-training settings: no task tokens."""
    kw.setdefault("task_specific_tokens", False)
    return R.RefConfig(**kw)


def tiny_pretraining_config(**kw) -> R.RefConfig:
    kw.setdefault("task_specific_tokens", False)
    return R.tiny_config(**kw)


def pretraining_losses(prediction_scores_t, prediction_scores_v, seq_relationship_score, masked_lm_labels, image_label, image_target,
                       next_sentence_label):
    """The three losses of upstream's forward with labels, from the heads' scores (any float dtype; computed in that dtype)."""
    vocab = prediction_scores_t.shape[-1]
    ce = nn.CrossEntropyLoss(ignore_index=PRETRAINING_ASSUMPTIONS["ignore_index"])
    masked_lm_loss = ce(prediction_scores_t.reshape(-1, vocab), masked_lm_labels.reshape(-1))
    v = prediction_scores_v[:, 1:] if PRETRAINING_ASSUMPTIONS["image_loss_skips_global_row"] else prediction_scores_v
    img_loss = nn.KLDivLoss(reduction="none")(F.log_softmax(v, dim=2), image_target)
    picked = (image_label == 1)
    masked_img_loss = torch.sum(img_loss * picked.unsqueeze(2).to(img_loss.dtype)) / max(torch.sum(picked), 0)
    next_sentence_loss = ce(seq_relationship_score.reshape(-1, 2), next_sentence_label.reshape(-1))
    return masked_lm_loss.unsqueeze(0), masked_img_loss.unsqueeze(0), next_sentence_loss.unsqueeze(0)


class BertForMultiModalPreTraining(nn.Module):
    def __init__(self, config: R.RefConfig):
        super().__init__()
        self.config = config
        self.bert = R.BertModel(config)
        self.cls = R.BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight)

    @torch.no_grad()
    def forward(self, input_ids, image_feat, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                masked_lm_labels=None, image_label=None, image_target=None, next_sentence_label=None, collect: Optional[dict] = None):
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if image_attention_mask is None:
            image_attention_mask = torch.ones(image_feat.size(0), image_feat.size(1), dtype=torch.long)
        dt = self.cls.bi_seq_relationship.weight.dtype
        t, v, pooled_t, pooled_v, attn = self.bert(input_ids, image_feat.to(dt), image_loc.to(dt), token_type_ids, attention_mask,
                                                   image_attention_mask, None, collect)
        if collect is not None:
            collect["final"] = (t, v, pooled_t, pooled_v)
        scores_t, scores_v, seq_rel = self.cls(t, v, pooled_t, pooled_v)
        if masked_lm_labels is None:
            return scores_t, scores_v, seq_rel, attn
        return pretraining_losses(scores_t, scores_v, seq_rel, masked_lm_labels, image_label, image_target, next_sentence_label)


def build(config: Optional[R.RefConfig] = None, seed: int = 42) -> BertForMultiModalPreTraining:
    """Seeded synthetic pre-training model, weights drawn as ``vilbert_ref.init_weights`` draws them."""
    model = BertForMultiModalPreTraining(config or pretraining_config())
    R.init_weights(model, seed=seed)
    return model.eval()
