"""Synthetic checkpoints and request tensors with the reference's key names, shapes and dtypes.

There is no network on the build/bench boxes and the reference ships no checkpoint
(`save/multitask_model/pytorch_model_9.bin`, worker.py:470, is absent), so benchmarks and smoke runs use a
seeded random-init state_dict of the *architecture* (key list of SURVEY.md section 8b) and synthetic requests
shaped like the tensors worker.py:416-419, 452-455 builds.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .config import BertConfig


def state_dict_spec(config: BertConfig, num_labels: int = 3129, gqa_labels: int = 1533) -> Dict[str, tuple]:
    """Upstream key -> shape for VILBertForVLTasks (the audit list the engine enforces)."""
    c = config
    H, Hv, Hb = c.hidden_size, c.v_hidden_size, c.bi_hidden_size
    spec: Dict[str, tuple] = {}

    def lin(p, n, k):
        spec[p + ".weight"] = (n, k)
        spec[p + ".bias"] = (n,)

    def ln(p, n):
        spec[p + ".weight"] = (n,)
        spec[p + ".bias"] = (n,)

    spec["bert.embeddings.word_embeddings.weight"] = (c.vocab_size, H)
    spec["bert.embeddings.position_embeddings.weight"] = (c.max_position_embeddings, H)
    spec["bert.embeddings.token_type_embeddings.weight"] = (c.type_vocab_size, H)
    if c.task_specific_tokens:
        spec["bert.embeddings.task_embeddings.weight"] = (getattr(c, "num_task_tokens", 20), H)
    ln("bert.embeddings.LayerNorm", H)
    lin("bert.v_embeddings.image_embeddings", Hv, c.v_feature_size)
    lin("bert.v_embeddings.image_location_embeddings", Hv, 5)
    ln("bert.v_embeddings.LayerNorm", Hv)

    def layer(p, hid, inter):
        for n in ("query", "key", "value"):
            lin(f"{p}.attention.self.{n}", hid, hid)
        lin(f"{p}.attention.output.dense", hid, hid)
        ln(f"{p}.attention.output.LayerNorm", hid)
        lin(f"{p}.intermediate.dense", inter, hid)
        lin(f"{p}.output.dense", hid, inter)
        ln(f"{p}.output.LayerNorm", hid)

    for i in range(c.num_hidden_layers):
        layer(f"bert.encoder.layer.{i}", H, c.intermediate_size)
    for i in range(c.v_num_hidden_layers):
        layer(f"bert.encoder.v_layer.{i}", Hv, c.v_intermediate_size)
    for i in range(len(c.v_biattention_id)):
        p = f"bert.encoder.c_layer.{i}"
        for n in ("query1", "key1", "value1"):
            lin(f"{p}.biattention.{n}", Hb, Hv)
        for n in ("query2", "key2", "value2"):
            lin(f"{p}.biattention.{n}", Hb, H)
        lin(f"{p}.biOutput.dense1", Hv, Hb)
        ln(f"{p}.biOutput.LayerNorm1", Hv)
        lin(f"{p}.biOutput.q_dense1", Hv, Hb)
        lin(f"{p}.biOutput.dense2", H, Hb)
        ln(f"{p}.biOutput.LayerNorm2", H)
        lin(f"{p}.biOutput.q_dense2", H, Hb)
        lin(f"{p}.v_intermediate.dense", c.v_intermediate_size, Hv)
        lin(f"{p}.v_output.dense", Hv, c.v_intermediate_size)
        ln(f"{p}.v_output.LayerNorm", Hv)
        lin(f"{p}.t_intermediate.dense", c.intermediate_size, H)
        lin(f"{p}.t_output.dense", H, c.intermediate_size)
        ln(f"{p}.t_output.LayerNorm", H)
    lin("bert.t_pooler.dense", Hb, H)
    lin("bert.v_pooler.dense", Hb, Hv)
    spec["cls.predictions.bias"] = (c.vocab_size,)
    lin("cls.predictions.transform.dense", H, H)
    ln("cls.predictions.transform.LayerNorm", H)
    spec["cls.predictions.decoder.weight"] = (c.vocab_size, H)          # tied to the word table
    lin("cls.bi_seq_relationship", 2, Hb)
    lin("cls.imagePredictions.transform.dense", Hv, Hv)
    ln("cls.imagePredictions.transform.LayerNorm", Hv)
    lin("cls.imagePredictions.decoder", c.v_target_size, Hv)

    def simple(p, i, h, o):
        lin(f"{p}.logit_fc.0", h, i)
        ln(f"{p}.logit_fc.2", h)
        lin(f"{p}.logit_fc.3", o, h)

    simple("vil_prediction", Hb, 2 * Hb, num_labels)
    simple("vil_prediction_gqa", Hb, 2 * Hb, gqa_labels)
    simple("vil_binary_prediction", 2 * Hb, 2 * Hb, 2)
    lin("vil_logit", 1, Hb)
    lin("vil_tri_prediction", 3, Hb)
    lin("vision_logit", 1, Hv)
    lin("linguisic_logit", 1, H)
    return spec


def synthetic_state_dict(config: BertConfig, num_labels: int = 3129, gqa_labels: int = 1533, seed: int = 42,
                         bf16_exact: bool = True) -> Dict[str, torch.Tensor]:
    """Random-init checkpoint of the architecture: weights ~ N(0, 0.02), LayerNorm gamma ~ 1 + N(0, 0.1),
    beta ~ N(0, 0.1), biases ~ N(0, 0.05) (seed 42 echoes worker.py:477)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for k, shape in state_dict_spec(config, num_labels, gqa_labels).items():
        if k == "cls.predictions.decoder.weight":
            continue
        is_ln = ".LayerNorm" in k or ".logit_fc.2." in k
        if len(shape) == 2:
            w = torch.randn(shape, generator=g) * 0.02
            if bf16_exact and "embeddings.weight" not in k:
                w = w.to(torch.bfloat16).float()
            sd[k] = w
        elif is_ln and k.endswith(".weight"):
            sd[k] = 1.0 + torch.randn(shape, generator=g) * 0.1
        elif is_ln:
            sd[k] = torch.randn(shape, generator=g) * 0.1
        else:
            sd[k] = torch.randn(shape, generator=g) * 0.05
    sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    return sd


# the task heads of a multi-task checkpoint: absent from a pre-training one (upstream BertForMultiModalPreTraining has bert + cls)
TASK_HEAD_PREFIXES = ("vil_prediction.", "vil_prediction_gqa.", "vil_binary_prediction.", "vil_logit.", "vil_tri_prediction.",
                      "vision_logit.", "linguisic_logit.")


def synthetic_pretraining_state_dict(config: BertConfig, seed: int = 42, bf16_exact: bool = True) -> Dict[str, torch.Tensor]:
    """Random-init pre-training checkpoint (``bert.*`` and ``cls.*``, no task heads) drawn as ``synthetic_state_dict``.  The
    config must have ``task_specific_tokens`` off, as upstream's pre-training config does (no task embedding table)."""
    if getattr(config, "task_specific_tokens", False):
        raise ValueError("a pre-training checkpoint has no task embeddings: set task_specific_tokens = False")
    sd = synthetic_state_dict(config, num_labels=2, gqa_labels=2, seed=seed, bf16_exact=bf16_exact)
    return {k: v for k, v in sd.items() if not k.startswith(TASK_HEAD_PREFIXES)}


def synthetic_masked_batch(batch: int, n_tokens: int = 36, n_regions: int = 37, seed: int = 0, vocab_size: int = 30522,
                           v_feature_size: int = 2048, v_target_size: int = 1601, mask_prob: float = 0.15):
    """A masked pre-training batch shaped like upstream's Conceptual Captions loader output, for BertForMultiModalPreTraining.forward:
    dict of ``input_ids`` / ``token_type_ids`` / ``attention_mask`` [B, n_tokens], ``image_feat`` [B, V, F] / ``image_loc`` [B, V, 5]
    / ``image_attention_mask`` [B, V] (V = n_regions, the global row first), ``masked_lm_labels`` [B, n_tokens] (the original id at
    about ``mask_prob`` of the word tokens, now [MASK] = 103; -1 elsewhere), ``image_label`` [B, V - 1] (1 at about ``mask_prob`` of
    the regions, whose features are zeroed; -1 elsewhere), ``image_target`` [B, V - 1, v_target_size] (detector class distributions:
    softmax rows with some classes exactly 0, renormalised) and ``next_sentence_label`` [B] (0 / 1, some -1)."""
    B, V = batch, n_regions
    q, feats, spatials, segment_ids, input_mask, image_mask, _, _ = synthetic_request(
        B, n_tokens, V, seed=seed, v_feature_size=v_feature_size, vocab_size=vocab_size, full_masks=False)
    g = torch.Generator().manual_seed(seed + 1)
    words = (q != 101) & (q != 102) & (input_mask == 1)
    masked = words & (torch.rand(q.shape, generator=g) < mask_prob)
    lm_labels = torch.where(masked, q, torch.full_like(q, -1))
    q = torch.where(masked, torch.full_like(q, 103), q)
    region = torch.rand(B, V - 1, generator=g) < mask_prob
    image_label = torch.where(region, torch.ones(B, V - 1, dtype=torch.long), torch.full((B, V - 1), -1, dtype=torch.long))
    feats[:, 1:][region] = 0.0
    target = torch.softmax(torch.randn(B, V - 1, v_target_size, generator=g) * 3.0, dim=-1)
    target = target * (torch.rand(B, V - 1, v_target_size, generator=g) > 0.2)
    target = target / target.sum(-1, keepdim=True)
    nsp = torch.randint(0, 2, (B,), generator=g)
    nsp[torch.rand(B, generator=g) < 0.1] = -1
    return dict(input_ids=q, image_feat=feats, image_loc=spatials, token_type_ids=segment_ids, attention_mask=input_mask,
                image_attention_mask=image_mask, masked_lm_labels=lm_labels, image_label=image_label, image_target=target,
                next_sentence_label=nsp)


def synthetic_detections(n_images: int, n_proposals=1000, n_classes: int = 1601, feature_size: int = 2048, seed: int = 0,
                         margin: Optional[float] = None, n_clusters: int = 12, n_dominant: int = 24, im_scale: float = 1.6):
    """Raw detector heads per image, shaped like the Faster R-CNN outputs the reference worker's feature extraction reads
    (worker.py:123-176): ``[(proposals [n, 4], scores [n, C], features [n, F], im_scale)]``, CPU fp32.  ``n_proposals`` is one count
    or one per image.

    Boxes (at the detector's input scale, ``im_scale`` times the image) are drawn around ``n_clusters`` centres, so neighbours
    overlap and the NMS has real work.  Every proposal has a dominant class among ``n_dominant``; features are relu(N(0, 1)) * 1.5.
    Logits: with ``margin=None`` N(0, 2) plus 6 on the dominant class.  With a ``margin`` d, the dominant logit is 0 and every other
    one is -26 - d * u for an integer u < 55 / d: the exponentials of the others sum below half an ulp of 1, so every softmax sum
    is exactly 1 in any summation order, and two probabilities of different logits differ by a factor of at least exp(d), so the
    selection does not depend on rounding; equal logits give equal probabilities and fall to the index tie rule."""
    g = torch.Generator().manual_seed(seed)
    counts = [int(n_proposals)] * n_images if isinstance(n_proposals, int) else [int(n) for n in n_proposals]
    n_dominant = min(n_dominant, n_classes - 1)
    dominant = torch.randperm(n_classes - 1, generator=g)[:n_dominant] + 1
    out = []
    for n in counts:
        img = torch.tensor([1333.0, 800.0]) * im_scale
        centres = torch.rand(n_clusters, 2, generator=g) * img * 0.8 + img * 0.1
        cl = torch.randint(0, n_clusters, (n,), generator=g)
        size = (0.05 + torch.rand(n, 2, generator=g) * 0.3) * img
        c = centres[cl] + torch.randn(n, 2, generator=g) * size * 0.15
        x1y1 = (c - size / 2).clamp(min=0.0)
        x2y2 = torch.minimum(c + size / 2, img - 1)
        proposals = torch.cat([x1y1, torch.maximum(x2y2, x1y1 + 1)], dim=1).float()
        dom = dominant[torch.randint(0, n_dominant, (n,), generator=g)]
        if margin is None:
            scores = torch.randn(n, n_classes, generator=g) * 2.0
            scores[torch.arange(n), dom] += 6.0
        else:
            u = torch.randint(0, max(1, int(55.0 / margin)), (n, n_classes), generator=g).float()
            scores = -26.0 - float(margin) * u
            scores[torch.arange(n), dom] = 0.0
        features = torch.relu(torch.randn(n, feature_size, generator=g)) * 1.5
        out.append((proposals, scores.float().contiguous(), features, float(im_scale)))
    return out


def synthetic_request(batch: int, n_tokens: int = 30, n_regions: int = 36, seed: int = 1234, task_id: int = 1,
                      v_feature_size: int = 2048, vocab_size: int = 30522, full_masks: bool = True):
    """Request tensors as the worker builds them (worker.py:402-455): features = relu(N(0,1))*1.5 with the
    mean-pooled global row first, normalised boxes with [0,0,1,1,1] first, [CLS] ids [SEP] pad."""
    g = torch.Generator().manual_seed(seed)
    B, L, V = batch, n_tokens, n_regions
    feats = torch.relu(torch.randn(B, V, v_feature_size, generator=g)) * 1.5
    if V > 1:
        feats[:, 0] = feats[:, 1:].mean(dim=1)
    xy = torch.rand(B, V, 2, generator=g) * 0.7
    wh = 0.05 + torch.rand(B, V, 2, generator=g) * 0.25
    x2y2 = (xy + wh).clamp(max=1.0)
    spatials = torch.cat([xy, x2y2, ((x2y2 - xy)[..., 0] * (x2y2 - xy)[..., 1]).unsqueeze(-1)], dim=-1)
    spatials[:, 0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
    question = torch.zeros(B, L, dtype=torch.long)
    input_mask = torch.zeros(B, L, dtype=torch.long)
    lens = torch.full((B,), L - 2) if full_masks else torch.randint(min(5, L - 2), L - 1, (B,), generator=g)
    for b in range(B):
        n = int(lens[b])
        question[b, 0] = 101
        question[b, 1:1 + n] = torch.randint(1000, vocab_size, (n,), generator=g)
        question[b, 1 + n] = 102
        input_mask[b, :n + 2] = 1
    segment_ids = torch.zeros(B, L, dtype=torch.long)
    image_mask = torch.ones(B, V, dtype=torch.uint8)
    co_attention_mask = torch.zeros(B, V, L)
    task_tokens = torch.full((B, 1), task_id, dtype=torch.long)
    return question, feats, spatials, segment_ids, input_mask, image_mask, co_attention_mask, task_tokens
