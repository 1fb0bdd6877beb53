"""Task / prediction API of the reference worker, minus Django, RabbitMQ and the detector.

Same call signatures, same validation, same per-task output dictionaries as
worker.py:

    custom_prediction(query, task, features, infos, task_id)                      worker.py:388-458
    prediction(question, features, spatials, segment_ids, input_mask, image_mask,
               co_attention_mask, task_tokens, task_id, infos)                    worker.py:248-386
    shape_result(task_id, answer, image_path)   (the `result` dicts of callback)  worker.py:564-645

Differences that do not change results: the model call goes to the sm_90a engine; only the heads a task
reads are computed (the reference computes all ten outputs and drops nine); top-N uses `topk` instead of a
full sort + per-element `.item()`; label maps are loaded once instead of per request (worker.py:299-300,
311-315); `eval(task_id)` (worker.py:562) is `int(task_id)`.
"""
from __future__ import annotations

import functools
import os
import pickle
import re
import unicodedata
from itertools import accumulate
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L

# ------------------------------------------------------------------------------------------ module state
# (the reference keeps `model`, `tokenizer`, `feature_extractor` as module globals, worker.py:464-466)
model = None
tokenizer = None
# One engine handle serves one host thread at a time (plan cache and last_error are per handle, unlocked): every model call
# of this module -- prediction(), prediction_batch(), the MicroBatchWorker thread -- takes this lock.
import threading as _threading
model_lock = _threading.RLock()
label_maps: Dict[str, Optional[list]] = {"vqa": None, "gqa": None}

MAX_LENGTH = 37                     # worker.py:408
SINGLE_IMAGE_TASKS = ("1", "15", "13", "11", "4", "16")   # worker.py:256
PAIR_TASKS = ("12",)                # worker.py:258
RETRIEVAL_TASKS = ("7",)            # worker.py:260
GROUNDING_TASKS = ("11", "4", "16")  # worker.py:374
# task id -> which element of the 10-tuple the decode reads (worker.py:295-374)
TASK_OUTPUT = {"1": L.OUT_VIL_PREDICTION, "2": L.OUT_VIL_PREDICTION, "15": L.OUT_VIL_PREDICTION_GQA,
               "12": L.OUT_VIL_BINARY_PREDICTION, "13": L.OUT_VIL_TRI_PREDICTION, "7": L.OUT_VIL_LOGIT,
               "11": L.OUT_VISION_LOGIT, "4": L.OUT_VISION_LOGIT, "16": L.OUT_VISION_LOGIT}
# task-id -> name table of the demo page (demo/templates/vilbert_multitask/result.html:321-335)
TASK_NAMES = {"1": "VQA", "2": "VG-QA", "15": "GQA", "12": "NLVR2", "13": "SNLI-VE", "7": "Image Retrieval",
              "11": "RefCOCO", "4": "Visual7W", "16": "GuessWhat"}


def load_vilbert_model(from_pretrained, config_file, num_labels: int = 3129, device: int = 0, vocab_file=None,
                       label2ans: Optional[Dict[str, str]] = None, tokenizer_obj=None, max_rows_per_sample: int = 256, **engine_kw):
    """worker.py:463-539 without the detector: config mutation (worker.py:509-522), from_pretrained, eval, cuda.
    max_rows_per_sample (256..1024): the longest query (wordpieces + the task token) or image (boxes + the global row) the model
    serves; text stays bounded by max_position_embeddings as well."""
    global model, tokenizer
    from .config import BertConfig
    from .model import VILBertForVLTasks
    config = config_file if isinstance(config_file, BertConfig) else BertConfig.from_json_file(config_file)
    config.v_target_size = 1601            # predict_feature=False, worker.py:512-514
    config.predict_feature = False
    config.task_specific_tokens = True     # worker.py:516-517
    config.visualization = True            # worker.py:522
    m = VILBertForVLTasks.from_pretrained(from_pretrained, config=config, num_labels=num_labels, default_gpu=True,
                                          max_rows_per_sample=max_rows_per_sample, **engine_kw)
    m.eval()
    m = m.cuda(device)
    model = m
    tokenizer = tokenizer_obj if tokenizer_obj is not None else (WordpieceTokenizer(vocab_file) if vocab_file else None)
    for key, path in (label2ans or {}).items():
        with open(path, "rb") as f:
            label_maps[key] = pickle.load(f)
    return m


def _label(kind: str, idx: int):
    m = label_maps.get(kind)
    if m is None:       # no trainval_label2ans.pkl on this box (worker.py:299, 311 read them from save/...)
        return f"<{kind}:{idx}>"
    return m[idx]


def _top(prob_1d: torch.Tensor, n: int):
    val, idx = torch.topk(prob_1d, n)      # == sort descending + first n (worker.py:297, 314, 330, 346, 360, 376)
    return val.tolist(), idx.tolist()


def _validate(task_id, infos):
    """Image-count rules of worker.py:255-262."""
    if task_id in SINGLE_IMAGE_TASKS:
        assert len(infos) == 1, "task require 1 image"
    elif task_id in PAIR_TASKS:
        assert len(infos) == 2, "task require 2 images"
    elif task_id in RETRIEVAL_TASKS:
        assert len(infos) > 1 and len(infos) <= 10, "task require 2-10 images"
    else:
        raise ValueError("task not valid.")


def _expand_text(task_id, n_rows, question, input_mask, segment_ids, task_tokens):
    """The text is repeated per image for NLVR2 pairs and retrieval candidates (worker.py:266-284)."""
    rep = 2 if task_id == "12" else (n_rows if task_id == "7" else 1)
    if rep > 1:
        question, input_mask = question.repeat(rep, 1), input_mask.repeat(rep, 1)
        segment_ids, task_tokens = segment_ids.repeat(rep, 1), task_tokens.repeat(rep, 1)
    return question, input_mask, segment_ids, task_tokens


def _decode(task_id, out, spatials, infos):
    """Logits of ONE request -> the reference's answer (worker.py:295-386): softmax over the task's output flattened, top-N, and
    for grounding the top rows' boxes in pixels.  Grounding ranks ALL rows of vision_logit, the synthetic global box included
    (worker.py:374-385), and reads the boxes from the image's spatials [1, V, 5]."""
    top = len(infos) if task_id == "7" else 2 if task_id == "12" else 3          # worker.py:250-253
    # OUT_* bit k selects element k of the 10-tuple
    conf, idx = _top(torch.softmax(out[TASK_OUTPUT[task_id].bit_length() - 1].view(-1), dim=0), top)
    boxes = None
    if task_id in GROUNDING_TASKS:
        w, h = infos[0]["image_width"], infos[0]["image_height"]
        boxes = [[int(b[0] * w), int(b[1] * h), int(b[2] * w), int(b[3] * h)]
                 for b in spatials[0][torch.as_tensor(idx, device=spatials.device)][:, :4].tolist()]
    return _answer(task_id, idx, conf, boxes)


def _check_decode(decode):
    if decode not in ("host", "device"):
        raise ValueError(f"decode must be 'host' or 'device', not {decode!r}")


def decode_messages(tasks, spans, v_off):
    """The descriptors of `model.decode_answers` for the requests of one forward, with `_decode`'s N and segments.

    `tasks` maps a request to its `(task_id, infos)`, `spans` a request to the batch rows `(lo, hi)` it took, and `v_off` gives
    the first `vision_logit` row of every batch row (B + 1 entries: multiples of V for a dense forward, prefix sums of the rows per
    image for a packed one).  An NLVR2 pair (even lo) reads pair row lo // 2, retrieval its hi - lo rows with N = len(infos), grounding
    the image's vision rows [v_off[lo], v_off[hi]), the global box included, with the image size of infos[0].
    Returns `[(request, (task_id, first, count, top_n, image_wh))]` in the order of `spans`."""
    msgs = []
    for i, (lo, hi) in spans.items():
        task_id, infos = tasks[i]
        wh = None
        if task_id in GROUNDING_TASKS:
            first, count, top = int(v_off[lo]), int(v_off[hi]) - int(v_off[lo]), 3
            wh = (infos[0]["image_width"], infos[0]["image_height"])
        elif task_id == "12":
            first, count, top = lo // 2, hi // 2 - lo // 2, 2
        else:
            first, count, top = lo, hi - lo, (len(infos) if task_id == "7" else 3)
        msgs.append((i, (task_id, first, count, top, wh)))
    return msgs


def _answer(task_id, idx, conf, boxes):
    """The answer dict of one request from its top-N indices, probabilities and, for grounding, pixel boxes [x1, y1, x2, y2]
    (as `_decode` and `model.decode_answers` rank them)."""
    if task_id in ("1", "2"):
        return {"top3_answer": [_label("vqa", i) for i in idx], "top3_confidence": conf}
    if task_id == "15":
        return {"top3_answer": [_label("gqa", i) for i in idx], "top3_confidence": conf}
    if task_id == "12":
        names = {0: "False", 1: "True"}
        return {"top3_answer": [names[i] for i in idx], "top3_confidence": conf}
    if task_id == "13":
        names = {0: "contradiction (false)", 1: "neutral", 2: "entailment (true)"}
        return {"top3_answer": [names[i] for i in idx], "top3_confidence": conf}
    if task_id == "7":
        return {"top3_answer": idx, "top3_confidence": conf}
    return [{"y1": b[1], "y2": b[3], "x1": b[0], "x2": b[2], "confidence": c * 100} for b, c in zip(boxes, conf)]


def _row_layout(accepted, bucket, select):
    """The batch rows of one model call.  `accepted` lists the requests in order as `(request, task_id, its rows)`.

    An NLVR2 pair starts on an even row -- the binary head consumes adjacent rows as one pair (worker.py:266-276) -- with ONE
    filler row in front when needed.  The engine keeps one plan per batch size and select, so that a long-running worker sees a
    small, fixed set of plans: the batch is padded with filler rows to a multiple of `bucket` (and to an even count when the pair
    head is computed), and `select` (default: the seven task heads) is ORed with the heads the requests read.
    Returns (the rows, None at filler positions; spans {request: (first row, end row)}; the select mask)."""
    rows, spans, need = [], {}, 0
    for i, task_id, own in accepted:
        if task_id in PAIR_TASKS and len(rows) % 2 == 1:
            rows.append(None)
        spans[i] = (len(rows), len(rows) + len(own))
        rows += own
        need |= TASK_OUTPUT[task_id]
    sel = (L.OUT_TASK_HEADS if select is None else int(select)) | need
    target = -(-len(rows) // bucket) * bucket
    if target % 2 == 1 and (sel & L.OUT_VIL_BINARY_PREDICTION):
        target += 1
    return rows + [None] * (target - len(rows)), spans, sel


def _split_outputs(out, spatials, lo, hi, v_off, t_off, task_id):
    """Rows [lo, hi) of a forward's outputs -> the 10-tuple and spatials `_decode` reads for one request.  Per-image outputs are
    sliced and the pair head keeps the request's pair.  Per-row outputs and spatials, packed [rows, ...], keep the request's vision
    rows [v_off[lo], v_off[hi]) and text rows [t_off[lo], t_off[hi]), shaped [1, rows, ...] for a single image."""
    sl = [None if o is None else o[lo:hi] for o in out[:5]] + [None] * 4 + [[]]
    if out[3] is not None:
        sl[3] = out[3][lo // 2:hi // 2] if task_id == "12" else out[3][0:0]
    one = hi - lo == 1
    for k, offs in ((5, v_off), (6, v_off), (7, t_off), (8, t_off)):
        if out[k] is not None:
            r = out[k][int(offs[lo]):int(offs[hi])]
            sl[k] = r.reshape(1, -1, r.shape[-1]) if one else r
    sp = spatials[int(v_off[lo]):int(v_off[hi])]
    return tuple(sl), (sp.reshape(1, -1, 5) if one else sp)


def _answer_spans(answers, out, spatials, tasks, spans, v_off, t_off, decode):
    """Fill in `answers[i]` for every request i of `spans` from one forward's outputs; `tasks` maps a request to `(task_id, infos)`
    and `v_off` / `t_off` give the first vision / text row of every batch row (see `_split_outputs`).  decode="device": one
    `model.decode_answers` call for all of them, given the spatials only when a grounding request reads them; "host": `_decode`
    per request on its slice of the outputs and spatials."""
    if decode == "device":
        msgs = decode_messages(tasks, spans, v_off)
        sp = None
        if any(m[0] in GROUNDING_TASKS for _, m in msgs):
            sp = spatials.to(device=torch.device("cuda", model._device), dtype=torch.float32).contiguous()
        with model_lock:
            res = model.decode_answers(out, [m for _, m in msgs], sp)
        for (i, m), r in zip(msgs, res):
            answers[i] = _answer(m[0], *r)
        return answers
    for i, (lo, hi) in spans.items():
        task_id, infos = tasks[i]
        sl, sp = _split_outputs(out, spatials, lo, hi, v_off, t_off, task_id)
        answers[i] = _decode(task_id, sl, sp, infos)
    return answers


def prediction(question, features, spatials, segment_ids, input_mask, image_mask, co_attention_mask, task_tokens,
               task_id, infos):
    """Validate, expand the text for pair / retrieval tasks, run the model once, decode.  worker.py:248-386."""
    _validate(task_id, infos)
    question, input_mask, segment_ids, task_tokens = _expand_text(task_id, features.size(0), question, input_mask,
                                                                  segment_ids, task_tokens)
    with model_lock:
        out = model(question, features, spatials, segment_ids, input_mask, image_mask, co_attention_mask, task_tokens,
                    output_all_attention_masks=True, select=TASK_OUTPUT[task_id])
    return _decode(task_id, out, spatials, infos)


def prediction_batch(requests, bucket: int = 8, select: Optional[int] = None, *, decode: str = "host"):
    """Micro-batching across requests (SURVEY.md section 8f-4; the reference handles one message at a time, worker.py:664-673).

    `requests` is a list of argument tuples of `prediction()`.  Requests whose tensors have the same text length, region count
    and feature width go through ONE model call; every pair's forward is independent of its batch neighbours, so each answer is
    what `prediction()` returns for that request alone.  NLVR2 requests (task 12) are placed on even rows -- the binary head
    consumes adjacent rows as one pair (worker.py:266-276) -- with ONE filler row in front when needed.  A request that fails
    validation gets its exception as its answer; the others are unaffected.

    The engine keeps one plan (workspace + CUDA graph) per (batch, text length, regions, select): so that a long-running worker
    sees a small, fixed set of plans, the batch is padded with filler rows to a multiple of `bucket` (even, so the binary
    head always has whole pairs) and `select` defaults to the seven task heads whatever tasks happen to be pending.

    `decode="device"` answers every request of a model call with one decode kernel and one device-to-host copy
    (`model.decode_answers`) instead of `_decode` per request; the answers have `_decode`'s structure."""
    if bucket < 1:
        raise ValueError("bucket must be >= 1")
    _check_decode(decode)
    answers = [None] * len(requests)
    groups = {}
    for i, r in enumerate(requests):
        (question, features, spatials, segment_ids, input_mask, image_mask, co_mask, task_tokens, task_id, infos) = r
        try:
            _validate(task_id, infos)
        except (AssertionError, ValueError) as e:
            answers[i] = e
            continue
        key = (question.shape[1], features.shape[1], features.shape[2])
        groups.setdefault(key, []).append(i)
    for idxs in groups.values():
        accepted = []
        for i in idxs:
            (question, features, spatials, segment_ids, input_mask, image_mask, co_mask, task_tokens, task_id, infos) = requests[i]
            q, im, seg, tk = _expand_text(task_id, features.size(0), question, input_mask, segment_ids, task_tokens)
            if co_mask is None:
                co_mask = torch.zeros(features.size(0), features.size(1), question.size(1), device=features.device)
            # every row of the request refers to the request's tensors, which go into the batch once
            accepted.append((i, task_id, [(q, features, spatials, seg, im, image_mask, co_mask, tk)] * features.size(0)))
        rows, spans, sel = _row_layout(accepted, bucket, select)
        parts = []                                         # filler rows: copies of the row before them, results discarded
        for r in rows:
            if r is None:
                parts.append(tuple(t[-1:] for t in parts[-1]))
            elif not parts or r is not parts[-1]:
                parts.append(r)
        cat = [torch.cat([r[k] for r in parts], dim=0) for k in range(8)]
        with model_lock:
            out = model(*cat, output_all_attention_masks=True, select=sel)
        # the per-row outputs [B, rows, ...] and the spatials in the packed layout [B * rows, ...]
        V, T = cat[1].shape[1], next((o.shape[1] for o in out[7:9] if o is not None), 0)
        out = tuple(o.flatten(0, 1) if 5 <= k <= 8 and o is not None else o for k, o in enumerate(out))
        _answer_spans(answers, out, cat[2].flatten(0, 1), {i: (requests[i][8], requests[i][9]) for i in idxs}, spans,
                      [k * V for k in range(len(rows) + 1)], [k * T for k in range(len(rows) + 1)], decode)
    return answers


def _prefix_len(mask_row):
    """Length of a 0/1 text mask that is a run of ones followed by zeros (>= 1), else None."""
    m = [int(x) for x in mask_row.tolist()]
    k = sum(1 for x in m if x != 0)
    return k if k >= 1 and all(x == 1 for x in m[:k]) and all(x == 0 for x in m[k:]) else None


def prediction_packed(requests, bucket: int = 8, select: Optional[int] = None, *, decode: str = "host"):
    """`prediction_batch` in ONE model call whatever the requests' shapes: a packed variable-length batch
    (`model.forward_packed`).  Padded text tokens are dropped (the `input_mask` must be a prefix of ones), region rows are kept
    as given (the `image_mask` must be all ones); a request that breaks either rule, or fails validation, gets a `ValueError` /
    its exception as its answer.  NLVR2 pairs go on even rows and the batch is padded to a multiple of `bucket`, both with
    filler rows of one token and one region.  The plan capacities are the widest padded text and the most regions among the
    requests (37 tokens from the worker's tokenizer), so a long-running worker sees one plan per batch bucket.  `decode` as for
    `prediction_batch`."""
    if bucket < 1:
        raise ValueError("bucket must be >= 1")
    _check_decode(decode)
    answers = [None] * len(requests)
    accepted = []                               # rows: (tokens [Tin], segments [Tin], task [1], features [V, F], spatials [V, 5])
    max_tin, max_v, F, dev = 1, 1, None, None
    for i, r in enumerate(requests):
        (question, features, spatials, segment_ids, input_mask, image_mask, co_mask, task_tokens, task_id, infos) = r
        try:
            _validate(task_id, infos)
            if image_mask is not None and not bool((image_mask != 0).all()):
                raise ValueError("prediction_packed: image_mask must be all ones (packed rows are all real)")
            q, im, seg, tk = _expand_text(task_id, features.size(0), question, input_mask, segment_ids, task_tokens)
            lens = [_prefix_len(im[j]) for j in range(features.size(0))]
            if any(k is None for k in lens):
                raise ValueError("prediction_packed: input_mask must be a prefix of ones")
        except (AssertionError, ValueError) as e:
            answers[i] = e
            continue
        F, dev = features.size(2), features.device
        accepted.append((i, task_id, [(q[j, :k], seg[j, :k], tk[j].reshape(1), features[j], spatials[j]) for j, k in enumerate(lens)]))
        max_tin, max_v = max(max_tin, q.size(1)), max(max_v, features.size(1))
    if not accepted:
        return answers
    samples, spans, sel = _row_layout(accepted, bucket, select)
    filler = (torch.zeros(1, dtype=torch.long, device=dev), torch.zeros(1, dtype=torch.long, device=dev),
              torch.zeros(1, dtype=torch.long, device=dev), torch.zeros(1, F, device=dev), torch.zeros(1, 5, device=dev))
    samples = [filler if smp is None else smp for smp in samples]
    cat = [torch.cat([smp[k] for smp in samples], dim=0) for k in range(5)]
    n_tokens = [int(smp[0].numel()) for smp in samples]
    n_regions = [int(smp[3].shape[0]) for smp in samples]
    with model_lock:
        out = model.forward_packed(cat[0], cat[3], cat[4], cat[1], cat[2].view(-1, 1), n_tokens, n_regions, select=sel,
                                   max_tokens=max_tin, max_regions=max_v)
    return _answer_spans(answers, out, cat[4], {i: (requests[i][8], requests[i][9]) for i in spans}, spans,
                         list(accumulate(n_regions, initial=0)),
                         list(accumulate([n + 1 for n in n_tokens], initial=0)),    # each text: its tokens and the task token
                         decode)


def build_inputs(query, task, features, infos, device, tok=None):
    """The tensor construction half of custom_prediction (worker.py:402-455), returned instead of consumed."""
    tokens, input_mask, segment_ids = tokenize_query(query, tok)
    text = torch.tensor(tokens, dtype=torch.long, device=device).unsqueeze(0)
    input_mask = torch.tensor(input_mask, dtype=torch.long, device=device).unsqueeze(0)
    segment_ids = torch.tensor(segment_ids, dtype=torch.long, device=device).unsqueeze(0)
    task_t = torch.tensor(np.array(task), dtype=torch.long, device=device).unsqueeze(0)

    feats, locs, masks = [], [], []
    for feature, info in zip(features, infos):
        w, h = float(info["image_width"]), float(info["image_height"])
        feature = torch.as_tensor(feature).to(device)
        n = feature.shape[0]
        g_feat = feature.sum(dim=0) / n                                   # mean-pooled global row (worker.py:432-434)
        feats.append(torch.cat([g_feat.view(1, -1), feature], dim=0))
        boxes = np.asarray(info["bbox"], dtype=np.float32)
        loc = np.zeros((boxes.shape[0], 5), dtype=np.float32)
        loc[:, :4] = boxes
        loc[:, 4] = (loc[:, 3] - loc[:, 1]) * (loc[:, 2] - loc[:, 0]) / (w * h)
        loc[:, [0, 2]] /= w
        loc[:, [1, 3]] /= h
        loc = np.concatenate([np.array([[0, 0, 1, 1, 1]], dtype=np.float32), loc], axis=0)   # worker.py:443-444
        locs.append(torch.from_numpy(loc))
        masks.append(torch.ones(n + 1, dtype=torch.uint8))
    features_t = torch.stack(feats, dim=0).float().to(device)              # requires equal n across images
    spatials = torch.stack(locs, dim=0).float().to(device)
    image_mask = torch.stack(masks, dim=0).to(device)
    co_attention_mask = torch.zeros((len(infos), features_t.shape[1], text.shape[1]), device=device)
    return text, features_t, spatials, segment_ids, input_mask, image_mask, co_attention_mask, task_t


def tokenize_query(query, tok=None):
    """worker.py:402-414: encode, add [CLS]/[SEP], pad (never truncate) to 37 -> (tokens, input_mask, segment_ids) lists."""
    tok = tok if tok is not None else tokenizer
    if tok is None:
        raise L.VilbertB200Error("no tokenizer: pass vocab_file= (bert-base-uncased vocab.txt) to load_vilbert_model")
    tokens = tok.add_special_tokens_single_sentence(tok.encode(query))
    segment_ids, input_mask = [0] * len(tokens), [1] * len(tokens)
    if len(tokens) < MAX_LENGTH:
        pad = [0] * (MAX_LENGTH - len(tokens))
        tokens, input_mask, segment_ids = tokens + pad, input_mask + pad, segment_ids + pad
    return tokens, input_mask, segment_ids


def custom_prediction(query, task, features, infos, task_id):
    """worker.py:388-458 (the GuessWhat dialog rewrite at 391-400 builds `tokens` and then discards it).

    The image half of the reference's tensor construction (global mean row, cat, box normalisation, [0,0,1,1,1], masks,
    stack -- worker.py:422-453) runs inside the engine's region-pack kernel: the detector's box features go to the device
    as they are and are written straight into the image-embedding GEMM's 16-bit operand (`model.forward_regions`).  Images
    with different box counts -- which `torch.stack` at worker.py:452 cannot take -- are padded and masked."""
    _validate(task_id, infos)
    device = torch.device("cuda", model._device)
    tokens, input_mask, segment_ids = tokenize_query(query)
    n_img = len(infos)
    rep = n_img if task_id in PAIR_TASKS + RETRIEVAL_TASKS else 1          # text repeated per image (worker.py:266-284)
    text = torch.tensor([tokens] * rep, dtype=torch.long)
    mask_t = torch.tensor([input_mask] * rep, dtype=torch.long)
    seg_t = torch.tensor([segment_ids] * rep, dtype=torch.long)
    task_t = torch.tensor(np.array(task), dtype=torch.long).view(1, -1)[:, :1].repeat(rep, 1)
    counts = [int(f.shape[0]) for f in features]
    n = max(counts)
    feats = torch.zeros(n_img, n, features[0].shape[1], dtype=torch.float32)
    boxes = torch.zeros(n_img, n, 4, dtype=torch.float32)
    for i, (f, info) in enumerate(zip(features, infos)):
        feats[i, :counts[i]] = torch.as_tensor(f, dtype=torch.float32)
        boxes[i, :counts[i]] = torch.as_tensor(np.asarray(info["bbox"], dtype=np.float32))[:counts[i], :4]
    wh = torch.tensor([[float(info["image_width"]), float(info["image_height"])] for info in infos], dtype=torch.float32)
    num_boxes = None if min(counts) == n else torch.tensor(counts, dtype=torch.int32)
    with model_lock:
        out, spatials = model.forward_regions(text.to(device), seg_t.to(device), mask_t.to(device), task_t.to(device),
                                              feats.to(device), boxes.to(device), wh.to(device), num_boxes,
                                              select=TASK_OUTPUT[task_id], output_all_attention_masks=True)
    return _decode(task_id, out, spatials, infos)


def real_tokens(query, tok=None):
    """tokenize_query without the padding: the input_mask prefix of (tokens, segment_ids)."""
    tokens, input_mask, segment_ids = tokenize_query(query, tok)
    k = sum(1 for m in input_mask if m)
    return tokens[:k], segment_ids[:k]


def _max_rows() -> int:
    """Rows per sample the loaded model accepts in either stream (its max_rows_per_sample; 256 for a model without the knob): a
    query holds at most this - 1 tokens (+ the task token), an image this - 1 boxes (+ the global mean row)."""
    return int(getattr(model, "max_rows_per_sample", 256))


def _region_text(query, tok, max_rows):
    """The text half of a packed region request: the query's real tokens and segments, at most `max_rows` - 1 of them."""
    tokens, segs = real_tokens(query, tok)
    if len(tokens) + 1 > max_rows:
        raise ValueError(f"query of {len(tokens)} tokens: packed rows hold at most {max_rows - 1}")
    return tokens, segs


def _region_rows(task_id, task, tokens, segs, imgs):
    """The rows of a packed region request, `(tokens, segments, task token) + image half`: the text repeated per image for NLVR2
    and retrieval (worker.py:266-284), else with the first image only."""
    t = int(np.array(task).reshape(-1)[0])
    return [(tokens, segs, t) + img for img in (imgs if task_id in PAIR_TASKS + RETRIEVAL_TASKS else imgs[:1])]


def pack_region_requests(requests, bucket: int = 8, select: Optional[int] = None, max_boxes: int = 100, tok=None):
    """The host half of `custom_prediction_packed`: `custom_prediction` argument tuples `(query, task, features, infos, task_id)` ->
    the inputs of ONE `forward_regions_packed` call, as CPU tensors.

    Every text keeps its real tokens only and is repeated per image for NLVR2 / retrieval; every image keeps its own box count.
    NLVR2 pairs start on even rows and the batch is padded to a multiple of `bucket` (even when the pair head is computed), both with
    filler rows of one token and one zero box in a 1 x 1 image.  The capacities are max(MAX_LENGTH, longest query) tokens and
    max(`max_boxes`, most boxes): with the defaults a long-running worker keeps one plan per batch size.  A request that fails
    validation gets its exception in `answers` and takes no row.  Returns a dict: answers, spans {request: (first row, end row)},
    n_tokens, n_boxes, question, segment_ids, task_tokens [B, 1], box_features, boxes, image_wh, select, max_tokens, max_boxes."""
    if bucket < 1:
        raise ValueError("bucket must be >= 1")
    max_rows = _max_rows()
    answers = [None] * len(requests)
    accepted, F = [], None                        # rows: (tokens, segments, task, box features [n, F], boxes [n, 4], (w, h))
    for i, (query, task, features, infos, task_id) in enumerate(requests):
        try:
            _validate(task_id, infos)
            if len(features) != len(infos):
                raise ValueError(f"{len(features)} feature arrays for {len(infos)} images")
            tokens, segs = _region_text(query, tok, max_rows)
            imgs = []
            for f, info in zip(features, infos):
                f = torch.as_tensor(f, dtype=torch.float32)
                n = int(f.shape[0]) if f.dim() == 2 else 0
                if n < 1 or n + 1 > max_rows or (F is not None and f.shape[1] != F):
                    raise ValueError(f"box features of shape {tuple(f.shape)}: need [n, F] with 1 <= n <= {max_rows - 1}"
                                     + (f" and F = {F}" if F is not None else ""))
                bx = torch.as_tensor(np.asarray(info["bbox"], dtype=np.float32))
                if bx.dim() != 2 or bx.shape[0] < n or bx.shape[1] < 4:
                    raise ValueError(f"bbox of shape {tuple(bx.shape)} for {n} boxes")
                imgs.append((f, bx[:n, :4], (float(info["image_width"]), float(info["image_height"]))))
            own = _region_rows(task_id, task, tokens, segs, imgs)
        except Exception as e:                      # noqa: BLE001 -- the request's answer, as callback()'s catch-all (worker.py:653-655)
            answers[i] = e
            continue
        F = int(imgs[0][0].shape[1])
        accepted.append((i, task_id, own))
    rows, spans, sel = _row_layout(accepted, bucket, select)
    filler = ([0], [0], 0, torch.zeros(1, F or 1), torch.zeros(1, 4), (1.0, 1.0))
    rows = [filler if r is None else r for r in rows]
    n_tokens = [len(r[0]) for r in rows]
    n_boxes = [int(r[3].shape[0]) for r in rows]
    return dict(answers=answers, spans=spans, n_tokens=n_tokens, n_boxes=n_boxes,
                question=torch.tensor([x for r in rows for x in r[0]], dtype=torch.long),
                segment_ids=torch.tensor([x for r in rows for x in r[1]], dtype=torch.long),
                task_tokens=torch.tensor([[r[2]] for r in rows], dtype=torch.long),
                box_features=torch.cat([r[3] for r in rows], dim=0) if rows else torch.zeros(0, 1),
                boxes=torch.cat([r[4] for r in rows], dim=0) if rows else torch.zeros(0, 4),
                image_wh=torch.tensor([list(r[5]) for r in rows], dtype=torch.float32).reshape(-1, 2),
                select=sel, max_tokens=max([MAX_LENGTH] + n_tokens), max_boxes=max([int(max_boxes)] + n_boxes))


def _answer_regions(answers, requests, out, spatials, spans, n_tokens, n_boxes, decode):
    """`_answer_spans` for a `forward_regions_packed` call on `custom_prediction` argument tuples."""
    return _answer_spans(answers, out, spatials, {i: (requests[i][4], requests[i][3]) for i in spans}, spans,
                         list(accumulate([n + 1 for n in n_boxes], initial=0)),     # each image: the global row, then the boxes
                         list(accumulate([n + 1 for n in n_tokens], initial=0)),    # each text: its tokens and the task token
                         decode)


def custom_prediction_packed(requests, bucket: int = 8, select: Optional[int] = None, max_boxes: int = 100, *, decode: str = "host"):
    """`custom_prediction` for many requests in ONE model call (`model.forward_regions_packed`): every question at its own length,
    every image at its own box count, no padding and no masks.  `requests` are argument tuples of `custom_prediction`:
    `(query, task, features, infos, task_id)`; the answers come back in the same order, a request that fails validation gets its
    exception.  The host packing is `pack_region_requests`.  Answers agree with `custom_prediction` within tolerance; they are not
    guaranteed bit for bit, because dropping the text padding may change the accumulation.  `decode` as for `prediction_batch`."""
    _check_decode(decode)
    p = pack_region_requests(requests, bucket, select, max_boxes)
    answers = p["answers"]
    if not p["spans"]:
        return answers
    with model_lock:
        out, spatials = model.forward_regions_packed(p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"],
                                                     p["image_wh"], p["n_tokens"], p["n_boxes"], select=p["select"],
                                                     max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
    return _answer_regions(answers, requests, out, spatials, p["spans"], p["n_tokens"], p["n_boxes"], decode)


def ablation_messages(requests, spans, tokens=None, boxes=None):
    """The `model.message_ablation` messages of packed region requests: request i, which took batch rows `spans[i] = (lo, hi)`,
    attributes its answer over images [lo, hi) -- one for VQA, GQA, SNLI-VE and grounding, the pair for NLVR2, every candidate for
    retrieval -- with its task id as the family.  Returns `{request: (task_id, lo, hi - lo, None, tokens, boxes)}`."""
    return {i: (requests[i][4], lo, hi - lo, None, tokens, boxes) for i, (lo, hi) in spans.items()}


def _pixel_box(info, row):
    """Row `row` of a grounding segment as a pixel box [x1, y1, x2, y2]: row 0 is the whole image, row r >= 1 box r - 1 of `info`."""
    if row == 0:
        return [0.0, 0.0, float(info["image_width"]), float(info["image_height"])]
    return [float(v) for v in np.asarray(info["bbox"], dtype=np.float32)[row - 1, :4]]


def _explain_packed(requests, max_boxes, messages, explain):
    """What the `custom_*_packed` explainers share: the requests packed by `pack_region_requests`, then under `model_lock` their
    answers (`custom_prediction_packed`, decode="device") and `explain(args, msgs, mask, kw)` on the same batch: `args` the
    batch's arguments of `model.forward_regions_packed`, `msgs` the list of `messages(spans)` ({request: message}), `mask` the
    tokenizer's [MASK] id and `kw` the plan capacities.  Returns (answers, the packed batch `p`, the message dict, explain's
    results); with no request that passes validation, or no message, nothing is explained."""
    p = pack_region_requests(requests, max_boxes=max_boxes)
    if not p["spans"]:
        return p["answers"], p, {}, []
    args = (p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"], p["image_wh"], p["n_tokens"], p["n_boxes"])
    msgs = messages(p["spans"])
    mask = (tokenizer.vocab.get("[MASK]", 103) if tokenizer is not None and hasattr(tokenizer, "vocab") else 103)
    kw = dict(max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
    with model_lock:
        out, spatials = model.forward_regions_packed(*args, select=p["select"], **kw)
        res = explain(args, list(msgs.values()), mask, kw) if msgs else []
    answers = _answer_regions(p["answers"], requests, out, spatials, p["spans"], p["n_tokens"], p["n_boxes"], "device")
    return answers, p, msgs, res


def custom_ablation_packed(requests, max_boxes: int = 100, *, tokens=None, boxes=None):
    """Why each answer: `custom_prediction_packed` (decode="device") for `custom_prediction` argument tuples
    `(query, task, features, infos, task_id)`, plus the answer's ablation over its question tokens and detector boxes
    (`model.message_ablation`) for every task: one image for VQA, GQA, SNLI-VE and grounding, the pair for NLVR2, every candidate for
    retrieval.  `tokens` / `boxes`: one (begin, end) range for every request, or None for the defaults (positions 1 .. Tin - 2, every
    box of an image with at least two).  The rows are those of `pack_region_requests`, unchanged.
    Returns per request `{"answer": <custom_prediction_packed's answer>, "ablation": <message_ablation's dict>}` -- whose `boxes` are
    `(image, box)` pairs, with `box_pixels` their [x1, y1, x2, y2] from `infos`, and for grounding `answer_box` the pixel box of the
    attributed row -- or the exception of a request that fails validation."""
    answers, _, msgs, ab = _explain_packed(requests, max_boxes, lambda spans: ablation_messages(requests, spans, tokens, boxes),
                                           lambda args, m, mask, kw: model.message_ablation(*args, m, mask_token=mask, **kw))
    for i, a in zip(msgs, ab):
        infos = requests[i][3]
        a["box_pixels"] = [_pixel_box(infos[img], b + 1) for img, b in a["boxes"]]
        if requests[i][4] in GROUNDING_TASKS:
            a["answer_box"] = _pixel_box(infos[0], a["answer"])
        answers[i] = {"answer": answers[i], "ablation": a}
    return answers


def custom_head_ablation_packed(requests, max_boxes: int = 100, *, entries=None):
    """Which attention heads each answer depends on: `custom_prediction_packed` (decode="device") for `custom_prediction` argument
    tuples `(query, task, features, infos, task_id)`, plus the answer's head ablation (`model.head_ablation`) over the images the
    answer reads, as `custom_ablation_packed` chooses them.  `entries`: one (begin, end) range of attention entries for every
    request, or None for all.  Returns per request `{"answer": <custom_prediction_packed's answer>, "ablation": <head_ablation's
    dict>}`, or the exception of a request that fails validation."""
    answers, _, msgs, ab = _explain_packed(
        requests, max_boxes, lambda spans: {i: m[:4] + (entries,) for i, m in ablation_messages(requests, spans).items()},
        lambda args, m, mask, kw: model.head_ablation(*args, m, **kw))
    for i, a in zip(msgs, ab):
        answers[i] = {"answer": answers[i], "ablation": a}
    return answers


def custom_shapley_packed(requests, max_boxes: int = 100, *, units=None, permutations: int = 8, seed: int = 0, antithetic: bool = True):
    """Shapley values of each answer's question tokens and detector boxes: `custom_prediction_packed` (decode="device") for
    `custom_prediction` argument tuples `(query, task, features, infos, task_id)`, plus `model.shapley` over the images the answer
    reads, as `custom_ablation_packed` chooses them.  `units`: None for the defaults (one unit per position 1 .. Tin - 2 and per box),
    or `(positions, boxes)` groups applied to every request.  Returns per request `{"answer": <custom_prediction_packed's answer>,
    "shapley": <shapley's dict>}` -- with `box_pixels`, per unit the [x1, y1, x2, y2] of its boxes from `infos` -- or the exception of
    a request that fails validation.  Grounding requests get a ValueError: their answer is a box, which a coalition would renumber."""
    return _coalition_packed(requests, max_boxes, "custom_shapley_packed", "shapley",
                             lambda args, m, mask, kw: model.shapley(*args, m, units=None if units is None else [units] * len(m),
                                                                     permutations=permutations, seed=seed, antithetic=antithetic,
                                                                     mask_token=mask, **kw))


def custom_interactions_packed(requests, max_boxes: int = 100, *, pairs="cross", units=None, permutations: int = 8, seed: int = 0,
                               antithetic: bool = True):
    """Which words work together with which boxes for each answer: `custom_prediction_packed` (decode="device") for
    `custom_prediction` argument tuples `(query, task, features, infos, task_id)`, plus `model.shapley_interactions` over the images
    the answer reads, as `custom_ablation_packed` chooses them.  `pairs`: "cross" (every word unit with every box unit) or a list of
    `(a, b)` unit indices, applied to every request; `units` as for `custom_shapley_packed`.  Returns per request
    `{"answer": <custom_prediction_packed's answer>, "interactions": <shapley_interactions' dict>}` -- with `box_pixels`, per unit
    the [x1, y1, x2, y2] of its boxes from `infos` -- or the exception of a request that fails validation.  Grounding requests get
    the ValueError `custom_shapley_packed` gives them."""
    return _coalition_packed(requests, max_boxes, "custom_interactions_packed", "interactions",
                             lambda args, m, mask, kw: model.shapley_interactions(
                                 *args, m, [pairs] * len(m), units=None if units is None else [units] * len(m),
                                 permutations=permutations, seed=seed, antithetic=antithetic, mask_token=mask, **kw))


def _coalition_packed(requests, max_boxes, name, key, explain):
    """What the coalition explainers share: `_explain_packed` with every request but grounding as a message, `explain(args, msgs,
    mask, kw)` the model call, and per answered request `{"answer": ..., key: <its dict with box_pixels per unit>}`."""
    answers, p, msgs, sh = _explain_packed(
        requests, max_boxes,
        lambda spans: {i: m[:4] for i, m in ablation_messages(requests, spans).items() if requests[i][4] not in GROUNDING_TASKS},
        explain)
    for i in p["spans"]:
        if i not in msgs:
            answers[i] = ValueError(f"{name}: a grounding answer is a box, which a coalition would renumber")
    for i, s in zip(msgs, sh):
        infos, lo = requests[i][3], p["spans"][i][0]
        first = list(accumulate([p["n_boxes"][lo + k] for k in range(len(infos))], initial=0))     # each image's first box

        def pixels(b):
            k = max(k for k in range(len(infos)) if first[k] <= b)
            return _pixel_box(infos[k], b - first[k] + 1)
        s["box_pixels"] = [[pixels(b) for b in bs] for _, bs in s["units"]]
        answers[i] = {"answer": answers[i], key: s}
    return answers


def _per_image(x, counts):
    """A per-image sequence as given, or one tensor over all images' rows split by `counts` (the reference's `.split`)."""
    if torch.is_tensor(x) or isinstance(x, np.ndarray):
        return list(torch.as_tensor(x).split(counts))
    return list(x)


def process_feature_extraction(proposals, scores, feats, im_scales, im_infos, conf_thresh=0, background=False, num_features=100):
    """The detector's feature extraction step (worker.py:123-176) on the device, one `model.select_regions` call for every image.

    `proposals` holds each image's boxes [n_i, 4] at the detector's input scale; `scores` ([n_i, C] logits, column 0 background)
    and `feats` ([n_i, F] fc6) are per-image sequences or, as the detector returns them, one tensor over all images' rows.
    `im_scales` / `im_infos` ({"width", "height"}) as the worker's image transform returns them.  Returns the reference's
    `(feat_list, info_list)`: feat_list[i] the k_i = min(num_features, n_i) kept feature rows (a device tensor), info_list[i] a dict
    of bbox (float32 [k_i, 4], original pixels), num_boxes (int), objects (int64 [k_i - start], the argmax of kept rows start..,
    start = 0 with `background` else 1), image_width, image_height and cls_prob (float32 [k_i, C])."""
    props = list(proposals)
    counts = [int(torch.as_tensor(p).shape[0]) for p in props]
    dets = list(zip(props, _per_image(scores, counts), _per_image(feats, counts), im_scales))
    start = 0 if background else 1
    with model_lock:
        r = model.select_regions(dets, num_features, float(conf_thresh), bool(background), cls_prob=True, objects=True)
    host = {k: r[k].cpu().numpy() for k in ("boxes", "num_boxes", "cls_prob", "objects")}
    feat_list, info_list = [], []
    for i, (lo, k) in enumerate(zip(r["dst_rows"], r["n_boxes"])):
        feat_list.append(r["box_features"][lo:lo + k])
        info_list.append({"bbox": host["boxes"][lo:lo + k], "num_boxes": int(host["num_boxes"][i]),
                          "objects": host["objects"][lo + start:lo + k], "image_width": im_infos[i]["width"],
                          "image_height": im_infos[i]["height"], "cls_prob": host["cls_prob"][lo:lo + k]})
    return feat_list, info_list


def custom_prediction_detections(requests, bucket: int = 8, select: Optional[int] = None, max_boxes: int = 100, *,
                                 decode: str = "host"):
    """`custom_prediction_packed` for requests that carry their images' raw detector heads instead of selected features: the
    region selection (`process_feature_extraction`'s, with the worker's defaults conf_thresh 0, no background class) writes
    straight into the packed box rows of ONE `forward_regions_packed` call, so no feature row passes through the host.

    `requests` are `(query, task, detections, infos, task_id)`: `detections[j]` = `(proposals [n, 4], scores [n, C], features
    [n, F], im_scale)` of image j (as `synthetic.synthetic_detections` returns them), `infos[j]` its dict with image_width /
    image_height.  Each image keeps k = min(max_boxes, n) boxes.  Rows, NLVR2 alignment, fillers (one token, one zero box in a 1 x 1
    image), capacities and `decode` follow `custom_prediction_packed`; the answers equal `custom_prediction_packed` on the features
    and boxes `process_feature_extraction` selects.  A request that fails validation gets its exception: every limit of
    `vb200_select_regions` on an image (1 <= n <= 2048 proposals, 2 <= C <= 2048 score columns, F the model's feature width, a
    positive finite im_scale, C the same as every other image of the call) is checked here, so one bad image does not fail the call."""
    if bucket < 1:
        raise ValueError("bucket must be >= 1")
    _check_decode(decode)
    max_rows = _max_rows()
    F = int(model._dims["v_feature_size"])
    answers = [None] * len(requests)
    accepted, CF = [], None                        # rows: (tokens, segments, task, detections, (w, h))
    for i, (query, task, detections, infos, task_id) in enumerate(requests):
        try:
            _validate(task_id, infos)
            if len(detections) != len(infos):
                raise ValueError(f"{len(detections)} detector outputs for {len(infos)} images")
            tokens, segs = _region_text(query, None, max_rows)
            imgs, cf = [], CF                       # cf: the (C, F) this request's images must share with the call
            for (prop, sc, ft, scale), info in zip(detections, infos):
                n = int(prop.shape[0])
                shape = (int(sc.shape[-1]), int(ft.shape[-1]))
                if not (1 <= n <= 2048 and 2 <= shape[0] <= 2048 and shape[1] == F
                        and tuple(prop.shape) == (n, 4) and tuple(sc.shape) == (n, shape[0]) and tuple(ft.shape) == (n, F)) \
                        or (cf is not None and shape != cf):
                    raise ValueError(f"detector output of shapes {tuple(prop.shape)}, {tuple(sc.shape)}, {tuple(ft.shape)}: need "
                                     f"[n, 4], [n, C], [n, F] with 1 <= n <= 2048, 2 <= C <= 2048 and F = {F} (the model's feature "
                                     "width)" + (f" and C = {cf[0]}" if cf else ""))
                if not 0.0 < float(scale) <= float(np.finfo(np.float32).max):
                    raise ValueError(f"im_scale {scale}: need a positive finite scale")
                cf = shape
                imgs.append(((prop, sc, ft, float(scale)), (float(info["image_width"]), float(info["image_height"]))))
            own = _region_rows(task_id, task, tokens, segs, imgs)
        except Exception as e:                      # noqa: BLE001 -- the request's answer, as callback()'s catch-all (worker.py:653-655)
            answers[i] = e
            continue
        CF = cf
        accepted.append((i, task_id, own))
    if not accepted:
        return answers
    rows, spans, sel = _row_layout(accepted, bucket, select)
    filler = ([0], [0], 0, None, (1.0, 1.0))
    rows = [filler if r is None else r for r in rows]
    n_tokens = [len(r[0]) for r in rows]
    n_boxes = [1 if r[3] is None else min(int(max_boxes), int(r[3][0].shape[0])) for r in rows]
    offs = np.concatenate([[0], np.cumsum(n_boxes)])
    # the engine needs a GPU; the CPU is only ever reached by a stand-in model when no GPU is visible (as in MicroBatchWorker._run)
    device = torch.device("cuda", model._device) if torch.cuda.is_available() else torch.device("cpu")
    box_features = torch.zeros(int(offs[-1]), CF[1], dtype=torch.float32, device=device)   # filler rows keep their zero box
    boxes = torch.zeros(int(offs[-1]), 4, dtype=torch.float32, device=device)
    real = [j for j, r in enumerate(rows) if r[3] is not None]
    question = torch.tensor([x for r in rows for x in r[0]], dtype=torch.long)
    segment_ids = torch.tensor([x for r in rows for x in r[1]], dtype=torch.long)
    task_tokens = torch.tensor([[r[2]] for r in rows], dtype=torch.long)
    image_wh = torch.tensor([list(r[4]) for r in rows], dtype=torch.float32).reshape(-1, 2)
    with model_lock:
        model.select_regions([rows[j][3] for j in real], int(max_boxes), dst_rows=[int(offs[j]) for j in real],
                             box_features=box_features, boxes=boxes)
        out, spatials = model.forward_regions_packed(question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens,
                                                     n_boxes, select=sel, max_tokens=max([MAX_LENGTH] + n_tokens),
                                                     max_boxes=max([int(max_boxes)] + n_boxes))
    return _answer_regions(answers, requests, out, spatials, spans, n_tokens, n_boxes, decode)


def shape_result(task_id: str, answer, image_path: Sequence[str], image_names: Optional[List[str]] = None):
    """The JSON-able `result` dict callback() pushes to the WebSocket, per task family (worker.py:564-645).
    Box drawing / file writing (cv2, worker.py:596-600) is left to the caller; pass the names it chose."""
    if task_id in ("1", "15", "2", "13"):
        return {"task_id": task_id, "result": [{"answer": answer["top3_answer"][i],
                                                "confidence": round(answer["top3_confidence"][i] * 100, 2)}
                                               for i in range(3)]}
    if task_id in ("4", "16", "11"):
        names = image_names if image_names is not None else [str(i) for i in range(len(answer))]
        return {"task_id": task_id, "image_name_list": names[:3],
                "confidence_list": [round(a["confidence"], 2) for a in answer[:3]]}
    if task_id == "12":
        return {"task_id": task_id, "result": [{"answer": answer["top3_answer"][i],
                                                "confidence": round(answer["top3_confidence"][i] * 100, 2)}
                                               for i in range(2)]}
    if task_id == "7":
        prefix = "demo/" if "demo" in image_path[0].split("/") else "test2014/"
        ext = str(image_path[0].split("/")[-1].split(".")[1])
        names = [prefix + os.path.split(image_path[i])[1].split(".")[0] + "." + ext for i in answer["top3_answer"]]
        return {"task_id": task_id, "image_name_list": names,
                "confidence_list": [round(c * 100, 2) for c in answer["top3_confidence"]]}
    raise ValueError("task not valid.")


def handle_request(body: dict, features, infos):
    """callback() minus transport (worker.py:556-563): body = {image_path, question, socket_id, task_id}."""
    task_id = str(body["task_id"])
    answer = custom_prediction(body["question"], [int(task_id)], features, infos, task_id)
    return shape_result(task_id, answer, body["image_path"])


# ------------------------------------------------------------------------------------------ tokenizer
class MicroBatchWorker(object):
    """Dependency-light stand-in for the reference's consumer loop (`callback` / `main`, worker.py:542-673) with micro-batching.

    `submit(body, features, infos)` takes the JSON message of demo/sender.py:19-24 (`image_path, question, socket_id, task_id`)
    plus the detector output for its images (the detector itself, worker.py:59-223, is out of scope) and returns a
    `concurrent.futures.Future` whose result is `{"socket_id": ..., "result": <the dict callback() pushes to the WebSocket,
    worker.py:564-649>}`.  A background thread drains the queue: it waits at most `max_wait_ms` after the first pending message
    for up to `max_rows` image rows, runs them through `prediction_batch` (one model call per shape group) and resolves the
    futures; a failing request resolves to its exception, like the try/except of callback (worker.py:653-655).

    `packed=True` hands the raw detector output of the pending messages to `custom_prediction_packed` instead: ONE model call
    whatever their text lengths and box counts (images of one message may have different box counts too), with no host-side
    feature construction.  Answers agree with the dense path within tolerance; they are not guaranteed bit for bit, because dropping
    the text padding may change the accumulation.  The default stays dense; making packed the default and deleting the dense
    branch is a follow-up, to be decided on the A/B of scripts/regions_packed_bench.py.

    `decode="device"` decodes every answer of a model call in one kernel (`model.decode_answers`) instead of one softmax, top-N
    and host synchronisation per message; the default stays on the host.

    `source="detections"` serves messages that carry the detector network's raw heads instead of selected features:
    `submit(body, detections, infos)` takes per image `(proposals [n, 4], scores [n, C], features [n, F], im_scale)` (the layout of
    `synthetic.synthetic_detections`) and `infos[j]` with image_width / image_height.  Each micro-batch goes through
    `custom_prediction_detections`: ONE region selection (the top `max_boxes` boxes per image, the detector's num_features) straight
    into the packed rows of ONE `forward_regions_packed`, and with `decode="device"` one decode.  `packed` only applies to
    `source="features"`.  Heads may be device tensors on any GPU: for each GPU that holds some, `submit` records an event on the
    submitting thread's current stream there and the worker's stream there waits for it before the selection, so heads written on
    any stream need no synchronisation, and the worker keeps them alive until its reads are done, so the caller may drop its
    references right after `submit`.  A message whose heads
    break a limit of the selection resolves to its own `ValueError`; the rest of its micro-batch is answered.  The default source
    stays "features"; changing it, like the dense default, waits for an A/B (scripts/worker_detections_bench.py)."""

    def __init__(self, max_rows: int = 64, max_wait_ms: float = 2.0, bucket: int = 8, packed: bool = False, *, decode: str = "host",
                 source: str = "features", max_boxes: int = 100):
        import queue
        import threading
        _check_decode(decode)
        if source not in ("features", "detections"):
            raise ValueError(f"source must be 'features' or 'detections', not {source!r}")
        if not 1 <= int(max_boxes) <= _max_rows() - 1:
            raise ValueError(f"max_boxes = {max_boxes} outside [1, {_max_rows() - 1}]")
        self.max_rows, self.max_wait, self.bucket = int(max_rows), float(max_wait_ms) * 1e-3, int(bucket)
        self.packed = bool(packed)
        self.decode = decode
        self.source, self.max_boxes = source, int(max_boxes)
        self._q = queue.Queue()
        self._stop = False
        self.batches = []                      # rows per model call group, for tests / monitoring
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()

    def submit(self, body: dict, features, infos):
        """Queue one message; `features` are the selected box features per image, or with `source="detections"` the raw heads."""
        from concurrent.futures import CancelledError, Future
        fut = Future()
        if self._stop:
            fut.set_exception(CancelledError("MicroBatchWorker closed"))
            return fut
        ready = []                             # per GPU: (event, heads) the worker's stream there waits for and keeps alive
        if self.source == "detections":
            by_device = {}
            for det in features:
                for t in (det[:3] if isinstance(det, (tuple, list)) else ()):
                    if torch.is_tensor(t) and t.is_cuda:
                        by_device.setdefault(t.device, []).append(t)
            for dev, heads in by_device.items():
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(dev))
                ready.append((ev, heads))
        self._q.put((body, features, infos, fut, ready))
        return fut

    def close(self):
        """Stop the consumer thread.  Messages still queued (behind the sentinel, or submitted after close) are cancelled:
        their futures raise `concurrent.futures.CancelledError` instead of blocking their callers for ever."""
        import queue
        from concurrent.futures import CancelledError
        self._stop = True
        self._q.put(None)
        self._thread.join(timeout=30.0)
        while True:
            try:
                item = self._q.get_nowait()
            except queue.Empty:
                break
            if item is not None and not item[3].done():
                item[3].set_exception(CancelledError("MicroBatchWorker closed"))

    def _loop(self):
        import queue
        import time
        while not self._stop:
            item = self._q.get()
            if item is None:
                break
            pending, rows = [item], len(item[2])
            deadline = time.monotonic() + self.max_wait
            while rows < self.max_rows:
                left = deadline - time.monotonic()
                if left <= 0:
                    break
                try:
                    nxt = self._q.get(timeout=left)
                except queue.Empty:
                    break
                if nxt is None:
                    self._stop = True
                    break
                pending.append(nxt)
                rows += len(nxt[2])
            self._run(pending)

    def _run(self, pending):
        if self.source == "detections":
            return self._run_detections(pending)
        if self.packed:
            return self._run_packed(pending, custom_prediction_packed)
        device = torch.device("cuda", model._device) if torch.cuda.is_available() else torch.device("cpu")
        reqs, live = [], []
        for body, features, infos, fut, _ in pending:
            try:
                task_id = str(body["task_id"])
                reqs.append(build_inputs(body["question"], [int(task_id)], features, infos, device) + (task_id, infos))
                live.append((body, fut, task_id))
            except Exception as e:             # noqa: BLE001 -- mirrors callback()'s catch-all (worker.py:653-655)
                fut.set_exception(e)
        if not reqs:
            return
        try:
            answers = prediction_batch(reqs, bucket=self.bucket, decode=self.decode)
        except Exception as e:                 # noqa: BLE001
            for _, fut, _ in live:
                fut.set_exception(e)
            return
        self.batches.append(sum(r[1].shape[0] for r in reqs))
        self._resolve(live, answers)

    def _run_detections(self, pending):
        """Order this thread's stream on each GPU that holds heads after the message's event there (the selection reads heads on
        the model's GPU in place, and copies heads on another GPU on this thread's stream of that GPU), keep the heads alive until
        the work enqueued on them is done (`record_stream`: the allocator does not reuse their memory before that, even when the
        call raises after enqueuing), then answer the micro-batch."""
        for *_, ready in pending:
            for ev, heads in ready:
                stream = torch.cuda.current_stream(heads[0].device)
                stream.wait_event(ev)
                for t in heads:
                    t.record_stream(stream)
        self._run_packed(pending, functools.partial(custom_prediction_detections, max_boxes=self.max_boxes))

    def _run_packed(self, pending, predict):
        reqs, live = [], []
        for body, features, infos, fut, _ in pending:
            try:
                task_id = str(body["task_id"])
                reqs.append((body["question"], [int(task_id)], features, infos, task_id))
                live.append((body, fut, task_id))
            except Exception as e:             # noqa: BLE001
                fut.set_exception(e)
        if not reqs:
            return
        try:
            answers = predict(reqs, bucket=self.bucket, decode=self.decode)
        except Exception as e:                 # noqa: BLE001
            for _, fut, _ in live:
                fut.set_exception(e)
            return
        self.batches.append(sum(len(r[3]) for r, a in zip(reqs, answers) if not isinstance(a, Exception)))
        self._resolve(live, answers)

    def _resolve(self, live, answers):
        for (body, fut, task_id), ans in zip(live, answers):
            if isinstance(ans, Exception):
                fut.set_exception(ans)
            else:
                try:
                    fut.set_result({"socket_id": body.get("socket_id"), "result": shape_result(task_id, ans, body["image_path"])})
                except Exception as e:         # noqa: BLE001
                    fut.set_exception(e)


class WordpieceTokenizer(object):
    """bert-base-uncased style tokenizer (lower-case, accent strip, punctuation split, greedy WordPiece) with the two
    methods the worker calls (worker.py:402-403).  Needs the user's vocab.txt: none ships with the reference."""

    def __init__(self, vocab, do_lower_case: bool = True, unk_token="[UNK]", cls_token="[CLS]", sep_token="[SEP]"):
        if isinstance(vocab, (str, os.PathLike)):
            with open(vocab, "r", encoding="utf-8") as f:
                vocab = {line.rstrip("\n"): i for i, line in enumerate(f)}
        self.vocab = dict(vocab)
        self.lower = do_lower_case
        self.unk, self.cls, self.sep = unk_token, cls_token, sep_token

    @staticmethod
    def _is_punct(ch):
        cp = ord(ch)
        if 33 <= cp <= 47 or 58 <= cp <= 64 or 91 <= cp <= 96 or 123 <= cp <= 126:
            return True
        return unicodedata.category(ch).startswith("P")

    def _basic(self, text):
        if self.lower:
            text = unicodedata.normalize("NFD", text.lower())
            text = "".join(c for c in text if unicodedata.category(c) != "Mn")
        out = []
        for word in text.split():
            cur = ""
            for ch in word:
                if self._is_punct(ch):
                    if cur:
                        out.append(cur)
                    out.append(ch)
                    cur = ""
                else:
                    cur += ch
            if cur:
                out.append(cur)
        return out

    def tokenize(self, text):
        pieces = []
        for word in self._basic(text):
            if len(word) > 100:
                pieces.append(self.unk)
                continue
            start, sub = 0, []
            while start < len(word):
                end, cur = len(word), None
                while start < end:
                    s = word[start:end] if start == 0 else "##" + word[start:end]
                    if s in self.vocab:
                        cur = s
                        break
                    end -= 1
                if cur is None:
                    sub = [self.unk]
                    break
                sub.append(cur)
                start = end
            pieces.extend(sub)
        return pieces

    def encode(self, text):
        return [self.vocab.get(t, self.vocab.get(self.unk, 0)) for t in self.tokenize(text)]

    def add_special_tokens_single_sentence(self, ids):
        return [self.vocab[self.cls]] + list(ids) + [self.vocab[self.sep]]
