"""VILBertForVLTasks: the object protocol of the reference worker on top of the C ABI.

    config = BertConfig.from_json_file(path)                                   worker.py:495, 506
    model  = VILBertForVLTasks.from_pretrained(ckpt, config=config,
                                               num_labels=3129, default_gpu=True)   worker.py:530-532
    model.eval(); model.cuda(0)                                                worker.py:534-536
    out10  = model(question, features, spatials, segment_ids, input_mask, image_mask,
                   co_attention_mask, task_tokens, output_all_attention_masks=True)  worker.py:286-289

Everything between the input tensors and the ten outputs runs in libvilbert_b200.so (hand-written sm_90a
kernels).  torch is used only as the tensor container and for the CUDA stream.  No CPU path exists: calling
the model without an H100 raises.
"""
from __future__ import annotations

import ctypes as C
import json
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from .config import BertConfig

_DTYPES = {torch.float32: L.F32, torch.float16: L.F16, torch.bfloat16: L.BF16}


def _normalise_state_dict(sd) -> Dict[str, torch.Tensor]:
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    if isinstance(sd, dict) and "model_state_dict" in sd and isinstance(sd["model_state_dict"], dict):
        sd = sd["model_state_dict"]
    out = {}
    for k, v in sd.items():
        if not torch.is_tensor(v):
            continue
        if v.dtype in (torch.int64, torch.int32, torch.bool) or v.dim() == 0 or v.dim() > 2:
            continue                      # e.g. position_ids buffers, num_batches_tracked
        if v.dtype not in _DTYPES:
            v = v.float()
        out[k] = v.detach().cpu().contiguous()
    return out


def _host_ints(x):
    return [int(v) for v in (x.tolist() if torch.is_tensor(x) else x)]


def _int32s(values):
    """Host ints as the ``int32_t*`` of a C ABI length array (the array lives as long as the returned pointer)."""
    return C.cast((C.c_int32 * max(len(values), 1))(*values), C.c_void_p)


def _to_device(t, dtype, device):
    """``t`` as a contiguous ``dtype`` tensor on ``device``; a tensor that already is one is passed through without a copy."""
    if not torch.is_tensor(t):
        t = torch.as_tensor(t)
    if t.dtype != dtype:
        t = t.to(dtype)
    if t.device != device:
        t = t.to(device, non_blocking=True)
    return t.contiguous()


def _task_rows(task_tokens, n, device):
    """The task token of each of n samples as [n, 1] int64 on ``device`` (the first entry of each sample's row)."""
    return _to_device(task_tokens, torch.int64, device).reshape(n, -1)[:, :1].contiguous()


def head_mask_shape(config):
    """``(n_entries, max_heads)`` of a head mask (vb200_model_dim "head_mask_entries" / "head_mask_heads"): one entry per text
    and image layer and two per connection layer (text-query, then image-query direction) in execution order, each with a slot
    for every head of the configuration's widest attention."""
    entries = config.num_hidden_layers + config.v_num_hidden_layers + 2 * len(config.v_biattention_id)
    return entries, max(config.num_attention_heads, config.v_num_attention_heads, config.bi_num_attention_heads)


def head_mask_rows(head_mask, batch: int, shape, device):
    """A packed forward's ``head_mask`` as the engine's contiguous fp32 ``[batch, n_entries, max_heads]`` on ``device``:
    ``[n_entries, max_heads]`` applies to every sample, ``[batch, n_entries, max_heads]`` gives each sample its own."""
    m = head_mask if torch.is_tensor(head_mask) else torch.as_tensor(head_mask)
    if tuple(m.shape) == tuple(shape):
        m = m.unsqueeze(0).expand(batch, *shape)
    elif tuple(m.shape) != (batch, *shape):
        raise ValueError(f"head_mask has shape {tuple(m.shape)}: expected {tuple(shape)} (every sample) or "
                         f"{(batch, *shape)} (per sample)")
    return _to_device(m, torch.float32, device)


def packed_offsets(lengths, extra: int = 0):
    """Row offsets [n + 1] of n items stored back to back with lengths[i] + extra rows each (extra = 1: the task-token row of
    a caption state)."""
    offs = [0]
    for n in lengths:
        offs.append(offs[-1] + int(n) + extra)
    return offs


class PackedRegionBatch:
    """A packed detector-output batch, ``forward_regions_packed``'s inputs, checked and staged on the engine's ``device`` once.
    ``name`` (the calling method) starts every error message.  ``inputs`` is the batch's vb200_packed_region_inputs, valid while the
    batch lives; ``subset`` the batch of some of its samples, their rows packed back to back."""

    @staticmethod
    def lengths(name, n_tokens, n_boxes):
        """``n_tokens`` / ``n_boxes`` as host int lists of the same, positive length."""
        nt, nb = _host_ints(n_tokens), _host_ints(n_boxes)
        if len(nb) != len(nt) or not nt:
            raise ValueError(f"{name}: n_tokens and n_boxes must have the same, positive length")
        return nt, nb

    def __init__(self, name, device, feature_size, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes):
        nt, nb = self.lengths(name, n_tokens, n_boxes)
        B = len(nt)
        q = _to_device(question, torch.int64, device).reshape(-1)
        seg = _to_device(segment_ids if segment_ids is not None else torch.zeros_like(q), torch.int64, device).reshape(-1)
        tk = _task_rows(task_tokens if task_tokens is not None else torch.zeros(B, 1, dtype=torch.int64), B, device)
        bf = _to_device(box_features, torch.float32, device).reshape(-1, feature_size)
        bx = _to_device(boxes, torch.float32, device).reshape(-1, 4)
        wh = _to_device(image_wh, torch.float32, device)
        if q.numel() != sum(nt) or seg.numel() != sum(nt) or bf.shape[0] != sum(nb) or bx.shape[0] != sum(nb) or tuple(wh.shape) != (B, 2):
            raise ValueError(f"{name}: question / segment_ids need sum(n_tokens) entries, box_features / boxes sum(n_boxes) rows, "
                             "image_wh [B, 2]")
        self.name, self.device, self.feature_size = name, device, feature_size
        self.nt, self.nb, self.tensors = nt, nb, (q, seg, tk, bf, bx, wh)

    def subset(self, samples):
        t_off, b_off = packed_offsets(self.nt), packed_offsets(self.nb)
        tcat = lambda t: torch.cat([t[t_off[i]:t_off[i + 1]] for i in samples])
        bcat = lambda t: torch.cat([t[b_off[i]:b_off[i + 1]] for i in samples])
        q, seg, tk, bf, bx, wh = self.tensors
        return PackedRegionBatch(self.name, self.device, self.feature_size, tcat(q), tcat(seg), tk[samples], bcat(bf), bcat(bx),
                                 wh[samples], [self.nt[i] for i in samples], [self.nb[i] for i in samples])

    def inputs(self, max_tokens: int = 0, max_boxes: int = 0, spatials=None):
        return L.PackedRegionInputs(len(self.nt), int(max_tokens), int(max_boxes), _int32s(self.nt), _int32s(self.nb),
                                    *[t.data_ptr() for t in self.tensors], spatials)


def _structs(cls, rows):
    """A ctypes array of ``cls``, one per tuple of field values in ``rows``."""
    return (cls * len(rows))(*[cls(*r) for r in rows])


# the families whose answer is one row of one image (vb200_answer_ablation)
ABLATION_FAMILIES = {"vqa": L.DECODE_VQA, "gqa": L.DECODE_GQA, "snli_ve": L.DECODE_SNLI_VE}


def ablation_ranges(n_tokens, n_boxes, tokens=None, boxes_range=None):
    """Each sample's (token_begin, token_end, box_begin, box_end) for answer ablation.  By default the question positions
    1 .. Tin - 2 are masked (the [CLS] and [SEP] kept) and every box of an image with at least two boxes is dropped.  ``tokens`` /
    ``boxes_range``: None (the default), one (begin, end) pair for every sample, or a list of one pair or None per sample."""
    n = len(n_tokens)

    def per_sample(r, name):
        if r is None:
            return [None] * n
        if len(r) == 2 and all(isinstance(x, int) for x in r):
            return [tuple(r)] * n
        if len(r) != n:
            raise ValueError(f"answer_ablation: {name} needs one (begin, end) pair, or one per sample ({n}), got {len(r)} entries")
        return [None if x is None else tuple(x) for x in r]

    tk, bx = per_sample(tokens, "tokens"), per_sample(boxes_range, "boxes_range")
    out = []
    for i, (tin, nb) in enumerate(zip(n_tokens, n_boxes)):
        tb, te = tk[i] if tk[i] is not None else (1, max(1, tin - 1))
        bb, be = bx[i] if bx[i] is not None else (0, nb if nb >= 2 else 0)
        if not 0 <= tb <= te <= tin:
            raise ValueError(f"answer_ablation: sample {i} has the token range [{tb}, {te}), reversed or outside [0, {tin}]")
        if not 0 <= bb <= be <= nb:
            raise ValueError(f"answer_ablation: sample {i} has the box range [{bb}, {be}), reversed or outside [0, {nb}]")
        if be > bb and nb < 2:
            raise ValueError(f"answer_ablation: sample {i} drops a box of an image with {nb} box (box ablation needs >= 2)")
        out.append((int(tb), int(te), int(bb), int(be)))
    return out


def ablation_calls(ranges, cap: int = L.ABLATION_MAX_VARIANTS):
    """The engine calls for these per-sample ranges: each call a list of (sample, (token_begin, token_end, box_begin, box_end))
    pieces whose variants (1 + tokens + boxes each) number at most ``cap``.  A batch is split at sample boundaries; a sample with more
    than ``cap`` variants is split into pieces of its units (tokens first, then boxes), each with its own unablated variant."""
    return message_calls([r for i, (tb, te, bb, be) in enumerate(ranges)
                          for r in [(i, 0, -1, 1)] + [(i, 1, p, 1) for p in range(tb, te)] + [(i, 2, j, 1) for j in range(bb, be)]], cap)


def ablation_variants(call):
    """The variants of one engine call in the engine's order: (sample, kind, unit) with kind "base" (unit None), "token" (the masked
    position) or "box" (the dropped box)."""
    out = []
    for i, (tb, te, bb, be) in call:
        out.append((i, "base", None))
        out += [(i, "token", p) for p in range(tb, te)]
        out += [(i, "box", j) for j in range(bb, be)]
    return out


# every decode family by name (vb200_message_ablation); a worker task id (_lib.TASK_DECODE_FAMILY) or a DECODE_* value works too
MESSAGE_FAMILIES = {"vqa": L.DECODE_VQA, "gqa": L.DECODE_GQA, "nlvr2": L.DECODE_NLVR2, "snli_ve": L.DECODE_SNLI_VE,
                    "retrieval": L.DECODE_RETRIEVAL, "grounding": L.DECODE_GROUNDING}
_FAMILY_IMAGES = {L.DECODE_VQA: 1, L.DECODE_GQA: 1, L.DECODE_NLVR2: 2, L.DECODE_SNLI_VE: 1, L.DECODE_GROUNDING: 1}


def message_family(family):
    """A decode family from its name, a worker task id or its ``_lib.DECODE_*`` value."""
    if isinstance(family, str):
        f = MESSAGE_FAMILIES.get(family, L.TASK_DECODE_FAMILY.get(family))
    else:
        f = int(family)
    if f not in MESSAGE_FAMILIES.values():
        raise ValueError(f"message_ablation: unknown family {family!r} (one of {sorted(MESSAGE_FAMILIES)}, a task id or a DECODE_* value)")
    return f


def _message_head(name, i, family, image_begin, n_images, answer, batch: int, top1: str = "the unablated top-1"):
    """``(family, image_begin, n_images, answer)`` of message i of an ablation call checked against a batch of ``batch`` images:
    the family by name, task id or value; the images it reads (``n_images`` right for the family, all inside the batch); the
    answer an index >= 0, or None / -1 (``top1``).  ``name`` starts every error message."""
    f = message_family(family)
    ib, k = int(image_begin), int(n_images)
    want = _FAMILY_IMAGES.get(f)
    if (k != want) if want else k < 1:
        raise ValueError(f"{name}: message {i} has n_images {k} (the family reads {want or '>= 1'})")
    if ib < 0 or ib + k > batch:
        raise ValueError(f"{name}: message {i} has images [{ib}, {ib + k}) outside the batch of {batch}")
    a = -1 if answer is None else int(answer)
    if a < -1:
        raise ValueError(f"{name}: message {i} has answer {a} (an index >= 0, or None / -1: {top1})")
    return f, ib, k, a


def message_pieces(messages, n_tokens, n_boxes):
    """The engine messages (``_lib.AblationMessage`` fields as tuples) for ``message_ablation``'s ``messages`` and the batch's
    lengths, and for each the index of the message it belongs to.  A message is ``(family, image_begin, n_images, answer=None,
    tokens=None, boxes=None)``; by default positions 1 .. Tin - 2 of image_begin's question are masked and every box of the
    message's images with at least two boxes is dropped (boxes numbered across the message's images).  The default boxes of a
    message with a one-box image between others run as separate pieces, each with its own unablated variant."""
    out = []
    for i, m in enumerate(messages):
        m = tuple(m) + (None,) * (6 - len(m))
        if len(m) != 6:
            raise ValueError(f"message_ablation: message {i} has {len(m)} fields (family, image_begin, n_images, answer, tokens, boxes)")
        f, ib, k, a = _message_head("message_ablation", i, *m[:4], len(n_tokens))
        tokens, boxes = m[4:]
        tin, nb = int(n_tokens[ib]), [int(n) for n in n_boxes[ib:ib + k]]
        first = [sum(nb[:j]) for j in range(k + 1)]            # each image's first box in the message's numbering
        tb, te = (1, max(1, tin - 1)) if tokens is None else (int(tokens[0]), int(tokens[1]))
        if not 0 <= tb <= te <= tin:
            raise ValueError(f"message_ablation: message {i} has the token range [{tb}, {te}), reversed or outside [0, {tin}]")
        if boxes is None:                                      # runs of adjacent images with >= 2 boxes
            runs = []
            for j in range(k):
                if nb[j] < 2:
                    continue
                if runs and runs[-1][1] == first[j]:
                    runs[-1] = (runs[-1][0], first[j + 1])
                else:
                    runs.append((first[j], first[j + 1]))
        else:
            bb, be = int(boxes[0]), int(boxes[1])
            if not 0 <= bb <= be <= first[k]:
                raise ValueError(f"message_ablation: message {i} has the box range [{bb}, {be}), reversed or outside [0, {first[k]}]")
            for j in range(k):
                if nb[j] < 2 and bb < first[j + 1] and be > first[j]:
                    raise ValueError(f"message_ablation: message {i} drops a box of its image {j}, which has {nb[j]} box")
            runs = [(bb, be)] if be > bb else []
        runs = runs or [(0, 0)]
        out.append(((f, ib, k, a, tb, te) + runs[0], i))
        out += [((f, ib, k, a, 0, 0) + r, i) for r in runs[1:]]
    return out


def _span(units):
    """``(first, last + 1)`` of consecutive units, ``(0, 0)`` for none."""
    return (units[0], units[-1] + 1) if units else (0, 0)


def _layout_calls(variants, cap, name, per):
    """The engine calls of an ablation layout, split greedily: ``variants`` are its records ``(message, kind, unit, samples)`` in
    layout order, each message's first (kind 0) its unablated variant.  Consecutive records of one ``(kind, unit)`` are one atom,
    which stays in one call.  Each message is cut into pieces of consecutive atoms of at most ``cap`` forward samples, each piece
    with the message's unablated variant, and the pieces are packed into calls in order.  Each call is a list of pieces
    ``(message, atoms)``, an atom ``[kind, unit, samples]``; ``name`` and ``per`` word the error of a message that cannot fit."""
    groups, last = [], None
    for m, kind, unit, samples in variants:
        if kind == 0:
            groups.append((m, samples, atoms := []))
            last = None
        elif last is not None and last[1] == unit and last[0] == kind:
            last[2] += samples
        else:
            atoms.append(last := [kind, unit, samples])
    pieces = []
    for m, base, atoms in groups:
        if base + max([a[2] for a in atoms], default=0) > cap:
            raise ValueError(f"{name}: message {m} runs {base} samples per {per}, too many for {cap} per call")
        chunk, size = [], base
        for a in atoms:
            n = a[2]
            if size + n > cap:
                pieces.append((m, chunk, size))
                chunk, size = [], base
            chunk.append(a)
            size += n
        pieces.append((m, chunk, size))
    calls, size = [], cap + 1
    for m, chunk, n in pieces:
        if size + n > cap:
            calls.append([])
            size = 0
        calls[-1].append((m, chunk))
        size += n
    return calls


def message_calls(variants, cap: int = L.ABLATION_MAX_VARIANTS):
    """The engine calls for a message ablation layout: ``variants`` are its records ``(message, kind, unit, samples)`` in layout order
    (``vb200_message_ablation_layout``).  Each call is a list of pieces ``(message, (token_begin, token_end, box_begin, box_end))``
    whose variants run at most ``cap`` forward samples.  Messages are kept whole where they fit; a message above ``cap`` is split
    into pieces of its units (positions first, then boxes), each with its own unablated variant."""
    calls = _layout_calls(variants, cap, "message_ablation", "unablated variant")
    return [[(m, _span([u for k, u, _ in a if k == 1]) + _span([u for k, u, _ in a if k == 2])) for m, a in call] for call in calls]


def head_messages(messages, batch: int, n_entries: int):
    """The engine messages (``_lib.HeadAblationMessage`` fields as tuples) for ``head_ablation``'s ``messages``: each is
    ``(family, image_begin, n_images, answer=None, entries=None)``, entries a ``(begin, end)`` range of the head mask's entry
    order (None: every entry)."""
    out = []
    for i, m in enumerate(messages):
        m = tuple(m)
        if not 3 <= len(m) <= 5:
            raise ValueError(f"head_ablation: message {i} has {len(m)} fields (family, image_begin, n_images, answer, entries)")
        m += (None,) * (5 - len(m))
        f, ib, k, a = _message_head("head_ablation", i, *m[:4], batch)
        entries = m[4]
        eb, ee = (0, n_entries) if entries is None else (int(entries[0]), int(entries[1]))
        if not 0 <= eb <= ee <= n_entries:
            raise ValueError(f"head_ablation: message {i} has the entry range [{eb}, {ee}), reversed or outside [0, {n_entries}]")
        out.append((f, ib, k, a, eb, ee))
    return out


def head_calls(variants, max_heads: int, cap: int = L.ABLATION_MAX_VARIANTS):
    """The engine calls for a head ablation layout: ``variants`` are its records ``(message, kind, unit, samples)`` in layout order
    (``vb200_head_ablation_layout``).  Each call is a list of pieces ``(message, (entry_begin, entry_end))`` whose variants run at
    most ``cap`` forward samples.  Messages are kept whole where they fit; a message above ``cap`` is split at entry boundaries, each
    piece with its own unablated variant."""
    calls = _layout_calls([(m, kind, unit // max_heads, n) for m, kind, unit, n in variants], cap, "head_ablation", "variant")
    return [[(m, _span([e for _, e, _ in a])) for m, a in call] for call in calls]


# the families a coalition can attribute (grounding's answer is a box, which a coalition would renumber)
COALITION_FAMILIES = {L.DECODE_VQA, L.DECODE_GQA, L.DECODE_NLVR2, L.DECODE_SNLI_VE, L.DECODE_RETRIEVAL}


def coalition_messages(messages, batch: int):
    """The engine messages ``(family, image_begin, n_images, answer)`` for ``coalition_ablation`` / ``shapley``'s ``messages``:
    each is ``(family or task id, image_begin, n_images, answer=None)``, any decode family except grounding."""
    out = []
    for i, m in enumerate(messages):
        m = tuple(m)
        if not 3 <= len(m) <= 4:
            raise ValueError(f"coalition_ablation: message {i} has {len(m)} fields (family, image_begin, n_images, answer)")
        if message_family(m[0]) not in COALITION_FAMILIES:
            raise ValueError(f"coalition_ablation: message {i} is a grounding message (its answer is a box, which a coalition would "
                             "renumber)")
        out.append(_message_head("coalition_ablation", i, *m + (None,) * (4 - len(m)), batch, "the full input's top-1"))
    return out


def coalition_units(units, tin: int, boxes: int, i: int = 0):
    """One message's units as ``(positions, boxes)`` tuples of ints.  ``units`` None: one unit per question position 1 .. Tin - 2 and
    one per box of the message's ``boxes`` (numbered across its images); else a list of ``(positions, boxes)`` groups, e.g. the word
    pieces of one word or the boxes of one class.  Each unit non-empty, no position or box in two units, at most
    ``_lib.COALITION_MAX_UNITS`` units."""
    if units is None:
        out = [((p,), ()) for p in range(1, max(1, tin - 1))] + [((), (b,)) for b in range(boxes)]
    else:
        out = []
        for u, g in enumerate(units):
            if len(g) != 2:
                raise ValueError(f"coalition_ablation: message {i} unit {u} needs (positions, boxes), got {g!r}")
            out.append((tuple(int(x) for x in g[0]), tuple(int(x) for x in g[1])))
    if not 1 <= len(out) <= L.COALITION_MAX_UNITS:
        raise ValueError(f"coalition_ablation: message {i} has {len(out)} units (1 .. {L.COALITION_MAX_UNITS})")
    seen_p, seen_b = {}, {}
    for u, (ps, bs) in enumerate(out):
        if not ps and not bs:
            raise ValueError(f"coalition_ablation: message {i} unit {u} is empty (no position and no box)")
        for x, lim, seen, what in [(p, tin, seen_p, "position") for p in ps] + [(b, boxes, seen_b, "box") for b in bs]:
            if not 0 <= x < lim:
                raise ValueError(f"coalition_ablation: message {i} unit {u} has {what} {x} outside [0, {lim})")
            if x in seen:
                raise ValueError(f"coalition_ablation: message {i} unit {u} has {what} {x}, which unit {seen[x]} already holds")
            seen[x] = u
    return out


def coalition_bitmaps(present, n_units: int):
    """Presence bitmaps of coalitions: ``present`` is a bool / 0-1 array [n_coalitions, n_units] (True: the unit is present).
    Returns a uint64 numpy array [n_coalitions, ceil(n_units / 64)], bit u % 64 of word u // 64 for unit u."""
    a = np.asarray(present, dtype=bool)
    if a.ndim != 2 or a.shape[1] != n_units:
        raise ValueError(f"coalition_ablation: coalitions need shape [n_coalitions, {n_units}], got {tuple(a.shape)}")
    W = (n_units + 63) // 64
    padded = np.zeros((a.shape[0], W * 64), dtype=np.uint64)
    padded[:, :n_units] = a
    weights = np.left_shift(np.uint64(1), np.arange(64, dtype=np.uint64))
    return (padded.reshape(-1, W, 64) * weights).sum(axis=2, dtype=np.uint64)


def coalition_calls(variants, cap: int = L.ABLATION_MAX_VARIANTS):
    """The engine calls for a coalition ablation layout: ``variants`` are its records ``(message, kind, unit, samples)`` in layout
    order (``vb200_coalition_ablation_layout``).  Each call is a list of pieces ``(message, (coalition_begin, coalition_end))``
    whose variants run at most ``cap`` forward samples; a message above that is split into runs of its coalitions, each piece with
    its own full-input variant."""
    calls = _layout_calls(variants, cap, "coalition_ablation", "variant")
    return [[(m, _span([c for _, c, _ in a])) for m, a in call] for call in calls]


def shapley_permutations(n_units: int, permutations: int, generator, antithetic: bool = True):
    """``permutations`` rows of a permutation of 0 .. n_units - 1 drawn with ``torch.randperm`` from ``generator`` (a CPU
    ``torch.Generator``); with ``antithetic`` row 2i + 1 is row 2i reversed and ``permutations`` must be even.  int64 [P, n]."""
    P = int(permutations)
    if P < 1:
        raise ValueError(f"shapley: permutations must be >= 1, got {P}")
    if antithetic and P % 2:
        raise ValueError(f"shapley: antithetic sampling needs an even number of permutations, got {P}")
    rows = []
    for _ in range(P // 2 if antithetic else P):
        r = torch.randperm(n_units, generator=generator)
        rows += [r, r.flip(0)] if antithetic else [r]
    return torch.stack(rows)


def shapley_chain(perm):
    """The coalitions a permutation estimate evaluates beyond the full input: the empty coalition, then for each row p of ``perm``
    the chain S^p_1 .. S^p_{n-1} (the first j units of row p).  bool [1 + P (n - 1), n], True: present."""
    perm = torch.as_tensor(perm, dtype=torch.int64)
    P, n = perm.shape
    rank = torch.empty_like(perm)
    rank.scatter_(1, perm, torch.arange(n).expand(P, n).contiguous())        # rank[p, u]: position of unit u in row p
    j = torch.arange(1, n).view(1, -1, 1)
    chain = rank.view(P, 1, n) < j                                            # [P, n - 1, n]
    return torch.cat([torch.zeros(1, n, dtype=torch.bool), chain.reshape(-1, n)])


def shapley_reference(values, perm, group: int, dtype=np.float32):
    """numpy float64 restatement of vb200_shapley_values for one message: ``values`` [2 + P (n - 1)] (v(empty), v(all), the chains),
    ``perm`` [P, n].  Returns (phi, stderr), each step the header's, in its order, rounded to ``dtype`` (float32: the device's
    outputs; float64: before that rounding)."""
    v = np.asarray(values, dtype=np.float32).astype(np.float64)
    perm = np.asarray(perm, dtype=np.int64)
    P, n = perm.shape
    c = np.empty((P, n + 1), dtype=np.float64)
    c[:, 0], c[:, n] = v[0], v[1]
    c[:, 1:n] = v[2:].reshape(P, n - 1)
    d = np.empty((P, n), dtype=np.float64)
    for p in range(P):
        for j in range(n):
            d[p, perm[p, j]] = c[p, j + 1] - c[p, j]
    G = P // group
    phi, se = np.empty(n), np.empty(n)
    for u in range(n):
        s = 0.0
        for p in range(P):
            s = s + float(d[p, u])
        phi[u] = s / P
        ss = 0.0
        for q in range(G):
            m = 0.0
            for i in range(group):
                m = m + float(d[q * group + i, u])
            t = m / group - phi[u]
            ss = ss + t * t
        se[u] = math.sqrt(ss / (G - 1) / G) if G >= 2 else float("nan")
    return phi.astype(dtype), se.astype(dtype)


def cross_pairs(units):
    """Every (word unit, box unit) pair of one message's ``units`` (``(positions, boxes)`` tuples) in unit order: a word unit has
    positions only, a box unit boxes only; units with both are in no pair."""
    words = [u for u, (ps, bs) in enumerate(units) if ps and not bs]
    boxes = [u for u, (ps, bs) in enumerate(units) if bs and not ps]
    return [(w, b) for w in words for b in boxes]


def interaction_pairs(pairs, units):
    """``shapley_interactions``' ``pairs`` checked against each message's ``units``: per message ``"cross"`` (``cross_pairs``) or a
    list of ``(a, b)`` unit indices, a != b.  Returns int32 numpy arrays [Q, 2], at least one pair per message and at most
    ``_lib.INTERACTION_MAX_PAIRS`` over all messages."""
    pairs = list(pairs)
    if len(pairs) != len(units):
        raise ValueError(f"shapley_interactions: pairs need one entry per message ({len(units)})")
    out, total = [], 0
    for i, (p, us) in enumerate(zip(pairs, units)):
        n = len(us)
        if n < 2:
            raise ValueError(f"shapley_interactions: message {i} has {n} unit; a pair needs two")
        if isinstance(p, str):
            if p != "cross":
                raise ValueError(f"shapley_interactions: message {i} pairs {p!r}: a list of (a, b) or \"cross\"")
            p = cross_pairs(us)
        a = np.asarray([tuple(int(x) for x in ab) for ab in p], dtype=np.int64).reshape(-1, 2)
        if len(a) == 0:
            raise ValueError(f"shapley_interactions: message {i} has no pairs")
        for q, (x, y) in enumerate(a.tolist()):
            if not (0 <= x < n and 0 <= y < n):
                raise ValueError(f"shapley_interactions: message {i} pair {q} ({x}, {y}) has a unit outside [0, {n})")
            if x == y:
                raise ValueError(f"shapley_interactions: message {i} pair {q} pairs unit {x} with itself")
        total += len(a)
        if total > L.INTERACTION_MAX_PAIRS:
            raise ValueError(f"shapley_interactions: messages 0..{i} have {total} pairs, above {L.INTERACTION_MAX_PAIRS}")
        out.append(a.astype(np.int32))
    return out


def _ranks(perm):
    """rank[p, u]: the position of unit u in row p of ``perm`` (int64 [P, n])."""
    P, n = perm.shape
    rank = torch.empty_like(perm)
    rank.scatter_(1, perm, torch.arange(n).expand(P, n).contiguous())
    return rank


def interaction_coalitions(perm, pairs):
    """The coalitions the Shapley-Taylor pair indices add to ``shapley_chain(perm)``: for each row p of ``perm`` and pair q = (a, b)
    of ``pairs`` [Q, 2], with S the units ranked before the first of a and b in row p, S + {second} then S + {a, b}.
    bool [2 P Q, n], True: present."""
    perm = torch.as_tensor(perm, dtype=torch.int64)
    pairs = torch.as_tensor(np.asarray(pairs), dtype=torch.int64).reshape(-1, 2)
    P, n = perm.shape
    Q = pairs.shape[0]
    rank = _ranks(perm)
    ra, rb = rank[:, pairs[:, 0]], rank[:, pairs[:, 1]]                        # [P, Q]
    a, b = pairs[:, 0].expand(P, Q), pairs[:, 1].expand(P, Q)
    first, second = torch.where(ra < rb, a, b), torch.where(ra < rb, b, a)
    x1 = rank.view(P, 1, n) < torch.minimum(ra, rb).view(P, Q, 1)              # S
    x1.scatter_(2, second.unsqueeze(2), True)
    x2 = x1.clone()
    x2.scatter_(2, first.unsqueeze(2), True)
    return torch.stack([x1, x2], 2).reshape(2 * P * Q, n)


def interaction_reference(values, perm, pairs, group: int, dtype=np.float32):
    """numpy float64 restatement of vb200_interaction_values for one message: ``values`` [2 + P (n - 1) + 2 P Q] (v(empty), v(all),
    the chains, then x1, x2 per permutation and pair), ``perm`` [P, n], ``pairs`` [Q, 2].  Returns (interaction, stderr) [Q], each
    step the header's, in its order, rounded to ``dtype`` (float32: the device's outputs; float64: before that rounding)."""
    v = np.asarray(values, dtype=np.float32).astype(np.float64)
    perm = np.asarray(perm, dtype=np.int64)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    P, n = perm.shape
    Q = len(pairs)
    c = np.empty((P, n + 1), dtype=np.float64)
    c[:, 0], c[:, n] = v[0], v[1]
    c[:, 1:n] = v[2:2 + P * (n - 1)].reshape(P, n - 1)
    x = v[2 + P * (n - 1):].reshape(P, Q, 2)
    rank = _ranks(torch.from_numpy(perm)).numpy()
    r = np.minimum(rank[:, pairs[:, 0]], rank[:, pairs[:, 1]])                  # [P, Q]
    rows = np.arange(P)[:, None]
    d = ((x[:, :, 1] - c[rows, r + 1]) - x[:, :, 0]) + c[rows, r]             # elementwise: one rounding per step
    s = np.zeros(Q)
    for p in range(P):
        s = s + d[p]
    inter = s / P
    G = P // group
    ss = np.zeros(Q)
    for k in range(G):
        m = np.zeros(Q)
        for i in range(group):
            m = m + d[k * group + i]
        t = m / group - inter
        ss = ss + t * t
    se = np.sqrt(ss / (G - 1) / G) if G >= 2 else np.full(Q, np.nan)
    return inter.astype(dtype), se.astype(dtype)


def attention_list(kinds, layout_entry, entries):
    """The reference's attn_data_list from the maps of the selected entries: ``kinds`` / ``layout_entry`` are the full entry list's
    kinds and each entry's index in ``entries`` (-1: not selected) as ``attention_selection`` returns them.  One position per layer in
    execution order: a text or image layer (kinds 0 / 1) holds its entry, a connection layer (kinds 2 and 3, adjacent) the tuple
    ``(text->image, image->text)``; an entry left out of the selection is None, each direction of a connection layer on its own."""
    def get(e):
        return entries[layout_entry[e]] if layout_entry[e] >= 0 else None
    attn, e = [], 0
    while e < len(kinds):
        if kinds[e] == 2:
            attn.append((get(e), get(e + 1)))
            e += 2
        else:
            attn.append(get(e))
            e += 1
    return attn


def _full_selection(layout):
    """``attention_selection``'s (kinds, layout_entry) of a layout that holds every entry."""
    return [entry[-2] for entry in layout], list(range(len(layout)))


def split_packed_attention(flat, layout, t_rows, v_rows, selection=None):
    """The packed attention buffer (VB200_OUT_ATTENTION_PACKED) as the reference's attn_data_list: ``layout`` is
    ``[(heads, kind, float_offset)]`` of ``attention_layout_packed``, ``t_rows`` / ``v_rows`` the samples' T_b / V_b.  A text or image
    layer (kinds 0 / 1) gives a list of B views ``[heads, L_b, L_b]``; a connection layer (kinds 2 and 3, adjacent) a tuple of two
    such lists, ``[heads, T_b, V_b]`` and ``[heads, V_b, T_b]``.  Inside an entry sample b's block follows sample b - 1's.
    ``selection``: ``attention_selection``'s (kinds, layout_entry) when the layout holds a selection of the entries (None: every
    entry); positions follow ``attention_list`` (heads 1 under the head mean)."""
    dims = {0: (t_rows, t_rows), 1: (v_rows, v_rows), 2: (t_rows, v_rows), 3: (v_rows, t_rows)}
    entries = []
    for heads, kind, off in layout:
        shapes = [(heads, lq, lk) for lq, lk in zip(*dims[kind])]
        sizes = [h * lq * lk for h, lq, lk in shapes]
        parts = torch.split(flat[int(off):int(off) + sum(sizes)], sizes)
        entries.append([p.view(s) for p, s in zip(parts, shapes)])
    return attention_list(*(selection or _full_selection(layout)), entries)


def entry_mask_bits(entries, name: str = "attention_entries") -> int:
    """The bitmask of option ``name`` ("attention_entries" / "state_entries") from an iterable of entry indices."""
    if isinstance(entries, (str, bytes)) or not hasattr(entries, "__iter__"):
        raise TypeError(f"{name} must be an iterable of entry indices or None, got {entries!r}")
    mask = 0
    for e in entries:
        if isinstance(e, bool) or not isinstance(e, int):
            raise TypeError(f"{name}: entry index {e!r} is not an int")
        if not 0 <= e < 63:
            raise ValueError(f"{name}: entry index {e} outside [0, 63)")
        mask |= 1 << e
    if mask == 0:
        raise ValueError(f"{name}: select at least one entry (None selects every entry)")
    return mask


def attention_mask_bits(entries) -> int:
    """The "attention_entries" bitmask of an iterable of entry indices (``from_pretrained(attention_entries=...)``)."""
    return entry_mask_bits(entries, "attention_entries")


def state_list(layout_entry, entries):
    """The layer states as ``output_layer_states`` returns them: one position per entry of the full list (``state_selection``'s
    ``layout_entry``), ``entries[i]`` for an entry at layout index i and None for an entry left out."""
    return [entries[i] if i >= 0 else None for i in layout_entry]


def split_packed_states(flat, layout, t_rows, v_rows, rows_mode):
    """The entries of a packed layer-state buffer (VB200_OUT_LAYER_STATES): ``layout`` is ``[(kind, rows, width, float_offset)]`` of
    ``state_layout_packed``, ``t_rows`` / ``v_rows`` the samples' T_b / V_b.  Under ``rows_mode`` 0 an entry is a list of B
    ``[L_b, width]`` views, else a ``[B, width]`` view.  One ``torch.split`` of the entry's ``[rows, width]`` view along the rows:
    views made one by one cost about four times the host time, which at batch 64 was most of a call with every entry."""
    entries = []
    for kind, rows, width, off in layout:
        entry = flat[int(off):int(off) + rows * width].view(rows, width)
        entries.append(list(torch.split(entry, t_rows if kind == 0 else v_rows)) if rows_mode == 0 else entry)
    return entries


def relevance_entries(attn, kinds):
    """The maps of element 9 (``attention_list`` order) as ``attention_relevance`` reads them: (entries, packed, t_rows, v_rows).
    ``kinds`` is the full entry list's kinds (``attention_selection``); ``entries`` one tensor ``[B, heads, Lq, Lk]`` (dense) or one
    list of B ``[heads, Lq_b, Lk_b]`` views (packed) per entry in execution order; ``t_rows`` / ``v_rows`` each sample's T_b / V_b
    (dense: B copies of T / V), read from the shapes.  ValueError for an entry left out by the selection (None)."""
    entries = []
    for pos in attn:
        entries.extend(pos if isinstance(pos, tuple) else (pos,))
    if len(entries) != len(kinds):
        raise ValueError(f"attention_relevance: {len(entries)} attention entries, the model has {len(kinds)}")
    for e, x in enumerate(entries):
        if x is None:
            raise ValueError(f"attention_relevance: attention entry {e} is None (left out by attention_entries); "
                             "the rollout needs every entry")
    packed = not torch.is_tensor(entries[0])
    rows = {}                                             # stream (0 text, 1 image) -> per-sample rows
    for kind, x in zip(kinds, entries):
        lq, lk = {0: (0, 0), 1: (1, 1), 2: (0, 1), 3: (1, 0)}[kind]
        for stream, axis in ((lq, -2), (lk, -1)):
            if stream not in rows:
                rows[stream] = [int(m.shape[axis]) for m in x] if packed else [int(x.shape[axis])] * int(x.shape[0])
        if len(rows) == 2:
            break
    return entries, packed, rows[0], rows[1]


def maps_pointer(entries, packed, layout):
    """Device address of the flat map buffer behind ``entries`` (``relevance_entries``), checked against ``layout``: per entry
    (heads, float offset) of the buffer the engine's current selection describes.  Entry e (packed: its sample 0) must be a
    contiguous fp32 view at that offset of one buffer with that head count; ValueError otherwise."""
    if len(layout) != len(entries):
        raise ValueError(f"attention_relevance: {len(entries)} entries, the current map selection lays out {len(layout)}")
    first = [x[0] if packed else x for x in entries]
    base = first[0].data_ptr() - 4 * int(layout[0][1])
    for e, (x, (heads, off)) in enumerate(zip(first, layout)):
        if x.dtype != torch.float32 or not x.is_contiguous() or x.device != first[0].device:
            raise ValueError(f"attention_relevance: attention entry {e} is not a contiguous fp32 map on {first[0].device}")
        if x.data_ptr() != base + 4 * int(off) or int(x.shape[-3]) != heads:
            raise ValueError(f"attention_relevance: attention entry {e} is not where the current map selection puts it "
                             "(the maps must be element 9 of one forward under this selection)")
    return base


_ATTENTION_HEADS = {"all": 0, "mean": 1}
_STATE_ROWS = {"all": 0, "first": 1, "mean": 2}


class VILBertForVLTasks(object):
    """Drop-in for ``vilbert.vilbert.VILBertForVLTasks`` on the inference path the worker uses."""

    _create_fn = "vb200_create"            # the C ABI constructor of this model's checkpoint kind

    def __init__(self, config: BertConfig, num_labels: int = 3129, state_dict=None, default_gpu: bool = True,
                 use_cuda_graph: bool = True, use_pdl: Optional[bool] = None, strict: bool = True, compute_dtype: str = "fp16",
                 fused_layernorm: bool = False, return_attention: bool = False, max_plans: int = 0, max_rows_per_sample: int = 256,
                 attention_entries=None, attention_heads: str = "all", state_entries=None, state_rows: str = "all"):
        self.config = config
        self.num_labels = num_labels
        self._sd = _normalise_state_dict(state_dict) if state_dict is not None else None
        self._handle = None
        self._device = None
        if compute_dtype not in ("fp16", "bf16", "fp32x"):
            raise ValueError("compute_dtype must be 'fp16', 'bf16' or 'fp32x'")
        if fused_layernorm:
            raise ValueError("fused_layernorm=True: the cluster-LayerNorm GEMM epilogue was removed; every LayerNorm runs as "
                             "GEMM + row LayerNorm kernel")
        # Format of the tensor-core operands (weights and activations): fp16 (default), bf16, or "fp32x" -- the fp32-parity mode:
        # every operand as an fp16 hi/lo pair, three tensor-core products per k-step, fp32 attention (<= 1e-3 per logit against
        # the reference's fp32 forward, 3x the tensor work).  Accumulation, residual stream, LayerNorm, softmax and logits are
        # fp32 in every mode.
        # max_rows_per_sample (256..1024): the longest text (tokens + task token) or image (regions) sequence a call may bring.
        # Plans of up to 256 rows per sample keep their kernels; longer ones stream keys through the attention kernels.  Text is
        # bounded by max_position_embeddings (+ the task token) as well.
        if not 256 <= int(max_rows_per_sample) <= 1024:
            raise ValueError(f"max_rows_per_sample must be in [256, 1024], got {max_rows_per_sample}")
        # Which attention maps element 9 carries: attention_entries (entry indices of the full list in execution order, see
        # attention_selection; None: every entry) and attention_heads ("all", or "mean": each entry averaged over its heads, the
        # head axis kept as size 1).  Engine state, set when the engine is created and by set_option.
        if attention_heads not in _ATTENTION_HEADS:
            raise ValueError(f"attention_heads must be 'all' or 'mean', got {attention_heads!r}")
        # Which layer states output_layer_states returns: state_entries (entry indices of the full list, see state_selection; None:
        # every entry) and state_rows ("all" rows, each sample's "first" row, or each sample's "mean" over its real rows).
        if state_rows not in _STATE_ROWS:
            raise ValueError(f"state_rows must be 'all', 'first' or 'mean', got {state_rows!r}")
        self._opts = dict(use_cuda_graph=use_cuda_graph, use_pdl=use_pdl, strict=strict, compute_dtype=compute_dtype,
                          max_plans=int(max_plans), max_rows_per_sample=int(max_rows_per_sample),
                          attention_entries=None if attention_entries is None else attention_mask_bits(attention_entries),
                          attention_heads=_ATTENTION_HEADS[attention_heads],
                          state_entries=None if state_entries is None else entry_mask_bits(state_entries, "state_entries"),
                          state_rows=_STATE_ROWS[state_rows])
        # attn_data_list (element 9 of the tuple): the reference returns the 24 layers' attention probabilities when called with
        # output_all_attention_masks=True (worker.py:287-288) and never reads them; here they are computed only when this flag
        # is set as well (model.return_attention = True), otherwise element 9 is [].
        self.return_attention = bool(return_attention)
        self.training = False
        self._dims = {}

    # ------------------------------------------------------------------ reference construction protocol
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, config=None, num_labels=3129, default_gpu=True,
                        state_dict=None, **kwargs):
        if config is None:
            raise ValueError("config is required (worker.py:530-532 always passes it)")
        if state_dict is None:
            if isinstance(pretrained_model_name_or_path, dict):
                state_dict = pretrained_model_name_or_path
            else:
                state_dict = torch.load(pretrained_model_name_or_path, map_location="cpu")
        return cls(config, num_labels=num_labels, state_dict=state_dict, default_gpu=default_gpu, **kwargs)

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise L.VilbertB200Error("vilbert_b200 is an inference engine; train() is not supported")
        return self

    def cuda(self, device=0):
        if isinstance(device, torch.device):
            device = device.index or 0
        device = 0 if device is None else int(device)
        if self._handle is not None and self._device == device:
            return self
        self._create(device)
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise L.VilbertB200Error("vilbert_b200 runs on sm_90 GPUs only; there is no CPU path")
        return self.cuda(device.index or 0)

    def half(self):            # tensor-core operands are 16-bit already (compute_dtype); accepted for call-site compatibility
        return self

    def parameters(self):
        return iter(())

    def state_dict(self):
        return dict(self._sd) if self._sd is not None else {}

    # ------------------------------------------------------------------ engine lifetime
    def _config_json(self) -> bytes:
        d = {k: v for k, v in self.config.to_dict().items()
             if isinstance(v, (int, float, str, bool, list)) or v is None}
        return json.dumps(d).encode()

    def _create(self, device: int):
        lib = L.load()
        if self._sd is None:
            raise L.VilbertB200Error("no state_dict: build the model with from_pretrained(...)")
        if not torch.cuda.is_available():
            raise L.VilbertB200Error("no CUDA device visible; vilbert_b200 has no CPU fallback")
        self.close()
        names = [k.encode() for k in self._sd]
        arr = (L.Tensor * len(self._sd))()
        keep = []
        for i, (k, v) in enumerate(self._sd.items()):
            t = arr[i]
            t.name = names[i]
            t.dtype = _DTYPES[v.dtype]
            t.ndim = v.dim()
            t.shape[0] = v.shape[0]
            t.shape[1] = v.shape[1] if v.dim() == 2 else 0
            t.data = v.data_ptr()
            keep.append(v)
        opt = self._options(device)
        h = C.c_void_p()
        with torch.cuda.device(device):
            rc = getattr(lib, self._create_fn)(self._config_json(), len(self._sd), arr, C.byref(opt), C.byref(h))
        L.check(rc, None)
        self._handle, self._device = h, device
        L.check(lib.vb200_set_option(h, b"max_rows_per_sample", self._opts["max_rows_per_sample"]), h)
        for key in ("attention_entries", "attention_heads", "state_entries", "state_rows"):
            if self._opts[key]:
                L.check(lib.vb200_set_option(h, key.encode(), self._opts[key]), h)
        for key in ("hidden_size", "v_hidden_size", "bi_hidden_size", "vocab_size", "v_target_size",
                    "v_feature_size", "num_labels", "gqa_labels", "task_specific_tokens", "weight_bytes",
                    "operand_width_factor"):
            v = C.c_int64()
            L.check(lib.vb200_model_dim(h, key.encode(), C.byref(v)), h)
            self._dims[key] = v.value

    def _options(self, device: int):
        """The vb200_options of this model's constructor arguments (tri-state flags: 1 on, -1 off, 0 the engine default)."""
        opt = L.Options()
        opt.device = device
        opt.num_labels = int(self.num_labels or 0)
        opt.use_cuda_graph = 1 if self._opts["use_cuda_graph"] else -1
        # None: engine default (programmatic dependent launch on every kernel); True: the same, forced; False: none
        opt.use_pdl = 0 if self._opts["use_pdl"] is None else (1 if self._opts["use_pdl"] else -1)
        opt.strict = 1 if self._opts["strict"] else -1
        opt.act_fp16 = -1 if self._opts["compute_dtype"] == "bf16" else 1
        opt.split_fp32 = 1 if self._opts["compute_dtype"] == "fp32x" else 0
        opt.max_plans = self._opts["max_plans"]
        return opt

    def close(self):
        if self._handle is not None:
            L.load().vb200_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _engine_device(self) -> torch.device:
        """The engine's device; raises when the model has no engine (before any CUDA tensor or library call)."""
        if self._handle is None:
            raise L.VilbertB200Error("call model.cuda(i) first (worker.py:536); there is no CPU path")
        return torch.device("cuda", self._device)

    def _call(self, fn: str, *args):
        """``fn(handle, *args, stream)`` of the C ABI on the current stream of the engine's device; raises on a failed status."""
        device = self._engine_device()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            L.check(getattr(L.load(), fn)(self._handle, *args, C.c_void_p(stream)), self._handle)

    # ------------------------------------------------------------------ forward
    def _out_shapes(self, B, T, V, select):
        d = self._dims
        shapes = {
            "vil_prediction": (L.OUT_VIL_PREDICTION, (B, d["num_labels"])),
            "vil_prediction_gqa": (L.OUT_VIL_PREDICTION_GQA, (B, d["gqa_labels"])),
            "vil_logit": (L.OUT_VIL_LOGIT, (B, 1)),
            "vil_binary_prediction": (L.OUT_VIL_BINARY_PREDICTION, (B // 2, 2) if B % 2 == 0 else (B, 2)),
            "vil_tri_prediction": (L.OUT_VIL_TRI_PREDICTION, (B, 3)),
            "vision_prediction": (L.OUT_VISION_PREDICTION, (B, V, d["v_target_size"])),
            "vision_logit": (L.OUT_VISION_LOGIT, (B, V, 1)),
            "linguisic_prediction": (L.OUT_LINGUISIC_PREDICTION, (B, T, d["vocab_size"])),
            "linguisic_logit": (L.OUT_LINGUISIC_LOGIT, (B, T, 1)),
        }
        return {k: s for k, (bit, s) in shapes.items() if select & bit}

    def plan_info(self, batch, n_tokens, n_regions, select=L.OUT_TASK_HEADS):
        self._engine_device()
        n, f = C.c_int64(), C.c_double()
        L.check(L.load().vb200_plan_info(self._handle, batch, n_tokens, n_regions, select, C.byref(n), C.byref(f)),
                self._handle)
        return n.value, f.value

    def set_option(self, key, value):
        """Run-time knobs of the engine (include/vilbert_b200.h, vb200_set_option): "max_plans", "timeline", "profile_grid_pct",
        "gemm_kernel", "max_rows_per_sample", "attention_entries" (a bitmask), "attention_heads" (0 / 1), "state_entries" (a bitmask)
        and "state_rows" (0 / 1 / 2) -- the last five also applied to the engine a later .cuda() creates."""
        self._engine_device()
        L.check(L.load().vb200_set_option(self._handle, key.encode(), int(value)), self._handle)
        if key in ("max_rows_per_sample", "attention_entries", "attention_heads", "state_entries", "state_rows"):
            self._opts[key] = int(value)

    @property
    def max_rows_per_sample(self) -> int:
        """Longest text (tokens + task token) or image (regions) sequence a call of this model may bring."""
        return self._opts["max_rows_per_sample"]

    def profile_ops(self, batch, n_tokens, n_regions, select=L.OUT_TASK_HEADS, iters=5, grid_pct=0):
        """Per-launch device times (ms) of one forward: every kernel replayed alone from its own CUDA graph between two events.
        grid_pct (10..100): persistent-grid size of the GEMMs for THIS measurement only (production: 2/3 of the CTA slots)."""
        self._engine_device()
        if grid_pct:
            L.check(L.load().vb200_set_option(self._handle, b"profile_grid_pct", int(grid_pct)), self._handle)
        cap = 2048
        n = C.c_int32()
        kinds = (C.c_int32 * cap)()
        ms = (C.c_double * cap)()
        fl = (C.c_double * cap)()
        dims = (C.c_int32 * (4 * cap))()
        L.check(L.load().vb200_profile_ops(self._handle, batch, n_tokens, n_regions, select, iters, cap, C.byref(n), kinds, ms,
                                           fl, dims), self._handle)
        names = {0: "gemm", 1: "self_attention", 2: "co_attention", 3: "rowdot", 4: "layernorm", 5: "attention_f32", 7: "layer_state"}
        return [dict(kind=names.get(kinds[i], "?"), ms=ms[i], flops=fl[i], dims=list(dims[4 * i:4 * i + 4]))
                for i in range(min(n.value, cap))]

    def _prep(self, question, features, spatials, segment_ids, input_mask, image_mask, task_tokens, device):
        B, Tin = question.shape
        V = features.shape[1]
        q = _to_device(question, torch.int64, device)
        f = _to_device(features, torch.float32, device)
        s = _to_device(spatials, torch.float32, device)
        seg = _to_device(segment_ids if segment_ids is not None else torch.zeros_like(question), torch.int64, device)
        im = _to_device(input_mask if input_mask is not None else torch.ones_like(question), torch.int64, device)
        vm = _to_device(image_mask if image_mask is not None else torch.ones(B, V, dtype=torch.uint8), torch.uint8, device)
        tk = _task_rows(task_tokens if task_tokens is not None else torch.zeros(B, 1, dtype=torch.int64), B, device)
        if tuple(f.shape) != (B, V, self._dims["v_feature_size"]) or tuple(s.shape) != (B, V, 5) \
                or tuple(seg.shape) != (B, Tin) or tuple(im.shape) != (B, Tin) or tuple(vm.shape) != (B, V):
            raise ValueError("input shapes do not match the worker.py:416-455 layout")
        return q, f, s, seg, im, vm, tk

    def __call__(self, *args, **kwargs):
        return self.forward(*args, **kwargs)

    @torch.no_grad()
    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None,
                image_attention_mask=None, co_attention_mask=None, task_ids=None,
                output_all_encoded_layers=False, output_all_attention_masks=False,
                compute_pretraining_heads=False, select: Optional[int] = None, debug_taps: bool = False, slot: int = 0,
                output_layer_states: bool = False):
        """Positional signature and 10-tuple of worker.py:286-289.

        ``vision_prediction`` / ``linguisic_prediction`` (the pre-training heads, elements 5 and 7, never read
        by the worker) are computed only with ``compute_pretraining_heads=True`` and are ``None`` otherwise;
        ``attn_data_list`` (element 9, never read by the worker) is the list of the 24 layers' attention probabilities in
        execution order -- ``[B, heads, L, L]`` for a text / image layer, a ``(text->image [B, heads, T, V], image->text
        [B, heads, V, T])`` tuple for a connection layer -- when ``output_all_attention_masks`` AND ``self.return_attention``
        are set, else ``[]``; with ``attention_entries`` / ``attention_heads`` an entry left out is None (each direction of a
        connection layer on its own) and a head-mean entry is ``[B, 1, Lq, Lk]``.  ``slot`` selects one of 16 independent
        workspaces: calls on different slots may be in flight concurrently on different CUDA streams.  ``output_all_encoded_layers``
        is accepted and ignored.  With ``output_layer_states`` the call returns ``(result, states)``: ``result`` as without it,
        ``states`` the layer states of ``state_selection`` (None for an entry left out), ``[B, L, hidden]`` under ``state_rows="all"``
        (padding rows included), else ``[B, hidden]``.
        """
        if self._handle is None and torch.is_tensor(input_txt) and input_txt.is_cuda:
            self.cuda(input_txt.device.index)
        device = self._engine_device()
        if select is None:
            select = L.OUT_ALL if compute_pretraining_heads else L.OUT_TASK_HEADS
        q, f, s, seg, im, vm, tk = self._prep(input_txt, input_imgs, image_loc, token_type_ids, attention_mask,
                                              image_attention_mask, task_ids, device)
        B, Tin = q.shape
        V = f.shape[1]
        inp = L.Inputs(B, Tin, V, q.data_ptr(), f.data_ptr(), s.data_ptr(), seg.data_ptr(), im.data_ptr(),
                       vm.data_ptr(), None, tk.data_ptr())
        want_attn = bool(output_all_attention_masks and self.return_attention)
        outs, o, select = self._alloc_outputs(B, Tin, V, select, debug_taps, want_attn, device)
        if output_layer_states:
            select, states = self._dense_states(B, Tin, V, select, o, device)
        self._call("vb200_forward_slot", C.byref(inp), C.byref(o), select, slot)
        result = self._result(outs, B, Tin, V, debug_taps)
        return (result, states()) if output_layer_states else result

    # ------------------------------------------------------------------ shared output plumbing
    def attention_layout(self, B, Tin, V):
        """[(heads, Lq, Lk, kind, float_offset)] of the flat attention buffer + its size (vb200_attention_layout)."""
        self._engine_device()
        lib = L.load()
        n = C.c_int32()
        total = C.c_int64()
        L.check(lib.vb200_attention_layout(self._handle, B, Tin, V, 0, C.byref(n), None, None, C.byref(total)), self._handle)
        dims = (C.c_int32 * (4 * n.value))()
        offs = (C.c_int64 * n.value)()
        L.check(lib.vb200_attention_layout(self._handle, B, Tin, V, n.value, C.byref(n), dims, offs, C.byref(total)), self._handle)
        return [(dims[4 * i], dims[4 * i + 1], dims[4 * i + 2], dims[4 * i + 3], offs[i]) for i in range(n.value)], total.value

    def attention_selection(self):
        """(kinds, layout_entry) of the full attention-map entry list in execution order (vb200_attention_selection): each entry's
        kind (0 text, 1 image, 2 / 3 the text->image / image->text direction of a connection layer) and its index in the layouts of
        the current selection, -1 when it is not selected."""
        self._engine_device()
        lib = L.load()
        n = C.c_int32()
        L.check(lib.vb200_attention_selection(self._handle, 0, C.byref(n), None, None), self._handle)
        kinds, where = (C.c_int32 * n.value)(), (C.c_int32 * n.value)()
        L.check(lib.vb200_attention_selection(self._handle, n.value, C.byref(n), kinds, where), self._handle)
        return list(kinds), list(where)

    def attention_layout_packed(self, n_tokens, n_regions):
        """[(heads, kind, float_offset)] of the packed attention buffer of a batch with these Tin_b / V_b (for
        ``forward_regions_packed``, V_b = n_boxes_b + 1) + its size in floats (vb200_attention_layout_packed)."""
        self._engine_device()
        lib = L.load()
        nt, nr = _host_ints(n_tokens), _host_ints(n_regions)
        if len(nt) != len(nr):
            raise ValueError("attention_layout_packed: n_tokens and n_regions must have the same length")
        args = (self._handle, len(nt), _int32s(nt), _int32s(nr))
        n, total = C.c_int32(), C.c_int64()
        L.check(lib.vb200_attention_layout_packed(*args, 0, C.byref(n), None, None, C.byref(total)), self._handle)
        dims = (C.c_int32 * (2 * n.value))()
        offs = (C.c_int64 * n.value)()
        L.check(lib.vb200_attention_layout_packed(*args, n.value, C.byref(n), dims, offs, C.byref(total)), self._handle)
        return [(dims[2 * i], dims[2 * i + 1], offs[i]) for i in range(n.value)], total.value

    def attention_relevance(self, attn):
        """Relevance of every text and image position to the two rows the answer heads read, from element 9 of ``forward`` /
        ``forward_regions`` (dense) or ``forward_packed`` / ``forward_regions_packed`` (packed), on the device
        (vb200_attention_relevance): the residual-weighted attention rollout through both streams, row 0 the text CLS row and row 1
        the image global row, each ``T + V`` floats (text columns first) that sum to 1.  Returns a device tensor ``[B, 2, T + V]``
        (dense; padded positions are 0) or a list of B ``[2, T_b + V_b]`` views of one buffer (packed).  Every entry must be in the
        maps (ValueError for a None entry); heads may be kept or averaged.  Asynchronous on the current stream."""
        kinds, _ = self.attention_selection()
        entries, packed, t_rows, v_rows = relevance_entries(attn, kinds)
        task = 1 if self._dims["task_specific_tokens"] else 0
        tin = [t - task for t in t_rows]
        B = len(t_rows)
        if packed:
            layout = [(h, off) for h, kind, off in self.attention_layout_packed(tin, v_rows)[0]]
            nt, nv = _int32s(tin), _int32s(v_rows)
        else:
            layout = [(h, off) for h, lq, lk, kind, off in self.attention_layout(B, tin[0], v_rows[0])[0]]
            nt, nv = _int32s(tin[:1]), _int32s(v_rows[:1])
        ptr = maps_pointer(entries, packed, layout)
        device = self._engine_device()
        if (entries[0][0] if packed else entries[0]).device != device:
            raise ValueError(f"attention_relevance: the maps are not on the engine's device {device}")
        sizes = [2 * (t + v) for t, v in zip(t_rows, v_rows)]
        out = torch.empty(sum(sizes), dtype=torch.float32, device=device)
        self._call("vb200_attention_relevance", C.c_void_p(ptr), B, nt, nv, int(packed), out.data_ptr())
        if packed:
            return [p.view(2, s // 2) for p, s in zip(torch.split(out, sizes), sizes)]
        return out.view(B, 2, t_rows[0] + v_rows[0])

    def state_selection(self):
        """(kinds, layout_entry) of the full layer-state list in execution order (vb200_state_selection): each entry's kind (0 text,
        1 image) and its index in the layouts of the current selection, -1 when it is not selected."""
        self._engine_device()
        lib = L.load()
        n = C.c_int32()
        L.check(lib.vb200_state_selection(self._handle, 0, C.byref(n), None, None), self._handle)
        kinds, where = (C.c_int32 * n.value)(), (C.c_int32 * n.value)()
        L.check(lib.vb200_state_selection(self._handle, n.value, C.byref(n), kinds, where), self._handle)
        return list(kinds), list(where)

    def _state_layout(self, fn, *args):
        """[(kind, rows, width, float_offset)] of the selected layer states and the buffer size (vb200_state_layout[_packed])."""
        self._engine_device()
        lib = L.load()
        n, total = C.c_int32(), C.c_int64()
        L.check(getattr(lib, fn)(self._handle, *args, 0, C.byref(n), None, None, None, C.byref(total)), self._handle)
        kinds, dims, offs = (C.c_int32 * n.value)(), (C.c_int32 * (2 * n.value))(), (C.c_int64 * n.value)()
        L.check(getattr(lib, fn)(self._handle, *args, n.value, C.byref(n), kinds, dims, offs, C.byref(total)), self._handle)
        return [(kinds[i], dims[2 * i], dims[2 * i + 1], offs[i]) for i in range(n.value)], total.value

    def state_layout(self, B, Tin, V):
        """[(kind, rows, width, float_offset)] of a dense forward's layer-state buffer + its size in floats."""
        return self._state_layout("vb200_state_layout", B, Tin, V)

    def state_layout_packed(self, n_tokens, n_regions):
        """[(kind, rows, width, float_offset)] of a packed forward's layer-state buffer for these Tin_b / V_b + its size in floats."""
        nt, nr = _host_ints(n_tokens), _host_ints(n_regions)
        if len(nt) != len(nr):
            raise ValueError("state_layout_packed: n_tokens and n_regions must have the same length")
        return self._state_layout("vb200_state_layout_packed", len(nt), _int32s(nt), _int32s(nr))

    def _dense_states(self, B, Tin, V, select, o, device):
        """Flat layer-state buffer of a dense forward bound to ``o.layer_states``: (select, states)."""
        layout, total = self.state_layout(B, Tin, V)
        flat = torch.empty(total, dtype=torch.float32, device=device)
        o.layer_states = flat.data_ptr()
        every_row = self._opts["state_rows"] == 0
        entries = [flat[off:off + rows * width].view((B, rows // B, width) if every_row else (B, width))
                   for kind, rows, width, off in layout]
        where = self.state_selection()[1]
        return select | L.OUT_LAYER_STATES, lambda: state_list(where, entries)

    def _packed_states(self, nt, nv, select, o, device):
        """Flat layer-state buffer of a packed forward with Tin_b = nt, V_b = nv bound to ``o.layer_states``: (select, states)."""
        layout, total = self.state_layout_packed(nt, nv)
        flat = torch.empty(total, dtype=torch.float32, device=device)
        o.layer_states = flat.data_ptr()
        task = 1 if self._dims["task_specific_tokens"] else 0
        entries = split_packed_states(flat, layout, [t + task for t in nt], nv, self._opts["state_rows"])
        where = self.state_selection()[1]
        return select | L.OUT_LAYER_STATES, lambda: state_list(where, entries)

    def _packed_attention(self, nt, nv, select, o, device):
        """Flat buffer of the packed attention maps for Tin_b = nt, V_b = nv, bound to ``o.attention_probs``: (select, flat, split)."""
        layout, total = self.attention_layout_packed(nt, nv)
        flat = torch.empty(total, dtype=torch.float32, device=device)
        o.attention_probs = flat.data_ptr()
        task = 1 if self._dims["task_specific_tokens"] else 0
        sel = self.attention_selection()
        return select | L.OUT_ATTENTION_PACKED, lambda: split_packed_attention(flat, layout, [t + task for t in nt], nv, sel)

    @staticmethod
    def _with_attention(result, attn, debug_taps):
        """``_result``'s tuple with element 9 replaced by ``attn``."""
        if debug_taps:
            return result[0][:9] + (attn,), result[1]
        return result[:9] + (attn,)

    def _alloc_outputs(self, B, Tin, V, select, debug_taps, want_attn, device):
        T = Tin + (1 if self._dims["task_specific_tokens"] else 0)
        outs = {k: torch.empty(shape, dtype=torch.float32, device=device)
                for k, shape in self._out_shapes(B, T, V, select).items()}
        if debug_taps:
            outs["sequence_output_t"] = torch.empty(B, T, self._dims["hidden_size"], dtype=torch.float32, device=device)
            outs["sequence_output_v"] = torch.empty(B, V, self._dims["v_hidden_size"], dtype=torch.float32, device=device)
            outs["pooled_output"] = torch.empty(B, self._dims["bi_hidden_size"], dtype=torch.float32, device=device)
        if want_attn:
            _, total = self.attention_layout(B, Tin, V)
            outs["attention_probs"] = torch.empty(total, dtype=torch.float32, device=device)
            select |= L.OUT_ATTENTION
        o = L.StateOutputs()
        for k, t in outs.items():
            setattr(o, k, t.data_ptr())
        return outs, o, select

    def _result(self, outs, B, Tin, V, debug_taps):
        g = outs.get
        attn = []
        if "attention_probs" in outs:
            flat = outs["attention_probs"]
            layout, _ = self.attention_layout(B, Tin, V)
            entries = [flat[off:off + B * heads * lq * lk].view(B, heads, lq, lk) for heads, lq, lk, kind, off in layout]
            attn = attention_list(*self.attention_selection(), entries)
        result = (g("vil_prediction"), g("vil_prediction_gqa"), g("vil_logit"), g("vil_binary_prediction"),
                  g("vil_tri_prediction"), g("vision_prediction"), g("vision_logit"), g("linguisic_prediction"),
                  g("linguisic_logit"), attn)
        if debug_taps:
            return result, {k: outs[k] for k in ("sequence_output_t", "sequence_output_v", "pooled_output")}
        return result

    # ------------------------------------------------------------------ detector output in, logits out (worker.py:388-458)
    @torch.no_grad()
    def forward_regions(self, question, segment_ids, input_mask, task_tokens, box_features, boxes, image_wh, num_boxes=None,
                        select: Optional[int] = None, output_all_attention_masks=False, slot: int = 0, return_spatials=True,
                        output_layer_states: bool = False):
        """``custom_prediction``'s tensor construction fused into the forward: ``box_features [B, n, F]`` (what the detector
        returned, no global row), pixel ``boxes [B, n, 4]``, ``image_wh [B, 2]`` -> the 10-tuple (and the ``spatials``
        tensor ``[B, n+1, 5]`` the reference would have built: the grounding decode reads it, worker.py:379).  With
        ``output_layer_states``: ``(result, states)`` as ``forward`` returns them."""
        device = self._engine_device()
        q, seg, im = (_to_device(t, torch.int64, device) for t in (question, segment_ids, input_mask))
        B, Tin = q.shape
        tk = _task_rows(task_tokens, B, device)
        bf, bx, wh = (_to_device(t, torch.float32, device) for t in (box_features, boxes, image_wh))
        n = bf.shape[1]
        if tuple(bf.shape) != (B, n, self._dims["v_feature_size"]) or tuple(bx.shape) != (B, n, 4) or tuple(wh.shape) != (B, 2) \
                or tuple(seg.shape) != (B, Tin) or tuple(im.shape) != (B, Tin):
            raise ValueError("forward_regions: box_features [B,n,F], boxes [B,n,4], image_wh [B,2], text [B,Tin] expected")
        nb = _to_device(num_boxes, torch.int32, device) if num_boxes is not None else None
        sp = torch.empty(B, n + 1, 5, dtype=torch.float32, device=device) if return_spatials else None
        if select is None:
            select = L.OUT_TASK_HEADS
        inp = L.RegionInputs(B, Tin, n, q.data_ptr(), seg.data_ptr(), im.data_ptr(), tk.data_ptr(), bf.data_ptr(), bx.data_ptr(),
                             wh.data_ptr(), nb.data_ptr() if nb is not None else None, sp.data_ptr() if sp is not None else None)
        want_attn = bool(output_all_attention_masks and self.return_attention)
        outs, o, select = self._alloc_outputs(B, Tin, n + 1, select, False, want_attn, device)
        if output_layer_states:
            select, states = self._dense_states(B, Tin, n + 1, select, o, device)
        self._call("vb200_forward_regions", C.byref(inp), C.byref(o), select, slot)
        result = self._result(outs, B, Tin, n + 1, False), sp
        return (result, states()) if output_layer_states else result

    # ------------------------------------------------------------------ packed variable-length batches
    @torch.no_grad()
    def forward_packed(self, question, features, spatials, segment_ids, task_tokens, n_tokens, n_regions,
                       select: int = L.OUT_TASK_HEADS, slot: int = 0, debug_taps: bool = False, max_tokens: int = 0,
                       max_regions: int = 0, output_all_attention_masks: bool = False, output_layer_states: bool = False,
                       head_mask=None):
        """One forward of B samples with their own text lengths and region counts, stored back to back without padding:
        ``question`` / ``segment_ids`` ``[sum Tin_i]``, ``features`` ``[sum V_i, F]``, ``spatials`` ``[sum V_i, 5]``,
        ``task_tokens`` ``[B, 1]``; ``n_tokens`` / ``n_regions`` (lists or CPU int tensors) give Tin_i and V_i.  Every row is real
        (no masks).  Returns the 10-tuple: per-sample outputs as in ``forward``, per-row outputs packed (``vision_logit``
        ``[sum V_i, 1]``, ``linguisic_logit`` ``[sum T_i, 1]`` with T_i = Tin_i + 1, ...).  Element 9 is ``[]``, or with
        ``output_all_attention_masks`` AND ``self.return_attention`` the 24 layers' attention probabilities at each sample's own
        lengths (``split_packed_attention``: per layer a list of B ``[heads, L_i, L_i]`` tensors, a connection layer a tuple of two
        such lists), views of one flat buffer.  ``max_tokens`` / ``max_regions`` (0: this call's maxima) are the plan's capacities:
        calls with the same batch size and capacities share one plan and CUDA graph whatever their lengths.  With
        ``output_layer_states``: ``(result, states)``, each selected entry a list of B ``[L_i, hidden]`` views of one flat buffer
        under ``state_rows="all"``, else ``[B, hidden]``; None for an entry left out.  ``head_mask`` (``head_mask_shape(config)``
        for every sample, or ``[B, *that]`` per sample; None: no gate) scales each attention head's context by its factor, as
        ``pytorch_transformers``' ``attention_probs * head_mask`` does, through vb200_forward_packed_gated; the maps are then the
        gated ones."""
        device = self._engine_device()
        nt, nr = _host_ints(n_tokens), _host_ints(n_regions)
        B = len(nt)
        if len(nr) != B or B < 1:
            raise ValueError("forward_packed: n_tokens and n_regions must have the same, positive length")
        F = self._dims["v_feature_size"]
        q = _to_device(question, torch.int64, device).reshape(-1)
        seg = _to_device(segment_ids if segment_ids is not None else torch.zeros_like(q), torch.int64, device).reshape(-1)
        f = _to_device(features, torch.float32, device).reshape(-1, F)
        s = _to_device(spatials, torch.float32, device).reshape(-1, 5)
        tk = _task_rows(task_tokens if task_tokens is not None else torch.zeros(B, 1, dtype=torch.int64), B, device)
        sum_tin, sum_v = sum(nt), sum(nr)
        if q.numel() != sum_tin or seg.numel() != sum_tin or f.shape[0] != sum_v or s.shape[0] != sum_v:
            raise ValueError("forward_packed: question / segment_ids need sum(n_tokens) rows, features / spatials sum(n_regions)")
        rows_t = sum_tin + (B if self._dims["task_specific_tokens"] else 0)
        outs, o = self._alloc_packed_outputs(B, rows_t, sum_v, select, debug_taps, device)
        want_attn = bool(output_all_attention_masks and self.return_attention)
        if want_attn:
            select, maps = self._packed_attention(nt, nr, select, o, device)
        if output_layer_states:
            select, states = self._packed_states(nt, nr, select, o, device)
        inp = L.PackedInputs(B, int(max_tokens), int(max_regions), _int32s(nt), _int32s(nr), q.data_ptr(), seg.data_ptr(), f.data_ptr(),
                             s.data_ptr(), tk.data_ptr())
        if head_mask is None:
            self._call("vb200_forward_packed", C.byref(inp), C.byref(o), select, slot)
        else:
            gate = head_mask_rows(head_mask, B, head_mask_shape(self.config), device)
            self._call("vb200_forward_packed_gated", C.byref(inp), gate.data_ptr(), C.byref(o), select, slot)
        result = self._result(outs, B, 0, 0, debug_taps)
        result = self._with_attention(result, maps(), debug_taps) if want_attn else result
        return (result, states()) if output_layer_states else result

    @torch.no_grad()
    def forward_regions_packed(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes,
                               select: int = L.OUT_TASK_HEADS, slot: int = 0, max_tokens: int = 0, max_boxes: int = 0,
                               debug_taps: bool = False, return_spatials: bool = True, output_all_attention_masks: bool = False,
                               output_layer_states: bool = False, head_mask=None):
        """``forward_regions`` with every image at its own box count and every text at its own length, stored back to back without
        padding: ``question`` / ``segment_ids`` ``[sum Tin_i]`` (text already repeated per image), ``task_tokens`` ``[B, 1]``,
        ``box_features`` ``[sum n_boxes_i, F]`` and pixel ``boxes`` ``[sum n_boxes_i, 4]`` as the detector returned them,
        ``image_wh`` ``[B, 2]``; ``n_tokens`` / ``n_boxes`` (lists or CPU int tensors) give Tin_i and the box counts.  Image i has
        V_i = n_boxes_i + 1 regions (its global mean row first).  Returns ``(10-tuple, spatials)``: the tuple as ``forward_packed``
        returns it (per-image outputs ``[B, ...]``, per-row outputs packed over sum V_i / sum T_i rows), ``spatials`` the packed
        ``[sum V_i, 5]`` locations the reference would have built (None with ``return_spatials=False``).  Each image's rows are
        bit-identical to ``forward_regions`` of that image alone.  ``max_tokens`` / ``max_boxes`` (0: this call's maxima) are the
        plan's capacities; the plan is the one ``forward_packed`` uses at ``max_regions = max_boxes + 1``.  Element 9 follows
        ``forward_packed``: the attention maps at each image's own T_i / V_i with ``output_all_attention_masks`` and
        ``self.return_attention``, else ``[]``.  ``output_layer_states`` returns ``(result, states)`` and ``head_mask`` gates the
        heads as in ``forward_packed`` (vb200_forward_regions_packed_gated)."""
        device = self._engine_device()
        batch = PackedRegionBatch("forward_regions_packed", device, self._dims["v_feature_size"], question, segment_ids, task_tokens,
                                  box_features, boxes, image_wh, n_tokens, n_boxes)
        nt, nb = batch.nt, batch.nb
        B = len(nt)
        rows_t = sum(nt) + (B if self._dims["task_specific_tokens"] else 0)
        rows_v = sum(nb) + B
        sp = torch.empty(rows_v, 5, dtype=torch.float32, device=device) if return_spatials else None
        outs, o = self._alloc_packed_outputs(B, rows_t, rows_v, select, debug_taps, device)
        want_attn = bool(output_all_attention_masks and self.return_attention)
        if want_attn:
            select, maps = self._packed_attention(nt, [n + 1 for n in nb], select, o, device)
        if output_layer_states:
            select, states = self._packed_states(nt, [n + 1 for n in nb], select, o, device)
        inp = batch.inputs(max_tokens, max_boxes, sp.data_ptr() if sp is not None else None)
        if head_mask is None:
            self._call("vb200_forward_regions_packed", C.byref(inp), C.byref(o), select, slot)
        else:
            gate = head_mask_rows(head_mask, B, head_mask_shape(self.config), device)
            self._call("vb200_forward_regions_packed_gated", C.byref(inp), gate.data_ptr(), C.byref(o), select, slot)
        result = self._result(outs, B, 0, 0, debug_taps)
        result = (self._with_attention(result, maps(), debug_taps) if want_attn else result), sp
        return (result, states()) if output_layer_states else result

    def _alloc_packed_outputs(self, B, rows_t, rows_v, select, debug_taps, device):
        """Outputs of a packed call: per-sample outputs [B, ...], per-row outputs and taps [rows_t or rows_v, ...]."""
        d = self._dims
        packed = {"vision_prediction": (rows_v, d["v_target_size"]), "vision_logit": (rows_v, 1),
                  "linguisic_prediction": (rows_t, d["vocab_size"]), "linguisic_logit": (rows_t, 1)}
        outs = {k: torch.empty(packed.get(k, shape), dtype=torch.float32, device=device)
                for k, shape in self._out_shapes(B, 1, 1, select).items()}
        if debug_taps:
            outs["sequence_output_t"] = torch.empty(rows_t, d["hidden_size"], dtype=torch.float32, device=device)
            outs["sequence_output_v"] = torch.empty(rows_v, d["v_hidden_size"], dtype=torch.float32, device=device)
            outs["pooled_output"] = torch.empty(B, d["bi_hidden_size"], dtype=torch.float32, device=device)
        o = L.StateOutputs()
        for k, t in outs.items():
            setattr(o, k, t.data_ptr())
        return outs, o

    # ------------------------------------------------------------------ answer ablation
    @torch.no_grad()
    def answer_ablation(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, family="vqa",
                        answer=None, tokens=None, boxes_range=None, mask_token: int = 103, max_tokens: int = 0, max_boxes: int = 0,
                        slot: int = 0, return_logits: bool = False):
        """How much each question token and each detector box holds up an answer (vb200_answer_ablation): for every image of a
        packed detector-output batch (the inputs of ``forward_regions_packed``), the answer's probability with each question position
        replaced by ``mask_token`` in turn and with each box dropped in turn, every variant a forward of the engine built and scored
        on the device.  ``family``: "vqa", "gqa" or "snli_ve" (or the ``_lib.DECODE_*`` value).  ``answer``: None (each sample's
        unablated top-1), one column for every sample, or a list with one column (or None) per sample.  ``tokens`` / ``boxes_range``:
        see ``ablation_ranges`` (default: positions 1 .. Tin - 2 and every box).  Batches above the engine's 1024 variants per call
        are split across calls (``ablation_calls``).
        Returns one dict per sample: ``answer`` (the attributed column), ``prob`` / ``top1`` / ``top1_prob`` of the unablated input,
        ``tokens`` / ``boxes`` (the ablated positions and boxes) with ``token_prob`` / ``box_prob`` (the answer's probability without
        that unit) and ``token_top1`` / ``box_top1`` (the variant's own top-1), CPU tensors; with ``return_logits`` also ``logits``,
        a device tensor [1 + tokens + boxes, width] in that variant order."""
        nt, nb = PackedRegionBatch.lengths("answer_ablation", n_tokens, n_boxes)
        B = len(nt)
        fam = ABLATION_FAMILIES.get(family, 0) if isinstance(family, str) else int(family)
        if fam not in ABLATION_FAMILIES.values():
            raise ValueError(f"answer_ablation: family {family!r} is not one of {sorted(ABLATION_FAMILIES)} (NLVR2, retrieval and "
                             "grounding answers are not ablated)")
        if answer is None or isinstance(answer, int):
            answers = [-1 if answer is None else int(answer)] * B
        else:
            answers = [-1 if a is None else int(a) for a in answer]
            if len(answers) != B:
                raise ValueError(f"answer_ablation: answer has {len(answers)} entries for {B} samples")
        if any(a < -1 for a in answers):
            raise ValueError("answer_ablation: an answer column must be >= 0 (or None / -1: the unablated top-1)")
        calls = ablation_calls(ablation_ranges(nt, nb, tokens, boxes_range))
        batch = PackedRegionBatch("answer_ablation", self._engine_device(), self._dims["v_feature_size"], question, segment_ids,
                                  task_tokens, box_features, boxes, image_wh, nt, nb)
        d = self._dims
        width = {L.DECODE_VQA: d["num_labels"], L.DECODE_GQA: d["gqa_labels"], L.DECODE_SNLI_VE: 3}[fam]
        res = [dict(tokens=[], token_prob=[], token_top1=[], boxes=[], box_prob=[], box_top1=[], logits=[]) for _ in range(B)]
        for call in calls:
            sub = batch if len(calls) == 1 else batch.subset([i for i, _ in call])   # this call's samples (or pieces of one)
            msgs = _structs(L.AblationMsg, [(answers[i],) + r for i, r in call])
            variants = ablation_variants(call)
            logits, col, prob, top1, top1_prob = self._ablation_run("vb200_answer_ablation", sub.inputs(max_tokens, max_boxes),
                                                                    (msgs, fam, int(mask_token)), len(variants) * width,
                                                                    len(variants), slot)
            logits = logits.view(len(variants), width)
            for k, (i, kind, unit) in enumerate(variants):
                r = res[i]
                if kind == "base":
                    if "answer" not in r:
                        r.update(answer=col[k], prob=prob[k], top1=top1[k], top1_prob=top1_prob[k])
                        r["logits"].append(logits[k:k + 1])
                    continue
                r["tokens" if kind == "token" else "boxes"].append(unit)
                r[kind + "_prob"].append(prob[k])
                r[kind + "_top1"].append(top1[k])
                r["logits"].append(logits[k:k + 1])
        for r in res:
            for k in ("token_prob", "box_prob"):
                r[k] = torch.tensor(r[k], dtype=torch.float32)
            for k in ("token_top1", "box_top1"):
                r[k] = torch.tensor(r[k], dtype=torch.int64)
            logits = r.pop("logits")
            if return_logits:
                r["logits"] = torch.cat(logits)
        return res

    def _ablation_layout(self, fn, n_tokens, n_boxes, arr):
        """``fn`` (vb200_message / head / coalition_ablation_layout) for the engine messages ``arr``: the records ``(message, kind,
        unit, samples, offset, length)`` and the floats they need."""
        lib, nv, nf, ns = L.load(), C.c_int64(), C.c_int64(), C.c_int64()
        args = (len(n_tokens), _int32s(n_tokens), _int32s(n_boxes), arr, len(arr))
        L.check(getattr(lib, fn)(self._handle, *args, None, C.byref(nv), C.byref(nf), C.byref(ns)), self._handle)
        recs = (L.AblationVariant * max(nv.value, 1))()
        L.check(getattr(lib, fn)(self._handle, *args, recs, C.byref(nv), C.byref(nf), C.byref(ns)), self._handle)
        return [(r.message, r.kind, r.unit, r.samples, r.offset, r.length) for r in recs[:nv.value]], nf.value

    def _message_layout(self, n_tokens, n_boxes, msgs):
        """vb200_message_ablation_layout of messages given as ``_lib.AblationMessage`` field tuples: the records, the floats they
        need and the struct array."""
        arr = _structs(L.AblationMessage, msgs)
        return (*self._ablation_layout("vb200_message_ablation_layout", n_tokens, n_boxes, arr), arr)

    def _head_layout(self, n_tokens, n_boxes, msgs):
        """vb200_head_ablation_layout of messages given as ``_lib.HeadAblationMessage`` field tuples: the records, the floats they
        need and the struct array."""
        arr = _structs(L.HeadAblationMessage, msgs)
        return (*self._ablation_layout("vb200_head_ablation_layout", n_tokens, n_boxes, arr), arr)

    def _coalition_layout(self, n_tokens, n_boxes, arr):
        """vb200_coalition_ablation_layout of a ``_lib.CoalitionMessage`` array: the records and the floats they need."""
        return self._ablation_layout("vb200_coalition_ablation_layout", n_tokens, n_boxes, arr)

    def _ablation_run(self, fn, inp, args, n_floats, n_variants, slot):
        """One ablation call: ``fn`` on the batch ``inp`` with its message arguments ``args``.  Returns the variants' segments, a
        device tensor of ``n_floats``, and their scores (vb200_ablation_score) as lists: answer, prob, top1, top1_prob."""
        device = self._engine_device()
        logits = torch.empty(n_floats, dtype=torch.float32, device=device)
        scores = torch.empty(n_variants, 4, dtype=torch.int32, device=device)       # vb200_ablation_score
        self._call(fn, C.byref(inp), *args, logits.data_ptr(), scores.data_ptr(), int(slot))
        sc = scores.cpu()
        return logits, sc[:, 0].tolist(), sc[:, 1].view(torch.float32).tolist(), sc[:, 2].tolist(), sc[:, 3].view(torch.float32).tolist()

    @torch.no_grad()
    def head_ablation(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages,
                      max_tokens: int = 0, max_boxes: int = 0, slot: int = 0, return_logits: bool = False):
        """Head ablation for every decode family (vb200_head_ablation): the packed detector-output batch of ``message_ablation`` and
        messages ``(family, image_begin, n_images, answer=None, entries=None)``; each head of each entry in ``entries`` (a ``(begin,
        end)`` range of ``head_mask_shape``'s entry order, None: all) is removed in turn from every sample of the message, all variants
        in packed forwards of at most 1024 samples (a message above that is split at entry boundaries).  Returns per message a dict:
        ``answer`` / ``prob`` / ``top1`` / ``top1_prob`` of the unablated input and, as ``[n_entries, max_heads]`` tensors,
        ``head_prob`` (the attributed answer's probability with that head removed) and ``head_top1`` (the variant's top-1), NaN / -1
        where no variant ran (an entry outside the range, or a slot past the entry's head count); with ``return_logits`` the segments
        in layout order."""
        nt, nb = PackedRegionBatch.lengths("head_ablation", n_tokens, n_boxes)
        if not messages:
            raise ValueError("head_ablation: no messages")
        E, H = head_mask_shape(self.config)
        msgs = head_messages(messages, len(nt), E)
        batch = PackedRegionBatch("head_ablation", self._engine_device(), self._dims["v_feature_size"], question, segment_ids,
                                  task_tokens, box_features, boxes, image_wh, nt, nb)
        inp = batch.inputs(max_tokens, max_boxes)
        recs, _, _ = self._head_layout(nt, nb, msgs)
        res = [dict(head_prob=torch.full((E, H), float("nan")), head_top1=torch.full((E, H), -1, dtype=torch.int64), logits=[])
               for _ in msgs]
        for call in head_calls([r[:4] for r in recs], H):
            crecs, n_floats, arr = self._head_layout(nt, nb, [msgs[p][:4] + r for p, r in call])
            logits, col, prob, top1, top1_prob = self._ablation_run("vb200_head_ablation", inp, (arr, len(arr)), n_floats, len(crecs),
                                                                    slot)
            for k, (m, kind, unit, _, off, n) in enumerate(crecs):
                r = res[call[m][0]]
                if kind == 0:
                    if "answer" in r:
                        continue
                    r.update(answer=col[k], prob=prob[k], top1=top1[k], top1_prob=top1_prob[k])
                else:
                    r["head_prob"][unit // H, unit % H] = prob[k]
                    r["head_top1"][unit // H, unit % H] = top1[k]
                r["logits"].append(logits[off:off + n])
        for r in res:
            logits = r.pop("logits")
            if return_logits:
                r["logits"] = logits
        return res

    @torch.no_grad()
    def message_ablation(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages,
                         mask_token: int = 103, max_tokens: int = 0, max_boxes: int = 0, slot: int = 0, return_logits: bool = False):
        """Answer ablation for every decode family (vb200_message_ablation): the packed detector-output batch of ``answer_ablation``
        (laid out as the worker lays it out: the text repeated per image, an NLVR2 pair on an even sample) and ``messages``, each
        ``(family or task id, image_begin, n_images, answer=None, tokens=None, boxes=None)`` -- see ``message_pieces`` for the
        defaults.  ``answer`` indexes the message's segment: a head column, 0 / 1 for NLVR2, the image for retrieval, the row of
        ``vision_logit`` (0: the global box) for grounding.  Calls above the engine's 1024 forward samples are split along the
        engine's own layout records (``message_calls``).
        Returns one dict per message: ``answer``, ``prob``, ``top1``, ``top1_prob`` of the unablated input; ``tokens`` with
        ``token_prob`` / ``token_top1``; ``boxes`` as ``(image of the message, box)`` pairs with ``box_prob`` / ``box_top1`` (CPU
        tensors; grounding reports rows in the unablated image's numbering, answer -1 / prob 0 where the attributed box is dropped);
        with ``return_logits`` also ``logits``, the variants' segments (device tensors) in that order."""
        nt, nb = PackedRegionBatch.lengths("message_ablation", n_tokens, n_boxes)
        if not messages:
            raise ValueError("message_ablation: no messages")
        pieces = message_pieces(messages, nt, nb)
        batch = PackedRegionBatch("message_ablation", self._engine_device(), self._dims["v_feature_size"], question, segment_ids,
                                  task_tokens, box_features, boxes, image_wh, nt, nb)
        inp = batch.inputs(max_tokens, max_boxes)
        msgs = [p for p, _ in pieces]
        recs, _, _ = self._message_layout(nt, nb, msgs)
        res = [dict(tokens=[], token_prob=[], token_top1=[], boxes=[], box_prob=[], box_top1=[], logits=[]) for _ in messages]
        for call in message_calls([r[:4] for r in recs]):
            crecs, n_floats, arr = self._message_layout(nt, nb, [msgs[p][:4] + r for p, r in call])
            logits, col, prob, top1, top1_prob = self._ablation_run("vb200_message_ablation", inp, (arr, len(arr), int(mask_token)),
                                                                    n_floats, len(crecs), slot)
            for k, (m, kind, unit, _, off, n) in enumerate(crecs):
                p = call[m][0]
                r = res[pieces[p][1]]
                seg_k = logits[off:off + n]
                if kind == 0:
                    if "answer" not in r:
                        r.update(answer=col[k], prob=prob[k], top1=top1[k], top1_prob=top1_prob[k])
                        r["logits"].append(seg_k)
                    continue
                if kind == 1:
                    r["tokens"].append(unit)
                else:
                    first = [0]
                    for j in range(msgs[p][2]):
                        first.append(first[-1] + nb[msgs[p][1] + j])
                    img = max(j for j in range(msgs[p][2]) if first[j] <= unit)
                    r["boxes"].append((img, unit - first[img]))
                name = "token" if kind == 1 else "box"
                r[name + "_prob"].append(prob[k])
                r[name + "_top1"].append(top1[k])
                r["logits"].append(seg_k)
        for r in res:
            for k in ("token_prob", "box_prob"):
                r[k] = torch.tensor(r[k], dtype=torch.float32)
            for k in ("token_top1", "box_top1"):
                r[k] = torch.tensor(r[k], dtype=torch.int64)
            logits = r.pop("logits")
            if return_logits:
                r["logits"] = logits
        return res

    # ------------------------------------------------------------------ coalition ablation and Shapley values
    @staticmethod
    def _coalition_structs(msgs, units, bitmaps):
        """``_lib.CoalitionMessage`` array for engine messages ``msgs`` with their units and uint64 bitmaps; the arrays the structs
        point at are returned with it and must outlive every call that reads it."""
        keep, out = [], []
        for m, us, bm in zip(msgs, units, bitmaps):
            po = np.cumsum([0] + [len(p) for p, _ in us]).astype(np.int32)
            bo = np.cumsum([0] + [len(b) for _, b in us]).astype(np.int32)
            ps = np.array([x for p, _ in us for x in p] or [0], dtype=np.int32)
            bs = np.array([x for _, b in us for x in b] or [0], dtype=np.int32)
            bm = np.ascontiguousarray(bm, dtype=np.uint64)
            keep += [po, bo, ps, bs, bm]
            out.append(L.CoalitionMessage(*m, len(us), po.ctypes.data, ps.ctypes.data, bo.ctypes.data, bs.ctypes.data, bm.shape[0],
                                          bm.ctypes.data if bm.shape[0] else None))
        return (L.CoalitionMessage * len(out))(*out), keep

    def _coalition_run(self, name, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages, units,
                       coalitions, mask_token, max_tokens, max_boxes, slot, return_logits):
        """What ``coalition_ablation`` and ``shapley`` share: the messages checked, the layout split along its records into calls of
        at most 1024 samples, and per message its full input's score and its coalitions' probabilities and top-1s as lists."""
        nt, nb = PackedRegionBatch.lengths(name, n_tokens, n_boxes)
        if not messages:
            raise ValueError(f"{name}: no messages")
        msgs = coalition_messages(messages, len(nt))
        if len(units) != len(msgs) or len(coalitions) != len(msgs):
            raise ValueError(f"{name}: units and coalitions need one entry per message ({len(msgs)})")
        us = [coalition_units(u, nt[ib], sum(nb[ib:ib + k]), i) for i, (u, (_, ib, k, _)) in enumerate(zip(units, msgs))]
        bms = [coalition_bitmaps(c, len(u)) for c, u in zip(coalitions, us)]
        batch = PackedRegionBatch(name, self._engine_device(), self._dims["v_feature_size"], question, segment_ids, task_tokens,
                                  box_features, boxes, image_wh, nt, nb)
        inp = batch.inputs(max_tokens, max_boxes)
        arr, keep = self._coalition_structs(msgs, us, bms)
        recs, _ = self._coalition_layout(nt, nb, arr)
        res = [dict(units=u, prob_d=[], top1_d=[], logits=[], samples=0) for u in us]
        for call in coalition_calls([r[:4] for r in recs]):
            carr, ckeep = self._coalition_structs([msgs[m] for m, _ in call], [us[m] for m, _ in call],
                                                  [bms[m][c0:c1] for m, (c0, c1) in call])
            crecs, n_floats = self._coalition_layout(nt, nb, carr)
            logits, col, prob, top1, top1_prob = self._ablation_run("vb200_coalition_ablation", inp, (carr, len(carr), int(mask_token)),
                                                                    n_floats, len(crecs), slot)
            at = 0
            for m, (c0, c1) in call:
                r = res[m]
                n = c1 - c0
                if "answer" not in r:
                    r.update(answer=col[at], prob=prob[at], top1=top1[at], top1_prob=top1_prob[at])
                    if return_logits:
                        r["logits"].append(logits[crecs[at][4]:crecs[at][4] + crecs[at][5]])
                r["prob_d"] += prob[at + 1:at + 1 + n]
                r["top1_d"] += top1[at + 1:at + 1 + n]
                if return_logits:
                    r["logits"] += [logits[o:o + k] for *_, o, k in crecs[at + 1:at + 1 + n]]
                r["samples"] += sum(c[3] for c in crecs[at:at + 1 + n])
                at += 1 + n
            del carr, ckeep
        del arr, keep
        return res

    @torch.no_grad()
    def coalition_ablation(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages, units,
                           coalitions, mask_token: int = 103, max_tokens: int = 0, max_boxes: int = 0, slot: int = 0,
                           return_logits: bool = False):
        """The answer with any set of units removed at once (vb200_coalition_ablation): the packed detector-output batch of
        ``message_ablation``, ``messages`` ``(family or task id, image_begin, n_images, answer=None)`` of every family but grounding,
        per message its ``units`` (None: the defaults of ``coalition_units``; else ``(positions, boxes)`` groups, boxes numbered across
        the message's images) and its ``coalitions``, a bool [n_coalitions, n_units] array (True: the unit is present).  An absent
        unit's positions are replaced by ``mask_token`` in every image and its boxes dropped from their images.  Calls above the
        engine's 1024 forward samples are split along its layout records (``coalition_calls``), each piece with its full input.
        Returns per message ``answer`` / ``prob`` / ``top1`` / ``top1_prob`` of the full input, ``units``, ``coalition_prob`` (the
        attributed answer's probability, v(S)) and ``coalition_top1`` as CPU tensors, ``samples`` (the forward samples run); with
        ``return_logits`` the segments (device tensors), the full input's first, then the coalitions' in order."""
        res = self._coalition_run("coalition_ablation", question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens,
                                  n_boxes, messages, units, coalitions, mask_token, max_tokens, max_boxes, slot, return_logits)
        for r in res:
            r["coalition_prob"] = torch.tensor(r.pop("prob_d"), dtype=torch.float32)
            r["coalition_top1"] = torch.tensor(r.pop("top1_d"), dtype=torch.int64)
            logits = r.pop("logits")
            if return_logits:
                r["logits"] = logits
        return res

    @torch.no_grad()
    def shapley(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages, units=None,
                permutations: int = 8, seed: int = 0, antithetic: bool = True, mask_token: int = 103, max_tokens: int = 0,
                max_boxes: int = 0, slot: int = 0):
        """Permutation-sampled Shapley values of each message's units for its answer (``coalition_ablation``, then
        vb200_shapley_values on the device).  ``messages`` as for ``coalition_ablation``; ``units`` None (the defaults of
        ``coalition_units`` for every message) or one entry per message (None or ``(positions, boxes)`` groups).  ``permutations`` P
        rows per message are drawn message by message from one CPU ``torch.Generator`` seeded with ``seed``; with ``antithetic`` row
        2i + 1 reverses row 2i and the standard error is taken over the P / 2 pair means.  v(empty) and v(all) are evaluated once per
        message and the P (n - 1) interior chain coalitions after them.  Returns per message ``answer``, ``prob`` (v(all)),
        ``empty_prob`` (v(empty)), ``units``, ``phi`` and ``stderr`` (float32 CPU tensors [n_units]), ``perm`` and ``samples`` (the
        forward samples run)."""
        nt, nb = PackedRegionBatch.lengths("shapley", n_tokens, n_boxes)
        msgs = coalition_messages(messages, len(nt))
        units = [None] * len(msgs) if units is None else list(units)
        if len(units) != len(msgs):
            raise ValueError(f"shapley: units need one entry per message ({len(msgs)})")
        units = [coalition_units(u, nt[ib], sum(nb[ib:ib + k]), i) for i, (u, (_, ib, k, _)) in enumerate(zip(units, msgs))]
        gen = torch.Generator().manual_seed(int(seed))
        perms = [shapley_permutations(len(u), permutations, gen, antithetic) for u in units]
        res = self._coalition_run("shapley", question, segment_ids, task_tokens, box_features, boxes, image_wh, nt, nb,
                                  [m for m in msgs], units, [shapley_chain(p) for p in perms], mask_token, max_tokens, max_boxes, slot,
                                  False)
        device = self._engine_device()
        g = 2 if antithetic else 1
        values, descs, at_v, at_p, at_o = [], [], 0, 0, 0
        for r, p in zip(res, perms):
            P, n = p.shape
            values += r["prob_d"][:1] + [r["prob"]] + r["prob_d"][1:]
            descs.append(L.ShapleyMessage(n, P, g, at_p, at_v, at_o))
            at_v, at_p, at_o = at_v + 2 + P * (n - 1), at_p + P * n, at_o + n
        vals = torch.tensor(values, dtype=torch.float32, device=device)
        perm_d = torch.cat([p.reshape(-1) for p in perms]).to(device=device, dtype=torch.int32)
        phi = torch.empty(at_o, dtype=torch.float32, device=device)
        se = torch.empty(at_o, dtype=torch.float32, device=device)
        arr = (L.ShapleyMessage * len(descs))(*descs)
        self._call("vb200_shapley_values", arr, len(descs), perm_d.data_ptr(), vals.data_ptr(), phi.data_ptr(), se.data_ptr())
        phi, se = phi.cpu(), se.cpu()
        out = []
        for r, p, d in zip(res, perms, descs):
            o, n = d.out_offset, d.n_units
            out.append(dict(answer=r["answer"], prob=r["prob"], empty_prob=float(r["prob_d"][0]), units=r["units"],
                            phi=phi[o:o + n], stderr=se[o:o + n], perm=p, samples=r["samples"]))
        return out

    @torch.no_grad()
    def shapley_interactions(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, messages,
                             pairs, units=None, permutations: int = 8, seed: int = 0, antithetic: bool = True, mask_token: int = 103,
                             max_tokens: int = 0, max_boxes: int = 0, slot: int = 0):
        """Shapley-Taylor interaction indices of order 2 for chosen pairs of each message's units (Sundararajan et al. 2020): for a
        pair {a, b}, the mean over permutations of v(S + {a, b}) - v(S + {a}) - v(S + {b}) + v(S), S the units before the first
        of a and b -- positive when the answer needs both units, negative when either is enough.  ``messages``, ``units``,
        ``permutations``, ``seed`` and ``antithetic`` as for ``shapley``, whose permutations and chains this call draws and
        evaluates in the same way, so its ``phi`` and ``stderr`` are ``shapley``'s bits.  ``pairs``: per message ``"cross"`` (every
        word unit with every box unit, ``cross_pairs``) or a list of ``(a, b)`` unit indices.  Beyond the chains each permutation
        and pair adds the two coalitions of ``interaction_coalitions``; everything runs in one ``coalition_ablation`` pass (split at
        the engine's 1024 samples per call), then vb200_shapley_values and vb200_interaction_values on the device.
        Cost per message: (2 + P (n - 1) + 2 P Q) x its samples per variant (1, 2 for NLVR2, K for retrieval) forward samples,
        plus the full input once more for every engine call past the first.
        Returns per message ``answer``, ``prob`` (v(all)), ``empty_prob`` (v(empty)), ``units``, ``pairs`` (int64 [Q, 2]),
        ``interaction`` and ``interaction_stderr`` (float32 CPU tensors [Q]), ``phi`` and ``stderr`` ([n_units]), ``perm`` and
        ``samples`` (the forward samples run)."""
        nt, nb = PackedRegionBatch.lengths("shapley_interactions", n_tokens, n_boxes)
        msgs = coalition_messages(messages, len(nt))
        units = [None] * len(msgs) if units is None else list(units)
        if len(units) != len(msgs):
            raise ValueError(f"shapley_interactions: units need one entry per message ({len(msgs)})")
        units = [coalition_units(u, nt[ib], sum(nb[ib:ib + k]), i) for i, (u, (_, ib, k, _)) in enumerate(zip(units, msgs))]
        prs = interaction_pairs(pairs, units)
        gen = torch.Generator().manual_seed(int(seed))
        perms = [shapley_permutations(len(u), permutations, gen, antithetic) for u in units]
        coal = [torch.cat([shapley_chain(p), interaction_coalitions(p, q)]) for p, q in zip(perms, prs)]
        res = self._coalition_run("shapley_interactions", question, segment_ids, task_tokens, box_features, boxes, image_wh, nt, nb,
                                  msgs, units, coal, mask_token, max_tokens, max_boxes, slot, False)
        device = self._engine_device()
        g = 2 if antithetic else 1
        values, sdesc, idesc, at_v, at_p, at_o, at_q = [], [], [], 0, 0, 0, 0
        for r, p, q in zip(res, perms, prs):
            P, n = p.shape
            values += r["prob_d"][:1] + [r["prob"]] + r["prob_d"][1:]
            sdesc.append(L.ShapleyMessage(n, P, g, at_p, at_v, at_o))
            idesc.append(L.InteractionMessage(n, P, g, len(q), at_p, at_v, at_q, q.ctypes.data))
            at_v, at_p, at_o, at_q = at_v + 2 + P * (n - 1) + 2 * P * len(q), at_p + P * n, at_o + n, at_q + len(q)
        vals = torch.tensor(values, dtype=torch.float32, device=device)
        perm_d = torch.cat([p.reshape(-1) for p in perms]).to(device=device, dtype=torch.int32)
        phi, se = (torch.empty(at_o, dtype=torch.float32, device=device) for _ in range(2))
        inter, ise = (torch.empty(at_q, dtype=torch.float32, device=device) for _ in range(2))
        sarr, iarr = (L.ShapleyMessage * len(sdesc))(*sdesc), (L.InteractionMessage * len(idesc))(*idesc)
        self._call("vb200_shapley_values", sarr, len(sdesc), perm_d.data_ptr(), vals.data_ptr(), phi.data_ptr(), se.data_ptr())
        self._call("vb200_interaction_values", iarr, len(idesc), perm_d.data_ptr(), vals.data_ptr(), inter.data_ptr(), ise.data_ptr())
        phi, se, inter, ise = phi.cpu(), se.cpu(), inter.cpu(), ise.cpu()
        out = []
        for r, p, q, sd, idd in zip(res, perms, prs, sdesc, idesc):
            o, n, oq, k = sd.out_offset, sd.n_units, idd.out_offset, idd.n_pairs
            out.append(dict(answer=r["answer"], prob=r["prob"], empty_prob=float(r["prob_d"][0]), units=r["units"],
                            pairs=torch.from_numpy(q.astype(np.int64)), interaction=inter[oq:oq + k], interaction_stderr=ise[oq:oq + k],
                            phi=phi[o:o + n], stderr=se[o:o + n], perm=p, samples=r["samples"]))
        return out

    # ------------------------------------------------------------------ answer decode (worker.py:295-386)
    def decode_answers(self, out, messages, spatials=None):
        """prediction()'s decode for many messages in one kernel and one device-to-host copy (vb200_decode_answers_host).

        ``out`` is the 10-tuple a forward returned, dense or packed.  ``messages`` is a list of ``(family or task_id, first, count,
        top_n, image_wh)``: a str is a worker task id ("1", "15", "12", ...), an int a family (``_lib.DECODE_*``); the message's
        segment is rows [first, first + count) of its family's output, flattened (an NLVR2 pair row is image row // 2; grounding
        rows are rows of ``vision_logit`` flattened to [rows, 1]); ``image_wh`` is the (width, height) of a grounding message's
        image, else ignored.  ``spatials`` (grounding): the locations the forward read or wrote, dense [B, V, 5] or packed [rows, 5].
        Returns one ``(indices, probs, boxes)`` per message: top_n indices in the segment, best first (equal probabilities: lower
        index first), the fp32 softmax probabilities as Python floats, and for grounding top_n ``[x1, y1, x2, y2]`` pixel boxes
        (``int(spatial * size)``, worker.py:381-384), else None."""
        self._engine_device()
        args, families = self._decode_args(out, messages, spatials)
        n = len(messages)
        answers = (L.Answer * max(n, 1))()
        self._call("vb200_decode_answers_host", *args, answers)
        res = []
        for a, fam in zip(answers[:n], families):
            k = a.n
            boxes = [list(a.box[j]) for j in range(k)] if fam == L.DECODE_GROUNDING else None
            res.append((list(a.index[:k]), list(a.prob[:k]), boxes))
        return res

    def _decode_args(self, out, messages, spatials):
        """(msgs, n, outputs, batch, vision_rows, spatials) of vb200_decode_answers[_host] for a forward's 10-tuple, and the
        messages' families."""
        n = len(messages)
        msgs = (L.DecodeMsg * max(n, 1))()
        families = []
        for i, (fam, first, count, top_n, wh) in enumerate(messages):
            f = L.TASK_DECODE_FAMILY.get(fam, 0) if isinstance(fam, str) else int(fam)
            w, h = (float(wh[0]), float(wh[1])) if wh is not None else (0.0, 0.0)
            msgs[i] = L.DecodeMsg(f, int(first), int(count), int(top_n), w, h)
            families.append(f)
        o = L.Outputs()
        for k, name in ((0, "vil_prediction"), (1, "vil_prediction_gqa"), (2, "vil_logit"), (3, "vil_binary_prediction"),
                        (4, "vil_tri_prediction"), (6, "vision_logit")):
            t = out[k]
            if t is None:
                continue
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise ValueError(f"decode_answers: {name} must be a contiguous fp32 device tensor")
            setattr(o, name, t.data_ptr())
        # the per-sample row count: the pair head alone has B / 2 rows for an even B and B rows for an odd one, so 2 R is consistent
        batch = next((int(out[k].shape[0]) for k in (0, 1, 2, 4) if out[k] is not None),
                     2 * int(out[3].shape[0]) if out[3] is not None else 0)
        vision_rows = int(out[6].numel()) if out[6] is not None else 0
        sp = None
        if spatials is not None:
            if spatials.dtype != torch.float32 or not spatials.is_cuda or not spatials.is_contiguous() or spatials.shape[-1] != 5:
                raise ValueError("decode_answers: spatials must be a contiguous fp32 device tensor [..., 5]")
            if out[6] is not None and spatials.numel() // 5 != vision_rows:
                raise ValueError(f"decode_answers: spatials has {spatials.numel() // 5} rows, vision_logit {vision_rows}")
            sp = spatials.data_ptr()
        return (msgs, n, C.byref(o), batch, vision_rows, sp), families

    # ------------------------------------------------------------------ pre-training heads at chosen rows
    @torch.no_grad()
    def pretraining_heads(self, taps, text_rows=None, image_rows=None, pair_rows=None, top_k: int = 0):
        """The checkpoint's three pre-training objectives at the rows a caller lists (vb200_pretraining_heads), from the final states
        a forward returned as taps: ``taps`` is the dict of ``forward(..., debug_taps=True)``, ``forward_packed``,
        ``forward_regions_packed`` or ``forward_cached_packed`` with ``debug_taps=True``.  Rows index the flattened states: dense text
        row b * T + t of ``sequence_output_t`` [B, T, hidden] (T = Tin + 1 with the task token), packed rows as the packed taps hold
        them; image rows likewise in ``sequence_output_v``, pair rows in ``pooled_output`` [B, bi_hidden].

        Returns a dict of device tensors: ``token_logits`` [n_t, vocab] (masked-token prediction, ``cls.predictions``),
        ``region_logits`` [n_v, v_target_size] (masked-region prediction, ``cls.imagePredictions``) and ``alignment`` [n_p, 2]
        (``cls.bi_seq_relationship`` on pooled_t * pooled_v) for each list given, each row bit-identical to that row of the forward's
        full-row heads (element 3 of a batch-1 forward for the alignment).  Which alignment column means "matched" is an upstream
        convention not confirmed here: both logits are returned in the head's order.  With ``top_k`` (1..10), ``token_top`` /
        ``region_top`` are ``(indices [n, top_k] int32, probabilities [n, top_k] fp32)``: each row's softmax over its logits, best
        first, equal probabilities ranking the lower index first -- computed on the device, like everything else here, so the call
        returns as soon as its work is enqueued."""
        device = self._engine_device()
        inp, groups, keep = self._pretrain_rows("pretraining_heads", taps, text_rows, image_rows, pair_rows, device)
        inp.top_k = int(top_k)
        out = L.PretrainOut()
        res = {}
        for n, n_out, (logits, top) in groups:
            res[logits] = torch.empty(n, n_out, dtype=torch.float32, device=device)
            setattr(out, logits, res[logits].data_ptr())
            if top is not None and top_k:
                res[top] = torch.empty(n, C.sizeof(L.Answer) // 4, dtype=torch.int32, device=device)
                setattr(out, top, res[top].data_ptr())
        self._call("vb200_pretraining_heads", C.byref(inp), C.byref(out))
        k = int(top_k)
        for head in ("token", "region"):
            ans = res.get(head + "_top")
            if ans is not None:            # vb200_answer as int32 words: n, index[10], prob[10], box[10][4]
                res[head + "_top"] = (ans[:, 1:1 + k], ans[:, 1 + L.DECODE_MAX_TOP:1 + L.DECODE_MAX_TOP + k].view(torch.float32))
        return res

    def _pretrain_rows(self, api, taps, text_rows, image_rows, pair_rows, device):
        """vb200_pretrain_rows of the lists given (None: not part of the call) over the taps' flattened states; returns it, one
        ``(count, logits columns, (logits output, top output))`` per list given, and the host arrays the struct points to."""
        d = self._dims
        # (list, its rows, tap, width, logits columns, vb200_pretrain_rows fields: state, state rows, count, list; outputs: logits, top)
        specs = (("text_rows", text_rows, "sequence_output_t", d["hidden_size"], d["vocab_size"],
                  ("text_state", "t_rows", "n_t", "text_rows"), ("token_logits", "token_top")),
                 ("image_rows", image_rows, "sequence_output_v", d["v_hidden_size"], d["v_target_size"],
                  ("image_state", "v_rows", "n_v", "image_rows"), ("region_logits", "region_top")),
                 ("pair_rows", pair_rows, "pooled_output", d["bi_hidden_size"], 2,
                  ("pooled_state", "p_rows", "n_p", "pair_rows"), ("alignment", None)))
        inp, groups, keep = L.PretrainRows(), [], []
        for name, rows, tap, width, n_out, fields, outputs in specs:
            if rows is None:
                continue
            rows = _host_ints(rows)
            state = taps.get(tap)
            if state is None:
                raise ValueError(f"{api}: {name} needs the {tap} tap")
            if state.dtype != torch.float32 or state.device != device or not state.is_contiguous() or state.shape[-1] != width:
                raise ValueError(f"{api}: {tap} must be a contiguous fp32 [..., {width}] tensor on {device}")
            state = state.view(-1, width)
            arr = _int32s(rows)
            keep += [state, arr]
            for field, value in zip(fields, (state.data_ptr(), state.shape[0], len(rows), arr)):
                setattr(inp, field, value)
            groups.append((len(rows), n_out, outputs))
        return inp, groups, keep

    @torch.no_grad()
    def pretraining_objectives(self, taps, text_rows=None, token_labels=None, image_rows=None, image_targets=None, pair_rows=None,
                               pair_labels=None):
        """The three pre-training objectives at the rows a caller lists (vb200_pretraining_objectives), on the device: the heads of
        ``pretraining_heads`` at those rows, then each row's loss from its logits and each list's mean.  ``taps`` and the row lists
        are as for ``pretraining_heads``; ``token_labels`` gives one vocabulary id per text row, ``image_targets`` one
        [v_target_size] target distribution per image row (any float tensor, [n_v, v_target_size]), ``pair_labels`` one 0 / 1 class
        per pair row.

        Returns a dict of device tensors: ``token_loss`` [n_t] (masked-token cross-entropy), ``region_loss`` [n_v] (KL divergence of
        the target from the row's softmax, as ``torch.nn.functional.kl_div`` computes it), ``pair_loss`` [n_p] (alignment
        cross-entropy), and ``masked_lm_loss``, ``masked_img_loss``, ``next_sentence_loss`` ([1] each): the mean of each list, NaN for
        an empty list, as upstream's losses are for batches without a masked token, region or labelled pair."""
        device = self._engine_device()
        lists = (text_rows, image_rows, pair_rows)
        inp, _, keep = self._pretrain_rows("pretraining_objectives", taps, *lists, device)
        n_t, n_v, n_p = (len(_host_ints(r)) if r is not None else 0 for r in lists)
        tg = L.PretrainTargets()
        for field, labels, n in (("token_labels", token_labels, n_t), ("pair_labels", pair_labels, n_p)):
            if n:
                values = _host_ints(labels if labels is not None else [])
                if len(values) != n:
                    raise ValueError(f"pretraining_objectives: {field} needs one label per row ({n}), got {len(values)}")
                arr = _int32s(values)
                keep.append(arr)
                setattr(tg, field, arr)
        if n_v:
            t = _to_device(image_targets, torch.float32, device) if image_targets is not None else None
            if t is None or tuple(t.shape) != (n_v, self._dims["v_target_size"]):
                raise ValueError(f"pretraining_objectives: image_targets must be [{n_v}, {self._dims['v_target_size']}]")
            keep.append(t)
            tg.image_targets = t.data_ptr()
        res = {"token_loss": torch.empty(n_t, dtype=torch.float32, device=device),
               "region_loss": torch.empty(n_v, dtype=torch.float32, device=device),
               "pair_loss": torch.empty(n_p, dtype=torch.float32, device=device)}
        reduced = torch.empty(3, dtype=torch.float32, device=device)
        out = L.PretrainLosses(*(res[k].data_ptr() if res[k].numel() else None for k in ("token_loss", "region_loss", "pair_loss")),
                               reduced.data_ptr())
        self._call("vb200_pretraining_objectives", C.byref(inp), C.byref(tg), C.byref(out))
        res.update(masked_lm_loss=reduced[0:1], masked_img_loss=reduced[1:2], next_sentence_loss=reduced[2:3])
        return res

    # ------------------------------------------------------------------ detector-region selection (worker.py:123-176)
    @torch.no_grad()
    def select_regions(self, detections, max_boxes: int = 100, conf_thresh: float = 0.0, background: bool = False,
                       nms_iou: float = 0.5, *, dst_rows=None, out_rows: Optional[int] = None, box_features=None, boxes=None,
                       cls_prob: bool = False, objects: bool = False):
        """The detector's feature extraction step for every image in one call (vb200_select_regions): per-proposal softmax, per-class
        NMS on the original-pixel boxes, per-box maximum confidence, the top ``max_boxes`` of each image.

        ``detections`` is a sequence of ``(proposals [n_i, 4], scores [n_i, C], features [n_i, F], im_scale)`` per image: the boxes
        at the detector's input scale, the class logits (column 0 background) and the fc6 features.  Image i's k_i = min(max_boxes,
        n_i) rows go to rows ``dst_rows[i] ...`` of the outputs (default: back to back in image order, the layout
        ``forward_regions_packed`` takes with ``n_boxes = k_i``).  ``box_features`` [out_rows, F] / ``boxes`` [out_rows, 4] may be
        caller tensors (e.g. a packed batch with rows left free for filler images); rows outside the images' ranges are not
        written.  Returns a dict of device tensors: box_features, boxes (original pixels), num_boxes [n] int32, keep_index
        [out_rows] int32, max_conf [out_rows] (the sorted scores), cls_prob [out_rows, C] and objects [out_rows] int64 (the argmax of
        each cls_prob row) when asked for, else None; and the host lists ``n_boxes`` (k_i) and ``dst_rows``."""
        device = self._engine_device()
        n = len(detections)
        if n < 1:
            raise ValueError("select_regions: no images")
        heads, k = [], []
        for prop, sc, ft, scale in detections:
            prop, sc, ft = (_to_device(t, torch.float32, device) for t in (prop, sc, ft))
            if prop.dim() != 2 or prop.shape[1] != 4 or sc.dim() != 2 or ft.dim() != 2 or not prop.shape[0] == sc.shape[0] == ft.shape[0]:
                raise ValueError(f"select_regions: image {len(heads)} needs proposals [n, 4], scores [n, C] and features [n, F]")
            heads.append((prop, sc, ft, float(scale)))
            k.append(min(int(max_boxes), int(prop.shape[0])))
        Cn, F = int(heads[0][1].shape[1]), int(heads[0][2].shape[1])
        if any(int(h[1].shape[1]) != Cn or int(h[2].shape[1]) != F for h in heads):
            raise ValueError("select_regions: every image needs the same number of score columns and feature width")
        if dst_rows is None:
            dst_rows = packed_offsets(k)[:-1]
        dst_rows = [int(r) for r in dst_rows]
        if len(dst_rows) != n:
            raise ValueError("select_regions: one dst_row per image")
        if out_rows is None:
            out_rows = int(box_features.shape[0]) if box_features is not None else max(r + kk for r, kk in zip(dst_rows, k))

        def buf(t, shape, dtype):
            if t is None:
                return torch.empty(shape, dtype=dtype, device=device)
            if tuple(t.shape) != shape or t.dtype != dtype or t.device != device or not t.is_contiguous():
                raise ValueError(f"select_regions: output of shape {tuple(t.shape)} / {t.dtype}, need {shape} {dtype} on {device}")
            return t
        res = dict(box_features=buf(box_features, (out_rows, F), torch.float32), boxes=buf(boxes, (out_rows, 4), torch.float32),
                   num_boxes=torch.empty(n, dtype=torch.int32, device=device),
                   keep_index=torch.empty(out_rows, dtype=torch.int32, device=device),
                   max_conf=torch.empty(out_rows, dtype=torch.float32, device=device),
                   cls_prob=torch.empty(out_rows, Cn, dtype=torch.float32, device=device) if cls_prob else None,
                   objects=torch.empty(out_rows, dtype=torch.int64, device=device) if objects else None)
        imgs = (L.Detections * n)()
        for i, ((prop, sc, ft, scale), r) in enumerate(zip(heads, dst_rows)):
            imgs[i] = L.Detections(int(prop.shape[0]), r, scale, prop.data_ptr(), sc.data_ptr(), ft.data_ptr())
        params = L.SelectParams(Cn, F, int(max_boxes), float(conf_thresh), float(nms_iou), int(bool(background)), int(out_rows))
        sel = L.Selected(*[res[name].data_ptr() if res[name] is not None else None for name, _ in L.Selected._fields_])
        self._call("vb200_select_regions", imgs, n, C.byref(params), C.byref(sel))
        res["n_boxes"], res["dst_rows"] = k, dst_rows
        return res

    # ------------------------------------------------------------------ retrieval reuse (SURVEY.md section 8e)
    def _dense_state(self, kind, n, rows, device, **lengths):
        """An empty prefix state of n items with ``rows`` rows each: f32 and 16-bit rows of the ``kind`` stream and the key mask."""
        H = self._dims["hidden_size" if kind == "text" else "v_hidden_size"]
        S = self._dims["operand_width_factor"]
        return dict(kind=kind, n=n, **lengths, f32=torch.empty(n, rows, H, dtype=torch.float32, device=device),
                    h16=torch.empty(n, rows, H * S, dtype=torch.int16, device=device),
                    mask=torch.empty(n, rows, dtype=torch.float32, device=device))

    def _packed_state(self, kind, lengths, device, extra=0):
        """An empty packed prefix state: item i's rows (lengths[i] + extra) back to back from ``offsets[i]``, no mask; ``max_len`` is
        the longest of ``lengths``."""
        offs = packed_offsets(lengths, extra)
        H = self._dims["hidden_size" if kind == "text" else "v_hidden_size"]
        return dict(kind=kind, n=len(lengths), offsets=torch.tensor(offs, dtype=torch.int32), max_len=max(lengths),
                    f32=torch.empty(offs[-1], H, dtype=torch.float32, device=device),
                    h16=torch.empty(offs[-1], H, dtype=torch.int16, device=device))

    @torch.no_grad()
    def encode_text(self, question, segment_ids, input_mask, task_tokens):
        """Everything ahead of the first connection layer that depends on the caption alone (embeddings + text layers T0..),
        once per caption.  Returns an opaque state for ``forward_cached``."""
        device = self._engine_device()
        q = _to_device(question, torch.int64, device)
        n, Tin = q.shape
        seg, im = _to_device(segment_ids, torch.int64, device), _to_device(input_mask, torch.int64, device)
        tk = _task_rows(task_tokens, n, device)
        st = self._dense_state("text", n, Tin + (1 if self._dims["task_specific_tokens"] else 0), device, Tin=Tin)
        self._call("vb200_encode_text", n, Tin, q.data_ptr(), seg.data_ptr(), im.data_ptr(), tk.data_ptr(), st["f32"].data_ptr(),
                   st["h16"].data_ptr(), st["mask"].data_ptr())
        return st

    @torch.no_grad()
    def encode_image(self, features, spatials, image_mask):
        """The image-side prefix (image embedding, plus image layers scheduled ahead of the first connection layer), once per image."""
        device = self._engine_device()
        f = _to_device(features, torch.float32, device)
        n, V = f.shape[0], f.shape[1]
        s, vm = _to_device(spatials, torch.float32, device), _to_device(image_mask, torch.uint8, device)
        st = self._dense_state("image", n, V, device, V=V)
        self._call("vb200_encode_image", n, V, f.data_ptr(), s.data_ptr(), vm.data_ptr(), st["f32"].data_ptr(), st["h16"].data_ptr(),
                   st["mask"].data_ptr())
        return st

    @torch.no_grad()
    def forward_cached(self, text_state, text_index, image_state, image_index, select: int = L.OUT_VIL_LOGIT, slot: int = 0):
        """Pair b = (caption text_index[b], image image_index[b]) from cached states: the connection layers onwards.  Results are
        bit-identical to the full forward of the same pairs."""
        device = self._engine_device()
        ti, vi = _to_device(text_index, torch.int32, device), _to_device(image_index, torch.int32, device)
        B = ti.numel()
        if vi.numel() != B:
            raise ValueError("text_index and image_index must have the same length")
        Tin, V = text_state["Tin"], image_state["V"]
        outs, o, select = self._alloc_outputs(B, Tin, V, select, False, False, device)
        self._call("vb200_forward_cached", B, Tin, V, ti.data_ptr(), text_state["n"], text_state["f32"].data_ptr(),
                   text_state["h16"].data_ptr(), text_state["mask"].data_ptr(), vi.data_ptr(), image_state["n"],
                   image_state["f32"].data_ptr(), image_state["h16"].data_ptr(), image_state["mask"].data_ptr(), C.byref(o), select, slot)
        return self._result(outs, B, Tin, V, False)

    # ------------------------------------------------------------------ packed retrieval: every caption / image at its own length
    @torch.no_grad()
    def encode_text_packed(self, question, segment_ids, task_tokens, n_tokens, max_tokens: int = 0):
        """``encode_text`` of n captions stored back to back without padding: ``question`` / ``segment_ids`` ``[sum Tin_c]``,
        ``task_tokens`` ``[n, 1]``, ``n_tokens`` (list or CPU tensor) the Tin_c.  Returns an opaque state for
        ``forward_cached_packed``: caption c's rows sit at ``offsets[c]`` (T_c = Tin_c + 1 rows with the task token) and equal
        ``encode_text`` of that caption alone.  ``max_tokens`` (0: this call's maximum) is the plan capacity."""
        device = self._engine_device()
        nt = _host_ints(n_tokens)
        n = len(nt)
        q = _to_device(question, torch.int64, device).reshape(-1)
        seg = _to_device(segment_ids, torch.int64, device).reshape(-1)
        tk = _task_rows(task_tokens, n, device)
        if n < 1 or q.numel() != sum(nt) or seg.numel() != sum(nt):
            raise ValueError("encode_text_packed: question / segment_ids need sum(n_tokens) entries for n >= 1 captions")
        st = self._packed_state("text", nt, device, extra=1 if self._dims["task_specific_tokens"] else 0)
        self._call("vb200_encode_text_packed", n, int(max_tokens), _int32s(nt), q.data_ptr(), seg.data_ptr(), tk.data_ptr(),
                   st["f32"].data_ptr(), st["h16"].data_ptr())
        return st

    @torch.no_grad()
    def encode_image_packed(self, features, spatials, n_regions, max_regions: int = 0):
        """``encode_image`` of n images stored back to back without padding: ``features`` ``[sum V_i, F]``, ``spatials``
        ``[sum V_i, 5]``, ``n_regions`` the V_i.  Image i's state rows sit at ``offsets[i]`` and equal ``encode_image`` of that
        image alone."""
        device = self._engine_device()
        nr = _host_ints(n_regions)
        n = len(nr)
        f = _to_device(features, torch.float32, device).reshape(-1, self._dims["v_feature_size"])
        s = _to_device(spatials, torch.float32, device).reshape(-1, 5)
        if n < 1 or f.shape[0] != sum(nr) or s.shape[0] != sum(nr):
            raise ValueError("encode_image_packed: features / spatials need sum(n_regions) rows for n >= 1 images")
        st = self._packed_state("image", nr, device)
        self._call("vb200_encode_image_packed", n, int(max_regions), _int32s(nr), f.data_ptr(), s.data_ptr(), st["f32"].data_ptr(),
                   st["h16"].data_ptr())
        return st

    @torch.no_grad()
    def encode_regions_packed(self, box_features, boxes, image_wh, n_boxes, max_boxes: int = 0):
        """``encode_image_packed`` from detector output, as ``forward_regions_packed`` takes it: ``box_features`` ``[sum n_boxes_i, F]``,
        pixel ``boxes`` ``[sum n_boxes_i, 4]``, ``image_wh`` ``[n, 2]``, ``n_boxes`` (list or CPU tensor) the box counts.  Image i's
        state is V_i = n_boxes_i + 1 rows, its global mean row first, built on the device by the region pack of
        ``forward_regions_packed``: ``forward_cached_packed`` on these states gives that forward's scores bit for bit.
        ``max_boxes`` (0: this call's maximum) is the plan capacity; the plan is ``encode_image_packed``'s at ``max_regions =
        max_boxes + 1``."""
        device = self._engine_device()
        nb = _host_ints(n_boxes)
        n = len(nb)
        bf = _to_device(box_features, torch.float32, device).reshape(-1, self._dims["v_feature_size"])
        bx = _to_device(boxes, torch.float32, device).reshape(-1, 4)
        wh = _to_device(image_wh, torch.float32, device)
        if n < 1 or bf.shape[0] != sum(nb) or bx.shape[0] != sum(nb) or tuple(wh.shape) != (n, 2):
            raise ValueError("encode_regions_packed: box_features / boxes need sum(n_boxes) rows and image_wh [n, 2] for n >= 1 images")
        st = self._packed_state("image", [k + 1 for k in nb], device)
        self._call("vb200_encode_regions_packed", n, int(max_boxes), _int32s(nb), bf.data_ptr(), bx.data_ptr(), wh.data_ptr(),
                   st["f32"].data_ptr(), st["h16"].data_ptr())
        return st

    @torch.no_grad()
    def encode_detections_packed(self, detections, image_wh, max_boxes: int = 100, conf_thresh: float = 0.0, background: bool = False):
        """A retrieval gallery from the detector's raw heads: one ``select_regions`` of every image (``detections`` as there) into a
        packed device buffer, then one ``encode_regions_packed`` of the k_i = min(max_boxes, n_i) selected boxes with the images'
        ``image_wh`` ``[n, 2]``.  No feature row passes through the host.  Returns the ``encode_regions_packed`` state; the plan
        capacity is ``max_boxes``, so galleries of any proposal counts share one plan."""
        r = self.select_regions(detections, max_boxes, conf_thresh, background)
        return self.encode_regions_packed(r["box_features"], r["boxes"], image_wh, r["n_boxes"], max_boxes=max_boxes)

    @torch.no_grad()
    def forward_cached_packed(self, text_state, text_index, image_state, image_index, select: int = L.OUT_VIL_LOGIT, slot: int = 0,
                              max_tokens: Optional[int] = None, max_regions: Optional[int] = None, debug_taps: bool = False):
        """Pair b = (caption text_index[b], image image_index[b]) from packed states, every pair at its own lengths.  Index tensors may
        be on the CPU or the GPU (they are read on the host).  Returns the 10-tuple as ``forward_packed`` does (per-row outputs packed,
        pair after pair), bit-identical to ``forward_packed`` of the same pairs.  Capacities default to the states' longest caption /
        largest image, so every call on the same states and batch size shares one plan."""
        if text_state.get("kind") != "text" or image_state.get("kind") != "image" or "offsets" not in text_state \
                or "offsets" not in image_state:
            raise ValueError("forward_cached_packed: pass the states of encode_text_packed and encode_image_packed")
        device = self._engine_device()
        ti = torch.as_tensor(text_index).to(device="cpu", dtype=torch.int32).reshape(-1).contiguous()
        vi = torch.as_tensor(image_index).to(device="cpu", dtype=torch.int32).reshape(-1).contiguous()
        B = ti.numel()
        if vi.numel() != B:
            raise ValueError("text_index and image_index must have the same length")
        toffs, voffs = text_state["offsets"], image_state["offsets"]
        mt = text_state["max_len"] if max_tokens is None else int(max_tokens)
        mr = image_state["max_len"] if max_regions is None else int(max_regions)
        # row totals for the per-row outputs (indices clamped here; the engine rejects out-of-range ones)
        rows_t = int((toffs[1:] - toffs[:-1])[ti.long().clamp(0, text_state["n"] - 1)].sum())
        rows_v = int((voffs[1:] - voffs[:-1])[vi.long().clamp(0, image_state["n"] - 1)].sum())
        outs, o = self._alloc_packed_outputs(B, rows_t, rows_v, select, debug_taps, device)
        pairs = L.PackedPairs(B, mt, mr, ti.data_ptr(), vi.data_ptr(), text_state["n"], toffs.data_ptr(), text_state["f32"].data_ptr(),
                              text_state["h16"].data_ptr(), image_state["n"], voffs.data_ptr(), image_state["f32"].data_ptr(),
                              image_state["h16"].data_ptr())
        self._call("vb200_forward_cached_packed", C.byref(pairs), C.byref(o), select, slot)
        return self._result(outs, B, 0, 0, debug_taps)

    # ------------------------------------------------------------------ host-buffer entry (bench e2e, serving)
    def forward_host(self, question, features, spatials, segment_ids, input_mask, image_mask, task_tokens,
                     out: Dict[str, torch.Tensor], select: int = L.OUT_VIL_PREDICTION, slot: int = 0, synchronize: bool = True):
        """vb200_forward_host[_slot]: HOST (ideally pinned) tensors in, HOST tensors out; H2D + forward + D2H (+ stream sync).
        With ``synchronize=False`` the call returns after enqueueing on the current stream; synchronise that stream before
        reading ``out`` or re-using the input buffers."""
        B, Tin = question.shape
        V = features.shape[1]
        inp = L.Inputs(B, Tin, V, question.data_ptr(), features.data_ptr(), spatials.data_ptr(),
                       segment_ids.data_ptr(), input_mask.data_ptr(), image_mask.data_ptr(), None,
                       task_tokens.data_ptr())
        o = L.Outputs()
        for k, t in out.items():
            setattr(o, k, t.data_ptr())
        self._call("vb200_forward_host_slot", C.byref(inp), C.byref(o), select, slot, 1 if synchronize else 0)
        return out
