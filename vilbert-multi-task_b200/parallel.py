"""Multi-GPU layer: one process per GPU, batch sharding with no data-path collective, and the single
all-gather that caption-image retrieval needs (SURVEY.md section 8e).

The reference is single-process / single-GPU (`model.cuda(0)`, worker.py:536; `distributed=False`,
worker.py:481) -- there is nothing to mirror, only the sharding the north_star asks for:

* every pair's forward is independent, except that NLVR2 consumes adjacent samples as one pair
  (`pooled.view(-1, 2048)` [UPSTREAM]; pairing visible at worker.py:266-276) -> shard on even boundaries;
* retrieval (task 7, worker.py:278-284, 359) needs the whole candidate row before its softmax/sort ->
  rank r scores a contiguous block of captions against ALL images, then ONE all-gather of the fp32
  score blocks gives every rank the full [n_captions, n_images] matrix.
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import torch
import torch.distributed as dist

from .worker_api import _prefix_len


def shard_range(n: int, rank: int, world: int, pair_aligned: bool = False) -> Tuple[int, int]:
    """Contiguous slice [lo, hi) of `n` samples for `rank`; sizes differ by at most one unit
    (a unit is 2 samples when `pair_aligned`, so an NLVR2 pair is never split across ranks)."""
    unit = 2 if pair_aligned else 1
    if pair_aligned and n % 2 != 0:
        raise ValueError("pair-aligned sharding needs an even number of samples")
    units = n // unit
    base, extra = divmod(units, world)
    lo = rank * base + min(rank, extra)
    hi = lo + base + (1 if rank < extra else 0)
    return lo * unit, hi * unit


def shard_batch(tensors: Sequence[torch.Tensor], rank: int, world: int, pair_aligned: bool = False):
    lo, hi = shard_range(tensors[0].shape[0], rank, world, pair_aligned)
    return [t[lo:hi] for t in tensors]


def all_gather_rows(local: torch.Tensor, n_total: int, group=None, comm=None) -> torch.Tensor:
    """Concatenate per-rank row blocks (block sizes from `shard_range`) into [n_total, ...] on every rank with ONE
    collective: blocks are padded to the largest block, gathered, and trimmed.  With `comm` (a `nccl_comm.NcclComm`) the
    all-gather is a raw ncclAllGather enqueued on the CURRENT CUDA stream -- the stream the engine's kernels ran on -- instead of
    a torch.distributed call (which hops to the process group's own stream, and is what the CPU / gloo tests use)."""
    if not (dist.is_available() and dist.is_initialized()):
        return local
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    sizes = [shard_range(n_total, r, world)[1] - shard_range(n_total, r, world)[0] for r in range(world)]
    assert local.shape[0] == sizes[rank], (local.shape, sizes, rank)
    m = max(sizes)
    if local.shape[0] == m:
        pad = local.contiguous()
    else:
        pad = local.new_zeros((m,) + tuple(local.shape[1:]))
        pad[: local.shape[0]] = local
    out = local.new_empty((world * m,) + tuple(local.shape[1:]))
    if comm is not None and local.is_cuda:
        comm.all_gather_f32(pad.float(), out)
    else:
        dist.all_gather_into_tensor(out, pad, group=group)
    if all(sz == m for sz in sizes):
        return out
    return torch.cat([out[r * m: r * m + sizes[r]] for r in range(world)], dim=0)


def retrieval_scores(score_pairs: Callable[[int, torch.Tensor], torch.Tensor], n_captions: int, n_images: int,
                     image_chunk: int = 64, group=None) -> torch.Tensor:
    """Full [n_captions, n_images] score matrix on every rank.

    `score_pairs(c, image_idx)` returns the vil_logit of caption `c` paired with each image in `image_idx`
    (the worker does exactly this for task 7: the text is repeated per image, worker.py:278-284, and
    `vil_logit` is read, worker.py:359).  Captions are sharded contiguously over ranks, images are walked in
    chunks of `image_chunk` pairs per forward; one all-gather at the end.
    """
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    lo, hi = shard_range(n_captions, rank, world)
    rows: List[torch.Tensor] = []
    for c in range(lo, hi):
        parts = []
        for s in range(0, n_images, image_chunk):
            idx = torch.arange(s, min(n_images, s + image_chunk))
            parts.append(score_pairs(c, idx).reshape(-1).float())
        rows.append(torch.cat(parts))
    device = rows[0].device if rows else torch.device("cpu")
    local = torch.stack(rows) if rows else torch.empty(0, n_images, device=device)
    return all_gather_rows(local, n_captions, group)


def make_pair_scorer(model, captions, images):
    """Glue for `retrieval_scores`: `captions` = (question[n_cap,T], segment_ids, input_mask), `images` =
    (features[n_img,V,F], spatials[n_img,V,5], image_mask[n_img,V]) resident on the model's device."""
    from . import _lib as L
    q, seg, im = captions
    f, s, vm = images

    def score(c: int, idx: torch.Tensor) -> torch.Tensor:
        n = idx.numel()
        idx = idx.to(f.device)
        task = torch.full((n, 1), 7, dtype=torch.long, device=f.device)
        out = model(q[c:c + 1].repeat(n, 1), f[idx], s[idx], seg[c:c + 1].repeat(n, 1), im[c:c + 1].repeat(n, 1),
                    vm[idx], None, task, select=L.OUT_VIL_LOGIT)
        return out[2]
    return score


def retrieval_scores_cached(model, captions, images, task_id: int = 7, pair_batch: int = 256, group=None, comm=None,
                            timings=None) -> torch.Tensor:
    """The same [n_captions, n_images] matrix with the reuse SURVEY.md section 7/8e describes: the caption-only part of the forward
    (embeddings + text layers ahead of the first connection layer) runs once per caption of this rank's block, the image-only
    part once per image, and only the connection layers onwards run per pair (`model.forward_cached`) -- 19 % fewer FLOPs at
    36 regions x 30 tokens, scores bit-identical to `retrieval_scores` (same kernels, same rows).  One all-gather at the end.

    `captions` = (question[n_cap, Tin], segment_ids, input_mask), `images` = (features[n_img, V, F], spatials, image_mask), on the
    model's device.  `timings` (dict) receives CUDA-event milliseconds: encode / pairs / gather."""
    from . import _lib as L
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    q, seg, im = captions
    f, s, vm = images
    n_cap, n_img = q.shape[0], f.shape[0]
    lo, hi = shard_range(n_cap, rank, world)
    dev = f.device
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timings is not None else None
    if ev:
        ev[0].record()
    task = torch.full((hi - lo, 1), task_id, dtype=torch.long, device=dev)
    vs = model.encode_image(f, s, vm)
    ts = model.encode_text(q[lo:hi], seg[lo:hi], im[lo:hi], task)
    if ev:
        ev[1].record()
    total = (hi - lo) * n_img
    padded = -(-total // pair_batch) * pair_batch            # one plan: the last chunk repeats pair 0, its scores are dropped
    flat = torch.arange(padded, dtype=torch.int64, device=dev)
    flat = torch.where(flat < total, flat, torch.zeros_like(flat))
    ci, ii = (flat // n_img).to(torch.int32), (flat % n_img).to(torch.int32)
    scores = torch.empty(padded, dtype=torch.float32, device=dev)
    for s0 in range(0, padded, pair_batch):
        out = model.forward_cached(ts, ci[s0:s0 + pair_batch], vs, ii[s0:s0 + pair_batch], select=L.OUT_VIL_LOGIT)
        scores[s0:s0 + pair_batch] = out[2].view(-1)
    local = scores[:total].view(hi - lo, n_img)
    if ev:
        ev[2].record()
    full = all_gather_rows(local, n_cap, group, comm)
    if ev:
        ev[3].record()
        torch.cuda.synchronize(dev)
        timings.update(encode_ms=ev[0].elapsed_time(ev[1]), pairs_ms=ev[1].elapsed_time(ev[2]), gather_ms=ev[2].elapsed_time(ev[3]),
                       local_captions=hi - lo, pairs=total)
    return full


def strip_padding(mask: torch.Tensor, name: str = "mask") -> List[int]:
    """Real length of every row of a padded batch: each row of `mask` must be a run of ones followed by zeros, with at least one
    one; anything else raises ValueError (packed rows are all real, so a hole in the mask cannot be represented)."""
    lens = [_prefix_len(row) for row in mask.detach().cpu()]
    bad = [i for i, k in enumerate(lens) if k is None]
    if bad:
        raise ValueError(f"{name} row {bad[0]} is not a prefix of ones")
    return lens


def pack_rows(x: torch.Tensor, lens: Sequence[int]) -> torch.Tensor:
    """The first lens[i] rows of every item of a padded [n, L, ...] tensor, back to back: [sum(lens), ...]."""
    keep = torch.arange(x.shape[1], device=x.device)[None, :] < torch.as_tensor(list(lens), device=x.device)[:, None]
    return x[keep]


def retrieval_pairs(n_captions: int, n_images: int, pair_batch: int):
    """Caption and image index (CPU int32) of every pair of an n_captions x n_images block, caption-major, padded with pair 0 to a
    multiple of `pair_batch` (one plan for every chunk; the padded pairs' scores are dropped), and the number of real pairs."""
    total = n_captions * n_images
    flat = torch.arange(-(-total // pair_batch) * pair_batch, dtype=torch.int64)
    flat = torch.where(flat < total, flat, torch.zeros_like(flat))
    return (flat // n_images).to(torch.int32), (flat % n_images).to(torch.int32), total


def retrieval_scores_packed(model, captions, images, task_id: int = 7, pair_batch: int = 256, group=None, comm=None,
                            timings=None, score: str = "vil_logit") -> torch.Tensor:
    """`retrieval_scores_cached` without padding: the same padded inputs, but every caption and image runs at its own length.
    `input_mask` and `image_mask` must have every row a prefix of ones (ValueError otherwise).  The real rows are packed, this rank's
    captions and all images are encoded once (`model.encode_text_packed` / `encode_image_packed`), and pairs are scored in chunks of
    `pair_batch` from the packed states (`model.forward_cached_packed`, one plan per chunk size).  Each score equals the
    unpadded forward of its pair; with uniform lengths and no padding it is bit-identical to `retrieval_scores_cached`.  One
    all-gather at the end.  `timings` (dict) receives CUDA-event milliseconds: encode / pairs / gather.

    `score`: "vil_logit" (default) returns the retrieval head's [n_captions, n_images] matrix; "alignment" returns the pre-training
    image-text alignment head instead (`cls.bi_seq_relationship`, the score of ViLBERT's zero-shot caption-based retrieval) as
    [n_captions, n_images, 2], both logits of each pair computed from the pair's pooled state (`model.pretraining_heads`).  Which
    column means "matched" is an upstream convention this code does not fix."""
    f, s, vm = images
    v_lens = strip_padding(vm, "image_mask")
    return _score_packed_states(model, captions, lambda: model.encode_image_packed(pack_rows(f, v_lens), pack_rows(s, v_lens), v_lens),
                                f.shape[0], task_id, pair_batch, group, comm, timings, score)


def retrieval_scores_regions(model, captions, gallery, task_id: int = 7, pair_batch: int = 256, max_boxes: int = 0, group=None,
                             comm=None, timings=None, score: str = "vil_logit") -> torch.Tensor:
    """`retrieval_scores_packed` with the gallery as the detector returns it: `gallery` = (box_features [sum n_boxes_i, F], pixel
    boxes [sum n_boxes_i, 4], image_wh [n_img, 2], n_boxes), the images' selected boxes back to back, on the model's device.  The
    gallery is encoded once with `model.encode_regions_packed` (capacity `max_boxes`, 0: the largest image), which builds each
    image's global mean row and locations on the device as `forward_regions_packed` does, so every score is bit-identical to that
    forward of its (caption, image) pair.  `captions` (padded, prefix masks), sharding, pair chunks, the all-gather and `timings`
    and `score` follow `retrieval_scores_packed`."""
    bf, bx, wh, n_boxes = gallery
    return _score_packed_states(model, captions, lambda: model.encode_regions_packed(bf, bx, wh, n_boxes, max_boxes=max_boxes),
                                len(n_boxes), task_id, pair_batch, group, comm, timings, score)


def _score_packed_states(model, captions, encode_gallery, n_img, task_id, pair_batch, group, comm, timings, score) -> torch.Tensor:
    """What the packed retrieval calls share: this rank's block of the padded `captions` (prefix masks), the gallery states of
    `encode_gallery()`, every pair scored in chunks of `pair_batch` from the packed states (`model.forward_cached_packed`; with
    score="alignment" its pooled tap through `model.pretraining_heads`), and one all-gather."""
    from . import _lib as L
    if score not in ("vil_logit", "alignment"):
        raise ValueError(f'score must be "vil_logit" or "alignment", got {score!r}')
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    q, seg, im = captions
    n_cap, dev = q.shape[0], q.device
    lo, hi = shard_range(n_cap, rank, world)
    t_lens = strip_padding(im[lo:hi], "input_mask")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timings is not None else None
    if ev:
        ev[0].record()
    task = torch.full((hi - lo, 1), task_id, dtype=torch.long, device=dev)
    vs = encode_gallery()
    ts = model.encode_text_packed(pack_rows(q[lo:hi], t_lens), pack_rows(seg[lo:hi], t_lens), task, t_lens)
    if ev:
        ev[1].record()
    ci, ii, total = retrieval_pairs(hi - lo, n_img, pair_batch)
    if score == "alignment":
        scores = torch.empty(ci.numel(), 2, dtype=torch.float32, device=dev)
        for s0 in range(0, ci.numel(), pair_batch):
            _, taps = model.forward_cached_packed(ts, ci[s0:s0 + pair_batch], vs, ii[s0:s0 + pair_batch], select=0, debug_taps=True)
            scores[s0:s0 + pair_batch] = model.pretraining_heads(taps, pair_rows=range(pair_batch))["alignment"]
        local = scores[:total].view(hi - lo, n_img, 2)
    else:
        scores = torch.empty(ci.numel(), dtype=torch.float32, device=dev)
        for s0 in range(0, ci.numel(), pair_batch):
            out = model.forward_cached_packed(ts, ci[s0:s0 + pair_batch], vs, ii[s0:s0 + pair_batch], select=L.OUT_VIL_LOGIT)
            scores[s0:s0 + pair_batch] = out[2].view(-1)
        local = scores[:total].view(hi - lo, n_img)
    if ev:
        ev[2].record()
    full = all_gather_rows(local, n_cap, group, comm)
    if ev:
        ev[3].record()
        torch.cuda.synchronize(dev)
        timings.update(encode_ms=ev[0].elapsed_time(ev[1]), pairs_ms=ev[1].elapsed_time(ev[2]), gather_ms=ev[2].elapsed_time(ev[3]),
                       local_captions=hi - lo, pairs=total)
    return full
