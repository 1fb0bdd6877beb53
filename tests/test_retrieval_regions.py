"""Host logic of caption-image retrieval from detector output (parallel.retrieval_scores_regions) on a stub model: caption shard bounds,
the gallery's packed box rows and counts, the pair chunks, and the gathered matrix under a gloo world of 2.  The same stub checks that
retrieval_scores_packed makes the calls it made before its pair loop was shared.  The engine calls themselves are covered on the GPU by
tests/test_gpu_retrieval_regions.py."""
import os
import re

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vilbert_b200 import _lib as L
from vilbert_b200 import parallel as P
from vilbert_b200.model import packed_offsets
import support

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 8


class StubModel:
    """Records every engine call.  A caption's first token is its index and every box feature row of image i holds i, so the states
    carry the caption / image each packed item came from; a pair's score is table[caption, image]."""

    def __init__(self, table):
        self.table, self.calls = table, []

    def encode_text_packed(self, question, segment_ids, task_tokens, n_tokens, max_tokens=0):
        offs = packed_offsets(n_tokens)
        assert question.numel() == segment_ids.numel() == offs[-1]
        self.calls.append(("encode_text_packed", list(n_tokens), question[offs[:-1]].tolist(), task_tokens.tolist()))
        return dict(kind="text", ids=question[offs[:-1]])

    def encode_image_packed(self, features, spatials, n_regions, max_regions=0):
        offs = packed_offsets(n_regions)
        assert features.shape[0] == spatials.shape[0] == offs[-1]
        self.calls.append(("encode_image_packed", list(n_regions)))
        return dict(kind="image", ids=features[offs[:-1], 0].long())

    def encode_regions_packed(self, box_features, boxes, image_wh, n_boxes, max_boxes=0):
        offs = packed_offsets(n_boxes)
        assert box_features.shape == (offs[-1], F) and boxes.shape == (offs[-1], 4) and image_wh.shape == (len(n_boxes), 2)
        for i in range(len(n_boxes)):               # every box row of image i is at its packed offset
            assert torch.all(box_features[offs[i]:offs[i + 1]] == i)
        self.calls.append(("encode_regions_packed", list(n_boxes), max_boxes))
        return dict(kind="image", ids=box_features[offs[:-1], 0].long())

    def forward_cached_packed(self, ts, text_index, vs, image_index, select=0):
        self.calls.append(("forward_cached_packed", text_index.tolist(), image_index.tolist(), select))
        s = self.table[ts["ids"][text_index.long()], vs["ids"][image_index.long()]]
        return (None, None, s.unsqueeze(1)) + (None,) * 7


def _captions(n_cap, t_pad=6):
    """Padded captions (question, segment_ids, input_mask) with first token = caption index and 1..t_pad real tokens."""
    lens = [1 + (3 * c) % t_pad for c in range(n_cap)]
    q, seg, im = (torch.zeros(n_cap, t_pad, dtype=torch.long) for _ in range(3))
    for c, k in enumerate(lens):
        q[c, :k], im[c, :k] = torch.arange(c, c + k), 1
    return (q, seg, im), lens


def _gallery(n_img):
    n_boxes = [1 + (7 * i) % 5 for i in range(n_img)]
    bf = torch.cat([torch.full((k, F), float(i)) for i, k in enumerate(n_boxes)])
    return (bf, torch.rand(sum(n_boxes), 4), torch.full((n_img, 2), 100.0), n_boxes)


def _expected_pairs(lo, hi, n_img, pair_batch):
    ci, ii, _ = P.retrieval_pairs(hi - lo, n_img, pair_batch)
    return [("forward_cached_packed", ci[s:s + pair_batch].tolist(), ii[s:s + pair_batch].tolist(), L.OUT_VIL_LOGIT)
            for s in range(0, ci.numel(), pair_batch)]


def _check(rank, world, n_cap, n_img, pair_batch):
    """Both packed retrieval calls on this rank: the gathered matrix equals the table, and the calls are the expected ones."""
    g = torch.Generator().manual_seed(3)
    table = torch.randn(n_cap, n_img, generator=g)
    caps, t_lens = _captions(n_cap)
    lo, hi = P.shard_range(n_cap, rank, world)
    task = [[7]] * (hi - lo)
    text_call = ("encode_text_packed", t_lens[lo:hi], list(range(lo, hi)), task)
    pairs = _expected_pairs(lo, hi, n_img, pair_batch)

    m = StubModel(table)
    gallery = _gallery(n_img)
    full = P.retrieval_scores_regions(m, caps, gallery, pair_batch=pair_batch, max_boxes=6)
    assert torch.equal(full, table)
    assert m.calls == [("encode_regions_packed", gallery[3], 6), text_call] + pairs

    m = StubModel(table)
    images, v_lens = support.padded_gallery(n_img, F)
    full = P.retrieval_scores_packed(m, caps, images, pair_batch=pair_batch)
    assert torch.equal(full, table)
    assert m.calls == [("encode_image_packed", v_lens), text_call] + pairs
    return True


def _worker(rank, world, port, n_cap, n_img, pair_batch, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        try:
            ok = _check(rank, world, n_cap, n_img, pair_batch)
        except AssertionError as e:
            ok = repr(e)
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_cap,n_img,pair_batch", [(5, 6, 4), (8, 3, 8), (3, 7, 5)])
def test_retrieval_regions_gloo_world2(n_cap, n_img, pair_batch):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = support.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n_cap, n_img, pair_batch, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]


def test_retrieval_regions_single_process():
    assert _check(0, 1, 4, 5, 6)


def test_retrieval_regions_rejects_non_prefix_caption_mask():
    caps, _ = _captions(3)
    caps[2][1, 0] = 0                                  # input_mask row 1 with a hole at the front
    with pytest.raises(ValueError, match="input_mask row 1 is not a prefix of ones"):
        P.retrieval_scores_regions(StubModel(torch.zeros(3, 2)), caps, _gallery(2))


def test_encode_regions_packed_symbol_in_header_and_exports():
    hdr = open(os.path.join(ROOT, "include", "vilbert_b200.h")).read()
    m = re.search(r"int vb200_encode_regions_packed\(([^;]*)\);", hdr)
    assert m and "vb200_encode_regions_packed" in L.EXPORTS
    params = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")
    assert len(params) == len(L.load().vb200_encode_regions_packed.argtypes) == 10


def test_encode_regions_packed_rejects_null_handle():
    assert L.load().vb200_encode_regions_packed(None, 1, 0, None, None, None, None, None, None, None) == -1


def test_encode_regions_packed_needs_a_device():
    import vilbert_b200 as vb
    model = vb.VILBertForVLTasks(vb.BertConfig())
    with pytest.raises(L.VilbertB200Error, match="no CPU path"):
        model.encode_regions_packed(torch.zeros(2, 2048), torch.zeros(2, 4), torch.ones(1, 2), [2])
