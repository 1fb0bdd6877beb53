"""worker_api.prediction_packed on CPU with a stub in place of the engine: how requests become one packed batch (padding stripped,
offsets, NLVR2 pairs on even rows, filler rows, per-request rejections) and how the packed outputs are split back per request.
The engine side is covered by tests/test_gpu_packed.py."""
import numpy as np
import pytest
import torch

from vilbert_b200 import worker_api as W


class StubPackedModel:
    """forward_packed with the engine's output layout: per-sample outputs [B, ...], per-row outputs packed.  Each output row
    carries its row index, so a split that picks the wrong rows is visible."""
    _device = 0

    def __init__(self):
        self.calls = []

    def forward_packed(self, question, features, spatials, segment_ids, task_tokens, n_tokens, n_regions, select=None,
                       max_tokens=0, max_regions=0):
        self.calls.append(dict(question=question.clone(), segment_ids=segment_ids.clone(), task=task_tokens.clone(),
                               features=features.clone(), n_tokens=list(n_tokens), n_regions=list(n_regions), select=select,
                               max_tokens=max_tokens, max_regions=max_regions))
        B, rv, rt = len(n_tokens), sum(n_regions), sum(n_tokens) + len(n_tokens)
        idx = lambda n, w: (torch.arange(n, dtype=torch.float32)[:, None] * 0.01 + torch.arange(w, dtype=torch.float32)[None] * 1e-4)
        return (idx(B, 3129), idx(B, 1533), idx(B, 1), idx(B // 2, 2) if B % 2 == 0 else idx(B, 2), idx(B, 3), None, idx(rv, 1), None,
                idx(rt, 1), [])


def _req(task, n_img, V, words, T=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(1, T, dtype=torch.long)
    q[0, :words] = torch.randint(5, 100, (words,), generator=g)
    im = torch.zeros(1, T, dtype=torch.long)
    im[0, :words] = 1
    seg = torch.zeros(1, T, dtype=torch.long)
    seg[0, :words] = torch.arange(words) % 2
    f = torch.randn(n_img, V, 8, generator=g)
    s = torch.rand(n_img, V, 5, generator=g)
    infos = [{"image_width": 640, "image_height": 480}] * n_img
    return (q, f, s, seg, im, torch.ones(n_img, V, dtype=torch.uint8), None, torch.tensor([[int(task)]]), task, infos)


def test_packing_strips_padding_and_builds_offsets():
    W.model = StubPackedModel()
    reqs = [_req("1", 1, 5, 7, seed=1), _req("7", 3, 4, 11, seed=2), _req("13", 1, 9, 3, seed=3)]
    W.prediction_packed(reqs, bucket=8)
    assert len(W.model.calls) == 1
    c = W.model.calls[0]
    # 1 + 3 + 1 real rows, then fillers of one token and one region up to the bucket
    assert c["n_tokens"] == [7, 11, 11, 11, 3, 1, 1, 1]
    assert c["n_regions"] == [5, 4, 4, 4, 9, 1, 1, 1]
    assert c["max_tokens"] == 37 and c["max_regions"] == 9
    q = c["question"]
    assert q.numel() == sum(c["n_tokens"])
    assert torch.equal(q[:7], reqs[0][0][0, :7])                          # padding dropped, tokens back to back
    assert torch.equal(q[7:18], reqs[1][0][0, :11]) and torch.equal(q[18:29], reqs[1][0][0, :11])
    assert torch.equal(c["segment_ids"][:7], reqs[0][3][0, :7])
    assert torch.equal(c["features"][:5], reqs[0][1][0]) and torch.equal(c["features"][5:9], reqs[1][1][0])
    assert c["features"].shape[0] == sum(c["n_regions"])
    assert c["task"].view(-1).tolist() == [1, 7, 7, 7, 13, 0, 0, 0]


def test_nlvr2_pairs_on_even_rows():
    W.model = StubPackedModel()
    reqs = [_req("1", 1, 5, 7, seed=1), _req("12", 2, 6, 9, seed=2)]
    ans = W.prediction_packed(reqs, bucket=1)
    c = W.model.calls[0]
    assert c["n_tokens"] == [7, 1, 9, 9]                                   # one filler row so that the pair starts on row 2
    assert c["n_regions"] == [5, 1, 6, 6]
    assert set(ans[1]["top3_answer"]) == {"True", "False"}
    # the pair's binary logits are row 1 of the [B/2, 2] head
    out = StubPackedModel().forward_packed(c["question"], c["features"], None, c["segment_ids"], c["task"], c["n_tokens"], c["n_regions"])
    want = torch.softmax(out[3][1], dim=0).tolist()
    assert sorted(ans[1]["top3_confidence"]) == pytest.approx(sorted(want))


def test_odd_bucket_made_even_for_the_pair_head():
    W.model = StubPackedModel()
    W.prediction_packed([_req("12", 2, 4, 5)], bucket=3)
    assert len(W.model.calls[0]["n_tokens"]) == 4


def test_rejections_are_per_request():
    W.model = StubPackedModel()
    holes = _req("1", 1, 5, 7, seed=1)
    holes[4][0, 2] = 0                                                     # input_mask 1 1 0 1 ...: not a prefix
    masked = list(_req("15", 1, 5, 7, seed=2))
    masked[5] = masked[5].clone()
    masked[5][0, -1] = 0                                                   # a padded region
    bad_task = _req("1", 2, 5, 7, seed=3)                                  # VQA with two images
    good = _req("13", 1, 6, 4, seed=4)
    ans = W.prediction_packed([holes, tuple(masked), bad_task, good], bucket=2)
    assert isinstance(ans[0], ValueError) and "prefix" in str(ans[0])
    assert isinstance(ans[1], ValueError) and "image_mask" in str(ans[1])
    assert isinstance(ans[2], AssertionError)
    assert isinstance(ans[3], dict)
    assert W.model.calls[0]["n_tokens"] == [4, 1]


def test_outputs_split_back_per_request():
    W.model = StubPackedModel()
    reqs = [_req("1", 1, 5, 7, seed=1), _req("11", 1, 6, 4, seed=2), _req("7", 3, 4, 11, seed=3)]
    ans = W.prediction_packed(reqs, bucket=8)
    c = W.model.calls[0]
    out = StubPackedModel().forward_packed(c["question"], c["features"], None, c["segment_ids"], c["task"], c["n_tokens"], c["n_regions"])
    conf, idx = torch.topk(torch.softmax(out[0][0], dim=0), 3)
    assert ans[0]["top3_confidence"] == pytest.approx(conf.tolist())
    assert ans[0]["top3_answer"] == [f"<vqa:{i}>" for i in idx.tolist()]
    # grounding reads ITS OWN regions: packed rows 5..10 of vision_logit
    v = out[6][5:11].view(-1)
    conf, idx = torch.topk(torch.softmax(v, dim=0), 3)
    assert [a["confidence"] for a in ans[1]] == pytest.approx([x * 100 for x in conf.tolist()])
    boxes = reqs[1][2][0][idx][:, :4]
    assert [a["x1"] for a in ans[1]] == [int(b[0] * 640) for b in boxes.tolist()]
    # retrieval: rows 2..4 of vil_logit
    conf, idx = torch.topk(torch.softmax(out[2][2:5].view(-1), dim=0), 3)
    assert ans[2]["top3_answer"] == idx.tolist()
    assert np.allclose(ans[2]["top3_confidence"], conf.tolist())
