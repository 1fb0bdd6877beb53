"""MicroBatchWorker(source="detections") on CPU, with a stub in place of the engine: raw detector heads in, one region selection and
one packed forward per micro-batch, per-message rejections, the constructor's checks, close(), and source="features" unchanged.
The engine itself is covered by tests/test_gpu_worker_detections.py."""
import concurrent.futures as cf

import pytest
import torch

from vilbert_b200 import worker_api as W

VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "a", "dog", "on", "grass"])}


class StubDetectionModel:
    """select_regions and forward_regions_packed with the engine's layouts.  The selection keeps each image's first k = min(max_boxes,
    n) proposals (features, and boxes divided by im_scale) in its destination rows; every forward output row carries its row index."""
    _device = 0
    _dims = {"v_feature_size": 8}

    def __init__(self, max_rows_per_sample=256):
        self.max_rows_per_sample = max_rows_per_sample
        self.calls = []

    def select_regions(self, detections, max_boxes=100, conf_thresh=0.0, background=False, nms_iou=0.5, *, dst_rows=None,
                       out_rows=None, box_features=None, boxes=None, cls_prob=False, objects=False):
        k = [min(int(max_boxes), int(d[0].shape[0])) for d in detections]
        self.calls.append(dict(op="select", n=[int(d[0].shape[0]) for d in detections], C=[int(d[1].shape[1]) for d in detections],
                               max_boxes=max_boxes, dst_rows=list(dst_rows), out_rows=int(box_features.shape[0])))
        for (prop, _, feat, scale), r, kk in zip(detections, dst_rows, k):
            box_features[r:r + kk] = torch.as_tensor(feat)[:kk]
            boxes[r:r + kk] = torch.as_tensor(prop)[:kk] / scale
        return dict(box_features=box_features, boxes=boxes, n_boxes=k, dst_rows=list(dst_rows))

    def forward_regions_packed(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, select=None,
                               max_tokens=0, max_boxes=0):
        self.calls.append(dict(op="forward", question=question.clone(), segment_ids=segment_ids.clone(), task=task_tokens.clone(),
                               box_features=box_features.clone(), boxes=boxes.clone(), image_wh=image_wh.clone(),
                               n_tokens=list(n_tokens), n_boxes=list(n_boxes), select=select, max_tokens=max_tokens,
                               max_boxes=max_boxes))
        B, rv, rt = len(n_tokens), sum(n_boxes) + len(n_boxes), sum(n_tokens) + len(n_tokens)
        idx = lambda n, w: (torch.arange(n, dtype=torch.float32)[:, None] * 0.01 + torch.arange(w, dtype=torch.float32)[None] * 1e-4)
        sp = torch.rand(rv, 5, generator=torch.Generator().manual_seed(rv))
        return (idx(B, 3129), idx(B, 1533), idx(B, 1), idx(B // 2, 2) if B % 2 == 0 else idx(B, 2), idx(B, 3), None, idx(rv, 1), None,
                idx(rt, 1), []), sp


def _heads(counts, seed, Cn=11, F=8, scale=1.5):
    """Raw heads per image: proposals [n, 4] at the input scale, logits [n, C], fc6 features [n, F]."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in counts:
        xy = torch.rand(n, 2, generator=g) * 400
        out.append((torch.cat([xy, xy + 10 + torch.rand(n, 2, generator=g) * 100], 1), torch.randn(n, Cn, generator=g),
                    torch.rand(n, F, generator=g), scale))
    return out


def _message(k, task_id, counts, question, **kw):
    body = {"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": question, "socket_id": f"s{k}",
            "task_id": task_id}
    infos = [{"image_width": 640.0 + j, "image_height": 480.0} for j in range(len(counts))]
    return body, _heads(counts, seed=100 + k, **kw), infos


def _requests(msgs):
    return [(b["question"], [int(b["task_id"])], d, i, b["task_id"]) for b, d, i in msgs]


def _same_calls(a, b):
    assert [c["op"] for c in a] == [c["op"] for c in b]
    for x, y in zip(a, b):
        assert x.keys() == y.keys()
        for key in x:
            assert (torch.equal(x[key], y[key]) if torch.is_tensor(x[key]) else x[key] == y[key]), key


def _run(msgs, **kw):
    worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=300.0, **kw)
    futs = [worker.submit(*m) for m in msgs]
    for f in futs:
        f.exception(timeout=60)
    worker.close()
    return worker, futs


@pytest.fixture(autouse=True)
def _tokenizer():
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.label_maps.update(vqa=None, gqa=None)
    yield
    W.tokenizer = None


MIXED = [("1", [30], "what is the man holding?"), ("12", [50, 7], "the man is holding a dog"),
         ("7", [120, 20, 5], "a dog on the grass"), ("11", [60], "the man")]


def test_mixed_micro_batch_is_one_selection_and_one_forward():
    """VQA, an NLVR2 pair of unequal proposal counts, retrieval over three images and grounding: one select_regions and one
    forward_regions_packed, with the rows custom_prediction_detections builds for the same requests."""
    msgs = [_message(k, *m) for k, m in enumerate(MIXED)]
    W.model = StubDetectionModel()
    worker, futs = _run(msgs, source="detections")
    got = W.model.calls
    assert [c["op"] for c in got] == ["select", "forward"]
    # VQA on row 0, a filler so that the pair starts on row 2, retrieval on rows 4..6, grounding on row 7; 120 proposals keep 100
    assert got[0]["n"] == [30, 50, 7, 120, 20, 5, 60] and got[0]["max_boxes"] == 100
    assert got[0]["dst_rows"] == [0, 31, 81, 88, 188, 208, 213] and got[0]["out_rows"] == 273
    assert got[1]["n_boxes"] == [30, 1, 50, 7, 100, 20, 5, 60] and got[1]["n_tokens"] == [9, 1, 9, 9, 7, 7, 7, 4]
    assert got[1]["max_boxes"] == 100 and got[1]["max_tokens"] == W.MAX_LENGTH
    assert bool((got[1]["box_features"][30:31] == 0).all()), "the filler row keeps its zero box"
    assert torch.equal(got[1]["box_features"][81:88].cpu(), msgs[1][1][1][2])
    assert worker.batches == [7]
    W.model = StubDetectionModel()
    want = W.custom_prediction_detections(_requests(msgs), bucket=8, max_boxes=100)
    _same_calls(got, W.model.calls)
    for f, (b, _, _), a in zip(futs, msgs, want):
        assert f.result() == {"socket_id": b["socket_id"], "result": W.shape_result(b["task_id"], a, b["image_path"])}


def test_max_boxes_reaches_the_selection_and_the_plan():
    W.model = StubDetectionModel(max_rows_per_sample=512)
    _, futs = _run([_message(0, "1", [400], "what")], source="detections", max_boxes=300)
    assert futs[0].exception() is None
    assert W.model.calls[0]["max_boxes"] == 300 and W.model.calls[1]["n_boxes"][0] == 300 and W.model.calls[1]["max_boxes"] == 300


def test_bad_heads_fail_their_own_message_only():
    W.model = StubDetectionModel()
    good = [_message(0, "1", [30], "what is the man holding?"), _message(1, "11", [40], "the man"), _message(2, "7", [5, 6], "a dog")]
    bad = {"n = 2049": _message(3, "1", [2049], "what"),
           "odd F": _message(4, "1", [20], "what", F=7),
           "F = 0": _message(5, "1", [20], "what", F=0),
           "C = 1": _message(6, "1", [20], "what", Cn=1),
           "C = 2049": _message(7, "1", [20], "what", Cn=2049),
           "C of the batch": _message(8, "1", [20], "what", Cn=12),
           "F of the model": _message(9, "1", [20], "what", F=16),
           "im_scale": _message(10, "1", [20], "what", scale=0.0)}
    b, d, i = _message(11, "12", [20, 20], "the man is holding a dog")
    bad["images of one message"] = (b, [d[0], _heads([20], seed=5, Cn=12)[0]], i)
    b, d, i = _message(12, "1", [20], "what")
    bad["shapes"] = (b, [(d[0][0][:, :3], d[0][1], d[0][2], d[0][3])], i)
    msgs = good[:1] + list(bad.values()) + good[1:]
    _, futs = _run(msgs, source="detections")
    for name, f in zip(bad, futs[1:-2]):
        assert isinstance(f.exception(), ValueError), name
    for f in futs[:1] + futs[-2:]:
        assert f.exception() is None and f.result()["socket_id"] in ("s0", "s1", "s2")
    assert [c["op"] for c in W.model.calls] == ["select", "forward"]
    assert W.model.calls[0]["n"] == [30, 40, 5, 6]                  # only the good messages' images were selected


def test_a_wrong_feature_width_first_does_not_fail_the_window():
    """The feature width is the model's, not the first message's: a first message with another multiple of 4 fails alone."""
    W.model = StubDetectionModel()
    msgs = [_message(0, "1", [20], "what", F=12), _message(1, "1", [30], "what is the man holding?"), _message(2, "11", [40], "the man")]
    _, futs = _run(msgs, source="detections")
    assert isinstance(futs[0].exception(), ValueError) and "F = 8" in str(futs[0].exception())
    assert [f.result()["socket_id"] for f in futs[1:]] == ["s1", "s2"]
    assert W.model.calls[0]["n"] == [30, 40]


def test_constructor_rejections():
    W.model = StubDetectionModel()
    with pytest.raises(ValueError, match="source"):
        W.MicroBatchWorker(source="heads")
    for bad in (0, -1, 256):
        with pytest.raises(ValueError, match="max_boxes"):
            W.MicroBatchWorker(source="detections", max_boxes=bad)
    W.model = StubDetectionModel(max_rows_per_sample=512)
    with pytest.raises(ValueError, match="511"):
        W.MicroBatchWorker(source="detections", max_boxes=512)
    W.MicroBatchWorker(source="detections", max_boxes=511).close()


def test_close_cancels_queued_messages():
    W.model = StubDetectionModel()
    worker = W.MicroBatchWorker(max_rows=4, max_wait_ms=1.0, source="detections")
    worker.close()
    with pytest.raises(cf.CancelledError):
        worker.submit(*_message(0, "1", [10], "what")).result(timeout=5)
    worker = W.MicroBatchWorker(max_rows=4, max_wait_ms=1.0, source="detections")
    worker._q.put(None)                                             # a message behind the sentinel is cancelled by close() as well
    late = cf.Future()
    b, d, i = _message(1, "1", [10], "what")
    worker._q.put((b, d, i, late, []))
    worker.close()
    with pytest.raises(cf.CancelledError):
        late.result(timeout=5)
    assert W.model.calls == []


def test_source_features_is_unchanged():
    """The default source takes selected features as before: MicroBatchWorker(packed=True) makes the calls custom_prediction_packed
    makes, and no selection."""
    g = torch.Generator().manual_seed(3)
    msgs = []
    for k, (task_id, counts, q) in enumerate(MIXED):
        feats = [torch.rand(n, 8, generator=g) for n in counts]
        infos = [{"image_width": 640, "image_height": 480,
                  "bbox": (torch.rand(n, 4, generator=g) * 300).numpy()} for n in counts]
        msgs.append(({"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": q, "socket_id": f"s{k}",
                      "task_id": task_id}, feats, infos))
    W.model = StubDetectionModel()
    worker, futs = _run(msgs, packed=True)
    got = W.model.calls
    assert [c["op"] for c in got] == ["forward"] and worker.source == "features"
    W.model = StubDetectionModel()
    want = W.custom_prediction_packed(_requests(msgs), bucket=8)
    _same_calls(got, W.model.calls)
    for f, (b, _, _), a in zip(futs, msgs, want):
        assert f.result()["result"] == W.shape_result(b["task_id"], a, b["image_path"])
    assert W.MicroBatchWorker.__init__.__defaults__ == (64, 2.0, 8, False)
    assert W.MicroBatchWorker.__init__.__kwdefaults__ == {"decode": "host", "source": "features", "max_boxes": 100}
