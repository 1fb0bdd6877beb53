"""MicroBatchWorker(source="detections") on the engine: raw detector heads in, WebSocket result dicts out.  `-m gpu` only.

Packed outputs of a sample are bit-identical whatever its batch neighbours and the plan's capacities (DESIGN.md §4.3), and the
region selection is per image and deterministic, so every message answered inside a micro-batch must equal, exactly, the same
message answered alone by custom_prediction_detections; and the answers must equal those of the host-side path the worker had
before (process_feature_extraction per message, then MicroBatchWorker(packed=True)).
"""
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "a", "dog", "on", "grass"])}
MIXED = [("1", [1000], "what is the man holding?"), ("12", [300, 80], "the man is holding a dog"),
         ("7", [60, 1000, 40], "a dog on the grass"), ("11", [500], "the man"), ("13", [37], "a dog"), ("1", [7], "what color")]


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16"))


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _worker_api(m):
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = m
    return W


def _messages(m, mix, seed, device="cpu"):
    """(body, heads, infos) per message: synthetic heads (1601 classes, the model's feature width) per image."""
    from vilbert_b200 import synthetic as S
    F = m._dims["v_feature_size"]
    msgs = []
    for k, (task_id, counts, q) in enumerate(mix):
        heads = S.synthetic_detections(len(counts), counts, feature_size=F, seed=seed + k)
        heads = [tuple(t.to(device) if torch.is_tensor(t) else t for t in d) for d in heads]
        body = {"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": q, "socket_id": f"s{k}",
                "task_id": task_id}
        msgs.append((body, heads, [{"image_width": 640.0 + j, "image_height": 480.0 - j} for j in range(len(counts))]))
    return msgs


def _serve(W, msgs, **kw):
    worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=500.0, **kw)
    futs = [worker.submit(*msg) for msg in msgs]
    for f in futs:
        f.exception(timeout=300)
    worker.close()
    return worker, futs


def _alone(W, msg, decode):
    body, heads, infos = msg
    ans = W.custom_prediction_detections([(body["question"], [int(body["task_id"])], heads, infos, body["task_id"])], decode=decode)[0]
    return {"socket_id": body["socket_id"], "result": W.shape_result(body["task_id"], ans, body["image_path"])}


@pytest.mark.parametrize("engine,decode", [("fp16", "host"), ("bf16", "device"), ("full", "host"), ("full", "device")])
def test_every_message_equals_its_own_call(request, engine, decode):
    """One micro-batch of mixed tasks, heads on the host and on the device: each result == the message alone, exactly."""
    m = request.getfixturevalue("full") if engine == "full" else request.getfixturevalue("tiny")[engine]
    W = _worker_api(m)
    msgs = _messages(m, MIXED, seed=700) + _messages(m, MIXED[:3], seed=800, device="cuda")
    worker, futs = _serve(W, msgs, source="detections", decode=decode)
    assert worker.batches == [sum(len(i) for _, _, i in msgs)]            # every message in one micro-batch
    for f, msg in zip(futs, msgs):
        assert f.result() == _alone(W, msg, decode)


@pytest.mark.parametrize("decode", ["host", "device"])
def test_answers_equal_host_selected_features(full, decode):
    """source="detections" against process_feature_extraction per message followed by MicroBatchWorker(packed=True)."""
    W = _worker_api(full)
    msgs = _messages(full, MIXED + [("15", [90], "what is the color of the dog")], seed=900, device="cuda")
    selected = []
    for body, heads, infos in msgs:
        props, scores, feats, scales = zip(*heads)
        f, inf = W.process_feature_extraction(props, scores, feats, scales, [{"width": i["image_width"], "height": i["image_height"]}
                                                                            for i in infos])
        selected.append((body, [x.cpu() for x in f], inf))
    _, want = _serve(W, selected, packed=True, decode=decode)
    _, got = _serve(W, msgs, source="detections", decode=decode)
    for g, w in zip(got, want):
        assert g.result() == w.result()


@pytest.mark.parametrize("head_device", [0, 1], ids=["model_device", "other_device"])
@pytest.mark.parametrize("decode", ["host", "device"])
def test_heads_written_on_a_side_stream(tiny, decode, head_device):
    """Heads zeroed, then written on another stream behind a ~0.5 s kernel, and submitted without synchronising: the worker's micro-batch
    is full at the last submit, so its selection is enqueued while the side stream is still sleeping, and only the stream ordering
    makes it read the written heads.  The answers equal those from heads that were synchronised first.  The caller drops its
    references right after submit (the worker's queue item holds them until the micro-batch is answered).  With heads on a second
    GPU the selection copies them to the model's device on the worker's stream of that GPU, which must wait as well."""
    if torch.cuda.device_count() <= head_device:
        pytest.skip("needs a second GPU")
    m = tiny["bf16"]
    W = _worker_api(m)
    msgs = _messages(m, MIXED, seed=1000, device=f"cuda:{head_device}")
    torch.cuda.synchronize(head_device)
    _, want = _serve(W, msgs, source="detections", decode=decode)
    want = [f.result() for f in want]
    worker = W.MicroBatchWorker(max_rows=sum(len(i) for _, _, i in msgs), max_wait_ms=500.0, source="detections", decode=decode)
    with torch.cuda.device(head_device), torch.cuda.stream(torch.cuda.Stream(head_device)):
        late = [[tuple(torch.zeros_like(t) if torch.is_tensor(t) else t for t in d) for d in heads] for _, heads, _ in msgs]
        torch.cuda._sleep(1_000_000_000)                            # ~0.5 s at 1980 MHz before the heads are written
        for lh, (_, heads, _) in zip(late, msgs):
            for d, src in zip(lh, heads):
                for t, s in zip(d[:3], src[:3]):
                    t.copy_(s)
        futs = [worker.submit(body, lh, infos) for lh, (body, _, infos) in zip(late, msgs)]
        del late, lh, d, t
    got = [f.result(timeout=300) for f in futs]
    worker.close()
    assert worker.batches == [sum(len(i) for _, _, i in msgs)]
    assert got == want


def test_bad_heads_fail_their_own_message_only(tiny):
    from vilbert_b200 import synthetic as S
    m = tiny["fp16"]
    W = _worker_api(m)
    F = m._dims["v_feature_size"]
    msgs = _messages(m, MIXED[:4], seed=1100, device="cuda")
    bad = []
    for k, (counts, C, Fb) in enumerate([([2049], 1601, F), ([20], 1601, F - 2), ([20], 1600, F), ([20], 1601, F + 4)]):
        heads = [tuple(t.cuda() if torch.is_tensor(t) else t for t in d)
                 for d in S.synthetic_detections(1, counts, n_classes=C, feature_size=Fb, seed=1200 + k)]
        bad.append(({"image_path": ["/m/demo/x.jpg"], "question": "what", "socket_id": f"b{k}", "task_id": "1"}, heads,
                    [{"image_width": 640.0, "image_height": 480.0}]))
    order = bad[3:] + msgs[:1] + bad[:3] + msgs[1:]                  # first: a feature width the model does not take
    _, futs = _serve(W, order, source="detections")
    for f, msg in zip(futs, order):
        if msg[0]["socket_id"].startswith("b"):
            assert isinstance(f.exception(), ValueError), msg[0]["socket_id"]
        else:
            assert f.result() == _alone(W, msg, "host")
