"""Answer decode on the device (vb200_decode_answers[_host] / VILBertForVLTasks.decode_answers / decode="device" in the worker).
`-m gpu` only.

The kernel computes the softmax as torch.softmax(x.view(-1), 0) does, with only the summation order differing, so indices must equal
`_decode`'s exactly wherever the ranking is unambiguous, probabilities agree within 1e-6, and grounding boxes equal the reference's
int(spatial * size) on Python floats bit for bit.  Ties rank the lower index first.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

WIDTHS = {"1": 3129, "15": 1533, "12": 2, "13": 3}
DT = ("fp16", "bf16")
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "un", "##aff", "##able", ",", "a", "dog", "on", "grass"])}


@pytest.fixture(scope="module")
def eng():
    """A small engine with the worker's head widths (3129 VQA labels, 1533 GQA labels): the decode reads widths from the engine."""
    import vilbert_b200 as vb
    from vilbert_b200 import synthetic as S
    cfg = support.tiny_cfg()
    m = vb.VILBertForVLTasks.from_pretrained(S.synthetic_state_dict(cfg, num_labels=3129, gqa_labels=1533, seed=3), config=cfg,
                                             num_labels=3129).eval().cuda(0)
    yield m
    m.close()


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.engines(full_oracle, DT)


def _gapped(n, g, planted=11):
    """n logits whose `planted` largest sit at random positions with softmax gaps far above 1e-4; the rest lie well below them."""
    x = torch.rand(n, generator=g) * 3.0 - 3.0
    k = min(n, planted)
    pos = torch.randperm(n, generator=g)[:k]
    x[pos] = 4.0 - 0.25 * torch.arange(k, dtype=torch.float32)
    return x


def _outputs(**t):
    """A forward's 10-tuple with the given elements (fp32 device tensors), the rest None."""
    names = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction", "vision_prediction",
             "vision_logit", "linguisic_prediction", "linguisic_logit"]
    return tuple(t.get(n) for n in names) + ([],)


def _boundary_spatials(rows, sizes, g):
    """[rows, 5] spatials whose x / y values sit at or just below k / size in fp32, so that an fp32 product and the reference's
    double product truncate to different integers for many of them; also returns how many such values there are."""
    sp = torch.rand(rows, 5, generator=g)
    w, h = sizes
    k = torch.randint(1, 400, (rows, 4), generator=g).double()
    scale = torch.tensor([w, h, w, h], dtype=torch.float64)
    v = (k / scale).float().numpy()
    v = np.where(torch.rand(rows, 4, generator=g).numpy() < 0.5, np.nextafter(v, np.float32(0)), v)
    sp[:, :4] = torch.from_numpy(v.astype(np.float32))
    f32 = (sp[:, :4] * torch.tensor([w, h, w, h], dtype=torch.float32)).trunc().int()
    ref = (sp[:, :4].double() * scale).trunc().int()
    return sp, int((f32 != ref).sum())


def _expect(seg, n):
    """`_decode`'s ranking of one segment: softmax over the flattened logits, topk (worker_api._top)."""
    from vilbert_b200 import worker_api as W
    p = torch.softmax(seg.reshape(-1), dim=0)
    conf, idx = W._top(p, n)
    return idx, p


def test_decode_every_family_against_host(eng):
    """VQA (3129), GQA (1533), NLVR2 (2), SNLI-VE (3), retrieval with 2-10 rows and grounding with 1, 37 and 101 rows, all in one
    call: indices equal `_decode`'s ranking, probabilities within 1e-6 of torch.softmax, boxes equal int(float(s) * float(size))."""
    from vilbert_b200 import _lib as L
    g = torch.Generator().manual_seed(11)
    B = 64
    vqa = torch.stack([_gapped(3129, g) for _ in range(B)])
    gqa = torch.stack([_gapped(1533, g) for _ in range(B)])
    tri = torch.stack([_gapped(3, g) for _ in range(B)])
    binary = torch.stack([_gapped(2, g) for _ in range(B // 2)])
    vil_logit = torch.cat([_gapped(c, g) for c in range(2, 11)] + [torch.zeros(B - 54)]).view(B, 1)
    g_rows, sizes = (1, 37, 101), ((640.0, 480.0), (333.0, 517.0), (1024.0, 768.0))
    vision = torch.cat([_gapped(r, g) for r in g_rows]).view(-1, 1)
    parts = [_boundary_spatials(r, s, g) for r, s in zip(g_rows, sizes)]
    spatials = torch.cat([p[0] for p in parts])
    assert sum(p[1] for p in parts) > 0, "no spatial value separates the fp32 product from the double one"
    out = _outputs(vil_prediction=vqa.cuda(), vil_prediction_gqa=gqa.cuda(), vil_logit=vil_logit.cuda(), vil_binary_prediction=binary.cuda(),
                   vil_tri_prediction=tri.cuda(), vision_logit=vision.cuda())
    msgs, want = [], []
    for r in (0, 5, 63):
        msgs.append(("1", r, 1, 3, None)); want.append((vqa[r], 3, None))
        msgs.append(("15", r, 1, 10, None)); want.append((gqa[r], 10, None))
        msgs.append(("13", r, 1, 3, None)); want.append((tri[r], 3, None))
        msgs.append(("12", r // 2, 1, 2, None)); want.append((binary[r // 2], 2, None))
    first = 0
    for c in range(2, 11):
        msgs.append(("7", first, c, c, None)); want.append((vil_logit[first:first + c], c, None))
        first += c
    first = 0
    for r, s in zip(g_rows, sizes):
        n = min(r, 3) if r < 3 else (10 if r == 101 else 3)
        msgs.append((L.DECODE_GROUNDING, first, r, n, s)); want.append((vision[first:first + r], n, (spatials[first:first + r], s)))
        first += r
    got = eng.decode_answers(out, msgs, spatials.cuda())
    assert len(got) == len(msgs)
    for m, (idx, prob, boxes), (seg, n, grd) in zip(msgs, got, want):
        ref_idx, p = _expect(seg, n)
        assert idx == ref_idx, m
        assert max(abs(a - float(p[i])) for a, i in zip(prob, idx)) <= 1e-6, m
        if grd is None:
            assert boxes is None
            continue
        sp, (w, h) = grd
        exp = [[int(float(sp[i, 0]) * float(w)), int(float(sp[i, 1]) * float(h)), int(float(sp[i, 2]) * float(w)),
                int(float(sp[i, 3]) * float(h))] for i in idx]
        assert boxes == exp, m


def test_decode_ties_rank_lower_index_first(eng):
    """Repeated maxima: the order is numpy.argsort(-p, kind="stable"), i.e. equal probabilities by ascending index."""
    g = torch.Generator().manual_seed(5)
    vqa = torch.randint(0, 3, (16, 3129), generator=g).float()          # batch 16, as vil_logit
    vil_logit = torch.zeros(16, 1)
    vil_logit[3:7] = 1.0
    vision = torch.randint(0, 2, (40, 1), generator=g).float()
    sp = torch.rand(40, 5, generator=g)
    out = _outputs(vil_prediction=vqa.cuda(), vil_logit=vil_logit.cuda(), vision_logit=vision.cuda())
    msgs = [("1", r, 1, 10, None) for r in range(4)] + [("7", 0, 10, 10, None), ("7", 2, 8, 8, None), ("4", 0, 40, 10, (640, 480))]
    segs = [vqa[r] for r in range(4)] + [vil_logit[0:10], vil_logit[2:10], vision]
    got = eng.decode_answers(out, msgs, sp.cuda())
    for m, seg, (idx, prob, _) in zip(msgs, segs, got):
        p = torch.softmax(seg.reshape(-1), 0).numpy()
        assert idx == np.argsort(-p, kind="stable")[:m[3]].tolist(), m


# ----------------------------------------------------------------------------------------------- real forwards
def _image(tin, n, seed, F, vocab, wh):
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(1, vocab, (tin,), generator=g)
    f = torch.relu(torch.randn(n, F, generator=g)) * 1.5
    w, h = wh
    x1, y1 = torch.rand(n, generator=g) * 0.7 * w, torch.rand(n, generator=g) * 0.7 * h
    x2 = torch.minimum(x1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * w, torch.tensor(float(w)))
    y2 = torch.minimum(y1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * h, torch.tensor(float(h)))
    return q, f, torch.stack([x1, y1, x2, y2], 1), wh


# rows 0-9 of a batch: VQA, GQA, SNLI-VE, grounding, NLVR2 pair (rows 4, 5), retrieval over rows 6-9
TASK_ROWS = [("1", 0, 1), ("15", 1, 2), ("13", 2, 3), ("11", 3, 4), ("12", 4, 6), ("7", 6, 10)]
WHS = ((640, 480), (500, 375), (333, 517), (1024, 768))


def _check_forward(model, out, spatials, v_off, infos):
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    spans = {k: (lo, hi) for k, (_, lo, hi) in enumerate(TASK_ROWS)}
    tasks = {k: (t, infos[k]) for k, (t, _, _) in enumerate(TASK_ROWS)}
    msgs = W.decode_messages(tasks, spans, v_off)
    got = model.decode_answers(out, [m for _, m in msgs], spatials)
    for (k, m), (idx, prob, boxes) in zip(msgs, got):
        task_id, lo, hi = TASK_ROWS[k]
        if task_id in W.GROUNDING_TASKS:
            a, b = int(v_off[lo]), int(v_off[hi])
            seg = out[6].reshape(-1)[a:b]
            sl = _outputs(vision_logit=seg.view(1, -1, 1))
            host = W._decode(task_id, sl, spatials.reshape(-1, 5)[a:b].view(1, -1, 5), infos[k])
            assert [(d["x1"], d["y1"], d["x2"], d["y2"]) for d in host] == [tuple(b_) for b_ in boxes], task_id
        else:
            seg = out[3][lo // 2:hi // 2] if task_id == "12" else out[{"1": 0, "15": 1, "13": 4, "7": 2}[task_id]][lo:hi]
        ref_idx, p = _expect(seg, m[3])
        assert idx == ref_idx, task_id
        assert max(abs(a - float(p[i])) for a, i in zip(prob, idx)) <= 1e-6, task_id


def _infos():
    """infos of every TASK_ROWS request: one per image row it took (retrieval's N is its image count)."""
    return [[{"image_width": WHS[r % 4][0], "image_height": WHS[r % 4][1]} for r in range(lo, hi)] for _, lo, hi in TASK_ROWS]


@pytest.mark.parametrize("which", ["tiny-fp16", "tiny-bf16", "full-fp16", "full-bf16"])
def test_decode_real_forwards(which, request):
    """Dense forward_regions and packed forward_regions_packed outputs of mixed tasks and box counts, decoded on the device, match
    `_decode` on the same outputs."""
    size, dtype = which.split("-")
    model = request.getfixturevalue(size)[dtype]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    B = 10
    infos = _infos()
    # dense: every image 36 boxes, 12 tokens
    imgs = [_image(12, 36, 900 + i, F, vocab, WHS[i % 4]) for i in range(B)]
    q = torch.stack([im[0] for im in imgs]).cuda()
    ones = torch.ones_like(q)
    tk = torch.tensor([[1]] * B).cuda()
    (out, sp) = model.forward_regions(q, torch.zeros_like(q), ones, tk, torch.stack([im[1] for im in imgs]).cuda(),
                                      torch.stack([im[2] for im in imgs]).cuda(), torch.tensor([list(im[3]) for im in imgs]).float().cuda())
    torch.cuda.synchronize()
    _check_forward(model, out, sp, [k * 37 for k in range(B + 1)], infos)
    # packed: own lengths and box counts
    counts = [5, 100, 17, 63, 1, 40, 9, 77, 2, 31]
    imgs = [_image(3 + i, counts[i], 950 + i, F, vocab, WHS[i % 4]) for i in range(B)]
    out, sp = model.forward_regions_packed(torch.cat([im[0] for im in imgs]).cuda(), None, tk, torch.cat([im[1] for im in imgs]).cuda(),
                                           torch.cat([im[2] for im in imgs]).cuda(),
                                           torch.tensor([list(im[3]) for im in imgs]).float().cuda(), [len(im[0]) for im in imgs], counts)
    torch.cuda.synchronize()
    _check_forward(model, out, sp, np.concatenate([[0], np.cumsum([c + 1 for c in counts])]), infos)


# ----------------------------------------------------------------------------------------------- the worker
MESSAGES = [("1", [36], "what is the man holding?"), ("12", [20, 20], "the man is holding a dog"), ("7", [30, 30, 30], "a dog on the grass"),
            ("11", [25], "the man"), ("13", [8], "a dog"), ("15", [100], "what is the color of the dog"), ("4", [50], "a dog"),
            ("16", [12], "the grass")]


def _same(a, b):
    """Device and host answers: equal labels, indices and boxes, confidences within 1e-4 after * 100."""
    if isinstance(a, list):
        assert [{k: v for k, v in x.items() if k != "confidence"} for x in a] == [{k: v for k, v in x.items() if k != "confidence"} for x in b]
        assert list(a[0]) == list(b[0])
        assert [x["confidence"] for x in a] == pytest.approx([x["confidence"] for x in b], abs=1e-4)
    else:
        assert list(a) == list(b) and a["top3_answer"] == b["top3_answer"]
        assert [c * 100 for c in a["top3_confidence"]] == pytest.approx([c * 100 for c in b["top3_confidence"]], abs=1e-4)
        assert all(type(c) is float for c in a["top3_confidence"])


def test_worker_device_decode_matches_host(full):
    """MicroBatchWorker(packed=True, decode="device") against decode="host" on the same messages, and prediction_batch likewise."""
    from vilbert_b200 import worker_api as W
    model = full["fp16"]
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = model
    F = model._dims["v_feature_size"]
    msgs = []
    for k, (task_id, counts, q) in enumerate(MESSAGES):
        feats, infos = support.detector_output(counts, F, wh=WHS, seed=700 + k)
        body = {"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": q, "socket_id": f"s{k}", "task_id": task_id}
        msgs.append((body, feats, infos))
    res = {}
    for mode in ("host", "device"):
        worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=500.0, packed=True, decode=mode)
        futs = [worker.submit(*m) for m in msgs]
        res[mode] = [f.result(timeout=120) for f in futs]
        worker.close()
        assert len(worker.batches) == 1
    for a, b in zip(res["device"], res["host"]):
        assert a["socket_id"] == b["socket_id"] and a["result"]["task_id"] == b["result"]["task_id"]
        ra, rb = a["result"], b["result"]
        if "result" in rb:
            assert [x["answer"] for x in ra["result"]] == [x["answer"] for x in rb["result"]]
            assert [x["confidence"] for x in ra["result"]] == pytest.approx([x["confidence"] for x in rb["result"]], abs=1e-4)
        else:
            assert ra["image_name_list"] == rb["image_name_list"]
            assert ra["confidence_list"] == pytest.approx(rb["confidence_list"], abs=1e-4)
    # the answer dicts themselves: custom_prediction_packed and prediction_batch (dense), device against host
    reqs = [(q, [int(t)], *support.detector_output(c, F, wh=WHS, seed=800 + k), t) for k, (t, c, q) in enumerate(MESSAGES)]
    for a, b in zip(W.custom_prediction_packed(reqs, decode="device"), W.custom_prediction_packed(reqs, decode="host")):
        _same(a, b)
    dev = torch.device("cuda", 0)
    dense = [W.build_inputs(q, [int(t)], feats, infos, dev) + (t, infos) for q, _, feats, infos, t in reqs]
    host = W.prediction_batch(dense, decode="host")
    for a, b in zip(W.prediction_batch(dense, decode="device"), host):
        _same(a, b)
    for a, b in zip(W.prediction_packed(dense, decode="device"), W.prediction_packed(dense, decode="host")):
        _same(a, b)


# ----------------------------------------------------------------------------------------------- the C entry points
def _c_args(eng, out, msgs, spatials):
    args, _ = eng._decode_args(out, msgs, spatials)
    return args


def _answers_from(dev_bytes, n):
    from vilbert_b200 import _lib as L
    return (L.Answer * n).from_buffer_copy(dev_bytes.cpu().numpy().tobytes())


def test_decode_rejections(eng):
    """Every invalid descriptor is VB200_ERR_INVALID with a message naming the message index, before anything is enqueued: the
    answer buffer keeps its sentinel."""
    from vilbert_b200 import _lib as L
    lib = L.load()
    B, Vr = 6, 20
    full_out = _outputs(vil_prediction=torch.zeros(B, 3129, device="cuda"), vil_prediction_gqa=torch.zeros(B, 1533, device="cuda"),
                        vil_logit=torch.zeros(B, 1, device="cuda"), vil_binary_prediction=torch.zeros(B // 2, 2, device="cuda"),
                        vil_tri_prediction=torch.zeros(B, 3, device="cuda"), vision_logit=torch.zeros(Vr, 1, device="cuda"))
    sp = torch.zeros(Vr, 5, device="cuda")
    good = [("1", 0, 1, 3, None), ("4", 0, Vr, 3, (10, 10))]
    cases = [
        ((0, 0, 1, 1, None), "unknown family"), ((7, 0, 1, 1, None), "unknown family"), (("99", 0, 1, 1, None), "unknown family"),
        (("13", 0, 1, 0, None), "top_n"), (("1", 0, 1, 11, None), "top_n"), (("13", 0, 1, 4, None), "top_n"), (("7", 0, 3, 4, None), "top_n"),
        (("1", -1, 1, 3, None), "outside"), (("1", 5, 2, 3, None), "outside"), (("1", 0, 0, 3, None), "outside"),
        (("12", 3, 1, 2, None), "outside"), (("4", 10, 11, 3, (1, 1)), "outside"), (("7", 6, 1, 1, None), "outside"),
    ]
    ans = torch.full((4 * C.sizeof(L.Answer),), 0x5A, dtype=torch.uint8, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for bad, needle in cases:
        for fn in ("device", "host"):
            args = _c_args(eng, full_out, good + [bad], sp)
            if fn == "device":
                rc = lib.vb200_decode_answers(eng._handle, *args, C.c_void_p(ans.data_ptr()), stream)
            else:
                host = (L.Answer * 3)()
                rc = lib.vb200_decode_answers_host(eng._handle, *args, host, stream)
            msg = lib.vb200_last_error(eng._handle).decode()
            assert rc == -1 and "message 2" in msg and needle in msg, (bad, fn, rc, msg)
    # a NULL source for a family that is used; spatials missing for grounding
    for k, fam in ((0, "1"), (1, "15"), (2, "7"), (3, "12"), (4, "13"), (6, "4")):
        out = list(full_out)
        out[k] = None
        ok = ("13", 0, 1, 3, None) if fam != "13" else ("7", 0, 2, 2, None)
        args = _c_args(eng, tuple(out), [ok, ok, (fam, 0, 1, 1, (1, 1))], sp)
        rc = lib.vb200_decode_answers(eng._handle, *args, C.c_void_p(ans.data_ptr()), stream)
        msg = lib.vb200_last_error(eng._handle).decode()
        assert rc == -1 and "message 2" in msg and "NULL" in msg, (fam, msg)
    args = _c_args(eng, full_out, [good[0], good[0], ("11", 0, 2, 1, (1, 1))], None)
    rc = lib.vb200_decode_answers(eng._handle, *args, C.c_void_p(ans.data_ptr()), stream)
    assert rc == -1 and "message 2" in lib.vb200_last_error(eng._handle).decode() and "spatials" in lib.vb200_last_error(eng._handle).decode()
    args = list(_c_args(eng, full_out, good, sp))
    args[1] = 0
    assert lib.vb200_decode_answers(eng._handle, *args, C.c_void_p(ans.data_ptr()), stream) == -1
    assert "n must be positive" in lib.vb200_last_error(eng._handle).decode()
    with pytest.raises(L.VilbertB200Error, match="message 0 has unknown family"):
        eng.decode_answers(full_out, [("3", 0, 1, 1, None)])
    torch.cuda.synchronize()
    assert bool((ans == 0x5A).all()), "a rejected call wrote answers"


def test_decode_staging_back_to_back(eng):
    """Unsynchronised calls on one stream, each with its own descriptors and answer buffer, queued behind a long kernel so that the
    first call's descriptor copy is still pending when the second call stages its own (the third one also grows the staging buffer
    past its first 256 entries): every answer is right."""
    from vilbert_b200 import _lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(2)
    vqa = torch.stack([_gapped(3129, g) for _ in range(8)]).cuda()
    tri = torch.stack([_gapped(3, g) for _ in range(8)]).cuda()
    out = _outputs(vil_prediction=vqa, vil_tri_prediction=tri)
    calls = [[("1", r, 1, 10, None) for r in range(8)], [("13", 7 - r, 1, 3, None) for r in range(8)],
             [("1", (5 * r) % 8, 1, 1 + r % 10, None) for r in range(300)]]
    bufs = [torch.zeros(len(m) * C.sizeof(L.Answer), dtype=torch.uint8, device="cuda") for m in calls]
    torch.cuda.synchronize()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda._sleep(200_000_000)
    for m, buf in zip(calls, bufs):
        L.check(lib.vb200_decode_answers(eng._handle, *_c_args(eng, out, m, None), C.c_void_p(buf.data_ptr()), stream), eng._handle)
    torch.cuda.synchronize()
    for msgs, buf in zip(calls, bufs):
        got = _answers_from(buf, len(msgs))
        for m, a in zip(msgs, got):
            seg = (vqa if m[0] == "1" else tri)[m[1]]
            ref_idx, p = _expect(seg.cpu(), m[3])
            assert a.n == m[3] and list(a.index[:a.n]) == ref_idx, m
            assert list(a.index[a.n:]) == [-1] * (10 - a.n) and list(a.prob[a.n:]) == [0.0] * (10 - a.n)
            assert max(abs(a.prob[j] - float(p[ref_idx[j]])) for j in range(a.n)) <= 1e-6
