"""Packed detector-output batches (vb200_forward_regions_packed / VILBertForVLTasks.forward_regions_packed /
worker_api.custom_prediction_packed / MicroBatchWorker(packed=True)).  `-m gpu` only.

The packed region pack writes each image's operand rows exactly as the dense region pack writes them for that image alone (same
sequential fp32 mean, same conversions), and the rest of the forward is the packed forward of tests/test_gpu_packed.py.  So every
image's outputs are compared with forward_regions of that image alone bit for bit, and with the fp32 oracle on the host-built,
padded batch at the tolerances of test_gpu_packed.py.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 mode vs the fp32 oracle (test_gpu_packed.py)
DT = ("fp16", "bf16")
ROW_OUT = {5: "regions", 6: "regions", 7: "tokens", 8: "tokens"}    # per-row outputs of the 10-tuple
TAPS = ("sequence_output_t", "sequence_output_v", "pooled_output")
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "un", "##aff", "##able", ",", "a", "dog", "on", "grass"])}


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle)


def _images(model, lens, seed):
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    whs = ((640, 480), (500, 375), (320, 240))
    return [support.image(t, n, seed + i, F, vocab, whs[i % 3]) for i, (t, n) in enumerate(lens)]


def _packed(model, imgs, select, **kw):
    out = model.forward_regions_packed(*support.packed_image_args(imgs), select=select, **kw)
    torch.cuda.synchronize()
    return out


def _check_bitwise(model, imgs, packed):
    import vilbert_b200 as vb
    (out, taps), sp = packed
    B = len(imgs)
    t_rows = [len(im[0]) + model._dims["task_specific_tokens"] for im in imgs]
    v_rows = [im[2].shape[0] + 1 for im in imgs]
    for i, im in enumerate(imgs):
        (ref, rtaps), rsp = support.regions_alone(model, im, vb.OUT_ALL, debug_taps=True)
        for k in range(9):
            if k in ROW_OUT:
                got = support.split_rows(out[k], v_rows if ROW_OUT[k] == "regions" else t_rows)[i]
                want = ref[k][0]
            elif k == 3:
                if B % 2 == 0:
                    continue            # the pair head reads two images: covered by pooled_output below and the oracle test
                got, want = out[3][i], ref[3][0]
            else:
                got, want = out[k][i], ref[k][0]
            assert torch.equal(got, want), f"image {i}: output {k} differs from forward_regions of the image alone"
        assert torch.equal(support.split_rows(taps["sequence_output_t"], t_rows)[i], rtaps["sequence_output_t"][0]), f"image {i}: text tap"
        assert torch.equal(support.split_rows(taps["sequence_output_v"], v_rows)[i], rtaps["sequence_output_v"][0]), f"image {i}: image tap"
        assert torch.equal(taps["pooled_output"][i], rtaps["pooled_output"][0]), f"image {i}: pooled tap"
        assert torch.equal(support.split_rows(sp, v_rows)[i], rsp[0]), f"image {i}: spatials"


# (Tin, boxes): Tin in {1, 3, 12, 37, 155}, boxes in {1, 9, 35, 100, 255} (V = 256, the attention kernels' limit)
CORNERS = [(1, 100), (3, 1), (12, 255), (37, 9), (155, 35), (37, 255), (1, 1)]


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("B", [7, 6])
def test_regions_packed_bitwise_equals_regions_per_image(tiny, mode, B):
    """All nine outputs, the three taps and the spatials rows of every image equal forward_regions of that image alone, bit for bit."""
    import vilbert_b200 as vb
    model = tiny[mode]
    imgs = _images(model, CORNERS[:B], seed=50 + B)
    _check_bitwise(model, imgs, _packed(model, imgs, vb.OUT_ALL, debug_taps=True))


def _host_batch(imgs, tok_lens, F):
    """worker.py:422-455 on the host (worker_api.build_inputs) per image, padded to a common (Tin, V) with masks."""
    from vilbert_b200 import worker_api as W
    rows, tok = [], W.WordpieceTokenizer(VOCAB)
    for im in imgs:                                  # the image half of build_inputs (the text comes from the image row itself)
        _, _, f, bx, wh, task = im
        info = {"image_width": float(wh[0]), "image_height": float(wh[1]), "bbox": bx.numpy()}
        _, ff, ss, _, _, _, _, _ = W.build_inputs("", [task], [f], [info], torch.device("cpu"), tok)
        rows.append((ff[0], ss[0]))
    B, Tm, Vm = len(imgs), max(tok_lens), max(r[0].shape[0] for r in rows)
    q, seg, mask = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (im, (ff, ss)) in enumerate(zip(imgs, rows)):
        t = len(im[0])
        q[b, :t], seg[b, :t], mask[b, :t] = im[0], im[1], 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    return q, f, s, seg, mask, vm, torch.tensor([[im[5]] for im in imgs])


def test_regions_packed_full_model_bitwise_and_oracle(full_oracle, full):
    """The 268 M model with 8 images of detector-like box counts (10..100) and worker-like question lengths: bit-identical per image
    to forward_regions of the image alone, and within the packed tests' tolerance of the fp32 oracle on the host-built padded batch."""
    import vilbert_b200 as vb
    lens = [(9, 36), (30, 100), (14, 10), (37, 63), (7, 99), (22, 17), (5, 12), (28, 72)]
    imgs = _images(full, lens, seed=7)
    packed = _packed(full, imgs, vb.OUT_ALL, debug_taps=True)
    _check_bitwise(full, imgs, packed)
    (out, _), _ = packed
    q, f, s, seg, mask, vm, task = _host_batch(imgs, [t for t, _ in lens], full._dims["v_feature_size"])
    ref = full_oracle(q, f, s, seg, mask, vm, None, task, compute_pretraining_heads=False)
    for k in (0, 1, 2, 3, 4, 6, 8):                 # the task heads
        if ref[k] is None:
            continue
        if k in ROW_OUT:
            per = [r[:(t + 1) if ROW_OUT[k] == "tokens" else n + 1] for r, (t, n) in zip(ref[k], lens)]
            want = torch.cat(per, dim=0).reshape(out[k].shape)
        else:
            want = ref[k]
        err = float((out[k].cpu() - want).abs().max())
        assert err < TOL, f"output {k} vs fp32 oracle: {err} >= {TOL}"


def test_regions_packed_spatials_match_host_construction(tiny):
    import vilbert_b200 as vb
    model = tiny["fp16"]
    lens = [(5, 20), (9, 1), (3, 57), (12, 8)]
    imgs = _images(model, lens, seed=31)
    _, sp = _packed(model, imgs, vb.OUT_VIL_PREDICTION)
    _, _, s, _, _, vm, _ = _host_batch(imgs, [t for t, _ in lens], model._dims["v_feature_size"])
    want = torch.cat([s[b, :n + 1] for b, (_, n) in enumerate(lens)])
    assert sp.shape == (sum(n + 1 for _, n in lens), 5)
    assert float((sp.cpu() - want).abs().max()) < 1e-6


def test_regions_packed_shares_the_packed_plan(tiny):
    """At fixed capacities (37 tokens, 100 boxes) calls with different lengths share one plan, and forward_packed at the same
    capacities (101 regions) uses that plan too."""
    import vilbert_b200 as vb
    model = tiny["fp16"]
    sel = vb.OUT_TASK_HEADS
    cap = dict(max_tokens=37, max_boxes=100)
    _packed(model, _images(model, [(3, 10), (20, 99), (37, 1), (8, 40)], seed=61), sel, **cap)
    n = support.n_plans(model)
    _packed(model, _images(model, [(1, 2), (5, 5), (12, 7), (2, 3)], seed=62), sel, **cap)
    assert support.n_plans(model) == n
    F = model._dims["v_feature_size"]
    model.forward_packed(torch.ones(4 * 6, dtype=torch.long).cuda(), torch.rand(4 * 30, F).cuda(), torch.rand(4 * 30, 5).cuda(), None,
                         torch.zeros(4, 1, dtype=torch.long).cuda(), [6] * 4, [30] * 4, select=sel, max_tokens=37, max_regions=101)
    torch.cuda.synchronize()
    assert support.n_plans(model) == n


def test_regions_packed_rejections(tiny_oracle, tiny):
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    sel = vb.OUT_TASK_HEADS
    ok = _images(model, [(5, 3), (4, 2)], seed=71)
    err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: .*" + pat)
    with err("VB200_OUT_ATTENTION"):
        _packed(model, ok, sel | L.OUT_ATTENTION)
    with err("image 1 has n_boxes 0"):
        F = model._dims["v_feature_size"]
        model.forward_regions_packed(torch.ones(9, dtype=torch.long), None, torch.zeros(2, 1, dtype=torch.long), torch.rand(3, F),
                                     torch.rand(3, 4), torch.ones(2, 2), [5, 4], [3, 0])
    with err("n_boxes 3, above the capacity max_boxes 2"):
        _packed(model, ok, sel, max_boxes=2)
    with err("n_boxes 256"):
        _packed(model, _images(model, [(5, 256)], seed=72), sel)
    with err("n_tokens 256"):
        _packed(model, _images(model, [(256, 3)], seed=73), sel)
    with err("n_tokens 200 > max_position_embeddings"):
        _packed(model, _images(model, [(200, 3)], seed=74), sel)
    with err("n_tokens 5, above the capacity"):
        _packed(model, ok, sel, max_tokens=4)
    with err("negative capacity max_tokens"):
        _packed(model, ok, sel, max_tokens=-1)
    with err("negative capacity max_boxes"):
        _packed(model, ok, sel, max_boxes=-1)
    with err("max_boxes 300"):
        _packed(model, ok, sel, max_boxes=300)
    # a NULL required pointer (box features), through the C ABI directly
    nt, nb = (C.c_int32 * 1)(3), (C.c_int32 * 1)(2)
    q = torch.ones(3, dtype=torch.long, device="cuda")
    tk = torch.zeros(1, 1, dtype=torch.long, device="cuda")
    bx, wh = torch.rand(2, 4, device="cuda"), torch.ones(1, 2, device="cuda")
    inp = L.PackedRegionInputs(1, 0, 0, C.cast(nt, C.c_void_p), C.cast(nb, C.c_void_p), q.data_ptr(), q.data_ptr(), tk.data_ptr(), None,
                               bx.data_ptr(), wh.data_ptr(), None)
    o = L.Outputs()
    assert L.load().vb200_forward_regions_packed(model._handle, C.byref(inp), C.byref(o), sel, 0, None) == -1
    assert b"vb200_packed_region_inputs has a NULL required pointer" in L.load().vb200_last_error(model._handle)
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        with err("fp32x"):
            _packed(x, ok, sel)
    finally:
        x.close()


# ----------------------------------------------------------------------------------------------- the worker on the engine
def _same_answer(a, b):
    """The tolerances of test_gpu_round2.py: same labels / boxes, confidences within 5e-3 (boxes: 0.5 percentage points)."""
    if isinstance(a, list):
        assert [(x["x1"], x["y1"], x["x2"], x["y2"]) for x in a] == [(x["x1"], x["y1"], x["x2"], x["y2"]) for x in b]
        assert [x["confidence"] for x in a] == pytest.approx([x["confidence"] for x in b], abs=0.5)
    else:
        assert a["top3_answer"] == b["top3_answer"]
        assert a["top3_confidence"] == pytest.approx(b["top3_confidence"], abs=5e-3)


def test_custom_prediction_packed_matches_custom_prediction(full):
    """One engine call for VQA, NLVR2, retrieval (images with unequal box counts), RefCOCO, SNLI-VE and GQA plus one invalid request:
    every answer matches custom_prediction of that request alone, and the invalid one gets its exception."""
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = full
    F = full._dims["v_feature_size"]
    reqs = []
    for k, (task_id, counts, q) in enumerate([("1", [36], "what is the man holding?"), ("12", [20, 33], "the man is holding a dog"),
                                               ("7", [20, 11, 57], "a dog on the grass"), ("11", [45], "the man"),
                                               ("13", [10], "a dog"), ("15", [100], "what is the color of the dog")]):
        feats, infos = support.detector_output(counts, F, seed=300 + k)
        reqs.append((q, [int(task_id)], feats, infos, task_id))
    bad_feats, bad_infos = support.detector_output([5, 5], F, seed=399)
    reqs.insert(3, ("what", [1], bad_feats, bad_infos, "1"))          # VQA with two images
    calls = []
    orig = full.forward_regions_packed

    def counted(*a, **kw):
        calls.append(1)
        return orig(*a, **kw)
    full.forward_regions_packed = counted
    try:
        got = W.custom_prediction_packed(reqs)
    finally:
        del full.forward_regions_packed
    assert len(calls) == 1
    assert isinstance(got[3], AssertionError)
    for r, ans in zip(reqs, got):
        if r is reqs[3]:
            continue
        _same_answer(ans, W.custom_prediction(*r))


def test_micro_batch_worker_packed_on_engine(full):
    """MicroBatchWorker(packed=True): every pending message in one forward, a retrieval message with unequal box counts included
    (the dense worker's torch.stack cannot take it), every result equal to handle_request() of that message alone."""
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = full
    F = full._dims["v_feature_size"]
    msgs = []
    for k, (task_id, counts, q) in enumerate([("1", [36], "what is the man holding?"), ("12", [20, 20], "the man is holding a dog"),
                                               ("7", [30, 12, 64], "a dog on the grass"), ("11", [25], "the man"), ("13", [8], "a dog"),
                                               ("15", [100], "what is the color of the dog")]):
        feats, infos = support.detector_output(counts, F, seed=600 + k)
        body = {"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": q, "socket_id": f"s{k}", "task_id": task_id}
        msgs.append((body, feats, infos))
    want = [W.handle_request(*m) for m in msgs]
    worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=500.0, packed=True)
    futs = [worker.submit(*m) for m in msgs]
    res = [f.result(timeout=120) for f in futs]
    worker.close()
    assert len(worker.batches) == 1 and worker.batches[0] == 9          # all six messages shared one forward (9 images)
    for r, w, m in zip(res, want, msgs):
        assert r["socket_id"] == m[0]["socket_id"] and r["result"]["task_id"] == w["task_id"]
        if "result" in w:
            assert [x["answer"] for x in r["result"]["result"]] == [x["answer"] for x in w["result"]]
            assert [x["confidence"] for x in r["result"]["result"]] == pytest.approx([x["confidence"] for x in w["result"]], abs=0.3)
        else:
            assert r["result"]["image_name_list"] == w["image_name_list"]
            assert r["result"]["confidence_list"] == pytest.approx(w["confidence_list"], abs=0.3)
