"""Caption-image retrieval from detector output (VILBertForVLTasks.encode_regions_packed / encode_detections_packed and
parallel.retrieval_scores_regions).  `-m gpu` only.

encode_regions_packed runs the region pack of forward_regions_packed (the same kernel at the same packed image offsets) in front of the
packed image prefix of encode_image_packed, and forward_cached_packed the same kernels on the same rows as a packed forward.  So scores
from region states are compared bit for bit with forward_regions_packed of the same (caption, image) pairs, which is what the worker
runs for a task-7 message; the fp32 oracle on the custom_prediction-built padded batch is compared at the packed tests' tolerance.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # the packed retrieval tests' tolerance against the fp32 oracle
DT = ("fp16", "bf16")
TAPS = ("sequence_output_t", "sequence_output_v", "pooled_output")
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "a", "dog", "on", "the", "grass", "man"])}


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle)


def _captions(model, lens, seed):
    """[(tokens [Tin], segments [Tin], task id)] per caption."""
    vocab = model._dims["vocab_size"]
    out = []
    for i, tin in enumerate(lens):
        g = torch.Generator().manual_seed(seed + i)
        out.append((torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g),
                    int(torch.randint(0, 20, (1,), generator=g))))
    return out


def _gallery(model, counts, seed):
    """[(box features [n, F], pixel boxes [n, 4] inside the image, image (w, h))] per image."""
    F = model._dims["v_feature_size"]
    whs = ((640.0, 480.0), (500.0, 375.0), (320.0, 240.0))
    out = []
    for i, n in enumerate(counts):
        g = torch.Generator().manual_seed(seed + 1000 + i)
        w, h = whs[i % 3]
        f = torch.relu(torch.randn(n, F, generator=g)) * 1.5
        x1, y1 = torch.rand(n, generator=g) * 0.7 * w, torch.rand(n, generator=g) * 0.7 * h
        x2 = torch.minimum(x1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * w, torch.tensor(w))
        y2 = torch.minimum(y1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * h, torch.tensor(h))
        out.append((f, torch.stack([x1, y1, x2, y2], 1), torch.tensor([w, h])))
    return out


def _encode_text(model, caps):
    cat = lambda xs: torch.cat(xs).cuda()
    return model.encode_text_packed(cat([c[0] for c in caps]), cat([c[1] for c in caps]), torch.tensor([[c[2]] for c in caps]).cuda(),
                                    [len(c[0]) for c in caps])


def _encode_gallery(model, imgs, max_boxes=0):
    cat = lambda k: torch.cat([im[k] for im in imgs]).cuda()
    return model.encode_regions_packed(cat(0), cat(1), torch.stack([im[2] for im in imgs]).cuda(), [im[0].shape[0] for im in imgs],
                                       max_boxes=max_boxes)


def _regions_pairs(model, caps, imgs, ti, ii, select):
    """forward_regions_packed of the pairs (caption ti[b], image ii[b]): the worker's forward for them."""
    pc, pi = [caps[t] for t in ti], [imgs[i] for i in ii]
    cat = lambda xs: torch.cat(xs).cuda()
    (out, taps), _ = model.forward_regions_packed(cat([c[0] for c in pc]), cat([c[1] for c in pc]), torch.tensor([[c[2]] for c in pc]).cuda(),
                                                  cat([i[0] for i in pi]), cat([i[1] for i in pi]), torch.stack([i[2] for i in pi]).cuda(),
                                                  [len(c[0]) for c in pc], [i[0].shape[0] for i in pi], select=select, debug_taps=True,
                                                  return_spatials=False)
    torch.cuda.synchronize()
    return out, taps


def _assert_same(got, want, what):
    (go, gt), (wo, wt) = got, want
    for k in range(9):
        assert (go[k] is None) == (wo[k] is None), (what, k)
        if go[k] is not None:
            assert torch.equal(go[k], wo[k]), f"{what}: output {k} differs from forward_regions_packed of the same pairs"
    for k in TAPS:
        assert torch.equal(gt[k], wt[k]), f"{what}: tap {k} differs"


# Tin 1 .. 155 (tiny max_position_embeddings is 160); boxes 1 .. 100, unequal, all below the capacity 100 but one
CAP_LENS = [1, 12, 37, 155, 9]
BOX_COUNTS = [1, 100, 37, 9, 64, 2]


@pytest.mark.parametrize("mode", DT)
def test_region_states_score_as_forward_regions_packed(tiny, mode):
    """All nine outputs (per-row outputs packed) and the three taps of forward_cached_packed on caption states and region states equal
    forward_regions_packed of the same pairs, bit for bit, with the gallery encoded at a capacity above most images' counts."""
    import vilbert_b200 as vb
    model = tiny[mode]
    caps, imgs = _captions(model, CAP_LENS, seed=1), _gallery(model, BOX_COUNTS, seed=1)
    ts, vs = _encode_text(model, caps), _encode_gallery(model, imgs, max_boxes=100)
    assert vs["offsets"].tolist()[-1] == sum(BOX_COUNTS) + len(BOX_COUNTS)
    ti, ii = [0, 4, 1, 2, 3, 0, 2], [1, 0, 5, 3, 2, 4, 1]
    got = model.forward_cached_packed(ts, torch.tensor(ti), vs, torch.tensor(ii), select=vb.OUT_ALL, debug_taps=True)
    torch.cuda.synchronize()
    _assert_same(got, _regions_pairs(model, caps, imgs, ti, ii, vb.OUT_ALL), mode)


@pytest.mark.parametrize("mode", DT)
def test_region_states_per_image_independent(tiny, mode):
    """Every image's state rows equal encode_regions_packed of that image alone (fp32 rows and 16-bit operand)."""
    model = tiny[mode]
    imgs = _gallery(model, BOX_COUNTS, seed=2)
    vs = _encode_gallery(model, imgs, max_boxes=100)
    torch.cuda.synchronize()
    vo = vs["offsets"].tolist()
    for i, im in enumerate(imgs):
        one = _encode_gallery(model, [im])
        torch.cuda.synchronize()
        assert one["offsets"].tolist() == [0, im[0].shape[0] + 1]
        assert torch.equal(vs["f32"][vo[i]:vo[i + 1]], one["f32"]), f"image {i}: fp32 rows"
        assert torch.equal(vs["h16"][vo[i]:vo[i + 1]], one["h16"]), f"image {i}: 16-bit rows"


def _heads(model, counts, seed, device="cuda"):
    from vilbert_b200 import synthetic as S
    heads = S.synthetic_detections(len(counts), counts, feature_size=model._dims["v_feature_size"], seed=seed)
    return [tuple(t.to(device) if torch.is_tensor(t) else t for t in d) for d in heads]


@pytest.mark.parametrize("mode", DT)
def test_encode_detections_equals_select_then_encode(tiny, mode):
    """encode_detections_packed == select_regions, then encode_regions_packed of the selected rows, bit for bit."""
    model = tiny[mode]
    heads = _heads(model, [60, 300, 7, 1000], seed=3)
    wh = torch.tensor([[640.0, 480.0], [500.0, 375.0], [320.0, 240.0], [800.0, 600.0]])
    got = model.encode_detections_packed(heads, wh, max_boxes=100)
    r = model.select_regions(heads, 100)
    want = _encode_gallery(model, [(r["box_features"][lo:lo + k], r["boxes"][lo:lo + k], wh[i])
                                   for i, (lo, k) in enumerate(zip(r["dst_rows"], r["n_boxes"]))], max_boxes=100)
    torch.cuda.synchronize()
    assert r["n_boxes"] == [60, 100, 7, 100]
    assert torch.equal(got["offsets"], want["offsets"])
    assert torch.equal(got["f32"], want["f32"]) and torch.equal(got["h16"], want["h16"])


def _task7_message(W, model, counts, seed):
    """A task-7 request answered by custom_prediction_detections with the device decode; returns the query's tokens, the heads, the
    image sizes, the worker's answer and the vil_logit rows of its one forward_regions_packed call."""
    heads = _heads(model, counts, seed)
    infos = [{"image_width": 640.0 + j, "image_height": 480.0 - j} for j in range(len(counts))]
    query = "a dog on the grass"
    seen = []
    orig = model.forward_regions_packed

    def spy(*a, **kw):
        res = orig(*a, **kw)
        seen.append(res[0][2].clone())
        return res
    model.forward_regions_packed = spy
    try:
        ans = W.custom_prediction_detections([(query, [7], heads, infos, "7")], decode="device")[0]
    finally:
        del model.forward_regions_packed
    torch.cuda.synchronize()
    assert len(seen) == 1
    tokens, segs = W.real_tokens(query)
    wh = torch.tensor([[i["image_width"], i["image_height"]] for i in infos])
    return tokens, segs, heads, wh, ans, seen[0][:len(counts)]


@pytest.mark.parametrize("engine", ["fp16", "bf16", "full"])
def test_task7_message_from_cached_states(request, engine):
    """A task-7 message: the caption state and the gallery encoded from the raw heads score every image exactly as the worker's
    forward (one selection, then forward_regions_packed) does, and decode_answers of those scores gives the worker's answer."""
    from vilbert_b200 import worker_api as W
    model = request.getfixturevalue("full") if engine == "full" else request.getfixturevalue("tiny")[engine]
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = model
    counts = [60, 1000, 40]
    tokens, segs, heads, wh, ans, want = _task7_message(W, model, counts, seed=700)
    ts = model.encode_text_packed(torch.tensor(tokens).cuda(), torch.tensor(segs).cuda(), torch.tensor([[7]]).cuda(), [len(tokens)])
    vs = model.encode_detections_packed(heads, wh, max_boxes=100)
    n = len(counts)
    out = model.forward_cached_packed(ts, torch.zeros(n, dtype=torch.int32), vs, torch.arange(n, dtype=torch.int32))
    torch.cuda.synchronize()
    assert torch.equal(out[2], want), "vil_logit from cached states differs from the worker's forward"
    (idx, probs, _), = model.decode_answers(out, [("7", 0, n, n, None)])
    assert idx == ans["top3_answer"] and probs == ans["top3_confidence"]


def test_full_model_bitwise_oracle_and_multi_gpu_path(full, full_oracle):
    """The 268 M model on a 5 x 8 block: bit-identical to forward_regions_packed; retrieval_scores_regions gives the same matrix; vil_logit
    within the packed tests' tolerance of the fp32 oracle on the custom_prediction-built padded batch (first 10 pairs)."""
    import vilbert_b200 as vb
    from vilbert_b200 import parallel as P
    from vilbert_b200 import worker_api as W
    caps = _captions(full, [7, 30, 12, 19, 9], seed=4)
    counts = [36, 10, 100, 57, 1, 80, 23, 99]
    imgs = _gallery(full, counts, seed=4)
    ts, vs = _encode_text(full, caps), _encode_gallery(full, imgs, max_boxes=100)
    ti = [c for c in range(5) for _ in range(8)]
    ii = [i for _ in range(5) for i in range(8)]
    got = full.forward_cached_packed(ts, torch.tensor(ti), vs, torch.tensor(ii), select=vb.OUT_TASK_HEADS, debug_taps=True)
    torch.cuda.synchronize()
    _assert_same(got, _regions_pairs(full, caps, imgs, ti, ii, vb.OUT_TASK_HEADS), "full 5 x 8")
    # the multi-GPU entry point (one process): padded captions with prefix masks, the gallery as packed box rows
    Tm = max(len(c[0]) for c in caps)
    q, seg, im = (torch.zeros(len(caps), Tm, dtype=torch.long) for _ in range(3))
    for c, (qq, sg, _) in enumerate(caps):
        q[c, :len(qq)], seg[c, :len(qq)], im[c, :len(qq)] = qq, sg, 1
    gallery = (torch.cat([i[0] for i in imgs]).cuda(), torch.cat([i[1] for i in imgs]).cuda(), torch.stack([i[2] for i in imgs]).cuda(),
               counts)
    matrix = P.retrieval_scores_regions(full, (q.cuda(), seg.cuda(), im.cuda()), gallery, task_id=caps[0][2], pair_batch=16, max_boxes=100)
    torch.cuda.synchronize()
    ts0 = full.encode_text_packed(torch.cat([c[0] for c in caps]).cuda(), torch.cat([c[1] for c in caps]).cuda(),
                                  torch.full((len(caps), 1), caps[0][2]).cuda(), [len(c[0]) for c in caps])
    same_task = full.forward_cached_packed(ts0, torch.tensor(ti), vs, torch.tensor(ii))
    torch.cuda.synchronize()
    assert torch.equal(matrix, same_task[2].view(5, 8))
    # fp32 oracle on custom_prediction's inputs, built on the host per image and padded
    n = 10
    tok = W.WordpieceTokenizer(VOCAB)
    rows = []
    for i in ii[:n]:
        f, bx, wh = imgs[i]
        info = {"image_width": float(wh[0]), "image_height": float(wh[1]), "bbox": bx.numpy()}
        _, ff, ss, _, _, _, _, _ = W.build_inputs("", [7], [f], [info], torch.device("cpu"), tok)
        rows.append((ff[0], ss[0]))
    Vm, F = max(r[0].shape[0] for r in rows), full._dims["v_feature_size"]
    Tn = max(len(caps[t][0]) for t in ti[:n])
    q, seg, im = (torch.zeros(n, Tn, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(n, Vm, F), torch.zeros(n, Vm, 5), torch.zeros(n, Vm, dtype=torch.uint8)
    for b, (t, (ff, ss)) in enumerate(zip(ti[:n], rows)):
        k, v = len(caps[t][0]), ff.shape[0]
        q[b, :k], seg[b, :k], im[b, :k] = caps[t][0], caps[t][1], 1
        f[b, :v], s[b, :v], vm[b, :v] = ff, ss, 1
    ref = full_oracle(q, f, s, seg, im, vm, None, torch.tensor([[caps[t][2]] for t in ti[:n]]))
    err = float((got[0][2][:n].cpu() - ref[2]).abs().max())
    assert err < TOL, f"vil_logit vs fp32 oracle: {err}"


def test_plan_shared_with_encode_image_packed(tiny):
    """encode_image_packed at max_regions = k + 1 and encode_regions_packed at max_boxes = k (same image count) use one plan."""
    model = tiny["fp16"]
    F = model._dims["v_feature_size"]
    k, lens = 40, [41, 3, 17, 30]
    model.encode_image_packed(torch.rand(sum(lens), F).cuda(), torch.rand(sum(lens), 5).cuda(), lens, max_regions=k + 1)
    torch.cuda.synchronize()
    n = support.n_plans(model)
    _encode_gallery(model, _gallery(model, [40, 1, 22, 7], seed=5), max_boxes=k)
    torch.cuda.synchronize()
    assert support.n_plans(model) == n


def test_back_to_back_calls(tiny):
    """Two calls on different galleries with no synchronisation in between: each state equals that call run alone."""
    model = tiny["bf16"]
    a, b = _gallery(model, [5, 77, 12], seed=6), _gallery(model, [90, 1, 33], seed=7)
    want_a = _encode_gallery(model, a, max_boxes=100)
    torch.cuda.synchronize()
    want_b = _encode_gallery(model, b, max_boxes=100)
    torch.cuda.synchronize()
    got_a = _encode_gallery(model, a, max_boxes=100)
    got_b = _encode_gallery(model, b, max_boxes=100)
    torch.cuda.synchronize()
    for got, want in ((got_a, want_a), (got_b, want_b)):
        assert torch.equal(got["f32"], want["f32"]) and torch.equal(got["h16"], want["h16"])


def test_encode_regions_packed_rejections(tiny_oracle, tiny):
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    F = model._dims["v_feature_size"]
    ok = _gallery(model, [3, 2], seed=8)
    err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: vb200_encode_regions_packed: " + pat)
    with err("image 1 has n_boxes 0"):
        model.encode_regions_packed(torch.rand(3, F), torch.rand(3, 4), torch.ones(2, 2), [3, 0])
    with err("image 0 has n_boxes 3, above the capacity max_boxes 2"):
        _encode_gallery(model, ok, max_boxes=2)
    with err("negative capacity max_boxes -1"):
        _encode_gallery(model, ok, max_boxes=-1)
    with err("capacity max_boxes 300 above 255"):
        _encode_gallery(model, ok, max_boxes=300)
    with err(r"image 0 has n_boxes 256 \(V = n_boxes \+ 1 must be <= 256\)"):
        _encode_gallery(model, _gallery(model, [256], seed=9))
    lib = L.load()
    nb = (C.c_int32 * 1)(2)
    bf, bx, wh = torch.rand(2, F, device="cuda"), torch.rand(2, 4, device="cuda"), torch.ones(1, 2, device="cuda")
    st = torch.empty(3, model._dims["v_hidden_size"], device="cuda")
    for null in range(6):
        args = [C.cast(nb, C.c_void_p), bf.data_ptr(), bx.data_ptr(), wh.data_ptr(), st.data_ptr(), st.data_ptr()]
        args[null] = None
        assert lib.vb200_encode_regions_packed(model._handle, 1, 0, *args, None) == -1
        assert b"vb200_encode_regions_packed: NULL pointer" in lib.vb200_last_error(model._handle)
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        with err("packed batches are not supported in split_fp32"):
            _encode_gallery(x, ok)
    finally:
        x.close()
