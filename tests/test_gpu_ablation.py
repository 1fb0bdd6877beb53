"""Answer ablation (vb200_answer_ablation / VILBertForVLTasks.answer_ablation).  `-m gpu` only.

Every variant is the engine's own forward of a well-defined input -- the question with one position replaced by [MASK], or the
detector output without one box -- so each variant's logits are compared bit for bit with forward_regions_packed of that input built
on the host, the scores with vb200_decode_answers on those logits, and the logits with the fp32 oracle on the same inputs at the
tolerance of tests/test_gpu_regions_packed.py.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 / bf16 vs the fp32 oracle (test_gpu_regions_packed.py)
MASK = 103
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]"])}     # the text comes from each sample itself
FAMILY_OUT = {"vqa": 0, "gqa": 1, "snli_ve": 4}          # element of the 10-tuple each family's head is


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16"))


@pytest.fixture(scope="module")
def tiny_long(tiny_oracle):
    yield from support.one_engine(tiny_oracle, compute_dtype="bf16", max_rows_per_sample=1024)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _images(model, lens, seed):
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    return [support.image(t, n, seed + i, F, vocab, ((640, 480), (500, 375))[i % 2]) for i, (t, n) in enumerate(lens)]


def _ablate(model, imgs, **kw):
    out = model.answer_ablation(*support.packed_image_args(imgs), return_logits=True, mask_token=MASK, **kw)
    torch.cuda.synchronize()
    return out


def _variant_inputs(imgs, res):
    """Every variant's input built on the host, in the engine's order: (question, segments, box features, boxes, wh, task)."""
    out = []
    for im, r in zip(imgs, res):
        q, seg, f, bx, wh, task = im
        out.append((q, seg, f, bx, wh, task))
        for p in r["tokens"]:
            qm = q.clone()
            qm[p] = MASK
            out.append((qm, seg, f, bx, wh, task))
        for j in r["boxes"]:
            keep = torch.arange(f.shape[0]) != j
            out.append((q, seg, f[keep], bx[keep], wh, task))
    return out


def _forward(model, variants, family, **kw):
    """forward_regions_packed of the host-built variants: their head rows [n, width]."""
    import vilbert_b200 as vb
    bit = {"vqa": vb.OUT_VIL_PREDICTION, "gqa": vb.OUT_VIL_PREDICTION_GQA, "snli_ve": vb.OUT_VIL_TRI_PREDICTION}[family]
    out, _ = model.forward_regions_packed(*support.packed_image_args(variants), select=bit, return_spatials=False, **kw)
    torch.cuda.synchronize()
    return out[FAMILY_OUT[family]]


def _check_bitwise(model, imgs, res, family, alone=True):
    """All variants against one host-built packed forward, and each sample's first and last variants against a forward alone."""
    variants = _variant_inputs(imgs, res)
    got = torch.cat([r["logits"] for r in res])
    assert got.shape[0] == len(variants)
    want = _forward(model, variants, family)
    for k in range(len(variants)):
        assert torch.equal(got[k], want[k]), f"variant {k} differs from forward_regions_packed of its input"
    if alone:
        k0 = 0
        for r in res:
            n = 1 + len(r["tokens"]) + len(r["boxes"])
            for k in {k0, k0 + n - 1}:
                assert torch.equal(got[k], _forward(model, [variants[k]], family)[0]), f"variant {k} differs from its forward alone"
            k0 += n
    return got


def _check_scores(model, res, family, answers):
    """scores against vb200_decode_answers on the variant logits: top-1 and its probability bit for bit, the attributed column's
    probability equal to the decode's softmax, answer -1 resolved to the unablated top-1."""
    for r, a in zip(res, answers):
        logits = r["logits"]
        n = logits.shape[0]
        top_n = min(3, logits.shape[1])
        out = [None] * 10
        out[FAMILY_OUT[family]] = logits.contiguous()
        fam = {"vqa": 1, "gqa": 2, "snli_ve": 4}[family]
        dec = model.decode_answers(out, [(fam, k, 1, top_n, None) for k in range(n)])
        base_top1 = dec[0][0][0]
        col = base_top1 if a is None else a
        assert r["answer"] == col and r["top1"] == base_top1 and r["top1_prob"] == dec[0][1][0]
        top1 = [r["top1"]] + r["token_top1"].tolist() + r["box_top1"].tolist()
        top1_prob = [r["top1_prob"]]
        probs = [r["prob"]] + r["token_prob"].tolist() + r["box_prob"].tolist()
        assert top1 == [d[0][0] for d in dec]
        for k, (idx, p, _) in enumerate(dec):
            if k == 0:
                assert top1_prob[0] == p[0]
            if col in idx:                   # the decode reports the attributed column: the same bits
                assert probs[k] == p[idx.index(col)], f"variant {k}: attributed probability"
            else:                            # below the decode's top_n: the same softmax up to the order of its sum
                sm = torch.softmax(logits[k].double(), 0)[col].item()
                assert abs(probs[k] - sm) <= 2e-5 * sm + 1e-12, f"variant {k}: attributed probability"


# (Tin, boxes): 1, 2 and 100 boxes, Tin 3 .. 37
LENS = [(3, 1), (12, 2), (37, 100), (5, 9)]


@pytest.mark.parametrize("mode", ["fp16", "bf16"])
def test_variants_bitwise_and_scores_tiny(tiny, mode):
    """Empty, full and partial ranges on mixed samples: every variant's logits equal forward_regions_packed of its input, and the
    scores equal the decode of those logits."""
    model = tiny[mode]
    imgs = _images(model, LENS, seed=11)
    tokens = [(0, 3), (1, 11), (2, 30), (0, 0)]                  # full, default-like, partial, empty
    boxes = [(0, 0), (0, 2), (10, 100), (3, 7)]                  # empty (one box), full, partial, partial
    answers = [None, 5, None, 199]
    res = _ablate(model, imgs, family="vqa", answer=answers, tokens=tokens, boxes_range=boxes)
    assert [r["tokens"] for r in res] == [list(range(*t)) for t in tokens]
    assert [r["boxes"] for r in res] == [list(range(*b)) for b in boxes]
    _check_bitwise(model, imgs, res, "vqa")
    _check_scores(model, res, "vqa", answers)


@pytest.mark.parametrize("family", ["gqa", "snli_ve"])
def test_other_families(tiny, family):
    model = tiny["bf16"]
    imgs = _images(model, [(9, 6), (20, 3)], seed=23)
    res = _ablate(model, imgs, family=family)
    assert [r["tokens"] for r in res] == [list(range(1, 8)), list(range(1, 19))]
    assert [r["boxes"] for r in res] == [list(range(6)), list(range(3))]
    _check_bitwise(model, imgs, res, family, alone=False)
    _check_scores(model, res, family, [None, None])


def test_full_model_two_samples(full):
    """The 268 M model in bf16 at the demo's shapes."""
    imgs = _images(full, [(37, 100), (14, 36)], seed=5)
    res = _ablate(full, imgs, family="vqa", tokens=[(1, 36), (1, 13)], boxes_range=[(0, 100), (0, 36)])
    _check_bitwise(full, imgs, res, "vqa", alone=False)
    _check_scores(full, res, "vqa", [None, None])


def test_past_256_rows(tiny_long):
    """An image of 300 boxes (V = 301) and a 155-token question on an engine with max_rows_per_sample 1024."""
    imgs = _images(tiny_long, [(155, 300), (4, 270)], seed=3)
    res = _ablate(tiny_long, imgs, family="vqa", tokens=[(100, 154), (1, 3)], boxes_range=[(290, 300), (0, 5)])
    _check_bitwise(tiny_long, imgs, res, "vqa", alone=False)


def test_fillers_change_nothing(tiny):
    """A call of exactly 64 variants (no fillers) and one that needs fillers give the same bits for the shared sample."""
    model = tiny["fp16"]
    imgs = _images(model, [(30, 35), (6, 4)], seed=41)
    a = _ablate(model, imgs[:1], family="vqa")                   # 1 + 28 + 35 = 64
    assert a[0]["logits"].shape[0] == 64
    b = _ablate(model, imgs, family="vqa")                       # 64 + 1 + 4 + 4 = 73 -> 128
    assert torch.equal(a[0]["logits"], b[0]["logits"])
    for k in ("answer", "prob", "top1", "top1_prob"):
        assert a[0][k] == b[0][k]
    for k in ("token_prob", "box_prob", "token_top1", "box_top1"):
        assert torch.equal(a[0][k], b[0][k])


def test_against_the_oracle(tiny, tiny_oracle):
    """Each variant's logits within the packed tests' tolerance of the fp32 oracle on the reduced, host-built inputs."""
    from vilbert_b200 import worker_api as W
    model = tiny["fp16"]
    imgs = _images(model, [(10, 5), (4, 12)], seed=17)
    res = _ablate(model, imgs, family="vqa", tokens=[(1, 9), (0, 4)])
    variants = _variant_inputs(imgs, res)
    rows = []
    for q, seg, f, bx, wh, task in variants:                      # worker.py:422-455 on the host, then padded with masks
        info = {"image_width": float(wh[0]), "image_height": float(wh[1]), "bbox": bx.numpy()}
        _, ff, ss, _, _, _, _, _ = W.build_inputs("", [task], [f], [info], torch.device("cpu"), W.WordpieceTokenizer(VOCAB))
        rows.append((ff[0], ss[0]))
    B, Tm, Vm, F = len(variants), max(len(v[0]) for v in variants), max(r[0].shape[0] for r in rows), model._dims["v_feature_size"]
    q, seg, mask = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (v, (ff, ss)) in enumerate(zip(variants, rows)):
        t = len(v[0])
        q[b, :t], seg[b, :t], mask[b, :t] = v[0], v[1], 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.tensor([[v[5]] for v in variants])
    ref = tiny_oracle(q, f, s, seg, mask, vm, None, task, compute_pretraining_heads=False)[0]
    got = torch.cat([r["logits"] for r in res]).cpu()
    err = float((got - ref).abs().max())
    assert err < TOL, f"variant logits vs fp32 oracle: {err} >= {TOL}"


def test_plans_are_shared_and_forwards_unchanged(tiny):
    """Calls with other lengths in the same bucket and capacities build no plan; forwards around a call keep their bits."""
    model = tiny["bf16"]
    imgs = _images(model, [(12, 20), (7, 9), (20, 30)], seed=61)
    fwd = lambda: _forward(model, imgs, "vqa", max_tokens=20, max_boxes=30)
    before = fwd()
    _ablate(model, imgs[:2], family="vqa", max_tokens=20, max_boxes=30)          # 1+10+20 + 1+5+9 = 46 -> 64
    n = support.n_plans(model)
    _ablate(model, imgs[1:], family="vqa", tokens=(1, 3), boxes_range=[(0, 9), (0, 20)], max_tokens=20, max_boxes=30)   # 13+23 -> 64
    assert support.n_plans(model) == n
    assert torch.equal(fwd(), before)


def test_back_to_back_calls_need_no_synchronisation(tiny):
    """Calls enqueued back to back with different inputs give what the same calls give with a synchronisation after each."""
    import vilbert_b200 as vb
    model = tiny["fp16"]
    sets = [_images(model, lens, seed=s) for s, lens in ((71, [(8, 5), (3, 2)]), (72, [(15, 40)]), (73, [(6, 3), (9, 9), (4, 2)]))]
    args = [support.packed_image_args(imgs) for imgs in sets]

    def run(sync):
        outs = []
        for a in args:
            nt, nb = a[6], a[7]
            n = sum(1 + max(0, t - 2) + (b if b >= 2 else 0) for t, b in zip(nt, nb))
            logits = torch.full((n, model._dims["num_labels"]), float("nan"), device="cuda")
            scores = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
            from vilbert_b200 import _lib as L
            msgs = (L.AblationMsg * len(nt))(*[L.AblationMsg(-1, 1, max(1, t - 1), 0, b if b >= 2 else 0) for t, b in zip(nt, nb)])
            inp = L.PackedRegionInputs(len(nt), 0, 0, vb.model._int32s(nt), vb.model._int32s(nb), a[0].data_ptr(), a[1].data_ptr(),
                                       a[2].data_ptr(), a[3].data_ptr(), a[4].data_ptr(), a[5].data_ptr(), None)
            model._call("vb200_answer_ablation", C.byref(inp), msgs, L.DECODE_VQA, MASK, logits.data_ptr(), scores.data_ptr(), 0)
            if sync:
                torch.cuda.synchronize()
            outs.append((logits, scores))
        torch.cuda.synchronize()
        return outs

    for (la, sa), (lb, sb) in zip(run(False), run(True)):
        assert torch.equal(la, lb) and torch.equal(sa, sb)


def test_rejections(tiny, tiny_oracle):
    """Every rejection is VB200_ERR_INVALID, names its cause, and leaves the sentinel-filled outputs untouched."""
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    imgs = _images(model, [(6, 3), (5, 1)], seed=81)
    a = list(support.packed_image_args(imgs))
    width = model._dims["num_labels"]
    logits = torch.full((64, width), 7.0, device="cuda")
    scores = torch.full((64, 4), 7, dtype=torch.int32, device="cuda")
    lib = L.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(m=model, msgs=None, family=L.DECODE_VQA, mask=MASK, lg=logits, nt=None, nb=None, bf=None, max_boxes=0, handle=None):
        nt, nb = nt or a[6], nb or a[7]
        msgs = msgs or [(-1, 1, 5, 0, 3), (-1, 0, 0, 0, 0)]
        arr = (L.AblationMsg * len(msgs))(*[L.AblationMsg(*x) for x in msgs])
        inp = L.PackedRegionInputs(len(nt), 0, max_boxes, vb.model._int32s(nt), vb.model._int32s(nb), a[0].data_ptr(), a[1].data_ptr(),
                                   a[2].data_ptr(), (bf if bf is not None else a[3].data_ptr()), a[4].data_ptr(), a[5].data_ptr(), None)
        h = handle or m._handle
        rc = lib.vb200_answer_ablation(h, C.byref(inp), arr, family, mask, lg.data_ptr() if lg is not None else None, scores.data_ptr(),
                                       0, stream)
        torch.cuda.synchronize()
        return rc, lib.vb200_last_error(h).decode()

    cases = [
        (dict(family=L.DECODE_NLVR2), "NLVR2"),
        (dict(family=L.DECODE_RETRIEVAL), "retrieval"),
        (dict(family=L.DECODE_GROUNDING), "grounding"),
        (dict(family=99), "unknown family"),
        (dict(msgs=[(-1, 0, 7, 0, 0), (-1, 0, 0, 0, 0)]), "sample 0 has the token range"),
        (dict(msgs=[(-1, 3, 2, 0, 0), (-1, 0, 0, 0, 0)]), "sample 0 has the token range"),
        (dict(msgs=[(-1, 0, 0, 0, 4), (-1, 0, 0, 0, 0)]), "sample 0 has the box range"),
        (dict(msgs=[(-1, 0, 0, 0, 0), (-1, 0, 0, 0, 1)]), "sample 1 drops a box"),
        (dict(mask=model._dims["vocab_size"]), "mask_token"),
        (dict(mask=-1), "mask_token"),
        (dict(msgs=[(width, 0, 0, 0, 0), (-1, 0, 0, 0, 0)]), "sample 0 has answer"),
        (dict(msgs=[(-2, 0, 0, 0, 0), (-1, 0, 0, 0, 0)]), "sample 0 has answer"),
        (dict(lg=None), "NULL"),
        (dict(lg=logits.view(-1).view(torch.uint8)[2:]), "variant_logits is not 4-byte aligned"),
        (dict(bf=a[3].data_ptr() + 4), "16-byte aligned"),
        (dict(nt=[6, 0]), "n_tokens 0"),
        (dict(nb=[3, 0]), "n_boxes 0"),
        (dict(max_boxes=2), "above the capacity"),
    ]
    for kw, match in cases:
        rc, msg = call(**kw)
        assert rc == -1 and match in msg, (kw, rc, msg)
        assert bool((logits == 7.0).all()) and bool((scores == 7).all()), kw
    # more than 1024 variants: 8 samples of 1 + 35 + 100 = 136
    big = _images(model, [(37, 100)] * 8, seed=90)
    b = support.packed_image_args(big)
    arr = (L.AblationMsg * 8)(*[L.AblationMsg(-1, 1, 36, 0, 100)] * 8)
    inp = L.PackedRegionInputs(8, 0, 0, vb.model._int32s(b[6]), vb.model._int32s(b[7]), *[t.data_ptr() for t in b[:6]], None)
    rc = lib.vb200_answer_ablation(model._handle, C.byref(inp), arr, L.DECODE_VQA, MASK, logits.data_ptr(), scores.data_ptr(), 0, stream)
    assert rc == -1 and "above 1024" in lib.vb200_last_error(model._handle).decode()
    # split_fp32 engines
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        rc, msg = call(m=x)
        assert rc == -1 and "split_fp32" in msg
    finally:
        x.close()
    assert bool((logits == 7.0).all()) and bool((scores == 7).all())


def test_pretraining_engine_is_rejected():
    from oracle import pretraining_ref as P
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    ref = P.build(P.tiny_pretraining_config(), seed=7)
    cfg = vb.BertConfig.from_dict(ref.config.to_dict())
    m = vb.BertForMultiModalPreTraining.from_pretrained(ref.state_dict(), config=cfg).eval().cuda(0)
    try:
        imgs = _images(m, [(5, 3)], seed=1)
        a = support.packed_image_args(imgs)
        arr = (L.AblationMsg * 1)(L.AblationMsg(-1, 1, 4, 0, 3))
        inp = L.PackedRegionInputs(1, 0, 0, vb.model._int32s(a[6]), vb.model._int32s(a[7]), *[t.data_ptr() for t in a[:6]], None)
        logits = torch.full((8, 4), 7.0, device="cuda")
        rc = L.load().vb200_answer_ablation(m._handle, C.byref(inp), arr, L.DECODE_VQA, MASK, logits.data_ptr(), None, 0,
                                            C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -1 and "pre-training" in L.load().vb200_last_error(m._handle).decode()
        assert bool((logits == 7.0).all())
    finally:
        m.close()
