"""BertForMultiModalPreTraining on the engine (vb200_create_pretraining) and the pre-training objectives on the device
(vb200_pretraining_objectives).  `-m gpu` only.

The pre-training checkpoint has the encoder and the `cls` heads and no task heads, and its config has task_specific_tokens off (no
other suite builds an engine with the flag off).  The no-label forward is checked against the fp32 oracle (oracle/pretraining_ref.py)
and row by row, bit for bit, against vb200_pretraining_heads on the same taps; the packed, detector-output and cached forwards
against dense forwards of each sample alone.  The objectives are checked against fp64 torch on the engine's own logits and against the
oracle's losses.
"""
import contextlib
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import support

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16", "fp32x")
TOL = {"fp16": 1e-2, "bf16": 3.5e-2, "fp32x": 1e-3}     # vs the fp32 oracle; bf16 x max(1, logit std), as tests/test_gpu_model.py
TOL_LOSS = {"fp16": 1e-2, "bf16": 3.5e-2, "fp32x": 1e-3}
KEYS = ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")
LABELS = ("masked_lm_labels", "image_label", "image_target", "next_sentence_label")


def _both():
    L = support.lib()
    return L.OUT_LINGUISIC_PREDICTION | L.OUT_VISION_PREDICTION


@pytest.fixture(scope="module")
def pt_oracle():
    from oracle import pretraining_ref as P
    return P.build(P.tiny_pretraining_config(), seed=7)


@pytest.fixture(scope="module")
def tiny(pt_oracle):
    import vilbert_b200 as vb
    yield from support.engines(pt_oracle, MODES, vb.BertForMultiModalPreTraining)


@pytest.fixture(scope="module")
def full_pt():
    from oracle import pretraining_ref as P
    import vilbert_b200 as vb
    oracle = P.build(seed=42)
    with contextlib.closing(support.engine(oracle, vb.BertForMultiModalPreTraining, compute_dtype="bf16")) as m:
        yield oracle, m


def _batch(model, B, Tin, V, seed):
    from vilbert_b200 import synthetic as S
    d = model._dims
    b = S.synthetic_masked_batch(B, Tin, V, seed=seed, vocab_size=d["vocab_size"], v_feature_size=d["v_feature_size"],
                                 v_target_size=d["v_target_size"])
    return b


def _dense(model, inputs, select):
    """VILBertForVLTasks.forward on the pre-training engine: (10-tuple, taps)."""
    import vilbert_b200 as vb
    return vb.VILBertForVLTasks.forward(model, *[t.cuda() for t in inputs], None, None, select=select, debug_taps=True)


def _err(a, r):
    return float((a.cpu() - r).abs().max())


# ------------------------------------------------------------------ engine flags
def test_engine_dims(tiny):
    L = support.lib()
    for m in tiny.values():
        assert m._dims["task_specific_tokens"] == 0 and m._dims["num_labels"] == 0 and m._dims["gqa_labels"] == 0
        v = C.c_int64()
        assert L.load().vb200_model_dim(m._handle, b"gqa_labels", C.byref(v)) == 0 and v.value == 0


# ------------------------------------------------------------------ the no-label forward
def _check_no_label_forward(oracle, model, mode, B, Tin, V, seed):
    from oracle import vilbert_ref as R
    b = _batch(model, B, Tin, V, seed)
    inp = [b[k] for k in KEYS]
    t, v, align, attn = model(*[x.cuda() for x in inp])
    out, taps = _dense(model, inp, _both())
    torch.cuda.synchronize()
    assert attn == [] and t.shape == (B, Tin, model._dims["vocab_size"]) and v.shape == (B, V, model._dims["v_target_size"])
    assert align.shape == (B, 2)
    assert torch.equal(t, out[7]) and torch.equal(v, out[5])
    # every row equals vb200_pretraining_heads on the same taps, bit for bit
    heads = model.pretraining_heads(taps, text_rows=range(B * Tin), image_rows=range(B * V), pair_rows=range(B))
    torch.cuda.synchronize()
    assert torch.equal(heads["token_logits"], t.reshape(B * Tin, -1))
    assert torch.equal(heads["region_logits"], v.reshape(B * V, -1))
    assert torch.equal(heads["alignment"], align)
    ref = oracle(*inp)
    for name, got, r in (("prediction_scores_t", t, ref[0]), ("prediction_scores_v", v, ref[1]), ("seq_relationship", align, ref[2])):
        tol = TOL[mode] * (max(1.0, float(r.std())) if mode == "bf16" else 1.0)
        err = _err(got, r)
        print(f"PARITY pretraining forward {mode} {name}: max abs err {err:.3e} (std {float(r.std()):.3f})")
        assert err < tol, (mode, name, err, tol)
    return b, out, taps


@pytest.mark.parametrize("mode", MODES)
def test_no_label_forward_matches_oracle_and_rows(tiny, pt_oracle, mode):
    _check_no_label_forward(pt_oracle, tiny[mode], mode, 3, 24, 11, seed=1)


def test_full_model_no_label_forward(full_pt):
    oracle, model = full_pt
    _check_no_label_forward(oracle, model, "bf16", 2, 36, 37, seed=2)


def test_attention_maps_on_pretraining_engine(tiny):
    model = tiny["fp16"]
    model.return_attention = True
    try:
        b = _batch(model, 2, 12, 7, seed=3)
        _, _, _, attn = model(*[b[k].cuda() for k in KEYS], output_all_attention_masks=True)
        torch.cuda.synchronize()
        assert len(attn) > 0
    finally:
        model.return_attention = False


# ------------------------------------------------------------------ packed, detector-output and cached forwards
def _alone(model, q, f, s, seg):
    """Dense batch-1 forward of one sample at its own lengths: token / region logits and the alignment of its pooled tap."""
    ones_t = torch.ones(1, q.numel(), dtype=torch.long)
    ones_v = torch.ones(1, f.shape[0], dtype=torch.uint8)
    out, taps = _dense(model, [q[None], f[None], s[None], seg[None], ones_t, ones_v], _both())
    return out[7][0], out[5][0], model.pretraining_heads(taps, pair_rows=[0])["alignment"]


def _packed_inputs(model, nt, nv, seed):
    g = torch.Generator().manual_seed(seed)
    vocab, Fd = model._dims["vocab_size"], model._dims["v_feature_size"]
    return (torch.randint(1, vocab, (sum(nt),), generator=g), torch.relu(torch.randn(sum(nv), Fd, generator=g)),
            torch.rand(sum(nv), 5, generator=g), torch.randint(0, 2, (sum(nt),), generator=g))


def _check_per_sample(model, out, taps, alone, nt, nv):
    heads = model.pretraining_heads(taps, pair_rows=range(len(nt)))
    torch.cuda.synchronize()
    t0 = v0 = 0
    for i, (tl, vl, al) in enumerate(alone):
        assert torch.equal(out[7][t0:t0 + nt[i]], tl), ("token", i)
        assert torch.equal(out[5][v0:v0 + nv[i]], vl), ("region", i)
        assert torch.equal(heads["alignment"][i:i + 1], al), ("alignment", i)
        t0, v0 = t0 + nt[i], v0 + nv[i]


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_packed_and_cached_packed_per_sample(tiny, mode):
    model = tiny[mode]
    nt, nv = [20, 7, 33], [12, 30, 5]
    q, f, s, seg = _packed_inputs(model, nt, nv, 4)
    offs_t, offs_v = [0, 20, 27, 60], [0, 12, 42, 47]
    alone = [_alone(model, q[offs_t[i]:offs_t[i + 1]], f[offs_v[i]:offs_v[i + 1]], s[offs_v[i]:offs_v[i + 1]],
                    seg[offs_t[i]:offs_t[i + 1]]) for i in range(3)]
    out, taps = model.forward_packed(q.cuda(), f.cuda(), s.cuda(), seg.cuda(), None, nt, nv, select=_both(), debug_taps=True)
    _check_per_sample(model, out, taps, alone, nt, nv)
    ts = model.encode_text_packed(q.cuda(), seg.cuda(), torch.zeros(3, 1, dtype=torch.long), nt)
    vs = model.encode_image_packed(f.cuda(), s.cuda(), nv)
    idx = torch.arange(3, dtype=torch.int32)
    out, taps = model.forward_cached_packed(ts, idx, vs, idx, select=_both(), debug_taps=True)
    _check_per_sample(model, out, taps, alone, nt, nv)


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_regions_packed_per_sample(tiny, mode):
    model = tiny[mode]
    nt, nb = [15, 40], [9, 22]
    g = torch.Generator().manual_seed(5)
    Fd = model._dims["v_feature_size"]
    q = torch.randint(1, model._dims["vocab_size"], (sum(nt),), generator=g)
    seg = torch.zeros(sum(nt), dtype=torch.long)
    bf = torch.relu(torch.randn(sum(nb), Fd, generator=g))
    x1, y1 = torch.rand(sum(nb), generator=g) * 300, torch.rand(sum(nb), generator=g) * 200
    bx = torch.stack([x1, y1, x1 + 30, y1 + 40], 1)
    wh = torch.tensor([[640.0, 480.0], [500.0, 400.0]])
    (out, taps), _ = model.forward_regions_packed(q.cuda(), seg.cuda(), None, bf.cuda(), bx.cuda(), wh.cuda(), nt, nb,
                                                  select=_both(), debug_taps=True)
    alone = []
    for i in range(2):
        ts = slice(sum(nt[:i]), sum(nt[:i + 1]))
        vs = slice(sum(nb[:i]), sum(nb[:i + 1]))
        # the dense detector-output forward of the image alone for the logits, the batch-1 packed one for its pooled tap
        o1, _ = model.forward_regions(q[ts][None], seg[ts][None], torch.ones(1, nt[i], dtype=torch.long),
                                      torch.zeros(1, 1, dtype=torch.long), bf[vs][None], bx[vs][None], wh[i:i + 1], select=_both())
        (_, tp), _ = model.forward_regions_packed(q[ts].cuda(), seg[ts].cuda(), None, bf[vs].cuda(), bx[vs].cuda(), wh[i:i + 1].cuda(),
                                                  [nt[i]], [nb[i]], select=0, debug_taps=True)
        alone.append((o1[7][0], o1[5][0], model.pretraining_heads(tp, pair_rows=[0])["alignment"]))
    _check_per_sample(model, out, taps, alone, nt, [n + 1 for n in nb])


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_dense_cached_matches_dense(tiny, mode):
    model = tiny[mode]
    b = _batch(model, 2, 16, 9, seed=6)
    ref, _ = _dense(model, [b[k] for k in KEYS], _both())
    ts = model.encode_text(b["input_ids"].cuda(), b["token_type_ids"].cuda(), b["attention_mask"].cuda(), torch.zeros(2, 1, dtype=torch.long))
    vs = model.encode_image(b["image_feat"].cuda(), b["image_loc"].cuda(), b["image_attention_mask"].cuda())
    idx = torch.arange(2, dtype=torch.int32)
    out = model.forward_cached(ts, idx, vs, idx, select=_both())
    torch.cuda.synchronize()
    assert torch.equal(out[7], ref[7]) and torch.equal(out[5], ref[5])


# ------------------------------------------------------------------ the objectives
def _torch_losses(tl, rl, pl, token_labels, targets, pair_labels):
    """fp64 per-row losses on the engine's own logits."""
    ce_t = F.cross_entropy(tl.double(), token_labels.long(), reduction="none")
    kl = F.kl_div(F.log_softmax(rl.double(), dim=1), targets.double(), reduction="none").sum(1)
    ce_p = F.cross_entropy(pl.double(), pair_labels.long(), reduction="none")
    return ce_t, kl, ce_p


def _rel(a, b):
    return float(((a.double() - b).abs() / b.abs().clamp(min=1e-6)).max()) if b.numel() else 0.0


def _targets(n, vt, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.softmax(torch.randn(n, vt, generator=g) * 2, 1) * (torch.rand(n, vt, generator=g) > 0.3)
    t[0] = 0.0
    t[0, vt - 1] = 1.0                                           # a one-hot target
    return (t / t.sum(1, keepdim=True)).cuda()


@pytest.mark.parametrize("mode", MODES)
def test_objectives_per_row_and_reduced(tiny, mode):
    model = tiny[mode]
    B, Tin, V = 3, 60, 50
    b = _batch(model, B, Tin, V, seed=7)
    _, taps = _dense(model, [b[k] for k in KEYS], 0)
    vocab, vt = model._dims["vocab_size"], model._dims["v_target_size"]
    tr = [0, 127, 128, B * Tin - 1, 5, 5, 64]
    vr = [0, 127, 128, B * V - 1, 3, 3]
    pr = [0, 2, 1, 1]
    tlab = torch.tensor([0, vocab - 1, 5, 17, 3, 3, vocab // 2], dtype=torch.int32)
    plab = torch.tensor([0, 1, 1, 0], dtype=torch.int32)
    tg = _targets(len(vr), vt, 8)
    res = model.pretraining_objectives(taps, text_rows=tr, token_labels=tlab, image_rows=vr, image_targets=tg, pair_rows=pr,
                                       pair_labels=plab)
    heads = model.pretraining_heads(taps, text_rows=tr, image_rows=vr, pair_rows=pr)
    torch.cuda.synchronize()
    ce_t, kl, ce_p = _torch_losses(heads["token_logits"], heads["region_logits"], heads["alignment"], tlab.cuda(), tg, plab.cuda())
    for name, got, ref in (("token", res["token_loss"], ce_t), ("region", res["region_loss"], kl), ("pair", res["pair_loss"], ce_p)):
        assert _rel(got, ref) < 1e-5, (mode, name, _rel(got, ref))
    assert float(res["token_loss"][4]) == float(res["token_loss"][5])          # duplicates
    for key, ref in (("masked_lm_loss", ce_t.mean()), ("masked_img_loss", kl.mean()), ("next_sentence_loss", ce_p.mean())):
        assert res[key].shape == (1,) and abs(float(res[key]) - float(ref)) <= 1e-5 * abs(float(ref)), (mode, key)


@pytest.mark.parametrize("mode", MODES)
def test_forward_with_labels_matches_torch_and_oracle(tiny, pt_oracle, mode):
    from oracle import pretraining_ref as P
    model = tiny[mode]
    B, Tin, V = 4, 36, 37
    b = _batch(model, B, Tin, V, seed=9)
    lm, img, nsp = model(*[b[k].cuda() for k in KEYS], *[b[k].cuda() for k in LABELS])
    t, v, align, _ = model(*[b[k].cuda() for k in KEYS])
    torch.cuda.synchronize()
    labels = [b[k] for k in LABELS]
    # torch's CrossEntropyLoss(ignore_index=-1) / KLDivLoss pipeline on the engine's own scores, in fp64
    ref = P.pretraining_losses(t.double().cpu(), v.double().cpu(), align.double().cpu(), labels[0], labels[1], labels[2].double(), labels[3])
    for name, got, r in zip(("masked_lm_loss", "masked_img_loss", "next_sentence_loss"), (lm, img, nsp), ref):
        assert got.shape == (1,) and abs(float(got) - float(r)) <= 1e-5 * abs(float(r)), (mode, name, float(got), float(r))
    oracle_losses = pt_oracle(*[b[k] for k in KEYS], *labels)
    for name, got, r in zip(("masked_lm_loss", "masked_img_loss", "next_sentence_loss"), (lm, img, nsp), oracle_losses):
        err = abs(float(got) - float(r))
        print(f"PARITY pretraining loss {mode} {name}: {float(got):.6f} vs oracle {float(r):.6f} (abs err {err:.3e})")
        assert err < TOL_LOSS[mode] * max(1.0, abs(float(r))), (mode, name, err)


def test_full_model_losses(full_pt):
    oracle, model = full_pt
    b = _batch(model, 2, 36, 37, seed=10)
    got = model(*[b[k].cuda() for k in KEYS], *[b[k].cuda() for k in LABELS])
    ref = oracle(*[b[k] for k in KEYS], *[b[k] for k in LABELS])
    torch.cuda.synchronize()
    for g, r in zip(got, ref):
        assert abs(float(g) - float(r)) < TOL_LOSS["bf16"] * max(1.0, abs(float(r))), (float(g), float(r))


def test_empty_lists_give_nan(tiny):
    model = tiny["fp16"]
    b = _batch(model, 2, 10, 6, seed=11)
    _, taps = _dense(model, [b[k] for k in KEYS], 0)
    res = model.pretraining_objectives(taps, text_rows=[], token_labels=[], image_rows=[], image_targets=None, pair_rows=[1],
                                       pair_labels=[1])
    torch.cuda.synchronize()
    assert math.isnan(float(res["masked_lm_loss"])) and math.isnan(float(res["masked_img_loss"]))
    assert not math.isnan(float(res["next_sentence_loss"]))
    # a batch with no masked token, region or labelled pair: NaN for all three, as upstream's 0 / 0
    lab = dict(masked_lm_labels=torch.full((2, 10), -1), image_label=torch.full((2, 5), -1),
               image_target=b["image_target"], next_sentence_label=torch.full((2,), -1))
    out = model(*[b[k].cuda() for k in KEYS], **lab)
    torch.cuda.synchronize()
    assert all(math.isnan(float(x)) for x in out)


@pytest.mark.parametrize("mode", ("fp16", "fp32x"))
def test_repeated_and_back_to_back_calls_same_bits(tiny, mode):
    model = tiny[mode]
    b = _batch(model, 3, 60, 50, seed=12)
    _, taps = _dense(model, [b[k] for k in KEYS], 0)
    vocab, vt = model._dims["vocab_size"], model._dims["v_target_size"]
    g = torch.Generator().manual_seed(13)
    calls = []
    for n_t, n_v in ((5, 3), (150, 140), (1, 300), (183, 1)):
        tr = torch.randint(0, 180, (n_t,), generator=g)
        vr = torch.randint(0, 150, (n_v,), generator=g)
        calls.append(dict(text_rows=tr, token_labels=torch.randint(0, vocab, (n_t,), generator=g), image_rows=vr,
                          image_targets=_targets(n_v, vt, n_v), pair_rows=[2, 0], pair_labels=[1, 0]))
    plans = support.n_plans(model)
    alone = []
    for c in calls:
        alone.append(model.pretraining_objectives(taps, **c))
        torch.cuda.synchronize()
    again = [model.pretraining_objectives(taps, **c) for c in calls]       # no synchronisation in between
    torch.cuda.synchronize()
    for a, r in zip(alone, again):
        for k in a:
            assert torch.equal(a[k], r[k]) or (torch.isnan(a[k]).all() and torch.isnan(r[k]).all()), k
    assert support.n_plans(model) == plans


def test_objectives_on_multitask_engine(tiny_oracle):
    import vilbert_b200 as vb
    from oracle import vilbert_ref as R
    cfg = vb.BertConfig.from_dict(tiny_oracle.config.to_dict())
    model = vb.VILBertForVLTasks.from_pretrained(tiny_oracle.state_dict(), config=cfg, num_labels=200).eval().cuda(0)
    try:
        inp = list(R.make_inputs(2, 20, 9, seed=14, vocab_size=cfg.vocab_size))
        inp[1] = inp[1][..., :cfg.v_feature_size].contiguous()
        _, taps = model(*[t.cuda() for t in inp], select=0, debug_taps=True)
        tg = _targets(3, cfg.v_target_size, 15)
        res = model.pretraining_objectives(taps, text_rows=[1, 2, 40], token_labels=[7, 8, 9], image_rows=[0, 4, 17], image_targets=tg,
                                           pair_rows=[0, 1], pair_labels=[1, 0])
        heads = model.pretraining_heads(taps, text_rows=[1, 2, 40], image_rows=[0, 4, 17], pair_rows=[0, 1])
        torch.cuda.synchronize()
        ce_t, kl, ce_p = _torch_losses(heads["token_logits"], heads["region_logits"], heads["alignment"],
                                       torch.tensor([7, 8, 9]).cuda(), tg, torch.tensor([1, 0]).cuda())
        assert _rel(res["token_loss"], ce_t) < 1e-5 and _rel(res["region_loss"], kl) < 1e-5 and _rel(res["pair_loss"], ce_p) < 1e-5
    finally:
        model.close()


# ------------------------------------------------------------------ zero-shot retrieval
def test_zero_shot_retrieval_alignment(tiny):
    from vilbert_b200 import parallel as P
    model = tiny["fp16"]
    b = _batch(model, 3, 14, 8, seed=16)
    im = torch.ones(3, 14, dtype=torch.long)
    im[1, 10:] = 0
    vm = torch.ones(3, 8, dtype=torch.uint8)
    vm[2, 6:] = 0
    caps = (b["input_ids"].cuda(), b["token_type_ids"].cuda(), im.cuda())
    imgs = (b["image_feat"].cuda(), b["image_loc"].cuda(), vm.cuda())
    scores = P.retrieval_scores_packed(model, caps, imgs, pair_batch=4, score="alignment")
    torch.cuda.synchronize()
    assert scores.shape == (3, 3, 2)
    for c in range(3):
        lt = int(im[c].sum())
        for i in range(3):
            lv = int(vm[i].sum())
            ones_t, ones_v = torch.ones(1, lt, dtype=torch.long), torch.ones(1, lv, dtype=torch.uint8)
            _, _, align, _ = model(b["input_ids"][c:c + 1, :lt].cuda(), b["image_feat"][i:i + 1, :lv].cuda(),
                                   b["image_loc"][i:i + 1, :lv].cuda(), b["token_type_ids"][c:c + 1, :lt].cuda(), ones_t.cuda(),
                                   ones_v.cuda())
            torch.cuda.synchronize()
            assert torch.equal(scores[c, i], align[0]), (c, i)


# ------------------------------------------------------------------ rejections
def test_task_head_select_bits_rejected(tiny):
    L = support.lib()
    model = tiny["fp16"]
    b = _batch(model, 2, 10, 6, seed=17)
    names = {L.OUT_VIL_PREDICTION: "vil_prediction", L.OUT_VIL_PREDICTION_GQA: "vil_prediction_gqa", L.OUT_VIL_LOGIT: "vil_logit",
             L.OUT_VIL_BINARY_PREDICTION: "vil_binary_prediction", L.OUT_VIL_TRI_PREDICTION: "vil_tri_prediction",
             L.OUT_VISION_LOGIT: "vision_logit", L.OUT_LINGUISIC_LOGIT: "linguisic_logit"}
    q, seg = b["input_ids"][0], b["token_type_ids"][0]
    f, s = b["image_feat"][0], b["image_loc"][0]
    ts = model.encode_text_packed(q.cuda(), seg.cuda(), torch.zeros(1, 1, dtype=torch.long), [10])
    vs = model.encode_image_packed(f.cuda(), s.cuda(), [6])
    one = torch.zeros(1, dtype=torch.int32)
    calls = {
        "dense": lambda sel: _dense(model, [b[k] for k in KEYS], sel),
        "packed": lambda sel: model.forward_packed(q.cuda(), f.cuda(), s.cuda(), seg.cuda(), None, [10], [6], select=sel),
        "cached_packed": lambda sel: model.forward_cached_packed(ts, one, vs, one, select=sel),
        "plan_info": lambda sel: model.plan_info(1, 10, 6, select=sel),
    }
    plans = support.n_plans(model)
    for bit, name in names.items():
        for kind, call in calls.items():
            with pytest.raises(L.VilbertB200Error, match=f"task head {name} "):
                call(bit)
    assert support.n_plans(model) == plans


def test_decode_families_rejected(tiny):
    L = support.lib()
    model = tiny["fp16"]
    t = torch.zeros(4, 3, device="cuda")
    fields = {L.DECODE_VQA: "vil_prediction", L.DECODE_GQA: "vil_prediction_gqa", L.DECODE_NLVR2: "vil_binary_prediction",
              L.DECODE_SNLI_VE: "vil_tri_prediction", L.DECODE_RETRIEVAL: "vil_logit", L.DECODE_GROUNDING: "vision_logit"}
    for fam, field in fields.items():
        o = L.Outputs()
        setattr(o, field, t.data_ptr())
        msgs = (L.DecodeMsg * 1)(L.DecodeMsg(fam, 0, 1, 1, 1.0, 1.0))
        answers = torch.full((1, C.sizeof(L.Answer) // 4), 7, dtype=torch.int32, device="cuda")
        rc = L.load().vb200_decode_answers(model._handle, msgs, 1, C.byref(o), 4, 4, t.data_ptr(), answers.data_ptr(), None)
        torch.cuda.synchronize()
        msg = L.load().vb200_last_error(model._handle).decode()
        assert rc == -1 and f"task head {field}," in msg, msg
        assert bool((answers == 7).all())


def _raw_objectives(model, taps, t_rows=(), t_labels=(), v_rows=(), targets=None, p_rows=(), p_labels=(), top_k=0):
    L = support.lib()
    keep = []

    def arr(v):
        a = (C.c_int32 * max(len(v), 1))(*v)
        keep.append(a)
        return C.cast(a, C.c_void_p)
    st = [taps["sequence_output_t"], taps["sequence_output_v"], taps["pooled_output"]]
    n_state = [st[0].numel() // st[0].shape[-1], st[1].numel() // st[1].shape[-1], st[2].shape[0]]
    rows = [list(t_rows), list(v_rows), list(p_rows)]
    r = L.PretrainRows(*(s.data_ptr() for s in st), *n_state, *(len(x) for x in rows), *(arr(x) for x in rows), top_k)
    tg = L.PretrainTargets(arr(list(t_labels)), targets, arr(list(p_labels)))
    outs = [torch.full((max(len(x), 1),), 7.0, device="cuda") for x in rows] + [torch.full((3,), 7.0, device="cuda")]
    o = L.PretrainLosses(*(x.data_ptr() for x in outs))
    torch.cuda.synchronize()
    plans = support.n_plans(model)
    rc = L.load().vb200_pretraining_objectives(model._handle, C.byref(r), C.byref(tg), C.byref(o), None)
    torch.cuda.synchronize()
    assert support.n_plans(model) == plans
    return rc, L.load().vb200_last_error(model._handle).decode(), outs


def test_objective_rejections_leave_outputs(tiny):
    model = tiny["fp16"]
    b = _batch(model, 2, 10, 6, seed=18)
    _, taps = _dense(model, [b[k] for k in KEYS], 0)
    vocab, vt = model._dims["vocab_size"], model._dims["v_target_size"]
    tg = torch.full((2, vt), 1.0 / vt, device="cuda")
    raw = torch.zeros(2 * vt + 1, device="cuda")
    cases = [
        (dict(t_rows=[0, 1], t_labels=[3, vocab]), f"token_labels[1] = {vocab} is outside [0, {vocab})"),
        (dict(t_rows=[0], t_labels=[-1]), "token_labels[0] = -1"),
        (dict(p_rows=[0, 1], p_labels=[1, 2]), "pair_labels[1] = 2 is not 0 or 1"),
        (dict(p_rows=[0, 1], p_labels=[0, -1]), "pair_labels[1] = -1"),
        (dict(v_rows=[0, 1], targets=None), "image_targets is NULL for 2 image rows"),
        (dict(v_rows=[0, 1], targets=raw.data_ptr() + 2), "image_targets is not 4-byte aligned"),
        (dict(t_rows=[0, 20], t_labels=[1, 1]), "text_rows[1] = 20"),
        (dict(v_rows=[12], targets=tg.data_ptr()), "image_rows[0] = 12"),
        (dict(p_rows=[2], p_labels=[0]), "pair_rows[0] = 2"),
        (dict(t_rows=[0], t_labels=[1], top_k=2), "top_k 2"),
    ]
    for kw, needle in cases:
        rc, msg, outs = _raw_objectives(model, taps, **kw)
        assert rc == -1 and needle in msg, (kw, msg)
        for t in outs:
            assert bool((t == 7).all()), kw
    rc, msg, outs = _raw_objectives(model, taps, t_rows=[0], t_labels=[vocab - 1], v_rows=[0, 11], targets=tg.data_ptr(), p_rows=[1],
                                    p_labels=[0])
    assert rc == 0, msg


def test_audit_on_device():
    import vilbert_b200 as vb
    from oracle import pretraining_ref as P
    from oracle import vilbert_ref as R
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    sd = oracle.state_dict()
    with pytest.raises(vb.VilbertB200Error, match='missing key "cls.imagePredictions.decoder.bias"'):
        bad = dict(sd)
        del bad["cls.imagePredictions.decoder.bias"]
        vb.BertForMultiModalPreTraining.from_pretrained(bad, config=cfg).cuda(0)
    # a multi-task checkpoint missing its task heads still fails vb200_create with the same message as before
    multi = R.build(R.tiny_config(), seed=7, num_labels=200)
    heads_off = {k: v for k, v in multi.state_dict().items() if not k.startswith("vil_")}
    with pytest.raises(vb.VilbertB200Error, match='checkpoint is missing key "vil_prediction.logit_fc.3.weight"'):
        vb.VILBertForVLTasks.from_pretrained(heads_off, config=vb.BertConfig.from_dict(multi.config.to_dict()), num_labels=200).cuda(0)
