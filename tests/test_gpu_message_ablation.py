"""Message ablation (vb200_message_ablation / VILBertForVLTasks.message_ablation / worker_api.custom_ablation_packed).  `-m gpu` only.

Every variant is the engine's own forward of a well-defined input in the worker's layout -- the message's question repeated per
image, one position replaced by [MASK], or one image without one box -- so each variant's segment is compared bit for bit with the
same floats of forward_regions_packed of that input built on the host (a retrieval box variant with all K images), and the scores
with vb200_decode_answers on those segments.
"""
import ctypes as C
import random

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 / bf16 vs the fp32 oracle (test_gpu_regions_packed.py)
MASK = 103
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6
POOLED = 1 | 2 | 4 | 8 | 16            # OUT_VIL_PREDICTION | _GQA | VIL_LOGIT | VIL_BINARY_PREDICTION | VIL_TRI_PREDICTION
HEAD = {VQA: 0, GQA: 1, SNLI: 4}       # element of the 10-tuple a one-row family reads
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing", "?", "a",
                                     "dog", "on", "grass"])}


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16"))


@pytest.fixture(scope="module")
def tiny_long(tiny_oracle):
    yield from support.one_engine(tiny_oracle, compute_dtype="bf16", max_rows_per_sample=1024)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _batch(model, groups, seed):
    """The worker's layout: per group (tin, [boxes per image]) the group's text repeated on each of its images.  Returns the samples
    and each group's first sample."""
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs, first = [], []
    for gi, (tin, counts) in enumerate(groups):
        first.append(len(imgs))
        for k, n in enumerate(counts):
            q, seg, f, bx, wh, task = support.image(tin, n, seed + 31 * gi + k, F, vocab, ((640, 480), (500, 375))[k % 2])
            if k > 0:
                q, seg, task = imgs[first[-1]][0], imgs[first[-1]][1], imgs[first[-1]][5]
            imgs.append((q, seg, f, bx, wh, task))
    return imgs, first


def _ablate(model, imgs, messages, **kw):
    out = model.message_ablation(*support.packed_image_args(imgs), messages, return_logits=True, mask_token=MASK, **kw)
    torch.cuda.synchronize()
    return out


def _variants(imgs, fam, ib, K, r):
    """The message's variants built on the host in the worker's layout: per variant its samples (a retrieval box variant: all K
    images) and, for a box variant, the changed image and the dropped row."""
    q, seg, task = imgs[ib][0], imgs[ib][1], imgs[ib][5]
    own = [(q, seg) + imgs[ib + k][2:5] + (task,) for k in range(K)]
    out = [(own, None)]
    for p in r["tokens"]:
        qm = q.clone()
        qm[p] = MASK
        out.append(([(qm,) + s[1:] for s in own], None))
    for k, j in r["boxes"]:
        keep = torch.arange(own[k][2].shape[0]) != j
        changed = own[k][:2] + (own[k][2][keep], own[k][3][keep]) + own[k][4:]
        samples = [changed if i == k else s for i, s in enumerate(own)]
        out.append((samples if fam in (NLVR2, RET) else [changed], (k, j)))
    return out


def _reference(model, imgs, fam, ib, K, r):
    """forward_regions_packed of every host-built variant of one message: each variant's segment."""
    import vilbert_b200 as vb
    var = _variants(imgs, fam, ib, K, r)
    samples = [s for v, _ in var for s in v]
    sel = POOLED | (vb.OUT_VISION_LOGIT if fam == GRD else 0)
    out, _ = model.forward_regions_packed(*support.packed_image_args(samples), select=sel, return_spatials=False)
    torch.cuda.synchronize()
    segs, at = [], 0
    voff = [0]
    for s in samples:
        voff.append(voff[-1] + s[2].shape[0] + 1)
    for v, _ in var:
        if fam in HEAD:
            segs.append(out[HEAD[fam]][at])
        elif fam == NLVR2:
            assert at % 2 == 0
            segs.append(out[3][at // 2])
        elif fam == RET:
            segs.append(out[2][at:at + K].reshape(-1))
        else:
            segs.append(out[6][voff[at]:voff[at + 1]].reshape(-1))
        at += len(v)
    return segs


def _check_bitwise(model, imgs, msgs, res):
    for (fam, ib, K, *_), r in zip(msgs, res):
        want = _reference(model, imgs, fam, ib, K, r)
        got = r["logits"]
        assert len(got) == len(want) == 1 + len(r["tokens"]) + len(r["boxes"])
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), f"family {fam}: variant {k} differs from forward_regions_packed of its input"


def _check_scores(model, msgs, res):
    """Scores against vb200_decode_answers of each segment; grounding's rows mapped back to the unablated numbering on the host."""
    for (fam, ib, K, *rest), r in zip(msgs, res):
        segs = r["logits"]
        flat = torch.cat(segs).reshape(-1, 1).contiguous()
        out = [None] * 10
        out[2] = flat
        offs = [0]
        for s in segs:
            offs.append(offs[-1] + s.numel())
        dec = model.decode_answers(out, [(RET, offs[k], s.numel(), min(10, s.numel()), None) for k, s in enumerate(segs)])
        answer = rest[0] if rest and rest[0] is not None else None
        col = dec[0][0][0] if answer is None else answer
        assert r["answer"] == col and r["top1"] == dec[0][0][0] and r["top1_prob"] == dec[0][1][0]
        drops = [None] * (1 + len(r["tokens"])) + [j + 1 if fam == GRD else None for _, j in r["boxes"]]
        probs = [r["prob"]] + r["token_prob"].tolist() + r["box_prob"].tolist()
        top1 = [r["top1"]] + r["token_top1"].tolist() + r["box_top1"].tolist()
        for k, ((idx, p, _), d) in enumerate(zip(dec, drops)):
            t = idx[0]
            assert top1[k] == (t + 1 if d is not None and t >= d else t), f"family {fam}: variant {k} top-1"
            if d is not None and col == d:
                assert probs[k] == 0.0, f"family {fam}: variant {k} dropped the attributed row"
                continue
            at = col - 1 if d is not None and col > d else col
            if at in idx:
                assert probs[k] == p[idx.index(at)], f"family {fam}: variant {k} attributed probability"
            else:
                sm = torch.softmax(segs[k].double(), 0)[at].item()
                assert abs(probs[k] - sm) <= 2e-5 * sm + 1e-12


def _scores_raw(res):
    return [(r["answer"], r["prob"], r["top1"], r["top1_prob"], r["token_prob"].tolist(), r["box_prob"].tolist(),
             r["token_top1"].tolist(), r["box_top1"].tolist()) for r in res]


# (Tin, box counts per image) and the message over that group: (family, answer, tokens, boxes)
GROUPS = [(9, [6, 2]), (12, [3, 1, 5]), (5, [4]), (7, [9]), (20, [2]), (6, [8]), (4, [3])]


def _messages(first):
    return [(NLVR2, first[0], 2, None, (1, 8), None), (RET, first[1], 3, 1, (0, 4), None), (GRD, first[2], 1, 2, None, None),
            (VQA, first[3], 1, None, (1, 6), (2, 9)), (GQA, first[4], 1, 7, None, None), (SNLI, first[5], 1, None, (0, 6), (0, 3)),
            (GRD, first[6], 1, None, (1, 3), (0, 3))]


@pytest.mark.parametrize("mode", ["fp16", "bf16"])
def test_every_family_bitwise_and_scores(tiny, mode):
    model = tiny[mode]
    imgs, first = _batch(model, GROUPS, seed=11)
    msgs = _messages(first)
    res = _ablate(model, imgs, msgs)
    assert res[1]["boxes"] == [(0, 0), (0, 1), (0, 2), (2, 0), (2, 1), (2, 2), (2, 3), (2, 4)]     # the one-box image is skipped
    assert res[2]["boxes"] == [(0, j) for j in range(4)] and res[2]["tokens"] == [1, 2, 3]
    _check_bitwise(model, imgs, msgs, res)
    _check_scores(model, msgs, res)
    assert res[2]["box_prob"][1].item() == 0.0                   # grounding answer row 2 is box 1


@pytest.mark.parametrize("K", [1, 3, 10])
def test_retrieval_sizes(tiny, K):
    """Retrieval with K images of mixed box counts: box variants run one image and equal the whole K-image variant."""
    model = tiny["bf16"]
    counts = [(2, 7, 1, 30)[k % 4] for k in range(K)]
    imgs, first = _batch(model, [(8, counts)], seed=100 + K)
    msgs = [(RET, 0, K, None, (1, 3), None)]
    res = _ablate(model, imgs, msgs)
    _check_bitwise(model, imgs, msgs, res)
    _check_scores(model, msgs, res)


def test_grounding_attributed_box_dropped(tiny):
    """Grounding with the attributed row dropped reports -1 / 0.0; top-1 rows after the dropped box map back by +1."""
    model = tiny["fp16"]
    imgs, first = _batch(model, [(6, [12])], seed=5)
    for answer in (0, 1, 5, 12, None):
        msgs = [(GRD, 0, 1, answer, (0, 0), None)]
        res = _ablate(model, imgs, msgs)
        col = res[0]["answer"]
        for j, (ans, p) in enumerate(zip([s for s in _raw_answers(model, imgs, msgs)], res[0]["box_prob"].tolist())):
            if col == j + 1:
                assert ans == -1 and p == 0.0
            else:
                assert ans == col
        _check_scores(model, msgs, res)


def _raw_answers(model, imgs, msgs):
    """The answer field of every box variant's score, read through the C ABI."""
    from vilbert_b200 import _lib as L
    import vilbert_b200 as vb
    a = support.packed_image_args(imgs)
    arr = (L.AblationMessage * len(msgs))(*[L.AblationMessage(m[0], m[1], m[2], -1 if m[3] is None else m[3], *m[4],
                                                                  0, int(a[7][m[1]])) for m in msgs])
    recs, n_floats, _ = model._message_layout(a[6], a[7], [tuple(getattr(x, f) for f, _ in L.AblationMessage._fields_) for x in arr])
    logits = torch.empty(n_floats, device="cuda")
    scores = torch.empty(len(recs), 4, dtype=torch.int32, device="cuda")
    inp = L.PackedRegionInputs(len(a[6]), 0, 0, vb.model._int32s(a[6]), vb.model._int32s(a[7]), *[t.data_ptr() for t in a[:6]], None)
    model._call("vb200_message_ablation", C.byref(inp), arr, len(msgs), MASK, logits.data_ptr(), scores.data_ptr(), 0)
    return [int(s) for s, r in zip(scores[:, 0].tolist(), recs) if r[1] == 2]


def test_mixed_call_matches_one_call_per_message(tiny):
    """All six families in one call, in shuffled order, give each message the bits of a call of its own."""
    model = tiny["bf16"]
    imgs, first = _batch(model, GROUPS, seed=13)
    msgs = _messages(first)
    order = list(range(len(msgs)))
    random.Random(3).shuffle(order)
    mixed = _ablate(model, imgs, [msgs[i] for i in order])
    for pos, i in enumerate(order):
        alone = _ablate(model, imgs, [msgs[i]])[0]
        assert all(torch.equal(a, b) for a, b in zip(mixed[pos]["logits"], alone["logits"]))
        assert _scores_raw([mixed[pos]]) == _scores_raw([alone])


def test_agrees_with_answer_ablation(tiny):
    """Single-image VQA, GQA and SNLI-VE messages: the bits of vb200_answer_ablation."""
    model = tiny["fp16"]
    imgs, first = _batch(model, [(9, [6]), (14, [3]), (5, [1])], seed=17)
    for fam, name in ((VQA, "vqa"), (GQA, "gqa"), (SNLI, "snli_ve")):
        old = model.answer_ablation(*support.packed_image_args(imgs), family=name, return_logits=True, mask_token=MASK)
        new = _ablate(model, imgs, [(fam, i, 1) for i in range(3)])
        for o, n in zip(old, new):
            assert torch.equal(o["logits"], torch.stack(n["logits"]))
            for k in ("answer", "prob", "top1", "top1_prob"):
                assert o[k] == n[k]
            for k in ("token_prob", "box_prob", "token_top1", "box_top1"):
                assert torch.equal(o[k], n[k])
            assert n["boxes"] == [(0, j) for j in o["boxes"]]


def test_full_model(full):
    """The 268 M model in bf16: one message per family at 37 tokens and 100 boxes, ranges trimmed."""
    groups = [(37, [100, 100]), (37, [100, 100, 100]), (37, [100]), (37, [100]), (37, [100]), (37, [100])]
    imgs, first = _batch(full, groups, seed=5)
    msgs = [(NLVR2, first[0], 2, None, (1, 4), (98, 102)), (RET, first[1], 3, None, (1, 3), (150, 153)),
            (GRD, first[2], 1, None, (1, 3), (0, 4)), (VQA, first[3], 1, None, (34, 36), (97, 100)),
            (GQA, first[4], 1, None, (1, 3), (0, 2)), (SNLI, first[5], 1, None, (1, 3), (0, 2))]
    res = _ablate(full, imgs, msgs)
    _check_bitwise(full, imgs, msgs, res)
    _check_scores(full, msgs, res)


def test_past_256_rows(tiny_long):
    """Grounding with 300 boxes and retrieval with two 300-box images on a max_rows_per_sample=1024 engine."""
    imgs, first = _batch(tiny_long, [(40, [300]), (10, [300, 300])], seed=3)
    msgs = [(GRD, first[0], 1, None, (1, 3), (290, 300)), (RET, first[1], 2, None, (1, 2), (298, 302))]
    res = _ablate(tiny_long, imgs, msgs)
    _check_bitwise(tiny_long, imgs, msgs, res)
    _check_scores(tiny_long, msgs, res)


def test_against_the_oracle(tiny, tiny_oracle):
    """The unablated segments within the packed tests' tolerance of the fp32 oracle: an NLVR2 pair, VQA, retrieval and grounding."""
    from vilbert_b200 import worker_api as W
    model = tiny["fp16"]
    imgs, first = _batch(model, [(8, [5, 7]), (10, [4]), (6, [3, 9, 2]), (7, [6]), (5, [2])], seed=19)
    msgs = [(NLVR2, 0, 2, None, (0, 0), (0, 0)), (VQA, 2, 1, None, (0, 0), (0, 0)), (RET, 3, 3, None, (0, 0), (0, 0)),
            (GRD, 6, 1, None, (0, 0), (0, 0))]
    res = _ablate(model, imgs, msgs)
    rows = []
    for q, seg, f, bx, wh, task in imgs:                         # worker.py:422-455 on the host, then padded with masks
        info = {"image_width": float(wh[0]), "image_height": float(wh[1]), "bbox": bx.numpy()}
        _, ff, ss, _, _, _, _, _ = W.build_inputs("", [task], [f], [info], torch.device("cpu"), W.WordpieceTokenizer(VOCAB))
        rows.append((ff[0], ss[0]))
    B, Tm, Vm, F = len(imgs), max(len(v[0]) for v in imgs), max(r[0].shape[0] for r in rows), model._dims["v_feature_size"]
    q, seg, mask = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (v, (ff, ss)) in enumerate(zip(imgs, rows)):
        t = len(v[0])
        q[b, :t], seg[b, :t], mask[b, :t] = v[0], v[1], 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.tensor([[v[5]] for v in imgs])
    ref = tiny_oracle(q, f, s, seg, mask, vm, None, task, compute_pretraining_heads=False)
    want = [ref[3][0], ref[0][2], ref[2][3:6].reshape(-1), ref[6][6, :rows[6][0].shape[0]].reshape(-1)]
    for r, w in zip(res, want):
        err = float((r["logits"][0].cpu() - w).abs().max())
        assert err < TOL, f"unablated segment vs fp32 oracle: {err} >= {TOL}"


def _call(model, imgs, msgs, logits, scores, mask=MASK, handle=None, n_msgs=None, inp_kw=None, bf=None):
    from vilbert_b200 import _lib as L
    import vilbert_b200 as vb
    a = support.packed_image_args(imgs)
    kw = dict(nt=a[6], nb=a[7], max_boxes=0)
    kw.update(inp_kw or {})
    arr = (L.AblationMessage * max(len(msgs), 1))(*[L.AblationMessage(*m) for m in msgs])
    inp = L.PackedRegionInputs(len(kw["nt"]), 0, kw["max_boxes"], vb.model._int32s(kw["nt"]), vb.model._int32s(kw["nb"]),
                               a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), bf if bf is not None else a[3].data_ptr(),
                               a[4].data_ptr(), a[5].data_ptr(), None)
    lib = L.load()
    h = handle or model._handle
    rc = lib.vb200_message_ablation(h, C.byref(inp), arr, len(msgs) if n_msgs is None else n_msgs, mask,
                                    logits.data_ptr() if logits is not None else None, scores.data_ptr() if scores is not None else None,
                                    0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, lib.vb200_last_error(h).decode()


def test_layout_matches_the_call(tiny):
    """The layout records give the variant order, the sample counts and the segments the call writes, and nothing past them."""
    model = tiny["fp16"]
    imgs, first = _batch(model, GROUPS, seed=23)
    msgs = [(NLVR2, first[0], 2, -1, 1, 3, 5, 7), (RET, first[1], 3, 2, 0, 2, 4, 6), (GRD, first[2], 1, 0, 1, 2, 0, 2),
            (VQA, first[3], 1, -1, 0, 1, 0, 1)]
    a = support.packed_image_args(imgs)
    recs, n_floats, _ = model._message_layout(a[6], a[7], msgs)
    K = {0: 2, 1: 3, 2: 1, 3: 1}
    length = {0: 2, 1: 3, 2: 5, 3: model._dims["num_labels"]}
    want = []
    for m, (fam, ib, k, ans, tb, te, bb, be) in enumerate(msgs):
        want.append((m, 0, -1, K[m]))
        want += [(m, 1, p, K[m]) for p in range(tb, te)]
        want += [(m, 2, u, 2 if fam == NLVR2 else 1) for u in range(bb, be)]
    assert [r[:4] for r in recs] == want
    off = 0
    for r in recs:
        box = r[1] == 2 and msgs[r[0]][0] == GRD
        assert r[4] == off and r[5] == length[r[0]] - (1 if box else 0)
        off += r[5]
    assert off == n_floats
    logits = torch.full((n_floats + 64,), float("nan"), device="cuda")
    scores = torch.full((len(recs) + 4, 4), 7, dtype=torch.int32, device="cuda")
    rc, msg = _call(model, imgs, msgs, logits, scores)
    assert rc == 0, msg
    assert not logits[:n_floats].isnan().any() and logits[n_floats:].isnan().all()
    assert not (scores[:len(recs)] == 7).all(1).any() and (scores[len(recs):] == 7).all()


def test_plans_are_shared_and_forwards_unchanged(tiny):
    """Repeated calls in the same bucket and capacities add no plans; forwards around a call keep their bits."""
    model = tiny["bf16"]
    imgs, first = _batch(model, GROUPS, seed=61)
    fwd = lambda: model.forward_regions_packed(*support.packed_image_args(imgs), max_tokens=20, max_boxes=30)[0][0].clone()
    before = fwd()
    msgs = _messages(first)
    _ablate(model, imgs, msgs, max_tokens=20, max_boxes=30)
    _ablate(model, imgs, msgs[3:5], max_tokens=20, max_boxes=30)          # pooled only
    n = support.n_plans(model)
    _ablate(model, imgs, msgs[::-1], max_tokens=20, max_boxes=30)
    _ablate(model, imgs, msgs[4:6], max_tokens=20, max_boxes=30)
    assert support.n_plans(model) == n
    assert torch.equal(fwd(), before)


def test_back_to_back_calls_need_no_synchronisation(tiny):
    from vilbert_b200 import _lib as L
    import vilbert_b200 as vb
    model = tiny["fp16"]
    sets = []
    for s, groups in ((71, GROUPS), (72, [(15, [40, 3])]), (73, [(6, [3]), (9, [9, 2, 4])])):
        imgs, first = _batch(model, groups, seed=s)
        msgs = [(m[0], m[1], m[2], -1 if m[3] is None else m[3]) + (m[4] or (0, 0)) + (m[5] or (0, 2)) for m in _messages(first)] \
            if s == 71 else ([(NLVR2, 0, 2, -1, 1, 14, 0, 43)] if s == 72 else [(GRD, 0, 1, -1, 1, 5, 0, 3), (RET, 1, 3, -1, 0, 9, 0, 15)])
        a = support.packed_image_args(imgs)
        recs, n_floats, arr = model._message_layout(a[6], a[7], msgs)
        inp = L.PackedRegionInputs(len(a[6]), 0, 0, vb.model._int32s(a[6]), vb.model._int32s(a[7]), *[t.data_ptr() for t in a[:6]], None)
        sets.append((inp, arr, len(msgs), n_floats, len(recs), a))

    def run(sync):
        outs = []
        for inp, arr, n, nf, nv, _ in sets:
            logits = torch.full((nf,), float("nan"), device="cuda")
            scores = torch.zeros(nv, 4, dtype=torch.int32, device="cuda")
            model._call("vb200_message_ablation", C.byref(inp), arr, n, MASK, logits.data_ptr(), scores.data_ptr(), 0)
            if sync:
                torch.cuda.synchronize()
            outs.append((logits, scores))
        torch.cuda.synchronize()
        return outs

    for (la, sa), (lb, sb) in zip(run(False), run(True)):
        assert torch.equal(la, lb) and torch.equal(sa, sb)


def test_rejections(tiny, tiny_oracle):
    """Every rejection is VB200_ERR_INVALID, names its cause and message, and leaves the sentinel-filled outputs untouched."""
    model = tiny["fp16"]
    imgs, first = _batch(model, [(6, [3, 4]), (5, [1]), (7, [2])], seed=81)
    logits = torch.full((4096,), 7.0, device="cuda")
    scores = torch.full((256, 4), 7, dtype=torch.int32, device="cuda")
    ok = [(NLVR2, 0, 2, -1, 1, 5, 0, 7), (VQA, 2, 1, -1, 0, 0, 0, 0)]
    a = support.packed_image_args(imgs)
    cases = [
        (dict(msgs=[(99, 0, 1, -1, 0, 0, 0, 0)]), "message 0 has unknown family"),
        (dict(msgs=[(NLVR2, 0, 1, -1, 0, 0, 0, 0)]), "message 0 (family 3) has n_images 1"),
        (dict(msgs=[ok[0], (VQA, 2, 2, -1, 0, 0, 0, 0)]), "message 1 (family 1) has n_images 2"),
        (dict(msgs=[(RET, 0, 0, -1, 0, 0, 0, 0)]), "has n_images 0"),
        (dict(msgs=[(RET, 3, 2, -1, 0, 0, 0, 0)]), "outside the batch"),
        (dict(msgs=[(VQA, -1, 1, -1, 0, 0, 0, 0)]), "outside the batch"),
        (dict(msgs=[(NLVR2, 0, 2, 2, 0, 0, 0, 0)]), "message 0 has answer 2"),
        (dict(msgs=[(RET, 0, 3, 3, 0, 0, 0, 0)]), "message 0 has answer 3"),
        (dict(msgs=[(GRD, 0, 1, 4, 0, 0, 0, 0)]), "message 0 has answer 4"),
        (dict(msgs=[(VQA, 0, 1, -2, 0, 0, 0, 0)]), "has answer -2"),
        (dict(msgs=[(VQA, 0, 1, -1, 0, 7, 0, 0)]), "token range"),
        (dict(msgs=[(VQA, 0, 1, -1, 3, 2, 0, 0)]), "token range"),
        (dict(msgs=[(NLVR2, 0, 2, -1, 0, 0, 0, 8)]), "box range"),
        (dict(msgs=[(NLVR2, 0, 2, -1, 0, 0, 4, 3)]), "box range"),
        (dict(msgs=[(RET, 1, 2, -1, 0, 0, 4, 5)]), "drops a box of its image 1"),
        (dict(msgs=[(VQA, 2, 1, -1, 0, 0, 0, 1)]), "drops a box"),
        (dict(msgs=ok, n_msgs=0), "n_msgs"),
        (dict(msgs=ok, mask=model._dims["vocab_size"]), "mask_token"),
        (dict(msgs=ok, logits=None), "NULL"),
        (dict(msgs=ok, bf=a[3].data_ptr() + 4), "16-byte aligned"),
        (dict(msgs=ok, inp_kw=dict(nt=[6, 6, 0, 7])), "n_tokens 0"),
        (dict(msgs=ok, inp_kw=dict(max_boxes=2)), "above the capacity"),
    ]
    for kw, match in cases:
        msgs = kw.pop("msgs")
        rc, msg = _call(model, imgs, msgs, kw.pop("logits", logits), scores, **kw)
        assert rc == -1 and match in msg, (msgs, kw, rc, msg)
        assert bool((logits == 7.0).all()) and bool((scores == 7).all()), kw
    # more than 1024 samples: retrieval, 3 images, 37 tokens, 120 boxes -> 3 + 35 * 3 + 120 ... in 4 messages
    big, _ = _batch(model, [(37, [100, 100, 100])], seed=90)
    rc, msg = _call(model, big, [(RET, 0, 3, -1, 1, 36, 0, 300)] * 4, logits, scores)
    assert rc == -1 and "above 1024" in msg, msg
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        rc, msg = _call(x, imgs, ok, logits, scores)
        assert rc == -1 and "split_fp32" in msg
    finally:
        x.close()
    assert bool((logits == 7.0).all()) and bool((scores == 7).all())


def test_pretraining_engine_is_rejected():
    from oracle import pretraining_ref as P
    import vilbert_b200 as vb
    ref = P.build(P.tiny_pretraining_config(), seed=7)
    cfg = vb.BertConfig.from_dict(ref.config.to_dict())
    m = vb.BertForMultiModalPreTraining.from_pretrained(ref.state_dict(), config=cfg).eval().cuda(0)
    try:
        imgs, _ = _batch(m, [(5, [3])], seed=1)
        logits = torch.full((8,), 7.0, device="cuda")
        rc, msg = _call(m, imgs, [(VQA, 0, 1, -1, 1, 4, 0, 3)], logits, None)
        assert rc == -1 and "pre-training" in msg
        assert bool((logits == 7.0).all())
    finally:
        m.close()


def test_worker_answers_match_custom_prediction_packed(tiny):
    """custom_ablation_packed: per request the answer of custom_prediction_packed(decode="device") and its attribution."""
    import numpy as np
    from vilbert_b200 import worker_api as W
    model = tiny["bf16"]
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = model
    def det(counts, seed):
        imgs, _ = _batch(model, [(3, counts)], seed=seed)
        return [im[2] for im in imgs], [{"image_width": float(im[4][0]), "image_height": float(im[4][1]), "bbox": im[3].numpy()}
                                        for im in imgs]

    reqs = [("what is the man holding ?", [1], *det([12], 1), "1"), ("a dog on the grass", [12], *det([5, 6], 2), "12"),
            ("the man", [11], *det([9], 3), "11"), ("a dog", [7], *det([4, 1, 3], 4), "7"), ("the dog", [15], *det([6], 5), "15"),
            ("a man", [13], *det([2], 6), "13"), ("bad", [1], *det([3, 3], 7), "1")]
    got = W.custom_ablation_packed(reqs, tokens=(1, 3))
    want = W.custom_prediction_packed(reqs, decode="device")
    assert isinstance(got[-1], AssertionError) and isinstance(want[-1], AssertionError)
    for i, (g, w) in enumerate(zip(got[:-1], want[:-1])):
        assert g["answer"] == w, i
        a = g["ablation"]
        assert a["tokens"] == [1, 2]
        infos = reqs[i][3]
        assert a["box_pixels"] == [[float(v) for v in np.asarray(infos[k]["bbox"], dtype=np.float32)[j, :4]] for k, j in a["boxes"]]
    assert got[3]["ablation"]["boxes"] == [(0, j) for j in range(4)] + [(2, j) for j in range(3)]
    assert "answer_box" in got[2]["ablation"]
