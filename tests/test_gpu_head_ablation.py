"""Head ablation (vb200_head_ablation / vb200_head_ablation_layout / VILBertForVLTasks.head_ablation /
worker_api.custom_head_ablation_packed).  `-m gpu` only.

Every variant is the gated forward of a well-defined input: the message's samples in the worker's layout with one gate at 0.  So each
segment the call writes is compared bit for bit with vb200_forward_regions_packed_gated run on that variant's samples and gate row
alone, for every decode family; the unablated segment with message ablation's; the scores with a softmax of the same segment.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6
POOLED = 1 | 2 | 4 | 8 | 16            # OUT_VIL_PREDICTION | _GQA | VIL_LOGIT | VIL_BINARY_PREDICTION | VIL_TRI_PREDICTION
VISION_LOGIT = 1 << 6
ERR_INVALID = -1
ENTRIES = (5, 11)                       # T5, both directions of C0, T6, V0, C1's text-query direction


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16"), max_rows_per_sample=1024)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _batch(model, groups, seed):
    """The worker's layout: per group (tin, [boxes per image]) the group's text repeated on each of its images."""
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = []
    for gi, (tin, counts) in enumerate(groups):
        first = len(imgs)
        for k, n in enumerate(counts):
            q, seg, f, bx, wh, task = support.image(tin, n, seed + 31 * gi + k, F, vocab)
            if k > 0:
                q, seg, task = imgs[first][0], imgs[first][1], imgs[first][5]
            imgs.append((q, seg, f, bx, wh, task))
    return imgs


def _call(model, imgs, msgs):
    """One raw vb200_head_ablation call: (layout records, logits, scores [n, 4] int32)."""
    L = support.lib()
    args = support.packed_image_args(imgs)
    nt, nb = args[6], args[7]
    recs, n_floats, arr = model._head_layout(nt, nb, msgs)
    logits = torch.full((n_floats,), float("nan"), device="cuda")
    scores = torch.full((len(recs), 4), -7, dtype=torch.int32, device="cuda")
    inp = L.PackedRegionInputs(len(imgs), 0, 0, C.cast((C.c_int32 * len(nt))(*nt), C.c_void_p),
                               C.cast((C.c_int32 * len(nb))(*nb), C.c_void_p), args[0].data_ptr(), args[1].data_ptr(),
                               args[2].data_ptr(), args[3].data_ptr(), args[4].data_ptr(), args[5].data_ptr(), None)
    model._call("vb200_head_ablation", C.byref(inp), arr, len(msgs), logits.data_ptr(), scores.data_ptr(), 0)
    torch.cuda.synchronize()
    return recs, logits, scores


def _reference(model, imgs, fam, ib, K, unit):
    """The variant's segment from vb200_forward_regions_packed_gated on its own samples and gate row."""
    from vilbert_b200.model import head_mask_shape
    E, H = head_mask_shape(model.config)
    mask = torch.ones(K, E, H)
    if unit >= 0:
        mask[:, unit // H, unit % H] = 0.0
    sel = POOLED | (VISION_LOGIT if fam == GRD else 0)
    (out, _) = model.forward_regions_packed(*support.packed_image_args(imgs[ib:ib + K]), select=sel, head_mask=mask)
    torch.cuda.synchronize()
    if fam == VQA:
        return out[0][0]
    if fam == GQA:
        return out[1][0]
    if fam == SNLI:
        return out[4][0]
    if fam == NLVR2:
        return out[3][0]
    if fam == RET:
        return out[2][:K, 0]
    return out[6][:, 0]


def _check_message(model, imgs, msg, recs, logits, scores, m):
    fam, ib, K, answer = msg[:4]
    mine = [(k, r) for k, r in enumerate(recs) if r[0] == m]
    E_lo, E_hi = msg[4], msg[5]
    kinds = model.attention_selection()[0]
    c = model.config
    heads = [c.num_attention_heads if k == 0 else c.v_num_attention_heads if k == 1 else c.bi_num_attention_heads for k in kinds]
    from vilbert_b200.model import head_mask_shape
    H = head_mask_shape(c)[1]
    want_units = [-1] + [e * H + h for e in range(E_lo, E_hi) for h in range(heads[e])]
    assert [r[2] for _, r in mine] == want_units
    assert [r[1] for _, r in mine] == [0] + [3] * (len(want_units) - 1)
    assert all(r[3] == K for _, r in mine)
    base = None
    for k, (_, kind, unit, _, off, n) in mine:
        seg = logits[off:off + n]
        ref = _reference(model, imgs, fam, ib, K, unit)
        assert seg.shape == ref.shape and support.eq32(seg, ref.contiguous()), f"message {m} unit {unit}"
        if kind == 0:
            base = seg
        # scores: the attributed column's probability and the variant's own top-1, as a softmax of the segment gives them
        col = int(scores[k, 0])
        want_col = int(base.argmax()) if answer < 0 else answer
        assert col == want_col
        p = torch.softmax(seg.double(), 0)
        assert abs(float(scores[k, 1:2].view(torch.float32)) - float(p[col])) < 1e-6
        assert int(scores[k, 2]) == int(seg.argmax())


FAMILIES = [(VQA, [(9, [12])]), (GQA, [(5, [7])]), (SNLI, [(11, [3])]), (GRD, [(6, [9])]), (NLVR2, [(8, [5, 6])]),
            (RET, [(7, [4])]), (RET, [(7, [4, 2, 6])])]


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("fam,groups", FAMILIES, ids=["vqa", "gqa", "snli", "grounding", "nlvr2", "ret1", "ret3"])
def test_every_family_bitwise_and_scores(tiny, mode, fam, groups):
    model = tiny[mode]
    imgs = _batch(model, groups, seed=11 + fam)
    msg = (fam, 0, len(groups[0][1]), -1 if fam != VQA else 3) + ENTRIES
    recs, logits, scores = _call(model, imgs, [msg])
    _check_message(model, imgs, msg, recs, logits, scores.cpu(), 0)


def test_shuffled_multi_family_call_matches_one_call_per_message(tiny):
    model = tiny["bf16"]
    imgs = _batch(model, [(9, [12]), (8, [5, 6]), (6, [9]), (7, [4, 2, 6])], seed=3)
    msgs = [(RET, 4, 3, -1, 12, 14), (VQA, 0, 1, 5, 0, 2), (GRD, 3, 1, -1, 28, 30), (NLVR2, 1, 2, -1, 6, 8)]
    recs, logits, _ = _call(model, imgs, msgs)
    for m, msg in enumerate(msgs):
        r1, l1, _ = _call(model, imgs, [msg])
        mine = [r for r in recs if r[0] == m]
        assert [r[1:4] for r in mine] == [r[1:4] for r in r1]
        for a, b in zip(mine, r1):
            assert support.eq32(logits[a[4]:a[4] + a[5]], l1[b[4]:b[4] + b[5]])
    assert not torch.isnan(logits).any()            # the layout's floats are every float the call writes


def test_unablated_matches_message_ablation(tiny):
    model = tiny["fp16"]
    imgs = _batch(model, [(9, [12]), (8, [5, 6])], seed=5)
    recs, logits, _ = _call(model, imgs, [(VQA, 0, 1, -1, 0, 1), (NLVR2, 1, 2, -1, 0, 1)])
    ma = model.message_ablation(*support.packed_image_args(imgs), [(VQA, 0, 1, None, (0, 0), (0, 0)), (NLVR2, 1, 2, None, (0, 0), (0, 0))],
                                return_logits=True)
    for m in range(2):
        r = [x for x in recs if x[0] == m and x[1] == 0][0]
        assert support.eq32(logits[r[4]:r[4] + r[5]], ma[m]["logits"][0])


def test_full_model(full):
    imgs = _batch(full, [(9, [12])], seed=7)
    msg = (VQA, 0, 1, -1, 26, 30)                   # the last entries: connection directions and text layers, 12 / 8 heads
    recs, logits, scores = _call(full, imgs, [msg])
    _check_message(full, imgs, msg, recs, logits, scores.cpu(), 0)


def test_past_256_rows(tiny):
    model = tiny["bf16"]
    imgs = _batch(model, [(20, [299])], seed=9)
    msg = (VQA, 0, 1, -1, 9, 11)                    # V0 (streaming self-attention) and C1 (streaming co-attention)
    recs, logits, scores = _call(model, imgs, [msg])
    _check_message(model, imgs, msg, recs, logits, scores.cpu(), 0)


def test_python_results_and_splitting(tiny):
    """head_ablation: its [n_entries, max_heads] results, for an every-head NLVR2 message and a retrieval K = 3 message in one
    call, equal the scores of raw calls of each message alone."""
    from vilbert_b200.model import head_mask_shape
    model = tiny["bf16"]
    E, H = head_mask_shape(model.config)
    imgs = _batch(model, [(8, [5, 6]), (7, [4, 2, 6])], seed=13)
    args = support.packed_image_args(imgs)
    res = model.head_ablation(*args, [(NLVR2, 0, 2), ("retrieval", 2, 3, None, (0, 30))])
    for m, msg in enumerate([(NLVR2, 0, 2, -1, 0, 30), (RET, 2, 3, -1, 0, 30)]):
        recs, _, scores = _call(model, imgs, [msg])
        sc = scores.cpu()
        assert res[m]["answer"] == int(sc[0, 0])
        for k, r in enumerate(recs[1:], 1):
            assert float(res[m]["head_prob"][r[2] // H, r[2] % H]) == float(sc[k, 1:2].view(torch.float32))
            assert int(res[m]["head_top1"][r[2] // H, r[2] % H]) == int(sc[k, 2])
        assert res[m]["head_prob"].shape == (E, H)


def test_rejections_leave_outputs_untouched(tiny, tiny_oracle):
    L = support.lib()
    model = tiny["bf16"]
    imgs = _batch(model, [(9, [12])], seed=15)
    args = support.packed_image_args(imgs)
    nt, nb = args[6], args[7]
    inp = L.PackedRegionInputs(1, 0, 0, C.cast((C.c_int32 * 1)(*nt), C.c_void_p), C.cast((C.c_int32 * 1)(*nb), C.c_void_p),
                               args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(), args[3].data_ptr(), args[4].data_ptr(),
                               args[5].data_ptr(), None)
    logits = torch.full((4096,), 7.0, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cases = [((VQA, 0, 1, -1, 3, 31), b"entry range"), ((VQA, 0, 1, -1, 5, 4), b"entry range"), ((VQA, 0, 2, -1, 0, 1), b"n_images"),
             ((NLVR2, 0, 1, -1, 0, 1), b"n_images"), ((9, 0, 1, -1, 0, 1), b"unknown family"), ((VQA, 0, 1, 5000, 0, 1), b"answer")]
    for msg, needle in cases:
        arr = (L.HeadAblationMessage * 1)(L.HeadAblationMessage(*msg))
        rc = L.load().vb200_head_ablation(model._handle, C.byref(inp), arr, 1, logits.data_ptr(), None, 0, st)
        assert rc == ERR_INVALID and needle in L.load().vb200_last_error(model._handle), msg
    arr = (L.HeadAblationMessage * 1)(L.HeadAblationMessage(VQA, 0, 1, -1, 0, 1))
    assert L.load().vb200_head_ablation(model._handle, C.byref(inp), arr, 0, logits.data_ptr(), None, 0, st) == ERR_INVALID
    assert L.load().vb200_head_ablation(model._handle, C.byref(inp), arr, 1, None, None, 0, st) == ERR_INVALID
    torch.cuda.synchronize()
    assert torch.all(logits == 7.0)
    exact = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        with pytest.raises(L.VilbertB200Error, match="split_fp32"):
            exact.head_ablation(*args, [(VQA, 0, 1, None, (0, 1))])
    finally:
        exact.close()


def test_worker_answers_match_custom_prediction_packed(tiny):
    from vilbert_b200 import worker_api as W
    model = tiny["bf16"]
    vocab = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "a", "dog"])}
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(vocab)
    W.model = model

    def det(counts, seed):
        imgs = _batch(model, [(3, counts)], seed=seed)
        return [im[2] for im in imgs], [{"image_width": float(im[4][0]), "image_height": float(im[4][1]), "bbox": im[3].numpy()}
                                        for im in imgs]

    reqs = [("what is the man", [1], *det([12], 1), "1"), ("a dog", [12], *det([5, 6], 2), "12"), ("the man", [11], *det([9], 3), "11")]
    got = W.custom_head_ablation_packed(reqs, entries=(0, 2))
    want = W.custom_prediction_packed(reqs, decode="device")
    for g, w in zip(got, want):
        assert g["answer"] == w
        hp = g["ablation"]["head_prob"]
        assert not torch.isnan(hp[:2, :2]).any() and torch.isnan(hp[2:]).all()
