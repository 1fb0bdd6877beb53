"""Coalition ablation and Shapley values (vb200_coalition_ablation / vb200_shapley_values / VILBertForVLTasks.coalition_ablation /
.shapley / worker_api.custom_shapley_packed).  `-m gpu` only.

A coalition variant is the engine's own forward of a well-defined input in the worker's layout -- the message's question with the
absent units' positions replaced by [MASK] on every image, each image without the absent units' boxes -- so every segment is
compared bit for bit with forward_regions_packed of that input built on the host.  The estimator is compared bit for bit with the
numpy float64 restatement on the engine's own values, and with exact Shapley values where every permutation is enumerated.
"""
import ctypes as C
import itertools
import math
import random

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 / bf16 vs the fp32 oracle (test_gpu_regions_packed.py)
MASK = 103
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6
POOLED = 1 | 2 | 4 | 8 | 16
HEAD = {VQA: 0, GQA: 1, SNLI: 4}
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
    """The worker's layout: per group (tin, [boxes per image]) the group's text repeated on each of its images."""
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


def _units(model, imgs, msg, units):
    from vilbert_b200 import model as M
    _, ib, K = msg[:3]
    return M.coalition_units(units, len(imgs[ib][0]), sum(imgs[ib + k][2].shape[0] for k in range(K)))


def _coalition_samples(imgs, msg, units, present):
    """The coalition's samples built on the host: the masked question on each image, each image's kept boxes."""
    _, ib, K = msg[:3]
    q, seg, task = imgs[ib][0].clone(), imgs[ib][1], imgs[ib][5]
    gone_b = set()
    for u, (ps, bs) in enumerate(units):
        if not present[u]:
            for p in ps:
                q[p] = MASK
            gone_b.update(bs)
    out, b0 = [], 0
    for k in range(K):
        f, bx, wh = imgs[ib + k][2:5]
        keep = torch.tensor([b0 + j not in gone_b for j in range(f.shape[0])])
        out.append((q, seg, f[keep], bx[keep], wh, task))
        b0 += f.shape[0]
    return out


def _reference(model, imgs, msg, units, coalitions):
    """forward_regions_packed of the full input and every host-built coalition: each one's segment."""
    fam, ib, K = msg[:3]
    rows = [[True] * len(units)] + [list(map(bool, c)) for c in coalitions]
    var = [_coalition_samples(imgs, msg, units, c) for c in rows]
    samples = [s for v in var for s in v]
    out, _ = model.forward_regions_packed(*support.packed_image_args(samples), select=POOLED, return_spatials=False)
    torch.cuda.synchronize()
    segs, at = [], 0
    for v in var:
        segs.append(out[HEAD[fam]][at] if fam in HEAD else out[3][at // 2] if fam == NLVR2 else out[2][at:at + K].reshape(-1))
        at += len(v)
    return segs


def _random_coalitions(rng, units, imgs, msg, n):
    """n random presence rows, each keeping at least one box of every image (an image without boxes is tested on its own)."""
    _, ib, K = msg[:3]
    counts = [imgs[ib + k][2].shape[0] for k in range(K)]
    first = [sum(counts[:k]) for k in range(K + 1)]
    out = []
    while len(out) < n:
        row = [rng.random() < 0.5 for _ in units]
        kept = [0] * K
        boxes_kept = set(b for u, (_, bs) in enumerate(units) if row[u] for b in bs)
        owned = set(b for _, bs in units for b in bs)
        for k in range(K):
            kept[k] = sum(1 for b in range(first[k], first[k + 1]) if b in boxes_kept or b not in owned)
        if min(kept) >= 1:
            out.append(row)
    return out


def _check(model, imgs, msgs, units, coalitions, res):
    """Bitwise segments, and scores as the decode's softmax of each segment."""
    for msg, us, cs, r in zip(msgs, units, coalitions, res):
        want = _reference(model, imgs, msg, us, cs)
        got = r["logits"]
        assert len(got) == len(want) == 1 + len(cs)
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), f"message {msg}: variant {k} differs from forward_regions_packed of its input"
        flat = torch.cat(got).reshape(-1, 1).contiguous()
        out = [None] * 10
        out[2] = flat
        offs = [0]
        for s in got:
            offs.append(offs[-1] + s.numel())
        dec = model.decode_answers(out, [(RET, offs[k], s.numel(), min(10, s.numel()), None) for k, s in enumerate(got)])
        col = dec[0][0][0] if len(msg) < 4 or msg[3] is None else msg[3]
        assert r["answer"] == col and r["top1"] == dec[0][0][0] and r["top1_prob"] == dec[0][1][0]
        probs = [r["prob"]] + r["coalition_prob"].tolist()
        for k, ((idx, p, _), seg) in enumerate(zip(dec, got)):
            if k > 0:
                assert int(r["coalition_top1"][k - 1]) == idx[0]
            if col in idx:                                       # the decode reports it: the same arithmetic, the same bits
                assert probs[k] == p[idx.index(col)], f"message {msg}: variant {k} prob"
            else:
                assert abs(probs[k] - float(torch.softmax(seg.double(), 0)[col])) <= 1e-6


GROUPS = [(8, [5, 7]), (10, [4]), (6, [3, 9, 2]), (7, [6]), (5, [3]), (9, [5])]


def _messages(first):
    return [(NLVR2, first[0], 2), (VQA, first[1], 1, 17), (RET, first[2], 3), (GQA, first[3], 1), (SNLI, first[4], 1),
            (RET, first[5], 1)]


@pytest.mark.parametrize("mode", ["fp16", "bf16"])
def test_every_family_bitwise_and_scores(tiny, mode):
    model = tiny[mode]
    imgs, first = _batch(model, GROUPS, seed=5)
    msgs = _messages(first)
    custom = [None, [((1, 2), (0,)), ((3,), ()), ((), (1, 2, 3))], [((1,), (0, 5)), ((2, 3), ()), ((), tuple(range(6, 14)))],
              None, [((1, 2, 3), (1, 2))], None]
    units = [_units(model, imgs, m, u) for m, u in zip(msgs, custom)]
    rng = random.Random(3)
    coal = [_random_coalitions(rng, us, imgs, m, 6) + [[True] * len(us)] for m, us in zip(msgs, units)]
    res = model.coalition_ablation(*support.packed_image_args(imgs), msgs, custom, coal, mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    _check(model, imgs, msgs, units, coal, res)
    for r, us in zip(res, units):
        assert r["units"] == us


def test_full_model(full):
    model = full
    imgs, first = _batch(model, [(37, [100]), (20, [30, 40])], seed=11)
    msgs = [(VQA, first[0], 1), (NLVR2, first[1], 2)]
    units = [_units(model, imgs, m, None) for m in msgs]
    rng = random.Random(5)
    coal = [_random_coalitions(rng, us, imgs, m, 5) for m, us in zip(msgs, units)]
    res = model.coalition_ablation(*support.packed_image_args(imgs), msgs, [None, None], coal, mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    _check(model, imgs, msgs, units, coal, res)


def test_past_256_rows(tiny_long):
    model = tiny_long
    imgs, first = _batch(model, [(150, [280]), (40, [270, 5])], seed=13)
    msgs = [(VQA, first[0], 1), (RET, first[1], 2)]
    custom = [[(tuple(range(1, 75)), tuple(range(0, 140))), (tuple(range(75, 149)), ())], None]
    units = [_units(model, imgs, m, u) for m, u in zip(msgs, custom)]
    rng = random.Random(7)
    coal = [_random_coalitions(rng, us, imgs, m, 3) for m, us in zip(msgs, units)]
    res = model.coalition_ablation(*support.packed_image_args(imgs), msgs, custom, coal, mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    _check(model, imgs, msgs, units, coal, res)


def test_empty_image_is_the_global_row_alone(tiny):
    """Every box of the image absent: bit-identical to forward_packed of the one-row image (zero features, location 0, 0, 1, 1, 1)."""
    for mode in ("fp16", "bf16"):
        model = tiny[mode]
        imgs, _ = _batch(model, [(9, [6])], seed=17)
        units = [((2,), ()), ((), tuple(range(6))), ((4, 5), ())]
        coal = [[False, False, True], [True, False, False], [False, False, False]]
        res = model.coalition_ablation(*support.packed_image_args(imgs), [(VQA, 0, 1)], [units], [coal], mask_token=MASK,
                                       return_logits=True)
        F = model._dims["v_feature_size"]
        qs = []
        for c in coal:
            q = imgs[0][0].clone()
            for u, (ps, _) in enumerate(units):
                if not c[u]:
                    q[list(ps)] = MASK
            qs.append(q)
        n = len(qs)
        out = model.forward_packed(torch.cat(qs).cuda(), torch.zeros(n, F).cuda(), torch.tensor([[0., 0., 1., 1., 1.]] * n).cuda(),
                                   imgs[0][1].repeat(n).cuda(), torch.tensor([[imgs[0][5]]] * n).cuda(), [len(q) for q in qs], [1] * n)
        torch.cuda.synchronize()
        for k in range(n):
            assert torch.equal(res[0]["logits"][1 + k], out[0][k]), f"{mode}: coalition {k}"


def test_single_unit_coalitions_match_message_ablation(tiny):
    """All units but one present: the variants of message ablation, bit for bit (segments and probabilities)."""
    model = tiny["bf16"]
    imgs, first = _batch(model, [(8, [5, 7]), (10, [4])], seed=23)
    msgs = [(NLVR2, first[0], 2), (VQA, first[1], 1)]
    ab = model.message_ablation(*support.packed_image_args(imgs), msgs, mask_token=MASK, return_logits=True)
    units = [_units(model, imgs, m, None) for m in msgs]
    coal = [(~torch.eye(len(us), dtype=torch.bool)).tolist() for us in units]
    res = model.coalition_ablation(*support.packed_image_args(imgs), msgs, [None, None], coal, mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    for a, r in zip(ab, res):
        assert len(a["logits"]) == len(r["logits"])
        for x, y in zip(a["logits"], r["logits"]):
            assert torch.equal(x, y)
        assert r["prob"] == a["prob"] and r["answer"] == a["answer"]
        assert torch.equal(r["coalition_prob"], torch.cat([a["token_prob"], a["box_prob"]]))


def _values(model, imgs, msgs, res):
    """The engine's own coalition values for shapley's permutations: v(empty), v(all), the chains."""
    from vilbert_b200 import model as M
    out = []
    for m, r in zip(msgs, res):
        chain = M.shapley_chain(r["perm"])
        c = model.coalition_ablation(*support.packed_image_args(imgs), [m], [r["units"]], [chain], mask_token=MASK)[0]
        assert c["prob"] == r["prob"] and float(c["coalition_prob"][0]) == r["empty_prob"]
        out.append(np.concatenate([c["coalition_prob"][:1].numpy(), np.float32([c["prob"]]), c["coalition_prob"][1:].numpy()]))
    return out


def test_estimator_bitwise_efficiency_dummy_and_seed(tiny):
    from vilbert_b200 import model as M
    model = tiny["fp16"]
    imgs, first = _batch(model, [(9, [6]), (7, [4, 5]), (6, [3, 2, 4])], seed=29)
    q = imgs[0][0].clone()
    q[3] = MASK                                                  # a position that already holds the mask token: a dummy unit
    imgs[0] = (q,) + imgs[0][1:]
    msgs = [(VQA, first[0], 1), (NLVR2, first[1], 2), (RET, first[2], 3)]
    for P, anti in ((8, True), (6, False), (2, True)):
        res = model.shapley(*support.packed_image_args(imgs), msgs, permutations=P, seed=4, antithetic=anti, mask_token=MASK)
        torch.cuda.synchronize()
        for r, v in zip(res, _values(model, imgs, msgs, res)):
            phi, se = M.shapley_reference(v, r["perm"].numpy(), 2 if anti else 1)
            assert np.array_equal(r["phi"].numpy(), phi, equal_nan=True) and np.array_equal(r["stderr"].numpy(), se, equal_nan=True)
            total = float(r["phi"].double().sum())
            assert abs(total - (r["prob"] - r["empty_prob"])) <= 4e-7 * len(r["units"]), (total, r["prob"], r["empty_prob"])
        dummy = res[0]["units"].index(((3,), ()))
        assert res[0]["phi"][dummy] == 0.0
        if P // (2 if anti else 1) >= 2:
            assert res[0]["stderr"][dummy] == 0.0
        else:
            assert math.isnan(float(res[0]["stderr"][dummy]))
        again = model.shapley(*support.packed_image_args(imgs), msgs, permutations=P, seed=4, antithetic=anti, mask_token=MASK)
        for a, b in zip(res, again):
            assert torch.equal(a["phi"], b["phi"]) and torch.equal(a["stderr"].nan_to_num(-1), b["stderr"].nan_to_num(-1))
            assert torch.equal(a["perm"], b["perm"])


def test_exact_with_every_permutation(tiny):
    """4 units and all 24 permutations: phi equals exact Shapley from the 16 coalition values of one call."""
    import vilbert_b200 as vb
    from vilbert_b200 import model as M
    model = tiny["bf16"]
    imgs, _ = _batch(model, [(8, [6])], seed=31)
    units = [((1, 2), ()), ((3,), (0, 1)), ((), (2, 3, 4)), ((4, 5), (5,))]
    subsets = [[bool(s >> u & 1) for u in range(4)] for s in range(16)]
    c = model.coalition_ablation(*support.packed_image_args(imgs), [(VQA, 0, 1)], [units], [subsets], mask_token=MASK)[0]
    v = c["coalition_prob"].double().numpy()
    assert float(c["coalition_prob"][15]) == c["prob"]
    exact = np.zeros(4)
    for u in range(4):
        for s in range(16):
            if not s >> u & 1:
                k = bin(s).count("1")
                exact[u] += math.factorial(k) * math.factorial(3 - k) / 24 * (v[s | 1 << u] - v[s])
    perm = np.array(list(itertools.permutations(range(4))), dtype=np.int64)
    vals = [v[0], v[15]]
    for p in perm:
        s = 0
        for j in range(3):
            s |= 1 << int(p[j])
            vals.append(v[s])
    vals = np.float32(vals)
    est = M.shapley_reference(vals, perm, 1, dtype=np.float64)[0]
    assert np.abs(est - exact).max() <= 1e-12
    phi = torch.empty(4, device="cuda")
    se = torch.empty(4, device="cuda")
    pd = torch.from_numpy(perm).to(device="cuda", dtype=torch.int32)
    vd = torch.from_numpy(vals).cuda()
    arr = (vb._lib.ShapleyMessage * 1)(vb._lib.ShapleyMessage(4, 24, 1, 0, 0, 0))
    model._call("vb200_shapley_values", arr, 1, pd.data_ptr(), vd.data_ptr(), phi.data_ptr(), se.data_ptr())
    assert np.array_equal(phi.cpu().numpy(), est.astype(np.float32))


def _raw(model, imgs, msgs, logits, scores, mask=MASK, n_msgs=None, bf=None):
    """vb200_coalition_ablation with engine messages (family, ib, K, answer, units, bitmaps); returns (rc, last error)."""
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    a = support.packed_image_args(imgs)
    arr, keep = model._coalition_structs([m[:4] for m in msgs], [m[4] for m in msgs], [m[5] for m in msgs])
    ptrs = [t.data_ptr() for t in a[:6]]
    if bf is not None:
        ptrs[3] = bf
    inp = L.PackedRegionInputs(len(a[6]), 0, 0, vb.model._int32s(a[6]), vb.model._int32s(a[7]), *ptrs, None)
    with torch.cuda.device(0):
        rc = L.load().vb200_coalition_ablation(model._handle, C.byref(inp), arr, len(msgs) if n_msgs is None else n_msgs, mask,
                                              logits.data_ptr() if logits is not None else None,
                                              scores.data_ptr() if scores is not None else None, 0,
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, (L.load().vb200_last_error(model._handle) or b"").decode()


def test_rejections(tiny, tiny_oracle):
    """Every rejection is VB200_ERR_INVALID, names its cause and message or unit, and leaves the sentinel outputs untouched."""
    from vilbert_b200 import model as M
    model = tiny["fp16"]
    imgs, _ = _batch(model, [(6, [3, 4]), (5, [1]), (7, [2])], seed=41)
    logits = torch.full((4096,), 7.0, device="cuda")
    scores = torch.full((256, 4), 7, dtype=torch.int32, device="cuda")
    u2 = [((1,), ()), ((), (0, 4))]
    bm = lambda rows, n: M.coalition_bitmaps(rows, n)
    ok = (NLVR2, 0, 2, -1, u2, bm([[True, False]], 2))
    cases = [
        ([(GRD, 2, 1, -1, u2[:1], bm([[True]], 1))], "message 0 is a grounding message"),
        ([(99, 0, 1, -1, u2, bm([[True, False]], 2))], "message 0 has unknown family"),
        ([ok, (VQA, 2, 2, -1, u2, bm([[True, False]], 2))], "message 1 (family 1) has n_images 2"),
        ([(RET, 3, 2, -1, u2, bm([[True, False]], 2))], "outside the batch"),
        ([(VQA, 0, 1, 9999, u2[:1], bm([[True]], 1))], "message 0 has answer 9999"),
        ([(VQA, 0, 1, -1, [((1,), ()), ((), ())], bm([[True, True]], 2))], "message 0 unit 1 is empty"),
        ([(VQA, 0, 1, -1, [((6,), ())], bm([[True]], 1))], "message 0 unit 0 has position 6 outside [0, 6)"),
        ([(VQA, 0, 1, -1, [((1,), (3,))], bm([[True]], 1))], "message 0 unit 0 has box 3 outside [0, 3)"),
        ([(NLVR2, 0, 2, -1, [((1,), (6,)), ((2,), (6,))], bm([[True, True]], 2))], "message 0 unit 1 has box 6, which unit 0"),
        ([(NLVR2, 0, 2, -1, [((1, 2), ()), ((2,), ())], bm([[True, True]], 2))], "message 0 unit 1 has position 2, which unit 0"),
        ([(VQA, 0, 1, -1, u2[:1], np.array([[3]], dtype=np.uint64))], "message 0 coalition 0 sets a bit at or past n_units 1"),
        ([(VQA, 0, 1, -1, [((1,), ())] * 0, np.zeros((0, 0), dtype=np.uint64))], "n_units 0"),
        ([(VQA, 0, 1, -1, [((), (j % 3,)) for j in range(1025)], np.zeros((0, 17), dtype=np.uint64))], "n_units 1025"),
    ]
    for msgs, match in cases:
        rc, msg = _raw(model, imgs, msgs, logits, scores)
        assert rc == -1 and match in msg, (match, rc, msg)
        assert bool((logits == 7.0).all()) and bool((scores == 7).all()), match
    for kw, match in [(dict(n_msgs=0), "n_msgs"), (dict(mask=model._dims["vocab_size"]), "mask_token"), (dict(logits=None), "NULL")]:
        rc, msg = _raw(model, imgs, [ok], kw.pop("logits", logits), scores, **kw)
        assert rc == -1 and match in msg, (match, msg)
    big, _ = _batch(model, [(37, [100])], seed=43)
    us = [((), (j,)) for j in range(100)]
    rc, msg = _raw(model, big, [(VQA, 0, 1, -1, us, bm([[True] * 100] * 1100, 100))], logits, scores)
    assert rc == -1 and "above 1024" in msg, msg
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        rc, msg = _raw(x, imgs, [ok], logits, scores)
        assert rc == -1 and "split_fp32" in msg
    finally:
        x.close()
    assert bool((logits == 7.0).all()) and bool((scores == 7).all())
    # the estimator's own rejections
    import vilbert_b200 as vb
    L = vb._lib
    phi = torch.full((8,), 7.0, device="cuda")
    perm = torch.zeros(64, dtype=torch.int32, device="cuda")
    for d, match in [((0, 2, 1, 0, 0, 0), "n_units 0"), ((2, 0, 1, 0, 0, 0), "n_perm 0"), ((2, 2, 3, 0, 0, 0), "group 3"),
                     ((2, 3, 2, 0, 0, 0), "not a multiple"), ((2, 2, 1, -1, 0, 0), "negative offset")]:
        arr = (L.ShapleyMessage * 1)(L.ShapleyMessage(*d))
        with torch.cuda.device(0):
            rc = L.load().vb200_shapley_values(model._handle, arr, 1, perm.data_ptr(), phi.data_ptr(), phi.data_ptr(), phi.data_ptr(),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -1 and match in L.load().vb200_last_error(model._handle).decode()
    torch.cuda.synchronize()
    assert bool((phi == 7.0).all())


def test_plans_shared_forwards_unchanged_and_no_synchronisation(tiny):
    model = tiny["bf16"]
    imgs, first = _batch(model, GROUPS, seed=47)
    a = support.packed_image_args(imgs)
    fwd = lambda: model.forward_regions_packed(*a, max_tokens=20, max_boxes=30)[0][0].clone()
    before = fwd()
    # retrieval left out: a message-ablation box variant of it runs the changed image alone, so its sample count differs
    msgs = [(m[0], m[1], m[2]) for m in _messages(first) if m[0] != RET]
    model.message_ablation(*a, msgs, mask_token=MASK, max_tokens=20, max_boxes=30)
    n = support.n_plans(model)
    units = [_units(model, imgs, m, None) for m in msgs]
    single = [(~torch.eye(len(us), dtype=torch.bool)).tolist() for us in units]      # message ablation's samples, as coalitions
    model.coalition_ablation(*a, msgs, [None] * len(msgs), single, mask_token=MASK, max_tokens=20, max_boxes=30)
    assert support.n_plans(model) == n
    rng = random.Random(9)
    coal = [_random_coalitions(rng, us, imgs, m, 4) for m, us in zip(msgs, units)]
    r1 = model.coalition_ablation(*a, msgs, [None] * len(msgs), coal, mask_token=MASK, max_tokens=20, max_boxes=30, return_logits=True)
    model.shapley(*a, msgs[:2], permutations=2, mask_token=MASK, max_tokens=20, max_boxes=30)
    n = support.n_plans(model)
    model.shapley(*a, msgs[:2], permutations=2, seed=1, mask_token=MASK, max_tokens=20, max_boxes=30)
    assert support.n_plans(model) == n
    assert torch.equal(fwd(), before)
    # the same calls back to back without synchronisation, against one call at a time
    from vilbert_b200 import model as M
    raw = [[(*msgs[i], -1, units[i], M.coalition_bitmaps(coal[i], len(units[i])))] for i in range(len(msgs))]

    def run(sync):
        outs = []
        for m in raw:
            arr, keep = model._coalition_structs([x[:4] for x in m], [x[4] for x in m], [x[5] for x in m])
            recs, nf = model._coalition_layout(a[6], a[7], arr)
            logits = torch.full((nf,), float("nan"), device="cuda")
            scores = torch.zeros(len(recs), 4, dtype=torch.int32, device="cuda")
            from vilbert_b200 import _lib as L
            import vilbert_b200 as vb
            inp = L.PackedRegionInputs(len(a[6]), 20, 30, vb.model._int32s(a[6]), vb.model._int32s(a[7]), *[t.data_ptr() for t in a[:6]],
                                       None)
            model._call("vb200_coalition_ablation", C.byref(inp), arr, 1, MASK, logits.data_ptr(), scores.data_ptr(), 0)
            if sync:
                torch.cuda.synchronize()
            outs.append((logits, scores, arr, keep, inp))
        torch.cuda.synchronize()
        return outs

    for (la, sa, *_), (lb, sb, *_), r in zip(run(False), run(True), r1):
        assert torch.equal(la, lb) and torch.equal(sa, sb)
        assert torch.equal(la, torch.cat(r["logits"]))


def test_against_the_oracle(tiny, tiny_oracle):
    """Host-built coalitions of a VQA message through the fp32 oracle: the engine's segments within the packed tests' tolerance."""
    from vilbert_b200 import worker_api as W
    model = tiny["fp16"]
    imgs, _ = _batch(model, [(10, [6])], seed=53)
    units = [((1, 2), (0,)), ((3, 4), (1, 2)), ((), (3, 4, 5))]
    coal = [[True, False, True], [False, True, False], [False, False, True]]
    res = model.coalition_ablation(*support.packed_image_args(imgs), [(VQA, 0, 1)], [units], [coal], mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    for k, c in enumerate(coal):
        (q, seg, f, bx, wh, task), = _coalition_samples(imgs, (VQA, 0, 1), units, c)
        info = {"image_width": float(wh[0]), "image_height": float(wh[1]), "bbox": bx.numpy()}
        _, ff, ss, _, _, _, _, _ = W.build_inputs("", [task], [f], [info], torch.device("cpu"), W.WordpieceTokenizer(VOCAB))
        ref = tiny_oracle(q[None], ff, ss, seg[None], torch.ones(1, len(q), dtype=torch.long),
                          torch.ones(1, ff.shape[1], dtype=torch.uint8), None, torch.tensor([[task]]), compute_pretraining_heads=False)
        err = float((res[0]["logits"][1 + k].cpu() - ref[0][0]).abs().max())
        assert err < TOL, f"coalition {k} vs fp32 oracle: {err} >= {TOL}"


def test_worker_agrees_with_model_shapley(tiny):
    from vilbert_b200 import worker_api as W
    model = tiny["bf16"]
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = model

    def det(counts, seed):
        imgs, _ = _batch(model, [(3, counts)], seed=seed)
        return [im[2] for im in imgs], [{"image_width": float(im[4][0]), "image_height": float(im[4][1]), "bbox": im[3].numpy()}
                                        for im in imgs]

    reqs = [("what is the man holding ?", [1], *det([5], 1), "1"), ("a dog on the grass", [12], *det([3, 4], 2), "12"),
            ("the man", [11], *det([4], 3), "11"), ("a dog", [7], *det([2, 1, 3], 4), "7")]
    got = W.custom_shapley_packed(reqs, permutations=4, seed=2)
    want = W.custom_prediction_packed(reqs, decode="device")
    p = W.pack_region_requests(reqs)
    args = (p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"], p["image_wh"], p["n_tokens"], p["n_boxes"])
    msgs = [m[:4] for i, m in W.ablation_messages(reqs, p["spans"]).items() if reqs[i][4] != "11"]
    sh = model.shapley(*args, msgs, permutations=4, seed=2, mask_token=W.tokenizer.vocab.get("[MASK]", 103),
                       max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
    assert isinstance(got[2], ValueError)
    for i, s in zip([0, 1, 3], sh):
        assert got[i]["answer"] == want[i]
        g = got[i]["shapley"]
        assert torch.equal(g["phi"], s["phi"]) and g["units"] == s["units"]
        assert len(g["box_pixels"]) == len(g["units"])
