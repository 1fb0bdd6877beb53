"""Shapley-Taylor pair indices (vb200_interaction_values / VILBertForVLTasks.shapley_interactions /
worker_api.custom_interactions_packed).  `-m gpu` only.

The coalitions are coalition ablation's, checked bit for bit in test_gpu_shapley.py, so this suite checks what the new call adds:
the estimator bit for bit against the numpy float64 restatement on the engine's own coalition values, the exact index where every
permutation is enumerated, the value layout, pair order, dummy units, seeds, plans, rejections and the worker.
"""
import ctypes as C
import itertools
import math

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

MASK = 103
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6
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


def _lib():
    from vilbert_b200 import _lib as L
    return L


def _engine_values(model, imgs, msgs, res):
    """The engine's own coalition values for each result's permutations and pairs, in the call's layout: v(empty), v(all), the
    chains, then x1, x2 per permutation and pair (one coalition_ablation call per message)."""
    from vilbert_b200 import model as M
    out = []
    for m, r in zip(msgs, res):
        coal = torch.cat([M.shapley_chain(r["perm"]), M.interaction_coalitions(r["perm"], r["pairs"])])
        c = model.coalition_ablation(*support.packed_image_args(imgs), [m], [r["units"]], [coal], mask_token=MASK)[0]
        assert c["prob"] == r["prob"] and float(c["coalition_prob"][0]) == r["empty_prob"]
        out.append(np.concatenate([c["coalition_prob"][:1].numpy(), np.float32([c["prob"]]), c["coalition_prob"][1:].numpy()]))
    return out


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def test_estimator_bitwise_phi_layout_pair_order_dummy_and_seed(tiny):
    from vilbert_b200 import model as M
    for mode in ("fp16", "bf16"):
        model = tiny[mode]
        imgs, first = _batch(model, [(9, [6]), (7, [4, 5]), (6, [3, 2, 4])], seed=29)
        q = imgs[0][0].clone()
        q[3] = MASK                                                  # a position that already holds the mask token: a dummy unit
        imgs[0] = (q,) + imgs[0][1:]
        msgs = [(VQA, first[0], 1), (NLVR2, first[1], 2), (RET, first[2], 3)]
        # retrieval: a pair, its reverse and a duplicate, an adjacent-rank-prone pair of word units, a box pair
        pairs = ["cross", [(0, 5), (1, 7), (3, 12)], [(0, 5), (5, 0), (0, 5), (1, 2), (6, 10)]]
        adjacent = 0
        for P, anti in ((8, True), (6, False), (2, True)):
            g = 2 if anti else 1
            kw = dict(permutations=P, seed=4, antithetic=anti, mask_token=MASK)
            res = model.shapley_interactions(*support.packed_image_args(imgs), msgs, pairs, **kw)
            torch.cuda.synchronize()
            sh = model.shapley(*support.packed_image_args(imgs), msgs, **kw)
            for r, s, v in zip(res, sh, _engine_values(model, imgs, msgs, res)):
                assert torch.equal(r["perm"], s["perm"]) and r["units"] == s["units"]
                assert _same(r["phi"], s["phi"]) and _same(r["stderr"], s["stderr"]), f"{mode} P={P}: phi differs from shapley"
                inter, se = M.interaction_reference(v, r["perm"].numpy(), r["pairs"].numpy(), g)
                assert _same(r["interaction"], inter) and _same(r["interaction_stderr"], se), f"{mode} P={P}: estimator"
                n, Q = len(r["units"]), len(r["pairs"])
                assert len(v) == 2 + P * (n - 1) + 2 * P * Q
                # layout: a pair adjacent in a permutation has x2 = the chain value two past r
                c = np.concatenate([v[:1].reshape(1, 1).repeat(P, 0), v[2:2 + P * (n - 1)].reshape(P, n - 1),
                                    v[1:2].reshape(1, 1).repeat(P, 0)], 1)
                x = v[2 + P * (n - 1):].reshape(P, Q, 2)
                rank = np.argsort(r["perm"].numpy(), 1)
                for p in range(P):
                    for k, (a, b) in enumerate(r["pairs"].tolist()):
                        if abs(rank[p, a] - rank[p, b]) == 1:
                            assert x[p, k, 1] == c[p, min(rank[p, a], rank[p, b]) + 2]
                            adjacent += 1
            assert res[0]["pairs"].tolist() == [list(p) for p in M.cross_pairs(res[0]["units"])]
            # pair order and duplicates: the same bits
            ri = res[2]["interaction"].view(torch.int32)
            assert ri[0] == ri[1] == ri[2]
            assert res[2]["interaction_stderr"][:3].view(torch.int32).unique().numel() == 1
            # the dummy unit: every pair with it exactly 0, its standard error 0 (NaN with one group)
            dummy = res[0]["units"].index(((3,), ()))
            with_dummy = [k for k, (a, b) in enumerate(res[0]["pairs"].tolist()) if dummy in (a, b)]
            assert with_dummy and all(float(res[0]["interaction"][k]) == 0.0 for k in with_dummy)
            for k in with_dummy:
                se = float(res[0]["interaction_stderr"][k])
                assert se == 0.0 if P // g >= 2 else math.isnan(se)
            again = model.shapley_interactions(*support.packed_image_args(imgs), msgs, pairs, **kw)
            for a, b in zip(res, again):
                for key in ("interaction", "interaction_stderr", "phi", "stderr", "perm", "pairs"):
                    assert _same(a[key], b[key]), key
                assert a["samples"] == b["samples"]
        assert adjacent > 0


def _subset_values(v, perm, pairs):
    """The call's value layout from the values of every subset (bit u of the index: unit u present)."""
    from vilbert_b200 import model as M
    n = perm.shape[1]
    out = [v[0], v[(1 << n) - 1]]
    for p in perm:
        s = 0
        for j in range(n - 1):
            s |= 1 << int(p[j])
            out.append(v[s])
    for row in M.interaction_coalitions(torch.from_numpy(perm), pairs).int().numpy():
        out.append(v[int(sum(int(b) << u for u, b in enumerate(row)))])
    return np.float32(out)


def _call(model, descs, perm, vals, inter, se, n_msgs=None):
    """vb200_interaction_values on the current stream; returns (rc, last error)."""
    L = _lib()
    arr = (L.InteractionMessage * max(len(descs), 1))(*descs)
    ptr = lambda t: t if t is None or isinstance(t, int) else t.data_ptr()
    with torch.cuda.device(0):
        rc = L.load().vb200_interaction_values(model._handle, arr, len(descs) if n_msgs is None else n_msgs, ptr(perm), ptr(vals),
                                               ptr(inter), ptr(se), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, (L.load().vb200_last_error(model._handle) or b"").decode()


def test_exact_with_every_permutation(tiny):
    """4 units, all 24 permutations, all 6 pairs: the index from the 16 coalition values of one call, exact within 1e-12."""
    from vilbert_b200 import model as M
    L = _lib()
    model = tiny["bf16"]
    imgs, _ = _batch(model, [(8, [6])], seed=31)
    units = [((1, 2), ()), ((3,), (0, 1)), ((), (2, 3, 4)), ((4, 5), (5,))]
    subsets = [[bool(s >> u & 1) for u in range(4)] for s in range(16)]
    c = model.coalition_ablation(*support.packed_image_args(imgs), [(VQA, 0, 1)], [units], [subsets], mask_token=MASK)[0]
    v32 = c["coalition_prob"].numpy()
    v = v32.astype(np.float64)
    perm = np.array(list(itertools.permutations(range(4))), dtype=np.int64)
    pairs = np.array(list(itertools.combinations(range(4), 2)), dtype=np.int32)
    vals = _subset_values(v32, perm, pairs)
    exact = np.zeros(6)
    for k, (a, b) in enumerate(pairs):
        for T in range(16):
            if not (T >> a & 1 or T >> b & 1):
                t = bin(T).count("1")
                exact[k] += 2 * math.factorial(t) * math.factorial(3 - t) / 24 * (v[T | 1 << a | 1 << b] - v[T | 1 << a] - v[T | 1 << b] + v[T])
    est, _ = M.interaction_reference(vals, perm, pairs, 1, dtype=np.float64)
    assert np.abs(est - exact).max() <= 1e-12
    assert abs(sum(v[1 << i] - v[0] for i in range(4)) + est.sum() - (v[15] - v[0])) <= 1e-12
    inter = torch.full((6,), 7.0, device="cuda")
    se = torch.full((6,), 7.0, device="cuda")
    d = L.InteractionMessage(4, 24, 1, 6, 0, 0, 0, pairs.ctypes.data)
    rc, msg = _call(model, [d], torch.from_numpy(perm).to(device="cuda", dtype=torch.int32), torch.from_numpy(vals).cuda(), inter, se)
    assert rc == 0, msg
    assert np.array_equal(inter.cpu().numpy(), est.astype(np.float32))
    assert np.array_equal(se.cpu().numpy(), M.interaction_reference(vals, perm, pairs, 1)[1])


def test_non_permutation_row_is_nan_for_its_message_only(tiny):
    from vilbert_b200 import model as M
    L = _lib()
    model = tiny["fp16"]
    rng = np.random.default_rng(5)
    n, P = 6, 4
    perms = [np.stack([rng.permutation(n) for _ in range(P)]) for _ in range(2)]
    perms[1][2, 3] = perms[1][2, 4]                                # row 2 of message 1 repeats a unit
    pairs = [np.array([(0, 1), (2, 5), (4, 3)], dtype=np.int32), np.array([(1, 2), (0, 5)], dtype=np.int32)]
    n_vals = 2 + P * (n - 1) + 2 * P * 3
    vals = np.float32(rng.random(n_vals + 2 + P * (n - 1) + 2 * P * 2))
    descs = [L.InteractionMessage(n, P, 2, 3, 0, 0, 0, pairs[0].ctypes.data),
             L.InteractionMessage(n, P, 2, 2, P * n, n_vals, 3, pairs[1].ctypes.data)]
    inter = torch.full((5,), 7.0, device="cuda")
    se = torch.full((5,), 7.0, device="cuda")
    perm_d = torch.from_numpy(np.concatenate(perms).reshape(-1)).to(device="cuda", dtype=torch.int32)
    rc, msg = _call(model, descs, perm_d, torch.from_numpy(vals).cuda(), inter, se)
    assert rc == 0, msg
    want = M.interaction_reference(vals[:n_vals], perms[0], pairs[0], 2)
    assert _same(inter[:3].cpu(), want[0]) and _same(se[:3].cpu(), want[1])
    assert torch.isnan(inter[3:]).all() and torch.isnan(se[3:]).all()


def test_full_model(full):
    from vilbert_b200 import model as M
    model = full
    imgs, first = _batch(model, [(37, [100])], seed=11)
    msgs = [(VQA, first[0], 1)]
    res = model.shapley_interactions(*support.packed_image_args(imgs), msgs, [[(0, 35), (3, 100), (10, 134), (20, 21)]],
                                     permutations=2, seed=3, mask_token=MASK)
    torch.cuda.synchronize()
    r, = res
    assert len(r["units"]) == 135
    v, = _engine_values(model, imgs, msgs, res)
    inter, se = M.interaction_reference(v, r["perm"].numpy(), r["pairs"].numpy(), 2)
    assert _same(r["interaction"], inter) and _same(r["interaction_stderr"], se)


def test_past_256_rows(tiny_long):
    from vilbert_b200 import model as M
    model = tiny_long
    imgs, first = _batch(model, [(150, [280])], seed=13)
    msgs = [(VQA, first[0], 1)]
    units = [[(tuple(range(1, 50)), ()), (tuple(range(50, 100)), ()), (tuple(range(100, 149)), ()), ((), tuple(range(0, 140))),
              ((), tuple(range(140, 280)))]]
    res = model.shapley_interactions(*support.packed_image_args(imgs), msgs, ["cross"], units=units, permutations=4, seed=7,
                                     mask_token=MASK)
    torch.cuda.synchronize()
    r, = res
    assert r["pairs"].tolist() == [[0, 3], [0, 4], [1, 3], [1, 4], [2, 3], [2, 4]]
    v, = _engine_values(model, imgs, msgs, res)
    inter, se = M.interaction_reference(v, r["perm"].numpy(), r["pairs"].numpy(), 2)
    assert _same(r["interaction"], inter) and _same(r["interaction_stderr"], se)


def test_plans_unsynchronised_calls_and_rejections(tiny):
    from vilbert_b200 import model as M
    L = _lib()
    model = tiny["bf16"]
    imgs, first = _batch(model, [(8, [5, 7]), (10, [4])], seed=47)
    a = support.packed_image_args(imgs)
    # one VQA message of 12 units at P = 2: shapley runs 2 + 2 * 11 = 24 samples, the interactions 24 + 2 * 2 * Q, so both pad to 64
    msgs = [(VQA, first[1], 1)]
    kw = dict(permutations=2, mask_token=MASK, max_tokens=20, max_boxes=30)
    sh = model.shapley(*a, msgs, **kw)
    n = support.n_plans(model)
    pairs = [(i, 11 - i) for i in range(6)] + [(0, 1), (2, 3), (4, 8), (9, 10)]
    r = model.shapley_interactions(*a, msgs, [pairs], **kw)
    assert r[0]["samples"] == sh[0]["samples"] + 2 * 2 * 10 == 64
    assert support.n_plans(model) == n
    model.shapley_interactions(*a, msgs, [pairs[:5]], seed=5, **kw)
    assert support.n_plans(model) == n
    # back to back without synchronisation, against one call at a time
    rng = np.random.default_rng(9)
    jobs = []
    for k in range(4):
        nu, P, Q = 5 + k, 4, 3 + k
        perm = np.stack([rng.permutation(nu) for _ in range(P)])
        pairs = np.array([(i % nu, (i + 1 + k) % nu) for i in range(Q)], dtype=np.int32)
        vals = np.float32(rng.random(2 + P * (nu - 1) + 2 * P * Q))
        jobs.append((nu, P, Q, perm, pairs, vals))

    def run(sync):
        outs = []
        for nu, P, Q, perm, pairs, vals in jobs:
            inter = torch.full((Q,), float("nan"), device="cuda")
            se = torch.full((Q,), float("nan"), device="cuda")
            p = pairs.copy()
            rc, msg = _call(model, [L.InteractionMessage(nu, P, 1, Q, 0, 0, 0, p.ctypes.data)],
                            torch.from_numpy(perm.reshape(-1)).to(device="cuda", dtype=torch.int32), torch.from_numpy(vals).cuda(), inter, se)
            assert rc == 0, msg
            del p                                                  # the pairs are staged: the host array may go at once
            if sync:
                torch.cuda.synchronize()
            outs.append((inter, se))
        torch.cuda.synchronize()
        return outs

    for (ia, sa), (ib, sb), (_, P, _, perm, pairs, vals) in zip(run(False), run(True), jobs):
        assert _same(ia.cpu(), ib.cpu()) and _same(sa.cpu(), sb.cpu())
        want = M.interaction_reference(vals, perm, pairs, 1)
        assert _same(ia.cpu(), want[0]) and _same(sa.cpu(), want[1])
    # rejections: VB200_ERR_INVALID naming the message or pair, outputs untouched
    inter = torch.full((8,), 7.0, device="cuda")
    se = torch.full((8,), 7.0, device="cuda")
    perm = torch.zeros(64, dtype=torch.int32, device="cuda")
    vals = torch.zeros(256, device="cuda")
    ok_pairs = np.array([(0, 1)], dtype=np.int32)
    ok = (4, 2, 1, 1, 0, 0, 0, ok_pairs.ctypes.data)
    same = np.array([(1, 1)], dtype=np.int32)
    far = np.array([(0, 1), (0, 4)], dtype=np.int32)
    many = np.zeros((40000, 2), dtype=np.int32)
    many[:, 1] = 1
    cases = [
        ([(1, 2, 1, 1, 0, 0, 0, ok_pairs.ctypes.data)], "message 0 has n_units 1"),
        ([(1025, 2, 1, 1, 0, 0, 0, ok_pairs.ctypes.data)], "n_units 1025"),
        ([ok, (4, 0, 1, 1, 0, 0, 0, ok_pairs.ctypes.data)], "message 1 has n_perm 0"),
        ([(4, 2, 3, 1, 0, 0, 0, ok_pairs.ctypes.data)], "group 3"),
        ([(4, 3, 2, 1, 0, 0, 0, ok_pairs.ctypes.data)], "not a multiple"),
        ([(4, 2, 1, 1, 0, -1, 0, ok_pairs.ctypes.data)], "negative offset"),
        ([(4, 2, 1, 0, 0, 0, 0, ok_pairs.ctypes.data)], "message 0 has n_pairs 0"),
        ([(4, 2, 1, 1, 0, 0, 0, None)], "message 0 has NULL pairs"),
        ([ok, (4, 2, 1, 1, 0, 0, 0, same.ctypes.data)], "message 1 pair 0 pairs unit 1 with itself"),
        ([(4, 2, 1, 2, 0, 0, 0, far.ctypes.data)], "message 0 pair 1 (0, 4) has a unit outside [0, 4)"),
        ([(4, 2, 1, 40000, 0, 0, 0, many.ctypes.data)] * 2, "above 65536"),
    ]
    for descs, match in cases:
        rc, msg = _call(model, [L.InteractionMessage(*d) for d in descs], perm, vals, inter, se)
        assert rc == -1 and match in msg, (match, rc, msg)
    d = [L.InteractionMessage(*ok)]
    for args, match in [((perm, vals, inter, se, 0), "n_msgs"), ((perm, None, inter, se), "NULL"),
                        ((perm, vals, inter.data_ptr() + 2, se), "4-byte aligned"), ((perm, vals, inter, se.data_ptr() + 2), "4-byte aligned")]:
        rc, msg = _call(model, d, *args)
        assert rc == -1 and match in msg, (match, msg)
    torch.cuda.synchronize()
    assert bool((inter == 7.0).all()) and bool((se == 7.0).all())


def test_worker_agrees_with_model(tiny):
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
    got = W.custom_interactions_packed(reqs, permutations=4, seed=2)
    want = W.custom_prediction_packed(reqs, decode="device")
    p = W.pack_region_requests(reqs)
    args = (p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"], p["image_wh"], p["n_tokens"], p["n_boxes"])
    msgs = [m[:4] for i, m in W.ablation_messages(reqs, p["spans"]).items() if reqs[i][4] != "11"]
    si = model.shapley_interactions(*args, msgs, ["cross"] * len(msgs), permutations=4, seed=2,
                                    mask_token=W.tokenizer.vocab.get("[MASK]", 103), max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
    assert isinstance(got[2], ValueError) and "grounding answer is a box" in str(got[2])
    for i, s in zip([0, 1, 3], si):
        assert got[i]["answer"] == want[i]
        g = got[i]["interactions"]
        for key in ("interaction", "interaction_stderr", "phi", "pairs"):
            assert _same(g[key], s[key]), key
        assert g["units"] == s["units"] and len(g["box_pixels"]) == len(g["units"])
