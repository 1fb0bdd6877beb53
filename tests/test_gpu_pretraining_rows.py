"""Pre-training heads at chosen rows (VILBertForVLTasks.pretraining_heads / vb200_pretraining_heads).  `-m gpu` only.

The call gathers the listed rows of a forward's fp32 final states into the 16-bit operand the final LayerNorm writes from the same
values, and runs the forward's head GEMMs, LayerNorm and narrow-head kernels on them.  So the masked-token and masked-region logits
at a row are compared bit for bit with that row of the same forward run with both pre-training heads selected, and the alignment
score with element 3 of a batch-1 forward of the pair.  Parity with the fp32 oracle's `cls` heads is checked on the oracle's own
final states; top-k against a softmax of the returned logits.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16", "fp32x")
TOL = {"fp16": 1e-2, "bf16": 2e-2, "fp32x": 1e-3}   # vs the oracle's heads (16-bit modes: with the engine's operand rounding emulated)


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, MODES)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _both_heads():
    L = support.lib()
    return L.OUT_LINGUISIC_PREDICTION | L.OUT_VISION_PREDICTION


def _row_lists(total, seed):
    """A short list with the tile edges, the last row and duplicates, and a long one spanning several 128-row buckets."""
    g = torch.Generator().manual_seed(seed)
    short = [0, 127 % total, 128 % total, 129 % total, total - 1, 3 % total, 3 % total, total - 1]
    long = torch.randint(0, total, (300,), generator=g).tolist() + [0, total - 1, total - 1]
    return short, long


def _dense(model, B, Tin, V, seed, pad_regions=2):
    from oracle import vilbert_ref as R
    inp = list(R.make_inputs(B, Tin, V, seed=seed, vocab_size=model._dims["vocab_size"], pad_regions=pad_regions))
    inp[1] = inp[1][..., :model._dims["v_feature_size"]].contiguous()
    return inp


def _run_dense(model, inp, select):
    out, taps = model(*[t.cuda() for t in inp], select=select, debug_taps=True)
    return out, taps


def _check_rows(model, out_t, out_v, taps, t_lists, v_lists):
    """token / region logits at every list equal the full-row heads' rows bit for bit."""
    vocab, vt = model._dims["vocab_size"], model._dims["v_target_size"]
    full_t, full_v = out_t.reshape(-1, vocab), out_v.reshape(-1, vt)
    for tr, vr in zip(t_lists, v_lists):
        res = model.pretraining_heads(taps, text_rows=tr, image_rows=vr)
        torch.cuda.synchronize()
        assert torch.equal(res["token_logits"], full_t[torch.tensor(tr)]), (len(tr), "token")
        assert torch.equal(res["region_logits"], full_v[torch.tensor(vr)]), (len(vr), "region")


# ------------------------------------------------------------------ bit-identity with the full-row heads
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [2, 3])
def test_dense_rows_bit_identical(tiny, mode, B):
    model = tiny[mode]
    inp = _dense(model, B, 60, 50, seed=100 + B)
    out, taps = _run_dense(model, inp, _both_heads())
    T = 61
    _check_rows(model, out[7], out[5], taps, _row_lists(B * T, 1), _row_lists(B * 50, 2))


def _packed_inputs(model, nt, nv, seed):
    g = torch.Generator().manual_seed(seed)
    vocab, F = model._dims["vocab_size"], model._dims["v_feature_size"]
    q = torch.randint(1, vocab, (sum(nt),), generator=g)
    seg = torch.randint(0, 2, (sum(nt),), generator=g)
    f = torch.relu(torch.randn(sum(nv), F, generator=g))
    s = torch.rand(sum(nv), 5, generator=g)
    tk = torch.randint(0, 20, (len(nt), 1), generator=g)
    return q, f, s, seg, tk


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_packed_rows_bit_identical(tiny, mode):
    model = tiny[mode]
    nt, nv = [40, 7, 90, 33], [12, 60, 3, 81]
    q, f, s, seg, tk = _packed_inputs(model, nt, nv, 5)
    out, taps = model.forward_packed(q.cuda(), f.cuda(), s.cuda(), seg.cuda(), tk.cuda(), nt, nv, select=_both_heads(), debug_taps=True)
    rows_t, rows_v = sum(nt) + len(nt), sum(nv)
    _check_rows(model, out[7], out[5], taps, _row_lists(rows_t, 3), _row_lists(rows_v, 4))


def _detections(model, counts, seed):
    F = model._dims["v_feature_size"]
    g = torch.Generator().manual_seed(seed)
    n = sum(counts)
    bf = torch.relu(torch.randn(n, F, generator=g)) * 1.5
    x1, y1 = torch.rand(n, generator=g) * 300, torch.rand(n, generator=g) * 200
    bx = torch.stack([x1, y1, x1 + 20 + torch.rand(n, generator=g) * 100, y1 + 20 + torch.rand(n, generator=g) * 100], 1)
    wh = torch.tensor([[640.0, 480.0]] * len(counts))
    return bf, bx, wh


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_regions_packed_rows_bit_identical(tiny, mode):
    model = tiny[mode]
    nt, nb = [20, 55, 9], [70, 30, 64]
    q, _, _, seg, tk = _packed_inputs(model, nt, [1, 1, 1], 6)
    bf, bx, wh = _detections(model, nb, 7)
    (out, taps), _ = model.forward_regions_packed(q.cuda(), seg.cuda(), tk.cuda(), bf.cuda(), bx.cuda(), wh.cuda(), nt, nb,
                                                  select=_both_heads(), debug_taps=True)
    rows_t, rows_v = sum(nt) + len(nt), sum(nb) + len(nb)
    _check_rows(model, out[7], out[5], taps, _row_lists(rows_t, 8), _row_lists(rows_v, 9))


def test_full_model_rows_bit_identical(full):
    model = full
    inp = _dense(model, 2, 70, 72, seed=21)
    out, taps = _run_dense(model, inp, _both_heads())
    _check_rows(model, out[7], out[5], taps, _row_lists(2 * 71, 10), _row_lists(2 * 72, 11))
    nt, nv = [37, 12, 60], [101, 40, 77]
    q, f, s, seg, tk = _packed_inputs(model, nt, nv, 12)
    out, taps = model.forward_packed(q.cuda(), f.cuda(), s.cuda(), seg.cuda(), tk.cuda(), nt, nv, select=_both_heads(), debug_taps=True)
    _check_rows(model, out[7], out[5], taps, _row_lists(sum(nt) + 3, 13), _row_lists(sum(nv), 14))


# ------------------------------------------------------------------ alignment = element 3 of a batch-1 forward
def _element3_alone(model, inp, b):
    L = support.lib()
    one = [t[b:b + 1] for t in inp]
    return model(*[t.cuda() for t in one], select=L.OUT_VIL_BINARY_PREDICTION)[3]


@pytest.mark.parametrize("mode", MODES)
def test_alignment_from_even_dense_batch(tiny, mode):
    model = tiny[mode]
    inp = _dense(model, 4, 30, 36, seed=31)
    _, taps = _run_dense(model, inp, 0)
    res = model.pretraining_heads(taps, pair_rows=[3, 0, 2, 1, 1])
    torch.cuda.synchronize()
    for i, b in enumerate([3, 0, 2, 1, 1]):
        assert torch.equal(res["alignment"][i:i + 1], _element3_alone(model, inp, b)), (mode, b)


def _dense_alone(model, q, f, s, seg, tk, nt, nv, b):
    """Sample b of a packed batch as a dense batch-1 forward at its own lengths (no padding)."""
    t0, v0 = sum(nt[:b]), sum(nv[:b])
    ones = torch.ones(1, nt[b], dtype=torch.long)
    return (q[t0:t0 + nt[b]][None], f[v0:v0 + nv[b]][None], s[v0:v0 + nv[b]][None], seg[t0:t0 + nt[b]][None], ones,
            torch.ones(1, nv[b], dtype=torch.uint8), None, tk[b:b + 1])


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_alignment_from_packed_and_cached_packed(tiny, mode):
    L = support.lib()
    model = tiny[mode]
    nt, nv = [12, 30, 5, 22], [20, 9, 36, 14]
    q, f, s, seg, tk = _packed_inputs(model, nt, nv, 41)
    _, taps = model.forward_packed(q.cuda(), f.cuda(), s.cuda(), seg.cuda(), tk.cuda(), nt, nv, select=0, debug_taps=True)
    res = model.pretraining_heads(taps, pair_rows=range(4))
    alone = []
    for b in range(4):
        a = _dense_alone(model, q, f, s, seg, tk, nt, nv, b)
        alone.append(model(*[t.cuda() if t is not None else None for t in a], select=L.OUT_VIL_BINARY_PREDICTION)[3])
    torch.cuda.synchronize()
    assert torch.equal(res["alignment"], torch.cat(alone))
    # the same pairs scored from packed caption / image states
    ts = model.encode_text_packed(q.cuda(), seg.cuda(), tk.cuda(), nt)
    vs = model.encode_image_packed(f.cuda(), s.cuda(), nv)
    idx = torch.arange(4, dtype=torch.int32)
    _, taps = model.forward_cached_packed(ts, idx, vs, idx, select=0, debug_taps=True)
    res = model.pretraining_heads(taps, pair_rows=[0, 1, 2, 3])
    torch.cuda.synchronize()
    assert torch.equal(res["alignment"], torch.cat(alone))


# ------------------------------------------------------------------ parity with the oracle's cls heads on its own final states
@pytest.mark.parametrize("mode", MODES)
def test_oracle_parity(tiny, tiny_oracle, mode):
    from oracle import vilbert_ref as R
    model = tiny[mode]
    inp = _dense(model, 2, 30, 36, seed=51)
    collect = {}
    tiny_oracle(*inp, collect=collect)
    t, v, pt, pv = collect["final"]
    taps = {"sequence_output_t": t.contiguous().cuda(), "sequence_output_v": v.contiguous().cuda(),
            "pooled_output": (pt * pv).contiguous().cuda()}
    tr, vr, pr = [0, 5, 30, 61, 7, 7], [0, 35, 36, 71, 2], [1, 0]
    res = model.pretraining_heads(taps, text_rows=tr, image_rows=vr, pair_rows=pr)
    cls = tiny_oracle.cls
    H, Hv = t.shape[-1], v.shape[-1]

    def heads():
        with torch.no_grad():
            return (cls.predictions(t.reshape(-1, H)[tr]), cls.imagePredictions(v.reshape(-1, Hv)[vr]),
                    cls.bi_seq_relationship((pt * pv)[pr]))
    if mode == "fp32x":
        ref = heads()
    else:
        with R.emulate_activation_rounding(tiny_oracle, torch.float16 if mode == "fp16" else torch.bfloat16):
            ref = heads()
    for key, r in zip(("token_logits", "region_logits", "alignment"), ref):
        err = float((res[key].cpu() - r).abs().max())
        print(f"PARITY pretraining_heads {mode} {key}: max abs err {err:.3e} (logit std {float(r.std()):.3f})")
        assert err < TOL[mode], (mode, key, err)


# ------------------------------------------------------------------ top-k
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("k", [1, 5, 10])
def test_top_k_matches_softmax_of_logits(tiny, mode, k):
    model = tiny[mode]
    inp = _dense(model, 2, 40, 30, seed=61)
    _, taps = _run_dense(model, inp, 0)
    res = model.pretraining_heads(taps, text_rows=list(range(0, 82, 3)), image_rows=[59, 0, 0, 31], top_k=k)
    torch.cuda.synchronize()
    for logits, top in (("token_logits", "token_top"), ("region_logits", "region_top")):
        idx, prob = res[top]
        assert idx.shape == prob.shape == (res[logits].shape[0], k)
        p = torch.softmax(res[logits].double(), dim=1)
        ref_p, ref_i = torch.sort(p, dim=1, descending=True, stable=True)          # equal probabilities: lower index first
        picked = torch.gather(p, 1, idx.long())
        assert torch.allclose(picked, ref_p[:, :k], rtol=1e-5, atol=1e-9), top
        assert torch.allclose(prob.double(), picked, rtol=1e-5, atol=1e-9), top
        clear = (ref_p[:, :k] - ref_p[:, 1:k + 1]).min(dim=1).values > 1e-6    # rows without a near tie inside the top k + 1
        assert torch.equal(idx.long()[clear], ref_i[:, :k][clear]), top


# ------------------------------------------------------------------ independence and isolation
@pytest.mark.parametrize("mode", ("fp16", "fp32x"))
def test_back_to_back_calls_and_isolation(tiny, mode):
    L = support.lib()
    model = tiny[mode]
    inp = _dense(model, 3, 60, 50, seed=71)
    sel = L.OUT_TASK_HEADS
    before, taps = _run_dense(model, inp, sel)
    before = [x.clone() if torch.is_tensor(x) else x for x in before]
    plans = support.n_plans(model)
    lists = [([0, 1, 2], [5]), (list(range(150)), list(range(140, 0, -1))), ([182, 182], [149]), (list(range(183)), [0] * 300)]
    alone = []
    for tr, vr in lists:
        alone.append(model.pretraining_heads(taps, text_rows=tr, image_rows=vr, pair_rows=[2, 1], top_k=3))
        torch.cuda.synchronize()
    again = [model.pretraining_heads(taps, text_rows=tr, image_rows=vr, pair_rows=[2, 1], top_k=3) for tr, vr in lists]
    torch.cuda.synchronize()
    for a, b in zip(alone, again):
        for key in ("token_logits", "region_logits", "alignment"):
            assert torch.equal(a[key], b[key]), key
        for key in ("token_top", "region_top"):
            assert torch.equal(a[key][0], b[key][0]) and torch.equal(a[key][1], b[key][1]), key
    assert support.n_plans(model) == plans
    after, _ = _run_dense(model, inp, sel)
    torch.cuda.synchronize()
    for x, y in zip(before[:9], after[:9]):
        assert (x is None and y is None) or torch.equal(x, y)
    assert support.n_plans(model) == plans


# ------------------------------------------------------------------ rejections
def _raw_call(model, t_rows=None, v_rows=None, p_rows=None, top_k=0, states=(True, True, True), tops=(False, False), n_override=None):
    """vb200_pretraining_heads on a B=2 dense forward's taps with sentinel-filled outputs; returns (status, message, outputs).  The
    call leaves the forward-plan count as it was."""
    L = support.lib()
    inp = _dense(model, 2, 20, 16, seed=81)
    _, taps = _run_dense(model, inp, 0)
    d = model._dims
    keep = []

    def arr(v):
        a = (C.c_int32 * max(len(v), 1))(*v)
        keep.append(a)
        return C.cast(a, C.c_void_p)
    rows = [r or [] for r in (t_rows, v_rows, p_rows)]
    st = [taps["sequence_output_t"], taps["sequence_output_v"], taps["pooled_output"]]
    n_state = [2 * 21, 2 * 16, 2]
    r = L.PretrainRows(*(s.data_ptr() if on else None for s, on in zip(st, states)), *n_state,
                       *(n_override or [len(x) for x in rows]), *(arr(x) for x in rows), top_k)
    outs = {"token_logits": torch.full((max(len(rows[0]), 1), d["vocab_size"]), 7.0, device="cuda"),
            "region_logits": torch.full((max(len(rows[1]), 1), d["v_target_size"]), 7.0, device="cuda"),
            "alignment": torch.full((max(len(rows[2]), 1), 2), 7.0, device="cuda"),
            "token_top": torch.full((max(len(rows[0]), 1), 61), 7, dtype=torch.int32, device="cuda"),
            "region_top": torch.full((max(len(rows[1]), 1), 61), 7, dtype=torch.int32, device="cuda")}
    o = L.PretrainOut(outs["token_logits"].data_ptr(), outs["region_logits"].data_ptr(), outs["alignment"].data_ptr(),
                      outs["token_top"].data_ptr() if tops[0] else None, outs["region_top"].data_ptr() if tops[1] else None)
    torch.cuda.synchronize()
    plans = support.n_plans(model)
    rc = L.load().vb200_pretraining_heads(model._handle, C.byref(r), C.byref(o), None)
    torch.cuda.synchronize()
    msg = L.load().vb200_last_error(model._handle).decode()
    assert support.n_plans(model) == plans
    return rc, msg, outs


@pytest.mark.parametrize("case, needle", [
    (dict(t_rows=[0, 42]), "text_rows[1] = 42"),
    (dict(v_rows=[3, -1]), "image_rows[1] = -1"),
    (dict(p_rows=[0, 1, 2]), "pair_rows[2] = 2"),
    (dict(t_rows=[0], states=(False, True, True)), "text_state is NULL"),
    (dict(v_rows=[0], states=(True, False, True)), "image_state is NULL"),
    (dict(p_rows=[0], states=(True, True, False)), "pooled_state is NULL"),
    (dict(t_rows=[0], top_k=11, tops=(True, False)), "top_k 11"),
    (dict(t_rows=[0], top_k=-1), "top_k -1"),
    (dict(v_rows=[0], top_k=0, tops=(False, True)), "region_top is requested with top_k = 0"),
    (dict(t_rows=[0], top_k=0, tops=(True, False)), "token_top is requested with top_k = 0"),
    (dict(t_rows=[0], n_override=[-1, 0, 0]), "text_rows has a count of -1"),
])
def test_rejections_name_list_and_index(tiny, case, needle):
    rc, msg, outs = _raw_call(tiny["fp16"], **case)
    assert rc == -1 and needle in msg, (rc, msg)
    for key, t in outs.items():
        assert bool((t == 7).all()), key


def test_top_k_above_width_rejected():
    from oracle import vilbert_ref as R
    oracle = R.build(R.tiny_config(v_target_size=8), seed=7, num_labels=200)
    model = support.engine(oracle)
    try:
        rc, msg, outs = _raw_call(model, v_rows=[0, 1], top_k=9, tops=(False, True))
        assert rc == -1 and "top_k 9 is above the 8 logits of a region_top row" in msg, msg
        assert bool((outs["region_top"] == 7).all()) and bool((outs["region_logits"] == 7).all())
        rc, msg, _ = _raw_call(model, v_rows=[0, 1], top_k=8, tops=(False, True))
        assert rc == 0, msg
    finally:
        model.close()


def test_model_wrapper_errors(tiny):
    model = tiny["fp16"]
    with pytest.raises(ValueError, match="needs the pooled_output tap"):
        model.pretraining_heads({"sequence_output_t": torch.zeros(4, 128, device="cuda")}, pair_rows=[0])
    from vilbert_b200 import _lib as L
    with pytest.raises(L.VilbertB200Error, match="text_rows\\[0\\] = 4"):
        model.pretraining_heads({"sequence_output_t": torch.zeros(4, 128, device="cuda")}, text_rows=[4])
