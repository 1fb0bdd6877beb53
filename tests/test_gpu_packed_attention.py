"""Attention maps of packed batches (VB200_OUT_ATTENTION_PACKED: forward_packed / forward_regions_packed with
output_all_attention_masks, vb200_attention_layout_packed).  `-m gpu` only.

The packed probability launch is the dense fp32 attention kernel run at each sample's own lengths with the same arithmetic, so every
sample's maps are compared bit for bit with the maps of a dense forward of that sample alone, and with the fp32 oracle on the padded
batch at the tolerance of test_gpu_round2.py's attention test.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

DT = ("fp16", "bf16")
TOL_ATTN = 5e-3            # engine (fp16) vs the fp32 oracle's attention probabilities (test_gpu_round2.py)


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT, return_attention=True)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, return_attention=True)


def _packed(model, samples, select=None, maps=True, **kw):
    import vilbert_b200 as vb
    out = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_TASK_HEADS if select is None else select, debug_taps=True,
                               output_all_attention_masks=maps, **kw)
    torch.cuda.synchronize()
    return out


def _check_maps_bitwise(attn, refs):
    """attn: the packed list; refs[b]: the dense attn_data_list of sample b alone (batch 1)."""
    assert len(attn) == len(refs[0]) and len(attn) > 0
    for k, layer in enumerate(attn):
        if isinstance(refs[0][k], tuple):
            assert isinstance(layer, tuple) and len(layer) == 2
            for d in range(2):
                assert len(layer[d]) == len(refs)
                for b, ref in enumerate(refs):
                    assert torch.equal(layer[d][b], ref[k][d][0]), f"layer {k} direction {d} sample {b}"
        else:
            assert len(layer) == len(refs)
            for b, ref in enumerate(refs):
                assert torch.equal(layer[b], ref[k][0]), f"layer {k} sample {b}"


# (Tin, V): Tin = 1 and V = 1, T = Tin + 1 and V on both sides of 32 and 64, V = 256
CORNERS = [(1, 256), (31, 1), (32, 33), (63, 31), (64, 65), (12, 64), (1, 1)]


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("B", [1, 7, 6])
def test_packed_maps_bitwise_equal_dense_per_sample(tiny, mode, B):
    model = tiny[mode]
    samples = support.batch(model, CORNERS[:B], seed=80 + B)
    (out, _) = _packed(model, samples)
    _check_maps_bitwise(out[9], [support.dense_alone(model, s, output_all_attention_masks=True)[9] for s in samples])


# ------------------------------------------------------------------------------------------------ detector output
def _regions_packed(model, imgs, maps=True, **kw):
    import vilbert_b200 as vb
    (out, sp) = model.forward_regions_packed(*support.packed_image_args(imgs), select=vb.OUT_TASK_HEADS, output_all_attention_masks=maps,
                                             **kw)
    torch.cuda.synchronize()
    return out


def _regions_alone(model, im):
    q, seg, f, bx, wh, task = im
    (out, _) = model.forward_regions(q[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
                                     torch.tensor([[task]]).cuda(), f[None].cuda(), bx[None].cuda(), wh[None].cuda(),
                                     output_all_attention_masks=True)
    torch.cuda.synchronize()
    return out[9]


# (Tin, boxes): V = boxes + 1 on both sides of 32 and 64, V = 256, T on both sides of 32 and 64
REGION_CORNERS = [(1, 255), (31, 1), (32, 31), (63, 32), (64, 63), (5, 64), (2, 2)]


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("B", [1, 7, 6])
def test_regions_packed_maps_bitwise_equal_regions_per_image(tiny, mode, B):
    model = tiny[mode]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = [support.image(t, n, 90 + B + i, F, vocab) for i, (t, n) in enumerate(REGION_CORNERS[:B])]
    out = _regions_packed(model, imgs)
    _check_maps_bitwise(out[9], [_regions_alone(model, im) for im in imgs])


# ------------------------------------------------------------------------------------------------ full model, oracle
def test_full_model_maps_bitwise_and_oracle(full_oracle, full):
    lens = [(9, 37), (30, 101), (14, 11), (37, 64), (5, 2), (22, 18)]
    samples = support.batch(full, lens, seed=17)
    (out, _) = _packed(full, samples)
    _check_maps_bitwise(out[9], [support.dense_alone(full, s, output_all_attention_masks=True)[9] for s in samples])
    B, Tm, Vm = len(samples), max(t for t, _ in lens), max(v for _, v in lens)
    F = full._dims["v_feature_size"]
    q, seg, im = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (qq, sg, ff, ss, _) in enumerate(samples):
        q[b, :len(qq)], seg[b, :len(qq)], im[b, :len(qq)] = qq, sg, 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.tensor([[smp[4]] for smp in samples])
    ref = full_oracle(q, f, s, seg, im, vm, None, task, output_all_attention_masks=True, compute_pretraining_heads=False)[9]
    assert len(ref) == len(out[9]) == 24
    rows = {"t": [t + 1 for t, _ in lens], "v": [v for _, v in lens]}
    worst = 0.0
    for got, want in zip(out[9], ref):
        pairs = [(got[0], want[0], "t", "v"), (got[1], want[1], "v", "t")] if isinstance(want, tuple) else \
                [(got, want, *(("t", "t") if want.shape[-1] == Tm + 1 else ("v", "v")))]
        for per, w, rq, rk in pairs:
            for b, x in enumerate(per):
                lq, lk = rows[rq][b], rows[rk][b]
                assert tuple(x.shape[1:]) == (lq, lk)
                worst = max(worst, float((x.cpu() - w[b, :, :lq, :lk]).abs().max()))
                assert float((x.sum(-1) - 1).abs().max()) < 1e-4
    assert worst < TOL_ATTN, worst


# ------------------------------------------------------------------------------------------------ no side effects, layout, plans
@pytest.mark.parametrize("mode", DT)
def test_maps_change_no_other_output(tiny, mode):
    import vilbert_b200 as vb
    model = tiny[mode]
    samples = support.batch(model, [(5, 36), (30, 10), (12, 101), (1, 1), (37, 7)], seed=3)
    (a, ta) = _packed(model, samples, select=vb.OUT_ALL, maps=True)
    (b, tb) = _packed(model, samples, select=vb.OUT_ALL, maps=False)
    assert b[9] == [] and len(a[9]) > 0
    for k in range(9):
        assert (a[k] is None) == (b[k] is None)
        if a[k] is not None:
            assert torch.equal(a[k], b[k]), f"output {k} changes with the maps"
    for k in ta:
        assert torch.equal(ta[k], tb[k]), k
    model.return_attention = False
    try:
        assert _packed(model, samples, maps=True)[0][9] == []
    finally:
        model.return_attention = True


def _call_c(model, samples, buf, select, max_tokens=0, max_regions=0):
    """vb200_forward_packed through the C ABI with a caller-chosen attention_probs buffer (None: NULL); returns the status."""
    from vilbert_b200 import _lib as L
    cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda().contiguous()
    q, seg, f, s = cat(0), cat(1), cat(2), cat(3)
    tk = torch.tensor([[smp[4]] for smp in samples]).cuda()
    B = len(samples)
    nt, nr = (C.c_int32 * B)(*[len(x[0]) for x in samples]), (C.c_int32 * B)(*[x[2].shape[0] for x in samples])
    inp = L.PackedInputs(B, max_tokens, max_regions, C.cast(nt, C.c_void_p), C.cast(nr, C.c_void_p), q.data_ptr(), seg.data_ptr(),
                         f.data_ptr(), s.data_ptr(), tk.data_ptr())
    logits = torch.empty(B, model._dims["num_labels"], device="cuda")
    o = L.Outputs()
    o.vil_prediction = logits.data_ptr()
    o.attention_probs = buf.data_ptr() if buf is not None else None
    rc = L.load().vb200_forward_packed(model._handle, C.byref(inp), C.byref(o), select, 0,
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


def test_layout_total_and_untouched_tail(tiny):
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    lens = [(3, 40), (20, 1), (1, 70), (33, 9)]
    samples = support.batch(model, lens, seed=23)
    layout, total = model.attention_layout_packed([t for t, _ in lens], [v for _, v in lens])
    T, V = [t + 1 for t, _ in lens], [v for _, v in lens]
    sums = {0: sum(t * t for t in T), 1: sum(v * v for v in V), 2: sum(t * v for t, v in zip(T, V)), 3: sum(t * v for t, v in zip(T, V))}
    off = 0
    for heads, kind, o in layout:
        assert o == off
        off += heads * sums[kind]
    assert off == total
    tail = 1000
    buf = torch.full((total + tail,), float("nan"), device="cuda")
    assert _call_c(model, samples, buf, L.OUT_VIL_PREDICTION | L.OUT_ATTENTION_PACKED) == 0
    assert not bool(buf[:total].isnan().any()), "a float of the layout was not written"
    assert bool(buf[total:].isnan().all()), "the call wrote past the layout's total"
    from vilbert_b200.model import split_packed_attention
    _check_maps_equal(split_packed_attention(buf, layout, T, V), _packed(model, samples)[0][9])


def _check_maps_equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, tuple):
            for xs, ys in zip(x, y):
                assert all(torch.equal(u, w) for u, w in zip(xs, ys))
        else:
            assert all(torch.equal(u, w) for u, w in zip(x, y))


def test_plans_shared_across_lengths(tiny):
    model = tiny["bf16"]
    cap = dict(max_tokens=40, max_regions=120)
    a = support.batch(model, [(5, 36), (30, 10), (12, 101), (1, 1)], seed=41)
    b = support.batch(model, [(40, 120), (2, 3), (7, 64), (19, 33)], seed=42)
    _packed(model, a, maps=False, **cap)
    n = support.n_plans(model)
    _packed(model, a, maps=True, **cap)
    assert support.n_plans(model) == n + 1, "the first call with maps adds exactly one plan"
    _packed(model, b, maps=True, **cap)
    _packed(model, b, maps=False, **cap)
    assert support.n_plans(model) == n + 1, "calls at the same capacities share the plans whatever the lengths"


def test_back_to_back_calls_stage_their_own_destination(tiny):
    """Two calls on one slot and one stream, different lengths and buffers, no synchronisation between them: the destination pointer
    travels with each call's staged meta, so both get their own maps."""
    model = tiny["fp16"]
    cap = dict(max_tokens=40, max_regions=120)
    a = support.batch(model, [(5, 36), (30, 10), (12, 101), (1, 1)], seed=51)
    b = support.batch(model, [(40, 120), (2, 3), (7, 64), (19, 33)], seed=52)
    want_a, want_b = _packed(model, a, **cap)[0][9], _packed(model, b, **cap)[0][9]
    args_a, args_b = support.packed_sample_args(a), support.packed_sample_args(b)      # inputs on the device first: nothing below synchronises
    torch.cuda.synchronize()
    got_a = model.forward_packed(*args_a, output_all_attention_masks=True, **cap)[9]
    got_b = model.forward_packed(*args_b, output_all_attention_masks=True, **cap)[9]
    torch.cuda.synchronize()
    _check_maps_equal(got_a, want_a)
    _check_maps_equal(got_b, want_b)


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections(tiny_oracle, tiny):
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: .*" + pat)
    lib = L.load()
    ok = support.batch(model, [(5, 3), (4, 2)], seed=61)
    sel = L.OUT_VIL_PREDICTION | L.OUT_ATTENTION_PACKED
    # the bit without a destination
    assert _call_c(model, ok, None, sel) == -1
    assert b"attention_probs" in lib.vb200_last_error(model._handle)
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    im = support.image(5, 3, 62, F, vocab)
    nt, nb = (C.c_int32 * 1)(5), (C.c_int32 * 1)(3)
    dev = [t.cuda().contiguous() for t in (im[0], im[1], torch.tensor([[im[5]]]), im[2], im[3], im[4][None])]
    inp = L.PackedRegionInputs(1, 0, 0, C.cast(nt, C.c_void_p), C.cast(nb, C.c_void_p), *[t.data_ptr() for t in dev], None)
    logits = torch.empty(1, model._dims["num_labels"], device="cuda")
    o = L.Outputs()
    o.vil_prediction = logits.data_ptr()
    assert lib.vb200_forward_regions_packed(model._handle, C.byref(inp), C.byref(o), sel, 0, None) == -1
    assert b"attention_probs" in lib.vb200_last_error(model._handle)
    # the bit on the dense and the cached forwards
    q, seg, f, s, task = ok[0]
    dense = (q[None].cuda(), f[None].cuda(), s[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
             torch.ones(1, f.shape[0], dtype=torch.uint8).cuda(), None, torch.tensor([[task]]).cuda())
    with err("VB200_OUT_ATTENTION_PACKED"):
        model(*dense, select=vb.OUT_TASK_HEADS | L.OUT_ATTENTION_PACKED)
    with err("VB200_OUT_ATTENTION_PACKED"):
        model.forward_regions(dev[0][None], dev[1][None], torch.ones(1, 5, dtype=torch.long).cuda(), dev[2], dev[3][None], dev[4][None],
                              dev[5], select=vb.OUT_TASK_HEADS | L.OUT_ATTENTION_PACKED)
    ts = model.encode_text(dense[0], dense[3], dense[4], dense[7])
    vs = model.encode_image(dense[1], dense[2], dense[5])
    idx = torch.zeros(1, dtype=torch.long)
    with err("VB200_OUT_ATTENTION_PACKED"):
        model.forward_cached(ts, idx, vs, idx, select=L.OUT_VIL_LOGIT | L.OUT_ATTENTION_PACKED)
    tsp = model.encode_text_packed(q.cuda(), seg.cuda(), torch.tensor([[task]]).cuda(), [len(q)])
    vsp = model.encode_image_packed(f.cuda(), s.cuda(), [f.shape[0]])
    with err("VB200_OUT_ATTENTION_PACKED"):
        model.forward_cached_packed(tsp, idx, vsp, idx, select=L.OUT_VIL_LOGIT | L.OUT_ATTENTION_PACKED)
    torch.cuda.synchronize()
    # the layout call validates the lengths as the packed forwards do
    with err("n_tokens 0"):
        model.attention_layout_packed([3, 0], [4, 4])
    with err("n_regions 0"):
        model.attention_layout_packed([3, 3], [4, 0])
    with err("V=257"):
        model.attention_layout_packed([3], [257])
    with err("T=257"):
        model.attention_layout_packed([256], [4])
    # fp32x engines keep rejecting packed calls
    x = support.engine(tiny_oracle, compute_dtype="fp32x", return_attention=True)
    try:
        with err("fp32x"):
            _packed(x, ok)
    finally:
        x.close()
