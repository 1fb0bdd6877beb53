"""Pruned tail: a forward whose select and taps read no final row of a stream runs that stream's last layer after its
self-attention on each sample's first row only (DESIGN.md section 4.3).  `-m gpu` only.

Every pruned op is row-local and no kernel's per-element result depends on the row count, the row stride or the tile width, so
each case compares a pooled-only call with the same call made to keep every row (a per-row head or the sequence taps): the
pooled-based outputs and pooled_output must be bit-identical.
"""
import contextlib

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

# the heads that read pooled_output only; a plan selecting nothing else prunes both tails
POOLED = 0x1F           # VIL_PREDICTION | VIL_PREDICTION_GQA | VIL_LOGIT | VIL_BINARY_PREDICTION | VIL_TRI_PREDICTION
ROW_HEADS = (1 << 6) | (1 << 8)     # VISION_LOGIT | LINGUISIC_LOGIT: every final row of both streams is read


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16", "fp32x"), return_attention=True, max_plans=256)


@contextlib.contextmanager
def _pooled_tap_only(model):
    """debug_taps calls of `model` bind pooled_output alone: the sequence taps stay unbound (and unwritten), so the plan prunes."""
    names = ("_alloc_outputs", "_alloc_packed_outputs")

    def wrap(f):
        def alloc(*a, **k):
            r = f(*a, **k)
            r[1].sequence_output_t = None
            r[1].sequence_output_v = None
            return r
        return alloc
    for n in names:
        setattr(model, n, wrap(getattr(model, n)))
    try:
        yield
    finally:
        for n in names:
            delattr(model, n)


def _pruned_and_full(model, call, select=POOLED):
    """call(select, debug_taps) -> (10-tuple, taps), once with only pooled_output bound, once with every tap bound."""
    n = support.n_plans(model)
    with _pooled_tap_only(model):
        pruned = call(select, True)
    full = call(select, True)
    torch.cuda.synchronize()
    assert support.n_plans(model) == n + 2, "the pooled-only call and the taps call share a plan"
    return pruned, full


def _assert_pooled_equal(pruned, full, what, outputs=range(5)):
    (po, pt), (fo, ft) = pruned, full
    for k in outputs:
        assert (po[k] is None) == (fo[k] is None), (what, k)
        if po[k] is not None:
            assert torch.equal(po[k], fo[k]), f"{what}: output {k} differs with the pruned tail"
    assert torch.equal(pt["pooled_output"], ft["pooled_output"]), f"{what}: pooled_output differs with the pruned tail"


def _dense_inputs(model, B, Tin, V, seed, pad):
    from oracle import vilbert_ref as R
    inp = list(R.make_inputs(B, Tin, V, seed=seed, vocab_size=model._dims["vocab_size"], pad_regions=pad))
    inp[1] = inp[1][..., :model._dims["v_feature_size"]].contiguous()
    return [t.cuda() for t in inp]


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp32x"])
@pytest.mark.parametrize("B,Tin,V,pad", [(1, 12, 37, 0), (2, 30, 36, 3), (3, 16, 10, 2)])
def test_dense(tiny, dtype, B, Tin, V, pad):
    model = tiny[dtype]
    inp = _dense_inputs(model, B, Tin, V, 40 + B, pad)
    pruned, full = _pruned_and_full(model, lambda sel, taps: model(*inp, select=sel, debug_taps=taps))
    _assert_pooled_equal(pruned, full, f"{dtype} dense B={B}")


def _packed_samples(model, lens, seed):
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    out = []
    for i, (tin, v) in enumerate(lens):
        g = torch.Generator().manual_seed(seed + i)
        q, seg = torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g)
        f = torch.relu(torch.randn(v, F, generator=g)) * 1.5
        xy = torch.rand(v, 2, generator=g) * 0.7
        x2y2 = (xy + 0.05 + torch.rand(v, 2, generator=g) * 0.25).clamp(max=1.0)
        s = torch.cat([xy, x2y2, ((x2y2 - xy)[:, 0] * (x2y2 - xy)[:, 1])[:, None]], dim=-1)
        s[0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
        out.append((q, seg, f, s, int(torch.randint(0, 20, (1,), generator=g))))
    return out


LENS = [(20, 40), (3, 33), (25, 12), (1, 1), (30, 65)]


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_packed(tiny, dtype):
    model = tiny[dtype]
    smp = _packed_samples(model, LENS, 7)
    cat = lambda k: torch.cat([s[k] for s in smp]).cuda()
    task = torch.tensor([[s[4]] for s in smp]).cuda()
    nt, nv = [len(s[0]) for s in smp], [s[2].shape[0] for s in smp]
    pruned, full = _pruned_and_full(model, lambda sel, taps: model.forward_packed(cat(0), cat(2), cat(3), cat(1), task, nt, nv,
                                                                                  select=sel, debug_taps=taps))
    _assert_pooled_equal(pruned, full, f"{dtype} forward_packed")


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_regions_packed(tiny, dtype):
    model = tiny[dtype]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    g = torch.Generator().manual_seed(5)
    nt, nb = [9, 2, 17], [10, 1, 30]
    q = torch.randint(1, vocab, (sum(nt),), generator=g).cuda()
    seg = torch.randint(0, 2, (sum(nt),), generator=g).cuda()
    feats = (torch.relu(torch.randn(sum(nb), F, generator=g)) * 1.5).cuda()
    x1y1 = torch.rand(sum(nb), 2, generator=g) * 300
    boxes = torch.cat([x1y1, x1y1 + 20 + torch.rand(sum(nb), 2, generator=g) * 100], 1).cuda()
    wh = torch.tensor([[640.0, 480.0]] * len(nt)).cuda()
    task = torch.tensor([[1], [12], [11]]).cuda()
    pruned, full = _pruned_and_full(model, lambda sel, taps: model.forward_regions_packed(q, seg, task, feats, boxes, wh, nt, nb,
                                                                                         select=sel, debug_taps=taps)[0])
    _assert_pooled_equal(pruned, full, f"{dtype} forward_regions_packed")


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp32x"])
def test_cached(tiny, dtype):
    model = tiny[dtype]
    q, f, s, seg, im, vm, _, task = _dense_inputs(model, 3, 14, 20, 9, 2)
    ts, vs = model.encode_text(q, seg, im, task), model.encode_image(f, s, vm)
    ti, ii = torch.tensor([2, 0, 1, 1], dtype=torch.int32).cuda(), torch.tensor([0, 0, 2, 1], dtype=torch.int32).cuda()
    pruned = model.forward_cached(ts, ti, vs, ii, select=POOLED)
    full = model.forward_cached(ts, ti, vs, ii, select=POOLED | ROW_HEADS)
    torch.cuda.synchronize()
    for k in range(5):
        assert torch.equal(pruned[k], full[k]), f"{dtype} forward_cached: output {k} differs with the pruned tail"


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_cached_packed(tiny, dtype):
    model = tiny[dtype]
    smp = _packed_samples(model, LENS, 21)
    cat = lambda xs: torch.cat(xs).cuda()
    ts = model.encode_text_packed(cat([s[0] for s in smp]), cat([s[1] for s in smp]), torch.tensor([[s[4]] for s in smp]).cuda(),
                                  [len(s[0]) for s in smp])
    vs = model.encode_image_packed(cat([s[2] for s in smp]), cat([s[3] for s in smp]), [s[2].shape[0] for s in smp])
    ti, ii = torch.tensor([4, 0, 3, 1, 1, 2]), torch.tensor([0, 4, 2, 3, 1, 1])
    pruned, full = _pruned_and_full(model, lambda sel, taps: model.forward_cached_packed(ts, ti, vs, ii, select=sel, debug_taps=taps))
    _assert_pooled_equal(pruned, full, f"{dtype} forward_cached_packed")


def test_text_tail_only(tiny):
    """vision_logit reads every image row: only the text tail is pruned, and every output stays the same."""
    model = tiny["bf16"]
    inp = _dense_inputs(model, 4, 18, 25, 3, 1)
    sel = 1 | (1 << 3) | (1 << 6)        # the multitask workload: VIL_PREDICTION | VIL_BINARY_PREDICTION | VISION_LOGIT
    pruned, full = _pruned_and_full(model, lambda s, taps: model(*inp, select=s, debug_taps=taps), select=sel)
    _assert_pooled_equal(pruned, full, "multitask select", outputs=(0, 3, 6))


def test_attention_maps(tiny):
    """Attention maps come from Q and K of every row, which a pruned layer still computes."""
    model = tiny["fp16"]
    inp = _dense_inputs(model, 2, 21, 30, 17, 2)
    pruned, full = _pruned_and_full(model, lambda s, taps: model(*inp, select=s, debug_taps=taps, output_all_attention_masks=True))
    _assert_pooled_equal(pruned, full, "attention maps")
    pa, fa = pruned[0][9], full[0][9]
    assert len(pa) == len(fa) > 0
    for i, (p, f) in enumerate(zip(pa, fa)):
        for x, y in zip(p if isinstance(p, tuple) else (p,), f if isinstance(f, tuple) else (f,)):
            assert torch.equal(x, y), f"attention entry {i} differs with the pruned tail"


def test_taps_after_pruned_plan(tiny):
    """A taps call of a shape a pooled-only call has already planned builds its own plan and fills every tap."""
    model = tiny["bf16"]
    inp = _dense_inputs(model, 3, 11, 19, 29, 0)
    model(*inp, select=POOLED)
    n = support.n_plans(model)
    out, taps = model(*inp, select=POOLED, debug_taps=True)
    assert support.n_plans(model) == n + 1
    ref_out, ref_taps = model(*inp, select=POOLED | ROW_HEADS, debug_taps=True)
    torch.cuda.synchronize()
    for k in ("sequence_output_t", "sequence_output_v", "pooled_output"):
        assert torch.equal(taps[k], ref_taps[k]), f"tap {k} after a pruned plan of the same shape"
    for k in range(5):
        assert torch.equal(out[k], ref_out[k])


@pytest.fixture(scope="module")
def full_bf16(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16", max_plans=256)


def test_full_model_bench_shape(full_bf16):
    """The flagship shape: B = 64, 30 tokens, 36 regions, VQA head."""
    inp = _dense_inputs(full_bf16, 64, 30, 36, 123, 0)
    pruned, full = _pruned_and_full(full_bf16, lambda s, taps: full_bf16(*inp, select=s, debug_taps=taps), select=1)
    _assert_pooled_equal(pruned, full, "full model B=64", outputs=(0,))


def test_full_model_plan_flops(full_bf16):
    """Pruning removes exactly the row-local GEMMs of the last text and image layer past each sample's first row."""
    d = full_bf16._dims
    B, T, V = 64, 31, 36                       # T: 30 tokens + the task token
    H, Hv = d["hidden_size"], d["v_hidden_size"]
    inter, v_inter = 3072, 1024                # the default config's intermediate sizes
    _, pruned = full_bf16.plan_info(B, 30, V, 1)
    _, kept = full_bf16.plan_info(B, 30, V, 1 | ROW_HEADS)
    removed = 2 * B * (T - 1) * (H * H + 2 * H * inter) + 2 * B * (V - 1) * (Hv * Hv + 2 * Hv * v_inter)
    row_heads = 2 * B * T * H + 2 * B * V * Hv  # the two rowdot heads the kept plan adds
    assert kept - pruned == removed + row_heads
