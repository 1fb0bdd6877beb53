"""Head masks on the packed forwards (forward_packed / forward_regions_packed with head_mask, vb200_forward_packed_gated and
vb200_forward_regions_packed_gated).  `-m gpu` only.

The gate scales a head's context rows in fp32 before the 16-bit store, so a gate of 1.0 must give the ungated bits in every output,
a gated sample must leave its batch neighbours and its own earlier layers untouched bit for bit, and a gated forward must match the
fp32 oracle gated the same way (forward hooks that scale the head's context columns) at the packed forwards' tolerances.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

DT = ("fp16", "bf16")
TOL = 1e-2                 # fp16 mode vs the fp32 oracle (test_gpu_packed.py)
TOL_BF16_VS_FP32 = 3.5e-2  # bf16 mode vs the fp32 oracle, x max(1, logit std) (test_gpu_packed.py)
ERR_INVALID = -1           # VB200_ERR_INVALID


def _tol(mode, want):
    return TOL if mode == "fp16" else TOL_BF16_VS_FP32 * max(1.0, float(want.std()))


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT, return_attention=True, max_rows_per_sample=1024)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16", return_attention=True)


def _shape(model):
    from vilbert_b200.model import head_mask_shape
    return head_mask_shape(model.config)


def _packed(model, samples, select=None, **kw):
    import vilbert_b200 as vb
    out = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_TASK_HEADS if select is None else select,
                               debug_taps=True, output_all_attention_masks=True, output_layer_states=True, **kw)
    torch.cuda.synchronize()
    return out


def _regions(model, imgs, select=None, **kw):
    import vilbert_b200 as vb
    out = model.forward_regions_packed(*support.packed_image_args(imgs), select=vb.OUT_TASK_HEADS if select is None else select,
                                       debug_taps=True, output_all_attention_masks=True, output_layer_states=True, **kw)
    torch.cuda.synchronize()
    (res, sp), states = out
    return (res, states), sp


def _flat(x):
    """Every tensor of a nested result, in order (None entries skipped)."""
    if torch.is_tensor(x):
        return [x]
    if isinstance(x, dict):
        return [t for k in sorted(x) for t in _flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _flat(v)]
    return []


def _bit_equal(a, b):
    fa, fb = _flat(a), _flat(b)
    assert len(fa) == len(fb) and len(fa) > 0
    for i, (x, y) in enumerate(zip(fa, fb)):
        assert x.shape == y.shape and support.eq32(x.float(), y.float()), f"tensor {i} differs"


# (Tin, V) per sample: short and long keys on both sides of 64; LONG adds sequences past 256 rows (the streaming kernels)
LENS = [(9, 37), (30, 101), (14, 11), (63, 64), (5, 2)]
LONG = [(9, 300), (150, 20), (12, 7)]


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("lens", [LENS, LONG], ids=["staged", "streaming"])
@pytest.mark.parametrize("select", ["heads", "taps"])
def test_all_ones_gate_is_bit_identical(tiny, mode, lens, select):
    """A gate of 1.0 everywhere gives the ungated bits in every output: task heads, taps, layer states and packed maps.  "heads"
    selects no per-row output, so both streams' last layers run pruned; "taps" reads vision_logit / linguisic_logit, so they do not."""
    import vilbert_b200 as vb
    model = tiny[mode]
    sel = vb.OUT_TASK_HEADS if select == "heads" else vb.OUT_TASK_HEADS | vb.OUT_VISION_LOGIT | vb.OUT_LINGUISIC_LOGIT
    samples = support.batch(model, lens, seed=31)
    ref = _packed(model, samples, select=sel)
    got = _packed(model, samples, select=sel, head_mask=torch.ones(_shape(model)))
    _bit_equal(got, ref)


@pytest.mark.parametrize("mode", DT)
def test_all_ones_gate_regions_bit_identical(tiny, mode):
    model = tiny[mode]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = [support.image(t, n, 40 + i, F, vocab) for i, (t, n) in enumerate([(9, 36), (30, 100), (3, 1), (64, 63)])]
    ref, sp_ref = _regions(model, imgs)
    got, sp = _regions(model, imgs, head_mask=torch.ones(_shape(model)))
    _bit_equal(got, ref)
    assert support.eq32(sp, sp_ref)


def test_all_ones_gate_head_mean_bit_identical(tiny_oracle):
    model = support.engine(tiny_oracle, compute_dtype="bf16", return_attention=True, attention_heads="mean")
    try:
        samples = support.batch(model, LENS, seed=32)
        _bit_equal(_packed(model, samples, head_mask=torch.ones(_shape(model))), _packed(model, samples))
    finally:
        model.close()


def test_full_model_all_ones_bit_identical(full):
    """The 268 M model (12 / 8 / 8 heads): slots past an entry's own head count are ignored, even when they hold NaN."""
    E, H = _shape(full)
    assert (E, H) == (30, 12)
    m = torch.ones(E, H)
    for e, heads in enumerate(_entry_heads(full)):
        m[e, heads:] = float("nan")
    samples = support.batch(full, [(9, 37), (30, 101), (14, 11)], seed=33)
    _bit_equal(_packed(full, samples, head_mask=m), _packed(full, samples))


def _entry_heads(model):
    """Each entry's head count, in the head mask's entry order."""
    kinds, _ = model.attention_selection()
    c = model.config
    return [c.num_attention_heads if k == 0 else c.v_num_attention_heads if k == 1 else c.bi_num_attention_heads for k in kinds]


def test_model_dims_match_shape(tiny, full):
    for model in (tiny["bf16"], full):
        E, H = _shape(model)
        for key, want in (("head_mask_entries", E), ("head_mask_heads", H)):
            v = C.c_int64()
            L = support.lib()
            L.check(L.load().vb200_model_dim(model._handle, key.encode(), C.byref(v)), model._handle)
            assert v.value == want, key


# ------------------------------------------------------------------------------------------------ isolation
@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("e", [0, 5, 12, 13, 29])
def test_one_gated_head_isolated(tiny, mode, e):
    """Gating head (e, h) of sample 1 leaves every other sample, and sample 1's layer states before entry e, bit for bit; the gated
    head's map is exactly zero."""
    model = tiny[mode]
    E, H = _shape(model)
    samples = support.batch(model, LENS, seed=34)
    B = len(samples)
    ref_out, ref_states = _packed(model, samples)
    m = torch.ones(B, E, H)
    h = e % H
    m[1, e, h] = 0.0
    out, states = _packed(model, samples, head_mask=m)
    # per-sample task heads and pooled output: only sample 1 may change
    for k in (0, 1, 2, 4):
        a, b = out[0][k], ref_out[0][k]
        keep = [i for i in range(B) if i != 1]
        assert support.eq32(a[keep], b[keep]), f"output {k}"
    assert support.eq32(out[1]["pooled_output"][[0, 2, 3, 4]], ref_out[1]["pooled_output"][[0, 2, 3, 4]])
    assert not torch.equal(out[1]["pooled_output"][1], ref_out[1]["pooled_output"][1])
    # maps: the gated head's block is zero, every other sample's maps unchanged
    kinds, _ = model.attention_selection()
    layer, d = _entry_layer(kinds, e)
    got, want = out[0][9][layer], ref_out[0][9][layer]
    if d is not None:
        got, want = got[d], want[d]
    assert torch.count_nonzero(got[1][h]) == 0
    for i in range(B):
        if i != 1:
            assert support.eq32(got[i], want[i])
    # layer states: sample 1's states written before entry e are unchanged (state entry s is written after attention entry
    # state_before[s] - 1)
    for s, (a, b) in enumerate(zip(states, ref_states)):
        for i, (x, y) in enumerate(zip(a, b)):
            if i != 1 or _state_before_entry(model, s) <= e:
                assert support.eq32(x, y), f"state {s} sample {i}"


def _entry_layer(kinds, e):
    """Entry e's index in the 24-entry attention list and its direction (None for a text / image layer)."""
    layer, i = 0, 0
    while i < len(kinds):
        if kinds[i] == 2:
            if e in (i, i + 1):
                return layer, e - i
            i += 2
        else:
            if e == i:
                return layer, None
            i += 1
        layer += 1
    raise AssertionError(e)


def _state_schedule(model):
    """Per layer-state entry: (is text, the number of attention entries run before it is written)."""
    out = [(True, 0), (False, 0)]
    n = 0
    kinds, _ = model.attention_selection()
    i = 0
    while i < len(kinds):
        k = kinds[i]
        if k == 2:
            n += 2
            out += [(True, n), (False, n)]
            i += 2
        else:
            n += 1
            out.append((k == 0, n))
            i += 1
    return out


def _state_before_entry(model, s):
    return _state_schedule(model)[s][1]


# ------------------------------------------------------------------------------------------------ oracle
def _gate_oracle(oracle, mask):
    """Forward hooks on the oracle's attention.self / biattention modules that scale head h's context columns of sample b by
    mask[b, e, h] (e: the entry in execution order).  Returns the hook handles."""
    enc = oracle.bert.encoder
    handles, e = [], 0

    def scale(ctx, g, heads):
        b, l, w = ctx.shape
        return (ctx.view(b, l, heads, w // heads) * g[:, None, :heads, None].to(ctx.dtype)).view(b, l, w)

    for step in enc.schedule():
        kind, idx = step[0], int(step[1:])
        if kind in "TV":
            mod = (enc.layer if kind == "T" else enc.v_layer)[idx].attention.self
            g = mask[:, e]
            handles.append(mod.register_forward_hook(
                lambda m, i, o, g=g: (scale(o[0], g, m.num_attention_heads), o[1])))
            e += 1
        else:
            mod = enc.c_layer[idx].biattention
            g1, g2 = mask[:, e], mask[:, e + 1]
            handles.append(mod.register_forward_hook(
                lambda m, i, o, g1=g1, g2=g2: (scale(o[0], g1, m.num_attention_heads), scale(o[1], g2, m.num_attention_heads), o[2])))
            e += 2
    return handles


def _oracle_padded(oracle, samples, mask):
    B = len(samples)
    Tm, Vm = max(len(s[0]) for s in samples), max(s[2].shape[0] for s in samples)
    F = oracle.config.v_feature_size
    q, seg, im = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (qq, sg, ff, ss, _) in enumerate(samples):
        q[b, :len(qq)], seg[b, :len(qq)], im[b, :len(qq)] = qq, sg, 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.tensor([[smp[4]] for smp in samples])
    handles = _gate_oracle(oracle, mask)
    try:
        with torch.no_grad():
            return oracle(q, f, s, seg, im, vm, None, task, compute_pretraining_heads=False)
    finally:
        for hd in handles:
            hd.remove()


def _masks(E, H, B, seed):
    g = torch.Generator().manual_seed(seed)
    binary = (torch.rand(B, E, H, generator=g) > 0.3).float()
    frac = torch.rand(B, E, H, generator=g) * 1.5
    edges = torch.ones(B, E, H)
    edges[0, :, 0] = 0.0                 # first head of every entry off in sample 0
    edges[1, :, -1] = 0.0                # last slot in sample 1 (each entry's last head where it has H heads)
    return {"binary": binary, "fractional": frac, "edges": edges}


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("kind", ["binary", "fractional", "edges"])
def test_gated_against_gated_oracle(tiny_oracle, tiny, mode, kind):
    model = tiny[mode]
    E, H = _shape(model)
    samples = support.batch(model, LENS, seed=35)
    mask = _masks(E, H, len(samples), seed=36)[kind]
    (out, _), _ = _packed(model, samples, head_mask=mask)
    ref = _oracle_padded(tiny_oracle, samples, mask)
    plain = _oracle_padded(tiny_oracle, samples, torch.ones(len(samples), E, H))
    worst = 0.0
    for k in (0, 1, 2, 4):
        err = float((out[k].cpu() - ref[k]).abs().max())
        assert err < _tol(mode, ref[k]), f"output {k}: {err}"
        worst = max(worst, err)
    # the gate moved the oracle's answer by more than the engine's error: the comparison tests the gate, not the ungated path
    assert float((ref[0] - plain[0]).abs().max()) > worst


def test_full_model_gated_against_gated_oracle(full_oracle, full):
    E, H = _shape(full)
    samples = support.batch(full, [(9, 37), (30, 101), (14, 11)], seed=37)
    mask = _masks(E, H, len(samples), seed=38)["binary"]
    heads = _entry_heads(full)
    for e in range(E):
        mask[2, e, 0] = mask[2, e, heads[e] - 1] = 0.0      # first and last head of every entry
    (out, _), _ = _packed(full, samples, head_mask=mask)
    ref = _oracle_padded(full_oracle, samples, mask)
    for k in (0, 1, 2, 4):
        err = float((out[k].cpu() - ref[k]).abs().max())
        assert err < _tol("bf16", ref[k]), f"output {k}: {err}"


# ------------------------------------------------------------------------------------------------ plans and calls
def _count_kernels(model, fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in ev.name
               and "Memset" not in ev.name)


def test_launch_count_equals_ungated(tiny_oracle):
    """Eager launches (no CUDA graph): a gated call launches exactly the ungated call's kernels."""
    model = support.engine(tiny_oracle, compute_dtype="bf16", use_cuda_graph=False, return_attention=True)
    try:
        samples = support.batch(model, LENS, seed=39)
        args = support.packed_sample_args(samples)
        ones = torch.ones(_shape(model))
        for maps in (False, True):
            run = lambda **kw: model.forward_packed(*args, output_all_attention_masks=maps, **kw)
            run(), run(head_mask=ones)            # build both plans
            assert _count_kernels(model, run) == _count_kernels(model, lambda: run(head_mask=ones))
    finally:
        model.close()


def test_plan_reuse_and_back_to_back(tiny):
    """One gated plan serves calls with different gates; unsynchronised back-to-back calls each see their own gate."""
    model = tiny["bf16"]
    E, H = _shape(model)
    samples = support.batch(model, LENS, seed=40)
    args = support.packed_sample_args(samples)
    masks = list(_masks(E, H, len(samples), seed=41).values())
    ref = []
    for m in masks:
        ref.append(model.forward_packed(*args, head_mask=m.cuda())[0].clone())
        torch.cuda.synchronize()
    n = support.n_plans(model)
    got = [model.forward_packed(*args, head_mask=m.cuda())[0] for m in masks]
    torch.cuda.synchronize()
    assert support.n_plans(model) == n
    for a, b in zip(got, ref):
        assert support.eq32(a, b)
    assert not torch.equal(ref[0], ref[1])


def test_rejections(tiny):
    import vilbert_b200 as vb
    L = support.lib()
    model = tiny["bf16"]
    samples = support.batch(model, LENS[:2], seed=42)
    with pytest.raises(ValueError, match="head_mask has shape"):
        model.forward_packed(*support.packed_sample_args(samples), head_mask=torch.ones(3, 2))
    q, f, s, seg, tk, nt, nr = support.packed_sample_args(samples)
    outs, o = model._alloc_packed_outputs(2, sum(nt) + 2, sum(nr), vb.OUT_TASK_HEADS, False, torch.device("cuda", 0))
    inp = L.PackedInputs(2, 0, 0, C.cast((C.c_int32 * 2)(*nt), C.c_void_p), C.cast((C.c_int32 * 2)(*nr), C.c_void_p), q.data_ptr(),
                         seg.data_ptr(), f.data_ptr(), s.data_ptr(), tk.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = L.load().vb200_forward_packed_gated(model._handle, C.byref(inp), None, C.byref(o), vb.OUT_TASK_HEADS, 0, st)
    assert rc == ERR_INVALID and b"head_mask is NULL" in L.load().vb200_last_error(model._handle)
    mask = torch.ones(2, *_shape(model), device="cuda")
    rc = L.load().vb200_forward_packed_gated(model._handle, C.byref(inp), mask.data_ptr(), C.byref(o), L.OUT_ATTENTION, 0, st)
    assert rc == ERR_INVALID and b"VB200_OUT_ATTENTION" in L.load().vb200_last_error(model._handle)
    bad = L.PackedInputs(2, 0, 0, C.cast((C.c_int32 * 2)(0, 3), C.c_void_p), C.cast((C.c_int32 * 2)(*nr), C.c_void_p), q.data_ptr(),
                         seg.data_ptr(), f.data_ptr(), s.data_ptr(), tk.data_ptr())
    rc = L.load().vb200_forward_packed_gated(model._handle, C.byref(bad), mask.data_ptr(), C.byref(o), vb.OUT_TASK_HEADS, 0, st)
    assert rc == ERR_INVALID and b"n_tokens 0" in L.load().vb200_last_error(model._handle)
    rc = L.load().vb200_forward_regions_packed_gated(model._handle, None, mask.data_ptr(), C.byref(o), vb.OUT_TASK_HEADS, 0, st)
    assert rc == ERR_INVALID


def test_split_fp32_rejects_gated_calls(tiny_oracle):
    model = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        samples = support.batch(model, LENS[:2], seed=43)
        with pytest.raises(support.lib().VilbertB200Error, match="split_fp32"):
            model.forward_packed(*support.packed_sample_args(samples), head_mask=torch.ones(_shape(model)))
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------ streaming kernels, head mean
@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("e", [9, 10, 11, 6, 7])
def test_one_gated_head_isolated_streaming(tiny, mode, e):
    """LONG puts sample 0's image stream past 256 rows, so V0 (entry 9) and the connection layers (6 / 7, 10 / 11) run the streaming
    kernels: gating head (e, last head) of sample 0 zeroes that head's map, changes sample 0 and leaves the others bit for bit;
    gating the other direction of the same connection layer gives a different answer (the direction is honoured)."""
    model = tiny[mode]
    E, H = _shape(model)
    samples = support.batch(model, LONG, seed=44)
    B = len(samples)
    (ref, ref_taps), _ = _packed(model, samples)
    m = torch.ones(B, E, H)
    m[0, e, H - 1] = 0.0
    (out, taps), _ = _packed(model, samples, head_mask=m)
    assert support.eq32(taps["pooled_output"][1:], ref_taps["pooled_output"][1:])
    assert not torch.equal(taps["pooled_output"][0], ref_taps["pooled_output"][0])
    kinds, _ = model.attention_selection()
    layer, d = _entry_layer(kinds, e)
    got = out[9][layer] if d is None else out[9][layer][d]
    assert torch.count_nonzero(got[0][H - 1]) == 0 and torch.count_nonzero(got[0][0]) > 0
    if d is not None:
        other = torch.ones(B, E, H)
        other[0, e + (1 if d == 0 else -1), H - 1] = 0.0
        (_, taps2), _ = _packed(model, samples, head_mask=other)
        assert not torch.equal(taps2["pooled_output"][0], taps["pooled_output"][0])


def test_gated_head_mean_is_mean_of_gated_maps(tiny_oracle, tiny):
    """attention_heads="mean" with one gated head: each mean map is (sum over heads of the gated per-head maps, added left to right
    in fp32) / heads, bit for bit, the per-head maps coming from an engine that writes every head."""
    per_head = tiny["bf16"]
    mean = support.engine(tiny_oracle, compute_dtype="bf16", return_attention=True, attention_heads="mean", max_rows_per_sample=1024)
    try:
        E, H = _shape(mean)
        samples = support.batch(mean, LENS, seed=45)
        m = torch.ones(len(samples), E, H)
        m[1, :, 0] = 0.0                       # head 0 of every entry off in sample 1
        m[2, 3, 1] = 0.25
        (a, _), _ = _packed(mean, samples, head_mask=m)
        (b, _), _ = _packed(per_head, samples, head_mask=m)
        for la, lb in zip(a[9], b[9]):
            pairs = zip(la, lb) if isinstance(la, tuple) else [(la, lb)]
            for da, db in pairs:
                for s, (x, y) in enumerate(zip(da, db)):
                    acc = torch.zeros_like(y[0])
                    for h in range(y.shape[0]):
                        acc = acc + y[h]
                    assert support.eq32(x[0], acc / y.shape[0]), f"sample {s}"
    finally:
        mean.close()
