"""Sequences past 256 rows per sample (vb200_set_option "max_rows_per_sample", the streaming attention kernels).  `-m gpu` only.

Up to 256 rows per sample a plan stages each (sample, head) of attention whole in shared memory; a plan with more rows in a stream
streams that stream's keys through the streaming kernels, which run the staged kernels' per-key-block arithmetic in the same order.
So the streaming hooks are compared with the staged hooks bit for bit wherever both run, with the fp64 / emulated references past
256 rows, and every long forward with the fp32 oracle and with dense forwards of each sample alone.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kernel_refs as KR
from oracle import detections_ref as D
import support

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
NAN = float("nan")
# tests/test_gpu_kernel_parity.py's attention bounds: error / max(1, |ref|) against fp64
ATTN_TOL = {torch.bfloat16: 1.2e-2, torch.float16: 1.5e-3}
TOL = 1e-2                 # fp16 mode vs the fp32 oracle (tests/test_gpu_model.py)
TOL_BF16_VS_FP32 = 3.5e-2  # bf16 mode vs the fp32 oracle, x max(1, output std) (tests/test_gpu_model.py)
TOL_FP32X = 1e-3           # fp32-parity mode vs the fp32 oracle
BOTH_SIDES = [1, 15, 16, 17, 63, 64, 65, 128, 129, 256]
LONG = [257, 300, 511, 513, 777, 1024]


# ------------------------------------------------------------------------------------------------------------------ op hooks
def _f16(dt):
    return 1 if dt == torch.float16 else 0


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _offs(lengths):
    return [0] + [int(x) for x in np.cumsum(lengths)]


def _dev_i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _key_mask(L, b):
    """Interior masked keys (every (b % 3 + 2)-th) and, for odd b, a masked tail; key 0 always real."""
    m = torch.zeros(L)
    m[1::b % 3 + 2] = -10000.0
    if b % 2 and L > 4:
        m[L - L // 4:] = -10000.0
    m[0] = 0.0
    return m


def _self(hook, qkv, ld_qkv, H, mask, B, L, heads, d, dt, ld_ctx, offs=None, rows=None):
    ctx = torch.full(((rows if rows is not None else B * L) + 16, ld_ctx), NAN, dtype=dt, device="cuda")
    support.call(hook, qkv, ld_qkv, H, mask, ctx, ld_ctx, B, L, heads, d, _f16(dt), offs)
    return ctx


def _co(hook, qi, ld_i, qt, ld_t, H, mi, mt, B, T, V, heads, d, dt, ot=None, ov=None, rows_t=None, rows_v=None):
    ct = torch.full(((rows_t if rows_t is not None else B * T) + 16, H + 8), NAN, dtype=dt, device="cuda")
    ci = torch.full(((rows_v if rows_v is not None else B * V) + 16, H), NAN, dtype=dt, device="cuda")
    support.call(hook, qi, ld_i, qt, ld_t, H, mi, mt, ct, H + 8, ci, H, B, T, V, heads, d, _f16(dt), ot, ov)
    return ct, ci


def _attn_err(ctx, ref):
    return ((ctx.double() - ref).abs() / ref.abs().clamp(min=1.0)).max().item()


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_stream_self_equals_staged(d, dt):
    """Dense (batch 2, one call per length) and packed (every length in one call): the streaming self-attention writes the staged
    kernel's bits at every length both accept, and nothing outside the context rows."""
    heads, H = 2, 2 * d
    ld_qkv, ld_ctx = 3 * H + 8, H + 8
    for L in BOTH_SIDES:
        qkv = torch.randn(2 * L, ld_qkv, generator=_gen(L + d), device="cuda").to(dt)
        mask = torch.stack([_key_mask(L, b) for b in range(2)]).cuda()
        a = _self("vb200_self_attention_stream", qkv, ld_qkv, H, mask, 2, L, heads, d, dt, ld_ctx)
        b = _self("vb200_self_attention_packed", qkv, ld_qkv, H, mask, 2, L, heads, d, dt, ld_ctx, _dev_i32([0, L, 2 * L]))
        torch.cuda.synchronize()
        assert support.eq16(a, b), f"dense L = {L}"
    offs = _offs(BOTH_SIDES)
    qkv = torch.randn(offs[-1], ld_qkv, generator=_gen(d), device="cuda").to(dt)
    mask = torch.cat([_key_mask(L, b) for b, L in enumerate(BOTH_SIDES)]).cuda()
    o = _dev_i32(offs)
    a = _self("vb200_self_attention_stream", qkv, ld_qkv, H, mask, len(BOTH_SIDES), 256, heads, d, dt, ld_ctx, o, offs[-1])
    b = _self("vb200_self_attention_packed", qkv, ld_qkv, H, mask, len(BOTH_SIDES), 256, heads, d, dt, ld_ctx, o, offs[-1])
    torch.cuda.synchronize()
    assert support.eq16(a, b)


CO_PAIRS = [(1, 1), (15, 65), (65, 15), (16, 17), (63, 64), (64, 63), (129, 17), (17, 129), (256, 31), (31, 256), (128, 256)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_stream_co_equals_staged(d, dt):
    """Co-attention with T != V on both sides of 64 and up to 256, dense and packed: bit-identical to the staged kernel."""
    heads, H = 2, 2 * d
    ld_i, ld_t = 3 * H + 8, 3 * H + 24
    for T, V in CO_PAIRS:
        g = _gen(T * 7 + V + d)
        qi = torch.randn(2 * V, ld_i, generator=g, device="cuda").to(dt)
        qt = torch.randn(2 * T, ld_t, generator=g, device="cuda").to(dt)
        mi = torch.stack([_key_mask(V, b) for b in range(2)]).cuda()
        mt = torch.stack([_key_mask(T, b + 1) for b in range(2)]).cuda()
        a = _co("vb200_co_attention_stream", qi, ld_i, qt, ld_t, H, mi, mt, 2, T, V, heads, d, dt)
        b = _co("vb200_co_attention", qi, ld_i, qt, ld_t, H, mi, mt, 2, T, V, heads, d, dt)
        torch.cuda.synchronize()
        assert support.eq16(a[0], b[0]) and support.eq16(a[1], b[1]), f"dense T = {T}, V = {V}"
    T_l, V_l = [t for t, _ in CO_PAIRS], [v for _, v in CO_PAIRS]
    ot, ov = _offs(T_l), _offs(V_l)
    g = _gen(d + 5)
    qi = torch.randn(ov[-1], ld_i, generator=g, device="cuda").to(dt)
    qt = torch.randn(ot[-1], ld_t, generator=g, device="cuda").to(dt)
    mi = torch.cat([_key_mask(V, b) for b, V in enumerate(V_l)]).cuda()
    mt = torch.cat([_key_mask(T, b + 1) for b, T in enumerate(T_l)]).cuda()
    args = (qi, ld_i, qt, ld_t, H, mi, mt, len(T_l), 256, 256, heads, d, dt, _dev_i32(ot), _dev_i32(ov), ot[-1], ov[-1])
    a, b = _co("vb200_co_attention_stream", *args), _co("vb200_co_attention_packed", *args)
    torch.cuda.synchronize()
    assert support.eq16(a[0], b[0]) and support.eq16(a[1], b[1])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_stream_accuracy_past_256(d, dt, parity_log):
    """Streaming self- and co-attention at 257 ... 1024 rows against fp64 (and the emulated rounding points, logged), within the
    bounds of test_gpu_kernel_parity.py."""
    heads, H = 2, 2 * d
    ld = 3 * H
    worst = 0.0
    for L in LONG:
        qkv = torch.randn(L, ld, generator=_gen(L + d), device="cuda").to(dt)
        mask = _key_mask(L, L % 5)[None].cuda()
        ctx = _self("vb200_self_attention_stream", qkv, ld, H, mask, 1, L, heads, d, dt, H)
        torch.cuda.synchronize()
        x = qkv.view(1, L, ld)
        ref = KR.attention_fp64(x[..., :H], x[..., H:2 * H], x[..., 2 * H:], mask, heads)
        em = KR.attention_emulated(x[..., :H].cpu(), x[..., H:2 * H].cpu(), x[..., 2 * H:].cpu(), mask.cpu(), heads, dt == torch.float16)
        err = _attn_err(ctx[:L, :H].view(1, L, H), ref)
        parity_log(test="long_self_attention", L=L, d=d, dtype=str(dt), max_rel_err=err,
                   err_vs_emulated=_attn_err(ctx[:L, :H].view(1, L, H).cpu(), em), bound=ATTN_TOL[dt])
        worst = max(worst, err)
        assert torch.isnan(ctx[L:].float()).all()
    for T, V in [(300, 36), (31, 1024), (777, 513)]:
        g = _gen(T + V + d)
        qi = torch.randn(V, ld, generator=g, device="cuda").to(dt)
        qt = torch.randn(T, ld, generator=g, device="cuda").to(dt)
        mi, mt = _key_mask(V, 1)[None].cuda(), _key_mask(T, 2)[None].cuda()
        ct, ci = _co("vb200_co_attention_stream", qi, ld, qt, ld, H, mi, mt, 1, T, V, heads, d, dt)
        torch.cuda.synchronize()
        xi, xt = qi.view(1, V, ld), qt.view(1, T, ld)
        worst = max(worst, _attn_err(ct[:T, :H].view(1, T, H), KR.attention_fp64(xt[..., :H], xi[..., H:2 * H], xi[..., 2 * H:], mi, heads)),
                    _attn_err(ci[:V, :H].view(1, V, H), KR.attention_fp64(xi[..., :H], xt[..., H:2 * H], xt[..., 2 * H:], mt, heads)))
    assert worst < ATTN_TOL[dt], worst


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_stream_packed_mix_equals_dense(d, dt):
    """A packed batch of lengths 1 ... 1024: every sample equals a dense streaming call of that sample alone, bit for bit."""
    heads, H = 2, 2 * d
    ld = 3 * H + 8
    lens = [1024, 1, 300, 64, 513, 17, 256, 257, 65]
    offs = _offs(lens)
    qkv = torch.randn(offs[-1], ld, generator=_gen(d + 11), device="cuda").to(dt)
    mask = torch.cat([_key_mask(L, b) for b, L in enumerate(lens)]).cuda()
    packed = _self("vb200_self_attention_stream", qkv, ld, H, mask, len(lens), max(lens), heads, d, dt, H, _dev_i32(offs), offs[-1])
    rev = lens[::-1]
    ov = _offs(rev)
    qi = torch.randn(ov[-1], ld, generator=_gen(d + 12), device="cuda").to(dt)
    mi = torch.cat([_key_mask(V, b + 1) for b, V in enumerate(rev)]).cuda()
    ct, ci = _co("vb200_co_attention_stream", qi, ld, qkv, ld, H, mi, mask, len(lens), max(lens), max(rev), heads, d, dt,
                 _dev_i32(offs), _dev_i32(ov), offs[-1], ov[-1])
    for b, L in enumerate(lens):
        sl, sv = slice(offs[b], offs[b + 1]), slice(ov[b], ov[b + 1])
        dense = _self("vb200_self_attention_stream", qkv[sl], ld, H, mask[sl].contiguous(), 1, L, heads, d, dt, H)
        dt_, di_ = _co("vb200_co_attention_stream", qi[sv], ld, qkv[sl], ld, H, mi[sv].contiguous(), mask[sl].contiguous(), 1, L,
                       rev[b], heads, d, dt)
        torch.cuda.synchronize()
        assert support.eq16(packed[sl], dense[:L]), f"self sample {b} (L = {L})"
        assert support.eq16(ct[sl], dt_[:L]) and support.eq16(ci[sv], di_[:rev[b]]), f"co sample {b} (T = {L}, V = {rev[b]})"
    assert torch.isnan(packed[offs[-1]:].float()).all()


# ------------------------------------------------------------------------------------------------------------------ engines
@pytest.fixture(scope="module")
def long_oracle():
    from oracle import vilbert_ref as R
    return R.build(R.tiny_config(max_position_embeddings=1024), seed=7, num_labels=200)


@pytest.fixture(scope="module")
def long_tiny(long_oracle):
    yield from support.engines(long_oracle, ("fp16", "bf16"), max_rows_per_sample=1024)


def test_defaults_unchanged(long_oracle):
    """A default engine keeps the 256-row bound and its messages; the option accepts 256 ... 1024 only."""
    from vilbert_b200 import _lib as L
    m = support.engine(long_oracle)
    try:
        v = C.c_int64()
        L.check(L.load().vb200_model_dim(m._handle, b"max_rows_per_sample", C.byref(v)), m._handle)
        assert v.value == 256 and m.max_rows_per_sample == 256
        err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: .*" + pat)
        with err(r"sequence too long for the small-sequence attention kernels \(T=257, V=36, max 256\)"):
            m.plan_info(1, 256, 36)
        with err(r"\(T=31, V=257, max 256\)"):
            m.plan_info(1, 30, 257)
        with err(r"sample 0 too long for the small-sequence attention kernels \(V=257, max 256\)"):
            m.attention_layout_packed([3], [257])
        with err(r"max_boxes = 256 outside \[1, 255\]"):
            from vilbert_b200 import synthetic as S
            m.select_regions(S.synthetic_detections(1, [300], n_classes=20, feature_size=8, seed=1), 256)
        for bad in (255, 1025):
            with err("max_rows_per_sample must be in"):
                m.set_option("max_rows_per_sample", bad)
        assert m.max_rows_per_sample == 256
        with pytest.raises(ValueError):
            support.engine(long_oracle, max_rows_per_sample=1025)
        # raising and lowering the bound is validation only
        m.set_option("max_rows_per_sample", 300)
        m.plan_info(1, 256, 36)
        m.set_option("max_rows_per_sample", 256)
        with err("T=257"):
            m.plan_info(1, 256, 36)
    finally:
        m.close()


def test_default_plan_launches_unchanged(tiny_oracle):
    """The plan of a short shape is the same launch list whatever the bound."""
    a, b = support.engine(tiny_oracle), support.engine(tiny_oracle, max_rows_per_sample=1024)
    try:
        for shape in [(2, 30, 36), (1, 155, 256)]:
            assert a.plan_info(*shape) == b.plan_info(*shape)
    finally:
        a.close()
        b.close()


NAMES = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction",
         "vision_prediction", "vision_logit", "linguisic_prediction", "linguisic_logit"]


def _check_vs_oracle(oracle, model, inputs, tol_fn, tag, parity_log):
    ref = oracle(*inputs, compute_pretraining_heads=True)
    out = model(*[t.cuda() for t in inputs], compute_pretraining_heads=True)
    torch.cuda.synchronize()
    for i, name in enumerate(NAMES):
        r, o = ref[i], out[i]
        if r is None:
            assert o is None, name
            continue
        diff = (o.cpu() - r).abs()
        small = r.abs() < 1000
        err, std = float(diff[small].max()), float(r[small].std()) if small.sum() > 1 else 0.0
        parity_log(test=tag, output=name, max_abs_err=err, ref_std=std)
        assert err < tol_fn(std), f"{tag}: {name}: {err}"


@pytest.mark.parametrize("Tin,V", [(300, 36), (511, 257), (30, 1000)])
@pytest.mark.parametrize("mode", ["fp16", "bf16"])
def test_long_model_vs_oracle(long_oracle, long_tiny, mode, Tin, V, parity_log):
    """Tiny 12/6/6 model with 1024 positions and the bound at 1024: all nine outputs of dense long forwards vs the fp32 oracle."""
    tol = (lambda s: TOL) if mode == "fp16" else (lambda s: TOL_BF16_VS_FP32 * max(1.0, s))
    _check_vs_oracle(long_oracle, long_tiny[mode], support.tiny_inputs(long_oracle, 1, Tin, V, Tin + V), tol, f"long_{mode}_T{Tin}_V{V}",
                     parity_log)


def test_long_model_fp32x_vs_oracle(long_oracle, parity_log):
    """fp32-parity mode (fp32 attention kernel) on dense long forwards: 1e-3 against the fp32 oracle."""
    m = support.engine(long_oracle, compute_dtype="fp32x", max_rows_per_sample=1024)
    try:
        for Tin, V in [(300, 36), (511, 257), (30, 1000)]:
            _check_vs_oracle(long_oracle, m, support.tiny_inputs(long_oracle, 1, Tin, V, Tin + V), lambda s: TOL_FP32X, f"long_fp32x_T{Tin}_V{V}",
                             parity_log)
    finally:
        m.close()


def test_full_model_long(full_oracle, parity_log):
    """The 268 M model once at (Tin, V) = (511, 300) in bf16."""
    m = support.engine(full_oracle, compute_dtype="bf16", max_rows_per_sample=1024)
    try:
        _check_vs_oracle(full_oracle, m, list(support.tiny_inputs(full_oracle, 1, 511, 300, 5)), lambda s: TOL_BF16_VS_FP32 * max(1.0, s),
                         "long_full_bf16", parity_log)
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------------ packed
def _rows(t, counts):
    o = _offs(counts)
    return [t[o[i]:o[i + 1]] for i in range(len(counts))]


ROW_OUT = {5: "v", 6: "v", 7: "t", 8: "t"}


def _assert_per_sample(out, samples, dense_models, select_all):
    t_rows = [len(s[0]) + 1 for s in samples]
    v_rows = [s[2].shape[0] for s in samples]
    for i, smp in enumerate(samples):
        for model in dense_models(smp):
            ref = support.dense_alone(model, smp, select=select_all)
            for k in range(9):
                if k == 3 or out[k] is None:
                    continue            # the pair head reads two samples
                got = _rows(out[k], v_rows if ROW_OUT[k] == "v" else t_rows)[i] if k in ROW_OUT else out[k][i]
                assert torch.equal(got, ref[k][0]), f"sample {i} (T = {t_rows[i]}, V = {v_rows[i]}): output {k}"


LENS = [(300, 36), (30, 1000), (255, 256), (12, 257), (511, 100), (1, 1)]


def test_packed_long_equals_dense(tiny_oracle, long_oracle, long_tiny):
    """forward_packed with capacities above 256 and samples on both sides of 256 rows: each sample's outputs equal a dense forward of
    it alone; samples of at most 256 rows also equal a dense forward on a default engine (staged kernels)."""
    import vilbert_b200 as vb
    model = long_tiny["bf16"]
    default = support.engine(long_oracle, compute_dtype="bf16")
    try:
        F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
        samples = [support.sample(t, v, 30 + i, F, vocab) for i, (t, v) in enumerate(LENS)]
        cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda()
        task = torch.tensor([[s[4]] for s in samples]).cuda()
        out = model.forward_packed(cat(0), cat(2), cat(3), cat(1), task, [len(s[0]) for s in samples],
                                   [s[2].shape[0] for s in samples], select=vb.OUT_ALL)
        torch.cuda.synchronize()
        short = lambda s: len(s[0]) + 1 <= 256 and s[2].shape[0] <= 256
        _assert_per_sample(out, samples, lambda s: [model] + ([default] if short(s) else []), vb.OUT_ALL)
    finally:
        default.close()


def test_packed_long_attention_maps(long_oracle):
    """Packed attention maps at lengths past 256 equal each sample's dense maps."""
    import vilbert_b200 as vb
    model = support.engine(long_oracle, compute_dtype="bf16", max_rows_per_sample=1024, return_attention=True)
    try:
        F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
        lens = [(300, 20), (10, 280), (3, 3)]
        samples = [support.sample(t, v, 50 + i, F, vocab) for i, (t, v) in enumerate(lens)]
        cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda()
        task = torch.tensor([[s[4]] for s in samples]).cuda()
        out = model.forward_packed(cat(0), cat(2), cat(3), cat(1), task, [len(s[0]) for s in samples],
                                   [s[2].shape[0] for s in samples], select=vb.OUT_TASK_HEADS, output_all_attention_masks=True)
        torch.cuda.synchronize()
        for i, (q, seg, f, s, tk) in enumerate(samples):
            ref = model(q[None].cuda(), f[None].cuda(), s[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
                        torch.ones(1, f.shape[0], dtype=torch.uint8).cuda(), None, torch.tensor([[tk]]).cuda(),
                        select=vb.OUT_TASK_HEADS, output_all_attention_masks=True)
            torch.cuda.synchronize()
            assert len(out[9]) == len(ref[9])
            for layer, (p, r) in enumerate(zip(out[9], ref[9])):
                if isinstance(p, tuple):
                    assert torch.equal(p[0][i], r[0][0]) and torch.equal(p[1][i], r[1][0]), (i, layer)
                else:
                    assert torch.equal(p[i], r[0]), (i, layer)
    finally:
        model.close()


def test_regions_packed_long_equals_dense(long_oracle, long_tiny):
    """forward_regions_packed with images of up to 700 boxes and texts on both sides of 256 rows: each image's outputs and spatials
    equal a dense forward_regions of that image alone; images of at most 256 rows also equal it on a default engine (staged
    kernels), so the kernel the packed plan picked does not show."""
    import vilbert_b200 as vb
    model = long_tiny["fp16"]
    default = support.engine(long_oracle, compute_dtype="fp16")
    F = model._dims["v_feature_size"]
    g = torch.Generator().manual_seed(3)
    cases = [(300, 400), (20, 100), (5, 700), (254, 255), (255, 40)]
    imgs = []
    for tin, n in cases:
        x1, y1 = torch.rand(n, generator=g) * 400, torch.rand(n, generator=g) * 300
        bx = torch.stack([x1, y1, x1 + 10 + torch.rand(n, generator=g) * 100, y1 + 10 + torch.rand(n, generator=g) * 100], -1)
        imgs.append((torch.randint(1, 2000, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g),
                     torch.relu(torch.randn(n, F, generator=g)), bx, [640.0, 480.0], int(torch.randint(0, 20, (1,), generator=g))))
    try:
        out, sp = model.forward_regions_packed(torch.cat([b[0] for b in imgs]), torch.cat([b[1] for b in imgs]),
                                               torch.tensor([[b[5]] for b in imgs]), torch.cat([b[2] for b in imgs]),
                                               torch.cat([b[3] for b in imgs]), torch.tensor([b[4] for b in imgs]),
                                               [len(b[0]) for b in imgs], [b[2].shape[0] for b in imgs], select=vb.OUT_ALL)
        torch.cuda.synchronize()
        t_rows = [len(b[0]) + 1 for b in imgs]
        v_rows = [b[2].shape[0] + 1 for b in imgs]
        for i, b in enumerate(imgs):
            engines = [model] + ([default] if t_rows[i] <= 256 and v_rows[i] <= 256 else [])
            for eng in engines:
                ref, rsp = support.regions_alone(eng, b, vb.OUT_ALL)
                assert torch.equal(_rows(sp, v_rows)[i], rsp[0]), i
                for k in range(9):
                    if k == 3 or out[k] is None:
                        continue            # the pair head reads two images
                    got = _rows(out[k], v_rows if ROW_OUT[k] == "v" else t_rows)[i] if k in ROW_OUT else out[k][i]
                    assert torch.equal(got, ref[k][0]), (i, k, eng is default)
    finally:
        default.close()


def test_packed_bound_not_multiple_of_16(long_oracle):
    """A bound of 300 (packed capacities round up to 304): packed forwards, region forwards and retrieval calls with samples at the
    bound run and equal dense forwards; one row more is rejected, naming the option."""
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    m = support.engine(long_oracle, compute_dtype="fp16", max_rows_per_sample=300)
    try:
        F, vocab = m._dims["v_feature_size"], m._dims["vocab_size"]
        samples = [support.sample(299, 300, 90, F, vocab), support.sample(7, 291, 91, F, vocab), support.sample(290, 3, 92, F, vocab)]
        cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda()
        task = torch.tensor([[s[4]] for s in samples]).cuda()
        nt, nv = [len(s[0]) for s in samples], [s[2].shape[0] for s in samples]
        out = m.forward_packed(cat(0), cat(2), cat(3), cat(1), task, nt, nv, select=vb.OUT_ALL)
        torch.cuda.synchronize()
        _assert_per_sample(out, samples, lambda s: [m], vb.OUT_ALL)
        # capacities at the bound: max_tokens 299 (T = 300), max_boxes 299 (V = 300)
        wh = torch.tensor([[640.0, 480.0]] * 3)
        bx = torch.cat([torch.tensor([[10.0, 20.0, 200.0, 300.0]]).repeat(n - 1, 1) for n in nv])
        m.forward_regions_packed(cat(0), cat(1), task, torch.cat([s[2][1:] for s in samples]), bx, wh, nt, [n - 1 for n in nv],
                                 max_tokens=299, max_boxes=299)
        ts = m.encode_text_packed(cat(0), cat(1), task, nt, max_tokens=299)
        vs = m.encode_image_packed(cat(2), cat(3), nv, max_regions=300)
        cached = m.forward_cached_packed(ts, [0, 1, 2], vs, [0, 1, 2], select=vb.OUT_VIL_LOGIT)
        torch.cuda.synchronize()
        assert torch.equal(cached[2], out[2])
        err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: .*" + pat)
        with err(r"too long for this engine's max_rows_per_sample \(T=301, max 300\)"):
            m.forward_packed(cat(0)[:300], cat(2)[:1], cat(3)[:1], cat(1)[:300], task[:1], [300], [1])
        with err(r"sequence too long for this engine's max_rows_per_sample \(T=32, V=301, max 300\)"):
            m.plan_info(1, 31, 301)
    finally:
        m.close()


def test_retrieval_long_equals_forward_packed(long_tiny):
    """encode_text_packed / encode_image_packed / forward_cached_packed with captions and images past 256 rows: scores equal
    forward_packed of the same pairs, bit for bit."""
    import vilbert_b200 as vb
    model = long_tiny["fp16"]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    caps = [support.sample(t, 1, 70 + i, F, vocab) for i, t in enumerate([400, 12, 256])]
    ims = [support.sample(1, v, 80 + i, F, vocab) for i, v in enumerate([300, 36, 257])]
    pairs = [(0, 0), (1, 2), (2, 1), (0, 1), (2, 2)]
    task = 7
    nt = [len(c[0]) for c in caps]
    nv = [im[2].shape[0] for im in ims]
    ts = model.encode_text_packed(torch.cat([c[0] for c in caps]).cuda(), torch.cat([c[1] for c in caps]).cuda(),
                                  torch.full((len(caps), 1), task).cuda(), nt)
    vs = model.encode_image_packed(torch.cat([im[2] for im in ims]).cuda(), torch.cat([im[3] for im in ims]).cuda(), nv)
    cached = model.forward_cached_packed(ts, [p[0] for p in pairs], vs, [p[1] for p in pairs], select=vb.OUT_VIL_LOGIT)
    q = torch.cat([caps[a][0] for a, _ in pairs]).cuda()
    seg = torch.cat([caps[a][1] for a, _ in pairs]).cuda()
    f = torch.cat([ims[b][2] for _, b in pairs]).cuda()
    s = torch.cat([ims[b][3] for _, b in pairs]).cuda()
    full = model.forward_packed(q, f, s, seg, torch.full((len(pairs), 1), task).cuda(), [nt[a] for a, _ in pairs],
                                [nv[b] for _, b in pairs], select=vb.OUT_VIL_LOGIT)
    torch.cuda.synchronize()
    assert torch.equal(cached[2], full[2])


# ------------------------------------------------------------------------------------------------------------------ regions
def test_select_regions_600_boxes(long_tiny, tiny_oracle):
    """select_regions keeps up to bound - 1 boxes: 600 of 1000 proposals match the oracle; at max_boxes <= 255 a default engine and
    the raised bound give the same rows."""
    from vilbert_b200 import synthetic as S
    dets = S.synthetic_detections(3, [1000, 700, 2048], n_classes=301, feature_size=64, seed=4, margin=0.05)
    m = long_tiny["bf16"]
    r = m.select_regions(dets, 600, cls_prob=True, objects=True)
    torch.cuda.synchronize()
    for i, d in enumerate(dets):
        ref = D.select_image(*d, max_boxes=600)
        lo, k = r["dst_rows"][i], r["n_boxes"][i]
        assert k == ref["keep"].shape[0]
        np.testing.assert_array_equal(r["keep_index"][lo:lo + k].cpu().numpy(), ref["keep"])
        assert int(r["num_boxes"][i]) == ref["num_boxes"]
        np.testing.assert_array_equal(r["objects"][lo:lo + k].cpu().numpy(), ref["argmax"])
        assert torch.equal(r["boxes"][lo:lo + k].cpu(), torch.from_numpy(ref["bbox"]))
        assert torch.equal(r["box_features"][lo:lo + k].cpu(), torch.from_numpy(ref["features"]))
    default = support.engine(tiny_oracle, compute_dtype="bf16")
    try:
        for K in (100, 255):
            a = m.select_regions(dets, K, cls_prob=True, objects=True)
            b = default.select_regions(dets, K, cls_prob=True, objects=True)
            torch.cuda.synchronize()
            assert a["dst_rows"] == b["dst_rows"] and a["n_boxes"] == b["n_boxes"] and torch.equal(a["num_boxes"], b["num_boxes"])
            for i, (lo, k) in enumerate(zip(a["dst_rows"], a["n_boxes"])):
                for key in ("keep_index", "boxes", "box_features", "objects", "max_conf", "cls_prob"):
                    assert torch.equal(a[key][lo:lo + k].cpu(), b[key][lo:lo + k].cpu()), (K, i, key)
    finally:
        default.close()


# ------------------------------------------------------------------------------------------------------------------ worker
DIALOG_WORDS = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "is", "it", "the", "a", "dog", "on", "grass", "man", "holding", "red", "hat",
                "left", "one", "yes", "no", "?", ",", ".", "##s"]


def test_worker_long_dialog_and_many_boxes(full_oracle, tmp_path):
    """custom_prediction_packed and custom_prediction_detections on a GuessWhat dialog of about 300 wordpieces (vocab file written
    here) and an image with 400 boxes, on the full model loaded with max_rows_per_sample = 410 (not a multiple of 16): the answers
    equal the host decode of the oracle's logits on the reference tensor construction."""
    import vilbert_b200 as vb
    from vilbert_b200 import synthetic as S
    from vilbert_b200 import worker_api as W
    vocab = tmp_path / "vocab.txt"
    vocab.write_text("\n".join(DIALOG_WORDS) + "\n")
    cfg = vb.BertConfig.from_dict(full_oracle.config.to_dict())
    m = W.load_vilbert_model(full_oracle.state_dict(), cfg, num_labels=full_oracle.num_labels, vocab_file=str(vocab),
                             max_rows_per_sample=410)
    try:
        assert m.max_rows_per_sample == 410
        turn = "is it the dog on the grass ? no , is it a man holding a red hat ? yes . is it the left one ? no . "
        query = (turn * 10).strip()
        n_tok = len(W.real_tokens(query)[0])
        assert 280 <= n_tok <= 320, n_tok
        F = m._dims["v_feature_size"]
        dets = S.synthetic_detections(1, [1000], n_classes=1601, feature_size=F, seed=17, margin=0.05)
        sel = D.select_image(*dets[0], max_boxes=400)
        assert sel["features"].shape[0] == 400
        size = {"image_width": 640.0, "image_height": 480.0}
        host_info = dict(size, bbox=sel["bbox"])
        feats = torch.from_numpy(sel["features"])
        got_packed = W.custom_prediction_packed([(query, [16], [feats], [host_info], "16")], max_boxes=400)[0]
        got_det = W.custom_prediction_detections([(query, [16], dets, [dict(size)], "16")], max_boxes=400)[0]
        assert not isinstance(got_packed, Exception), got_packed
        assert not isinstance(got_det, Exception), got_det
        inp = W.build_inputs(query, [16], [feats], [host_info], torch.device("cpu"))
        assert inp[0].shape[1] == n_tok and inp[1].shape[1] == 401
        ref = full_oracle(*inp, compute_pretraining_heads=False)
        want = W._decode("16", ref, inp[2], [host_info])
        for got in (got_packed, got_det):
            assert [(a["x1"], a["y1"], a["x2"], a["y2"]) for a in got] == [(a["x1"], a["y1"], a["x2"], a["y2"]) for a in want]
            assert [a["confidence"] for a in got] == pytest.approx([a["confidence"] for a in want], abs=0.5)
        # one box more than the bound allows is the request's error, not the call's
        too_many = W.custom_prediction_packed([(query, [16], [torch.zeros(410, F)], [dict(size, bbox=np.zeros((410, 4)))], "16")])[0]
        assert isinstance(too_many, ValueError) and "409" in str(too_many)
    finally:
        m.close()
