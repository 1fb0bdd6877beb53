"""The ping-pong GEMM (gemm_pingpong.cuh, vb200_linear variant 5) against the cooperative persistent kernel (variant 0).  `-m gpu` only.

The ping-pong kernel applies the same element operations in the same order (one k-ordered fp32 accumulation per element, + bias,
activation, 16-bit conversion), so every comparison here is torch.equal on the raw output bytes.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _operands(M, N, K, f16, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.float16 if f16 else torch.bfloat16
    x = torch.randn(M, K, generator=g, device="cuda").to(dt)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).to(dt)
    b = torch.randn(N, generator=g, device="cuda")
    return x, w, b


def _linear(x, w, b, act, yb, yf, bn, variant, f16, pdl=0, m=None):
    L = support.lib()
    lib = L.load()
    M, K = x.shape
    N = w.shape[0]
    L.check(lib.vb200_linear(x.data_ptr(), K, w.data_ptr(), K, b.data_ptr() if b is not None else None, None, 0, None, None, 1e-12,
                             act, yb.data_ptr() if yb is not None else None, N, yf.data_ptr() if yf is not None else None, N,
                             M if m is None else m, N, K, bn, pdl, 1 if f16 else 0, variant, None, _stream()), None)


def _both(M, N, K, act, bn, f16, outs, seed=0, bias=True):
    """(variant 0, variant 5) outputs of one GEMM; outs = "16", "32" or "16+32"."""
    x, w, b = _operands(M, N, K, f16, seed)
    dt = x.dtype
    res = []
    for variant in (0, 5):
        yb = torch.full((M, N), 7.0, dtype=dt, device="cuda") if "16" in outs else None
        yf = torch.full((M, N), 7.0, device="cuda") if "32" in outs else None
        _linear(x, w, b if bias else None, act, yb, yf, bn, variant, f16)
        res.append((yb, yf))
    torch.cuda.synchronize()
    return res


def _assert_equal(res, what):
    (b0, f0), (b1, f1) = res
    if b0 is not None:
        assert torch.equal(b0.view(torch.int16), b1.view(torch.int16)), f"{what}: 16-bit output differs"
    if f0 is not None:
        assert torch.equal(f0.view(torch.int32), f1.view(torch.int32)), f"{what}: fp32 output differs"


B64_TEXT, B64_IMG = 64 * 31, 64 * 36
# (M, N, K, act, block_n)
CASES = [
    # the plain GEMMs of a batch-64 forward
    (B64_TEXT, 3072, 768, 1, 128), (B64_IMG, 3072, 1024, 0, 128), (B64_IMG, 1024, 1024, 0, 128), (B64_IMG, 1024, 1024, 1, 128),
    (B64_TEXT, 768, 3072, 0, 128), (B64_TEXT, 2304, 768, 0, 128), (B64_TEXT, 768, 768, 0, 128), (B64_TEXT, 768, 1024, 0, 128),
    (B64_IMG, 1024, 2112, 0, 128),
    # the same launches with 64-wide tiles
    (B64_TEXT, 768, 768, 0, 64), (B64_TEXT, 768, 3072, 0, 64), (B64_IMG, 1024, 1024, 1, 64), (B64_TEXT, 3072, 768, 1, 64),
    # ragged M
    (1, 256, 64, 2, 128), (127, 512, 192, 1, 64), (129, 384, 128, 0, 128), (1983, 768, 768, 2, 128), (1983, 768, 256, 1, 64),
    # K: one k-block, ragged k-blocks, long
    (256, 256, 64, 1, 128), (512, 1024, 2112, 0, 64), (384, 512, 3072, 2, 128), (300, 256, 200, 0, 128),
    # tiles per CTA (132 SMs): 100 tiles (one each), 132 (one each), 180 (two each), 324 (three each: one consumer walks one more),
    # 660 (five each)
    (1280, 1280, 256, 0, 128), (1408, 1536, 256, 1, 128), (1920, 1536, 256, 0, 128), (2304, 2304, 256, 2, 128),
    (2816, 3840, 128, 1, 128), (2304, 1152, 128, 0, 64),
]


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "M%d_N%d_K%d_act%d_bn%d" % c)
def test_pingpong_equals_persistent(case, f16):
    """Variant 5 equals variant 0 bit for bit with a 16-bit output, an fp32 output and both."""
    M, N, K, act, bn = case
    for outs in ("16", "32", "16+32"):
        _assert_equal(_both(M, N, K, act, bn, f16, outs, seed=M + N + K), f"{case} {outs}")


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
def test_pingpong_without_bias(f16):
    _assert_equal(_both(700, 512, 256, 1, 128, f16, "16+32", bias=False), "no bias")


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("m", [0, 1, 128, 129, 1000])
def test_pingpong_device_row_count(bn, m):
    """vb200_linear_rows (the ping-pong kernel by default) with m_rows = m at M = 1000: rows < m equal variant 0; every tile that starts
    at or past m is skipped, so rows from the next 128-row boundary on keep the sentinel."""
    L = support.lib()
    lib = L.load()
    M, N, K = 1000, 256, 192
    x, w, b = _operands(M, N, K, True, 5)
    rows = torch.tensor([m], dtype=torch.int32, device="cuda")
    y = torch.full((M, N), 12345.0, device="cuda")
    yb = torch.full((M, N), 3.0, dtype=torch.float16, device="cuda")
    L.check(lib.vb200_linear_rows(x.data_ptr(), K, w.data_ptr(), K, b.data_ptr(), 1, yb.data_ptr(), N, y.data_ptr(), N, M, N, K, bn, 1,
                                  rows.data_ptr(), _stream()), None)
    ref = torch.empty(M, N, device="cuda")
    refb = torch.empty(M, N, dtype=torch.float16, device="cuda")
    _linear(x, w, b, 1, refb, ref, bn, 0, True)
    torch.cuda.synchronize()
    assert torch.equal(y[:m], ref[:m]) and torch.equal(yb[:m], refb[:m])
    boundary = (m + 127) // 128 * 128
    assert bool((y[boundary:] == 12345.0).all()) and bool((yb[boundary:] == 3.0).all())


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
def test_pingpong_pdl_chain(f16):
    """Three dependent ping-pong launches (each reads the previous output) with programmatic dependent launch equal the same chain
    without it."""
    M, N, K = 1984, 768, 768
    x, _, _ = _operands(M, N, K, f16, 11)
    ws = [_operands(1, N, K, f16, 20 + i)[1:] for i in range(3)]
    outs = []
    for pdl in (0, 5):
        cur = x
        for act, (w, b) in zip((1, 0, 2), ws):
            y = torch.empty(M, N, dtype=x.dtype, device="cuda")
            _linear(cur, w, b, act, y, None, 64, 5, f16, pdl=pdl)
            cur = y
        torch.cuda.synchronize()
        outs.append(cur)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))


# ---------------------------------------------------------------- the full model: gemm_kernel 0 (cooperative) against 1 (ping-pong)
def _tensors(x):
    if torch.is_tensor(x):
        return [x.clone()]
    if isinstance(x, dict):
        return [t for k in sorted(x) for t in _tensors(x[k])]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _tensors(v)]
    return []


def _ab(model, run):
    got = []
    for kernel in (0, 1):
        model.set_option("gemm_kernel", kernel)
        out = run()
        torch.cuda.synchronize()
        got.append(_tensors(out))
    model.set_option("gemm_kernel", 1)
    assert len(got[0]) == len(got[1]) and len(got[0]) > 0
    for i, (a, b) in enumerate(zip(*got)):
        assert a.shape == b.shape and torch.equal(a, b), f"tensor {i} differs between the cooperative and the ping-pong kernel"


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_full_model_pingpong_bitwise(full_oracle, dtype):
    """268 M model: a batch-64 forward with the task heads, a packed batch with mixed lengths and a packed retrieval block give the
    same bits with either GEMM kernel."""
    import vilbert_b200 as vb
    from oracle import vilbert_ref as R
    model = support.engine(full_oracle, compute_dtype=dtype)
    try:
        inp = [t.cuda() for t in R.make_inputs(64, 30, 36, seed=3)]
        _ab(model, lambda: model(*inp, select=vb.OUT_TASK_HEADS, debug_taps=True))

        F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
        g = torch.Generator().manual_seed(9)
        tl, vl = [9, 30, 14, 37, 7, 22, 5, 28], [37, 101, 11, 64, 100, 18, 2, 73]
        q = torch.randint(1, vocab, (sum(tl),), generator=g).cuda()
        seg = torch.randint(0, 2, (sum(tl),), generator=g).cuda()
        f = (torch.relu(torch.randn(sum(vl), F, generator=g)) * 1.5).cuda()
        xy = torch.rand(sum(vl), 2, generator=g) * 0.7
        s = torch.cat([xy, xy + 0.2, torch.full((sum(vl), 1), 0.04)], dim=-1).cuda()
        task = torch.randint(0, 20, (len(tl), 1), generator=g).cuda()
        _ab(model, lambda: model.forward_packed(q, f, s, seg, task, tl, vl, select=vb.OUT_ALL, debug_taps=True))

        def retrieval():
            ts = model.encode_text_packed(q[:sum(tl[:6])], seg[:sum(tl[:6])], task[:6], tl[:6])
            vs = model.encode_image_packed(f, s, vl)
            ti = torch.tensor([c for c in range(6) for _ in range(8)])
            ii = torch.tensor([i for _ in range(6) for i in range(8)])
            return ts, vs, model.forward_cached_packed(ts, ti, vs, ii, select=vb.OUT_TASK_HEADS, debug_taps=True)
        _ab(model, retrieval)
    finally:
        model.close()
