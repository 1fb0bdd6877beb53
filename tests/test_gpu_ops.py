"""Kernel-level parity through the C ABI (vb200_linear / vb200_self_attention / vb200_co_attention)
against plain fp32 torch math on the same bf16-rounded operands.  `-m gpu` only."""
import ctypes as C
import math

import pytest
import torch

import support

pytestmark = pytest.mark.gpu


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


VARIANT = 0     # vb200_linear variant; 2 (the ABI name of the Blackwell CTA-pair kernel) selects the persistent kernel too


@pytest.fixture(params=[0, 2], ids=["persistent", "pair"])
def variant(request):
    global VARIANT
    VARIANT = request.param
    yield request.param
    VARIANT = 0


def run_linear(x, w, bias=None, act=0, block_n=0, want_bf16=True, want_f32=True, ld_f32=None, pdl=0):
    """x, w: both fp16 or both bf16 (wgmma needs matching operand formats); same format for the 16-bit output."""
    L = support.lib()
    lib = L.load()
    M, K = x.shape
    N = w.shape[0]
    dev = x.device
    f16 = 1 if x.dtype == torch.float16 else 0
    yb = torch.zeros(M, N, dtype=x.dtype, device=dev) if want_bf16 and N % 8 == 0 else None
    ldf = ld_f32 or N
    yf = torch.full((M, ldf), float("nan"), dtype=torch.float32, device=dev) if want_f32 else None
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.vb200_linear(_ptr(x), x.stride(0), _ptr(w), w.stride(0), _ptr(bias), None, 0, None, None, 1e-12, act,
                          _ptr(yb), N, _ptr(yf), ldf, M, N, K, block_n, pdl, f16, VARIANT, None, C.c_void_p(stream))
    L.check(rc, None)
    torch.cuda.synchronize()
    return yb, (yf[:, :N] if yf is not None else None)


def ref_linear(x, w, bias=None, act=0):
    y = x.double() @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if act == 1:
        y = y * 0.5 * (1.0 + torch.erf(y / math.sqrt(2.0)))
    elif act == 2:
        y = torch.relu(y)
    return y.float()


ACT = [torch.float16, torch.bfloat16]


def _mk(M, N, K, seed=0, act=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, generator=g, device="cuda").to(act)
    w = (torch.randn(N, K, generator=g, device="cuda") * (1.0 / math.sqrt(K))).to(act)
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    return x, w, b, g


@pytest.mark.parametrize("M,N,K,block_n", [
    (128, 128, 64, 128),        # one tile, one k-block
    (128, 128, 256, 128),       # k loop, ring not wrapped
    (256, 256, 1024, 128),      # ring wraps (16 k-blocks > 6 stages)
    (200, 384, 768, 128),       # ragged M
    (1984, 2304, 768, 128),     # text QKV at B=64
    (2304, 3072, 1024, 128),    # co-attention image QKV at B=64
    (1984, 3072, 768, 256),     # block_n 256: runs as 128-wide tiles
    (1984, 3072, 768, 192),     # 128x192 tiles: the N = 3072 GEMMs at batch 64 in 16 column tiles
    (2304, 3072, 1024, 192),
    (300, 384, 512, 192),       # ragged M, two N tiles
    (77, 64, 128, 64),          # narrow tile
    (64, 3129, 2048, 128),      # VQA logits: ragged N, M < tile
    (15872, 3072, 768, 128),    # B=512 text FFN-in: 2976 tiles, ~10 per persistent CTA
])
@pytest.mark.parametrize("act_dt", ACT)
def test_linear_bias(M, N, K, block_n, act_dt, variant, parity_log):
    if variant == 2 and block_n not in (128, 256):
        pytest.skip("variant 2 is the plain 128-wide tile (block_n 256 runs as 128)")
    x, w, b, _ = _mk(M, N, K, act=act_dt)
    ld = (N + 3) // 4 * 4
    yb, yf = run_linear(x, w, b, block_n=block_n, ld_f32=ld)
    ref = ref_linear(x, w, b)
    err = (yf - ref).abs().max().item()
    parity_log(test="linear_bias", M=M, N=N, K=K, block_n=block_n, act=str(act_dt), max_abs_err=err, ref_std=ref.std().item())
    assert err < 2e-3, f"fp32 output max abs err {err}"
    if yb is not None:
        errb = (yb.float() - ref).abs().max().item()
        assert errb < 3e-2, f"bf16 output max abs err {errb}"


@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("act", [1, 2])
def test_linear_act(act, act_dt, variant, parity_log):
    x, w, b, _ = _mk(300, 1024, 512, seed=1, act=act_dt)
    _, yf = run_linear(x, w, b, act=act)
    ref = ref_linear(x, w, b, act=act)
    err = (yf - ref).abs().max().item()
    parity_log(test="linear_act", act=act, max_abs_err=err)
    assert err < 2e-3


def test_linear_pdl_chain():
    """Two dependent GEMMs launched with programmatic dependent launch give the same result as without."""
    x, w, b, _ = _mk(512, 512, 512, seed=4)
    y1, _ = run_linear(x, w, b, pdl=0)
    y2a, _ = run_linear(x, w, b, pdl=1)
    assert torch.equal(y1, y2a)


def _attn_ref(q, k, v, mask_add, heads):
    B, Lq, H = q.shape
    Lk = k.shape[1]
    d = H // heads
    qh = q.float().view(B, Lq, heads, d).permute(0, 2, 1, 3)
    kh = k.float().view(B, Lk, heads, d).permute(0, 2, 1, 3)
    vh = v.float().view(B, Lk, heads, d).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(d) + mask_add[:, None, None, :]
    p = torch.softmax(s, dim=-1)
    return (p @ vh).permute(0, 2, 1, 3).reshape(B, Lq, H)


@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("B,L,heads,d", [(3, 31, 12, 64), (2, 38, 12, 64), (2, 36, 8, 128), (2, 101, 8, 128),
                                         (1, 129, 2, 64), (2, 17, 2, 128), (1, 256, 2, 128), (2, 1, 2, 64), (1, 2, 1, 128)])
def test_self_attention(B, L, heads, d, act_dt, parity_log):
    Lm = support.lib()
    lib = Lm.load()
    H = heads * d
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(B * L, 3 * H, generator=g, device="cuda").to(act_dt)
    mask = torch.zeros(B, L, device="cuda")
    mask[:, L - L // 4:] = -10000.0
    mask[0] = 0.0
    ctx = torch.zeros(B * L, H, dtype=act_dt, device="cuda")
    rc = lib.vb200_self_attention(_ptr(qkv), 3 * H, H, _ptr(mask), _ptr(ctx), H, B, L, heads, d,
                                  1 if act_dt == torch.float16 else 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    Lm.check(rc, None)
    torch.cuda.synchronize()
    x = qkv.view(B, L, 3 * H)
    ref = _attn_ref(x[..., :H], x[..., H:2 * H], x[..., 2 * H:], mask, heads)
    err = (ctx.view(B, L, H).float() - ref).abs().max().item()
    parity_log(test="self_attention", B=B, L=L, heads=heads, d=d, max_abs_err=err)
    assert err < 2e-2


@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("B,T,V,heads,d", [(3, 31, 36, 8, 128), (2, 38, 101, 8, 128), (2, 17, 10, 2, 128),
                                           (1, 129, 100, 8, 128), (1, 256, 256, 2, 128), (2, 2, 1, 2, 128), (1, 1, 200, 1, 64)])
def test_co_attention(B, T, V, heads, d, act_dt, parity_log):
    Lm = support.lib()
    lib = Lm.load()
    H = heads * d
    g = torch.Generator(device="cuda").manual_seed(6)
    qkv_i = torch.randn(B * V, 3 * H, generator=g, device="cuda").to(act_dt)
    qkv_t = torch.randn(B * T, 3 * H, generator=g, device="cuda").to(act_dt)
    mi = torch.zeros(B, V, device="cuda")
    mi[:, V - 3:] = -10000.0
    mt = torch.zeros(B, T, device="cuda")
    mt[:, T - 5:] = -10000.0
    ctx_t = torch.zeros(B * T, H, dtype=act_dt, device="cuda")
    ctx_i = torch.zeros(B * V, H, dtype=act_dt, device="cuda")
    rc = lib.vb200_co_attention(_ptr(qkv_i), 3 * H, _ptr(qkv_t), 3 * H, H, _ptr(mi), _ptr(mt), _ptr(ctx_t), H,
                                _ptr(ctx_i), H, B, T, V, heads, d, 1 if act_dt == torch.float16 else 0,
                                C.c_void_p(torch.cuda.current_stream().cuda_stream))
    Lm.check(rc, None)
    torch.cuda.synchronize()
    xi, xt = qkv_i.view(B, V, 3 * H), qkv_t.view(B, T, 3 * H)
    ref_t = _attn_ref(xt[..., :H], xi[..., H:2 * H], xi[..., 2 * H:], mi, heads)       # text queries, image keys/values
    ref_i = _attn_ref(xi[..., :H], xt[..., H:2 * H], xt[..., 2 * H:], mt, heads)       # image queries, text keys/values
    e1 = (ctx_t.view(B, T, H).float() - ref_t).abs().max().item()
    e2 = (ctx_i.view(B, V, H).float() - ref_i).abs().max().item()
    parity_log(test="co_attention", B=B, T=T, V=V, err_text_ctx=e1, err_image_ctx=e2)
    assert e1 < 2e-2 and e2 < 2e-2


@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("M,N,with_res", [(1984, 768, True), (2304, 1024, True), (64, 2048, False), (37, 128, True), (5, 256, False)])
def test_layernorm_row_kernel(M, N, with_res, act_dt, parity_log):
    """vb200_layernorm: LayerNorm(y + residual) with fp32 and 16-bit outputs (the LayerNorm after every residual GEMM)."""
    L = support.lib()
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(9)
    y = torch.randn(M, N, generator=g, device="cuda") * 3 + 0.5
    res = torch.randn(M, N, generator=g, device="cuda") if with_res else None
    gamma = 1.0 + 0.1 * torch.randn(N, generator=g, device="cuda")
    beta = 0.1 * torch.randn(N, generator=g, device="cuda")
    of = torch.empty(M, N, device="cuda")
    oh = torch.empty(M, N, dtype=act_dt, device="cuda")
    rc = lib.vb200_layernorm(_ptr(y), N, _ptr(res), N if with_res else 0, _ptr(gamma), _ptr(beta), 1e-12, _ptr(of), N, _ptr(oh), N,
                             M, N, 1 if act_dt == torch.float16 else 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    L.check(rc, None)
    torch.cuda.synchronize()
    x = (y + res if with_res else y).double()
    u = x.mean(-1, keepdim=True)
    ref = ((x - u) / torch.sqrt((x - u).pow(2).mean(-1, keepdim=True) + 1e-12) * gamma.double() + beta.double()).float()
    err = (of - ref).abs().max().item()
    parity_log(test="layernorm_row", M=M, N=N, max_abs_err=err)
    assert err < 1e-5
    assert (oh.float() - ref).abs().max().item() < 5e-2


# ----------------------------------------------------------------------------------------------- round 2
@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("act", [1, 2])
def test_linear_act_192(act, act_dt, parity_log):
    x, w, b, _ = _mk(1984, 3072, 768, seed=3, act=act_dt)
    yb, yf = run_linear(x, w, b, act=act, block_n=192)
    ref = ref_linear(x, w, b, act=act)
    err = (yf - ref).abs().max().item()
    parity_log(test="linear_act_192", act=act, max_abs_err=err)
    assert err < 2e-3
    assert (yb.float() - ref).abs().max().item() < 3e-2
    _, y128 = run_linear(x, w, b, act=act, block_n=128)
    assert torch.equal(yf, y128)                      # the tile width does not change a single bit


def test_linear_gelu_outliers():
    """ADVICE r1: FFN pre-activations far from the origin (real checkpoints have outliers): GELU(-50) must be 0, not
    -1.1e-5 * x, and GELU(+50) must be x."""
    x, w, b, _ = _mk(256, 256, 128, seed=9, act=torch.float16)
    b = b * 0.0
    b[:64] = -60.0
    b[64:128] = 60.0
    _, yf = run_linear(x, w, b, act=1)
    ref = ref_linear(x, w, b, act=1)
    assert (yf[:, :64] == 0).all(), yf[:, :64].abs().max().item()
    assert (yf - ref).abs().max().item() < 2e-3


def _split_act(x):
    """fp32 [M, K] (K % 64 == 0) -> fp16 hi | lo | hi per 64 columns, [M, 3K] (common.cuh split_col)."""
    hi = x.clamp(-65504, 65504).half()
    lo = (x - hi.float()).half()
    M, K = x.shape
    return torch.stack([hi.view(M, K // 64, 64), lo.view(M, K // 64, 64), hi.view(M, K // 64, 64)], dim=2).reshape(M, 3 * K).contiguous()


def _split_w(w):
    hi = w.half()
    lo = (w - hi.float()).half()
    N, K = w.shape
    return torch.stack([hi.view(N, K // 64, 64), hi.view(N, K // 64, 64), lo.view(N, K // 64, 64)], dim=2).reshape(N, 3 * K).contiguous()


def _unsplit(y3):
    """hi | lo | hi layout -> fp32 hi + lo (and check the second hi copy)."""
    M, K3 = y3.shape
    v = y3.view(M, K3 // 192, 3, 64).float()
    assert torch.equal(v[:, :, 0], v[:, :, 2])
    return (v[:, :, 0] + v[:, :, 1]).reshape(M, K3 // 3)


@pytest.mark.parametrize("M,N,K,act", [(128, 128, 64, 0), (300, 384, 768, 3), (1984, 768, 3072, 0), (64, 3136, 2048, 2),
                                        (77, 64, 128, 0)])
def test_linear_split_operands(M, N, K, act, parity_log):
    """fp32-parity mode GEMM: fp16 hi/lo split operands, K' = 3K; against fp64 math on the ORIGINAL fp32 operands."""
    L = support.lib()
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, K, generator=g, device="cuda") * 1.7
    w = torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    x3, w3 = _split_act(x), _split_w(w)
    y3 = torch.zeros(M, 3 * N, dtype=torch.float16, device="cuda")
    yf = torch.full((M, N), float("nan"), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    L.check(lib.vb200_linear_split(_ptr(x3), 3 * K, _ptr(w3), 3 * K, _ptr(b), act, _ptr(y3), 3 * N, _ptr(yf), N, M, N, 3 * K,
                                   C.c_void_p(st)), None)
    torch.cuda.synchronize()
    ref = ref_linear(x, w, b, act=1 if act == 3 else act)
    err = (yf - ref).abs().max().item()
    err16 = (_unsplit(y3) - ref).abs().max().item()
    parity_log(test="linear_split", M=M, N=N, K=K, act=act, max_abs_err=err, max_abs_err_hi_lo=err16, ref_std=ref.std().item())
    assert err < 2e-5 * max(1.0, ref.abs().max().item()), err          # ~fp32 (plain fp16 operands give 1e-3 here)
    assert err16 < 4e-5 * max(1.0, ref.abs().max().item()), err16


def test_layernorm_split_output(parity_log):
    L = support.lib()
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(6)
    M, N = 333, 768
    y, r = torch.randn(M, N, generator=g, device="cuda"), torch.randn(M, N, generator=g, device="cuda")
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g, device="cuda"), 0.1 * torch.randn(N, generator=g, device="cuda")
    of = torch.empty(M, N, device="cuda")
    o3 = torch.zeros(M, 3 * N, dtype=torch.float16, device="cuda")
    L.check(lib.vb200_layernorm_split(_ptr(y), N, _ptr(r), N, _ptr(gamma), _ptr(beta), 1e-12, _ptr(of), N, _ptr(o3), 3 * N, M, N,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)), None)
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm((y + r).double(), (N,), gamma.double(), beta.double(), 1e-12).float()
    assert (of - ref).abs().max().item() < 1e-5
    err = (_unsplit(o3) - of).abs().max().item()
    parity_log(test="layernorm_split", max_abs_err_hi_lo=err)
    assert err < 1e-6


@pytest.mark.parametrize("in_kind", [0, 1, 2])
@pytest.mark.parametrize("B,Lq,Lk,heads,d", [(3, 31, 36, 8, 128), (2, 36, 31, 8, 128), (2, 31, 31, 12, 64), (1, 101, 38, 2, 128),
                                             (2, 5, 200, 3, 64)])
def test_attention_f32(B, Lq, Lk, heads, d, in_kind, parity_log):
    """fp32 CUDA-core attention: context in every output format + the probability output, against fp64 torch math."""
    L = support.lib()
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(7)
    hid = heads * d
    dt = [torch.float32, torch.float16, torch.bfloat16][in_kind]
    q = torch.randn(B * Lq, hid, generator=g, device="cuda").to(dt)
    kv = torch.randn(B * Lk, 2 * hid, generator=g, device="cuda").to(dt)
    mask = torch.zeros(B, Lk, device="cuda")
    mask[:, -2:] = -10000.0
    probs = torch.full((B, heads, Lq, Lk), float("nan"), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    kp = C.c_void_p(kv.data_ptr())
    vp = C.c_void_p(kv.data_ptr() + hid * kv.element_size())
    qd = q.double().view(B, Lq, heads, d).permute(0, 2, 1, 3)
    kd = kv[:, :hid].double().view(B, Lk, heads, d).permute(0, 2, 1, 3)
    vd = kv[:, hid:].double().view(B, Lk, heads, d).permute(0, 2, 1, 3)
    p_ref = torch.softmax(qd @ kd.transpose(-1, -2) / math.sqrt(d) + mask.double()[:, None, None, :], dim=-1)
    c_ref = (p_ref @ vd).permute(0, 2, 1, 3).reshape(B * Lq, hid).float()
    for ctx_mode in (0, 1, 2, 3):
        ctx = None
        if ctx_mode in (1, 2):
            ctx = torch.zeros(B * Lq, hid, dtype=torch.float16 if ctx_mode == 1 else torch.bfloat16, device="cuda")
        elif ctx_mode == 3:
            ctx = torch.zeros(B * Lq, 3 * hid, dtype=torch.float16, device="cuda")
        L.check(lib.vb200_attention_f32(_ptr(q), hid, kp, vp, 2 * hid, in_kind, _ptr(mask), B, Lq, Lk, heads, d, _ptr(ctx),
                                        ctx.stride(0) if ctx is not None else 0, ctx_mode, _ptr(probs), st), None)
        torch.cuda.synchronize()
        perr = (probs - p_ref.float()).abs().max().item()
        assert perr < 2e-6, perr
        if ctx_mode == 3:
            cerr = (_unsplit(ctx) - c_ref).abs().max().item()
            assert cerr < 2e-5, cerr
        elif ctx_mode:
            cerr = (ctx.float() - c_ref).abs().max().item()
            assert cerr < (4e-3 if ctx_mode == 1 else 3e-2), cerr
    parity_log(test="attention_f32", B=B, Lq=Lq, Lk=Lk, heads=heads, d=d, in_kind=in_kind, probs_max_abs_err=perr)


@pytest.mark.parametrize("M,N,K,act", [
    (128, 128, 64, 0),          # one tile, one k-block
    (256, 256, 1024, 0),        # the 2-stage ring wraps eight times
    (200, 384, 768, 1),         # ragged M, GELU
    (1984, 3072, 768, 1),       # text FFN-in at batch 64: 384 tiles, about three per persistent CTA
    (2304, 3072, 1024, 0),      # image QKV: 432 tiles
    (64, 3129, 2048, 0),        # ragged N (per-lane remainder path)
    (15872, 768, 768, 2),       # 744 tiles: CTAs walk several tiles through one deposit area
])
@pytest.mark.parametrize("act_dt", ACT)
@pytest.mark.parametrize("kernel_variant", [2, 3, 4], ids=["cta_pair", "three_ctas_per_sm", "lone_cta_6_stages"])
def test_linear_three_ctas_per_sm(M, N, K, act, act_dt, kernel_variant, parity_log):
    """vb200_linear variants 2, 3 and 4 (ABI names of Blackwell kernel configurations; on sm_90a they select the persistent
    kernel) must give variant 0's bits, and the TMA-store epilogue (16-bit output only, yb3b) the same bits as the register-store
    one (fp32 + 16-bit outputs)."""
    global VARIANT
    x, w, b, _ = _mk(M, N, K, seed=5, act=act_dt)
    ld = (N + 3) // 4 * 4
    try:
        VARIANT = 0
        yb0, yf0 = run_linear(x, w, b, act=act, block_n=128, ld_f32=ld)
        VARIANT = kernel_variant
        yb3, yf3 = run_linear(x, w, b, act=act, block_n=128, ld_f32=ld)
        yb3b, _ = run_linear(x, w, b, act=act, block_n=128, want_f32=False)           # 16-bit only: the TMA-store epilogue
    finally:
        VARIANT = 0
    ref = ref_linear(x, w, b, act=act)
    err = (yf3 - ref).abs().max().item()
    parity_log(test="linear_variant_%d" % kernel_variant, M=M, N=N, K=K, act=act, dtype=str(act_dt), max_abs_err=err)
    assert err < 2e-3
    assert torch.equal(yf0, yf3)
    if yb0 is not None:
        assert torch.equal(yb0, yb3) and torch.equal(yb0, yb3b)


@pytest.mark.parametrize("M,N,K,act", [(31, 768, 768, 0), (36, 3072, 1024, 1), (248, 768, 3072, 0), (288, 1024, 1024, 2), (64, 3129, 2048, 0)])
@pytest.mark.parametrize("act_dt", ACT)
def test_linear_lone_cta_64_wide(M, N, K, act, act_dt, parity_log):
    """What a small forward (batch <= 8) runs: 64-wide tiles (variant 4 selects the persistent kernel).  The tile width does not
    change an element's accumulation order: the same bits as the default 128-wide kernel."""
    global VARIANT
    x, w, b, _ = _mk(M, N, K, seed=6, act=act_dt)
    ld = (N + 3) // 4 * 4
    try:
        VARIANT = 0
        yb0, yf0 = run_linear(x, w, b, act=act, block_n=128, ld_f32=ld)
        VARIANT = 4
        yb4, yf4 = run_linear(x, w, b, act=act, block_n=64, ld_f32=ld)
    finally:
        VARIANT = 0
    err = (yf4 - ref_linear(x, w, b, act=act)).abs().max().item()
    parity_log(test="linear_lone_cta_64_wide", M=M, N=N, K=K, act=act, dtype=str(act_dt), max_abs_err=err)
    assert err < 2e-3
    assert torch.equal(yf0, yf4)
    if yb0 is not None:
        assert torch.equal(yb0, yb4)
