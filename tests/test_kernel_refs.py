"""CPU checks of the references the op-level kernel tests rely on (oracle/kernel_refs.py): exact 16-bit rounding, the fp16 hi / lo
split, the float32 region-pack restatement against worker_api.build_inputs, and the attention rounding floor the GPU bounds rest on."""
import numpy as np
import pytest
import torch

from oracle import kernel_refs as R
from vilbert_b200 import worker_api as W


def _edge_values():
    one = np.float32(1.0)
    ulp_f16, ulp_bf16 = np.float32(2.0 ** -10), np.float32(2.0 ** -7)
    v = [0.0, -0.0, 1.0, -1.0, 65504.0, -65504.0, 65519.0, 65519.996, 65520.0, -65520.0, 65536.0, 1e5, -1e5, 3.0e38, -3.0e38,
         6.1e-5, 5.96e-8, 2.98e-8, 8.9e-8, 1e-40,
         one + ulp_f16 / 2, one + 3 * ulp_f16 / 2, one + ulp_bf16 / 2, one + 3 * ulp_bf16 / 2,   # ties: to the even neighbour
         -(one + ulp_f16 / 2), -(one + 3 * ulp_bf16 / 2), 2049.0, 2051.0, 4097.0, 257.0, 259.0]
    return np.array(v, dtype=np.float32)


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
def test_sat_rn_matches_independent_rounding(f16):
    """sat_rn (torch) == the numpy / integer implementation bit for bit: ties, +-65504, 65520 (the fp16 tie that rounds to inf
    without the clamp), huge values, subnormals, and a million random values over many binades."""
    g = np.random.default_rng(0)
    rnd = (g.standard_normal(1 << 20) * np.exp2(g.integers(-30, 30, 1 << 20))).astype(np.float32)
    x = np.concatenate([_edge_values(), rnd])
    got = R.bits16(R.sat_rn(torch.from_numpy(x), f16)).numpy().view(np.uint16)
    assert np.array_equal(got, R.sat_rn_bits_np(x, f16))


def test_sat_rn_edges():
    t = torch.tensor([65504.0, 65519.0, 65520.0, 1e5, -1e5, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11])
    h = R.sat_rn(t, True).float().tolist()
    assert h == [65504.0, 65504.0, 65504.0, 65504.0, -65504.0, 1.0, 1.0 + 2.0 ** -9]
    assert torch.isinf(torch.tensor([65520.0]).half()).all()          # what a store without the clamp would write
    b = R.sat_rn(torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1e5]), False).float().tolist()
    assert b == [1.0, 1.0 + 2.0 ** -6, 99840.0]


def test_split16_matches_gemm_test_helper():
    """The hi / lo split helper equals the one the fp32-parity GEMM tests build their operands with, and hi + lo carries x to
    2^-22 relative."""
    from test_gpu_ops import _split_act
    g = torch.Generator().manual_seed(3)
    x = torch.randn(37, 256, generator=g) * torch.exp2(torch.randint(-12, 12, (37, 256), generator=g).float())
    x[0, :4] = torch.tensor([7e4, -7e4, 65504.0, 1e-9])
    got = R.split16(x)
    assert torch.equal(R.bits16(got), R.bits16(_split_act(x)))
    far = R.split16(torch.full((1, 64), 1e6)).view(3, 64).float()         # past 2 x 65504 the lo part saturates too
    assert far[0].eq(65504).all() and far[1].eq(65504).all()
    v = got.view(37, 4, 3, 64)
    assert torch.equal(R.bits16(v[:, :, 0]), R.bits16(v[:, :, 2]))
    back = (v[:, :, 0].float() + v[:, :, 1].float()).reshape(37, 256)
    ok = x.abs() <= 65504
    assert ((back - x).abs()[ok] <= x.abs()[ok] * 2.0 ** -21 + 2.0 ** -24).all()


# ---------------------------------------------------------------------------------------------------------------- GELU restatement
def _all_f32(lo, hi):
    """Every fp32 value in [lo, hi] for 0 < lo < hi, ascending."""
    a, b = np.float32(lo).view(np.uint32), np.float32(hi).view(np.uint32)
    return np.arange(a, b + 1, dtype=np.uint32).view(np.float32)


def _all_finite_16(f16):
    """Every finite fp16 or bf16 value, as fp32."""
    u = np.arange(1 << 16, dtype=np.uint32)
    x = u.astype(np.uint16).view(np.float16).astype(np.float32) if f16 else (u << 16).view(np.float32)
    return x[np.isfinite(x)]


def _gelu_err(x):
    return np.abs(R.gelu_poly_f32(x).astype(np.float64) - R.gelu_fp64(torch.from_numpy(x)).numpy())


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
def test_gelu_poly_bound_every_16bit_value(f16):
    """|gelu_erf - GELU| <= 4.3e-5 (common.cuh) on every finite fp16 / bf16 input, and no NaN or inf.  Measured: 4.11e-5 (fp16),
    3.98e-5 (bf16)."""
    x = _all_finite_16(f16)
    assert len(x) == (63488 if f16 else 65280)
    y = R.gelu_poly_f32(x)
    assert np.isfinite(y).all()
    assert _gelu_err(x).max() <= R.GELU_BOUND


def test_gelu_poly_bound_dense_grid():
    """The same bound on a 10^7-point fp32 grid over [-12, 12] and on every fp32 value within 2^-8 of the worst grid point (near
    x = -4.2645; 4.27e-5 there)."""
    x = np.linspace(-12.0, 12.0, 10_000_001, dtype=np.float64).astype(np.float32)
    e = _gelu_err(x)
    worst = x[np.argmax(e)]
    assert e.max() <= R.GELU_BOUND and -4.4 < worst < -4.1, (e.max(), worst)
    near = -_all_f32(-worst - 2.0 ** -8, -worst + 2.0 ** -8)
    assert _gelu_err(near).max() <= R.GELU_BOUND


def test_gelu_poly_saturation_thresholds():
    """Below GELU_ZERO_BELOW the output is -0, above GELU_IDENTITY_ABOVE it is x bit for bit: every fp32 value with 2 <= |x| <= 16,
    then every 256th fp32 bit pattern out to FLT_MAX, every value around sqrt(FLT_MAX) (where x * x overflows) and FLT_MAX itself.
    Both thresholds are tight: the thresholds themselves give neither."""
    zb, ia = np.float32(R.GELU_ZERO_BELOW), np.float32(R.GELU_IDENTITY_ABOVE)
    dense = _all_f32(2.0, 16.0)
    a16 = np.float32(16.0).view(np.uint32)
    fmax = np.finfo(np.float32).max
    sparse = np.arange(a16, fmax.view(np.uint32), 256, dtype=np.uint32).view(np.float32)
    r = np.float32(np.sqrt(fmax)).view(np.uint32)
    overflow = np.arange(r - (1 << 14), r + (1 << 14), dtype=np.uint32).view(np.float32)
    pos = np.concatenate([dense, sparse, overflow, np.array([fmax], dtype=np.float32)])
    yp = R.gelu_poly_f32(pos)
    yn = R.gelu_poly_f32(-pos)
    assert np.isfinite(yp).all() and np.isfinite(yn).all()
    above = pos > ia
    assert np.array_equal(yp[above].view(np.uint32), pos[above].view(np.uint32))
    below = -pos < zb
    assert (yn[below] == 0).all() and np.signbit(yn[below]).all()
    y_zb, y_ia = R.gelu_poly_f32(np.array([zb, ia], dtype=np.float32))
    assert y_zb != 0 and y_ia != ia


def test_gelu_poly_small_inputs():
    """Zero gives +0, and small inputs follow x / 2 + x^2 / sqrt(2 pi) (the bound is absolute, so check the relative error too)."""
    x = np.array([0.0, -0.0, 1e-30, -1e-30, 1e-6, -1e-6, 1e-3], dtype=np.float32)
    y = R.gelu_poly_f32(x)
    assert y[0] == 0 and y[1] == 0
    ref = R.gelu_fp64(torch.from_numpy(x)).numpy()
    assert (np.abs(y[2:] - ref[2:]) <= np.abs(ref[2:]) * 1e-3).all()


# ---------------------------------------------------------------------------------------------------------------- exact GEMM operands
EXACT_SHAPES = [(1, 64, 64), (129, 1000, 200), (64, 3129, 2048), (300, 1601, 3072), (77, 64, 2112)]


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
@pytest.mark.parametrize("M,N,K", EXACT_SHAPES)
def test_exact_operands(M, N, K, f16):
    """The builder's operands are exact in the 16-bit format, every element stays inside the 2^24-unit budget (quarter-unit biases:
    sum |x w| + |b| < 2^22) and the largest reaches within a factor four of it; biases have 12 or 13 significant bits (exact in
    neither 16-bit format) and some are +-70000; columns of x past K are NaN."""
    ld_x = K + 8
    x, w, b = R.exact_operands(M, N, K, ld_x, f16, seed=M + N + K)
    dt = torch.float16 if f16 else torch.bfloat16
    assert x.dtype == dt and w.dtype == dt and x.shape == (M, ld_x) and w.shape == (N, K) and b.shape == (N,)
    assert torch.isnan(x[:, K:].float()).all() and not torch.isnan(x[:, :K].float()).any()
    s = R.exact_bound(x[:, :K], w, b)
    assert s.max().item() < 2.0 ** 22
    sxw = R.exact_bound(x[:, :K], w, None)
    assert 2.0 ** 20 <= sxw.max().item() < 2.0 ** 23
    if M >= 8:                                                  # amplitudes fall by 4x per row: many binades
        assert sxw.max().item() / sxw.min().item() > 2.0 ** 8
    assert ((b.double() * 4).remainder(2) == 1).sum().item() >= N - 2 * ((N + 95) // 97)    # odd quarters
    small = b.abs() < 70000
    assert not torch.equal(b[small].half().float(), b[small]) and not torch.equal(b[small].bfloat16().float(), b[small])
    if N > 2:
        assert (b == 70000).any() and (b == -70000).any()


@pytest.mark.parametrize("M,N,K", EXACT_SHAPES[:3])
def test_exact_linear_is_order_independent(M, N, K):
    """exact_linear equals fp32 accumulation in three different orders (forwards, backwards, pairwise by torch's fp32 matmul), bit
    for bit: the point of the exact-valued operands."""
    x, w, b = R.exact_operands(M, N, K, None, True, seed=7)
    ref = R.exact_linear(x, w, b, 0)
    xf, wf = x.float(), w.float()
    assert torch.equal((xf @ wf.t()) + b, ref)
    fwd = torch.zeros(M, N)
    bwd = torch.zeros(M, N)
    for k in range(K):
        fwd += xf[:, k:k + 1] * wf[:, k][None]
        bwd += xf[:, K - 1 - k:K - k] * wf[:, K - 1 - k][None]
    assert torch.equal(fwd + b, ref) and torch.equal(bwd + b, ref)
    assert torch.equal(R.exact_linear(x, w, b, 2), torch.relu(ref))
    mul = torch.exp2(torch.randint(-3, 4, (M, N)).float())
    assert torch.equal(R.exact_linear(x, w, b, 0, mul), ref * mul)


def test_exact_linear_catches_narrow_accumulators():
    """A 16-bit bias, or an accumulator rounded to tf32 (10 explicit mantissa bits) before the bias add, changes the result: the
    operands are built so that the exact tests see such defects."""
    x, w, b = R.exact_operands(256, 512, 768, None, False, seed=3)
    ref = R.exact_linear(x, w, b, 0)
    acc = x.double() @ w.double().t()
    assert not torch.equal((acc + b.half().double()).float(), ref)
    assert not torch.equal((acc + b.bfloat16().double()).float(), ref)
    m, e = torch.frexp(acc)
    tf32 = torch.ldexp(torch.round(m * 2 ** 11) / 2 ** 11, e)
    assert not torch.equal((tf32 + b.double()).float(), ref)


def test_split16_w_layout():
    """The weight split is hi | hi | lo per 64 columns and hi + lo carries w to 2^-22 relative."""
    g = torch.Generator().manual_seed(4)
    w = torch.randn(5, 128, generator=g)
    v = R.split16_w(w).view(5, 2, 3, 64).float()
    assert torch.equal(v[:, :, 0], v[:, :, 1])
    back = (v[:, :, 0] + v[:, :, 2]).reshape(5, 128)
    assert ((back - w).abs() <= w.abs() * 2.0 ** -21 + 2.0 ** -24).all()


class _Tok:
    def encode(self, s):
        return [5, 6, 7]

    def add_special_tokens_single_sentence(self, ids):
        return [2] + ids + [3]


@pytest.mark.parametrize("n,F", [(7, 2048), (36, 2048), (1, 64), (100, 40)])
def test_region_restatement_matches_build_inputs(n, F):
    """The float32 region-pack restatement against the host input builder: box rows and spatials bit for bit; the mean row (torch.sum
    adds in its own order) within one unit in the last place of the 16-bit formats."""
    g = np.random.default_rng(n * F)
    feats = (g.random((n, F), dtype=np.float32) * g.choice([0.01, 1.0, 300.0], size=(n, F))).astype(np.float32)
    x1 = g.integers(0, 300, n).astype(np.float32)
    y1 = g.integers(0, 200, n).astype(np.float32)
    boxes = np.stack([x1, y1, x1 + g.integers(1, 300, n), y1 + g.integers(1, 250, n)], axis=1).astype(np.float32)
    w, h = 640.0, 427.0
    info = {"image_width": w, "image_height": h, "bbox": boxes}
    _, f, s, *_ = W.build_inputs("q", [1], [torch.from_numpy(feats)], [info], torch.device("cpu"), _Tok())
    rows, loc, real = R.region_rows(feats, boxes, w, h, n)
    assert real.all()
    assert np.array_equal(rows[1:], f[0, 1:].numpy())
    assert np.array_equal(loc.view(np.uint32), s[0].numpy().view(np.uint32))
    mean_bi = f[0, 0].numpy()
    for f16 in (True, False):
        ulp = np.float32(2.0 ** (-10 if f16 else -7)) * np.exp2(np.floor(np.log2(np.maximum(np.abs(rows[0]), 2.0 ** -14))))
        assert (np.abs(rows[0] - mean_bi) <= ulp).all()


def test_region_restatement_padding():
    """nb < n: the mean over the valid boxes only, zero rows and zero locations for the padded ones; nb = 0: a zero mean row."""
    g = np.random.default_rng(1)
    feats = g.random((6, 16), dtype=np.float32)
    boxes = np.tile(np.array([[1, 2, 30, 40]], dtype=np.float32), (6, 1))
    rows, loc, real = R.region_rows(feats, boxes, 100.0, 50.0, 3)
    assert np.array_equal(rows[0], ((feats[0] + feats[1]) + feats[2]) / np.float32(3))
    assert not rows[4:].any() and not loc[4:].any() and real.tolist() == [True] * 4 + [False] * 3
    rows, loc, real = R.region_rows(feats, boxes, 100.0, 50.0, 0)
    assert not rows.any() and loc[0].tolist() == [0, 0, 1, 1, 1] and real.tolist() == [True] + [False] * 6


@pytest.mark.parametrize("L,d", [(16, 64), (17, 128), (31, 64), (65, 128), (129, 128), (256, 64)])
def test_attention_rounding_floor(L, d):
    """The CPU emulation of the tensor-core attention's rounding points (16-bit P before P V, 16-bit context) against fp64, at inputs
    like the GPU tests' (N(0, 1) Q / K / V in the 16-bit format, per-sample masks with interior masked keys), as the error over
    max(1, |reference|).  Measured at these shapes: at most 4.4e-3 (bf16) and 6.2e-4 (fp16).  The GPU attention tests bound the
    kernels at 1.2e-2 and 1.5e-3 of the same measure, about twice this floor."""
    heads = 2
    H = heads * d
    g = torch.Generator().manual_seed(L + d)
    for f16, bound in ((False, 1.2e-2), (True, 1.5e-3)):
        dt = torch.float16 if f16 else torch.bfloat16
        qkv = torch.randn(2, L, 3 * H, generator=g).to(dt)
        mask = torch.zeros(2, L)
        mask[0, 1:L:3] = -10000.0
        mask[1, L // 2 + 1:] = -10000.0
        q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
        ref = R.attention_fp64(q, k, v, mask, heads)
        err = ((R.attention_emulated(q, k, v, mask, heads, f16) - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
        assert err < bound / 2, (f16, err)


def _edge_masks(L):
    return torch.stack([R.edge_mask(p, L) for p in R.EDGE_MASKS])


def test_attention_probs_fp64_matches_softmax():
    """attention_probs_fp64 against an independent fp64 restatement (per-head scores, torch.softmax, P V as a sum over keys), at every
    edge mask: probabilities and context to fp64 rounding, rows summing to 1, and attention_fp64 returning the same context."""
    heads, d, Lq, Lk = 2, 64, 5, 130
    H = heads * d
    g = torch.Generator().manual_seed(11)
    mask = _edge_masks(Lk)
    B = mask.shape[0]
    q, k, v = (torch.randn(B, n, H, generator=g, dtype=torch.float64) for n in (Lq, Lk, Lk))
    p, ctx = R.attention_probs_fp64(q, k, v, mask, heads)
    assert p.shape == (B, heads, Lq, Lk) and ctx.shape == (B, Lq, H) and p.dtype == ctx.dtype == torch.float64
    for h in range(heads):
        c = slice(h * d, (h + 1) * d)
        s = torch.einsum("bid,bjd->bij", q[..., c], k[..., c]) / d ** 0.5 + mask.double()[:, None, :]
        ph = torch.softmax(s, dim=-1)
        assert torch.allclose(p[:, h], ph, rtol=0, atol=1e-15)
        assert torch.allclose(ctx[..., c], (ph[..., None] * v[:, None, :, c]).sum(2), rtol=0, atol=1e-13)
    assert torch.allclose(p.sum(-1), torch.ones(B, heads, Lq, dtype=torch.float64), rtol=0, atol=1e-14)
    assert torch.equal(R.attention_fp64(q, k, v, mask, heads), ctx)


def test_edge_masks():
    """The edge mask builder: one real key where the pattern puts it (clamped to the length), masks exactly 0 or -10000, and the
    straddle pattern masking the two keys around every multiple of 16."""
    for L in (1, 2, 16, 17, 64, 65, 129, 512):
        m = _edge_masks(L)
        assert ((m == 0) | (m == R.MASKED)).all()
        for p, row in zip(R.EDGE_MASKS, m):
            if p.startswith("single@"):
                at = p.split("@")[1]
                assert R.single_real_key(row) == (L - 1 if at == "last" else min(int(at), L - 1)), (p, L)
        assert (m[R.EDGE_MASKS.index("all_masked")] == R.MASKED).all() and (m[R.EDGE_MASKS.index("all_real")] == 0).all()
    s = R.edge_mask("straddle", 70)
    assert (s == R.MASKED).nonzero().flatten().tolist() == [15, 16, 31, 32, 47, 48, 63, 64]
    assert (R.edge_mask("real_below@17", 40) == 0).nonzero().flatten().tolist() == list(range(17))


def test_fully_masked_row_is_unmasked_softmax():
    """Every key masked: softmax(s - 10000) is softmax(s), so the fp64 reference of a fully masked sample is its unmasked one."""
    heads, d, L = 2, 64, 67
    H = heads * d
    g = torch.Generator().manual_seed(12)
    q, k, v = (torch.randn(1, L, H, generator=g) * 2 for _ in range(3))
    pm, cm = R.attention_probs_fp64(q, k, v, R.edge_mask("all_masked", L)[None], heads)
    pr, cr = R.attention_probs_fp64(q, k, v, R.edge_mask("all_real", L)[None], heads)
    assert torch.allclose(pm, pr, rtol=1e-10, atol=0) and torch.allclose(cm, cr, rtol=0, atol=1e-10)


@pytest.mark.parametrize("L,d", [(1, 64), (2, 128), (15, 64), (17, 128), (33, 64), (63, 128), (64, 64)])
def test_attention_rounding_floor_edge_masks(L, d):
    """test_attention_rounding_floor at every edge mask (one sample per pattern): the emulated rounding points stay within half the
    GPU attention bound of fp64, once the fully masked samples are allowed the rounding of their masked scores
    (masked_score_slack).  Without that allowance they exceed it (7.9e-4 at L = 2, fp16), so the slack is needed, and it is no
    licence for the others: the samples with a real key stay within half the bound on their own."""
    heads = 2
    H = heads * d
    g = torch.Generator().manual_seed(L * 3 + d)
    mask = _edge_masks(L)
    B = mask.shape[0]
    for f16, bound in ((False, 1.2e-2), (True, 1.5e-3)):
        dt = torch.float16 if f16 else torch.bfloat16
        qkv = torch.randn(B, L, 3 * H, generator=g).to(dt)
        q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
        p, ref = R.attention_probs_fp64(q, k, v, mask, heads)
        slack = R.masked_score_slack(p, mask == R.MASKED, v, ref, heads, R.MASKED_SCORE_ERR["tc"])
        assert not slack[~(mask == R.MASKED).all(1)].any()
        err = (R.attention_emulated(q, k, v, mask, heads, f16) - ref).abs()
        assert (err <= bound / 2 * ref.abs().clamp(min=1.0) + slack).all(), (f16, (err - slack).max().item())


@pytest.mark.parametrize("d", [64, 128])
def test_grid_qk_scores_exact(d):
    """The fp32 attention test's Q / K grid: fp32 scores accumulated key by key in the kernel's order (one fmaf per element) and in
    reverse equal the fp64 ones, at the largest Q amplitude and at the all-extreme corner; the values survive fp16 and bf16."""
    g = torch.Generator().manual_seed(d)
    q, k = R.grid_qk(64, d, 8.0, g), R.grid_qk(256, d, 1.0, g)
    q[0], k[0] = 8.0, -1.0
    exact = q.double() @ k.double().t()
    fwd, bwd = torch.zeros(64, 256), torch.zeros(64, 256)
    for i in range(d):
        fwd = torch.addcmul(fwd, q[:, i:i + 1], k[:, i][None])
        bwd = torch.addcmul(bwd, q[:, d - 1 - i:d - i], k[:, d - 1 - i][None])
    assert torch.equal(fwd.double(), exact) and torch.equal(bwd.double(), exact)
    assert exact[0, 0].item() == -8.0 * d
    for dt in (torch.float16, torch.bfloat16):
        assert torch.equal(q.to(dt).float(), q) and torch.equal(k.to(dt).float(), k)
