"""Plain references for the op-level kernel tests (tests/test_gpu_kernel_parity.py): the exact 16-bit conversions the kernels apply,
the fp16 hi / lo split of the fp32-parity mode, a float32 restatement of the detector-output input builder in the region-pack
kernel's order, fp64 attention with its probabilities, key masks at the attention kernels' block edges, and an emulation of the
tensor-core attention's rounding points.  CPU only; checked by tests/test_kernel_refs.py."""
from __future__ import annotations

import math

import numpy as np
import torch

F16_MAX = 65504.0


# ---------------------------------------------------------------------------------------------------------------- 16-bit rounding
def sat_rn(x: torch.Tensor, f16: bool) -> torch.Tensor:
    """The 16-bit value every saturating kernel store writes for the fp32 value x (common.cuh pack16x2_rt): fp16 clamps to +-65504
    and then rounds to nearest even; bf16 rounds to nearest even."""
    x = x.float()
    if f16:
        return x.clamp(-F16_MAX, F16_MAX).to(torch.float16)
    return x.to(torch.bfloat16)


def sat_rn_bits_np(x: np.ndarray, f16: bool) -> np.ndarray:
    """sat_rn as raw uint16 bits, computed without torch (numpy's fp16 cast; bf16 by integer round-to-nearest-even on the fp32
    bits), so the torch helper above can be checked against an independent implementation.  Finite inputs only."""
    x = np.asarray(x, dtype=np.float32)
    if f16:
        return np.clip(x, -F16_MAX, F16_MAX).astype(np.float16).view(np.uint16)
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bits16(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16)


def split16(x: torch.Tensor) -> torch.Tensor:
    """fp32 [M, K] (K % 64 == 0) -> the fp32-parity operand, fp16 [M, 3K]: per 64 columns hi | lo | hi with hi = sat_rn_fp16(x),
    lo = sat_rn_fp16(x - hi) (common.cuh split_col / split_lo; lo goes through the same saturating store as hi, which only matters
    past 2 x 65504, where x - hi itself leaves the fp16 range)."""
    x = x.float()
    hi = sat_rn(x, True)
    lo = sat_rn(x - hi.float(), True)
    M, K = x.shape
    g = K // 64
    return torch.stack([hi.view(M, g, 64), lo.view(M, g, 64), hi.view(M, g, 64)], dim=2).reshape(M, 3 * K).contiguous()


def split16_w(w: torch.Tensor) -> torch.Tensor:
    """fp32 [N, K] (K % 64 == 0) -> the fp32-parity weight, fp16 [N, 3K]: per 64 columns hi | hi | lo (engine.cu put_split_w), so
    that against the activation's hi | lo | hi the K' = 3K contraction adds hi.hi + lo.hi + hi.lo."""
    w = w.float()
    hi = sat_rn(w, True)
    lo = sat_rn(w - hi.float(), True)
    N, K = w.shape
    g = K // 64
    return torch.stack([hi.view(N, g, 64), hi.view(N, g, 64), lo.view(N, g, 64)], dim=2).reshape(N, 3 * K).contiguous()


# ---------------------------------------------------------------------------------------------------------------- GELU epilogues
# gelu_erf (common.cuh): x * sat(0.5 + x Q(x^2)), Q of degree 8 in x^2, evaluated in Horner order with one fp32 FMA per step.
GELU_Q = (4.547042257e-11, -4.515281038e-09, 1.986152114e-07, -5.147503089e-06, 8.848903963e-05, -1.079077483e-03, 9.718777612e-03,
          -6.619028002e-02, 3.988192081e-01)
GELU_BOUND = 4.3e-5             # the documented |gelu_erf - GELU| bound over the whole fp32 range
# Saturation thresholds of gelu_erf (checked by tests/test_kernel_refs.py on every fp32 value with 2 <= |x| <= 16 and a sample out to
# FLT_MAX): for x < GELU_ZERO_BELOW the output is -0 (x * 0), for x > GELU_IDENTITY_ABOVE it is x itself.  Each is the last input on
# its side whose output is neither (gelu(-4.2741566) = -1.44e-6).
GELU_ZERO_BELOW = float(np.float32(-4.2741566))
GELU_IDENTITY_ABOVE = float(np.float32(4.2741566))


def _fma32(a: np.ndarray, b: np.ndarray, c) -> np.ndarray:
    """fp32 fmaf(a, b, c): the product of two fp32 values is exact in fp64, the sum is rounded to fp64 and then to fp32 (a double
    rounding that can differ from the single one of the hardware FMA in rare ties)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return (a.astype(np.float64) * b.astype(np.float64) + np.float64(c)).astype(np.float32)


def gelu_poly_f32(x) -> np.ndarray:
    """gelu_erf restated in numpy float32: u = x * x rounded to fp32, Q in the kernel's Horner order with one emulated FMA per step,
    the FMA's saturation to [0, 1] (NaN -> 0, as __saturatef), then x * Phi rounded to fp32."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        u = (x * x).astype(np.float32)
        q = np.full(x.shape, np.float32(GELU_Q[0]), dtype=np.float32)
        for c in GELU_Q[1:]:
            q = _fma32(q, u, np.float32(c))
        t = _fma32(x, q, np.float32(0.5))
        t = np.clip(np.nan_to_num(t, nan=0.0, posinf=1.0, neginf=0.0), 0.0, 1.0).astype(np.float32)
        return (x * t).astype(np.float32)


def gelu_fp64(x) -> torch.Tensor:
    """GELU, erf form, in fp64 (torch.erf): the function gelu_erf and the act-3 GELU approximate."""
    x = torch.as_tensor(x).double()
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_as_fp64(x) -> torch.Tensor:
    """The act-3 GELU's formula (common.cuh gelu_erf_as: Abramowitz & Stegun 7.1.26 erf) evaluated in fp64: what the fp32 kernel
    computes, without its fp32 rounding, __fdividef and exp2f."""
    x = torch.as_tensor(x).double()
    z = x / math.sqrt(2.0)
    ax = z.abs()
    t = 1.0 / (1.0 + 0.3275911 * ax)
    p = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t
    return x * 0.5 * (1.0 + torch.copysign(1.0 - p * torch.exp(-ax * ax), z))


# ---------------------------------------------------------------------------------------------------------------- exact GEMMs
# Integer-valued operands whose fp32 result does not depend on the order of accumulation: every product is an integer, and the sum of
# the |products| plus |bias| of each output element stays below 2^24 in units of the smallest power of two anywhere in it (the bias
# has quarter units, so the budget is 2^22).  Every partial sum in any order is then an exactly representable fp32 value, and the
# correct fp32 output equals the fp64 one.  The budget is a parameter (`scale`) so that it can be lowered if a tensor core turns out
# to align its addends more narrowly; H100 wgmma (fp16 and bf16 operands, fp32 accumulation) is exact at the full budget
# (tests/test_gpu_gemm_exact.py test_exact_accumulation_at_full_budget).
EXACT_BUDGET_LOG2 = 22          # 2^24 in quarter units
BIAS_UNIT = 0.25
W_MAX = 15                      # weights: integers in [-15, 15]
X_MANT = 255                    # activations: integers in [-255, 255] times a power of two (8 significant bits: exact in bf16)
BIG_BIAS = 70000.0              # a few columns: fp16 outputs saturate


def exact_bound(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None) -> torch.Tensor:
    """Per output element: sum_k |x_k w_k| + |b| (fp64; exact for these integers)."""
    s = x.double().abs() @ w.double().abs().t()
    if b is not None:
        s = s + b.double().abs()
    return s


def exact_operands(M: int, N: int, K: int, ld_x: int | None = None, f16: bool = True, seed: int = 0, scale: int = EXACT_BUDGET_LOG2,
                   device="cpu"):
    """(x [M, ld_x] 16-bit, w [N, K] 16-bit, b [N] fp32) of an exact-valued GEMM (see above) with sum |x w| + |b| < 2^scale.

    Row 0 of x and row 0 of w are constant, so element (0, 0) accumulates monotonically to within a factor two of the budget; the
    other rows take amplitudes from the full budget down by powers of four, so the outputs span many binades.  Biases are odd
    multiples of 1/4 of 12 or 13 significant bits (exact in neither 16-bit format); every 97th column gets +-70000 instead.  Columns of
    x past K are NaN: a kernel that reads them writes NaN."""
    assert scale <= EXACT_BUDGET_LOG2
    ld_x = ld_x or K
    dt = torch.float16 if f16 else torch.bfloat16
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(seed)
    f64 = dict(dtype=torch.float64, device=dev)
    budget = 2.0 ** scale - BIG_BIAS - 1.0
    a_max = budget / (K * W_MAX)                                   # largest |x| that keeps every element inside the budget
    assert a_max >= 1.0, (K, scale)
    w = torch.randint(-W_MAX, W_MAX + 1, (N, K), generator=g, device=dev).double()
    w[0] = W_MAX
    amp = (a_max / 4.0 ** (torch.arange(M, device=dev) % 8).double()).clamp(min=1.0)
    shift = torch.clamp(torch.ceil(torch.log2(amp / X_MANT)), min=0.0)     # amp = mant * 2^shift, mant <= 255
    mant = torch.floor(amp / torch.exp2(shift))
    x = (torch.rand(M, K, generator=g, **f64) * 2.0 - 1.0) * mant[:, None]
    x = torch.round(x) * torch.exp2(shift)[:, None]
    x[0] = mant[0] * torch.exp2(shift[0])
    b = (torch.randint(2048, 4096, (N,), generator=g, device=dev) * 2 + 1).double() * BIAS_UNIT
    b = b * (torch.randint(0, 2, (N,), generator=g, device=dev) * 2 - 1)
    b[1::97] = BIG_BIAS
    b[2::97] = -BIG_BIAS
    b = b.float()
    assert torch.equal(x.to(dt).double(), x) and torch.equal(w.to(dt).double(), w)
    s = exact_bound(x, w, b)
    assert s.max().item() < 2.0 ** scale, s.max().item()
    if scale >= 12:
        assert s.max().item() >= 2.0 ** (scale - 2)
    xp = torch.full((M, ld_x), float("nan"), **f64)
    xp[:, :K] = x
    return xp.to(dt), w.to(dt), b


def exact_linear(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, act: int, mul: torch.Tensor | None = None) -> torch.Tensor:
    """fp32 result of act(x w^T + b) (* mul) for exact-valued operands: fp64 (exact on these integers, on the device too) converted to
    fp32 without rounding; act 0 or 2 (ReLU of an exact value is exact); mul (fp32 [M, N]) multiplies in fp32, the kernel's one
    rounding."""
    assert act in (0, 2)
    K = w.shape[1]
    y = x[:, :K].double() @ w.double().t()
    if b is not None:
        y = y + b.double()
    if act == 2:
        y = torch.relu(y)
    y32 = y.float()
    assert torch.equal(y32.double(), y), "the operands are not exact-valued"
    return y32 * mul.float() if mul is not None else y32


# ---------------------------------------------------------------------------------------------------------------- region pack
def region_rows(box_feats: np.ndarray, boxes: np.ndarray, w: float, h: float, nb: int):
    """One image of the region-pack kernel in float32, in the kernel's order of operations (worker.py:422-455 restated):
    box_feats [n, F], boxes [n, 4] pixel x1 y1 x2 y2, nb <= n valid boxes.  Returns (operand rows [n + 1, F] fp32, locations
    [n + 1, 5] fp32, real-row flags [n + 1]).  Row 0 is the mean of the valid boxes -- a sequential fp32 sum divided by max(nb, 1),
    so nb = 0 gives a zero row --, padded boxes are zero rows; the area (y2 - y1)(x2 - x1) / float(w h) is taken before the
    coordinates are divided by w and h."""
    box_feats = np.asarray(box_feats, dtype=np.float32)
    boxes = np.asarray(boxes, dtype=np.float32)
    n, F = box_feats.shape
    rows = np.zeros((n + 1, F), dtype=np.float32)
    s = np.zeros(F, dtype=np.float32)
    for r in range(nb):
        s = s + box_feats[r]                                     # float32 + float32, one box at a time
    rows[0] = s / np.float32(max(nb, 1))
    rows[1:nb + 1] = box_feats[:nb]
    w32, h32 = np.float32(w), np.float32(h)
    wh = np.float32(float(w32) * float(h32))
    loc = np.zeros((n + 1, 5), dtype=np.float32)
    loc[0] = [0, 0, 1, 1, 1]
    b = boxes[:nb]
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    loc[1:nb + 1, 4] = (y2 - y1) * (x2 - x1) / wh
    loc[1:nb + 1, 0] = x1 / w32
    loc[1:nb + 1, 1] = y1 / h32
    loc[1:nb + 1, 2] = x2 / w32
    loc[1:nb + 1, 3] = y2 / h32
    real = np.zeros(n + 1, dtype=bool)
    real[:nb + 1] = True
    return rows, loc, real


def operand_rows(feat: np.ndarray, loc: np.ndarray, Kp: int) -> np.ndarray:
    """[feat | loc | 0 ...] rows, Kp wide, fp32 (the image operand before its 16-bit conversion)."""
    R, F = feat.shape
    out = np.zeros((R, Kp), dtype=np.float32)
    out[:, :F] = feat
    out[:, F:F + 5] = loc
    return out


# ---------------------------------------------------------------------------------------------------------------- attention
def attention_probs_fp64(q, k, v, mask_add, heads):
    """softmax(Q K^T / sqrt(d) + mask) and its product with V, in fp64; q [B, Lq, H], k / v [B, Lk, H], mask_add [B, Lk] ->
    (probabilities [B, heads, Lq, Lk], context [B, Lq, H])."""
    B, Lq, H = q.shape
    Lk = k.shape[1]
    d = H // heads
    qh = q.double().reshape(B, Lq, heads, d).permute(0, 2, 1, 3)
    kh = k.double().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    vh = v.double().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(d) + mask_add.double()[:, None, None, :]
    p = torch.softmax(s, dim=-1)
    return p, (p @ vh).permute(0, 2, 1, 3).reshape(B, Lq, H)


def attention_fp64(q, k, v, mask_add, heads):
    """softmax(Q K^T / sqrt(d) + mask) V in fp64; q [B, Lq, H], k / v [B, Lk, H], mask_add [B, Lk] -> [B, Lq, H] fp64."""
    return attention_probs_fp64(q, k, v, mask_add, heads)[1]


# Key masks at the places the attention kernels skip or predicate work (tests/test_gpu_attention_edges.py): the 64-key blocks of the
# online softmax, the 16-key padding of the staged tiles, the 32-key chunks of the fp32 kernel, the key pairs of one mma column.
# A pattern is "kind" or "kind@position"; positions past the sample's length clamp to it.
MASKED = -10000.0               # the additive mask of a masked key (BERT's extended attention mask)
EDGE_MASKS = ("all_real", "key0_masked",
              "single@0", "single@last", "single@63", "single@64", "single@65",       # one real key
              "masked_below@63", "masked_below@64", "masked_below@65",                # first block masked, later keys real
              "masked_block@64", "masked_block@192",                                  # one middle block masked
              "straddle",                                                             # keys n - 1 and n masked at every n = 16 i
              "real_below@15", "real_below@17", "real_below@31", "real_below@33",     # real prefix ending one key either side of a
              "real_below@63", "real_below@65", "real_below@127", "real_below@129",   # 16 / 32 / 64 boundary
              "all_masked")


def edge_mask(pattern: str, L: int) -> torch.Tensor:
    """The additive key mask [L] (fp32, 0 or MASKED) of one EDGE_MASKS pattern."""
    kind, _, at = pattern.partition("@")
    m = torch.zeros(L)
    if kind == "all_real":
        pass
    elif kind == "all_masked":
        m[:] = MASKED
    elif kind == "key0_masked":
        m[0] = MASKED
    elif kind == "single":
        m[:] = MASKED
        m[L - 1 if at == "last" else min(int(at), L - 1)] = 0.0
    elif kind == "masked_below":
        m[:int(at)] = MASKED
    elif kind == "masked_block":
        m[int(at):int(at) + 64] = MASKED
    elif kind == "straddle":
        for n in range(16, L, 16):
            m[n - 1:n + 1] = MASKED
    elif kind == "real_below":
        m[int(at):] = MASKED
    else:
        raise ValueError(pattern)
    return m


# A masked score is s - 10000 (fp32 kernel, natural log) or s log2(e) - 14427 (tensor-core kernels, log2 domain), rounded to fp32
# where the ulp is 2^-10: each masked key's exponent carries up to 2^-11 of error.  Only rows with no real key give masked keys any
# weight; there that error is real (an fp32 PyTorch forward has it too) and comes on top of each kernel's rounding floor.
MASKED_SCORE_ERR = {"f32": 2.0 ** -11, "tc": 2.0 ** -11 * math.log(2.0)}     # natural-log units


def masked_score_slack(p, masked, v, ctx, heads, err):
    """Context error allowed for the rounding of masked scores, per element [B, Lq, H]: each weight p_j of a masked key is off by a
    factor exp(delta_j), |delta_j| <= err, so to first order the context moves by sum_j p_j (delta_j - mean delta) (v_j - c), at most
    2 err sum_j p_j |v_j - c| <= 2 err sqrt(sum_j p_j (v_j - c)^2) (Cauchy-Schwarz, sum_j p_j <= 1), summed over masked keys.  p: fp64
    probabilities [B, heads, Lq, Lk]; masked [B, Lk] bool; v [B, Lk, H]; ctx: the fp64 context [B, Lq, H].  Zero for rows with a
    real key (their masked weights underflow to 0 in fp64)."""
    B, Lq, H = ctx.shape
    Lk = v.shape[1]
    d = H // heads
    pm = p * masked.double()[:, None, None, :]
    vh = v.double().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    ch = ctx.double().reshape(B, Lq, heads, d).permute(0, 2, 1, 3)
    var = pm @ (vh * vh) - 2.0 * ch * (pm @ vh) + ch * ch * pm.sum(-1, keepdim=True)
    return (2.0 * err * var.clamp(min=0.0).sqrt()).permute(0, 2, 1, 3).reshape(B, Lq, H)


def single_real_key(mask: torch.Tensor) -> int | None:
    """The index of the only real key of a mask [L], or None when it has none or several."""
    real = (mask == 0).nonzero().flatten()
    return int(real[0]) if real.numel() == 1 else None


def grid_qk(rows: int, cols: int, amp: float, generator: torch.Generator) -> torch.Tensor:
    """[rows, cols] fp32 multiples of 1/4 in [-amp, amp], amp <= 8: Q elements at amp <= 8, K elements at amp = 1.  Each product q k
    is then a multiple of 2^-4 of magnitude <= 8, and every partial sum of a head's dot product (d <= 128) stays below 2^10 = 2^14
    units, so a score q . k is exact in fp32 in any order of accumulation; the values themselves are exact in fp16 and bf16 (at most
    6 significant bits).  Scores have a standard deviation of about amp / 3."""
    assert amp <= 8.0
    n = int(amp * 4)
    return torch.randint(-n, n + 1, (rows, cols), generator=generator, device=generator.device).float() / 4.0


def attention_emulated(q, k, v, mask_add, heads, f16: bool):
    """The tensor-core attention's rounding points on the CPU: fp32 scores s = fmaf(q.k, kLog2e / sqrtf(d), mask * kLog2e) and
    softmax numerators p = exp2(s - max) (log2 domain, as attention.cu), the denominator summed from the fp32 p, P rounded to the
    16-bit format before P V, the context rounded to the 16-bit format.  One key block, as attend_tile_short: past 64 keys the
    kernel's online softmax rounds P against the running max of each block (oracle/step_ref.py attention_blockwise restates
    that).  Returns the 16-bit context as fp64 [B, Lq, H]."""
    B, Lq, H = q.shape
    Lk = k.shape[1]
    d = H // heads
    dt = torch.float16 if f16 else torch.bfloat16
    qh = q.float().reshape(B, Lq, heads, d).permute(0, 2, 1, 3)
    kh = k.float().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    vh = v.float().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    log2e = torch.tensor(1.4426950408889634, dtype=torch.float32)
    scale = log2e / torch.sqrt(torch.tensor(float(d), dtype=torch.float32))
    raw = (qh.double() @ kh.double().transpose(-1, -2)).float()
    s = (raw.double() * scale.double() + (mask_add.float() * log2e).double()[:, None, None, :]).float()
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = (p.to(dt).double() @ vh.double()).float() * (1.0 / l)
    return o.to(dt).double().permute(0, 2, 1, 3).reshape(B, Lq, H)
