"""Every attention kernel against fp64 at its mask, length and key-block edges.  `-m gpu` only.

The attention paths all compute softmax(Q K^T / sqrt(d) + mask) V, but each skips or predicates work at its own places: the staged
kernels' 16-key tile padding and 64-key online-softmax blocks (attention.cu attend_tile_short / attend_tile), the streaming kernels'
ring of 64-key blocks, the fp32 kernel's 32-key chunks, its probability rows rounded up to 32 keys and its 8-query-row CTAs
(attention_f32.cu).  Every call here holds one sample per edge mask (oracle/kernel_refs.py EDGE_MASKS: one real key at 0, 63, 64,
65 or last, whole 64-key blocks masked, mask edges one key either side of each multiple of 16, key 0 masked, every key masked), at
lengths on both sides of those boundaries.

The 16-bit kernels are held to the bound of tests/test_gpu_kernel_parity.py (error over max(1, |fp64|)), bit for bit to one another
where two of them accept the same call, and exactly to V where a sample has one real key.  The fp32 kernel is held to a bound derived
from its fp32 arithmetic (_f32_bounds).  A sample whose keys are all masked is compared with the unmasked softmax: adding -10000 to
every score changes no probability.  Output buffers start as NaN, and every write outside a kernel's contract shows up there.
"""
import math

import pytest
import torch

from oracle import kernel_refs as R
import support

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
NAN = float("nan")
HEADS = 2
# tests/test_gpu_kernel_parity.py's attention bounds: error / max(1, |ref|) against fp64, about twice the rounding floor
ATTN_TOL = {torch.bfloat16: 1.2e-2, torch.float16: 1.5e-3}
STAGED = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256]      # every staged path, both sides of 16 / 64
LONG = [257, 511, 512]                                                                   # past the engine's staged plans
PATTERNS = R.EDGE_MASKS
P = len(PATTERNS)
# co-attention (T, V): T <= 64 < V and the reverse put the short path in one direction of a CTA and the block path in the other
CO_PAIRS = [(1, 65), (8, 9), (17, 129), (64, 65), (63, 256), (65, 64), (129, 17), (256, 1), (33, 127), (255, 32), (257, 64),
            (31, 511), (512, 65)]


def _f16(dt):
    return 1 if dt == torch.float16 else 0


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _offs(lengths):
    o = [0]
    for n in lengths:
        o.append(o[-1] + n)
    return o


def _dev_i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _is_nan(t):
    return bool(torch.isnan(t.float()).all())


def _masks(L, pats):
    """[len(pats), L] additive masks on the device, sample b with pattern pats[b]."""
    return torch.stack([R.edge_mask(p, L) for p in pats]).cuda()


def _rotate(shift):
    return [PATTERNS[(b + shift) % P] for b in range(P)]


def _staged_fits(d, L, n_mask):
    """The staged kernels' shared-memory check (attention.cu launch_self / launch_co): Q, K and V tiles of pad16(L) rows of d + 8
    16-bit elements, plus n_mask fp32 mask entries, within 227 KB."""
    return 3 * ((L + 15) // 16 * 16) * (d + 8) * 2 + 4 * n_mask <= 227 * 1024


def _reference(q, k, v, mask):
    """fp64 (probabilities, context) of a call; samples whose keys are all masked get the unmasked softmax."""
    full = (mask == R.MASKED).all(1)
    return R.attention_probs_fp64(q, k, v, torch.where(full[:, None], torch.zeros_like(mask), mask), HEADS)


def _note(worst, key, pats, per_sample):
    d = worst.setdefault(key, {})
    for p, e in zip(pats, per_sample.tolist()):
        d[p] = max(d.get(p, 0.0), e)


# ================================================================================================================ 16-bit kernels
def _check16(ctx, q, k, v, mask, dt, what):
    """One call's context [B, Lq, H] (16-bit, from the kernel) against fp64: within ATTN_TOL of error / max(1, |ref|), plus, where
    every key is masked, the rounding of the masked scores (kernel_refs.masked_score_slack); no NaN; a sample with one real key
    gets that key's V row exactly (its probability is exp2(0) = 1, the others exp2(about -14427) = 0, and 1 x v is exact in the fp32
    accumulator).  Returns the error measure per sample."""
    p, ref = _reference(q, k, v, mask)
    slack = R.masked_score_slack(p, mask == R.MASKED, v, ref, HEADS, R.MASKED_SCORE_ERR["tc"])
    assert not torch.isnan(ctx.float()).any(), what
    err = (ctx.double() - ref).abs()
    scale = ref.abs().clamp(min=1.0)
    bad = err > ATTN_TOL[dt] * scale + slack
    assert not bad.any(), f"{what}: samples {sorted(set(bad.nonzero()[:, 0].tolist()))}, worst {((err - slack) / scale).max().item():.3e}"
    for b in range(mask.shape[0]):
        j = R.single_real_key(mask[b])
        if j is not None:
            assert support.eq16(ctx[b], v[b, j][None].expand_as(ctx[b])), f"{what}: sample {b}, single real key {j}"
    return (err / scale).amax(dim=(1, 2))


def _self(hook, qkv, ld_qkv, H, mask, B, L, d, dt, rows, offs=None):
    ctx = torch.full((rows + 16, H + 8), NAN, dtype=dt, device="cuda")
    args = (qkv, ld_qkv, H, mask, ctx, H + 8, B, L, HEADS, d, _f16(dt))
    if hook != "vb200_self_attention":              # the dense staged hook has no row offsets
        args += (offs,)
    support.call(hook, *args)
    return ctx


def _co(hook, qi, qt, ld, H, mi, mt, B, T, V, d, dt, rows_t, rows_v, ot=None, ov=None):
    ct = torch.full((rows_t + 16, H + 8), NAN, dtype=dt, device="cuda")
    ci = torch.full((rows_v + 16, H), NAN, dtype=dt, device="cuda")
    args = (qi, ld, qt, ld, H, mi, mt, ct, H + 8, ci, H, B, T, V, HEADS, d, _f16(dt))
    if hook != "vb200_co_attention":
        args += (ot, ov)
    support.call(hook, *args)
    return ct, ci


def _split(x, H):
    return x[..., :H], x[..., H:2 * H], x[..., 2 * H:3 * H]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_self_attention_edges(d, dt, parity_log):
    """Dense self-attention, one sample per edge mask, at every staged length and past 256: the streaming kernel against fp64, and
    the staged kernel equal to it bit for bit wherever it accepts the length; nothing written outside the context."""
    H = HEADS * d
    ld = 3 * H + 8
    worst = {}
    for L in STAGED + LONG:
        pats = _rotate(L)
        qkv = torch.randn(P * L, ld, generator=_gen(L * 2 + d), device="cuda").to(dt)
        mask = _masks(L, pats)
        stream = _self("vb200_self_attention_stream", qkv, ld, H, mask, P, L, d, dt, P * L)
        torch.cuda.synchronize()
        q, k, v = _split(qkv[:, :3 * H].view(P, L, 3 * H), H)
        _note(worst, "stream", pats, _check16(stream[:P * L, :H].view(P, L, H), q, k, v, mask, dt, f"stream L = {L}"))
        assert _is_nan(stream[P * L:]) and _is_nan(stream[:, H:]), L
        if _staged_fits(d, L, L):
            staged = _self("vb200_self_attention", qkv, ld, H, mask, P, L, d, dt, P * L)
            torch.cuda.synchronize()
            assert support.eq16(staged, stream), f"staged != stream at L = {L}"
    parity_log(test="edge_self_attention", d=d, dtype=str(dt), bound=ATTN_TOL[dt], worst_rel_err=worst)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_self_attention_packed_edges(d, dt, parity_log):
    """One packed launch mixing every length with every edge mask: each sample equals a dense call of it alone bit for bit (staged
    kernel up to 256 rows, streaming kernel at every length), the packed staged and streaming launches agree bit for bit, fp64 holds,
    and the rows past the last sample keep the sentinel."""
    H = HEADS * d
    ld = 3 * H + 8
    lengths = STAGED + LONG
    n = 2 * len(lengths)
    samples = [(lengths[i % len(lengths)], PATTERNS[(3 * i + i // len(lengths)) % P]) for i in range(n)]
    worst = {}
    for hook, subset in (("vb200_self_attention_packed", [s for s in samples if s[0] <= 256]),
                         ("vb200_self_attention_stream", samples)):
        lens = [L for L, _ in subset]
        offs = _offs(lens)
        qkv = torch.randn(offs[-1], ld, generator=_gen(d + len(subset)), device="cuda").to(dt)
        mask = torch.cat([R.edge_mask(p, L) for L, p in subset]).cuda()
        o = _dev_i32(offs)
        packed = _self(hook, qkv, ld, H, mask, len(subset), max(lens), d, dt, offs[-1], o)
        if hook == "vb200_self_attention_packed":
            stream = _self("vb200_self_attention_stream", qkv, ld, H, mask, len(subset), max(lens), d, dt, offs[-1], o)
            torch.cuda.synchronize()
            assert support.eq16(packed, stream), "packed staged != packed streaming"
        dense_hook = "vb200_self_attention" if hook == "vb200_self_attention_packed" else hook
        for b, (L, pat) in enumerate(subset):
            sl = slice(offs[b], offs[b + 1])
            dense = _self(dense_hook, qkv[sl], ld, H, mask[sl].contiguous(), 1, L, d, dt, L)
            torch.cuda.synchronize()
            assert support.eq16(packed[sl], dense[:L]), f"{hook} sample {b} (L = {L}, {pat})"
            q, k, v = _split(qkv[sl, :3 * H].view(1, L, 3 * H), H)
            e = _check16(packed[sl, :H].view(1, L, H), q, k, v, mask[sl].view(1, L), dt, f"{hook} sample {b} (L = {L}, {pat})")
            _note(worst, hook, [pat], e)
        assert _is_nan(packed[offs[-1]:]) and _is_nan(packed[:, H:])
    parity_log(test="edge_self_attention_packed", d=d, dtype=str(dt), bound=ATTN_TOL[dt], worst_rel_err=worst)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_co_attention_edges(d, dt, parity_log):
    """Dense co-attention, one sample per edge-mask pair (text and image masks rotated against each other), T and V on either side of
    64 and past 256: both directions of the streaming kernel against fp64, the staged kernel equal to it bit for bit wherever it
    accepts the lengths (one CTA runs the short path in one direction and the block path in the other, over buffers sized for the
    longer stream); nothing written outside the contexts."""
    H = HEADS * d
    ld = 3 * H + 8
    worst = {}
    for T, V in CO_PAIRS:
        pt, pv = _rotate(T), _rotate(V + 11)
        g = _gen(T * 7 + V + d)
        qi = torch.randn(P * V, ld, generator=g, device="cuda").to(dt)
        qt = torch.randn(P * T, ld, generator=g, device="cuda").to(dt)
        mi, mt = _masks(V, pv), _masks(T, pt)
        ct, ci = _co("vb200_co_attention_stream", qi, qt, ld, H, mi, mt, P, T, V, d, dt, P * T, P * V)
        torch.cuda.synchronize()
        xi, xt = _split(qi[:, :3 * H].view(P, V, 3 * H), H), _split(qt[:, :3 * H].view(P, T, 3 * H), H)
        what = f"T = {T}, V = {V}"
        _note(worst, "stream_text", pv, _check16(ct[:P * T, :H].view(P, T, H), xt[0], xi[1], xi[2], mi, dt, "text ctx " + what))
        _note(worst, "stream_image", pt, _check16(ci[:P * V, :H].view(P, V, H), xi[0], xt[1], xt[2], mt, dt, "image ctx " + what))
        assert _is_nan(ct[P * T:]) and _is_nan(ct[:, H:]) and _is_nan(ci[P * V:]), what
        if _staged_fits(d, max(T, V), T + V):
            st, si = _co("vb200_co_attention", qi, qt, ld, H, mi, mt, P, T, V, d, dt, P * T, P * V)
            torch.cuda.synchronize()
            assert support.eq16(st, ct) and support.eq16(si, ci), f"staged != stream at {what}"
    parity_log(test="edge_co_attention", d=d, dtype=str(dt), bound=ATTN_TOL[dt], worst_rel_err=worst)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_co_attention_packed_edges(d, dt, parity_log):
    """One packed co-attention launch mixing every (T, V) pair with rotated edge masks: each sample equals a dense call of it alone
    bit for bit (staged up to 256 rows, streaming at every length), staged and streaming packed launches agree, fp64 holds, and the
    rows outside every sample keep the sentinel."""
    H = HEADS * d
    ld = 3 * H + 8
    n = 2 * len(CO_PAIRS)
    samples = [(*CO_PAIRS[i % len(CO_PAIRS)], PATTERNS[(3 * i) % P], PATTERNS[(5 * i + 1) % P]) for i in range(n)]
    worst = {}
    for hook, subset in (("vb200_co_attention_packed", [s for s in samples if max(s[0], s[1]) <= 256]),
                         ("vb200_co_attention_stream", samples)):
        T_l, V_l = [s[0] for s in subset], [s[1] for s in subset]
        ot, ov = _offs(T_l), _offs(V_l)
        g = _gen(d + 3 * len(subset))
        qi = torch.randn(ov[-1], ld, generator=g, device="cuda").to(dt)
        qt = torch.randn(ot[-1], ld, generator=g, device="cuda").to(dt)
        mi = torch.cat([R.edge_mask(s[3], s[1]) for s in subset]).cuda()
        mt = torch.cat([R.edge_mask(s[2], s[0]) for s in subset]).cuda()
        offs = (_dev_i32(ot), _dev_i32(ov))
        ct, ci = _co(hook, qi, qt, ld, H, mi, mt, len(subset), max(T_l), max(V_l), d, dt, ot[-1], ov[-1], *offs)
        if hook == "vb200_co_attention_packed":
            st, si = _co("vb200_co_attention_stream", qi, qt, ld, H, mi, mt, len(subset), max(T_l), max(V_l), d, dt, ot[-1], ov[-1],
                         *offs)
            torch.cuda.synchronize()
            assert support.eq16(ct, st) and support.eq16(ci, si), "packed staged != packed streaming"
        dense_hook = "vb200_co_attention" if hook == "vb200_co_attention_packed" else hook
        for b, (T, V, p_t, p_v) in enumerate(subset):
            s_t, s_v = slice(ot[b], ot[b + 1]), slice(ov[b], ov[b + 1])
            dct, dci = _co(dense_hook, qi[s_v], qt[s_t], ld, H, mi[s_v].contiguous(), mt[s_t].contiguous(), 1, T, V, d, dt, T, V)
            torch.cuda.synchronize()
            what = f"{hook} sample {b} (T = {T} {p_t}, V = {V} {p_v})"
            assert support.eq16(ct[s_t], dct[:T]) and support.eq16(ci[s_v], dci[:V]), what
            xi, xt = _split(qi[s_v, :3 * H].view(1, V, 3 * H), H), _split(qt[s_t, :3 * H].view(1, T, 3 * H), H)
            _note(worst, hook + "_text", [p_v], _check16(ct[s_t, :H].view(1, T, H), xt[0], xi[1], xi[2], mi[s_v].view(1, V), dt, what))
            _note(worst, hook + "_image", [p_t], _check16(ci[s_v, :H].view(1, V, H), xi[0], xt[1], xt[2], mt[s_t].view(1, T), dt, what))
        assert _is_nan(ct[ot[-1]:]) and _is_nan(ci[ov[-1]:]) and _is_nan(ct[:, H:])
    parity_log(test="edge_co_attention_packed", d=d, dtype=str(dt), bound=ATTN_TOL[dt], worst_rel_err=worst)


# ================================================================================================================ fp32 kernel
U = 2.0 ** -24          # unit roundoff of fp32
# (Lq, Lk): Lk on both sides of the 32-key chunks and past the 48 KB shared-memory opt-in (probability rows of 8 x Lkp floats: from
# Lk = 897 at d = 128 and Lk = 1217 at d = 64), Lq on both sides of the 8-row CTAs
F32_SHAPES = [(9, 1), (1, 2), (8, 31), (7, 32), (17, 33), (2, 63), (16, 64), (9, 65), (1, 255), (8, 256), (33, 257), (7, 1023),
              (9, 1024), (1, 1025), (8, 2047), (17, 2048)]
CTX_DT = {1: torch.float16, 2: torch.bfloat16, 3: torch.float16}


def _f32_bounds(p, s, mask, v):
    """Per-element bounds on |kernel - fp64| of attention_f32's probabilities [B, heads, Lq, Lk] and context [B, Lq, H] (before its
    16-bit store), for Q / K on kernel_refs.grid_qk's grid, whose dot products are exact in fp32.  s: the fp64 scores q.k / sqrt(d)
    [B, heads, Lq, Lk] without the mask; p: the fp64 probabilities.  First order in u = 2^-24, for one row of Lk keys:

      score    s^_j = fl(q.k * scale + mask_j), scale = 1 / sqrtf(d) within 2u of 1 / sqrt(d) (sqrtf and the division round once
               each), the product or the add rounding once more: |s^_j - s_j - mask_j| <= 3u |s_j|, plus, for a masked key, the
               rounding of a sum near -10000, half the ulp of [2^13, 2^14): 2^-11.
      shift    t_j = fl(s^_j - m), m the row maximum (exact): u |s_j + mask_j - m|.
      expf     2 ulp (CUDA C Programming Guide, no fast math): 4u relative.
               => e^_j = exp(s_j + mask_j - m) (1 + r_j), |r_j| <= 3u |s_j| + [masked] 2^-11 + u |s_j + mask_j - m| + 4u.
      sum      lane l adds keys l, l + 32, ... in order, then a 5-step butterfly: each term meets ceil(Lk / 32) + 5 roundings, so the
               fp32 sum is S (1 + sum_i p_i r_i + theta), |theta| <= (ceil(Lk / 32) + 5) u.
      1 / sum, e^_j * (1 / sum): one rounding each, 2u.
               => |p^_j - p_j| <= p_j (r_j + sum_i p_i r_i + (ceil(Lk / 32) + 7) u) =: b_j
      context  c^ = fmaf over the keys in order, one rounding per key: |c^ - c| <= sum_j b_j |v_j| + Lk u sum_j p_j |v_j|.

    The sum term is the only one that grows with Lk: 12u at Lk = 200, 71u at Lk = 2048.  2^-10 of relative headroom and 2^-126 of
    absolute headroom cover the second-order terms and probabilities below fp32's normal range."""
    Lk = p.shape[-1]
    masked = (mask == R.MASKED).double()[:, None, None, :]
    sm = s + mask.double()[:, None, None, :]
    r = 3 * U * s.abs() + 2.0 ** -11 * masked + U * (sm - sm.amax(-1, keepdim=True)).abs() + 4 * U
    bp = p * (r + (p * r).sum(-1, keepdim=True) + (math.ceil(Lk / 32) + 7) * U)
    bp = bp * (1 + 2.0 ** -10) + 2.0 ** -126
    B, heads, Lq, _ = p.shape
    vh = v.double().abs().reshape(B, Lk, heads, -1).permute(0, 2, 1, 3)
    bc = bp @ vh + Lk * U * (p @ vh)
    return bp, (bc * (1 + 2.0 ** -10)).permute(0, 2, 1, 3).reshape(B, Lq, -1)


def _unsplit(y3, H):
    """fp16 hi | lo | hi per 64 columns -> hi + lo in fp32 (the second hi copy must equal the first)."""
    v = y3[:, :3 * H].reshape(y3.shape[0], H // 64, 3, 64).float()
    assert torch.equal(v[:, :, 0], v[:, :, 2])
    return (v[:, :, 0] + v[:, :, 1]).reshape(y3.shape[0], H)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("in_kind", [0, 1, 2], ids=["fp32", "fp16", "bf16"])
def test_attention_f32_edges(in_kind, d, parity_log):
    """The fp32 attention kernel, one sample per edge mask, Lk from 1 to 2048 and Lq on both sides of its 8-row CTAs, in every
    context mode: probabilities within _f32_bounds of fp64 and rows summing to 1 within the sum of those bounds; every masked key of
    a row with a real key exactly 0; one real key exactly one-hot, its context exactly that V row in the output format; fully masked
    rows equal to the unmasked softmax; probabilities identical in ctx modes 0 - 3; the context within _f32_bounds plus its store's
    rounding; nothing written outside the outputs."""
    H = HEADS * d
    dt = [torch.float32, torch.float16, torch.bfloat16][in_kind]
    worst = {}
    worst_ratio, worst_ctx = 0.0, {m: 0.0 for m in (1, 2, 3)}
    for Lq, Lk in F32_SHAPES:
        pats = _rotate(Lk)
        g = _gen(Lq * 4096 + Lk + d)
        amp = [1.0, 4.0, 8.0]                      # score spread about 0.3, 1.3 and 2.7: flat to peaked rows
        q = torch.cat([R.grid_qk(Lq, H, amp[b % 3], g) for b in range(P)]).to(dt)
        kv = torch.cat([R.grid_qk(P * Lk, H, 1.0, g), torch.randn(P * Lk, H, generator=g, device="cuda")], dim=1).to(dt)
        mask = _masks(Lk, pats)
        qd, kd, vd = q.view(P, Lq, H), kv[:, :H].view(P, Lk, H), kv[:, H:].view(P, Lk, H)
        p, c = _reference(qd, kd, vd, mask)
        qh = qd.double().view(P, Lq, HEADS, d).permute(0, 2, 1, 3)
        s = qh @ kd.double().view(P, Lk, HEADS, d).permute(0, 2, 3, 1) / math.sqrt(d)
        bp, bc = _f32_bounds(p, s, mask, vd)
        n = P * HEADS * Lq * Lk
        what = f"Lq = {Lq}, Lk = {Lk}"
        first = None
        for ctx_mode in (0, 1, 2, 3):
            probs = torch.full((n + 64,), NAN, device="cuda")
            ctx, ld = None, 0
            if ctx_mode:
                ld = (3 * H if ctx_mode == 3 else H) + 8
                ctx = torch.full((P * Lq + 8, ld), NAN, dtype=CTX_DT[ctx_mode], device="cuda")
            support.call("vb200_attention_f32", q, H, kv, kv.data_ptr() + H * kv.element_size(), 2 * H, in_kind, mask, P, Lq, Lk,
                         HEADS, d, ctx, ld, ctx_mode, probs)
            torch.cuda.synchronize()
            assert _is_nan(probs[n:]), what
            pk = probs[:n].view(P, HEADS, Lq, Lk)
            if first is None:
                first = pk
            else:
                assert support.eq32(pk, first), f"{what}: probabilities differ between ctx modes 0 and {ctx_mode}"
            if ctx is None:
                continue
            assert _is_nan(ctx[P * Lq:]) and _is_nan(ctx[:, 3 * H if ctx_mode == 3 else H:]), what
            got = _unsplit(ctx[:P * Lq], H) if ctx_mode == 3 else ctx[:P * Lq, :H].float()
            got = got.view(P, Lq, H).double()
            store = {1: 2.0 ** -11, 2: 2.0 ** -8, 3: 2.0 ** -22}[ctx_mode] * (c.abs() + bc) + (0.0 if ctx_mode == 2 else 2.0 ** -25)
            cerr = (got - c).abs()
            assert (cerr <= bc + store).all(), f"{what}, ctx mode {ctx_mode}: worst {(cerr / (bc + store)).max().item():.3f} of the bound"
            worst_ctx[ctx_mode] = max(worst_ctx[ctx_mode], cerr.max().item())
            for b in range(P):
                j = R.single_real_key(mask[b])
                if j is not None:
                    row = vd[b, j].float()[None].expand(Lq, H)
                    want = R.split16(row) if ctx_mode == 3 else R.sat_rn(row, ctx_mode == 1)
                    assert support.eq16(ctx[b * Lq:(b + 1) * Lq, :want.shape[1]], want), f"{what}, ctx mode {ctx_mode}: sample {b}"
        pk = first.double()
        assert torch.isfinite(pk).all(), what
        err = (pk - p).abs()
        bad = err > bp
        assert not bad.any(), f"{what}: samples {sorted(set(bad.nonzero()[:, 0].tolist()))}, worst {(err / bp).max().item():.3f} of the bound"
        row_err = (pk.sum(-1) - 1.0).abs()
        assert (row_err <= bp.sum(-1) + Lk * 2.0 ** -53).all(), f"{what}: row sums, worst {row_err.max().item():.3e}"
        real = (mask == 0).any(1)
        zero = (mask == R.MASKED)[:, None, None, :] & real[:, None, None, None]
        assert (pk[zero.expand_as(pk)] == 0).all(), f"{what}: a masked key of a row with a real key has a nonzero probability"
        for b in range(P):
            j = R.single_real_key(mask[b])
            if j is not None:
                one_hot = torch.zeros(Lk, dtype=torch.float64, device="cuda")
                one_hot[j] = 1.0
                assert torch.equal(pk[b], one_hot.expand_as(pk[b])), f"{what}: sample {b}, single real key {j}"
        _note(worst, "probs", pats, err.amax(dim=(1, 2, 3)))
        worst_ratio = max(worst_ratio, (err / bp).max().item())
    parity_log(test="edge_attention_f32", in_kind=in_kind, d=d, probs_worst_abs_err=worst["probs"], probs_worst_share_of_bound=worst_ratio,
               ctx_worst_abs_err=worst_ctx)
