"""The kernels and forwards the VB200_* launch switches reach, each checked against its oracle, with a digest of every output.

Not a test module: pytest does not collect it.  Each switch is read once per process, into a function-local static, at its first
launch, so a setting can only be tested in a fresh process: tests/test_gpu_switches.py runs this script once without any VB200_*
variable and once per setting, and compares the digests.

    python tests/switch_child.py --sections gemm,ln,attn,fwd[,full] --out OUT.json

Sections: gemm (every GEMM case; gemm_grid the tile-count cases alone, gemm_rows the vb200_linear_rows cases alone), ln, attn, fwd
(the tiny engine) and full (the full-size bf16 engine).  Every case checks itself: GEMMs bitwise on exact-valued operands, LayerNorm
and attention against fp64 at the bounds of the op suites, forwards free of NaN.  The first failed check ends the run with exit
status 1 and a message naming its case.  Otherwise OUT.json maps every output's name to the sha256 of its bytes (shape and dtype
included).  Output buffers start NaN-filled with padding rows and columns, and every check requires the padding to keep its NaN.
"""
import argparse
import hashlib
import json
import os
import re
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SECTIONS = ("gemm", "gemm_grid", "gemm_rows", "ln", "attn", "fwd", "full")
NAN = float("nan")


class CaseFailed(Exception):
    pass


def require(ok, case, msg=""):
    if not ok:
        raise CaseFailed(f"{case}: {msg}" if msg else case)


class Digests(dict):
    def add(self, name, obj):
        """sha256 of a tensor's shape, dtype and bytes, or of the repr of a host value; nested tuples, lists and dicts get one entry
        per leaf, named by its path."""
        import torch
        if isinstance(obj, (tuple, list)) and any(torch.is_tensor(o) or isinstance(o, (tuple, list, dict)) for o in obj):
            for i, o in enumerate(obj):
                self.add(f"{name}[{i}]", o)
        elif isinstance(obj, dict):
            for k, o in obj.items():
                self.add(f"{name}[{k}]", o)
        elif torch.is_tensor(obj):
            t = obj.detach().contiguous().cpu()
            h = hashlib.sha256(f"{tuple(t.shape)} {t.dtype}".encode())
            if t.numel():
                h.update(t.reshape(-1).view(torch.uint8).numpy().tobytes())
            self[name] = h.hexdigest()
        elif obj is not None:
            self[name] = hashlib.sha256(repr(obj).encode()).hexdigest()


def _atoi(s):
    """C atoi: optional whitespace and sign, then digits; 0 when there are none."""
    m = re.match(r"\s*([+-]?\d+)", s)
    return int(m.group(1)) if m else 0


# ============================================================================================================================ gemm
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_slots():
    """persistent_grid's slot count S (gemm_persistent.cuh): VB200_GRID_PCT clamped to 10..100, else 100; S = max(1, SMs pct / 100)."""
    e = os.environ.get("VB200_GRID_PCT")
    v = _atoi(e) if e is not None else 100
    pct = v if 10 <= v <= 100 else 100
    return max(1, sm_count() * pct // 100)


def grid_balanced():
    e = os.environ.get("VB200_GRID_BALANCE")
    return e is None or _atoi(e) != 0


def balanced_grid(tiles, slots):
    if tiles <= slots:
        return tiles
    per = -(-tiles // slots)
    return -(-tiles // per)


def persistent_grid(tiles):
    """The CTA count persistent_grid launches for `tiles` tiles in this process's environment."""
    slots = grid_slots()
    return balanced_grid(tiles, slots) if grid_balanced() else min(tiles, slots)


def _f16(dt):
    import torch
    return dt == torch.float16


def _dt_name(dt):
    import torch
    return "fp16" if dt == torch.float16 else "bf16"


def _all_nan(t):
    import torch
    return bool(torch.isnan(t.float()).all())


def _buffers(M, N, dt):
    """NaN-filled outputs with 8 padding rows and padding columns (ld16 = N rounded up to 8, plus 8; ld32 = N rounded up to 4, plus 4)."""
    import torch
    ld16, ld32 = (N + 7) // 8 * 8 + 8, (N + 3) // 4 * 4 + 4
    return (torch.full((M + 8, ld16), NAN, dtype=dt, device="cuda"), ld16,
            torch.full((M + 8, ld32), NAN, device="cuda"), ld32)


def _check_gemm(case, y16, y32, x, w, b, act, N, dt, rows):
    """Rows [0, rows) against the exact result -- y32 bitwise (act 0 / 2) or within GELU_BOUND of fp64 GELU of the exact
    pre-activation with gelu_erf's saturation (act 1), y16 == sat_rn(y32) --; padding columns keep their NaN."""
    import support
    from oracle import kernel_refs as R
    if act == 1:
        pre = R.exact_linear(x, w, b, 0)[:rows]
        got = y32[:rows, :N]
        err = (got.double() - R.gelu_fp64(pre.double())).abs().max().item()
        require(err <= R.GELU_BOUND, case, f"GELU output {err:.3e} from fp64 GELU (bound {R.GELU_BOUND})")
        lo, hi = pre < R.GELU_ZERO_BELOW, pre > R.GELU_IDENTITY_ABOVE
        require(bool((got[lo] == 0).all()) and support.eq32(got[hi], pre[hi]), case, "GELU saturation")
        ref = got
    else:
        ref = R.exact_linear(x, w, b, act)[:rows]
        bad = int((y32[:rows, :N] != ref).sum())
        require(support.eq32(y32[:rows, :N], ref), case, f"fp32 output differs from the exact result ({bad} elements)")
    require(support.eq16(y16[:rows, :N], R.sat_rn(ref, _f16(dt))), case, "16-bit output is not sat_rn of the fp32 output")
    require(_all_nan(y32[:, N:]) and _all_nan(y16[:, N:]), case, "padding columns written")


def _linear(case, d, M, N, K, dt, act, variant, bn, seed, stamps=False):
    """vb200_linear on exact operands, checked; with `stamps`, the CTA count and, on ping-pong, the tiles each CTA walked."""
    import support
    import torch
    from oracle import kernel_refs as R
    x, w, b = R.exact_operands(M, N, K, None, _f16(dt), seed, device="cuda")
    y16, ld16, y32, ld32 = _buffers(M, N, dt)
    sms = sm_count()
    timing = torch.zeros(sms, 16, dtype=torch.int64, device="cuda") if stamps else None
    support.call("vb200_linear", x, K, w, K, b, None, 0, None, None, 1e-12, act, y16, ld16, y32, ld32, M, N, K, bn, 0, int(_f16(dt)),
                 variant, timing)
    torch.cuda.synchronize()
    _check_gemm(case, y16, y32, x, w, b, act, N, dt, M)
    require(_all_nan(y32[M:]) and _all_nan(y16[M:]), case, "rows past M written")
    d.add(case + "/y16", y16)
    d.add(case + "/y32", y32)
    if stamps:
        tiles = (M + 127) // 128 * ((N + bn - 1) // bn)
        g = persistent_grid(tiles)
        stamped = timing[:, 0] != 0
        n = int(stamped.sum())
        require(n == g and bool(stamped[:g].all()), case, f"{n} CTAs stamped, persistent_grid predicts {g} for {tiles} tiles "
                f"(S = {grid_slots()}, balance {'on' if grid_balanced() else 'off'})")
        if variant == 5:
            walked = timing[:g, 11].cpu()
            want = torch.tensor([-(-(tiles - c) // g) for c in range(g)])
            require(torch.equal(walked, want), case, f"tiles per CTA {walked.tolist()} instead of the strided walk {want.tolist()}")
            require(int(walked.sum()) == tiles, case, "the CTAs walked a different number of tiles")


def gemm_grid(d):
    """vb200_linear, cooperative (variant 0) and ping-pong (5) at 64- and 128-wide tiles in fp16 and bf16, at tile counts around one,
    two and three times the grid's S slots, the last row tile ragged (M = 128 tiles - 5), K = 64; CTA count and tiles walked checked
    against persistent_grid.  CTA c of a grid g walks tiles c, c + g, ..., so with balancing on or off every CTA walks the floor or
    the ceiling of tiles / g: the balance switch shows in the CTA count, not in the spread of tiles per CTA."""
    import torch
    S = grid_slots()
    counts = sorted({t for t in (1, S - 1, S, S + 1, 2 * S - 1, 2 * S + 1, 3 * S + 2) if t >= 1})
    # the set must hold a tile count at which the balanced and the unbalanced grid differ, or the balance switch goes unchecked
    require(any(balanced_grid(t, S) != min(t, S) for t in counts), "gemm/grid", f"no tile count tells the grid modes apart at S = {S}")
    i = 0
    for variant, bn in ((0, 64), (0, 128), (5, 64), (5, 128)):
        for dt in (torch.float16, torch.bfloat16):
            for tiles in counts:
                act = (0, 2, 1)[i % 3]
                i += 1
                M = 128 * tiles - 5
                case = f"gemm/tiles{tiles}/v{variant}_bn{bn}_{_dt_name(dt)}_act{act}"
                _linear(case, d, M, bn, 64, dt, act, variant, bn, seed=tiles * 8 + variant + bn, stamps=True)


# (M, N, K, act): engine GEMMs -- the text FFN-in with GELU at batch 64, the image FFN-in at batch 64, the text attention output at
# batch 512 (about 57 tiles per CTA at S = 13), the VQA head's last layer (ragged N: cooperative only)
ENGINE_GEMMS = [(1984, 3072, 768, 1), (2304, 3072, 1024, 0), (15872, 768, 768, 2), (64, 3129, 2048, 0)]


def gemm_engine(d):
    import torch
    for i, (M, N, K, act) in enumerate(ENGINE_GEMMS):
        for dt in (torch.float16, torch.bfloat16):
            for variant in ((0, 5) if N % 128 == 0 else (0,)):
                case = f"gemm/engine_{M}x{N}x{K}/v{variant}_{_dt_name(dt)}_act{act}"
                _linear(case, d, M, N, K, dt, act, variant, 128, seed=100 + i, stamps=True)


def gemm_rows(d):
    """vb200_linear_rows (the process's default kernel: ping-pong unless VB200_GEMM=coop) with a device row count that ends mid-grid:
    rows below it exact, rows from the next 128-row boundary on untouched; the ragged-N form runs the cooperative kernel."""
    import support
    import torch
    from oracle import kernel_refs as R
    for N, K, M, m in ((256, 192, 4000, 2500), (1601, 768, 3000, 1300)):
        for dt in (torch.float16, torch.bfloat16):
            case = f"gemm/rows_{M}x{N}x{K}_m{m}/{_dt_name(dt)}"
            x, w, b = R.exact_operands(M, N, K, None, _f16(dt), N + m, device="cuda")
            y16, ld16, y32, ld32 = _buffers(M, N, dt)
            support.call("vb200_linear_rows", x, K, w, K, b, 0, y16, ld16, y32, ld32, M, N, K, 0, int(_f16(dt)),
                         torch.tensor([m], dtype=torch.int32, device="cuda"))
            torch.cuda.synchronize()
            _check_gemm(case, y16, y32, x, w, b, 0, N, dt, m)
            edge = (m + 127) // 128 * 128
            require(_all_nan(y32[edge:]) and _all_nan(y16[edge:]), case, "rows past the device row count's last tile written")
            d.add(case + "/y16", y16[:m])
            d.add(case + "/y32", y32[:m])


def gemm_split(d):
    """vb200_linear_split (fp32-parity mode, 64-wide cooperative tiles) on exact fp16 operands, lo parts zero: y32 exact and the split
    16-bit output split16 of it."""
    import support
    import torch
    from oracle import kernel_refs as R
    M, N, K = 2000, 384, 256
    case = f"gemm/split_{M}x{N}x{K}"
    x, w, b = R.exact_operands(M, N, K, None, True, 7, device="cuda")
    ref = R.exact_linear(x, w, b, 0)
    x3, w3 = R.split16(x.float()), R.split16_w(w.float())
    y3 = torch.full((M + 8, 3 * N + 64), NAN, dtype=torch.float16, device="cuda")
    y32 = torch.full((M + 8, N + 4), NAN, device="cuda")
    support.call("vb200_linear_split", x3, 3 * K, w3, 3 * K, b, 0, y3, 3 * N + 64, y32, N + 4, M, N, 3 * K)
    torch.cuda.synchronize()
    require(support.eq32(y32[:M, :N], ref), case, f"fp32 output differs from the exact result ({int((y32[:M, :N] != ref).sum())})")
    require(support.eq16(y3[:M, :3 * N], R.split16(ref)), case, "split 16-bit output is not split16 of the exact result")
    require(_all_nan(y32[:, N:]) and _all_nan(y3[:, 3 * N:]) and _all_nan(y32[M:]) and _all_nan(y3[M:]), case, "padding written")
    d.add(case + "/y3", y3)
    d.add(case + "/y32", y32)


# ============================================================================================================================== ln
LN_M = (1985, 17, 9, 8, 7, 3, 2, 1)
LN_N = (128, 768, 1024, 2048)


def _ln_inputs(M, N, ld, seed):
    """y (N(0.5, 3)) and residual (N(0, 1)) with row stride ld (NaN past N), gamma ~ 1 + N(0, 0.1), beta ~ N(0, 0.1)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.full((M, ld), NAN, device="cuda")
    res = torch.full((M, ld), NAN, device="cuda")
    y[:, :N] = torch.randn(M, N, generator=g, device="cuda") * 3 + 0.5
    res[:, :N] = torch.randn(M, N, generator=g, device="cuda")
    gamma = 1.0 + 0.1 * torch.randn(N, generator=g, device="cuda")
    beta = 0.1 * torch.randn(N, generator=g, device="cuda")
    return y, res, gamma, beta


def _ln_ref(y, res, gamma, beta, N):
    import torch
    x = y[:, :N].double() + (res[:, :N].double() if res is not None else 0.0)
    return torch.nn.functional.layer_norm(x, (N,), gamma.double(), beta.double(), 1e-12)


def ln(d):
    """vb200_layernorm at ragged and one-row M for every rows-per-CTA setting, with and without the residual, fp16 and bf16: fp32
    output within 1e-5 of fp64 (tests/test_gpu_ops.py test_layernorm_row_kernel), 16-bit output == sat_rn of the fp32 one
    (tests/test_gpu_kernel_parity.py test_layernorm_row_kernel_16bit_rounding), row M and padding columns untouched; then
    vb200_layernorm_split, its hi | lo | hi output split16 of the fp32 one."""
    import support
    import torch
    from oracle import kernel_refs as R
    for N in LN_N:
        ld = N + 8
        for M in LN_M:
            y, res, gamma, beta = _ln_inputs(M, N, ld, seed=M * 4096 + N)
            for with_res in (True, False):
                r = res if with_res else None
                ref = _ln_ref(y, r, gamma, beta, N)
                for dt in (torch.float16, torch.bfloat16):
                    case = f"ln/M{M}_N{N}_{'res' if with_res else 'nores'}_{_dt_name(dt)}"
                    of = torch.full((M + 1, ld), NAN, device="cuda")
                    oh = torch.full((M + 1, ld), NAN, dtype=dt, device="cuda")
                    support.call("vb200_layernorm", y, ld, r, ld if with_res else 0, gamma, beta, 1e-12, of, ld, oh, ld, M, N, int(_f16(dt)))
                    torch.cuda.synchronize()
                    require(not torch.isnan(of[:M, :N]).any(), case, "fp32 rows left NaN")
                    err = (of[:M, :N].double() - ref).abs().max().item()
                    require(err < 1e-5, case, f"fp32 output {err:.3e} from fp64 LayerNorm")
                    require(support.eq16(oh[:M, :N], R.sat_rn(of[:M, :N], _f16(dt))), case, "16-bit output is not sat_rn of the fp32 output")
                    require(_all_nan(of[M:]) and _all_nan(oh[M:]) and _all_nan(of[:, N:]) and _all_nan(oh[:, N:]), case, "padding written")
                    d.add(case + "/f32", of)
                    d.add(case + "/16", oh)
    N, ld = 768, 776
    for M in (1, 9, 333):
        case = f"ln/split_M{M}_N{N}"
        y, res, gamma, beta = _ln_inputs(M, N, ld, seed=M + 17)
        ref = _ln_ref(y, res, gamma, beta, N)
        of = torch.full((M + 1, ld), NAN, device="cuda")
        o3 = torch.full((M + 1, 3 * N + 8), NAN, dtype=torch.float16, device="cuda")
        support.call("vb200_layernorm_split", y, ld, res, ld, gamma, beta, 1e-12, of, ld, o3, 3 * N + 8, M, N)
        torch.cuda.synchronize()
        require(not torch.isnan(of[:M, :N]).any(), case, "fp32 rows left NaN")
        err = (of[:M, :N].double() - ref).abs().max().item()
        require(err < 1e-5, case, f"fp32 output {err:.3e} from fp64 LayerNorm")
        require(support.eq16(o3[:M, :3 * N], R.split16(of[:M, :N])), case, "split 16-bit output is not split16 of the fp32 output")
        require(_all_nan(of[M:]) and _all_nan(o3[M:]) and _all_nan(of[:, N:]) and _all_nan(o3[:, 3 * N:]), case, "padding written")
        d.add(case + "/f32", of)
        d.add(case + "/split16", o3)


# ============================================================================================================================ attn
HEADS = 2
# tests/test_gpu_attention_edges.py's bounds (those of tests/test_gpu_kernel_parity.py): error / max(1, |fp64|)
ATTN_TOL = {"fp16": 1.5e-3, "bf16": 1.2e-2}
SELF_L = (1, 15, 16, 17, 31, 48, 63, 64, 65, 100, 128, 129, 200, 256)
# (T, V): T <= 64 < V, V <= 64 < T, T = 1, V = 1, both long
CO_TV = ((1, 65), (17, 129), (63, 256), (129, 17), (256, 1), (65, 64), (8, 9), (256, 256))
PACKED_L = (1, 15, 17, 64, 65, 129, 200, 256, 31, 100)


def _attn_check(case, ctx, q, k, v, mask, dt):
    """ctx [B, Lq, H] against fp64 as tests/test_gpu_attention_edges.py _check16 does: error within ATTN_TOL x max(1, |ref|) plus the
    masked-score slack where every key is masked (the unmasked softmax is the reference there), no NaN, a sample with one real key
    equal to that key's V row bit for bit."""
    import support
    import torch
    from oracle import kernel_refs as R
    full = (mask == R.MASKED).all(1)
    p, ref = R.attention_probs_fp64(q, k, v, torch.where(full[:, None], torch.zeros_like(mask), mask), HEADS)
    slack = R.masked_score_slack(p, mask == R.MASKED, v, ref, HEADS, R.MASKED_SCORE_ERR["tc"])
    require(not torch.isnan(ctx.float()).any(), case, "context rows left NaN")
    err = (ctx.double() - ref).abs()
    scale = ref.abs().clamp(min=1.0)
    bad = err > ATTN_TOL[_dt_name(dt)] * scale + slack
    require(not bad.any(), case, f"samples {sorted(set(bad.nonzero()[:, 0].tolist()))} off fp64, worst "
            f"{((err - slack) / scale).max().item():.3e}")
    for b in range(mask.shape[0]):
        j = R.single_real_key(mask[b])
        if j is not None:
            require(support.eq16(ctx[b], v[b, j][None].expand_as(ctx[b])), case, f"sample {b}: single real key {j}")


def _qkv_split(x, H):
    return x[..., :H], x[..., H:2 * H], x[..., 2 * H:3 * H]


def attn(d):
    """The staged self- and co-attention kernels (dense and packed), one sample per edge mask, against fp64; contexts start NaN with
    padding rows and columns."""
    import support
    import torch
    from oracle import kernel_refs as R
    P = len(R.EDGE_MASKS)
    pats = lambda shift: [R.EDGE_MASKS[(b + shift) % P] for b in range(P)]
    masks = lambda L, ps: torch.stack([R.edge_mask(p, L) for p in ps]).cuda()
    for D in (64, 128):
        H = HEADS * D
        ld = 3 * H + 8
        for dt in (torch.float16, torch.bfloat16):
            tag = f"d{D}_{_dt_name(dt)}"
            f16 = int(_f16(dt))
            for L in SELF_L:
                case = f"attn/self_L{L}_{tag}"
                g = torch.Generator(device="cuda").manual_seed(L * 2 + D)
                qkv = torch.randn(P * L, ld, generator=g, device="cuda").to(dt)
                mask = masks(L, pats(L))
                ctx = torch.full((P * L + 16, H + 8), NAN, dtype=dt, device="cuda")
                support.call("vb200_self_attention", qkv, ld, H, mask, ctx, H + 8, P, L, HEADS, D, f16)
                torch.cuda.synchronize()
                q, k, v = _qkv_split(qkv[:, :3 * H].view(P, L, 3 * H), H)
                _attn_check(case, ctx[:P * L, :H].view(P, L, H), q, k, v, mask, dt)
                require(_all_nan(ctx[P * L:]) and _all_nan(ctx[:, H:]), case, "padding written")
                d.add(case, ctx)
            for T, V in CO_TV:
                case = f"attn/co_T{T}_V{V}_{tag}"
                g = torch.Generator(device="cuda").manual_seed(T * 7 + V + D)
                qi = torch.randn(P * V, ld, generator=g, device="cuda").to(dt)
                qt = torch.randn(P * T, ld, generator=g, device="cuda").to(dt)
                pv, pt = pats(V + 11), pats(T)
                mi, mt = masks(V, pv), masks(T, pt)
                ct = torch.full((P * T + 16, H + 8), NAN, dtype=dt, device="cuda")
                ci = torch.full((P * V + 16, H + 8), NAN, dtype=dt, device="cuda")
                support.call("vb200_co_attention", qi, ld, qt, ld, H, mi, mt, ct, H + 8, ci, H + 8, P, T, V, HEADS, D, f16)
                torch.cuda.synchronize()
                xi, xt = _qkv_split(qi[:, :3 * H].view(P, V, 3 * H), H), _qkv_split(qt[:, :3 * H].view(P, T, 3 * H), H)
                _attn_check(case + " text", ct[:P * T, :H].view(P, T, H), xt[0], xi[1], xi[2], mi, dt)
                _attn_check(case + " image", ci[:P * V, :H].view(P, V, H), xi[0], xt[1], xt[2], mt, dt)
                require(_all_nan(ct[P * T:]) and _all_nan(ct[:, H:]) and _all_nan(ci[P * V:]) and _all_nan(ci[:, H:]), case,
                        "padding written")
                d.add(case + "/text", ct)
                d.add(case + "/image", ci)
            _attn_packed(d, D, dt, tag)


def _offsets(lengths):
    o = [0]
    for n in lengths:
        o.append(o[-1] + n)
    return o


def _attn_packed(d, D, dt, tag):
    """vb200_self_attention_packed and vb200_co_attention_packed over mixed lengths, each sample with its own edge mask."""
    import support
    import torch
    from oracle import kernel_refs as R
    P = len(R.EDGE_MASKS)
    H = HEADS * D
    ld = 3 * H + 8
    f16 = int(_f16(dt))
    dev = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    case = f"attn/self_packed_{tag}"
    lens = list(PACKED_L)
    offs = _offsets(lens)
    pats = [R.EDGE_MASKS[(3 * i + 1) % P] for i in range(len(lens))]
    g = torch.Generator(device="cuda").manual_seed(D + 5)
    qkv = torch.randn(offs[-1], ld, generator=g, device="cuda").to(dt)
    mask = torch.cat([R.edge_mask(p, L) for p, L in zip(pats, lens)]).cuda()
    ctx = torch.full((offs[-1] + 16, H + 8), NAN, dtype=dt, device="cuda")
    support.call("vb200_self_attention_packed", qkv, ld, H, mask, ctx, H + 8, len(lens), max(lens), HEADS, D, f16, dev(offs))
    torch.cuda.synchronize()
    for b, L in enumerate(lens):
        sl = slice(offs[b], offs[b + 1])
        q, k, v = _qkv_split(qkv[sl, :3 * H].view(1, L, 3 * H), H)
        _attn_check(f"{case} sample {b} (L = {L}, {pats[b]})", ctx[sl, :H].view(1, L, H), q, k, v, mask[sl].view(1, L), dt)
    require(_all_nan(ctx[offs[-1]:]) and _all_nan(ctx[:, H:]), case, "padding written")
    d.add(case, ctx)

    case = f"attn/co_packed_{tag}"
    T_l, V_l = [t for t, _ in CO_TV], [v for _, v in CO_TV]
    ot, ov = _offsets(T_l), _offsets(V_l)
    pt = [R.EDGE_MASKS[(3 * i) % P] for i in range(len(CO_TV))]
    pv = [R.EDGE_MASKS[(5 * i + 1) % P] for i in range(len(CO_TV))]
    g = torch.Generator(device="cuda").manual_seed(D + 9)
    qi = torch.randn(ov[-1], ld, generator=g, device="cuda").to(dt)
    qt = torch.randn(ot[-1], ld, generator=g, device="cuda").to(dt)
    mi = torch.cat([R.edge_mask(p, V) for p, V in zip(pv, V_l)]).cuda()
    mt = torch.cat([R.edge_mask(p, T) for p, T in zip(pt, T_l)]).cuda()
    ct = torch.full((ot[-1] + 16, H + 8), NAN, dtype=dt, device="cuda")
    ci = torch.full((ov[-1] + 16, H + 8), NAN, dtype=dt, device="cuda")
    support.call("vb200_co_attention_packed", qi, ld, qt, ld, H, mi, mt, ct, H + 8, ci, H + 8, len(CO_TV), max(T_l), max(V_l), HEADS,
                 D, f16, dev(ot), dev(ov))
    torch.cuda.synchronize()
    for b, (T, V) in enumerate(CO_TV):
        s_t, s_v = slice(ot[b], ot[b + 1]), slice(ov[b], ov[b + 1])
        xi, xt = _qkv_split(qi[s_v, :3 * H].view(1, V, 3 * H), H), _qkv_split(qt[s_t, :3 * H].view(1, T, 3 * H), H)
        what = f"{case} sample {b} (T = {T} {pt[b]}, V = {V} {pv[b]})"
        _attn_check(what + " text", ct[s_t, :H].view(1, T, H), xt[0], xi[1], xi[2], mi[s_v].view(1, V), dt)
        _attn_check(what + " image", ci[s_v, :H].view(1, V, H), xi[0], xt[1], xt[2], mt[s_t].view(1, T), dt)
    require(_all_nan(ct[ot[-1]:]) and _all_nan(ci[ov[-1]:]) and _all_nan(ct[:, H:]) and _all_nan(ci[:, H:]), case, "padding written")
    d.add(case + "/text", ct)
    d.add(case + "/image", ci)


# ============================================================================================================================= fwd
def _no_nan(case, obj):
    import torch
    if torch.is_tensor(obj):
        require(not torch.isnan(obj.float()).any(), case, "NaN in an output")
    elif isinstance(obj, (tuple, list)):
        for o in obj:
            _no_nan(case, o)
    elif isinstance(obj, dict):
        for o in obj.values():
            _no_nan(case, o)


def fwd(d):
    """The tiny engine (tests/conftest.py tiny_oracle's weights) in fp16, bf16 and fp32x: dense batch 2 (64-wide lone tiles) and dense
    batch 9 at Tin = 36 (333 text rows: 128-wide tiles) with debug taps, every attention map and every layer state; in fp16 and bf16
    also forward_packed at mixed lengths with every attention map and layer state; forward_regions_packed; a head-gated packed forward with fractional gates
    and decode_answers on its VQA logits.  Checked free of NaN; the digests carry the comparison."""
    import support
    import torch
    from oracle import vilbert_ref as VR
    from vilbert_b200 import _lib as L
    from vilbert_b200.model import head_mask_shape
    oracle = VR.build(VR.tiny_config(), seed=7, num_labels=200)
    for mode in ("fp16", "bf16", "fp32x"):
        model = support.engine(oracle, compute_dtype=mode, return_attention=True)
        try:
            for B, Tin, V in ((2, 30, 36), (9, 36, 36)):
                case = f"fwd/{mode}/dense_B{B}_T{Tin}_V{V}"
                inp = [t.cuda() for t in support.tiny_inputs(oracle, B, Tin, V, seed=B * 31, pad=3)]
                out = model(*inp, output_all_attention_masks=True, compute_pretraining_heads=True, debug_taps=True,
                            output_layer_states=True)
                torch.cuda.synchronize()
                _no_nan(case, out)
                d.add(case, out)
            if mode == "fp32x":                  # packed batches run in the 16-bit modes only
                continue
            lens = [(5, 10), (36, 36), (1, 1), (20, 50), (12, 3)]
            args = support.packed_sample_args(support.batch(model, lens, seed=400))
            case = f"fwd/{mode}/packed"
            out = model.forward_packed(*args, select=L.OUT_ALL, debug_taps=True, output_all_attention_masks=True,
                                       output_layer_states=True)
            torch.cuda.synchronize()
            _no_nan(case, out)
            d.add(case, out)
            F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
            imgs = [support.image(t, n, 500 + i, F, vocab) for i, (t, n) in enumerate([(7, 9), (30, 36), (2, 1), (18, 60)])]
            case = f"fwd/{mode}/regions_packed"
            out = model.forward_regions_packed(*support.packed_image_args(imgs), debug_taps=True, output_all_attention_masks=True)
            torch.cuda.synchronize()
            _no_nan(case, out)
            d.add(case, out)
            case = f"fwd/{mode}/gated_packed"
            E, Hm = head_mask_shape(model.config)
            gate = torch.rand(len(lens), E, Hm, generator=torch.Generator().manual_seed(3))
            out = model.forward_packed(*args, head_mask=gate, output_all_attention_masks=True)
            torch.cuda.synchronize()
            _no_nan(case, out)
            d.add(case, out)
            dec = model.decode_answers(out, [(1, k, 1, 5, None) for k in range(len(lens))])
            d.add(f"fwd/{mode}/decode", [(list(i), list(p), b) for i, p, b in dec])
        finally:
            model.close()


def full(d):
    """The full-size bf16 engine with the synthetic seed-42 checkpoint: dense batch 8 at Tin = 36 and 36 regions (296 text rows: the
    lone-tile path at real widths) and batch 16 (592 rows: 128-wide tiles); the task heads checked free of NaN and digested."""
    import torch
    import vilbert_b200 as vb
    from oracle import vilbert_ref as VR
    from vilbert_b200 import synthetic as S
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = vb.VILBertForVLTasks.from_pretrained(S.synthetic_state_dict(cfg, seed=42), config=cfg, num_labels=3129,
                                                 compute_dtype="bf16").eval().cuda(0)
    try:
        for B in (8, 16):
            case = f"full/dense_B{B}_T36_V36"
            out = model(*[t.cuda() for t in VR.make_inputs(B, 36, 36, seed=B)])
            torch.cuda.synchronize()
            _no_nan(case, out)
            d.add(case, out)
    finally:
        model.close()


# ============================================================================================================================ main
def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sections", default="gemm,ln,attn,fwd", help="comma-separated: " + ", ".join(SECTIONS))
    ap.add_argument("--out", required=True, help="JSON file for {output name: sha256}")
    args = ap.parse_args(argv)
    sections = [s for s in args.sections.split(",") if s]
    unknown = [s for s in sections if s not in SECTIONS]
    if unknown:
        ap.error(f"unknown sections {unknown}")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("switch_child.py needs an H100: every case runs a CUDA kernel")
    d = Digests()
    runs = {"gemm": (gemm_grid, gemm_engine, gemm_rows, gemm_split), "gemm_grid": (gemm_grid,), "gemm_rows": (gemm_rows,),
            "ln": (ln,), "attn": (attn,), "fwd": (fwd,), "full": (full,)}
    for s in sections:
        for fn in runs[s]:
            try:
                fn(d)
            except CaseFailed as e:
                print(f"switch_child: FAILED {e}", file=sys.stderr)
                return 1
            except Exception:
                traceback.print_exc()
                print(f"switch_child: FAILED in {fn.__name__} (section {s}) after {len(d)} outputs", file=sys.stderr)
                return 1
    with open(args.out, "w") as f:
        json.dump(d, f, indent=0, sort_keys=True)
    print(f"switch_child: {len(d)} outputs from {','.join(sections)}, S = {grid_slots()}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
