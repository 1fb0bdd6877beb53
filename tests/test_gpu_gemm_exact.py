"""Exact-value oracles for every GEMM entry point and an exhaustive sweep of the activation epilogues.  `-m gpu` only.

The GEMMs here run on exact-valued operands (oracle/kernel_refs.py exact_operands): integer products whose partial sums stay inside
fp32's 24-bit significand in any order, so the correct fp32 output is the fp64 product converted without rounding, whatever order a
kernel accumulates in.  Every check is bitwise: y32 == exact and y16 == sat_rn(exact).  A defect the two GEMM kernels share -- a
16-bit bias, an accumulator narrower than fp32, a wrong tensor map, a missing k-block -- changes bits here, where the comparisons of
the kernels with each other (tests/test_gpu_gemm_pingpong.py) cannot see it and the 2e-3 fp64 bounds of tests/test_gpu_ops.py are
about a thousand times too loose to.  Output buffers start NaN-filled; padding columns past N and tiles past a device row count
must keep the NaN.

The activation sweep feeds every finite fp16 and bf16 value through identity weights, so the accumulator holds the input exactly and
the epilogue's bias add, activation and 16-bit conversion are compared, value by value, with their references: pre = fp32(x + b), the
documented 4.3e-5 bound and saturation thresholds of gelu_erf, and its float32 restatement gelu_poly_f32."""
import pytest
import torch

from oracle import kernel_refs as R
import support

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
NAN = float("nan")


def _f16(dt):
    return dt == torch.float16


def _all_nan(t):
    return bool(torch.isnan(t.float()).all())


def _operands(M, N, K, dt, seed, ld_x=None, scale=R.EXACT_BUDGET_LOG2):
    return R.exact_operands(M, N, K, ld_x, _f16(dt), seed, scale, device="cuda")


def _buffers(M, N, dt, outs, ld16=None, ld32=None):
    """NaN-filled outputs with padding columns: ld16 = N rounded up to 8, plus 8; ld32 = N rounded up to 4, plus 4."""
    ld16 = ld16 or (N + 7) // 8 * 8 + 8
    ld32 = ld32 or (N + 3) // 4 * 4 + 4
    y16 = torch.full((M, ld16), NAN, dtype=dt, device="cuda") if "16" in outs else None
    y32 = torch.full((M, ld32), NAN, device="cuda") if "32" in outs else None
    return y16, ld16, y32, ld32


def _linear(x, w, b, M, N, K, dt, act=0, outs="16+32", variant=0, bn=0, pdl=0, sync=True, y16=None, ld16=None):
    if y16 is None:
        y16, ld16, y32, ld32 = _buffers(M, N, dt, outs)
    else:
        y32, ld32 = None, 0
    support.call("vb200_linear", x, x.stride(0), w, w.stride(0), b, None, 0, None, None, 1e-12, act, y16, ld16 if y16 is not None else 0,
                 y32, ld32 if y32 is not None else 0, M, N, K, bn, pdl, int(_f16(dt)), variant, None)
    if sync:
        torch.cuda.synchronize()
    return y16, y32


def _check(y16, y32, ref, N, dt, rows=None, what=""):
    """y32 == ref and y16 == sat_rn(ref) bit for bit on rows [0, rows); padding columns past N keep their NaN."""
    m = ref.shape[0] if rows is None else rows
    if y32 is not None:
        assert support.eq32(y32[:m, :N], ref[:m]), f"{what}: fp32 output differs from the exact result " \
            f"({int((y32[:m, :N] != ref[:m]).sum())} elements)"
        assert _all_nan(y32[:, N:]), f"{what}: fp32 padding columns written"
    if y16 is not None:
        assert support.eq16(y16[:m, :N], R.sat_rn(ref[:m], _f16(dt))), f"{what}: 16-bit output is not sat_rn(exact)"
        assert _all_nan(y16[:, N:]), f"{what}: 16-bit padding columns written"


# ================================================================================================================ the assumption
@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("variant", [0, 5])
def test_exact_accumulation_at_full_budget(dt, variant):
    """wgmma with 16-bit operands and fp32 accumulation sums integer products exactly while every partial sum stays below 2^24 units:
    element (0, 0) accumulates 3072 equal products monotonically to within a factor two of the builder's 2^22 budget (in quarter
    units, 2^24), the other rows span many binades down to +-1 operands."""
    M, N, K = 256, 256, 3072
    x, w, b = _operands(M, N, K, dt, seed=1)
    ref = R.exact_linear(x, w, b, 0)
    assert ref[0, 0].abs().item() >= 2.0 ** 21
    y16, y32 = _linear(x, w, b, M, N, K, dt, variant=variant, bn=128)
    _check(y16, y32, ref, N, dt, what=f"variant {variant}")


# ================================================================================================================ entry points
# (variant, block_n) for every width each vb200_linear variant accepts: 0 persistent (256 runs as 128), 2 / 3 the 128-wide persistent
# tile, 4 the 128- or 64-wide one, 5 ping-pong
LINEAR_CONFIGS = [(0, 64), (0, 128), (0, 192), (0, 256), (2, 128), (2, 256), (3, 128), (3, 256), (4, 64), (4, 128), (4, 256),
                  (5, 64), (5, 128)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("variant,bn", LINEAR_CONFIGS, ids=["v%d_bn%d" % c for c in LINEAR_CONFIGS])
def test_linear_exact(variant, bn, dt):
    """vb200_linear with fp32 output only, 16-bit output only (the TMA-store epilogue) and both, act 0 and ReLU; ragged M, strided A
    (ld_x = K + 8, NaN past K)."""
    M, N, K = 300, 384, 768
    x, w, b = _operands(M, N, K, dt, seed=variant * 1000 + bn, ld_x=K + 8)
    for act in (0, 2):
        ref = R.exact_linear(x, w, b, act)
        for outs in ("32", "16", "16+32"):
            y16, y32 = _linear(x, w, b, M, N, K, dt, act=act, outs=outs, variant=variant, bn=bn)
            _check(y16, y32, ref, N, dt, what=f"act {act} outputs {outs}")


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_linear_exact_without_bias(dt):
    M, N, K = 200, 256, 512
    x, w, _ = _operands(M, N, K, dt, seed=2)
    ref = R.exact_linear(x, w, None, 0)
    for variant in (0, 5):
        y16, y32 = _linear(x, w, None, M, N, K, dt, variant=variant)
        _check(y16, y32, ref, N, dt, what=f"variant {variant}")


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("m", [0, 1, 127, 128, 129, 1000])
@pytest.mark.parametrize("N,K", [(256, 192), (1601, 768)], ids=["pingpong", "coop_ragged_n"])
def test_linear_rows_exact(N, K, m, dt):
    """vb200_linear_rows at M = 1000 with m_rows = m, on the ping-pong kernel (N = 256) and the cooperative kernel's device row count
    (ragged N, PCfg MODE 6): rows < m are exact; tiles are skipped whole, so rows from the next 128-row boundary on keep the NaN."""
    M = 1000
    x, w, b = _operands(M, N, K, dt, seed=N + m)
    ref = R.exact_linear(x, w, b, 0)
    y16, ld16, y32, ld32 = _buffers(M, N, dt, "16+32")
    support.call("vb200_linear_rows", x, K, w, K, b, 0, y16, ld16, y32, ld32, M, N, K, 0, int(_f16(dt)),
                 torch.tensor([m], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    _check(y16, y32, ref, N, dt, rows=m, what=f"m_rows {m}")
    boundary = (m + 127) // 128 * 128
    assert _all_nan(y32[boundary:]) and _all_nan(y16[boundary:])


# (M, N, K, ld_x, ld_mul): the pooler at batch 8 and 64 (A = the first token of each sample, ld_x = T H), a ragged N with an ld_mul
# that is not a multiple of 4 (the scalar multiply), ragged M with ld_mul % 4 != 0
PRODUCT_CASES = [(8, 1024, 1024, 37 * 1024, 1024), (64, 1024, 1024, 101 * 1024, 1024), (64, 1000, 768, 776, 1003),
                 (200, 1024, 1024, 1088, 1027)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("case", PRODUCT_CASES, ids=lambda c: "M%d_N%d_K%d_ldx%d_ldmul%d" % c)
def test_linear_product_exact(case, dt):
    """vb200_linear_product: act(x w^T + b) * mul with mul powers of two and small integers -- the fp32 multiply is the kernel's only
    rounding after the exact GEMM --, act 0 and ReLU, both outputs and the 16-bit one alone (TMA store)."""
    M, N, K, ld_x, ld_mul = case
    x, w, b = _operands(M, N, K, dt, seed=M + N + ld_mul, ld_x=ld_x)
    g = torch.Generator().manual_seed(ld_mul)
    pow2 = torch.exp2(torch.randint(-6, 7, (M, ld_mul), generator=g).float())
    ints = torch.randint(-7, 8, (M, ld_mul), generator=g).float()
    mul = torch.where(torch.rand(M, ld_mul, generator=g) < 0.5, pow2, ints).cuda()
    for act in (0, 2):
        ref = R.exact_linear(x, w, b, act, mul[:, :N])
        for outs in ("16+32", "16"):
            y16, ld16, y32, ld32 = _buffers(M, N, dt, outs)
            support.call("vb200_linear_product", x, ld_x, w, K, b, act, mul, ld_mul, y16, ld16, y32, ld32 if y32 is not None else 0, M, N, K,
                         0, int(_f16(dt)))
            torch.cuda.synchronize()
            _check(y16, y32, ref, N, dt, what=f"act {act} outputs {outs}")


def _split_operands(M, N, K, seed):
    """fp32 operands of the fp32-parity GEMM whose fp16 lo parts are non-zero and whose three terms hi.hi + lo.hi + hi.lo are exact:
    x alternates odd integers in +-[2049, 3071] (fp16 spacing 2 there, so lo = +-1) on even k with small integers on odd k; w holds
    integers in [-3, 3] plus, per row, one odd integer in +-[2049, 4095] on an odd k (lo = +-1 against a small x).  Every element's sum
    of |terms| + |b| stays below 2^22 (quarter-unit biases)."""
    g = torch.Generator().manual_seed(seed)
    big = (torch.randint(1024, 1536, (M, K // 2), generator=g) * 2 + 1).double()
    big = big * (torch.randint(0, 2, (M, K // 2), generator=g) * 2 - 1)
    x = torch.randint(-15, 16, (M, K), generator=g).double()
    x[:, 0::2] = big
    w = torch.randint(-3, 4, (N, K), generator=g).double()
    kk = torch.randint(0, K // 2, (N,), generator=g) * 2 + 1
    w[torch.arange(N), kk] = ((torch.randint(1024, 2048, (N,), generator=g) * 2 + 1) * (torch.randint(0, 2, (N,), generator=g) * 2 - 1)).double()
    b = ((torch.randint(2048, 4096, (N,), generator=g) * 2 + 1) * R.BIAS_UNIT).float()
    return x.float(), w.float(), b


def _split_ref(x, w, b, act):
    """hi.hi + lo.hi + hi.lo + b in fp64 (the documented contraction; the lo.lo term is dropped), with hi = fp16(v) and
    lo = fp16(v - hi) taken from the fp32 operands themselves, not from the split layouts fed to the kernel; then act.  Exact for
    _split_operands."""
    xh, wh = x.half().double(), w.half().double()
    xl, wl = (x - x.half().float()).half().double(), (w - w.half().float()).half().double()
    lh, hl = xl @ wh.t(), xh @ wl.t()
    y = xh @ wh.t() + lh + hl + b.double()
    terms = xh.abs() @ wh.abs().t() + xl.abs() @ wh.abs().t() + xh.abs() @ wl.abs().t()
    assert (terms + b.double().abs()).max().item() < 2.0 ** R.EXACT_BUDGET_LOG2
    assert lh.abs().sum().item() > 0 and hl.abs().sum().item() > 0
    if act == 2:
        y = torch.relu(y)
    assert torch.equal(y.float().double(), y)
    return y.float()


@pytest.mark.parametrize("act", [0, 2])
@pytest.mark.parametrize("M,N,K", [(200, 384, 256), (77, 64, 128), (64, 3136, 512)])
def test_linear_split_exact(M, N, K, act):
    """vb200_linear_split (fp32x, fp16 hi | lo | hi activations against hi | hi | lo weights): the fp32 output equals the documented
    hi.hi + lo.hi + hi.lo + b exactly, on operands with non-zero lo parts in both, and the split 16-bit output is split16 of it."""
    x, w, b = _split_operands(M, N, K, seed=M + N + act)
    ref = _split_ref(x, w, b, act)
    x3, w3, b = R.split16(x).cuda(), R.split16_w(w).cuda(), b.cuda()
    y3 = torch.full((M, 3 * N + 64), NAN, dtype=torch.float16, device="cuda")
    y32 = torch.full((M, N + 4), NAN, device="cuda")
    support.call("vb200_linear_split", x3, 3 * K, w3, 3 * K, b, act, y3, 3 * N + 64, y32, N + 4, M, N, 3 * K)
    torch.cuda.synchronize()
    ref = ref.cuda()
    assert support.eq32(y32[:, :N], ref), int((y32[:, :N] != ref).sum())
    assert support.eq16(y3[:, :3 * N], R.split16(ref))
    assert _all_nan(y32[:, N:]) and _all_nan(y3[:, 3 * N:])


# ================================================================================================================ shapes
# Every distinct (M, N, K) GEMM of the 12/6/6 plan (30 tokens, 36 regions, task heads) at batch 1, 8, 64 and 512, from
# vb200_profile_ops after one forward of the full engine.  test_plan_gemms_match_engine keeps the list in step with the plan builder.
PLAN_BATCHES = (1, 8, 64, 512)
PLAN_GEMMS = [(1, 1024, 768), (1, 1024, 1024), (1, 1533, 2048), (1, 2048, 1024), (1, 3129, 2048), (4, 2048, 2048),
              (8, 1024, 768), (8, 1024, 1024), (8, 1533, 2048), (8, 2048, 1024), (8, 3129, 2048), (31, 768, 768),
              (31, 768, 1024), (31, 768, 3072), (31, 2304, 768), (31, 3072, 768), (32, 2048, 2048), (36, 1024, 1024),
              (36, 1024, 2112), (36, 3072, 1024), (64, 1024, 768), (64, 1024, 1024), (64, 1533, 2048), (64, 2048, 1024),
              (64, 3129, 2048), (248, 768, 768), (248, 768, 1024), (248, 768, 3072), (248, 2304, 768), (248, 3072, 768),
              (256, 2048, 2048), (288, 1024, 1024), (288, 1024, 2112), (288, 3072, 1024), (512, 1024, 768), (512, 1024, 1024),
              (512, 1533, 2048), (512, 2048, 1024), (512, 3129, 2048), (1984, 768, 768), (1984, 768, 1024), (1984, 768, 3072),
              (1984, 2304, 768), (1984, 3072, 768), (2304, 1024, 1024), (2304, 1024, 2112), (2304, 3072, 1024),
              (15872, 768, 768), (15872, 768, 1024), (15872, 768, 3072), (15872, 2304, 768), (15872, 3072, 768),
              (18432, 1024, 1024), (18432, 1024, 2112), (18432, 3072, 1024)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_plan_gemms_exact(dt):
    """Every plan GEMM shape on the cooperative kernel at its default tile width and, where it applies, the ping-pong kernel."""
    assert PLAN_GEMMS
    for i, (M, N, K) in enumerate(PLAN_GEMMS):
        x, w, b = _operands(M, N, K, dt, seed=i)
        ref = R.exact_linear(x, w, b, 0)
        variants = (0, 5) if N % (64 if N <= 64 else 128) == 0 else (0,)
        for variant in variants:
            y16, y32 = _linear(x, w, b, M, N, K, dt, variant=variant)
            _check(y16, y32, ref, N, dt, what=f"plan GEMM {(M, N, K)} variant {variant}")


def test_plan_gemms_match_engine(full_oracle, parity_log):
    import vilbert_b200 as vb
    from oracle import vilbert_ref as VR
    cfg = vb.BertConfig.from_dict(full_oracle.config.to_dict())
    model = vb.VILBertForVLTasks.from_pretrained(full_oracle.state_dict(), config=cfg, num_labels=full_oracle.num_labels,
                                                 compute_dtype="bf16").eval().cuda(0)
    try:
        shapes = set()
        for B in PLAN_BATCHES:
            inp = [t.cuda() for t in VR.make_inputs(B, 30, 36, seed=B)]
            model(*inp, select=vb.OUT_TASK_HEADS)
            torch.cuda.synchronize()
            shapes |= {tuple(o["dims"][:3]) for o in model.profile_ops(B, 30, 36, vb.OUT_TASK_HEADS, iters=1) if o["kind"] == "gemm"}
    finally:
        model.close()
    parity_log(test="plan_gemms", shapes=sorted(shapes))
    assert sorted(shapes) == sorted(PLAN_GEMMS), f"the plan's GEMMs changed; PLAN_GEMMS = {sorted(shapes)}"


EDGE_M = (1, 63, 64, 127, 128, 129, 1983)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("K", [64, 200, 2112, 3072])
@pytest.mark.parametrize("N", [64, 1000, 1601, 3129])
def test_edge_shapes_exact(N, K, dt):
    """M in {1, 63, 64, 127, 128, 129, 1983} for every N and K here (one k-block, a ragged last k-block, the image embedding's 2112,
    the FFN-out's 3072; a single 64-wide column tile, N % 128 != 0, the ragged 1601 / 3129 heads), strided A; variant 0 at its
    default width and, for N = 64, the ping-pong kernel too."""
    for M in EDGE_M:
        x, w, b = _operands(M, N, K, dt, seed=M * 7 + N + K, ld_x=K + 8)
        ref = R.exact_linear(x, w, b, 2 if M % 2 else 0)
        for variant in ((0, 5) if N == 64 else (0,)):
            y16, y32 = _linear(x, w, b, M, N, K, dt, act=2 if M % 2 else 0, variant=variant)
            _check(y16, y32, ref, N, dt, what=f"M {M} variant {variant}")


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_unaligned_fp32_output_exact(dt):
    """N = 1003 with an fp32 output of row stride 1003 (not a multiple of 4: the scalar store path), no 16-bit output."""
    M, N, K = 300, 1003, 768
    x, w, b = _operands(M, N, K, dt, seed=3)
    ref = R.exact_linear(x, w, b, 0)
    y32 = torch.full((M + 1, N), NAN, device="cuda")
    support.call("vb200_linear", x, K, w, K, b, None, 0, None, None, 1e-12, 0, None, 0, y32, N, M, N, K, 0, 0, int(_f16(dt)), 0, None)
    torch.cuda.synchronize()
    assert support.eq32(y32[:M], ref) and _all_nan(y32[M:])


# M = 128 x (tiles - 1) + 1 .. 128 x tiles, one column tile: 131 / 132 / 133 and 263 / 264 / 265 tiles against 132 SMs
TILE_COUNTS = [131, 132, 133, 263, 264, 265]


@pytest.mark.parametrize("variant,bn", [(0, 64), (0, 128), (5, 64), (5, 128)], ids=["v0_bn64", "v0_bn128", "v5_bn64", "v5_bn128"])
def test_tile_counts_exact(variant, bn):
    """Tile counts just below, at and above one and two waves of the 132 SMs; the last row tile is ragged (M = 128 tiles - 5)."""
    dt = torch.bfloat16 if bn == 64 else torch.float16
    N, K = bn, 64
    for tiles in TILE_COUNTS:
        M = 128 * tiles - 5
        x, w, b = _operands(M, N, K, dt, seed=tiles)
        ref = R.exact_linear(x, w, b, 0)
        y16, y32 = _linear(x, w, b, M, N, K, dt, variant=variant, bn=bn)
        _check(y16, y32, ref, N, dt, what=f"{tiles} tiles")


# ================================================================================================================ PDL chains
def _chain_operands(Ns, K, seed):
    """Integer weights with at most 8 non-zeros of +-1 per row and biases in [-3, 3]: from x in {-1, 0, 1} every intermediate stays
    below 8 (8 + 3) + 3 = 91 < 2^8, exact in bf16 and fp16."""
    g = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for N in Ns:
        w = torch.zeros(N, K)
        idx = torch.randint(0, K, (N, 8), generator=g)
        w.scatter_(1, idx, (torch.randint(0, 2, (N, 8), generator=g) * 2 - 1).float())
        ws.append(w)
        bs.append(torch.randint(-3, 4, (N,), generator=g).float())
        K = N
    return ws, bs


def _chain_ref(x, ws, bs, acts, limit):
    """The fp64 chain; every intermediate (stored in 16 bits by the kernels) must be an integer below `limit`."""
    y = x.double()
    for i, (w, b, act) in enumerate(zip(ws, bs, acts)):
        if i:
            assert y.abs().max().item() < limit
        y = y @ w.double().t() + b.double()
        if act == 2:
            y = torch.relu(y)
    return y.float()


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_coop_pdl_chain_exact(dt):
    """The cooperative three-launch chain of test_coop_plain_gemm_pdl_chain (N = 768 16-bit, ragged N = 1000 16-bit, N = 3129 both
    outputs; no synchronize in between) under PDL modes 0, 1 and 5, on integer data: every intermediate 16-bit store is exact, so
    the final output must equal the fp64 chain, not only agree across modes."""
    M, K = 1984, 768
    acts = (0, 2, 0)
    ws, bs = _chain_operands((768, 1000, 3129), K, seed=31)
    g = torch.Generator().manual_seed(30)
    x = torch.randint(-1, 2, (M, K), generator=g).float()
    ref = _chain_ref(x, ws, bs, acts, 2 ** 8).cuda()
    x, ws, bs = x.to(dt).cuda(), [w.to(dt).cuda() for w in ws], [b.cuda() for b in bs]
    for pdl in (0, 1, 5):
        y1 = torch.full((M, 768), NAN, dtype=dt, device="cuda")
        y2 = torch.full((M, 1000), NAN, dtype=dt, device="cuda")
        _linear(x, ws[0], bs[0], M, 768, K, dt, act=acts[0], pdl=pdl, sync=False, y16=y1, ld16=768)
        _linear(y1, ws[1], bs[1], M, 1000, 768, dt, act=acts[1], pdl=pdl, sync=False, y16=y2, ld16=1000)
        y3b, y3 = _linear(y2, ws[2], bs[2], M, 3129, 1000, dt, act=acts[2], pdl=pdl, sync=False)
        torch.cuda.synchronize()
        _check(y3b, y3, ref, 3129, dt, what=f"pdl {pdl}")


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_pingpong_pdl_chain_exact(dt):
    """The ping-pong chain of test_pingpong_pdl_chain (three N = 768 launches, 64-wide tiles, 16-bit outputs) under PDL modes 0 and 5
    on integer data: the final 16-bit output equals sat_rn of the fp64 chain."""
    M, K = 1984, 768
    acts = (2, 0, 2)
    ws, bs = _chain_operands((768, 768, 768), K, seed=20)
    g = torch.Generator().manual_seed(11)
    x = torch.randint(-1, 2, (M, K), generator=g).float()
    ref = _chain_ref(x, ws, bs, acts, 2 ** 8).cuda()
    x, ws, bs = x.to(dt).cuda(), [w.to(dt).cuda() for w in ws], [b.cuda() for b in bs]
    for pdl in (0, 5):
        cur = x
        for w, b, act in zip(ws, bs, acts):
            y = torch.full((M, 768), NAN, dtype=dt, device="cuda")
            _linear(cur, w, b, M, 768, K, dt, act=act, variant=5, bn=64, pdl=pdl, sync=False, y16=y, ld16=768)
            cur = y
        torch.cuda.synchronize()
        assert support.eq16(cur, R.sat_rn(ref, _f16(dt))), f"pdl {pdl}"


# ================================================================================================================ activation sweep
def _every_16bit_value(dt):
    """Every finite fp16 / bf16 value, in bit order, zero-padded to a [256, 256] operand (65536 slots)."""
    u = torch.arange(1 << 16, dtype=torch.int32).to(torch.int16).view(dt)
    v = u[torch.isfinite(u.float())]
    a = torch.zeros(1 << 16, dtype=dt)
    a[:len(v)] = v
    return a.view(256, 256), len(v)


def _sweep_biases():
    """Per-column fp32 biases over many binades: zero, +-2^-24 .. +-2^9 scaled normals, and a few exact small integers."""
    g = torch.Generator().manual_seed(12)
    b = torch.randn(256, generator=g) * torch.exp2(torch.randint(-24, 10, (256,), generator=g).float())
    b[0] = 0.0
    b[1:9] = torch.tensor([1.0, -1.0, 0.5, -0.5, 3.0, -3.0, 4.25, -4.25])
    return b


def _ulp_distance(a, b):
    """|a - b| in fp32 units in the last place (finite values; +0 and -0 are the same point)."""
    def key(t):
        i = t.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


SWEEP_CONFIGS = [(0, 64), (0, 128), (5, 64), (5, 128)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("variant,bn", SWEEP_CONFIGS, ids=["v%d_bn%d" % c for c in SWEEP_CONFIGS])
def test_activation_epilogue_every_16bit_input(variant, bn, dt, parity_log):
    """Identity weights (K = N = M = 256) with every finite fp16 / bf16 value in the A rows, so that the accumulator is the input
    exactly; bias 0, then varied fp32 biases with pre = fp32(x + b), the kernel's one fp32 add.
      act 0: y32 == pre bit for bit.  act 2: y32 == max(pre, 0) by value.
      act 1: |y32 - GELU(pre)| <= 4.3e-5; -0 below GELU_ZERO_BELOW and pre itself above GELU_IDENTITY_ABOVE; no NaN or inf anywhere,
             +-65504 and +-3.39e38 included; within one fp32 ulp of gelu_poly_f32 (its emulated FMAs can double-round in rare ties).
      every act: the 16-bit output is sat_rn(y32).
    Subnormal inputs stay in the sweep: wgmma passes fp16 and bf16 subnormals through exactly (measured on an H100), so act 0 is
    bitwise on them too."""
    f16 = _f16(dt)
    a, n = _every_16bit_value(dt)
    x = a.cuda()
    w = torch.eye(256, dtype=dt, device="cuda")
    worst = 0.0
    for bias in (torch.zeros(256), _sweep_biases()):
        b = bias.cuda()
        pre = x.float() + b                                     # torch fp32: one rounding, as the kernel's
        for act in (0, 2, 1):
            y16, y32 = _linear(x, w, b, 256, 256, 256, dt, act=act, variant=variant, bn=bn)
            y16, y32 = y16[:, :256], y32[:, :256]
            assert support.eq16(y16, R.sat_rn(y32, f16)), act
            assert bool(torch.isfinite(y32).all()), act
            if act == 0:
                sub = (x.float().abs() < (2.0 ** -14 if f16 else 2.0 ** -126)) & (x.float() != 0)
                bad = y32.view(torch.int32) != pre.view(torch.int32)
                assert not bool(bad.any()), f"{int(bad.sum())} differ, {int((bad & sub).sum())} of them at subnormal inputs"
            elif act == 2:
                assert torch.equal(y32, pre.clamp(min=0.0))
            else:
                err = (y32.double() - R.gelu_fp64(pre.double())).abs()
                worst = max(worst, err.max().item())
                assert err.max().item() <= R.GELU_BOUND, err.max().item()
                lo, hi = pre < R.GELU_ZERO_BELOW, pre > R.GELU_IDENTITY_ABOVE
                assert bool((y32[lo] == 0).all()) and support.eq32(y32[hi], pre[hi])
                emu = torch.from_numpy(R.gelu_poly_f32(pre.cpu().numpy())).cuda()
                assert _ulp_distance(y32, emu).max().item() <= 1
    parity_log(test="gemm_exact_gelu_sweep", dtype=str(dt), variant=variant, block_n=bn, values=n, max_abs_err=worst, bound=R.GELU_BOUND)


# The act-3 GELU (gelu_erf_as: A&S erf with __fdividef and exp2f, fp32-parity mode) over this sweep, measured on one H100 80GB HBM3
# (700 W power limit) before the bound was set: max |y - GELU(pre)| = 4.54e-7.  The A&S form evaluated in fp64 is within 2.1e-7 of
# GELU on [-12, 12]; the rest is fp32 evaluation.  The bound is just under twice the measurement.
ACT3_BOUND = 9.0e-7
# Against the same A&S formula evaluated in fp64 (kernel_refs.gelu_as_fp64) on |pre| <= 2, where a coefficient error of the erf
# polynomial shows most (1.061405429 -> 1.0614 moves the output by 7.6e-7 near |x| = 0.6): a float32 emulation of the kernel's
# evaluation order on the CPU differs by 1.36e-7 there, the H100 (same card) by 1.41e-7; the bound is just under twice that.
ACT3_FORM_BOUND = 2.8e-7


def test_act3_gelu_every_fp16_input(parity_log):
    """vb200_linear_split with identity weights in the split layout (hi | hi | lo = I | I | 0) and every finite fp16 value as the hi
    part of the activations (lo = 0): the accumulator is the input exactly, and the A&S-erf GELU of pre = fp32(x + b) (bias 0, then
    varied biases) is within ACT3_BOUND = 9.0e-7 of fp64 GELU (measured on an H100: 4.54e-7) and, on |pre| <= 2, within
    ACT3_FORM_BOUND = 2.8e-7 of its own formula in fp64 (measured: 1.41e-7); no NaN or inf, and the split 16-bit output is split16
    of the fp32 one."""
    a, n = _every_16bit_value(torch.float16)
    x3 = R.split16(a.float()).cuda()
    w3 = R.split16_w(torch.eye(256)).cuda()
    worst = form = 0.0
    for bias in (torch.zeros(256), _sweep_biases()):
        b = bias.cuda()
        pre = a.float().cuda() + b
        y3 = torch.full((256, 768), NAN, dtype=torch.float16, device="cuda")
        y32 = torch.full((256, 256), NAN, device="cuda")
        support.call("vb200_linear_split", x3, 768, w3, 768, b, 3, y3, 768, y32, 256, 256, 256, 768)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(y32).all())
        assert support.eq16(y3, R.split16(y32))
        err = (y32.double() - R.gelu_fp64(pre.double())).abs()
        worst = max(worst, err.max().item())
        near = pre.abs() <= 2.0
        form = max(form, (y32.double() - R.gelu_as_fp64(pre.double())).abs()[near].max().item())
    parity_log(test="gemm_exact_act3_sweep", values=n, max_abs_err=worst, bound=ACT3_BOUND, max_abs_err_vs_formula=form,
               formula_bound=ACT3_FORM_BOUND)
    assert worst <= ACT3_BOUND, worst
    assert form <= ACT3_FORM_BOUND, form


# ================================================================================================================ narrow heads
@pytest.mark.parametrize("add,bias", [(True, True), (False, False), (True, False), (False, True)], ids=["add_bias", "plain", "add", "bias"])
@pytest.mark.parametrize("K", [768, 1024, 2048])
@pytest.mark.parametrize("n_out", [1, 2, 3, 4])
def test_rowdot_exact(n_out, K, add, bias):
    """vb200_rowdot accumulates in fp32 on CUDA cores: on integer x in [-63, 63] and w in [-31, 31], quarter-unit biases and an
    additive mask of -10000 plus small integers, every partial sum is exact and out == the fp64 result bit for bit.  M = 37, strided
    x (NaN past K), ld_out 6 (columns past n_out keep the NaN)."""
    M, ld_x, ld_out = 37, K + 4, 6
    g = torch.Generator().manual_seed(n_out * K + 2 * add + bias)
    x = torch.full((M, ld_x), NAN)
    x[:, :K] = torch.randint(-63, 64, (M, K), generator=g).float()
    x[0, :K] = 63.0
    w = torch.randint(-31, 32, (n_out, K), generator=g).float()
    w[0] = 31.0
    b = ((torch.randint(-4096, 4096, (n_out,), generator=g) * 2 + 1) * R.BIAS_UNIT).float() if bias else None
    a = None
    if add:
        a = torch.randint(-50, 51, (M,), generator=g).float()
        a[::3] = -10000.0
    ref = x[:, :K].double() @ w.double().t()
    scale = x[:, :K].double().abs() @ w.double().abs().t()
    if b is not None:
        ref, scale = ref + b.double(), scale + b.double().abs()
    if a is not None:
        ref, scale = ref + a.double()[:, None], scale + a.double().abs()[:, None]
    assert scale.max().item() < 2.0 ** R.EXACT_BUDGET_LOG2 and scale.max().item() > 2.0 ** 20
    out = torch.full((M, ld_out), NAN, device="cuda")
    support.call("vb200_rowdot", x.cuda(), ld_x, w.cuda(), b.cuda() if b is not None else None, a.cuda() if a is not None else None, out,
                 ld_out, M, K, n_out, None)
    torch.cuda.synchronize()
    assert support.eq32(out[:, :n_out], ref.float().cuda())
    assert _all_nan(out[:, n_out:])
