"""Op-level parity for every kernel the engine launches, against plain high-precision or bit-exact references (oracle/kernel_refs.py):
text embeddings, image / region packs, narrow heads, state gathers, packed self- and co-attention, the pooled-product GEMM, the
cooperative GEMM's device row count, exact 16-bit rounding on every GEMM store path and a dependent chain of cooperative GEMMs under
programmatic dependent launch.  `-m gpu` only.

Output buffers start out filled with a sentinel (NaN, or a marker value) so that a write outside a kernel's contract shows up.  Where
a kernel writes an fp32 value and its 16-bit copy, the 16-bit bits must equal sat_rn(fp32): fp16 clamps to +-65504 and rounds to
nearest even, bf16 rounds to nearest even."""
import math

import numpy as np
import pytest
import torch

from oracle import kernel_refs as R
import support

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
NAN = float("nan")


def _is_nan(t):
    return bool(torch.isnan(t.float()).all())


def _f16(dt):
    return 1 if dt == torch.float16 else 0


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _offs(lengths):
    return [0] + list(np.cumsum(lengths).astype(int))


def _dev_i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


# ================================================================================================================ text embeddings
class _Tables:
    def __init__(self, H, seed=0, vocab=50, max_pos=40, n_type=2, n_task=6):
        g = _gen(seed)
        self.H, self.vocab, self.max_pos, self.n_type, self.n_task = H, vocab, max_pos, n_type, n_task
        self.word = torch.randn(vocab, H, generator=g, device="cuda")
        self.pos = torch.randn(max_pos, H, generator=g, device="cuda") * 0.5
        self.type = torch.randn(n_type, H, generator=g, device="cuda") * 0.5
        self.task = torch.randn(n_task, H, generator=g, device="cuda")
        self.gamma = 1.0 + 0.1 * torch.randn(H, generator=g, device="cuda")
        self.beta = 0.1 * torch.randn(H, generator=g, device="cuda")

    def run(self, ids, seg, imask, task, B, Tin, tt, f16, split16=0, offs=None, rows=0, extra=3):
        n = rows if offs is not None else B * (Tin + tt)
        out = torch.full((n + extra, self.H), NAN, device="cuda")
        o16 = torch.full((n + extra, 3 * self.H if split16 else self.H), NAN, device="cuda",
                         dtype=torch.float16 if f16 else torch.bfloat16)
        mask = torch.full((n + extra,), NAN, device="cuda")
        support.call("vb200_text_embed", ids, seg, imask, task, self.word, self.pos, self.type, self.task,
                     self.gamma, self.beta, 1e-12, out, o16, mask, B, Tin, self.H, self.vocab, self.max_pos, self.n_type,
                     self.n_task, tt, f16, split16, offs, rows)
        torch.cuda.synchronize()
        return out, o16, mask, n

    def ref(self, ids_list, seg_list, task_list, tt):
        """fp64: LayerNorm(word + position + type) per output row, the task row at index 1; clamped ids / types / task ids and
        positions (embed_heads.cu text_embed_kernel)."""
        clamp = lambda v, n: min(max(int(v), 0), n - 1)
        wi, pi, si, ti, is_task = [], [], [], [], []
        for ids_b, seg_b, task_b in zip(ids_list, seg_list, task_list):
            for t in range(len(ids_b) + tt):
                task_row = bool(tt) and t == 1
                src = t - 1 if (tt and t >= 2) else t
                is_task.append(task_row)
                ti.append(clamp(task_b, self.n_task))
                wi.append(0 if task_row else clamp(ids_b[src], self.vocab))
                si.append(0 if task_row else clamp(seg_b[src], self.n_type))
                pi.append(0 if task_row else min(src, self.max_pos - 1))
        ix = lambda v: torch.tensor(v, device="cuda")
        x = self.word.double()[ix(wi)] + self.pos.double()[ix(pi)] + self.type.double()[ix(si)]
        x = torch.where(ix(is_task)[:, None], self.task.double()[ix(ti)], x)
        u = x.mean(-1, keepdim=True)
        var = (x - u).pow(2).mean(-1, keepdim=True)
        return (x - u) / torch.sqrt(var + 1e-12) * self.gamma.double() + self.beta.double()


def _text_inputs(B, Tin, tb, seed, out_of_range=False):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, tb.vocab, (B, Tin), generator=g)
    seg = torch.randint(0, 2, (B, Tin), generator=g)                        # token types 0 and 1
    task = torch.randint(0, tb.n_task, (B,), generator=g)
    imask = torch.zeros(B, Tin, dtype=torch.long)
    for b in range(B):
        imask[b, :max(1, Tin - 3 * b)] = 1                                  # per-sample padding
    if out_of_range:
        ids.view(-1)[::3] = torch.tensor([-3, tb.vocab, tb.vocab + 7])[torch.arange(ids.numel())[::3] % 3]
        seg.view(-1)[1::4] = torch.tensor([-1, 2, 5])[torch.arange(seg.numel())[1::4] % 3]
        task[:] = torch.tensor([-2, tb.n_task, tb.n_task + 3, 1, 0])[torch.arange(B) % 5]
    return ids, seg, imask, task


def _mask_ref(imask, tt):
    B, Tin = imask.shape
    m = torch.cat([torch.ones(B, 1, dtype=torch.long), imask], dim=1) if tt else imask
    return ((1.0 - m.float()) * -10000.0).reshape(-1)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("tt", [1, 0], ids=["task_tokens", "no_task_tokens"])
@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("Tin", [1, 2, 37])
@pytest.mark.parametrize("H", [128, 768, 1024])
def test_text_embed_dense(H, Tin, B, tt, dt, parity_log):
    tb = _Tables(H, seed=H + Tin)
    ids, seg, imask, task = _text_inputs(B, Tin, tb, seed=B * 100 + Tin)
    out, o16, mask, n = tb.run(ids.cuda(), seg.cuda(), imask.cuda(), task.cuda(), B, Tin, tt, _f16(dt))
    ref = tb.ref(ids.tolist(), seg.tolist(), task.tolist(), tt)
    err = (out[:n].double() - ref).abs().max().item()
    parity_log(test="kp_text_embed", H=H, Tin=Tin, B=B, tt=tt, dtype=str(dt), max_abs_err=err, bound=1e-5)
    assert err < 1e-5, err
    assert support.eq16(o16[:n], R.sat_rn(out[:n], dt == torch.float16))
    assert torch.equal(mask[:n].cpu(), _mask_ref(imask, tt))
    assert _is_nan(out[n:]) and _is_nan(o16[n:]) and _is_nan(mask[n:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("Tin", [40, 41], ids=["Tin_max_pos", "Tin_past_max_pos"])
def test_text_embed_clamping(Tin, dt, parity_log):
    """Out-of-range token ids, token types and task ids are clamped into their tables, positions past max_pos - 1 to the last one
    (max_pos = 40 here), as documented in vilbert_b200.h."""
    tb = _Tables(768, seed=Tin)
    B = 5
    ids, seg, imask, task = _text_inputs(B, Tin, tb, seed=Tin, out_of_range=True)
    for tt in (1, 0):
        out, o16, mask, n = tb.run(ids.cuda(), seg.cuda(), imask.cuda(), task.cuda(), B, Tin, tt, _f16(dt))
        ref = tb.ref(ids.tolist(), seg.tolist(), task.tolist(), tt)
        err = (out[:n].double() - ref).abs().max().item()
        parity_log(test="kp_text_embed_clamp", Tin=Tin, tt=tt, dtype=str(dt), max_abs_err=err, bound=1e-5)
        assert err < 1e-5, err
        assert support.eq16(o16[:n], R.sat_rn(out[:n], dt == torch.float16))
        assert torch.equal(mask[:n].cpu(), _mask_ref(imask, tt))


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("tt", [1, 0], ids=["task_tokens", "no_task_tokens"])
@pytest.mark.parametrize("H", [128, 768, 1024])
def test_text_embed_packed(H, tt, dt, parity_log):
    """Packed batch: every sample's rows equal a dense call of that sample alone, bit for bit; every row is real (mask 0); rows past
    offs[B] keep the sentinel."""
    tb = _Tables(H, seed=7 * H)
    lens = [1, 2, 37, 5, 16]
    g = torch.Generator().manual_seed(H)
    ids_l = [torch.randint(0, tb.vocab, (n,), generator=g) for n in lens]
    seg_l = [torch.randint(0, 2, (n,), generator=g) for n in lens]
    task = torch.randint(0, tb.n_task, (len(lens),), generator=g)
    offs = _offs([n + tt for n in lens])
    out, o16, mask, n = tb.run(torch.cat(ids_l).cuda(), torch.cat(seg_l).cuda(), None, task.cuda(), len(lens), 0, tt, _f16(dt),
                               offs=_dev_i32(offs), rows=offs[-1])
    ref = tb.ref([t.tolist() for t in ids_l], [t.tolist() for t in seg_l], task.tolist(), tt)
    err = (out[:n].double() - ref).abs().max().item()
    parity_log(test="kp_text_embed_packed", H=H, tt=tt, dtype=str(dt), max_abs_err=err, bound=1e-5)
    assert err < 1e-5, err
    assert _is_nan(out[n:]) and _is_nan(o16[n:]) and _is_nan(mask[n:])
    assert bool((mask[:n] == 0).all())
    for b, Tin in enumerate(lens):
        d_out, d16, d_mask, dn = tb.run(ids_l[b].view(1, -1).cuda(), seg_l[b].view(1, -1).cuda(),
                                        torch.ones(1, Tin, dtype=torch.long, device="cuda"), task[b:b + 1].cuda(), 1, Tin, tt, _f16(dt))
        sl = slice(offs[b], offs[b + 1])
        assert support.eq32(out[sl], d_out[:dn]) and support.eq16(o16[sl], d16[:dn]) and torch.equal(mask[sl], d_mask[:dn]), b


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_text_embed_split16(packed):
    """fp32-parity mode: the 16-bit output is fp16 hi | lo | hi per 64 columns with hi = sat_rn_fp16(x), lo = rn_fp16(x - hi)."""
    tb = _Tables(768, seed=3)
    B, Tin = 3, 19
    ids, seg, imask, task = _text_inputs(B, Tin, tb, seed=3)
    if packed:
        offs = [0, 20, 40, 60]
        out, o16, _, n = tb.run(ids.view(-1).cuda(), seg.view(-1).cuda(), None, task.cuda(), B, 0, 1, 1, split16=1,
                                offs=_dev_i32(offs), rows=60)
    else:
        out, o16, _, n = tb.run(ids.cuda(), seg.cuda(), imask.cuda(), task.cuda(), B, Tin, 1, 1, split16=1)
    assert support.eq16(o16[:n], R.split16(out[:n]))
    assert _is_nan(o16[n:])


# ================================================================================================================ image pack
def _feats(rows, F, seed, big=True):
    g = _gen(seed)
    f = torch.randn(rows, F, generator=g, device="cuda") * 3.0
    if big:                                                  # above the fp16 range: the fp16 operand must saturate
        f[0, :6] = torch.tensor([7e4, -1e5, 65504.0, 65519.0, 65520.0, -65520.0])
        f[1::5, 3] = 1e6
    return f


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("with_mask", [True, False], ids=["image_mask", "no_mask"])
@pytest.mark.parametrize("F,Kp", [(2048, 2056), (2048, 2112), (40, 48), (40, 128)])
def test_image_pack(F, Kp, with_mask, dt):
    """[feat | loc | 0 ...] in the 16-bit format, bit for bit; additive mask from image_mask (NULL: every row real)."""
    rows = 37
    feats = _feats(rows, F, seed=F + Kp)
    loc = torch.rand(rows, 5, generator=_gen(1), device="cuda")
    im = (torch.arange(rows, device="cuda") % 4 != 3).to(torch.uint8) if with_mask else None
    a = torch.full((rows + 2, Kp), NAN, dtype=dt, device="cuda")
    mask = torch.full((rows + 2,), NAN, device="cuda")
    support.call("vb200_image_pack", feats, loc, im, a, mask, rows, F, Kp, _f16(dt), 0)
    torch.cuda.synchronize()
    ref = torch.from_numpy(R.operand_rows(feats.cpu().numpy(), loc.cpu().numpy(), Kp)).cuda()
    assert support.eq16(a[:rows], R.sat_rn(ref, dt == torch.float16))
    want = (1.0 - im.float()) * -10000.0 if with_mask else torch.zeros(rows, device="cuda")
    assert torch.equal(mask[:rows], want)
    assert _is_nan(a[rows:]) and _is_nan(mask[rows:])


@pytest.mark.parametrize("F,Kp", [(2048, 2112), (40, 64)])
def test_image_pack_split16(F, Kp):
    rows = 21
    feats = _feats(rows, F, seed=F)
    loc = torch.rand(rows, 5, generator=_gen(2), device="cuda")
    a = torch.full((rows + 1, 3 * Kp), NAN, dtype=torch.float16, device="cuda")
    mask = torch.full((rows + 1,), NAN, device="cuda")
    support.call("vb200_image_pack", feats, loc, None, a, mask, rows, F, Kp, 1, 1)
    torch.cuda.synchronize()
    ref = torch.from_numpy(R.operand_rows(feats.cpu().numpy(), loc.cpu().numpy(), Kp)).cuda()
    assert support.eq16(a[:rows], R.split16(ref)) and _is_nan(a[rows:])


# ================================================================================================================ region pack
def _detector(B, n, F, seed):
    """Detector-like output: non-negative box features over several magnitudes (so the order of the mean's sum matters), pixel boxes
    inside differently sized images."""
    g = np.random.default_rng(seed)
    feats = (g.random((B, n, F), dtype=np.float32) * g.choice(np.array([0.01, 1.0, 300.0], dtype=np.float32), size=(B, n, F)))
    wh = np.stack([g.integers(200, 1000, B), g.integers(150, 800, B)], axis=1).astype(np.float32)
    x1 = (g.random((B, n)) * wh[:, :1] * 0.6).astype(np.float32).round()
    y1 = (g.random((B, n)) * wh[:, 1:] * 0.6).astype(np.float32).round()
    x2 = x1 + 1 + (g.random((B, n)) * wh[:, :1] * 0.39).round()
    y2 = y1 + 1 + (g.random((B, n)) * wh[:, 1:] * 0.39).round()
    boxes = np.stack([x1, y1, x2, y2], axis=-1).astype(np.float32)
    return feats.astype(np.float32), boxes, wh


class _Tok:
    def encode(self, s):
        return [5]

    def add_special_tokens_single_sentence(self, ids):
        return [2] + ids + [3]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("num_boxes", [True, False], ids=["num_boxes", "all_boxes"])
@pytest.mark.parametrize("F,Kp", [(2048, 2112), (40, 48)])
def test_region_pack_dense(F, Kp, num_boxes, dt):
    """Bit for bit against the float32 restatement (oracle/kernel_refs.region_rows): num_boxes {n, n - 3, 1, 0} -- nb = 0 gives a
    zero mean row with every box masked; padded boxes are zero rows with a -10000 mask.  Images with every box valid also match the
    host input builder (worker_api.build_inputs): box rows and spatials exactly, the mean row within one unit in the last place."""
    from vilbert_b200 import worker_api as W
    B, n = 4, 36
    feats, boxes, wh = _detector(B, n, F, seed=F)
    nbs = [n, n - 3, 1, 0] if num_boxes else [n] * B
    R_ = B * (n + 1)
    a = torch.full((R_ + 2, Kp), NAN, dtype=dt, device="cuda")
    mask = torch.full((R_ + 2,), NAN, device="cuda")
    sp = torch.full((R_ + 2, 5), NAN, device="cuda")
    nb_t = _dev_i32(nbs) if num_boxes else None
    support.call("vb200_region_pack", torch.from_numpy(feats).cuda(), torch.from_numpy(boxes).cuda(), torch.from_numpy(wh).cuda(),
                 nb_t, a, mask, sp, B, n, F, Kp, _f16(dt), 0, None)
    torch.cuda.synchronize()
    f16 = dt == torch.float16
    assert _is_nan(a[R_:]) and _is_nan(mask[R_:]) and _is_nan(sp[R_:])
    for b in range(B):
        rows, loc, real = R.region_rows(feats[b], boxes[b], wh[b, 0], wh[b, 1], nbs[b])
        sl = slice(b * (n + 1), (b + 1) * (n + 1))
        ref = torch.from_numpy(R.operand_rows(rows, loc, Kp)).cuda()
        assert support.eq16(a[sl], R.sat_rn(ref, f16)), b
        assert support.eq32(sp[sl], torch.from_numpy(loc).cuda()), b
        assert torch.equal(mask[sl].cpu(), torch.from_numpy(np.where(real, 0.0, -10000.0).astype(np.float32))), b
        if nbs[b] == n:
            info = {"image_width": float(wh[b, 0]), "image_height": float(wh[b, 1]), "bbox": boxes[b]}
            _, f_bi, s_bi, *_ = W.build_inputs("q", [1], [torch.from_numpy(feats[b])], [info], torch.device("cpu"), _Tok())
            got = a[sl][:, :F]
            assert support.eq16(got[1:], R.sat_rn(f_bi[0, 1:].cuda(), f16))
            assert support.eq32(sp[sl], s_bi[0].cuda())
            d = (got[0].view(torch.int16).int() - R.sat_rn(f_bi[0, 0].cuda(), f16).view(torch.int16).int()).abs()
            assert int(d.max()) <= 1


def test_region_pack_split16():
    B, n, F, Kp = 2, 10, 2048, 2112
    feats, boxes, wh = _detector(B, n, F, seed=5)
    R_ = B * (n + 1)
    a = torch.full((R_, 3 * Kp), NAN, dtype=torch.float16, device="cuda")
    mask = torch.full((R_,), NAN, device="cuda")
    support.call("vb200_region_pack", torch.from_numpy(feats).cuda(), torch.from_numpy(boxes).cuda(), torch.from_numpy(wh).cuda(),
                 _dev_i32([n, 4]), a, mask, None, B, n, F, Kp, 1, 1, None)
    torch.cuda.synchronize()
    for b, nb in enumerate([n, 4]):
        rows, loc, _ = R.region_rows(feats[b], boxes[b], wh[b, 0], wh[b, 1], nb)
        ref = torch.from_numpy(R.operand_rows(rows, loc, Kp)).cuda()
        assert support.eq16(a[b * (n + 1):(b + 1) * (n + 1)], R.split16(ref)), b


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("F,Kp", [(2048, 2112), (40, 48)])
def test_region_pack_packed(F, Kp, dt):
    """Packed detector output with box counts {1, 2, 36, 100}: bit for bit against the restatement; every row real; rows past
    offs[B] keep the sentinel."""
    counts = [1, 2, 36, 100]
    B = len(counts)
    g = np.random.default_rng(F)
    per = [_detector(1, c, F, seed=int(g.integers(1 << 30))) for c in counts]
    feats = np.concatenate([p[0][0] for p in per])
    boxes = np.concatenate([p[1][0] for p in per])
    wh = np.concatenate([p[2] for p in per])
    offs = _offs([c + 1 for c in counts])
    R_ = offs[-1]
    a = torch.full((R_ + 3, Kp), NAN, dtype=dt, device="cuda")
    mask = torch.full((R_ + 3,), NAN, device="cuda")
    sp = torch.full((R_ + 3, 5), NAN, device="cuda")
    support.call("vb200_region_pack", torch.from_numpy(feats).cuda(), torch.from_numpy(boxes).cuda(), torch.from_numpy(wh).cuda(),
                 None, a, mask, sp, B, 0, F, Kp, _f16(dt), 0, _dev_i32(offs))
    torch.cuda.synchronize()
    assert _is_nan(a[R_:]) and _is_nan(mask[R_:]) and _is_nan(sp[R_:])
    assert bool((mask[:R_] == 0).all())
    for b, c in enumerate(counts):
        rows, loc, _ = R.region_rows(per[b][0][0], per[b][1][0], wh[b, 0], wh[b, 1], c)
        sl = slice(offs[b], offs[b + 1])
        assert support.eq16(a[sl], R.sat_rn(torch.from_numpy(R.operand_rows(rows, loc, Kp)).cuda(), dt == torch.float16)), b
        assert support.eq32(sp[sl], torch.from_numpy(loc).cuda()), b


# ================================================================================================================ narrow heads
@pytest.mark.parametrize("cut", [None, 30], ids=["all_rows", "m_rows_30"])
@pytest.mark.parametrize("add,bias", [(True, True), (False, False), (True, False), (False, True)], ids=["add_bias", "plain", "add", "bias"])
@pytest.mark.parametrize("K", [768, 1024, 2048])
@pytest.mark.parametrize("n_out", [1, 2, 3, 4])
def test_rowdot(n_out, K, add, bias, cut, parity_log):
    """out[m, j] = x[m] . w[j] + bias[j] + add[m] against fp64, to 1e-5 of the row's sum of |terms|; M = 37 (not a multiple of the four
    rows per CTA), strided x, ld_out > n_out: columns past n_out and rows at or past the device row count keep the sentinel."""
    M, ld_x, ld_out = 37, K + 4, 6
    g = _gen(n_out * K)
    x = torch.randn(M, ld_x, generator=g, device="cuda")
    w = torch.randn(n_out, K, generator=g, device="cuda") / math.sqrt(K)
    b = torch.randn(n_out, generator=g, device="cuda") if bias else None
    a = None
    if add:                                                     # the vision-logit mask: 0 / -10000, plus noise
        a = torch.randn(M, generator=g, device="cuda")
        a[::3] = -10000.0
    out = torch.full((M, ld_out), NAN, device="cuda")
    rows = _dev_i32([cut]) if cut is not None else None
    support.call("vb200_rowdot", x, ld_x, w, b, a, out, ld_out, M, K, n_out, rows)
    torch.cuda.synchronize()
    m = cut if cut is not None else M
    terms = x[:, :K].double()[:, None, :] * w.double()[None]
    ref = terms.sum(-1)
    scale = terms.abs().sum(-1)
    if b is not None:
        ref, scale = ref + b.double(), scale + b.double().abs()
    if a is not None:
        ref, scale = ref + a.double()[:, None], scale + a.double().abs()[:, None]
    rel = ((out[:m, :n_out].double() - ref[:m]).abs() / scale[:m]).max().item()
    parity_log(test="kp_rowdot", n_out=n_out, K=K, add=add, bias=bias, cut=cut, max_rel_err=rel, bound=1e-5)
    assert rel < 1e-5, rel
    assert _is_nan(out[:, n_out:]) and _is_nan(out[m:])


# ================================================================================================================ state gathers
def test_gather_state():
    """Sample b of the destination = block clamp(idx[b]) of the source, bit for bit (fp32, 16-bit, mask); out-of-range indices clamp;
    the destination block past B keeps the sentinel."""
    n_src, B, L, H, H16 = 5, 7, 3, 64, 72
    g = _gen(11)
    s32 = torch.randn(n_src, L, H, generator=g, device="cuda")
    s16 = torch.randint(-32768, 32767, (n_src, L, H16), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    smask = torch.randn(n_src, L, generator=g, device="cuda")
    idx = [0, 4, -1, 9, 2, 2, 3]
    d32 = torch.full((B + 1, L, H), NAN, device="cuda")
    d16 = torch.full((B + 1, L, H16), 0x7E01, dtype=torch.int16, device="cuda")
    dmask = torch.full((B + 1, L), NAN, device="cuda")
    support.call("vb200_gather_state", _dev_i32(idx), n_src, s32, s16, smask, d32, d16, dmask, B, L, H, H16)
    torch.cuda.synchronize()
    src = torch.tensor([min(max(i, 0), n_src - 1) for i in idx], device="cuda")
    assert support.eq32(d32[:B], s32[src]) and torch.equal(d16[:B], s16[src]) and support.eq32(dmask[:B], smask[src])
    assert _is_nan(d32[B:]) and bool((d16[B:] == 0x7E01).all()) and _is_nan(dmask[B:])


def test_gather_state_packed_pooler_form():
    """The packed pooler's gather (engine: L = 1, H = H16 = the row stride, idx = the plan's row offsets, no fp32 / mask copy): row
    offs[b] of the packed 16-bit state -> row b."""
    lens = [1, 30, 7, 129, 16]
    offs = _offs(lens)
    ld = 768 + 8
    M = offs[-1]
    s16 = torch.randint(-32768, 32767, (M, ld), generator=_gen(12), device="cuda", dtype=torch.int32).to(torch.int16)
    d16 = torch.full((len(lens) + 1, ld), 0x7E01, dtype=torch.int16, device="cuda")
    support.call("vb200_gather_state", _dev_i32(offs), M, None, s16, None, None, d16, None, len(lens), 1, ld, ld)
    torch.cuda.synchronize()
    assert torch.equal(d16[:len(lens)], s16[torch.tensor(offs[:-1], device="cuda")])
    assert bool((d16[len(lens):] == 0x7E01).all())


def test_gather_packed_state():
    """Packed retrieval gather, both streams in one launch: pair b's rows [dst[b], dst[b+1]) = source rows from src[b], bit for bit;
    ragged offsets; destination rows past dst[B] keep the sentinel."""
    Ht, Hv = 768, 1024
    t_lens, v_lens = [5, 1, 37, 12], [36, 101, 1, 20]              # pair lengths
    t_src_rows, v_src_rows = 80, 170
    t_src_start, v_src_start = [3, 0, 40, 60], [100, 0, 169, 30]   # pairs may share a caption / an image, or overlap
    g = _gen(13)
    ts32, vs32 = torch.randn(t_src_rows, Ht, generator=g, device="cuda"), torch.randn(v_src_rows, Hv, generator=g, device="cuda")
    ts16 = torch.randn(t_src_rows, Ht, generator=g, device="cuda").half()
    vs16 = torch.randn(v_src_rows, Hv, generator=g, device="cuda").half()
    to, vo = _offs(t_lens), _offs(v_lens)
    td32 = torch.full((to[-1] + 2, Ht), NAN, device="cuda")
    td16 = torch.full((to[-1] + 2, Ht), NAN, dtype=torch.float16, device="cuda")
    vd32 = torch.full((vo[-1] + 2, Hv), NAN, device="cuda")
    vd16 = torch.full((vo[-1] + 2, Hv), NAN, dtype=torch.float16, device="cuda")
    support.call("vb200_gather_packed_state", len(t_lens), _dev_i32(to), _dev_i32(t_src_start), ts32, ts16, td32, td16,
                 Ht // 4, Ht // 8, _dev_i32(vo), _dev_i32(v_src_start), vs32, vs16, vd32, vd16, Hv // 4, Hv // 8)
    torch.cuda.synchronize()
    for b in range(len(t_lens)):
        st, sv = t_src_start[b], v_src_start[b]
        assert support.eq32(td32[to[b]:to[b + 1]], ts32[st:st + t_lens[b]]) and support.eq16(td16[to[b]:to[b + 1]], ts16[st:st + t_lens[b]]), b
        assert support.eq32(vd32[vo[b]:vo[b + 1]], vs32[sv:sv + v_lens[b]]) and support.eq16(vd16[vo[b]:vo[b + 1]], vs16[sv:sv + v_lens[b]]), b
    assert _is_nan(td32[to[-1]:]) and _is_nan(td16[to[-1]:]) and _is_nan(vd32[vo[-1]:]) and _is_nan(vd16[vo[-1]:])


# ================================================================================================================ attention
# error / max(1, |ref|), about twice the rounding floor: the CPU emulation of the kernels' rounding points (16-bit P before P V, 16-bit
# context; tests/test_kernel_refs.py::test_attention_rounding_floor) gives up to 4.4e-3 (bf16) and 6.2e-4 (fp16); measured on an H100
# SXM: up to 5.4e-3 (bf16, packed batches with 15-17-key samples) and 6.9e-4 (fp16)
ATTN_TOL = {torch.bfloat16: 1.2e-2, torch.float16: 1.5e-3}

LENGTHS = [1, 15, 16, 17, 63, 64, 65, 128, 129, 256]


def _key_mask(L, b):
    """A different additive mask per sample: interior masked keys (every (b % 3 + 2)-th key) and, for odd b, a masked tail; key 0
    always real."""
    m = torch.zeros(L)
    m[1::b % 3 + 2] = -10000.0
    if b % 2 and L > 4:
        m[L - L // 4:] = -10000.0
    m[0] = 0.0
    return m


def _attn_err(ctx, ref):
    return ((ctx.double() - ref).abs() / ref.abs().clamp(min=1.0)).max().item()


def _self_dense(qkv, ld_qkv, H, mask, B, L, heads, d, dt, ld_ctx):
    ctx = torch.full((B * L, ld_ctx), NAN, dtype=dt, device="cuda")
    support.call("vb200_self_attention", qkv, ld_qkv, H, mask, ctx, ld_ctx, B, L, heads, d, _f16(dt))
    return ctx


def _co_dense(qi, ld_i, qt, ld_t, H, mi, mt, B, T, V, heads, d, dt, ld_ct, ld_ci):
    ct = torch.full((B * T, ld_ct), NAN, dtype=dt, device="cuda")
    ci = torch.full((B * V, ld_ci), NAN, dtype=dt, device="cuda")
    support.call("vb200_co_attention", qi, ld_i, qt, ld_t, H, mi, mt, ct, ld_ct, ci, ld_ci, B, T, V, heads, d, _f16(dt))
    return ct, ci


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("B,L,heads,d", [(3, 31, 12, 64), (3, 65, 2, 128), (2, 129, 8, 64), (2, 256, 2, 128), (4, 17, 2, 64)])
def test_self_attention_masks_strides(B, L, heads, d, dt, parity_log):
    """Dense self-attention with a different mask per sample (interior and tail masked keys) and strided qkv / ctx rows."""
    H = heads * d
    ld_qkv, ld_ctx = 3 * H + 16, H + 8
    qkv = torch.randn(B * L, ld_qkv, generator=_gen(B * L + d), device="cuda").to(dt)
    mask = torch.stack([_key_mask(L, b) for b in range(B)]).cuda()
    ctx = _self_dense(qkv, ld_qkv, H, mask, B, L, heads, d, dt, ld_ctx)
    torch.cuda.synchronize()
    x = qkv[:, :3 * H].view(B, L, 3 * H)
    ref = R.attention_fp64(x[..., :H], x[..., H:2 * H], x[..., 2 * H:], mask, heads)
    err = _attn_err(ctx[:, :H].view(B, L, H), ref)
    parity_log(test="kp_self_attention", B=B, L=L, heads=heads, d=d, dtype=str(dt), max_rel_err=err, bound=ATTN_TOL[dt])
    assert err < ATTN_TOL[dt], err
    assert _is_nan(ctx[:, H:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("B,T,V,heads,d", [(3, 31, 36, 8, 128), (3, 37, 100, 2, 128), (2, 100, 37, 2, 64), (2, 129, 65, 2, 64),
                                           (2, 64, 256, 2, 128), (3, 1, 17, 2, 64)])
def test_co_attention_masks_strides(B, T, V, heads, d, dt, parity_log):
    """Dense co-attention with a different text and image mask per sample, T and V on both sides of 64, strided rows."""
    H = heads * d
    ld_i, ld_t, ld_ct, ld_ci = 3 * H + 8, 3 * H + 24, H + 16, H + 2
    g = _gen(B + T + V + d)
    qi = torch.randn(B * V, ld_i, generator=g, device="cuda").to(dt)
    qt = torch.randn(B * T, ld_t, generator=g, device="cuda").to(dt)
    mi = torch.stack([_key_mask(V, b) for b in range(B)]).cuda()
    mt = torch.stack([_key_mask(T, b + 1) for b in range(B)]).cuda()
    ct, ci = _co_dense(qi, ld_i, qt, ld_t, H, mi, mt, B, T, V, heads, d, dt, ld_ct, ld_ci)
    torch.cuda.synchronize()
    xi, xt = qi[:, :3 * H].view(B, V, 3 * H), qt[:, :3 * H].view(B, T, 3 * H)
    ref_t = R.attention_fp64(xt[..., :H], xi[..., H:2 * H], xi[..., 2 * H:], mi, heads)
    ref_i = R.attention_fp64(xi[..., :H], xt[..., H:2 * H], xt[..., 2 * H:], mt, heads)
    e1, e2 = _attn_err(ct[:, :H].view(B, T, H), ref_t), _attn_err(ci[:, :H].view(B, V, H), ref_i)
    parity_log(test="kp_co_attention", B=B, T=T, V=V, heads=heads, d=d, dtype=str(dt), err_text_ctx=e1, err_image_ctx=e2,
               bound=ATTN_TOL[dt])
    assert e1 < ATTN_TOL[dt] and e2 < ATTN_TOL[dt], (e1, e2)
    assert _is_nan(ct[:, H:]) and _is_nan(ci[:, H:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_self_attention_packed(d, dt, parity_log):
    """Packed self-attention over samples of length 1 ... 256: each sample's rows equal a dense call of that sample alone, bit for
    bit, and fp64 within the attention bound; rows past the last sample and columns past H keep the sentinel."""
    heads = 2
    H = heads * d
    ld_qkv, ld_ctx = 3 * H + 8, H + 8
    offs = _offs(LENGTHS)
    M = offs[-1]
    qkv = torch.randn(M, ld_qkv, generator=_gen(d), device="cuda").to(dt)
    mask = torch.cat([_key_mask(L, b) for b, L in enumerate(LENGTHS)]).cuda()
    ctx = torch.full((M + 16, ld_ctx), NAN, dtype=dt, device="cuda")
    support.call("vb200_self_attention_packed", qkv, ld_qkv, H, mask, ctx, ld_ctx, len(LENGTHS), max(LENGTHS), heads, d, _f16(dt),
                 _dev_i32(offs))
    worst = 0.0
    for b, L in enumerate(LENGTHS):
        sl = slice(offs[b], offs[b + 1])
        dense = _self_dense(qkv[sl], ld_qkv, H, mask[sl].contiguous(), 1, L, heads, d, dt, ld_ctx)
        torch.cuda.synchronize()
        assert support.eq16(ctx[sl, :H], dense[:, :H]), f"sample {b} (L = {L})"
        x = qkv[sl, :3 * H].view(1, L, 3 * H)
        ref = R.attention_fp64(x[..., :H], x[..., H:2 * H], x[..., 2 * H:], mask[sl].view(1, L), heads)
        worst = max(worst, _attn_err(ctx[sl, :H].view(1, L, H), ref))
    parity_log(test="kp_self_attention_packed", d=d, dtype=str(dt), max_rel_err=worst, bound=ATTN_TOL[dt])
    assert worst < ATTN_TOL[dt], worst
    assert _is_nan(ctx[M:]) and _is_nan(ctx[:, H:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_co_attention_packed(d, dt, parity_log):
    """Packed co-attention, text lengths 1 ... 256 against image lengths in the reverse order: each sample equals a dense call of it
    alone, bit for bit, and fp64 within the attention bound; rows outside every sample keep the sentinel."""
    heads = 2
    H = heads * d
    T_l, V_l = LENGTHS, LENGTHS[::-1]
    B = len(T_l)
    ld_i, ld_t, ld_ct, ld_ci = 3 * H + 8, 3 * H, H + 8, H
    ot, ov = _offs(T_l), _offs(V_l)
    g = _gen(d + 1)
    qi = torch.randn(ov[-1], ld_i, generator=g, device="cuda").to(dt)
    qt = torch.randn(ot[-1], ld_t, generator=g, device="cuda").to(dt)
    mi = torch.cat([_key_mask(V, b) for b, V in enumerate(V_l)]).cuda()
    mt = torch.cat([_key_mask(T, b + 1) for b, T in enumerate(T_l)]).cuda()
    ct = torch.full((ot[-1] + 16, ld_ct), NAN, dtype=dt, device="cuda")
    ci = torch.full((ov[-1] + 16, ld_ci), NAN, dtype=dt, device="cuda")
    support.call("vb200_co_attention_packed", qi, ld_i, qt, ld_t, H, mi, mt, ct, ld_ct, ci, ld_ci, B, max(T_l), max(V_l),
                 heads, d, _f16(dt), _dev_i32(ot), _dev_i32(ov))
    worst = 0.0
    for b in range(B):
        T, V = T_l[b], V_l[b]
        st, sv = slice(ot[b], ot[b + 1]), slice(ov[b], ov[b + 1])
        dt_, di_ = _co_dense(qi[sv], ld_i, qt[st], ld_t, H, mi[sv].contiguous(), mt[st].contiguous(), 1, T, V, heads, d, dt, ld_ct, ld_ci)
        torch.cuda.synchronize()
        assert support.eq16(ct[st, :H], dt_[:, :H]) and support.eq16(ci[sv, :H], di_[:, :H]), f"sample {b} (T = {T}, V = {V})"
        xi, xt = qi[sv, :3 * H].view(1, V, 3 * H), qt[st, :3 * H].view(1, T, 3 * H)
        ref_t = R.attention_fp64(xt[..., :H], xi[..., H:2 * H], xi[..., 2 * H:], mi[sv].view(1, V), heads)
        ref_i = R.attention_fp64(xi[..., :H], xt[..., H:2 * H], xt[..., 2 * H:], mt[st].view(1, T), heads)
        worst = max(worst, _attn_err(ct[st, :H].view(1, T, H), ref_t), _attn_err(ci[sv, :H].view(1, V, H), ref_i))
    parity_log(test="kp_co_attention_packed", d=d, dtype=str(dt), max_rel_err=worst, bound=ATTN_TOL[dt])
    assert worst < ATTN_TOL[dt], worst
    assert _is_nan(ct[ot[-1]:]) and _is_nan(ci[ov[-1]:]) and _is_nan(ct[:, H:])


STRUCT_LENGTHS = [1, 16, 17, 64, 65, 129, 256]


def _structured(L, heads, d, seed, dt):
    """Q / K / V rows for one sample in which query i of head h attends to key perm[h][i] with a score margin of about 30 (keys are
    random +-1 codes, the query is 10 x its key's code), and every V column of key j holds j: an indexing error is an O(1) error.
    Random permutations put the winning key in every 64-key block, so the online softmax rescales."""
    g = torch.Generator().manual_seed(seed)
    H = heads * d
    codes = torch.randint(0, 2, (L, heads, d), generator=g).float() * 2 - 1
    perm = torch.stack([torch.randperm(L, generator=g) for _ in range(heads)])            # [heads, L]
    q = torch.stack([10.0 * codes[perm[h], h] for h in range(heads)], dim=1)               # [L, heads, d]
    v = torch.arange(L).float()[:, None].expand(L, H)
    qkv = torch.cat([q.reshape(L, H), codes.reshape(L, H), v], dim=1).to(dt)
    expect = perm.t().float()[:, :, None].expand(L, heads, d).reshape(L, H)                # row i, head h -> perm[h][i]
    return qkv, expect


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("d", [64, 128])
def test_attention_structured(d, dt):
    """Dense (two samples per call) and packed self- and co-attention on the structured inputs: every output equals the index of the
    key its query was built to attend to."""
    heads = 2
    H = heads * d
    for L in STRUCT_LENGTHS:
        parts = [_structured(L, heads, d, seed=L * 10 + s, dt=dt) for s in range(2)]
        qkv = torch.cat([p[0] for p in parts]).cuda()
        expect = torch.cat([p[1] for p in parts]).cuda()
        mask = torch.zeros(2 * L, device="cuda")
        ctx = _self_dense(qkv, 3 * H, H, mask, 2, L, heads, d, dt, H)
        torch.cuda.synchronize()
        assert (ctx.float() - expect).abs().max().item() < 0.5, f"dense self L = {L}"
    parts = [_structured(L, heads, d, seed=L, dt=dt) for L in STRUCT_LENGTHS]
    offs = _offs(STRUCT_LENGTHS)
    qkv = torch.cat([p[0] for p in parts]).cuda()
    expect = torch.cat([p[1] for p in parts]).cuda()
    mask = torch.zeros(offs[-1], device="cuda")
    ctx = torch.full((offs[-1], H), NAN, dtype=dt, device="cuda")
    support.call("vb200_self_attention_packed", qkv, 3 * H, H, mask, ctx, H, len(STRUCT_LENGTHS), max(STRUCT_LENGTHS), heads, d,
                 _f16(dt), _dev_i32(offs))
    torch.cuda.synchronize()
    assert (ctx.float() - expect).abs().max().item() < 0.5, "packed self"
    # co-attention: text queries over image keys built for them (T = V per sample), and the image direction over the text keys
    ct = torch.full((offs[-1], H), NAN, dtype=dt, device="cuda")
    ci = torch.full((offs[-1], H), NAN, dtype=dt, device="cuda")
    o = _dev_i32(offs)
    support.call("vb200_co_attention_packed", qkv, 3 * H, qkv, 3 * H, H, mask, mask, ct, H, ci, H, len(STRUCT_LENGTHS),
                 max(STRUCT_LENGTHS), max(STRUCT_LENGTHS), heads, d, _f16(dt), o, o)
    torch.cuda.synchronize()
    assert (ct.float() - expect).abs().max().item() < 0.5 and (ci.float() - expect).abs().max().item() < 0.5, "packed co"
    for L in (17, 129):
        i = STRUCT_LENGTHS.index(L)
        sl = slice(offs[i], offs[i + 1])
        dct, dci = _co_dense(qkv[sl], 3 * H, qkv[sl], 3 * H, H, mask[sl], mask[sl], 1, L, L, heads, d, dt, H, H)
        torch.cuda.synchronize()
        assert (dct.float() - expect[sl]).abs().max().item() < 0.5 and (dci.float() - expect[sl]).abs().max().item() < 0.5, L


# ================================================================================================================ GEMMs
def _operands(M, N, K, dt, seed, ld_x=None):
    g = _gen(seed)
    x = torch.randn(M, ld_x or K, generator=g, device="cuda").to(dt)
    w = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).to(dt)
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    return x, w, b


def _linear(x, w, b, M, N, K, dt, outs="16+32", variant=0, bn=0, act=0, pdl=0, ld16=None, ld32=None, sync=True, y16=None, y32=None):
    ld16 = ld16 or (N + 7) // 8 * 8
    ld32 = ld32 or (N + 3) // 4 * 4
    if y16 is None and "16" in outs:
        y16 = torch.full((M, ld16), NAN, dtype=dt, device="cuda")
    if y32 is None and "32" in outs:
        y32 = torch.full((M, ld32), NAN, device="cuda")
    support.call("vb200_linear", x, x.stride(0), w, w.stride(0), b, None, 0, None, None, 1e-12, act, y16, ld16, y32, ld32, M, N, K, bn, pdl,
                 _f16(dt), variant, None)
    if sync:
        torch.cuda.synchronize()
    return (y16[:, :N] if y16 is not None else None), (y32[:, :N] if y32 is not None else None)


# (name, M, N, K, variant, block_n): the store paths of the two plain GEMM kernels
STORE_PATHS = [
    ("register_store", 256, 512, 256, 0, 128),         # 16-byte swizzled stores of both outputs
    ("ragged_n_remainder", 64, 3129, 2048, 0, 128),    # the per-lane remainder of the last, ragged 32-column chunk
    ("many_tiles_per_cta", 2304, 3072, 1024, 0, 128),  # several tiles per persistent CTA
    ("narrow_tiles", 300, 384, 512, 4, 64),
    ("pingpong", 1984, 768, 768, 5, 128),              # the ping-pong kernel: every output through the TMA
    ("pingpong_64", 1000, 1024, 256, 5, 64),
]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("path", STORE_PATHS, ids=[p[0] for p in STORE_PATHS])
def test_linear_16bit_is_sat_rn(path, dt):
    """The 16-bit output is sat_rn of the fp32 output written alongside it, bit for bit; the 16-bit-only run (the cooperative
    kernel's TMA-store epilogue for each CTA's last tile; the ping-pong kernel's 16-bit TMA map alone) gives the same bits."""
    _, M, N, K, variant, bn = path
    x, w, b = _operands(M, N, K, dt, seed=M + N)
    for act in (0, 1):
        y16, y32 = _linear(x, w, b, M, N, K, dt, variant=variant, bn=bn, act=act)
        assert support.eq16(y16, R.sat_rn(y32, dt == torch.float16)), act
        if N % 8 == 0:
            y16b, _ = _linear(x, w, b, M, N, K, dt, outs="16", variant=variant, bn=bn, act=act)
            assert support.eq16(y16b, y16), act


@pytest.mark.parametrize("path", STORE_PATHS, ids=[p[0] for p in STORE_PATHS])
def test_linear_fp16_saturates(path):
    """Bias +-1e5 in fp16: every GEMM store path writes +-65504, never inf (register, ragged remainder, TMA store, ping-pong)."""
    _, M, N, K, variant, bn = path
    x, w, b = _operands(M, N, K, torch.float16, seed=N)
    b[0::3] = 1e5
    b[1::3] = -1e5
    y16, y32 = _linear(x, w, b, M, N, K, torch.float16, variant=variant, bn=bn)
    assert bool((y32[:, 0::3] > 65504).all()) and bool((y32[:, 1::3] < -65504).all())
    assert support.eq16(y16, R.sat_rn(y32, True))
    assert bool((y16[:, 0::3] == 65504).all()) and bool((y16[:, 1::3] == -65504).all())
    if N % 8 == 0:
        y16b, _ = _linear(x, w, b, M, N, K, torch.float16, outs="16", variant=variant, bn=bn)
        assert support.eq16(y16b, y16) and not bool(torch.isinf(y16b.float()).any())


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_layernorm_row_kernel_16bit_rounding(dt):
    """The row LayerNorm's 16-bit output is the round-to-nearest-even of its fp32 output.  It converts with the non-saturating
    pack16x2 (an out-of-range fp16 value would become inf, where the GEMM stores clamp to +-65504), so this holds for in-range
    values only -- LayerNorm outputs are bounded by |gamma| sqrt(N) + |beta|, far inside the fp16 range."""
    M, N = 300, 768
    g = _gen(19)
    y, res = torch.randn(M, N, generator=g, device="cuda") * 3, torch.randn(M, N, generator=g, device="cuda")
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g, device="cuda"), 0.1 * torch.randn(N, generator=g, device="cuda")
    of = torch.full((M, N), NAN, device="cuda")
    oh = torch.full((M, N), NAN, dtype=dt, device="cuda")
    support.call("vb200_layernorm", y, N, res, N, gamma, beta, 1e-12, of, N, oh, N, M, N, _f16(dt))
    torch.cuda.synchronize()
    assert bool((of.abs() < 65504).all())
    assert support.eq16(oh, R.sat_rn(of, dt == torch.float16))


def _ref_product(x, w, b, act, mul):
    y = x.double() @ w.double().t() + b.double()
    if act == 2:
        y = torch.relu(y)
    return y * mul.double()


# (M, N, K, ld_x, ld_mul): the pooler at batch 1 / 8 / 64 (strided A: the first token of each sample, ld_x = T H), then a ragged N
# and an ld_mul that is not a multiple of 4 (the scalar multiply fallback)
PRODUCT_CASES = [(1, 1024, 1024, 37 * 1024, 1024), (8, 1024, 1024, 37 * 1024, 1024), (64, 1024, 1024, 101 * 1024, 1024),
                 (64, 1000, 768, 768, 1000), (64, 1000, 768, 768, 1003), (200, 1024, 1024, 1024, 1027)]


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("case", PRODUCT_CASES, ids=lambda c: "M%d_N%d_K%d_ldx%d_ldmul%d" % c)
def test_linear_product(case, dt, parity_log):
    """Pooled-product GEMM relu(x w^T + b) * mul against fp64, both outputs; the 16-bit output is sat_rn of the fp32 one, and the
    16-bit-only run (TMA store) gives the same bits."""
    M, N, K, ld_x, ld_mul = case
    x, w, b = _operands(M, N, K, dt, seed=M + N + ld_mul, ld_x=ld_x)
    mul = torch.rand(M, ld_mul, generator=_gen(ld_mul), device="cuda") * 2.0
    ref = _ref_product(x[:, :K], w, b, 2, mul[:, :N])
    ld16, ld32 = (N + 7) // 8 * 8, (N + 3) // 4 * 4
    y16 = torch.full((M, ld16), NAN, dtype=dt, device="cuda")
    y32 = torch.full((M, ld32), NAN, device="cuda")
    support.call("vb200_linear_product", x, ld_x, w, K, b, 2, mul, ld_mul, y16, ld16, y32, ld32, M, N, K, 0, _f16(dt))
    y16o = torch.full((M, ld16), NAN, dtype=dt, device="cuda")
    support.call("vb200_linear_product", x, ld_x, w, K, b, 2, mul, ld_mul, y16o, ld16, None, 0, M, N, K, 0, _f16(dt))
    torch.cuda.synchronize()
    err = (y32[:, :N].double() - ref).abs().max().item()
    parity_log(test="kp_linear_product", M=M, N=N, K=K, ld_mul=ld_mul, dtype=str(dt), max_abs_err=err, bound=2e-3)
    assert err < 2e-3, err
    assert support.eq16(y16[:, :N], R.sat_rn(y32[:, :N], dt == torch.float16))
    assert support.eq16(y16o[:, :N], y16[:, :N])
    assert _is_nan(y32[:, N:]) and _is_nan(y16[:, N:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("m", [0, 1, 128, 129, 1000])
@pytest.mark.parametrize("N", [1601, 3129])
def test_coop_device_row_count(N, m, dt):
    """vb200_linear_rows with a ragged N (the packed heads' img_decoder / VQA widths) runs the cooperative kernel's device row count
    (PCfg MODE 6): rows < m equal vb200_linear bit for bit, rows from the next 128-row boundary on keep the sentinel."""
    M, K = 1000, 768
    x, w, b = _operands(M, N, K, dt, seed=N)
    ld16, ld32 = (N + 7) // 8 * 8, (N + 3) // 4 * 4
    y16 = torch.full((M, ld16), NAN, dtype=dt, device="cuda")
    y32 = torch.full((M, ld32), NAN, device="cuda")
    support.call("vb200_linear_rows", x, K, w, K, b, 0, y16, ld16, y32, ld32, M, N, K, 0, _f16(dt), _dev_i32([m]))
    r16, r32 = _linear(x, w, b, M, N, K, dt)
    assert support.eq32(y32[:m, :N], r32[:m]) and support.eq16(y16[:m, :N], r16[:m])
    boundary = (m + 127) // 128 * 128
    assert _is_nan(y32[boundary:]) and _is_nan(y16[boundary:])
    assert _is_nan(y32[:, N:]) and _is_nan(y16[:, N:])


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_coop_plain_gemm_pdl_chain(dt):
    """Three dependent cooperative-kernel launches (variant 0) -- N = 768 with 16-bit output, a ragged N = 1000 with GELU, then N = 3129
    reading the previous output -- with no synchronize in between, under programmatic dependent launch modes 0, 1 and 5 (5 puts the weight
    tiles in flight before griddepcontrol.wait).  Intermediate buffers start as NaN, so a read before the previous launch has finished
    shows up; all three modes give the same bits."""
    M, K = 1984, 768
    x, w1, b1 = _operands(M, 768, K, dt, seed=31)
    _, w2, b2 = _operands(1, 1000, 768, dt, seed=32)
    _, w3, b3 = _operands(1, 3129, 1000, dt, seed=33)
    outs = []
    for pdl in (0, 1, 5):
        y1 = torch.full((M, 768), NAN, dtype=dt, device="cuda")
        y2 = torch.full((M, 1000), NAN, dtype=dt, device="cuda")
        _linear(x, w1, b1, M, 768, K, dt, outs="16", pdl=pdl, y16=y1, ld16=768, sync=False)
        _linear(y1, w2, b2, M, 1000, 768, dt, outs="16", pdl=pdl, act=1, y16=y2, ld16=1000, sync=False)
        y3b, y3 = _linear(y2, w3, b3, M, 3129, 1000, dt, pdl=pdl, sync=False)
        torch.cuda.synchronize()
        outs.append((y1, y2, y3b, y3))
    for o in outs:
        assert not _is_nan(o[3]) and not bool(torch.isnan(o[3]).any())
    for o in outs[1:]:
        assert support.eq16(o[0], outs[0][0]) and support.eq16(o[1], outs[0][1]) and support.eq16(o[2], outs[0][2]) \
            and support.eq32(o[3], outs[0][3])
    ref = R.sat_rn(outs[0][3], dt == torch.float16)
    assert support.eq16(outs[0][2], ref)
