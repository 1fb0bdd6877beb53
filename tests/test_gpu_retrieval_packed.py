"""Packed caption-image retrieval (VILBertForVLTasks.encode_text_packed / encode_image_packed / forward_cached_packed and
parallel.retrieval_scores_packed).  `-m gpu` only.

The packed prefixes run the same kernels on the same rows as a dense prefix of one caption / image alone, and the packed suffix
the same kernels on the same rows as vb200_forward_packed, so states and scores are compared bit for bit; the fp32 oracle and the
dense padded retrieval path are compared at the tolerances of test_gpu_packed.py.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 mode vs the fp32 oracle, and packed vs dense padded retrieval (test_gpu_model.py)
DT = ("fp16", "bf16")


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle)


def _captions(model, lens, seed):
    """[(tokens [Tin], segments [Tin], task id)] per caption."""
    vocab = model._dims["vocab_size"]
    out = []
    for i, tin in enumerate(lens):
        g = torch.Generator().manual_seed(seed + i)
        out.append((torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g),
                    int(torch.randint(0, 20, (1,), generator=g))))
    return out


def _images(model, lens, seed):
    """[(features [V, F], spatials [V, 5])] per image, global box first."""
    F = model._dims["v_feature_size"]
    out = []
    for i, v in enumerate(lens):
        g = torch.Generator().manual_seed(seed + 1000 + i)
        f = torch.relu(torch.randn(v, F, generator=g)) * 1.5
        xy = torch.rand(v, 2, generator=g) * 0.7
        x2y2 = (xy + 0.05 + torch.rand(v, 2, generator=g) * 0.25).clamp(max=1.0)
        s = torch.cat([xy, x2y2, ((x2y2 - xy)[:, 0] * (x2y2 - xy)[:, 1])[:, None]], dim=-1)
        s[0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
        out.append((f, s))
    return out


def _encode(model, caps, imgs, **kw):
    cat = lambda xs: torch.cat(xs).cuda()
    ts = model.encode_text_packed(cat([c[0] for c in caps]), cat([c[1] for c in caps]), torch.tensor([[c[2]] for c in caps]).cuda(),
                                  [len(c[0]) for c in caps], max_tokens=kw.get("max_tokens", 0))
    vs = model.encode_image_packed(cat([i[0] for i in imgs]), cat([i[1] for i in imgs]), [i[0].shape[0] for i in imgs],
                                   max_regions=kw.get("max_regions", 0))
    return ts, vs


def _forward_packed_pairs(model, caps, imgs, ti, ii, select):
    """vb200_forward_packed of the same pairs: the pairs' captions and images concatenated as one packed batch."""
    pc, pi = [caps[t] for t in ti], [imgs[i] for i in ii]
    cat = lambda xs: torch.cat(xs).cuda()
    out = model.forward_packed(cat([c[0] for c in pc]), cat([i[0] for i in pi]), cat([i[1] for i in pi]), cat([c[1] for c in pc]),
                               torch.tensor([[c[2]] for c in pc]).cuda(), [len(c[0]) for c in pc], [i[0].shape[0] for i in pi],
                               select=select, debug_taps=True)
    torch.cuda.synchronize()
    return out


def _assert_same(got, want, what):
    (go, gt), (wo, wt) = got, want
    for k in range(9):
        assert (go[k] is None) == (wo[k] is None), (what, k)
        if go[k] is not None:
            assert torch.equal(go[k], wo[k]), f"{what}: output {k} differs from forward_packed of the same pairs"
    for k in ("sequence_output_t", "sequence_output_v", "pooled_output"):
        assert torch.equal(gt[k], wt[k]), f"{what}: tap {k} differs"


# Tin 1, T = 63 / 64 / 65 keys either side of 64, Tin 155 (tiny max_position_embeddings is 160); V 1, 63 / 64 / 65, the 256-row limit
CAP_LENS = [1, 62, 63, 64, 155, 9]
IMG_LENS = [1, 63, 64, 65, 256]


@pytest.mark.parametrize("mode", DT)
def test_packed_states_equal_dense_encode_alone(tiny, mode):
    """Every caption's rows of the packed text state equal encode_text of that caption alone at its own length, bit for bit (fp32
    stream and 16-bit operand); the same for images."""
    model = tiny[mode]
    caps, imgs = _captions(model, CAP_LENS, seed=1), _images(model, IMG_LENS, seed=1)
    ts, vs = _encode(model, caps, imgs)
    torch.cuda.synchronize()
    to, vo = ts["offsets"].tolist(), vs["offsets"].tolist()
    assert to[-1] == sum(CAP_LENS) + len(CAP_LENS) and vo[-1] == sum(IMG_LENS)
    for c, (q, seg, task) in enumerate(caps):
        one = torch.ones(1, len(q), dtype=torch.long).cuda()
        ref = model.encode_text(q[None].cuda(), seg[None].cuda(), one, torch.tensor([[task]]).cuda())
        torch.cuda.synchronize()
        assert torch.equal(ts["f32"][to[c]:to[c + 1]], ref["f32"][0]), f"caption {c}: fp32 rows"
        assert torch.equal(ts["h16"][to[c]:to[c + 1]], ref["h16"][0]), f"caption {c}: 16-bit rows"
    for i, (f, s) in enumerate(imgs):
        ref = model.encode_image(f[None].cuda(), s[None].cuda(), torch.ones(1, f.shape[0], dtype=torch.uint8).cuda())
        torch.cuda.synchronize()
        assert torch.equal(vs["f32"][vo[i]:vo[i + 1]], ref["f32"][0]), f"image {i}: fp32 rows"
        assert torch.equal(vs["h16"][vo[i]:vo[i + 1]], ref["h16"][0]), f"image {i}: 16-bit rows"


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("B", [7, 6])
def test_cached_packed_bitwise_equals_forward_packed(tiny, mode, B):
    """All nine outputs (per-row outputs packed) and the three taps of forward_cached_packed equal forward_packed of the same pairs,
    bit for bit, with lengths at the corners mixed in one batch and captions / images repeated across pairs."""
    import vilbert_b200 as vb
    model = tiny[mode]
    caps, imgs = _captions(model, CAP_LENS, seed=2), _images(model, IMG_LENS, seed=2)
    ts, vs = _encode(model, caps, imgs)
    ti = [0, 4, 1, 2, 3, 5, 0][:B]
    ii = [4, 0, 3, 1, 2, 4, 0][:B]
    got = model.forward_cached_packed(ts, torch.tensor(ti), vs, torch.tensor(ii).cuda(), select=vb.OUT_ALL, debug_taps=True)
    torch.cuda.synchronize()
    _assert_same(got, _forward_packed_pairs(model, caps, imgs, ti, ii, vb.OUT_ALL), f"{mode} B={B}")


def test_cached_packed_full_model_block(full, full_oracle):
    """The 268 M model on a 6 x 10 block of retrieval pairs: bit-identical to forward_packed, and vil_logit within 1e-2 of the fp32
    oracle on the equivalent padded batch (checked on the first 12 pairs to keep the CPU oracle short)."""
    import vilbert_b200 as vb
    caps = _captions(full, [7, 30, 12, 19, 25, 9], seed=3)
    imgs = _images(full, [36, 10, 101, 57, 12, 80, 36, 23, 64, 99], seed=3)
    ts, vs = _encode(full, caps, imgs)
    ti = [c for c in range(6) for _ in range(10)]
    ii = [i for _ in range(6) for i in range(10)]
    got = full.forward_cached_packed(ts, torch.tensor(ti), vs, torch.tensor(ii), select=vb.OUT_TASK_HEADS, debug_taps=True)
    torch.cuda.synchronize()
    _assert_same(got, _forward_packed_pairs(full, caps, imgs, ti, ii, vb.OUT_TASK_HEADS), "full 6 x 10")
    n = 12
    Tm, Vm, F = max(len(caps[t][0]) for t in ti[:n]), max(imgs[i][0].shape[0] for i in ii[:n]), full._dims["v_feature_size"]
    q, seg, im = (torch.zeros(n, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(n, Vm, F), torch.zeros(n, Vm, 5), torch.zeros(n, Vm, dtype=torch.uint8)
    for b, (t, i) in enumerate(zip(ti[:n], ii[:n])):
        k, v = len(caps[t][0]), imgs[i][0].shape[0]
        q[b, :k], seg[b, :k], im[b, :k] = caps[t][0], caps[t][1], 1
        f[b, :v], s[b, :v], vm[b, :v] = imgs[i][0], imgs[i][1], 1
    task = torch.tensor([[caps[t][2]] for t in ti[:n]])
    ref = full_oracle(q, f, s, seg, im, vm, None, task)
    err = float((got[0][2][:n].cpu() - ref[2]).abs().max())
    assert err < TOL, f"vil_logit vs fp32 oracle: {err}"


def _retrieval_inputs(model, n_cap, n_img, T_pad, V_pad, t_lens, v_lens, seed):
    caps, imgs = _captions(model, t_lens, seed), _images(model, v_lens, seed)
    F = model._dims["v_feature_size"]
    q, seg, im = (torch.zeros(n_cap, T_pad, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(n_img, V_pad, F), torch.zeros(n_img, V_pad, 5), torch.zeros(n_img, V_pad, dtype=torch.uint8)
    for c, (qq, sg, _) in enumerate(caps):
        q[c, :len(qq)], seg[c, :len(qq)], im[c, :len(qq)] = qq, sg, 1
    for i, (ff, ss) in enumerate(imgs):
        f[i, :ff.shape[0]], s[i, :ff.shape[0]], vm[i, :ff.shape[0]] = ff, ss, 1
    return tuple(t.cuda() for t in (q, seg, im)), tuple(t.cuda() for t in (f, s, vm))


def test_retrieval_scores_packed_vs_cached(full):
    """Uniform lengths, no padding: the packed score matrix equals the dense cached one bit for bit.  Variable lengths padded to the
    block maximum: the two agree within 1e-2 (the dense path attends over masked padding keys)."""
    from vilbert_b200 import parallel as P
    caps, imgs = _retrieval_inputs(full, 5, 7, 20, 36, [20] * 5, [36] * 7, seed=4)
    dense = P.retrieval_scores_cached(full, caps, imgs, pair_batch=8)
    packed = P.retrieval_scores_packed(full, caps, imgs, pair_batch=8)
    torch.cuda.synchronize()
    assert packed.shape == (5, 7)
    assert torch.equal(packed, dense)
    caps, imgs = _retrieval_inputs(full, 5, 7, 30, 101, [7, 30, 12, 21, 9], [10, 101, 36, 55, 12, 80, 99], seed=5)
    dense = P.retrieval_scores_cached(full, caps, imgs, pair_batch=8)
    timings = {}
    packed = P.retrieval_scores_packed(full, caps, imgs, pair_batch=8, timings=timings)
    torch.cuda.synchronize()
    err = float((packed - dense).abs().max())
    assert err < TOL, err
    assert timings["pairs"] == 35 and timings["local_captions"] == 5


def test_packed_retrieval_plan_reuse(tiny):
    """Further chunks reuse the pair plan; a second run with other lengths under the same capacities builds no plan."""
    import vilbert_b200 as vb
    model = tiny["fp16"]
    caps, imgs = _captions(model, [5, 30, 12], seed=6), _images(model, [36, 101, 10, 7], seed=6)
    ts, vs = _encode(model, caps, imgs, max_tokens=30, max_regions=101)
    model.forward_cached_packed(ts, torch.tensor([0, 1, 2, 0]), vs, torch.tensor([0, 1, 2, 3]), select=vb.OUT_VIL_LOGIT)
    n = support.n_plans(model)
    model.forward_cached_packed(ts, torch.tensor([2, 2, 1, 0]), vs, torch.tensor([3, 1, 0, 2]), select=vb.OUT_VIL_LOGIT)
    assert support.n_plans(model) == n
    caps2, imgs2 = _captions(model, [2, 17, 9], seed=7), _images(model, [3, 50, 1, 88], seed=7)
    ts2, vs2 = _encode(model, caps2, imgs2, max_tokens=30, max_regions=101)
    got = model.forward_cached_packed(ts2, torch.tensor([1, 0, 2, 1]), vs2, torch.tensor([2, 3, 0, 1]), select=vb.OUT_VIL_LOGIT,
                                      max_tokens=30, max_regions=101)
    torch.cuda.synchronize()
    assert support.n_plans(model) == n
    # capacity changes no bit: the same pairs at this call's own maxima (another plan)
    ref = model.forward_cached_packed(ts2, torch.tensor([1, 0, 2, 1]), vs2, torch.tensor([2, 3, 0, 1]), select=vb.OUT_VIL_LOGIT)
    torch.cuda.synchronize()
    assert torch.equal(got[2], ref[2])


def test_packed_retrieval_rejections(tiny_oracle, tiny):
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    caps, imgs = _captions(model, [5, 4], seed=8), _images(model, [3, 2], seed=8)
    ts, vs = _encode(model, caps, imgs)
    idx = torch.tensor([0, 1])
    err = lambda pat: pytest.raises(L.VilbertB200Error, match=r"error -1: .*" + pat)
    with err("VB200_OUT_ATTENTION"):
        model.forward_cached_packed(ts, idx, vs, idx, select=L.OUT_VIL_LOGIT | L.OUT_ATTENTION)
    with err(r"text_index 2 outside \[0, 2\)"):
        model.forward_cached_packed(ts, torch.tensor([0, 2]), vs, idx)
    with err(r"image_index -1 outside \[0, 2\)"):
        model.forward_cached_packed(ts, idx, vs, torch.tensor([0, -1]))
    with err("text state 1 has 0 rows"):
        model.forward_cached_packed(dict(ts, offsets=torch.tensor([0, 6, 6], dtype=torch.int32)), idx, vs, idx)
    with err("image state 0 has -1 rows"):
        model.forward_cached_packed(ts, idx, dict(vs, offsets=torch.tensor([3, 2, 5], dtype=torch.int32)), idx)
    with err("capacity"):
        model.forward_cached_packed(ts, idx, vs, idx, max_tokens=4)
    with err("capacity"):
        model.forward_cached_packed(ts, idx, vs, idx, max_regions=2)
    with err("capacity"):
        _encode(model, caps, imgs, max_tokens=4)
    with err("T=257"):
        _encode(model, _captions(model, [256], seed=9), imgs)
    with err("V=257"):
        _encode(model, caps, _images(model, [257], seed=9))
    with err("max_position_embeddings"):
        _encode(model, _captions(model, [161], seed=9), imgs)
    with err("n_tokens 0"):
        model.encode_text_packed(torch.zeros(4, dtype=torch.long).cuda(), torch.zeros(4, dtype=torch.long).cuda(),
                                 torch.zeros(2, 1, dtype=torch.long).cuda(), [0, 4])
    with err("n_regions 0"):
        model.encode_image_packed(torch.zeros(3, model._dims["v_feature_size"]).cuda(), torch.zeros(3, 5).cuda(), [3, 0])
    lib = L.load()
    idx32 = idx.to(torch.int32)
    pairs = L.PackedPairs(2, 0, 0, idx32.data_ptr(), idx32.data_ptr(), 2, ts["offsets"].data_ptr(), None,
                          ts["h16"].data_ptr(), 2, vs["offsets"].data_ptr(), vs["f32"].data_ptr(), vs["h16"].data_ptr())
    assert lib.vb200_forward_cached_packed(model._handle, C.byref(pairs), C.byref(L.Outputs()), L.OUT_VIL_LOGIT, 0, None) == -1
    assert b"NULL" in lib.vb200_last_error(model._handle)
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        with err("fp32x"):
            _encode(x, caps, imgs)
    finally:
        x.close()
