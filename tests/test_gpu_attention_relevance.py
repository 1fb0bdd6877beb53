"""Attention relevance on the device (vb200_attention_relevance, model.attention_relevance).  `-m gpu` only.

Every sample's [2, T + V] rows are bit-identical to the float32 restatement of tests/relevance_ref.py run on the engine's own maps,
and within 1e-6 per entry of the float64 matrix product up to (Tin, V) = (37, 101).  Past 256 rows the float64 bound is derived
from the summation length: a step rounds each column once per product and add over at most L query rows, once per head of the mean
and twice more (the residual add and the halving), so it adds at most gamma_{L + heads + 2} = (L + heads + 2) u (u = 2^-24) to the
L1 norm of r; the steps after it are row-stochastic and do not grow an error in that norm, so n_steps (L + heads + 2) u bounds the
L1 error, and with it every entry.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from relevance_ref import attention_relevance_f32, attention_relevance_f64, sample_maps
import support

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL_F64 = 1e-6             # per entry, engine vs the float64 product on the same maps, up to 256 rows
TOL_ORACLE = 4e-5          # per entry, the bf16 engine's relevance vs the fp32 oracle's maps through the float64 product, 268 M model at
                           # (Tin, V) = (37, 101): measured 1.0e-5 on an H100 80GB HBM3 at 700 W; about 4x that
SENTINEL = -7.0


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16", "fp32x"), return_attention=True)


def _kinds(model):
    return model.attention_selection()[0]


def _task(model):
    return 1 if model._dims["task_specific_tokens"] else 0


def _dense(model, inp):
    out = model(*inp, output_all_attention_masks=True)
    torch.cuda.synchronize()
    return out[9]


def _check_refs(model, attn, rel, packed, tol_f64=TOL_F64):
    """rel (dense [B, 2, N] or packed list) == the float32 restatement on each sample's maps, bit for bit; within tol_f64 of float64.
    Returns the worst float64 difference."""
    kinds = _kinds(model)
    worst = 0.0
    B = len(rel)
    for b in range(B):
        maps = sample_maps(attn, b)
        T = maps[kinds.index(0)].shape[-1]
        V = maps[kinds.index(1)].shape[-1]
        got = rel[b].cpu().numpy()
        assert got.shape == (2, T + V)
        ref = attention_relevance_f32(maps, kinds, T, V)
        assert np.array_equal(got, ref), (b, np.abs(got - ref).max())
        d = float(np.abs(got - attention_relevance_f64(maps, kinds, T, V)).max())
        assert d < tol_f64, (b, d)
        assert np.abs(got.astype(np.float64).sum(1) - 1).max() < 1e-5
        worst = max(worst, d)
    return worst


# ------------------------------------------------------------------------------------------------------------ dense
@pytest.mark.parametrize("mode", ("fp16", "bf16", "fp32x"))
@pytest.mark.parametrize("B,pad", [(2, 0), (3, 4)])
def test_dense_bitwise(tiny, tiny_oracle, mode, B, pad):
    model = tiny[mode]
    inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, B, 16, 12, seed=31 + B, pad=pad)]
    attn = _dense(model, inp)
    rel = model.attention_relevance(attn)
    torch.cuda.synchronize()
    assert rel.shape == (B, 2, 16 + _task(model) + 12)
    _check_refs(model, attn, rel, packed=False)
    # padded positions (text: input_mask with the task row's 1 prepended; image: image_mask) are exactly 0
    tmask = torch.cat([torch.ones(B, 1, dtype=inp[4].dtype, device=inp[4].device), inp[4]], 1) if _task(model) else inp[4]
    real = torch.cat([tmask.bool(), inp[5].bool()], 1)
    assert (~real).any()
    assert torch.equal(rel.permute(1, 0, 2)[:, ~real], torch.zeros(2, int((~real).sum()), device=rel.device))


def test_heads_all_and_mean_same_bits(tiny, tiny_oracle):
    model = tiny["bf16"]
    inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 2, 9, 7, seed=5, pad=2)]
    samples = support.batch(model, [(4, 9), (13, 2)], seed=3)
    full_d = model.attention_relevance(_dense(model, inp))
    full_p = model.attention_relevance(_packed(model, samples))
    model.set_option("attention_heads", 1)
    try:
        mean_d = model.attention_relevance(_dense(model, inp))
        mean_p = model.attention_relevance(_packed(model, samples))
    finally:
        model.set_option("attention_heads", 0)
    torch.cuda.synchronize()
    assert torch.equal(full_d, mean_d)
    for a, b in zip(full_p, mean_p):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ packed
def _packed(model, samples):
    out = model.forward_packed(*support.packed_sample_args(samples), output_all_attention_masks=True)
    torch.cuda.synchronize()
    return out[9]


def _alone(model, smp):
    """Relevance of a batch-1 dense forward of one packed sample: [2, T + V]."""
    return model.attention_relevance(support.dense_alone(model, smp, output_all_attention_masks=True)[9])[0]


LENS = [(1, 40), (31, 1), (12, 64), (5, 17)]


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_packed_bitwise_and_alone(tiny, mode):
    model = tiny[mode]
    samples = support.batch(model, LENS, seed=11)
    attn = _packed(model, samples)
    rel = model.attention_relevance(attn)
    torch.cuda.synchronize()
    assert len(rel) == len(LENS)
    assert len({r.untyped_storage().data_ptr() for r in rel}) == 1          # views of one buffer
    _check_refs(model, attn, rel, packed=True)
    for b, smp in enumerate(samples):
        assert torch.equal(rel[b], _alone(model, smp)), b


def test_regions_packed_bitwise(tiny):
    model = tiny["bf16"]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = []
    for i, (tin, n) in enumerate([(7, 3), (1, 30), (20, 9)]):
        g = torch.Generator().manual_seed(70 + i)
        q, seg = torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g)
        f = torch.relu(torch.randn(n, F, generator=g))
        x1, y1 = torch.rand(n, generator=g) * 400, torch.rand(n, generator=g) * 300
        imgs.append((q, seg, f, torch.stack([x1, y1, x1 + 100, y1 + 80], 1), i + 1))
    cat = lambda k: torch.cat([im[k] for im in imgs], dim=0).cuda()
    (out, _) = model.forward_regions_packed(cat(0), cat(1), torch.tensor([[im[4]] for im in imgs]).cuda(), cat(2), cat(3),
                                            torch.tensor([[640.0, 480.0]] * 3).cuda(), [len(im[0]) for im in imgs],
                                            [im[2].shape[0] for im in imgs], output_all_attention_masks=True)
    rel = model.attention_relevance(out[9])
    torch.cuda.synchronize()
    assert [r.shape[-1] for r in rel] == [len(im[0]) + _task(model) + im[2].shape[0] + 1 for im in imgs]
    _check_refs(model, out[9], rel, packed=True)


def test_long_rows(tiny_oracle):
    """Past 256 rows (max_rows_per_sample 1024): bitwise against the restatement, each packed sample equal to its dense forward
    alone, and within the derived L1 bound of float64."""
    from oracle import vilbert_ref as R
    oracle = R.build(R.tiny_config(max_position_embeddings=1024), seed=7, num_labels=200)
    model = support.engine(oracle, compute_dtype="bf16", max_rows_per_sample=1024, return_attention=True)
    try:
        samples = support.batch(model, [(300, 20), (10, 1024), (3, 3)], seed=50)
        attn = _packed(model, samples)
        rel = model.attention_relevance(attn)
        torch.cuda.synchronize()
        kinds = _kinds(model)
        n_steps = len(kinds) - kinds.count(3)
        for b, smp in enumerate(samples):
            T, V = len(smp[0]) + _task(model), smp[2].shape[0]
            maps = sample_maps(attn, b)
            bound = n_steps * (max(T, V) + max(m.shape[0] for m in maps) + 2) * U
            got = rel[b].cpu().numpy()
            assert np.array_equal(got, attention_relevance_f32(maps, kinds, T, V)), b
            assert np.abs(got - attention_relevance_f64(maps, kinds, T, V)).sum(1).max() < bound, b
            assert torch.equal(rel[b], _alone(model, smp)), b
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------------ full model
def test_full_model_bf16(full_oracle, parity_log):
    from oracle import vilbert_ref as R
    model = support.engine(full_oracle, compute_dtype="bf16", return_attention=True)
    try:
        kinds = _kinds(model)
        assert len(kinds) == 30
        # the demo's largest shape, dense with padding: (Tin, V) = (37, 101)
        inp = [t.cuda() for t in R.make_inputs(2, 37, 101, seed=808, pad_regions=3)]
        attn = _dense(model, inp)
        rel = model.attention_relevance(attn)
        torch.cuda.synchronize()
        worst = _check_refs(model, attn, rel, packed=False)
        parity_log(test="relevance_full_bf16_vs_f64", max_abs_err=worst)
        # the oracle's fp32 maps of the same inputs through the float64 product
        with torch.no_grad():
            ref_attn = full_oracle(*[t.cpu() for t in inp], output_all_attention_masks=True)[9]
        d_oracle = 0.0
        for b in range(2):
            maps = sample_maps(ref_attn, b)
            T, V = maps[kinds.index(0)].shape[-1], maps[kinds.index(1)].shape[-1]
            d_oracle = max(d_oracle, float(np.abs(rel[b].cpu().numpy() - attention_relevance_f64(maps, kinds, T, V)).max()))
        parity_log(test="relevance_full_bf16_vs_oracle_maps", max_abs_err=d_oracle)
        assert d_oracle < TOL_ORACLE, d_oracle
        # packed samples == each sample's dense forward alone
        samples = support.batch(model, [(37, 101), (5, 10), (20, 36)], seed=90)
        prel = model.attention_relevance(_packed(model, samples))
        for b, smp in enumerate(samples):
            assert torch.equal(prel[b], _alone(model, smp)), b
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------------ raw calls
def _raw_args(model, attn):
    from vilbert_b200 import model as M
    entries, packed, t_rows, v_rows = M.relevance_entries(attn, _kinds(model))
    tin = [t - _task(model) for t in t_rows]
    if packed:
        layout = [(h, o) for h, _, o in model.attention_layout_packed(tin, v_rows)[0]]
        nt, nv = (C.c_int32 * len(tin))(*tin), (C.c_int32 * len(tin))(*v_rows)
    else:
        layout = [(h, o) for h, _, _, _, o in model.attention_layout(len(tin), tin[0], v_rows[0])[0]]
        nt, nv = (C.c_int32 * 1)(tin[0]), (C.c_int32 * 1)(v_rows[0])
    n = sum(2 * (t + v) for t, v in zip(t_rows, v_rows))
    return M.maps_pointer(entries, packed, layout), len(tin), nt, nv, int(packed), n


def _call(model, ptr, B, nt, nv, packed, out):
    L = support.lib()
    stream = torch.cuda.current_stream().cuda_stream
    return L.load().vb200_attention_relevance(model._handle, C.c_void_p(ptr), B, C.cast(nt, C.c_void_p), C.cast(nv, C.c_void_p),
                                              packed, C.c_void_p(out.data_ptr() if out is not None else None), C.c_void_p(stream))


def test_every_float_written_maps_unchanged_repeatable(tiny, tiny_oracle):
    model = tiny["fp16"]
    for attn in (_dense(model, [t.cuda() for t in support.tiny_inputs(tiny_oracle, 3, 10, 9, seed=2, pad=3)]),
                 _packed(model, support.batch(model, LENS, seed=4))):
        ptr, B, nt, nv, packed, n = _raw_args(model, attn)
        flat = attn[0] if not packed else attn[0][0]
        storage = flat.untyped_storage()
        before = torch.empty(storage.nbytes() // 4, dtype=torch.float32, device="cuda")
        before.untyped_storage().copy_(storage)
        plans = support.n_plans(model)
        outs = [torch.full((n,), float("nan"), device="cuda") for _ in range(3)]
        for o in outs:                                         # back to back, no synchronisation in between
            assert _call(model, ptr, B, nt, nv, packed, o) == 0
        torch.cuda.synchronize()
        assert not torch.isnan(outs[0]).any()
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
        after = torch.empty_like(before)
        after.untyped_storage().copy_(storage)
        assert torch.equal(before, after)
        assert support.n_plans(model) == plans


def test_rejections_leave_output_untouched(tiny, tiny_oracle):
    L = support.lib()
    model = tiny["fp16"]
    attn = _packed(model, support.batch(model, LENS, seed=4))
    ptr, B, nt, nv, packed, n = _raw_args(model, attn)
    out = torch.full((n,), SENTINEL, device="cuda")

    def rejected(rc, needle):
        assert rc == -1
        assert needle in L.load().vb200_last_error(model._handle).decode()
        torch.cuda.synchronize()
        assert bool((out == SENTINEL).all())

    bad = (C.c_int32 * B)(*nt)
    bad[2] = 0
    rejected(_call(model, ptr, B, bad, nv, 1, out), "n_tokens")
    big = (C.c_int32 * B)(*nv)
    big[1] = 257                                                 # past max_rows_per_sample 256
    rejected(_call(model, ptr, B, nt, big, 1, out), "too long")
    rejected(_call(model, ptr, 0, nt, nv, 1, out), "batch")
    rejected(_call(model, 0, B, nt, nv, 1, out), "NULL")
    rejected(_call(model, ptr, B, nt, nv, 2, out), "packed")
    assert L.load().vb200_attention_relevance(model._handle, C.c_void_p(ptr), B, None, None, 1, C.c_void_p(out.data_ptr()), None) == -1
    assert _call(model, ptr, B, nt, nv, 1, None) == -1
    model.set_option("attention_entries", ((1 << 30) - 1) & ~(1 << 3))
    try:
        rejected(_call(model, ptr, B, nt, nv, 1, out), "entry 3 ")
        sel = model.forward_packed(*support.packed_sample_args(support.batch(model, LENS, seed=4)), output_all_attention_masks=True)[9]
        with pytest.raises(ValueError, match="None"):
            model.attention_relevance(sel)
    finally:
        model.set_option("attention_entries", (1 << len(_kinds(model))) - 1)
    assert _call(model, ptr, B, nt, nv, 1, out) == 0
    torch.cuda.synchronize()
    assert not bool((out == SENTINEL).any())


def test_pretraining_engine():
    import vilbert_b200 as vb
    from oracle import pretraining_ref as P
    from oracle import vilbert_ref as R
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    model = vb.BertForMultiModalPreTraining.from_pretrained(oracle.state_dict(), config=cfg, return_attention=True).eval().cuda(0)
    try:
        inp = list(R.make_inputs(2, 10, 6, seed=4, vocab_size=cfg.vocab_size))
        inp[1] = inp[1][..., :cfg.v_feature_size].contiguous()
        attn = model(*[t.cuda() for t in inp[:6]], output_all_attention_masks=True)[3]
        rel = model.attention_relevance(attn)
        torch.cuda.synchronize()
        _check_refs(model, attn, rel, packed=False)
    finally:
        model.close()
