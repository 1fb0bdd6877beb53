"""The model-level numerics checks at checkpoint-like weights (oracle/trained_like.py): peaked and sink attention, GELU past its
saturation, outlier channels.  `-m gpu` only.

The cases and references are those of tests/test_gpu_step_parity.py, tests/test_gpu_fp32x_fp64.py and
tests/test_gpu_attention_relevance.py; only the weights differ:

* step parity in fp16 and bf16 (``StepRef`` teacher-forced on the engine's states): reduced-width dense shapes with padding and
  several key blocks, forward_packed and forward_regions_packed, sequences past 256 rows, the 268 M model at B = 2, held to
  ``step_ref.STEP_BOUNDS_TRAINED`` (the maps family logged only: near-tied sharp heads flip on one-ulp Q / K disagreements);
  the head-mean maps against the fp64 mean of the engine's per-head maps;
* fp32x against the fp64 oracle on both models, held to ``fp64.BOUNDS_TRAINED`` (peaked attention amplifies fp32 rounding, the
  fp32 oracle's own included, past ``fp64.BOUNDS``);
* relevance: bit-identical to the float32 restatement on the engine's peaked maps, and within the derived L1 bound of the float64
  definition on the fp32 oracle's maps;
* the regime itself on the engine's own maps, so a generator that drifts back to near-uniform attention fails here.
"""
import numpy as np
import pytest
import torch

import test_gpu_step_parity as P
from oracle import fp64 as X
from oracle import step_ref as S
from oracle import trained_like as TL
from relevance_ref import attention_relevance_f32, attention_relevance_f64, sample_maps

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16")
TINY_DENSE = [(4, 37, 101, 7), (1, 155, 256, 11), (2, 30, 36, 0), (3, 16, 10, 3)]
U = 2.0 ** -24


def _measured(model, name):
    """The weights the trained-regime bounds were measured on, bit for bit (trained_like.DIGESTS)."""
    assert TL.digest(model) == TL.DIGESTS[name], f"trained_like({name}) differs from the weights the bounds were measured on"
    return model


@pytest.fixture(scope="module")
def tiny_t(tiny_oracle):
    return _measured(TL.trained_like(tiny_oracle, TL.SEED), "tiny")


@pytest.fixture(scope="module")
def full_t(full_oracle):
    return _measured(TL.trained_like(full_oracle, TL.SEED), "full")


@pytest.fixture(scope="module")
def tiny(tiny_t):
    e = {m: P.engine(tiny_t, m) for m in MODES + ("fp32x",)}
    yield e
    for m in e.values():
        m.close()


def _assert(tag, mode, result, parity_log):
    fails = []
    for fam, errs in result.items():
        if not errs:
            continue
        bound = S.STEP_BOUNDS_TRAINED[mode][P.family(fam)]
        w = S.worst(errs)
        parity_log(test=f"trained_step_parity_{tag}_{mode}", family=fam, max_err=w[1], worst_step=w[0], where=w[2], bound=bound)
        if bound is None:           # the maps family: logged, no bound at these weights (step_ref.STEP_BOUNDS_TRAINED)
            continue
        first = S.first_over(errs, bound)
        if first is not None:
            fails.append((fam, first, bound))
    assert not fails, "; ".join(f"{fam}: first over {bound:g} at {lab} ({where}): {e:.3e}" for fam, (lab, e, where), bound in fails)


# ------------------------------------------------------------------------------------------------------------ step parity
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,Tin,V,pad", TINY_DENSE)
def test_step_parity_dense(tiny, tiny_t, mode, B, Tin, V, pad, parity_log):
    inp = P.tiny_inputs(tiny_t, B, Tin, V, seed=2000 + 7 * B + Tin, pad=pad)
    _assert(f"tiny_B{B}_T{Tin}_V{V}_pad{pad}", mode, P.run_dense(tiny[mode], tiny_t, mode, inp), parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_step_parity_packed_and_regions(tiny, tiny_t, mode, parity_log):
    model = tiny[mode]
    _assert("tiny_packed", mode, P.run_packed(model, tiny_t, mode, P.packed_samples(model, P.PACKED_LENS, 2100)), parity_log)
    imgs = P.region_images(model, P.REGION_LENS, 2200) + P.region_images(model, [P.REGION_LENS[0]], 2250)
    _assert("tiny_regions", mode, P.run_regions(model, tiny_t, mode, imgs), parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_step_parity_past_256_rows(mode, parity_log):
    oracle = _measured(TL.trained_like(P.long_oracle(), TL.SEED), "long")
    model = P.engine(oracle, mode, max_rows_per_sample=1024)
    try:
        for Tin, V in P.LONG:
            inp = P.tiny_inputs(oracle, 2, Tin, V, seed=2300 + Tin, pad=5)
            _assert(f"long_T{Tin}_V{V}", mode, P.run_dense(model, oracle, mode, inp), parity_log)
    finally:
        model.close()


@pytest.mark.parametrize("mode", MODES)
def test_step_parity_full_model(full_t, mode, parity_log):
    from oracle import vilbert_ref as R
    model = P.engine(full_t, mode)
    try:
        _assert("full_B2", mode, P.run_dense(model, full_t, mode, R.make_inputs(2, 30, 101, seed=2400, pad_regions=4)), parity_log)
    finally:
        model.close()


@pytest.mark.parametrize("mode", MODES)
def test_head_mean_maps(tiny, tiny_t, mode, parity_log):
    """The head-mean maps (attention_heads = 1) on peaked maps: the same forward's states bit for bit, and each map within float32
    rounding (heads + 1 ulps of 1) of the fp64 mean over heads of the engine's own per-head maps."""
    model = tiny[mode]
    inp = P.tiny_inputs(tiny_t, 2, 70, 101, seed=2500, pad=3)
    dev = [t.cuda() for t in inp]
    full, states = model(*dev, output_all_attention_masks=True, output_layer_states=True)
    model.set_option("attention_heads", 1)
    try:
        res, states2 = model(*dev, output_all_attention_masks=True, output_layer_states=True)
    finally:
        model.set_option("attention_heads", 0)
    torch.cuda.synchronize()
    for a, b in zip(states, states2):
        assert torch.equal(a, b)
    worst = ("", 0.0)
    for lab, got, heads in zip(S.map_labels(tiny_t.bert.encoder.schedule()), S.flat_maps(res[9]), S.flat_maps(full[9])):
        mean = heads.double().mean(1)
        e = float((got.double().reshape(mean.shape) - mean).abs().max())
        bound = (heads.shape[1] + 1) * 2.0 ** -23
        assert e < bound, (lab, e, bound)
        worst = max(worst, (lab, e), key=lambda x: x[1])
    parity_log(test=f"trained_head_mean_maps_{mode}", max_err=worst[1], worst_step=worst[0])


# ------------------------------------------------------------------------------------------------------------ fp32x vs fp64
def _fp32x_check(o64, eng, inp, tag, parity_log):
    collect = {}
    ref = o64(*inp, compute_pretraining_heads=True, output_all_attention_masks=True, collect=collect)
    out, taps = eng(*[t.cuda() for t in inp], compute_pretraining_heads=True, output_all_attention_masks=True, debug_taps=True)
    torch.cuda.synchronize()
    fams = {"logits": X.output_errs(out, ref), "states": X.state_errs(taps, collect["final"]),
            "attention": dict(X.attention_errs(out[9], ref[9], o64.bert.encoder.schedule()))}
    over = {}
    for fam, errs in fams.items():
        for name, e in errs.items():
            parity_log(test="trained_fp32x_vs_fp64_" + tag, family=fam, output=name, err_vs_fp64=e, bound=X.BOUNDS_TRAINED[fam])
            if not e < X.BOUNDS_TRAINED[fam]:
                over.setdefault(fam, {})[name] = e
    assert not over, f"{tag}: over fp64.BOUNDS_TRAINED: {over}"


@pytest.mark.parametrize("B,Tin,V,pad", [(4, 37, 101, 7), (1, 155, 256, 11), (2, 30, 36, 0)])
def test_fp32x_tiny(tiny, tiny_t, B, Tin, V, pad, parity_log):
    _fp32x_check(X.fp64(tiny_t), tiny["fp32x"], P.tiny_inputs(tiny_t, B, Tin, V, 2600 + B, pad), f"tiny_B{B}_T{Tin}_V{V}", parity_log)


def test_fp32x_full_model(full_t, parity_log):
    from oracle import vilbert_ref as R
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(full_t.config.to_dict())
    eng = vb.VILBertForVLTasks.from_pretrained(full_t.state_dict(), config=cfg, num_labels=full_t.num_labels, compute_dtype="fp32x",
                                               return_attention=True).eval().cuda(0)
    try:
        _fp32x_check(X.fp64(full_t), eng, R.make_inputs(2, 30, 101, seed=2700, pad_regions=3), "full_B2", parity_log)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------ relevance
def _l1_bound(kinds, maps, T, V):
    """n_steps (L + heads + 2) u: tests/test_gpu_attention_relevance.py's derivation of the float32 rollout's L1 error."""
    n_steps = len(kinds) - kinds.count(3)
    return n_steps * (max(T, V) + max(m.shape[0] for m in maps) + 2) * U


@pytest.mark.parametrize("mode", ("fp16", "bf16", "fp32x"))
def test_relevance_on_peaked_maps(tiny, tiny_t, mode, parity_log):
    """The engine's relevance, bit-identical to the float32 restatement on its own peaked maps and within the derived bound of the
    float64 definition on them; and on the fp32 oracle's maps of the same inputs, the float32 restatement within that bound of the
    float64 definition (the rollout's rounding at sink-heavy maps)."""
    model = tiny[mode]
    inp = P.tiny_inputs(tiny_t, 2, 70, 101, seed=2800, pad=4)
    out = model(*[t.cuda() for t in inp], output_all_attention_masks=True)
    rel = model.attention_relevance(out[9])
    torch.cuda.synchronize()
    kinds = model.attention_selection()[0]
    with torch.no_grad():
        ref_attn = tiny_t(*inp, output_all_attention_masks=True)[9]
    worst = 0.0
    for b in range(2):
        maps = sample_maps(out[9], b)
        T, V = maps[kinds.index(0)].shape[-1], maps[kinds.index(1)].shape[-1]
        got = rel[b].cpu().numpy()
        assert np.array_equal(got, attention_relevance_f32(maps, kinds, T, V)), b
        bound = _l1_bound(kinds, maps, T, V)
        d = float(np.abs(got - attention_relevance_f64(maps, kinds, T, V)).sum(1).max())
        assert d < bound, (b, d, bound)
        omaps = sample_maps(ref_attn, b)
        od = float(np.abs(attention_relevance_f32(omaps, kinds, T, V) - attention_relevance_f64(omaps, kinds, T, V)).sum(1).max())
        assert od < bound, (b, od, bound)
        worst = max(worst, d, od)
        # the sinks carry the flow: relevance is far from uniform over the rows
        assert got.max() > 5.0 / (T + V), got.max()
    parity_log(test=f"trained_relevance_{mode}_l1_vs_f64", max_err=worst)


# ------------------------------------------------------------------------------------------------------------ the regime
@pytest.mark.parametrize("mode", MODES)
def test_engine_maps_are_in_the_regime(tiny, tiny_t, mode):
    """The attention targets on the engine's own element-9 maps: a peaked head in every layer and direction, the model's median row
    max, winners past the first key block, and a sink head on each stream's key 0."""
    model = tiny[mode]
    inp = P.tiny_inputs(tiny_t, 2, 100, 101, seed=11, pad=5)          # tests/test_trained_like.py's attention inputs
    out = model(*[t.cuda() for t in inp], output_all_attention_masks=True)
    torch.cuda.synchronize()
    t_real, v_real = TL.real_rows(inp)
    reg = TL.attention_regime(out[9], tiny_t.bert.encoder.schedule(), t_real, v_real)
    TL.assert_attention_targets(reg)
