"""Checkpoint-like weights (oracle/trained_like.py) on CPU: the targets on the fp32 oracle for both model sizes, determinism, the
state_dict contract, and the defect catalog of oracle/step_ref.py at these weights.

* Targets: peaked attention in every layer and direction, sink heads on each stream's key 0, winners past the first 64-key block,
  FFN pre-activations past the polynomial GELU's saturation, LayerNorm and residual outlier channels, every 16-bit operand <= 4096.
* The catalog: ``step_ref.DEFECTS_TRAINED`` (the synthetic-weight catalog and the QKV bias added after rounding), fed the fp64
  oracle's own states on the 268 M model as tests/test_step_ref.py runs it, each moving its families by at least twice
  ``step_ref.STEP_BOUNDS_TRAINED`` in the modes it lists; the other ``NOT_SEPARABLE`` entries are printed, and each must stay under
  twice the states bound (one that grows past it belongs in the catalog).
"""
import hashlib

import pytest
import torch

from oracle import fp64 as X
from oracle import step_ref as S
from oracle import trained_like as TL
from oracle import vilbert_ref as R

TG = TL.TARGETS


@pytest.fixture(scope="module")
def tiny_t(tiny_oracle):
    return TL.trained_like(tiny_oracle, TL.SEED)


@pytest.fixture(scope="module")
def full_t(full_oracle):
    return TL.trained_like(full_oracle, TL.SEED)


def _inputs(oracle, B, Tin, V, seed, pad=0):
    inp = list(R.make_inputs(B, Tin, V, seed=seed, vocab_size=oracle.config.vocab_size, pad_regions=pad))
    inp[1] = inp[1][..., :oracle.config.v_feature_size].contiguous()
    return inp


def _digest(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


# ------------------------------------------------------------------------------------------------------------ targets
@pytest.mark.parametrize("size", ("tiny", "full"))
def test_targets(size, tiny_t, full_t, tiny_oracle, full_oracle):
    """Every target on the fp32 oracle, on inputs other than the calibration batch: the issue's (2, 30, 36) batch for the
    activation targets, and 100 tokens x 101 regions (both streams past one key block) for the attention ones."""
    m, base = (tiny_t, tiny_oracle) if size == "tiny" else (full_t, full_oracle)
    sched = m.bert.encoder.schedule()
    act, _ = TL.activation_regime(m, _inputs(m, 2, 30, 36, seed=1))
    long_inp = _inputs(m, 2, 100, 101, seed=11, pad=5)
    act_l, out = TL.activation_regime(m, long_inp)
    reg = TL.attention_regime(out[9], sched, *TL.real_rows(long_inp))
    base_reg = TL.attention_regime(base(*long_inp, output_all_attention_masks=True)[9], sched, *TL.real_rows(long_inp))
    print(f"TARGETS {size}: median row max {reg['model_rowmax']:.3f} (synthetic weights {base_reg['model_rowmax']:.3f}), "
          f"rows won past key 63 {reg['late']:.3f}")
    for lab, e in reg["maps"].items():
        print(f"  {lab:>16}: sharpest head {max(e['rowmax']):.3f}  sink {max(e['sink']):.3f}")
    TL.assert_attention_targets(reg)
    for a in (act, act_l):
        share = min(v[0] for v in a["ffn"].values())
        top = min(v[1] for v in a["ffn"].values())
        print(f"  FFN: smallest share past {TG['gelu_sat']} {share:.4f}, smallest max |x| {top:.1f}; LayerNorm input max "
              f"{a['ln_in']}; state max {a['state_max']}; largest 16-bit operand {a['operand_max']:.1f}")
        assert share >= TG["gelu_sat_share"] and top >= TG["gelu_max"], a["ffn"]
        for stream in ("text", "image"):
            assert a["ln_in"][stream] >= TG["residual_outlier"], (stream, a["ln_in"])
            assert a["state_max"][stream] >= TG["operand_outlier"], (stream, a["state_max"])
        assert a["operand_max"] <= TG["operand_max"], a["operand_max"]
    lo, hi = TG["ln_outlier"]
    for text in (True, False):
        for ln in TL._stream_layernorms(m, text):
            big = (ln.bias.abs() >= lo) & (ln.bias.abs() <= hi)
            assert int(big.sum()) >= TL.LN_OUTLIERS, int(big.sum())


# ------------------------------------------------------------------------------------------------------------ contract
def test_deterministic(tiny_oracle, tiny_t):
    """The same seed gives the same state_dict bit for bit; another seed does not; the source oracle is left as it was."""
    before = _digest(tiny_oracle.state_dict())
    again = TL.trained_like(tiny_oracle, TL.SEED)
    assert _digest(again.state_dict()) == _digest(tiny_t.state_dict())
    assert _digest(TL.trained_like(tiny_oracle, TL.SEED + 1).state_dict()) != _digest(tiny_t.state_dict())
    assert _digest(tiny_oracle.state_dict()) == before


@pytest.mark.parametrize("size", ("tiny", "full"))
def test_state_dict_contract(size, tiny_t, full_t, tiny_oracle, full_oracle):
    """Key names, shapes and dtypes of the oracle's state_dict, Linear weights bf16-representable, and the engine's from_pretrained
    takes it without a device (as tests/test_model_without_engine.py builds models)."""
    import vilbert_b200 as vb
    m, base = (tiny_t, tiny_oracle) if size == "tiny" else (full_t, full_oracle)
    sd, ref = m.state_dict(), base.state_dict()
    assert list(sd) == list(ref)
    for k in ref:
        assert sd[k].shape == ref[k].shape and sd[k].dtype == ref[k].dtype, k
        assert torch.isfinite(sd[k]).all(), k
    for name, mod in m.named_modules():
        if isinstance(mod, torch.nn.Linear):
            assert torch.equal(mod.weight, mod.weight.to(torch.bfloat16).float()), name
    cfg = vb.BertConfig.from_dict(m.config.to_dict())
    model = vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=m.num_labels).eval()
    assert model is not None


# ------------------------------------------------------------------------------------------------------------ defect catalog
# As tests/test_step_ref.py: the 268 M model, B = 2, 30 tokens and 101 regions with 7 padded, one text, one connection and one
# image layer, each fed the fp64 oracle's own states.
@pytest.fixture(scope="module")
def catalog(full_t):
    inp = R.make_inputs(2, 30, 101, seed=904, pad_regions=7)
    states, _, final, _ = _oracle_run(X.fp64(full_t), inp)
    tm, vm = S.key_masks(inp[4], inp[5])
    cache = {}

    def run(mode, defects=()):
        key = (mode, tuple(defects))
        if key not in cache:
            ref = S.StepRef(full_t, mode, defects)
            outs, maps = S.forced_steps(ref, states, tm, vm, ("T0", "C0", "V0"))
            t, v, pt, pv = final
            cache[key] = (outs, maps, ref.pooled(t[:, 0], v[:, 0]), ref.outputs(pt * pv, t, v, vm))
        return cache[key]
    return run


def _oracle_run(oracle64, inp):
    collect = {}
    with torch.no_grad():
        out = oracle64(*inp, compute_pretraining_heads=True, output_all_attention_masks=True, collect=collect)
    t, v = collect["emb"]
    states = [t, v]
    for step in oracle64.bert.encoder.schedule():
        t, v = collect[step]
        states += ([t] if step[0] != "V" else []) + ([v] if step[0] != "T" else [])
    return states, out[9], collect["final"], out[:9]


def _moved(a, b):
    return {"states": max(X.rel_err(x, y) for x, y in zip(b[0], a[0])),
            "maps": max(float((x - y).abs().max()) for x, y in zip(b[1], a[1])),
            "pooled": X.rel_err(b[2], a[2]),
            "logits": max(X.rel_err(x, y) for x, y in zip(b[3], a[3]))}


def _report(catalog, mode, defect):
    moved = _moved(catalog(mode), catalog(mode, (defect,)))
    b = S.STEP_BOUNDS_TRAINED[mode]
    print(f"TRAINED DEFECT {mode} {defect}: " + "  ".join(f"{k} {v:.2e}" + (f" ({v / b[k]:.1f}x bound)" if b[k] else " (no bound)")
                                                         for k, v in moved.items()))
    return moved


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("defect", list(S.DEFECTS_TRAINED))
def test_bounds_see_the_defect(catalog, mode, defect):
    desc, families, modes = S.DEFECTS_TRAINED[defect]
    moved = _report(catalog, mode, defect)
    if mode not in modes:
        pytest.skip(f"{desc}: not separable from the {mode} trained bounds (step_ref.DEFECTS_TRAINED)")
    for fam in families:
        assert moved[fam] >= 2 * S.STEP_BOUNDS_TRAINED[mode][fam], (desc, fam, moved[fam], S.STEP_BOUNDS_TRAINED[mode][fam])


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("defect", [d for d in S.NOT_SEPARABLE if d not in S.DEFECTS_TRAINED])
def test_not_separable_defects(catalog, mode, defect):
    moved = _report(catalog, mode, defect)
    assert moved["states"] < 2 * S.STEP_BOUNDS_TRAINED[mode]["states"], (defect, moved)

