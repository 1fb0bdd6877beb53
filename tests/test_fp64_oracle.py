"""The fp64 oracle and the bounds of tests/test_gpu_fp32x_fp64.py, on CPU.

* The oracles run end to end in fp64 (``oracle.fp64.fp64``) and the fp32 oracle sits within 1e-5 of that run on every output and the
  final states, 1e-6 on the attention maps: the fp32 floor the fp32-parity mode is measured against.
* The bounds can see the defects: one-line wiring mistakes of the fp32-parity mode (a 16-bit rounding where a hi/lo split belongs, the
  polynomial or tanh GELU in place of erf), restated here as hooks and patches on the fp64 oracle, move its outputs by at least twice
  the bound of every check family that must catch them (``oracle.fp64.BOUNDS``, one set for both models).  A change that loosens
  a bound fails here unless this catalog is revisited.
"""
import math

import pytest
import torch
from torch import nn

from oracle import fp64 as X
from oracle import vilbert_ref as R
import support

FLOOR = 1e-5             # fp32 oracle vs fp64 oracle: outputs and final states (rel_err)
FLOOR_ATTENTION = 1e-6   # ... and attention maps (max abs)


def _run(model, inp, pretraining=True):
    collect = {}
    out = model(*inp, compute_pretraining_heads=pretraining, output_all_attention_masks=True, collect=collect)
    return out, collect["final"]


def _taps(final):
    t, v, pt, pv = final
    return {"sequence_output_t": t, "sequence_output_v": v, "pooled_output": pt * pv}


def _errs(model, a, b):
    """(worst output rel_err, worst state rel_err, [(map, err)] of the attention maps) between two runs ``_run`` returned."""
    (oa, fa), (ob, fb) = a, b
    return (max(X.output_errs(oa, ob).values()), max(X.state_errs(_taps(fa), fb).values()),
            X.attention_errs(oa[9], ob[9], model.bert.encoder.schedule()))


@pytest.fixture(scope="module")
def tiny64(tiny_oracle):
    return X.fp64(tiny_oracle)


# ------------------------------------------------------------------ the fp64 oracle
def test_fp64_copy_leaves_the_oracle(tiny_oracle, tiny64):
    assert all(p.dtype == torch.float32 for p in tiny_oracle.parameters())
    assert all(p.dtype == torch.float64 for p in tiny64.parameters())
    assert tiny64.cls.predictions.decoder.weight is tiny64.bert.embeddings.word_embeddings.weight          # still tied
    for (n, p), q in zip(tiny_oracle.state_dict().items(), tiny64.state_dict().values()):
        assert torch.equal(p.double(), q), n


def test_fp64_oracle_runs_in_fp64(tiny64):
    inp = support.tiny_inputs(tiny64, 3, 16, 10, 9, pad=3)
    out, final = _run(tiny64, inp)
    for i, name in enumerate(X.OUTPUT_NAMES):
        assert out[i].dtype == torch.float64, name
    assert all(x.dtype == torch.float64 for x in final)
    assert all(p.dtype == torch.float64 for a in out[9] for p in (a if isinstance(a, tuple) else (a,)))
    assert float(out[6][:, -3:].max()) < -9000                       # the masked regions' vision_logit rows
    # float64 inputs give the same run as the float32 inputs converted inside the oracle
    again, _ = _run(tiny64, [t.double() if t.is_floating_point() else t for t in inp])
    for a, b in zip(out[:9], again[:9]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ the fp32 floor
def _check_floor(oracle, oracle64, inp, tag):
    out, s, attn = _errs(oracle, _run(oracle, inp), _run(oracle64, inp))
    worst_map = max(attn, key=lambda x: x[1])
    print(f"FLOOR {tag}: outputs {out:.2e}  states {s:.2e}  attention {worst_map[1]:.2e} ({worst_map[0]})")
    assert out < FLOOR and s < FLOOR, (tag, out, s)
    assert X.first_over(attn, FLOOR_ATTENTION) is None, (tag, X.first_over(attn, FLOOR_ATTENTION))


@pytest.mark.parametrize("B,Tin,V,pad", [(2, 30, 36, 0), (3, 16, 10, 3), (1, 12, 37, 0), (4, 37, 101, 7), (2, 70, 100, 0)])
def test_fp32_floor_tiny(tiny_oracle, tiny64, B, Tin, V, pad):
    _check_floor(tiny_oracle, tiny64, support.tiny_inputs(tiny_oracle, B, Tin, V, 500 + B, pad), f"tiny_B{B}_T{Tin}_V{V}")


def test_fp32_floor_full(full_oracle):
    _check_floor(full_oracle, X.fp64(full_oracle), R.make_inputs(2, 30, 36, seed=808, pad_regions=3), "full_B2_T30_V36")


def test_fp32_floor_pretraining_losses():
    from oracle import pretraining_ref as P
    from vilbert_b200 import synthetic as S
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    c = oracle.config
    b = S.synthetic_masked_batch(4, 36, 37, seed=9, vocab_size=c.vocab_size, v_feature_size=c.v_feature_size,
                                 v_target_size=c.v_target_size)
    args = [b[k] for k in ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask",
                           "masked_lm_labels", "image_label", "image_target", "next_sentence_label")]
    ref = X.fp64(oracle)(*args[:8], args[8].double(), args[9])
    got = oracle(*args)
    for g, r in zip(got, ref):
        assert r.dtype == torch.float64 and X.rel_err(g, r) < FLOOR, (float(g), float(r))


# ------------------------------------------------------------------ the defect catalog
def _round16(x):
    return x.half().to(x.dtype)


def _gelu_act1(x):
    """The GEMM epilogue's polynomial GELU (act 1, csrc/common.cuh gelu_erf): x * sat(0.5 + x Q(x^2)), Q of degree 8."""
    q = torch.full_like(x, 4.547042257e-11)
    u = x * x
    for c in (-4.515281038e-09, 1.986152114e-07, -5.147503089e-06, 8.848903963e-05, -1.079077483e-03, 9.718777612e-03,
              -6.619028002e-02, 3.988192081e-01):
        q = q * u + c
    return x * (0.5 + x * q).clamp(0.0, 1.0)


def _gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def _round_input(model, names):
    for name in names:
        model.get_submodule(name).register_forward_pre_hook(lambda _m, args: (_round16(args[0]),) + args[1:])


def _round_output(model, pred):
    for name, m in model.named_modules():
        if isinstance(m, nn.Linear) and pred(name):
            m.register_forward_hook(lambda _m, _a, out: _round16(out))


def _round_params(model, names):
    with torch.no_grad():
        for name in names:
            p = model.get_parameter(name)
            p.copy_(_round16(p))


def _context_inputs(model):
    names = [n + ".output.dense" for n, m in model.named_modules() if isinstance(m, R._Attention)]
    return names + [n + d for n, m in model.named_modules() if isinstance(m, R.BertBiOutput) for d in (".dense1", ".dense2")]


EMB = "bert.embeddings."
# name -> (what it does to the fp64 oracle, the check families that must see it)
DEFECTS = {
    "Q and K rounded to fp16": (lambda m, mp: _round_output(m, lambda n: n.rsplit(".", 1)[-1] in ("query", "key", "query1", "key1",
                                                                                                     "query2", "key2")),
                                ("attention",)),
    "act-1 polynomial GELU instead of act 3": (lambda m, mp: mp.setattr(R, "gelu", _gelu_act1), ("logits", "states")),
    "5-d box operand in fp16, no lo part": (lambda m, mp: _round_input(m, ["bert.v_embeddings.image_location_embeddings"]),
                                            ("logits", "states")),
    "tanh GELU instead of erf": (lambda m, mp: mp.setattr(R, "gelu", _gelu_tanh), ("logits", "states")),
    "Linear biases rounded to fp16": (lambda m, mp: _round_params(m, [n + ".bias" for n, x in m.named_modules()
                                                                      if isinstance(x, nn.Linear) and x.bias is not None]),
                                      ("logits", "states")),
    "classifier input (the pooled product) rounded to fp16": (lambda m, mp: _round_input(m, [h + ".logit_fc.0" for h in (
        "vil_prediction", "vil_prediction_gqa", "vil_binary_prediction")]), ("logits",)),
    "position table rounded to fp16": (lambda m, mp: _round_params(m, [EMB + "position_embeddings.weight"]), ("logits", "states")),
    "attention context rounded to fp16": (lambda m, mp: _round_input(m, _context_inputs(m)), ("logits", "states")),
    "word / position / type tables rounded to fp16": (lambda m, mp: _round_params(m, [EMB + t + "_embeddings.weight" for t in
                                                                                      ("word", "position", "token_type")]),
                                                      ("logits", "states")),
    "region features in fp16, no lo part": (lambda m, mp: _round_input(m, ["bert.v_embeddings.image_embeddings"]), ("logits", "states")),
}


@pytest.fixture(scope="module")
def catalog_run(tiny64):
    inp = support.tiny_inputs(tiny64, 4, 37, 101, 504, pad=7)
    return inp, _run(tiny64, inp)


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_bounds_see_the_defect(tiny_oracle, catalog_run, monkeypatch, defect):
    apply, families = DEFECTS[defect]
    inp, clean = catalog_run
    model = X.fp64(tiny_oracle)
    apply(model, monkeypatch)
    out, s, attn = _errs(model, _run(model, inp), clean)
    moved = {"logits": out, "states": s, "attention": max(e for _, e in attn)}
    print(f"DEFECT {defect}: " + "  ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    for fam in families:
        assert moved[fam] >= 2 * X.BOUNDS[fam], (defect, fam, moved[fam], X.BOUNDS[fam])
