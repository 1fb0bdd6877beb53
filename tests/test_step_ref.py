"""The one-step fp64 reference of the 16-bit engine (oracle/step_ref.py) and the bounds tests/test_gpu_step_parity.py holds the
engine to, on CPU.

* Restatement: with every rounding switched off, each step of ``StepRef`` equals the fp64 oracle's own module on the oracle's
  ``collect`` states to 1e-12, heads included, on the reduced-width and the 268 M model with padded batches.
* Attention: the block-wise attention equals ``kernel_refs.attention_emulated`` bit for bit on one key block, and past 64 keys it
  stays within the rounding floor of tests/test_kernel_refs.py against fp64.
* Defect catalog: each one-line mistake of ``step_ref.DEFECTS``, fed the fp64 oracle's own states, moves every check family that
  must catch it by at least twice that family's bound (``step_ref.STEP_BOUNDS``).  Each defect's end-to-end movement of the nine
  outputs (the defect in every step) is printed next to the end-to-end tolerances of tests/test_gpu_model.py.
"""
import pytest
import torch

from oracle import fp64 as X
from oracle import kernel_refs as K
from oracle import step_ref as S
from oracle import vilbert_ref as R
import support

EXACT = 1e-12
E2E_TOL = {"fp16": 1e-2, "bf16": 3.5e-2}    # tests/test_gpu_model.py: fp16 max abs, bf16 max abs / max(1, logit std)


def _oracle_run(oracle64, inp):
    """The fp64 oracle's full state list, attention maps, final states and outputs on ``inp``."""
    collect = {}
    with torch.no_grad():
        out = oracle64(*inp, compute_pretraining_heads=True, output_all_attention_masks=True, collect=collect)
    t, v = collect["emb"]
    states = [t, v]
    for step in oracle64.bert.encoder.schedule():
        t, v = collect[step]
        states += ([t] if step[0] != "V" else []) + ([v] if step[0] != "T" else [])
    return states, out[9], collect["final"], out[:9]


def _masks(inp, task_tokens=True):
    return S.key_masks(inp[4], inp[5], task_tokens)


# ------------------------------------------------------------------------------------------------------------ restatement
def _check_restatement(oracle, inp, tag):
    o64 = X.fp64(oracle)
    states, maps, final, outs = _oracle_run(o64, inp)
    ref = S.StepRef(oracle)
    tm, vm = _masks(inp, oracle.config.task_specific_tokens)
    emb_t = ref.text_embed(inp[0], inp[3], inp[7])
    emb_v = ref.image_embed(inp[1], inp[2])
    res = S.teacher_forced(ref, states, emb_t, emb_v, tm, vm, maps)
    assert len(res["states"]) == len(states) and len(res["maps"]) == len(S.flat_maps(maps))
    for fam in ("states", "maps"):
        w = S.worst(res[fam])
        print(f"RESTATEMENT {tag} {fam}: {w[1]:.1e} ({w[0]})")
        assert S.first_over(res[fam], EXACT) is None, (tag, fam, S.first_over(res[fam], EXACT))
    t, v, pt, pv = final
    assert X.rel_err(ref.pooled(t[:, 0], v[:, 0]), pt * pv) < EXACT
    got = ref.outputs(pt * pv, t, v, vm)
    errs = X.output_errs(got, outs)
    print(f"RESTATEMENT {tag} outputs: {max(errs.values()):.1e}")
    assert max(errs.values()) < EXACT, errs


@pytest.mark.parametrize("B,Tin,V,pad", [(3, 16, 10, 3), (4, 37, 101, 7), (1, 3, 1, 0), (5, 70, 66, 2)])
def test_restatement_tiny(tiny_oracle, B, Tin, V, pad):
    _check_restatement(tiny_oracle, support.tiny_inputs(tiny_oracle, B, Tin, V, 900 + B, pad), f"tiny_B{B}_T{Tin}_V{V}")


def test_restatement_full(full_oracle):
    _check_restatement(full_oracle, R.make_inputs(2, 30, 36, seed=901, pad_regions=3), "full_B2_T30_V36")


def test_restatement_regions(tiny_oracle):
    """The image embedding from forward_regions' operand rows (kernel_refs.region_rows) is the oracle's on the same rows."""
    import numpy as np
    g = np.random.default_rng(5)
    F = tiny_oracle.config.v_feature_size
    feats = np.maximum(g.standard_normal((7, F)), 0).astype(np.float32)
    xy = g.uniform(0, 300, (7, 2)).astype(np.float32)
    boxes = np.concatenate([xy, xy + 50], 1)
    rows, loc, _ = K.region_rows(feats, boxes, 640.0, 480.0, 5)
    rows, loc = torch.from_numpy(rows)[None], torch.from_numpy(loc)[None]
    o64 = X.fp64(tiny_oracle)
    with torch.no_grad():
        want = o64.bert.v_embeddings(rows.double(), loc.double())
    assert X.rel_err(S.StepRef(tiny_oracle).image_embed(rows, loc), want) < EXACT


# ------------------------------------------------------------------------------------------------------------ attention
def _attn_inputs(L, d, f16, seed):
    heads = 2
    H = heads * d
    g = torch.Generator().manual_seed(seed)
    dt = torch.float16 if f16 else torch.bfloat16
    qkv = torch.randn(2, L, 3 * H, generator=g).to(dt)
    mask = torch.zeros(2, L)
    mask[0, 1:L:3] = -10000.0
    mask[1, L // 2 + 1:] = -10000.0
    return qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:], mask, heads


@pytest.mark.parametrize("L,d", [(1, 64), (16, 64), (17, 128), (31, 64), (64, 128)])
@pytest.mark.parametrize("f16", (True, False))
def test_blockwise_attention_is_the_emulation_on_one_block(L, d, f16):
    q, k, v, mask, heads = _attn_inputs(L, d, f16, L + d)
    got = S.attention_blockwise(q, k, v, mask, heads, f16)
    assert torch.equal(got, K.attention_emulated(q, k, v, mask, heads, f16))


@pytest.mark.parametrize("L,d", [(65, 128), (100, 64), (129, 128), (256, 64), (301, 64)])
def test_blockwise_attention_floor_past_one_block(L, d):
    """Past 64 keys, against fp64, within half the bounds tests/test_kernel_refs.py test_attention_rounding_floor holds the
    one-block emulation to; and without rounding it is softmax(Q K^T / sqrt(d) + mask) V itself."""
    for f16, bound in ((False, 1.2e-2), (True, 1.5e-3)):
        q, k, v, mask, heads = _attn_inputs(L, d, f16, L + d)
        ref = K.attention_fp64(q, k, v, mask, heads)
        err = ((S.attention_blockwise(q, k, v, mask, heads, f16) - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
        assert err < bound / 2, (f16, err)
        assert (S.attention_blockwise(q, k, v, mask, heads) - ref).abs().max().item() < EXACT


# ------------------------------------------------------------------------------------------------------------ defect catalog
# Per step on the 268 M model (its steps carry the largest measured engine values, so the bounds are set by it): B = 2, 30 tokens
# (T = 31) and 101 regions with 7 padded -- two image key blocks, keys past pad16 boundaries, padded image keys.  A defect acts
# alike in every layer of a kind, so one text, one connection and one image layer run.  End to end on the reduced-width model
# (every step on the reference's own previous output): B = 4, 37 tokens, 101 regions, 7 padded.
CATALOG_STEPS = ("T0", "C0", "V0")


def _catalog(oracle, inp, only):
    states, _, final, _ = _oracle_run(X.fp64(oracle), inp)
    tm, vm = _masks(inp)
    cache = {}

    def run(mode, defects=()):
        """(entries, maps, pooled, outputs) of StepRef(mode, defects) fed the fp64 oracle's states, the outputs from the oracle's
        final states and pooled product."""
        key = (mode, tuple(defects))
        if key not in cache:
            ref = S.StepRef(oracle, mode, defects)
            outs, maps = S.forced_steps(ref, states, tm, vm, only)
            t, v, pt, pv = final
            cache[key] = (outs, maps, ref.pooled(t[:, 0], v[:, 0]), ref.outputs(pt * pv, t, v, vm))
        return cache[key]
    return run


@pytest.fixture(scope="module")
def catalog(full_oracle):
    return _catalog(full_oracle, R.make_inputs(2, 30, 101, seed=904, pad_regions=7), CATALOG_STEPS)


@pytest.fixture(scope="module")
def end_to_end(tiny_oracle):
    inp = support.tiny_inputs(tiny_oracle, 4, 37, 101, seed=905, pad=7)
    tm, vm = _masks(inp)
    cache = {}

    def run(mode, defects=()):
        key = (mode, tuple(defects))
        if key not in cache:
            ref = S.StepRef(tiny_oracle, mode, defects)
            tc, vc = ref.text_embed(inp[0], inp[3], inp[7]), ref.image_embed(inp[1], inp[2])
            for step in ref.schedule:
                if step[0] == "C":
                    tc, vc, _ = ref.connection(int(step[1:]), tc, vc, tm, vm)
                elif step[0] == "T":
                    tc = ref.layer(step, tc, tm)[0]
                else:
                    vc = ref.layer(step, vc, vm)[0]
            cache[key] = ref.outputs(ref.pooled(tc[:, 0], vc[:, 0]), tc, vc, vm)
        return cache[key]
    return run


def _moved(a, b):
    """How far run b moves each family from run a."""
    return {"states": max(X.rel_err(x, y) for x, y in zip(b[0], a[0])),
            "maps": max(float((x - y).abs().max()) for x, y in zip(b[1], a[1])),
            "pooled": X.rel_err(b[2], a[2]),
            "logits": max(X.rel_err(x, y) for x, y in zip(b[3], a[3]))}


def _e2e(a, b, mode):
    """The largest end-to-end movement of the nine outputs as a multiple of its tests/test_gpu_model.py tolerance (max abs, rows
    past 1000 excluded; bf16 x max(1, std))."""
    worst = (0.0, "")
    for name, x, y in zip(X.OUTPUT_NAMES, b, a):
        small = y.abs() < 1000
        d = float((x - y).abs()[small].max())
        tol = E2E_TOL[mode] * (max(1.0, float(y[small].std())) if mode == "bf16" else 1.0)
        worst = max(worst, (d / tol, name))
    return worst


def _report(catalog, end_to_end, mode, defect):
    moved = _moved(catalog(mode), catalog(mode, (defect,)))
    ratio, name = _e2e(end_to_end(mode), end_to_end(mode, (defect,)), mode)
    print(f"DEFECT {mode} {defect}: " + "  ".join(f"{k} {v:.2e} ({v / S.STEP_BOUNDS[mode][k]:.1f}x bound)" for k, v in moved.items())
          + f"  | end to end {ratio:.2f}x the tolerance ({name}){'  -- under the end-to-end bound' if ratio < 1 else ''}")
    return moved


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("defect", list(S.DEFECTS))
def test_bounds_see_the_defect(catalog, end_to_end, mode, defect):
    desc, families, modes = S.DEFECTS[defect]
    moved = _report(catalog, end_to_end, mode, defect)
    if mode not in modes:
        pytest.skip(f"{desc}: not separable from the {mode} bounds (step_ref.DEFECTS)")
    for fam in families:
        assert moved[fam] >= 2 * S.STEP_BOUNDS[mode][fam], (desc, fam, moved[fam], S.STEP_BOUNDS[mode][fam])


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("defect", list(S.NOT_SEPARABLE))
def test_not_separable_defects_stay_below_the_bounds(catalog, end_to_end, mode, defect):
    """The defects left out of the catalog: printed, and each still under twice its family's bound -- should one grow past it (a
    bound tightened, say), it belongs in the catalog."""
    moved = _report(catalog, end_to_end, mode, defect)
    assert moved["states"] < 2 * S.STEP_BOUNDS[mode]["states"], (defect, moved)


def test_clean_runs_sit_at_the_format_floor(catalog):
    """Sanity of the catalog's baseline: the fp16 and bf16 references sit at their format floors from the fp64 oracle's states."""
    exact = catalog(None)
    for mode, floor in (("fp16", 1e-2), ("bf16", 5e-2)):
        moved = _moved(exact, catalog(mode))
        assert moved["states"] < floor, (mode, moved)
