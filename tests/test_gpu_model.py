"""End-to-end parity of the CUDA engine (worker-facing Python protocol -> C ABI -> sm_90a kernels) against the
fp32 CPU oracle on identical seeded inputs.  `-m gpu` only.

Tolerances (BASELINE.json north_star: "within 1e-3 fp32 / 1e-2 bf16 per logit"):

* TOL = 1e-2 per logit against the fp32 oracle -- met by the DEFAULT engine mode (fp16 tensor-core operands,
  fp32 accumulation / residual stream / LayerNorm / softmax; same tensor-core rate as bf16).
* The bf16-operand mode (compute_dtype="bf16") cannot meet 1e-2 against fp32: rounding the ~150 GEMM operands of
  this network to an 8-bit significand moves the VQA logits (std 0.91) by up to ~1.9e-2 in *exact* arithmetic --
  the oracle itself shows it when its activations are rounded to bf16 at the same points
  (oracle.emulate_activation_rounding; tests/test_oracle.py pins that number on CPU).  That mode is therefore checked
  against the fp32 oracle at TOL_BF16_VS_FP32 = 3.5e-2 x max(1, logit std) (i.e. ~2x the format floor).

These bounds see only defects that move the logits by 1-3 %.  How the plan wires the kernels together in both 16-bit modes is
checked step by step in tests/test_gpu_step_parity.py: every layer state against oracle/step_ref.py (fp64, rounded where the
engine rounds) run on the engine's own previous state, at bounds ~4x the measured last-bit disagreement; the op-level tests pin
the kernels themselves.

The synthetic checkpoint is bf16-representable (oracle.init_weights(bf16_exact=True)), so both sides start from
identical parameters.  Measured numbers are appended to gpurun_out/parity.jsonl.
"""
import os

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # north_star, default mode vs fp32 oracle
TOL_BF16_VS_FP32 = 3.5e-2  # bf16 mode vs fp32 oracle, x max(1, logit std): the format floor is ~2 % of the logit spread
                           # (1.9e-2 on the VQA logits with std 0.91, see module docstring / tests/test_oracle.py)
# The distance to the oracle run WITH the same 16-bit rounding points (oracle.emulate_activation_rounding) is logged but not
# asserted: two runs that round at the same places decorrelate after a few layers (any last-bit difference in an fp32
# accumulation flips later roundings), so their distance is ~sqrt(2) x either one's distance to fp32 -- measured 0.026 vs
# 0.019 in bf16 mode.  The emulation's value is the CPU-side floor in tests/test_oracle.py, not a bitwise target.
NAMES = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction",
         "vision_prediction", "vision_logit", "linguisic_prediction", "linguisic_logit"]
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def tiny_engines(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full_engines(full_oracle):
    yield from support.engines(full_oracle, DT)


def _errs(ref, out):
    """max abs error per output, ignoring the -10000 rows of masked regions (checked on a relative scale)."""
    res = {}
    for i, name in enumerate(NAMES):
        r, o = ref[i], out[i]
        if r is None:
            assert o is None, name
            continue
        assert o is not None and tuple(o.shape) == tuple(r.shape), (name, None if o is None else o.shape, r.shape)
        diff = (o.cpu() - r).abs()
        big = r.abs() > 1000
        if big.any():
            assert float((diff[big] / r[big].abs()).max()) < 1e-3, name
        res[name] = (float(diff[~big].max()) if (~big).any() else 0.0, float(r[~big].std()) if (~big).sum() > 1 else 0.0)
    return res


def _check(oracle, engines, inputs, parity_log, tag, pretraining):
    from oracle import vilbert_ref as R
    ref32 = oracle(*inputs, compute_pretraining_heads=pretraining)
    dev = [t.cuda() for t in inputs]
    for mode, eng in engines.items():
        out = eng(*dev, output_all_attention_masks=True, compute_pretraining_heads=pretraining)
        torch.cuda.synchronize()
        assert out[9] == []
        with R.emulate_activation_rounding(oracle, DT[mode]):
            ref_em = oracle(*inputs, compute_pretraining_heads=pretraining)
        e32, eem = _errs(ref32, out), _errs(ref_em, out)

        for name in e32:
            parity_log(test=tag, mode=mode, output=name, err_vs_fp32=e32[name][0], err_vs_emulated=eem[name][0],
                       ref_std=e32[name][1])
        for name in e32:
            tol32 = TOL if mode == "fp16" else TOL_BF16_VS_FP32 * max(1.0, e32[name][1])
            assert e32[name][0] < tol32, f"{tag}/{mode}: {name} vs fp32 oracle: {e32[name][0]} >= {tol32}"


@pytest.mark.parametrize("B,Tin,V,pad", [(2, 30, 36, 0), (3, 16, 10, 3), (4, 37, 101, 7), (1, 12, 37, 0), (2, 128, 100, 0),
                                         (1, 3, 1, 0), (1, 155, 256, 11), (5, 3, 7, 2)])
def test_tiny_model_all_outputs(tiny_oracle, tiny_engines, parity_log, B, Tin, V, pad):
    """Structurally complete 12/6/6 model at reduced width: all nine outputs incl. the pre-training heads, ragged text
    lengths, masked regions, odd batch (binary head falls back to the seq-relationship score), and the corner of the
    BASELINE sweep (text 128, regions 100); extremes: three tokens ([CLS] id [SEP]) + one region, 155 tokens (the tiny model has 160 positions)
    x 256 regions (four key blocks in every attention kernel), an odd batch of tiny sequences."""
    _check(tiny_oracle, tiny_engines, support.tiny_inputs(tiny_oracle, B, Tin, V, 100 + B, pad), parity_log,
           f"tiny_B{B}_T{Tin}_V{V}", pretraining=True)


def test_tiny_model_eager_equals_graph(tiny_oracle, tiny_engines):
    """CUDA-graph replay and eager launches of the same plan give bit-identical outputs."""
    dev = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 2, 20, 12, 5)]
    eager = support.engine(tiny_oracle, use_cuda_graph=False)
    a = tiny_engines["fp16"](*dev)
    b = eager(*dev)
    c = tiny_engines["fp16"](*dev)
    torch.cuda.synchronize()
    for x, y, z in zip(a[:9], b[:9], c[:9]):
        if x is not None:
            assert torch.equal(x, y) and torch.equal(x, z)
    eager.close()


def test_tiny_model_pdl(tiny_oracle, tiny_engines):
    """Programmatic dependent launch changes scheduling only, never results: the default (every kernel), forced on
    (use_pdl=True) and none (use_pdl=False) agree bit for bit."""
    dev = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 2, 20, 12, 6)]
    a = tiny_engines["fp16"](*dev, compute_pretraining_heads=True)
    for mode in (True, False):
        other = support.engine(tiny_oracle, use_pdl=mode)
        for rep in range(3):
            b = other(*dev, compute_pretraining_heads=True)
            torch.cuda.synchronize()
            for x, y in zip(a[:9], b[:9]):
                if x is not None:
                    assert torch.equal(x, y)
        other.close()


def test_tiny_model_host_api(tiny_oracle, tiny_engines):
    """vb200_forward_host (pinned host buffers in/out) == vb200_forward (device pointers)."""
    from vilbert_b200 import _lib as L
    inp = support.tiny_inputs(tiny_oracle, 4, 20, 12, 8)
    eng = tiny_engines["fp16"]
    ref = eng(*[t.cuda() for t in inp])
    hin = [t.pin_memory() for i, t in enumerate(inp) if i != 6]
    out = {"vil_prediction": torch.empty(4, tiny_oracle.num_labels).pin_memory(),
           "vision_logit": torch.empty(4, 12, 1).pin_memory()}
    eng.forward_host(*hin, out, select=L.OUT_VIL_PREDICTION | L.OUT_VISION_LOGIT)
    assert torch.equal(out["vil_prediction"], ref[0].cpu()) and torch.equal(out["vision_logit"], ref[6].cpu())


def test_tiny_model_workspace_slots(tiny_oracle, tiny_engines):
    """vb200_forward_slot / vb200_forward_host_slot: batches in flight on different slots and streams do not disturb each
    other -- every slot returns bit-for-bit what slot 0 returns for the same batch."""
    from vilbert_b200 import _lib as L
    eng = tiny_engines["fp16"]
    batches = [support.tiny_inputs(tiny_oracle, 3, 20, 12, 40 + i, pad=i % 2) for i in range(6)]
    want = []
    for b in batches:
        want.append(eng(*[t.cuda() for t in b])[0].clone())
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    dev = [[t.cuda() for t in b] for b in batches]
    torch.cuda.synchronize()
    for rep in range(3):
        got = []
        for i, d in enumerate(dev):
            with torch.cuda.stream(streams[i % 3]):
                got.append(eng(*d, slot=i % 3)[0].clone())   # clone on the same stream: the slot's buffer is re-used
        torch.cuda.synchronize()
        for w, g in zip(want, got):
            assert torch.equal(w, g)
    # asynchronous host calls, two slots
    hin = [[t.pin_memory() for i, t in enumerate(b) if i != 6] for b in batches]
    houts = [{"vil_prediction": torch.empty(3, tiny_oracle.num_labels).pin_memory()} for _ in batches]
    for i, h in enumerate(hin):
        s = streams[i % 2]
        s.synchronize()
        with torch.cuda.stream(s):
            eng.forward_host(*h, houts[i], select=L.OUT_VIL_PREDICTION, slot=i % 2, synchronize=False)
    torch.cuda.synchronize()
    for w, h in zip(want, houts):
        assert torch.equal(w.cpu(), h["vil_prediction"])
    with pytest.raises(RuntimeError):
        eng(*dev[0], slot=99)


@pytest.mark.parametrize("B,Tin,V,pad", [(1, 30, 36, 0), (2, 30, 36, 0), (3, 37, 101, 5), (2, 16, 10, 0)])
def test_full_model_task_heads(full_oracle, full_engines, parity_log, B, Tin, V, pad):
    from oracle import vilbert_ref as R
    inp = R.make_inputs(B, Tin, V, seed=1234 + B, pad_regions=pad)
    _check(full_oracle, full_engines, inp, parity_log, f"full_B{B}_T{Tin}_V{V}", pretraining=False)


def test_full_model_pretraining_heads(full_oracle, full_engines, parity_log):
    from oracle import vilbert_ref as R
    inp = R.make_inputs(2, 30, 36, seed=77)
    _check(full_oracle, full_engines, inp, parity_log, "full_pretraining", pretraining=True)


def test_full_model_golden(full_engines, parity_log):
    """Committed fixtures (tests/golden/*.npz, made by tests/golden/make_golden.py from the fp32 oracle)."""
    from oracle import vilbert_ref as R
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    files = sorted(f for f in os.listdir(gdir) if f.endswith(".npz"))
    assert files, "no golden fixtures committed"
    for fn in files:
        z = np.load(os.path.join(gdir, fn))
        if int(z["weight_seed"]) != 42:
            continue          # fixtures of a real checkpoint (make_golden_from_upstream.py --checkpoint) need that checkpoint
        B, Tin, V, seed, pad = (int(z[k]) for k in ("B", "Tin", "V", "seed", "pad"))
        inp = R.make_inputs(B, Tin, V, seed=seed, pad_regions=pad)
        out = full_engines["fp16"](*[t.cuda() for t in inp])
        torch.cuda.synchronize()
        for i, name in enumerate(NAMES):
            if name in z.files:
                r = torch.from_numpy(z[name])
                small = r.abs() < 1000
                err = float((out[i].cpu() - r).abs()[small].max())
                parity_log(test="golden:" + fn, output=name, max_abs_err=err)
                assert err < TOL, (fn, name, err)


def test_batch64_shard_equivalence(full_oracle, full_engines, parity_log):
    """Full-size property (SURVEY 8e): a pair's logits do not depend on what else is in the batch --
    B=64 in one call == the same 64 pairs in 4 calls of 16 (what batch sharding over ranks does), bit for bit;
    plus a spot check of 4 of the 64 rows against the oracle (BASELINE.json configs[1] shape)."""
    from oracle import vilbert_ref as R
    eng = full_engines["fp16"]
    inp = R.make_inputs(64, 30, 36, seed=4321, full_masks=False)
    dev = [t.cuda() for t in inp]
    whole = eng(*dev)[0]
    parts = torch.cat([eng(*[t[i:i + 16] for t in dev])[0] for i in range(0, 64, 16)])
    torch.cuda.synchronize()
    d = float((whole - parts).abs().max())
    parity_log(test="batch64_shard_equivalence", max_abs_diff=d)
    assert d == 0.0
    idx = [0, 21, 42, 63]
    ref = full_oracle(*[t[idx] for t in inp], compute_pretraining_heads=False)[0]
    err = float((whole[idx].cpu() - ref).abs().max())
    parity_log(test="batch64_rows_vs_oracle", max_abs_err=err, ref_std=float(ref.std()))
    assert err < TOL


def test_checkpoint_file_ingestion(tiny_oracle, tiny_engines, tmp_path):
    """SURVEY.md 8f-3: the worker's loading path (worker.py:470-536) -- config JSON file + torch-saved flat state_dict with the
    DataParallel `module.` prefix and the tied/unused keys a real checkpoint carries -- gives the same engine as the in-memory
    dict: identical outputs, bit for bit."""
    import json
    import vilbert_b200 as vb
    cfg = tiny_oracle.config.to_dict()
    cfg_path = tmp_path / "bert_base_6layer_6conect.json"
    cfg_path.write_text(json.dumps(cfg))
    sd = {"module." + k: v.clone() for k, v in tiny_oracle.state_dict().items()}
    sd["module.cls.predictions.decoder.weight"] = sd["module.bert.embeddings.word_embeddings.weight"]     # tied copy
    ckpt = tmp_path / "pytorch_model_9.bin"
    torch.save(sd, ckpt)
    # (worker_api.load_vilbert_model forces v_target_size = 1601 as worker.py:513 does, which only fits the full-size
    # checkpoint; this reduced-width model goes through the same from_json_file / from_pretrained(path) calls directly)
    config = vb.BertConfig.from_json_file(str(cfg_path))
    m = vb.VILBertForVLTasks.from_pretrained(str(ckpt), config=config, num_labels=tiny_oracle.num_labels, default_gpu=True)
    m.eval()
    m.cuda(0)
    dev = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 3, 20, 12, 77, pad=1)]
    a = tiny_engines["fp16"](*dev, compute_pretraining_heads=True)
    b = m(*dev, compute_pretraining_heads=True)
    torch.cuda.synchronize()
    for x, y in zip(a[:9], b[:9]):
        assert torch.equal(x, y)
    m.close()
    sd.pop("module.bert.t_pooler.dense.bias")
    torch.save(sd, ckpt)
    with pytest.raises(RuntimeError, match="t_pooler.dense.bias"):
        vb.VILBertForVLTasks.from_pretrained(str(ckpt), config=config, num_labels=tiny_oracle.num_labels).cuda(0)
