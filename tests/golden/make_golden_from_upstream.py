"""Re-pin the oracle against the REAL upstream model the day it is importable.

    python tests/golden/make_golden_from_upstream.py [--checkpoint save/multitask_model/pytorch_model_9.bin]
                                                     [--config config/bert_base_6layer_6conect.json]

Status today: "parity unpinned".  The hot path's arithmetic lives in the third-party package `vilbert`
(facebookresearch/vilbert-multi-task, imported at worker.py:44-46, un-vendored and unpinned); neither it nor its
dependencies (pytorch_transformers, easydict) nor the checkpoint `pytorch_model_9.bin` (worker.py:470) exist on the build box, so
tests/golden/full_*.npz hold the outputs of oracle/vilbert_ref.py -- our restatement -- not of the reference.

What this script does on a box where `import vilbert.vilbert` works:

1. builds upstream `VILBertForVLTasks` exactly as the worker does (worker.py:495-536: `BertConfig.from_json_file` or the dict below,
   `v_target_size = 1601`, `task_specific_tokens = True`, `visualization = True`, `from_pretrained(..., num_labels=3129)`, `.eval()`),
   on CPU in fp32, loading either the real checkpoint (`--checkpoint`) or the seeded synthetic state_dict the test-suite uses
   (oracle.init_weights, seed 42 -- same key names, so `load_state_dict(strict=True)` doubles as a key audit of SURVEY.md 8b);
2. runs it on the seeded inputs of make_golden.py's CASES through the worker's positional call (worker.py:286-289);
3. compares every output with oracle/vilbert_ref.py on the same weights and inputs and prints the max abs difference per output
   (expected: fp32 round-off, ~1e-5; anything larger names the first mis-restated module through the per-layer taps);
4. writes `tests/golden/upstream_B*_T*_V*.npz` -- reference-generated fixtures.  tests/test_oracle.py::test_upstream_golden and
   tests/test_gpu_model.py::test_full_model_golden pick up every `*.npz` in this directory, so committing those files turns
   "parity: partial (unpinned)" into reference-pinned parity for both the oracle and the CUDA engine.

Without `vilbert` the script exits 3 after printing what is missing (the CPU test-suite asserts exactly that behaviour, so the
recipe cannot rot silently).
"""
import argparse
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

UPSTREAM_MODULES = ("vilbert.vilbert", "pytorch_transformers", "easydict")
OUT_NAMES = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction",
             "vision_prediction", "vision_logit", "linguisic_prediction", "linguisic_logit"]
KEEP = (0, 1, 2, 3, 4, 6, 8)          # the heads make_golden.py stores (the two pre-training heads are [B,T,30522]-sized)


def missing_modules():
    out = []
    for m in UPSTREAM_MODULES:
        try:
            importlib.import_module(m)
        except Exception as e:      # noqa: BLE001 -- any import-time failure means "not usable here"
            out.append(f"{m}: {type(e).__name__}: {e}")
    return out


def build_upstream(config_path, checkpoint, num_labels, oracle_model):
    """worker.py:495-536, on CPU."""
    import torch
    from vilbert.vilbert import BertConfig, VILBertForVLTasks
    if config_path:
        config = BertConfig.from_json_file(config_path)                      # worker.py:495
    else:
        config = BertConfig.from_dict(oracle_model.config.to_dict())
    config.v_target_size = 1601                                              # worker.py:512-514 (predict_feature False)
    config.predict_feature = False
    config.task_specific_tokens = True                                       # worker.py:516-517
    config.dynamic_attention = False                                         # worker.py:484, 519
    config.visualization = True                                              # worker.py:522
    if checkpoint:
        model = VILBertForVLTasks.from_pretrained(checkpoint, config=config, num_labels=num_labels, default_gpu=True)
        sd = {k[7:] if k.startswith("module.") else k: v for k, v in torch.load(checkpoint, map_location="cpu").items()}
    else:
        model = VILBertForVLTasks(config, num_labels=num_labels, default_gpu=True)
        sd = oracle_model.state_dict()
        missing, unexpected = model.load_state_dict(sd, strict=False)
        if missing or unexpected:
            raise SystemExit(f"key audit failed against upstream: missing {list(missing)[:8]} unexpected {list(unexpected)[:8]}")
    return model.eval(), sd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checkpoint", default="")
    ap.add_argument("--config", default="")
    ap.add_argument("--tol", type=float, default=1e-4, help="max abs difference oracle vs upstream that still counts as pinned")
    args = ap.parse_args()
    miss = missing_modules()
    if miss:
        print("upstream model not importable on this box -- parity stays unpinned:\n  " + "\n  ".join(miss))
        print("install facebookresearch/vilbert-multi-task (+ pytorch_transformers, easydict) and re-run; see the module docstring")
        return 3
    import numpy as np
    import torch
    from oracle import vilbert_ref as R
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from make_golden import CASES
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    oracle = R.build(seed=42)
    upstream, sd = build_upstream(args.config, args.checkpoint, oracle.num_labels, oracle)
    if args.checkpoint:
        oracle.load_state_dict(sd, strict=True)            # the oracle must accept the real checkpoint key for key
    here = os.path.dirname(os.path.abspath(__file__))
    worst = 0.0
    report = {}
    for B, Tin, V, seed, pad in CASES:
        inp = R.make_inputs(B, Tin, V, seed=seed, pad_regions=pad)
        with torch.no_grad():
            up = upstream(*inp, output_all_attention_masks=True)            # worker.py:286-289
            ours = oracle(*inp, compute_pretraining_heads=True, output_all_attention_masks=True)
        d = {}
        for i in range(9):
            diff = float((up[i].float() - ours[i]).abs()[ours[i].abs() < 1000].max())
            report[f"B{B}_T{Tin}_V{V}/{OUT_NAMES[i]}"] = diff
            worst = max(worst, diff)
            if i in KEEP:
                d[OUT_NAMES[i]] = up[i].float().numpy().astype(np.float32)
        d.update(B=B, Tin=Tin, V=V, seed=seed, pad=pad, weight_seed=-1 if args.checkpoint else 42)
        fn = os.path.join(here, f"upstream_B{B}_T{Tin}_V{V}.npz")
        np.savez_compressed(fn, **d)
        print("wrote", fn)
    print(json.dumps(report, indent=1))
    print(f"max |oracle - upstream| = {worst:.3e} (tolerance {args.tol:g})")
    if worst >= args.tol:
        print("ORACLE DISAGREES WITH UPSTREAM: fix oracle/vilbert_ref.py (see UPSTREAM_ASSUMPTIONS there) before trusting any parity claim")
        return 1
    print("oracle pinned: commit tests/golden/upstream_*.npz and drop the 'parity unpinned' notes (oracle header, DESIGN.md 1)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
