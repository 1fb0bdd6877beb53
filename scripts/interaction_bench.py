"""Shapley-Taylor pair indices against Shapley values alone on the same message (one JSON line).

Workload: the full synthetic model in bf16, one VQA message of 37 question tokens and 100 detector boxes, the default units (one per
question position 1 .. 35 and one per box: n = 135), P = 8 antithetic permutations, and Q = 128 pairs: the first 8 word units with
the first 16 box units, a word x box grid a user would inspect.
  (a) model.shapley: v(empty), v(all) and the P (n - 1) chain coalitions, then the Shapley estimator.
  (b) model.shapley_interactions: the same chains plus two coalitions per permutation and pair, then both estimators.
Each is timed with CUDA events around --steps calls, alternating window by window; the median of --rounds windows is reported as ms
per message.  The forward samples of each path are the engine's layout counts (computed, not timed): 2 + P (n - 1) and
2 + P (n - 1) + 2 P Q, plus the full input once more for every call past the first at 1024 samples.  The estimator kernel
(vb200_interaction_values) is timed alone with CUDA events over --kernel-iters launches on values of the call's size, and its numpy
restatement (model.interaction_reference) with the host clock, for scale.  The card name, power limit and the SM clock sampled while
the windows run are read in the same run.

    python scripts/interaction_bench.py [--steps 2] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

TIN, BOXES, P = 37, 100, 8
WORDS, BOX_UNITS = 8, 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timing windows per path; the median is reported")
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import numpy as np
    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    from vilbert_b200 import model as M

    harness.require_gpu("interaction_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(args.seed)
    bx = harness.pixel_boxes(g, BOXES)
    feats = torch.relu(torch.randn(BOXES, cfg.v_feature_size, generator=g)) * 1.5
    q = torch.randint(1000, cfg.vocab_size, (TIN,), generator=g)
    x = (q.to(dev), torch.zeros(TIN, dtype=torch.long, device=dev), torch.tensor([[1]], device=dev), feats.to(dev), bx.to(dev),
         torch.tensor([[640.0, 480.0]], device=dev), [TIN], [BOXES])
    msgs = [("vqa", 0, 1)]
    units = M.coalition_units(None, TIN, BOXES)
    n = len(units)
    words = [u for u, (ps, bs) in enumerate(units) if ps][:WORDS]
    boxes = [u for u, (ps, bs) in enumerate(units) if bs][:BOX_UNITS]
    pairs = [(w, b) for w in words for b in boxes]
    Q = len(pairs)

    def shapley():
        return model.shapley(*x, msgs, permutations=P, seed=args.seed)

    def interactions():
        return model.shapley_interactions(*x, msgs, [pairs], permutations=P, seed=args.seed)

    a, b = shapley()[0], interactions()[0]
    torch.cuda.synchronize()
    assert torch.equal(a["phi"], b["phi"]), "shapley_interactions' phi differs from shapley's"
    with harness.sampled_clock() as clock:
        ms = harness.alternate({"shapley": shapley, "shapley_interactions": interactions}, args.rounds, args.steps, args.warmup)
    ms = {k: [t / len(msgs) for t in v] for k, v in ms.items()}

    # the estimator alone: the call's permutations and pairs, values of the call's size (its time does not depend on them)
    perm = b["perm"].numpy()
    pr = np.ascontiguousarray(b["pairs"].numpy(), dtype=np.int32)
    vals = np.random.default_rng(args.seed).random(2 + P * (n - 1) + 2 * P * Q).astype(np.float32)
    perm_d = torch.from_numpy(perm.reshape(-1)).to(device=dev, dtype=torch.int32)
    vals_d = torch.from_numpy(vals).to(dev)
    inter, se = torch.empty(Q, device=dev), torch.empty(Q, device=dev)
    arr = (L.InteractionMessage * 1)(L.InteractionMessage(n, P, 2, Q, 0, 0, 0, pr.ctypes.data))

    def kernel():
        model._call("vb200_interaction_values", arr, 1, perm_d.data_ptr(), vals_d.data_ptr(), inter.data_ptr(), se.data_ptr())

    kernel_us = harness.timed(kernel, args.kernel_iters, 10) * 1000.0
    want = M.interaction_reference(vals, perm, pr, 2)
    assert np.array_equal(inter.cpu().numpy(), want[0]) and np.array_equal(se.cpu().numpy(), want[1])
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        M.interaction_reference(vals, perm, pr, 2)
    numpy_us = (time.perf_counter() - t0) / reps * 1e6

    card = harness.card(clock)
    chain = 2 + P * (n - 1)
    print(json.dumps({"workload": f"full synthetic model, bf16, one VQA message, {TIN} tokens and {BOXES} boxes, default units (n = {n}), "
                                  f"P = {P} antithetic, Q = {Q} pairs ({WORDS} word units x {BOX_UNITS} box units), seed {args.seed}",
                      "shapley_samples": a["samples"], "interaction_samples": b["samples"],
                      "shapley_samples_formula": chain, "interaction_samples_formula": chain + 2 * P * Q,
                      "shapley_ms_per_message": statistics.median(ms["shapley"]),
                      "interactions_ms_per_message": statistics.median(ms["shapley_interactions"]),
                      "windows_ms": ms, "estimator_kernel_us": kernel_us, "estimator_numpy_us": numpy_us,
                      "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
