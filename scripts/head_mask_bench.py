"""Cost of the head gate on the packed forward (one JSON line).

Workload: the full synthetic model in bf16, a batch-64 packed VQA forward (vil_prediction only) at bench.py's default shape, 30
question tokens and 36 regions per sample.  Two paths share one engine:
  (a) forward_packed without a head mask: the ungated PACKED plan, whose attention kernels get no gate;
  (b) forward_packed with an all-ones head mask: the gated plan, one device-to-device copy of the [64, 30, 12] mask, then the same
      kernels reading their gate.
The mask is built once, outside the timed loops.  Each is timed with CUDA events around --steps calls, alternating window by window for
--rounds windows; the median is reported in ms per forward, with the outputs' max absolute difference (0: an all-ones gate gives the
ungated bits).  A separate torch.profiler pass then splits each path's device time per call into its kernels and its copies.  The card name, power limit and the SM
clock sampled while the windows run are read in the same run.

    python scripts/head_mask_bench.py [--steps 200] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

B, TIN, V = 64, 30, 36


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5, help="alternating timing windows per path; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--profile-calls", type=int, default=20, help="calls per path in the profiled pass (device time split)")
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200.model import head_mask_shape

    harness.require_gpu("head_mask_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(args.seed)
    q = torch.randint(1000, cfg.vocab_size, (B * TIN,), generator=g).to(dev)
    f = (torch.relu(torch.randn(B * V, cfg.v_feature_size, generator=g)) * 1.5).to(dev)
    s = torch.rand(B * V, 5, generator=g).to(dev)
    seg, task = torch.zeros(B * TIN, dtype=torch.long, device=dev), torch.ones(B, 1, dtype=torch.long, device=dev)
    ones = torch.ones(B, *head_mask_shape(cfg), device=dev)
    x = (q, f, s, seg, task, [TIN] * B, [V] * B)
    paths = {"ungated": lambda: model.forward_packed(*x, select=vb.OUT_VIL_PREDICTION)[0],
             "gated_ones": lambda: model.forward_packed(*x, select=vb.OUT_VIL_PREDICTION, head_mask=ones)[0]}

    out = {k: fn().clone() for k, fn in paths.items()}
    torch.cuda.synchronize()
    diff = float((out["ungated"] - out["gated_ones"]).abs().max())
    with harness.sampled_clock() as clock:
        ms = harness.alternate(paths, args.rounds, args.steps, args.warmup)

    # device time per call in a separate profiled pass: the kernels' summed time and the copies', per path
    from torch.profiler import ProfilerActivity, profile
    device = {}
    for k, fn in paths.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_calls):
                fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        copy = [e for e in evs if "Memcpy" in e.name or "Memset" in e.name]
        kern = [e for e in evs if e not in copy]
        device[k] = {"kernel_us_per_call": sum(e.device_time for e in kern) / args.profile_calls,
                     "kernels_per_call": len(kern) / args.profile_calls,
                     "copy_us_per_call": sum(e.device_time for e in copy) / args.profile_calls,
                     "copies_per_call": len(copy) / args.profile_calls}

    card = harness.card(clock)
    print(json.dumps({"workload": f"full synthetic model, bf16, packed VQA forward, batch {B}, {TIN} tokens, {V} regions, seed {args.seed}",
                      **{f"{k}_ms": statistics.median(v) for k, v in ms.items()}, "windows_ms": ms, "device": device, "max_abs_diff": diff,
                      "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
