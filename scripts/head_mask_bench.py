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
    from vilbert_b200 import synthetic as S
    from vilbert_b200.model import head_mask_shape
    from bench import ClockSampler

    if not torch.cuda.is_available():
        raise SystemExit("head_mask_bench.py needs an H100: there is no CPU path")
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = vb.VILBertForVLTasks.from_pretrained(S.synthetic_state_dict(cfg, seed=42), config=cfg, num_labels=3129,
                                                 compute_dtype="bf16").eval().cuda(0)
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

    def timed(fn, steps):
        for _ in range(args.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / steps

    out = {k: fn().clone() for k, fn in paths.items()}
    torch.cuda.synchronize()
    diff = float((out["ungated"] - out["gated_ones"]).abs().max())
    ms = {k: [] for k in paths}
    clock = ClockSampler(0)
    clock.start()
    for _ in range(args.rounds):
        for k, fn in paths.items():
            ms[k].append(timed(fn, args.steps))
    clock.stop_flag = True
    clock.join()

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

    try:
        import pynvml as nv_
        nv_.nvmlInit()
        h = nv_.nvmlDeviceGetHandleByIndex(0)
        name = nv_.nvmlDeviceGetName(h)
        card = {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv_.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception as e:          # NVML missing: report it
        card = {"name": torch.cuda.get_device_name(0), "nvml_error": repr(e)}
    card.update(clock.result())
    print(json.dumps({"workload": f"full synthetic model, bf16, packed VQA forward, batch {B}, {TIN} tokens, {V} regions, seed {args.seed}",
                      **{f"{k}_ms": statistics.median(v) for k, v in ms.items()}, "windows_ms": ms, "device": device, "max_abs_diff": diff,
                      "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
