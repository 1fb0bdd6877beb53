"""Cost of attention maps by selection on the packed detector-output path (one JSON line).

Workload: packed_attention_bench.py's -- batch 64 VQA rows in the given dtype (default bf16), U{5..20} question tokens, U{10..100}
detector boxes per image, forward_regions_packed at fixed capacities 37 tokens / 100 boxes.  Four variants of the same call on one
engine, the map selection set (vb200_set_option "attention_entries" / "attention_heads") before each window:
  no_maps        -- output_all_attention_masks=False;
  all_maps       -- every entry, every head (the default selection);
  connection     -- the 12 connection-layer entries (both directions of the 6 connection layers), every head;
  t2i_mean       -- the 6 text->image connection entries, averaged over heads.
The variants alternate window by window after every plan is warm; each is timed with CUDA events around a loop of whole calls and the
median of --rounds windows is reported, with the fp32 map floats written per call and, from a torch.profiler pass of its own, the
device time per call of the probability kernels (attention_f32_kernel / attention_f32_mean_kernel).  The card name, power limit and
the SM clock sampled while the windows run are read in the same run.

    python scripts/attention_maps_bench.py [--batch 64] [--steps 50] [--dtype bf16]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import harness  # noqa: E402

T_CAP, BOX_CAP = 37, 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5, help="alternating timing windows per variant; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from packed_attention_bench import detector_rows

    harness.require_gpu("attention_maps_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype, return_attention=True)
    rows = detector_rows(args.batch, args.seed, cfg.v_feature_size, cfg.vocab_size)
    B = len(rows)
    tin, nb = [len(r[0]) for r in rows], [r[1].shape[0] for r in rows]
    dev = torch.device("cuda", 0)
    pq = torch.cat([r[0] for r in rows]).to(dev)
    packed_in = (pq, torch.zeros_like(pq), torch.ones(B, 1, dtype=torch.long, device=dev), torch.cat([r[1] for r in rows]).to(dev),
                 torch.cat([r[2] for r in rows]).to(dev), torch.tensor([list(r[3]) for r in rows]).to(dev), tin, nb)

    kinds, _ = model.attention_selection()
    full = (1 << len(kinds)) - 1
    conn = sum(1 << e for e, k in enumerate(kinds) if k >= 2)
    t2i = sum(1 << e for e, k in enumerate(kinds) if k == 2)
    # variant -> (maps, attention_entries, attention_heads)
    variants = {"no_maps": (False, full, 0), "all_maps": (True, full, 0), "connection": (True, conn, 0), "t2i_mean": (True, t2i, 1)}

    def select(name):
        _, mask, heads = variants[name]
        model.set_option("attention_entries", mask)
        model.set_option("attention_heads", heads)

    def call(name):
        return model.forward_regions_packed(*packed_in, select=vb.OUT_VIL_PREDICTION, max_tokens=T_CAP, max_boxes=BOX_CAP,
                                            return_spatials=False, output_all_attention_masks=variants[name][0])

    floats, logits = {}, {}
    for name, (maps, _, _) in variants.items():
        select(name)
        floats[name] = model.attention_layout_packed(tin, [n + 1 for n in nb])[1] if maps else 0
        logits[name] = call(name)[0][0]
    torch.cuda.synchronize()
    for name in variants:
        if not torch.equal(logits[name], logits["no_maps"]):
            raise SystemExit(f"VQA logits of {name} differ from the call without maps")

    def timed(name):
        select(name)
        return harness.timed(lambda: call(name), args.steps, args.warmup)

    with harness.sampled_clock() as clock:
        ms = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k in variants:
                ms[k].append(timed(k))

    from torch.profiler import ProfilerActivity, profile

    def map_kernel_ms(name, n=5):
        """Device ms per call of the probability kernels, from CUPTI kernel records."""
        select(name)
        call(name)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                call(name)
            torch.cuda.synchronize()
        t = 0.0
        for ev in prof.key_averages():
            d = getattr(ev, "device_time_total", None)
            d = ev.cuda_time_total if d is None else d
            if "attention_f32" in ev.key and ev.device_type is not None and "cuda" in str(ev.device_type).lower():
                t += d
        return t / n / 1e3
    kernel_ms = {k: map_kernel_ms(k) for k in variants}

    card = harness.card(clock)
    result = {k: {"ms_per_call": statistics.median(v), "windows_ms": v, "map_floats_per_call": floats[k],
                  "device_ms_per_call_map_kernels": kernel_ms[k]} for k, v in ms.items()}
    print(json.dumps({"workload": f"batch {B} VQA rows, U{{5..20}} tokens, U{{10..100}} boxes, seed {args.seed}, {args.dtype}, "
                                  f"forward_regions_packed at capacities {T_CAP} / {BOX_CAP}", **result, "steps": args.steps,
                      "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
