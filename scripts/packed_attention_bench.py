"""Cost of the attention maps (element 9 of the 10-tuple) on the detector-output path, packed and dense (one JSON line).

Workload (seeded): batch 64 VQA rows in the given dtype (default bf16), questions of U{5..20} real tokens, U{10..100} detector boxes
per image -- the regions_packed_bench.py detector workload with shorter questions.  Three arms over the same rows, timed as whole calls
with CUDA events in alternating windows after every plan they use is warm (median of --rounds):
  packed       -- forward_regions_packed, no maps (fixed capacities 37 tokens / 100 boxes);
  packed_maps  -- the same call with output_all_attention_masks=True (VB200_OUT_ATTENTION_PACKED): every sample's maps at its own
                  T_i / V_i, written straight into one flat buffer;
  dense_maps   -- forward_regions with output_all_attention_masks=True, padded to the batch's longest question and largest box count.
Reported per arm: ms per call (device events around a loop of whole calls: when the host side of a call is the slower part, this
is the host's rate), the fp32 map floats written per call, and -- from a torch.profiler pass of its own after the timing windows -- the
device time per call of all device activity (kernels and copies) and of the probability kernels (attention_f32_kernel) alone.  For packed_maps the host time of
split_packed_attention (the flat buffer -> per-layer, per-sample views) is timed separately.  The card name and power limit are read
through NVML in the same run, with the SM clock sampled while the windows run.

    python scripts/packed_attention_bench.py [--batch 64] [--steps 50] [--dtype bf16]
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

T_CAP, BOX_CAP = 37, 100


def detector_rows(batch, seed, F, vocab):
    """`batch` VQA rows: (token ids, box features [n, F], pixel boxes [n, 4], (w, h)), U{5..20} tokens and U{10..100} boxes."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sizes = ((640, 480), (500, 375), (800, 600), (480, 640))
    rows = []
    for i in range(batch):
        t = int(torch.randint(5, 21, (1,), generator=g))
        n = int(torch.randint(10, 101, (1,), generator=g))
        q = torch.randint(1000, vocab, (t,), generator=g)
        f = torch.relu(torch.randn(n, F, generator=g)) * 1.5
        w, h = sizes[i % len(sizes)]
        xy = torch.rand(n, 2, generator=g) * torch.tensor([0.7 * w, 0.7 * h])
        wh_box = (0.05 + 0.25 * torch.rand(n, 2, generator=g)) * torch.tensor([float(w), float(h)])
        bx = torch.cat([xy, torch.minimum(xy + wh_box, torch.tensor([float(w), float(h)]))], 1)
        rows.append((q, f, bx, (float(w), float(h))))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timing windows per arm; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb

    harness.require_gpu("packed_attention_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype, return_attention=True)
    sel = vb.OUT_VIL_PREDICTION
    rows = detector_rows(args.batch, args.seed, cfg.v_feature_size, cfg.vocab_size)
    B, F = len(rows), cfg.v_feature_size
    tin, nb = [len(r[0]) for r in rows], [r[1].shape[0] for r in rows]
    t_max, n_max = max(tin), max(nb)

    dev = torch.device("cuda", 0)
    q, im = torch.zeros(B, t_max, dtype=torch.long), torch.zeros(B, t_max, dtype=torch.long)
    f, bx = torch.zeros(B, n_max, F), torch.zeros(B, n_max, 4)
    for b, (qq, ff, bb, _) in enumerate(rows):
        q[b, :len(qq)], im[b, :len(qq)] = qq, 1
        f[b, :ff.shape[0]], bx[b, :ff.shape[0]] = ff, bb
    wh = torch.tensor([list(r[3]) for r in rows])
    task = torch.ones(B, 1, dtype=torch.long)
    nbox = torch.tensor(nb, dtype=torch.int32).to(dev)
    dense_in = [t.to(dev) for t in (q, torch.zeros_like(q), im, task, f, bx, wh)]
    pq = torch.cat([r[0] for r in rows]).to(dev)
    packed_in = (pq, torch.zeros_like(pq), task.to(dev), torch.cat([r[1] for r in rows]).to(dev), torch.cat([r[2] for r in rows]).to(dev),
                 wh.to(dev), tin, nb)
    arms = {
        "packed": lambda: model.forward_regions_packed(*packed_in, select=sel, max_tokens=T_CAP, max_boxes=BOX_CAP, return_spatials=False),
        "packed_maps": lambda: model.forward_regions_packed(*packed_in, select=sel, max_tokens=T_CAP, max_boxes=BOX_CAP,
                                                            return_spatials=False, output_all_attention_masks=True),
        "dense_maps": lambda: model.forward_regions(*dense_in, num_boxes=nbox, select=sel, return_spatials=False,
                                                    output_all_attention_masks=True),
    }
    floats = {"packed": 0, "packed_maps": model.attention_layout_packed(tin, [n + 1 for n in nb])[1],
              "dense_maps": model.attention_layout(B, t_max, n_max + 1)[1]}
    logits = {k: fn()[0][0] for k, fn in arms.items()}
    torch.cuda.synchronize()
    if not torch.equal(logits["packed"], logits["packed_maps"]):
        raise SystemExit("VQA logits differ with and without the packed maps")

    with harness.sampled_clock() as clock:
        ms = harness.alternate(arms, args.rounds, args.steps, args.warmup)

    from torch.profiler import ProfilerActivity, profile

    def device_ms(fn, n=5):
        """(all kernels, attention_f32_kernel) device ms per call, from CUPTI kernel records."""
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
        total = maps = 0.0
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            if ev.device_type is not None and "cuda" in str(ev.device_type).lower():
                total += t
                if "attention_f32_kernel" in ev.key:
                    maps += t
        return total / n / 1e3, maps / n / 1e3
    dev_ms = {k: device_ms(fn) for k, fn in arms.items()}

    from vilbert_b200.model import split_packed_attention
    layout, total_floats = model.attention_layout_packed(tin, [n + 1 for n in nb])
    flat = torch.empty(total_floats, device=dev)
    t_rows, v_rows = [t + 1 for t in tin], [n + 1 for n in nb]
    t0 = time.perf_counter()
    for _ in range(20):
        split_packed_attention(flat, layout, t_rows, v_rows)
    split_ms = (time.perf_counter() - t0) / 20 * 1e3

    card = harness.card(clock)
    result = {k: {"ms_per_call": statistics.median(v), "windows_ms": v, "map_floats_per_call": floats[k],
                  "device_ms_per_call_all_activity": dev_ms[k][0], "device_ms_per_call_map_kernels": dev_ms[k][1]}
              for k, v in ms.items()}
    result["packed_maps"]["host_ms_split_packed_attention"] = split_ms
    print(json.dumps({"workload": f"batch {B} VQA rows, U{{5..20}} tokens (max {t_max}), U{{10..100}} boxes (max {n_max}), "
                                  f"seed {args.seed}, {args.dtype}", **result, "steps": args.steps, "rounds": args.rounds,
                      "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
