"""Attention relevance on the device against a torch loop over the same maps (one JSON line).

Workload: batch 64 VQA rows, U{5..37} question tokens and U{10..100} detector boxes per image, the full synthetic model in bf16 with
head-mean maps (attention_heads="mean"), forward_regions_packed at capacities 37 tokens / 100 boxes.
  (a) the forward + model.attention_relevance (vb200_attention_relevance: one CTA per sample);
  (b) the forward + a torch loop: per sample, per step, the rollout's products on the device (what a caller without the kernel runs).
Each variant is timed with CUDA events around a loop of whole calls, alternating window by window; the median of --rounds windows is
reported.  Also: the relevance call alone (CUDA events around a loop of model.attention_relevance on one forward's maps), the device
time of attention_relevance_kernel per call from a torch.profiler pass of its own, and max |a - b|.  The card name, power limit and the
SM clock sampled while the windows run are read in the same run.

    python scripts/relevance_bench.py [--batch 64] [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

T_CAP, BOX_CAP = 37, 100


def rows(batch, seed, F, vocab):
    """`batch` VQA rows: (token ids, box features [n, F], pixel boxes [n, 4], (w, h)), U{5..37} tokens and U{10..100} boxes."""
    import torch
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(batch):
        t = int(torch.randint(5, T_CAP + 1, (1,), generator=g))
        n = int(torch.randint(10, BOX_CAP + 1, (1,), generator=g))
        bx = harness.pixel_boxes(g, n)
        out.append((torch.randint(1000, vocab, (t,), generator=g), torch.relu(torch.randn(n, F, generator=g)) * 1.5, bx,
                    (640.0, 480.0)))
    return out


def torch_relevance(attn, kinds):
    """The rollout of every sample with torch ops on the device: per sample, per step (last to first), r <- 0.5 (r + r M) on the
    covered columns.  attn: element 9 of a packed forward with head-mean maps (each entry a list of B [1, Lq, Lk] views)."""
    import torch
    flat, e = [], 0
    for pos in attn:
        flat.extend(pos if isinstance(pos, tuple) else (pos,))
    steps = []
    while e < len(kinds):
        steps.append((e, e + 1) if kinds[e] == 2 else (e,))
        e += 2 if kinds[e] == 2 else 1
    text, image = kinds.index(0), kinds.index(1)
    out = []
    for b in range(len(flat[0])):
        T, V = flat[text][b].shape[-1], flat[image][b].shape[-1]
        r = torch.zeros(2, T + V, device=flat[0][b].device)
        r[0, 0] = 1
        r[1, T] = 1
        for step in reversed(steps):
            acc = torch.zeros_like(r)
            lo, hi = (T, T + V) if kinds[step[0]] == 1 else (0, T if kinds[step[0]] == 0 else T + V)
            for k in step:
                q0, k0 = {0: (0, 0), 1: (T, T), 2: (0, T), 3: (T, 0)}[kinds[k]]
                m = flat[k][b][0]
                acc[:, k0:k0 + m.shape[1]] += r[:, q0:q0 + m.shape[0]] @ m
            r[:, lo:hi] = 0.5 * (r[:, lo:hi] + acc[:, lo:hi])
        out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5, help="alternating timing windows per variant; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb

    harness.require_gpu("relevance_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, "bf16", return_attention=True, attention_heads="mean")
    rs = rows(args.batch, args.seed, cfg.v_feature_size, cfg.vocab_size)
    B = len(rs)
    tin, nb = [len(r[0]) for r in rs], [r[1].shape[0] for r in rs]
    dev = torch.device("cuda", 0)
    pq = torch.cat([r[0] for r in rs]).to(dev)
    packed_in = (pq, torch.zeros_like(pq), torch.ones(B, 1, dtype=torch.long, device=dev), torch.cat([r[1] for r in rs]).to(dev),
                 torch.cat([r[2] for r in rs]).to(dev), torch.tensor([list(r[3]) for r in rs]).to(dev), tin, nb)
    kinds, _ = model.attention_selection()

    def forward():
        return model.forward_regions_packed(*packed_in, select=vb.OUT_VIL_PREDICTION, max_tokens=T_CAP, max_boxes=BOX_CAP,
                                            return_spatials=False, output_all_attention_masks=True)[0][9]

    variants = {"device": lambda: model.attention_relevance(forward()), "torch_loop": lambda: torch_relevance(forward(), kinds)}
    attn = forward()
    a, b = model.attention_relevance(attn), torch_relevance(attn, kinds)
    torch.cuda.synchronize()
    max_diff = max(float((x - y).abs().max()) for x, y in zip(a, b))

    with harness.sampled_clock() as clock:
        ms = {k: [] for k in variants}
        call_ms = []
        for _ in range(args.rounds):
            for k, fn in variants.items():
                ms[k].append(harness.timed(fn, args.steps, args.warmup))
            call_ms.append(harness.timed(lambda: model.attention_relevance(attn), 10 * args.steps, args.warmup))

    from torch.profiler import ProfilerActivity, profile
    n = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            model.attention_relevance(attn)
        torch.cuda.synchronize()
    kernel_us = 0.0
    for ev in prof.key_averages():
        d = getattr(ev, "device_time_total", None)
        d = ev.cuda_time_total if d is None else d
        if "attention_relevance_kernel" in ev.key:
            kernel_us += d
    kernel_us /= n

    card = harness.card(clock)
    print(json.dumps({"workload": f"batch {B} VQA rows, U{{5..{T_CAP}}} tokens, U{{10..{BOX_CAP}}} boxes, seed {args.seed}, bf16, "
                                  f"head-mean maps, forward_regions_packed at capacities {T_CAP} / {BOX_CAP}",
                      "forward_plus_device_ms": statistics.median(ms["device"]), "forward_plus_torch_loop_ms": statistics.median(ms["torch_loop"]),
                      "windows_ms": ms, "relevance_call_ms": statistics.median(call_ms), "relevance_kernel_device_us": kernel_us,
                      "max_abs_diff_device_vs_torch_loop": max_diff, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
