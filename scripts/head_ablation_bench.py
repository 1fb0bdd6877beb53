"""Head ablation on the device against variants replicated with torch ops (one JSON line).

Workload: the full synthetic model in bf16, one VQA message of 37 question tokens and 100 detector boxes, every head of every
attention entry removed in turn (1 + 288 = 289 variants, one forward sample each).
  (a) model.head_ablation: the variants' samples and gate rows built on the device from the batch's single copy, one gated packed
      forward, the segments gathered and scored on the device.
  (b) the message's input replicated 289 times with torch ops, a [289, entries, heads] head mask built with torch, one
      forward_regions_packed(head_mask=...) call (vb200_forward_regions_packed_gated), torch.softmax of the VQA rows.
Both end with the scores on the host.  Each is timed with CUDA events around --steps calls, alternating window by window; the median
of --rounds windows is reported as ms per message, with the max absolute difference of (a)'s segments from (b)'s logits.  The card
name, power limit and the SM clock sampled while the windows run are read in the same run.

    python scripts/head_ablation_bench.py [--steps 5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

TIN, BOXES = 37, 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5, help="alternating timing windows per path; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200.model import head_mask_shape

    harness.require_gpu("head_ablation_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    E, H = head_mask_shape(cfg)
    g = torch.Generator().manual_seed(args.seed)
    bx = harness.pixel_boxes(g, BOXES).to(dev)
    q = torch.randint(1000, cfg.vocab_size, (TIN,), generator=g).to(dev)
    f = (torch.relu(torch.randn(BOXES, cfg.v_feature_size, generator=g)) * 1.5).to(dev)
    seg, task, wh = torch.zeros(TIN, dtype=torch.long, device=dev), torch.ones(1, 1, dtype=torch.long, device=dev), \
        torch.tensor([[640.0, 480.0]], device=dev)
    x = (q, seg, task, f, bx, wh, [TIN], [BOXES])
    recs, _, _ = model._head_layout([TIN], [BOXES], [(1, 0, 1, -1, 0, E)])
    units = [r[2] for r in recs]                          # -1 (unablated), then entry * H + head in layout order
    n = len(units)

    def device_call():
        res = model.head_ablation(*x, [("vqa", 0, 1)], return_logits=True)
        return torch.stack(res[0]["logits"]), res[0]["head_prob"]

    def torch_call():
        mask = torch.ones(n, E, H, device=dev)
        idx = torch.tensor([u for u in units if u >= 0], device=dev)
        mask.view(n, E * H)[torch.arange(1, n, device=dev), idx] = 0.0
        (out, _) = model.forward_regions_packed(q.repeat(n), seg.repeat(n), task.repeat(n, 1), f.repeat(n, 1), bx.repeat(n, 1),
                                                wh.repeat(n, 1), [TIN] * n, [BOXES] * n, select=vb.OUT_VIL_PREDICTION,
                                                return_spatials=False, head_mask=mask)
        logits = out[0]
        p = torch.softmax(logits, dim=-1)
        col = int(p[0].argmax())
        return logits, p[:, col].cpu()

    a, _ = device_call()
    b, _ = torch_call()
    torch.cuda.synchronize()
    diff = float((a - b).abs().max())
    with harness.sampled_clock() as clock:
        ms = harness.alternate({"device": device_call, "torch": torch_call}, args.rounds, args.steps, args.warmup)
    card = harness.card(clock)
    print(json.dumps({"workload": f"full synthetic model, bf16, one VQA message of {TIN} tokens and {BOXES} boxes, every head removed "
                                  f"in turn, seed {args.seed}", "variants": n,
                      "device_ms_per_message": statistics.median(ms["device"]), "torch_ms_per_message": statistics.median(ms["torch"]),
                      "windows_ms": ms, "max_abs_diff": diff, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
