"""Answer ablation on the device against variants built with torch ops and scored with a torch softmax (one JSON line).

Workload: the full synthetic model in bf16, VQA, messages of 37 question tokens and 100 detector boxes (the demo's largest shape), each
ablated over positions 1..35 and all 100 boxes: 1 + 35 + 100 = 136 variants per message; 1 message and 8 messages (1088 variants,
two engine calls).
  (a) model.answer_ablation: the variants' text ids and operand rows built on the device from each message's single copy, one packed
      forward per call, the scores from the decode kernel;
  (b) the variants' inputs replicated with torch ops on the device (every variant's question, box features and boxes), one
      forward_regions_packed of them all and torch.softmax of the head rows.
Both end with the scores on the host.  Each is timed with CUDA events around a loop of whole calls, alternating window by window; the
median of --rounds windows is reported as ms per message.  Also: the bytes (b) builds, the variant count, and whether the logits of (a)
and (b) agree bit for bit.  The card name, power limit and the SM clock sampled while the windows run are read in the same run.

    python scripts/ablation_bench.py [--steps 5] [--rounds 3]
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


def messages(n, seed, F, vocab):
    """n messages: (token ids [TIN], box features [BOXES, F], pixel boxes [BOXES, 4], (w, h))."""
    import torch
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        bx = harness.pixel_boxes(g, BOXES)
        out.append((torch.randint(1000, vocab, (TIN,), generator=g), torch.relu(torch.randn(BOXES, F, generator=g)) * 1.5, bx,
                    (640.0, 480.0)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timing windows per variant; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb

    harness.require_gpu("ablation_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    mask_token = 103
    tokens, boxes_range = (1, TIN - 1), (0, BOXES)
    per_msg = 1 + (tokens[1] - tokens[0]) + (boxes_range[1] - boxes_range[0])

    def inputs(ms):
        B = len(ms)
        q = torch.cat([m[0] for m in ms]).to(dev)
        return (q, torch.zeros_like(q), torch.ones(B, 1, dtype=torch.long, device=dev), torch.cat([m[1] for m in ms]).to(dev),
                torch.cat([m[2] for m in ms]).to(dev), torch.tensor([list(m[3]) for m in ms], device=dev), [TIN] * B, [BOXES] * B)

    def device_call(x):
        res = model.answer_ablation(*x, family="vqa", tokens=tokens, boxes_range=boxes_range, mask_token=mask_token, return_logits=True)
        return torch.cat([r["logits"] for r in res]), [r["token_prob"] for r in res]

    def torch_call(x):
        """Every variant replicated with torch ops, one forward_regions_packed, torch.softmax of the answer column on the host."""
        q, seg, tk, bf, bx, wh, nt, nb = x
        B = len(nt)
        qs, fs, bs, whs, n_box = [], [], [], [], []
        for i in range(B):
            qi, fi, bi = q[i * TIN:(i + 1) * TIN], bf[i * BOXES:(i + 1) * BOXES], bx[i * BOXES:(i + 1) * BOXES]
            qs.append(qi)
            fs.append(fi)
            bs.append(bi)
            n_box.append(BOXES)
            for p in range(*tokens):
                qm = qi.clone()
                qm[p] = mask_token
                qs.append(qm)
                fs.append(fi)
                bs.append(bi)
                n_box.append(BOXES)
            for j in range(*boxes_range):
                keep = torch.cat([torch.arange(j, device=dev), torch.arange(j + 1, BOXES, device=dev)])
                qs.append(qi)
                fs.append(fi.index_select(0, keep))
                bs.append(bi.index_select(0, keep))
                n_box.append(BOXES - 1)
        n = len(qs)
        vq, vf, vb_ = torch.cat(qs), torch.cat(fs), torch.cat(bs)
        vwh = wh.repeat_interleave(per_msg, 0)
        vtk = tk.repeat_interleave(per_msg, 0)
        out, _ = model.forward_regions_packed(vq, torch.zeros_like(vq), vtk, vf, vb_, vwh, [TIN] * n, n_box,
                                              select=vb.OUT_VIL_PREDICTION, max_tokens=TIN, max_boxes=BOXES, return_spatials=False)
        logits = out[0]
        probs = torch.softmax(logits, 1)
        ans = logits.view(B, per_msg, -1)[:, 0].argmax(1)
        p = probs.view(B, per_msg, -1).gather(2, ans.view(B, 1, 1).expand(B, per_msg, 1)).cpu()
        return logits, p, vq.numel() * 8 + vf.numel() * 4 + vb_.numel() * 4

    results = {}
    with harness.sampled_clock() as clock:
        for n_msg in (1, 8):
            x = inputs(messages(n_msg, args.seed + n_msg, cfg.v_feature_size, cfg.vocab_size))
            a_logits, _ = device_call(x)
            b_logits, _, built = torch_call(x)
            torch.cuda.synchronize()
            ms = harness.alternate({"device": lambda: device_call(x), "torch": lambda: torch_call(x)}, args.rounds, args.steps,
                                   args.warmup)
            results[f"{n_msg}_messages"] = {
                "variants": n_msg * per_msg, "engine_calls": -(-n_msg * per_msg // 1024),
                "device_ms_per_message": statistics.median(ms["device"]) / n_msg,
                "torch_ms_per_message": statistics.median(ms["torch"]) / n_msg,
                "windows_ms": ms, "torch_bytes_built_per_message": built // n_msg,
                "logits_bitwise_equal": bool(torch.equal(a_logits, b_logits))}
    card = harness.card(clock)
    print(json.dumps({"workload": f"full synthetic model, bf16, VQA, messages of {TIN} tokens and {BOXES} boxes, positions "
                                  f"{tokens[0]}..{tokens[1] - 1} masked and every box dropped ({per_msg} variants per message), seed {args.seed}",
                      **results, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
