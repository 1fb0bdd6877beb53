"""Shapley values on the device against coalitions replicated with torch ops (one JSON line).

Workload: the full synthetic model in bf16, one VQA message and one NLVR2 message, 37 question tokens and 100 detector boxes per
image, the default units (one per question position 1 .. 35 and one per box: 135 and 235 units), P = 8 antithetic permutations
(1 + 8 * 134 = 1073 and 1 + 8 * 234 = 1873 coalitions beside the full input).
  (a) model.shapley: every coalition's samples built on the device from the batch's single copy, packed forwards of at most 1024
      samples, the segments gathered and scored on the device, the estimator in one kernel.
  (b) every coalition's input replicated with torch ops: the masked questions, and per image the operand rows the worker builds
      from its kept boxes (worker.py:422-455: the mean row, then the boxes, with normalised locations), through forward_packed in
      chunks of at most 1024 samples (forward_regions_packed needs a box per image, and early chain coalitions leave images
      without one), torch.softmax of the answer rows, and the estimator restated in torch float64.
Both end with phi on the host.  Each is timed with CUDA events around --steps calls, alternating window by window; the median of
--rounds windows is reported as ms per message, with the forward samples each path runs and the max absolute difference of phi
between them (the paths differ in the summation order of the softmax and of the mean row).  The card name, power limit and the SM
clock sampled while the windows run are read in the same run.

    python scripts/shapley_bench.py [--steps 2] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

TIN, BOXES, P = 37, 100, 8
CHUNK = 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timing windows per path; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import model as M

    harness.require_gpu("shapley_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(args.seed)

    def image():
        bx = harness.pixel_boxes(g, BOXES)
        return (torch.relu(torch.randn(BOXES, cfg.v_feature_size, generator=g)) * 1.5).to(dev), bx.to(dev)

    q = [torch.randint(1000, cfg.vocab_size, (TIN,), generator=g).to(dev) for _ in range(2)]
    imgs = [image() for _ in range(3)]                    # sample 0: the VQA image; samples 1, 2: the NLVR2 pair
    text = [q[0], q[1], q[1]]
    x = (torch.cat(text), torch.zeros(3 * TIN, dtype=torch.long, device=dev), torch.tensor([[1], [12], [12]], device=dev),
         torch.cat([f for f, _ in imgs]), torch.cat([b for _, b in imgs]), torch.tensor([[640.0, 480.0]] * 3, device=dev),
         [TIN] * 3, [BOXES] * 3)
    msgs = [("vqa", 0, 1), ("nlvr2", 1, 2)]
    wh = torch.tensor([640.0, 480.0], device=dev)

    def device_call():
        return model.shapley(*x, msgs, permutations=P, seed=args.seed)

    def torch_call():
        gen = torch.Generator().manual_seed(args.seed)
        out = []
        for (fam, ib, K), head in zip(msgs, (0, 3)):
            units = M.coalition_units(None, TIN, K * BOXES)
            n = len(units)
            perm = M.shapley_permutations(n, P, gen, True)
            present = torch.cat([torch.ones(1, n, dtype=torch.bool), M.shapley_chain(perm)]).to(dev)   # full input, empty, chains
            C = present.shape[0]
            pos_unit = torch.full((TIN,), n, dtype=torch.long, device=dev)
            box_unit = torch.full((K * BOXES,), n, dtype=torch.long, device=dev)
            for u, (ps, bs) in enumerate(units):
                pos_unit[list(ps)] = u
                box_unit[list(bs)] = u
            ext = torch.cat([present, torch.ones(C, 1, dtype=torch.bool, device=dev)], 1)
            qs = torch.where(ext[:, pos_unit], text[ib], torch.full_like(text[ib], 103))          # [C, TIN]
            kept = ext[:, box_unit]                                                              # [C, K * BOXES]
            feats = torch.stack([imgs[ib + k][0] for k in range(K)])                          # [K, BOXES, F]
            bx = torch.stack([imgs[ib + k][1] for k in range(K)])
            loc = torch.cat([bx[..., :2] / wh, bx[..., 2:] / wh, ((bx[..., 3] - bx[..., 1]) * (bx[..., 2] - bx[..., 0]) / (640.0 * 480.0))[..., None]], -1)
            g_loc = torch.tensor([[0.0, 0.0, 1.0, 1.0, 1.0]], device=dev)
            rows = []
            per = CHUNK // K
            for c0 in range(0, C, per):
                c1 = min(C, c0 + per)
                B = (c1 - c0) * K
                m = kept[c0:c1].view(B, BOXES)                                                   # sample (c, k)'s kept boxes
                f = feats.repeat(c1 - c0, 1, 1)
                cnt = m.sum(1, keepdim=True).clamp(min=1).float()
                mean = (f * m[..., None]).sum(1) / cnt
                valid = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), m], 1)
                rf = torch.cat([mean[:, None], f], 1)[valid]
                rs = torch.cat([g_loc.expand(B, 1, 5), loc.repeat(c1 - c0, 1, 1)], 1)[valid]
                o = model.forward_packed(qs[c0:c1].repeat_interleave(K, 0).reshape(-1), rf, rs, torch.zeros(B * TIN, dtype=torch.long, device=dev),
                                         x[2][ib:ib + 1].repeat(B, 1), [TIN] * B, (m.sum(1) + 1).tolist(),
                                         select=vb.OUT_VIL_PREDICTION | vb.OUT_VIL_BINARY_PREDICTION)
                rows.append(o[head])
            probs = torch.softmax(torch.cat(rows), dim=-1)
            col = int(probs[0].argmax())
            v = probs[:, col]
            vals = torch.cat([v[1:2], v[:1], v[2:]]).double()                                   # v(empty), v(all), the chains
            c = torch.cat([vals[0].expand(P, 1), vals[2:].view(P, n - 1), vals[1].expand(P, 1)], 1)
            d = torch.zeros(P, n, dtype=torch.float64, device=dev)
            d.scatter_(1, perm.to(dev), c[:, 1:] - c[:, :-1])
            s = torch.zeros(n, dtype=torch.float64, device=dev)
            for p in range(P):
                s = s + d[p]
            out.append(dict(phi=(s / P).float().cpu(), samples=C * K))
        return out

    a, b = device_call(), torch_call()
    torch.cuda.synchronize()
    diff = max(float((ra["phi"] - rb["phi"]).abs().max()) for ra, rb in zip(a, b))
    with harness.sampled_clock() as clock:
        ms = harness.alternate({"device": device_call, "torch": torch_call}, args.rounds, args.steps, args.warmup)
    ms = {k: [t / len(msgs) for t in v] for k, v in ms.items()}
    card = harness.card(clock)
    print(json.dumps({"workload": f"full synthetic model, bf16, one VQA and one NLVR2 message, {TIN} tokens and {BOXES} boxes per image, "
                                  f"default units, P = {P} antithetic, seed {args.seed}",
                      "device_samples": [r["samples"] for r in a], "torch_samples": [r["samples"] for r in b],
                      "device_ms_per_message": statistics.median(ms["device"]), "torch_ms_per_message": statistics.median(ms["torch"]),
                      "windows_ms": ms, "max_abs_phi_diff": diff, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
