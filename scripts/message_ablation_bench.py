"""Message ablation on the device against variants built with torch ops and scored with a torch softmax (one JSON line).

Workload: the full synthetic model in bf16 at the demo's largest messages -- 37 question tokens and 100 detector boxes per image, each
message ablated over positions 1..35 and every box -- one message each of grounding (1 image), NLVR2 (2 images) and retrieval with
K = 4 and K = 10 images.
  (a) model.message_ablation: the variants built on the device from the batch's single copy, one packed forward per engine call (at
      most 1024 samples), the segments gathered and scored on the device.  A retrieval box variant runs only the changed image.
  (b) every variant's full input replicated with torch ops on the device in the worker's layout (all K images of a retrieval box
      variant), forward_regions_packed in chunks of at most 1024 samples, torch.softmax of each segment.
Both end with the scores on the host.  Each is timed with CUDA events around a loop of whole calls, alternating window by window; the
median of --rounds windows is reported as ms per message.  (b) is timed where it fits in memory (not for K = 10, whose 10,360
replicated samples hold 8.5 GB of box features); the max absolute difference of (a)'s segments from (b)'s is reported for every
family.  The card name, power limit and the SM clock sampled while the windows run are read in the same run.

    python scripts/message_ablation_bench.py [--steps 3] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402

TIN, BOXES, CAP = 37, 100, 1024
NLVR2, RET, GRD = 3, 5, 6
FAMILIES = [("grounding", GRD, 1, True), ("nlvr2", NLVR2, 2, True), ("retrieval_k4", RET, 4, True), ("retrieval_k10", RET, 10, False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timing windows per path; the median is reported")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb

    harness.require_gpu("message_ablation_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, "bf16")
    dev = torch.device("cuda", 0)
    mask_token, tokens = 103, (1, TIN - 1)
    pooled = vb.OUT_VIL_PREDICTION | vb.OUT_VIL_PREDICTION_GQA | vb.OUT_VIL_LOGIT | vb.OUT_VIL_BINARY_PREDICTION | vb.OUT_VIL_TRI_PREDICTION

    def message(K, seed):
        """K images sharing one question: token ids [TIN], box features [K * BOXES, F], pixel boxes, image sizes."""
        g = torch.Generator().manual_seed(seed)
        bx = harness.pixel_boxes(g, K * BOXES)
        q = torch.randint(1000, cfg.vocab_size, (TIN,), generator=g)
        f = torch.relu(torch.randn(K * BOXES, cfg.v_feature_size, generator=g)) * 1.5
        return (q.repeat(K).to(dev), torch.zeros(K * TIN, dtype=torch.long, device=dev), torch.ones(K, 1, dtype=torch.long, device=dev),
                f.to(dev), bx.to(dev), torch.tensor([[640.0, 480.0]] * K, device=dev), [TIN] * K, [BOXES] * K)

    def device_call(x, fam, K):
        res = model.message_ablation(*x, [(fam, 0, K, None, tokens, None)], mask_token=mask_token, return_logits=True)
        return torch.cat(res[0]["logits"]), res[0]["token_prob"]

    def torch_variants(x, fam, K):
        """Each variant's samples as (question, box features, boxes) device tensors, in the engine's variant order."""
        q, f, bx = x[0][:TIN], x[3], x[4]
        imgs = [(f[k * BOXES:(k + 1) * BOXES], bx[k * BOXES:(k + 1) * BOXES]) for k in range(K)]
        out = [[(q,) + im for im in imgs]]
        for p in range(*tokens):
            qm = q.clone()
            qm[p] = mask_token
            out.append([(qm,) + im for im in imgs])
        for k in range(K):
            for j in range(BOXES):
                keep = torch.cat([torch.arange(j, device=dev), torch.arange(j + 1, BOXES, device=dev)])
                changed = (q, imgs[k][0].index_select(0, keep), imgs[k][1].index_select(0, keep))
                out.append([changed if i == k else (q,) + im for i, im in enumerate(imgs)] if fam != GRD else [changed])
        return out

    def torch_call(x, fam, K):
        """Every variant replicated, forward_regions_packed in chunks of whole variants, torch.softmax of each segment."""
        var = torch_variants(x, fam, K)
        segs, built, chunk = [], 0, []
        sel = pooled | (vb.OUT_VISION_LOGIT if fam == GRD else 0)

        def run(chunk):
            samples = [s for v in chunk for s in v]
            n = len(samples)
            vq, vf, vbx = torch.cat([s[0] for s in samples]), torch.cat([s[1] for s in samples]), torch.cat([s[2] for s in samples])
            nb = [s[1].shape[0] for s in samples]
            out, _ = model.forward_regions_packed(vq, torch.zeros_like(vq), torch.ones(n, 1, dtype=torch.long, device=dev), vf, vbx,
                                                  torch.tensor([[640.0, 480.0]] * n, device=dev), [TIN] * n, nb, select=sel,
                                                  max_tokens=TIN, max_boxes=BOXES, return_spatials=False)
            at, row = 0, 0
            for v in chunk:
                if fam == NLVR2:
                    segs.append(out[3][at // 2])
                elif fam == RET:
                    segs.append(out[2][at:at + K].reshape(-1))
                else:
                    segs.append(out[6][row:row + nb[at] + 1].reshape(-1))
                row += sum(b + 1 for b in nb[at:at + len(v)])
                at += len(v)
            return vq.numel() * 8 + vf.numel() * 4 + vbx.numel() * 4

        for v in var:
            if sum(len(c) for c in chunk) + len(v) > CAP:
                built += run(chunk)
                chunk = []
            chunk.append(v)
        built += run(chunk)
        probs = [torch.softmax(s, 0) for s in segs]
        p = torch.stack([pr[0] for pr in probs]).cpu()
        return torch.cat(segs), p, built, sum(len(v) for v in var)

    results = {}
    with harness.sampled_clock() as clock:
        for name, fam, K, time_torch in FAMILIES:
            x = message(K, args.seed + K)
            a, _ = device_call(x, fam, K)
            b, _, built, torch_samples = torch_call(x, fam, K)
            torch.cuda.synchronize()
            nt, nb = x[6], x[7]
            recs, _, _ = model._message_layout(nt, nb, [vb.model.message_pieces([(fam, 0, K, None, tokens, None)], nt, nb)[0][0]])
            r = {"device_samples": sum(rc[3] for rc in recs), "torch_samples": torch_samples,
                 "max_abs_diff": float((a - b).abs().max()) if a.shape == b.shape else None}
            del b
            paths = {"device": lambda: device_call(x, fam, K)}
            if time_torch:
                paths["torch"] = lambda: torch_call(x, fam, K)
            # "torch" stays [] where (b) is not timed
            ms = {"device": [], "torch": [], **harness.alternate(paths, args.rounds, args.steps, args.warmup)}
            r["device_ms_per_message"] = statistics.median(ms["device"])
            r["torch_ms_per_message"] = statistics.median(ms["torch"]) if time_torch else None
            r["torch_bytes_built_per_message"] = built
            r["windows_ms"] = ms
            results[name] = r

    card = harness.card(clock)
    print(json.dumps({"workload": f"full synthetic model, bf16, one message per family of {TIN} tokens and {BOXES} boxes per image, "
                                  f"positions {tokens[0]}..{tokens[1] - 1} masked and every box dropped, seed {args.seed}",
                      **results, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
