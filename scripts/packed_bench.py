"""Packed variable-length batches vs dense padded batches on a mixed VQA workload (one JSON line).

Workload (seeded): batch 64 of VQA requests as the worker builds them -- text padded to 37 tokens with U{5..28} real words plus
[CLS] / [SEP], and 1 + U{10..100} regions per image.  Two paths over the same requests, timed with CUDA events after every plan
they use is warm:
  dense  -- one forward at (37 tokens, the batch's largest region count) with input / image masks (what padding to the batch
            maximum costs);
  packed -- one vb200_forward_packed call on the real rows, fixed capacities 37 tokens / 101 regions (one plan for the batch size).
Reported per path: pairs/s, the useful algorithmic FLOPs (sum over samples of plan_info(1, Tin_i, V_i)) and the FLOPs as issued
(dense: plan_info of the padded batch; packed: the useful FLOPs -- GEMM tiles past the row totals are skipped; the at most 127 rows
that fill the last 128-row tile of each stream are not counted).  The card name, power limit and SM clock are read through NVML in
the same run, and the packed VQA logits of 4 samples are checked against the dense ones (max abs difference <= 1e-5).

    python scripts/packed_bench.py [--batch 64] [--steps 200] [--dtype bf16]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402


def workload(batch, seed, F, vocab):
    import torch
    g = torch.Generator().manual_seed(seed)
    tin = [int(torch.randint(5, 29, (1,), generator=g)) + 2 for _ in range(batch)]      # words + [CLS] / [SEP]
    nv = [1 + int(torch.randint(10, 101, (1,), generator=g)) for _ in range(batch)]
    samples = []
    for t, v in zip(tin, nv):
        q = torch.randint(1000, vocab, (t,), generator=g)
        q[0], q[-1] = 101, 102
        f = torch.relu(torch.randn(v, F, generator=g)) * 1.5
        f[0] = f[1:].mean(dim=0)
        xy = torch.rand(v, 2, generator=g) * 0.7
        x2y2 = (xy + 0.05 + torch.rand(v, 2, generator=g) * 0.25).clamp(max=1.0)
        s = torch.cat([xy, x2y2, ((x2y2 - xy)[:, 0] * (x2y2 - xy)[:, 1])[:, None]], dim=-1)
        s[0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
        samples.append((q, f, s))
    return samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternating dense / packed timing windows; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import statistics
    import torch
    import vilbert_b200 as vb

    harness.require_gpu("packed_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    B, T_PAD, V_CAP = args.batch, 37, 101
    sel = vb.OUT_VIL_PREDICTION
    samples = workload(B, args.seed, cfg.v_feature_size, cfg.vocab_size)
    tin, nv = [len(s[0]) for s in samples], [s[1].shape[0] for s in samples]
    v_max = max(nv)

    # FLOPs from shapes (plan_info builds the plans it is asked about: done before any timing)
    per = {}
    for t, v in set(zip(tin, nv)):
        per[(t, v)] = model.plan_info(1, t, v, sel)[1]
    useful = sum(per[(t, v)] for t, v in zip(tin, nv))
    dense_issued = model.plan_info(B, T_PAD, v_max, sel)[1]

    dev = torch.device("cuda", 0)
    q = torch.zeros(B, T_PAD, dtype=torch.long)
    im = torch.zeros(B, T_PAD, dtype=torch.long)
    f = torch.zeros(B, v_max, cfg.v_feature_size)
    s = torch.zeros(B, v_max, 5)
    vm = torch.zeros(B, v_max, dtype=torch.uint8)
    for b, (qq, ff, ss) in enumerate(samples):
        q[b, :len(qq)], im[b, :len(qq)] = qq, 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.ones(B, 1, dtype=torch.long)
    dense_in = [t.to(dev) for t in (q, f, s, torch.zeros_like(q), im, vm)] + [None, task.to(dev)]
    pq = torch.cat([smp[0] for smp in samples]).to(dev)
    packed_in = (pq, torch.cat([smp[1] for smp in samples]).to(dev), torch.cat([smp[2] for smp in samples]).to(dev),
                 torch.zeros_like(pq), task.to(dev), tin, nv)

    run_dense = lambda: model(*dense_in, select=sel)
    run_packed = lambda: model.forward_packed(*packed_in, select=sel, max_tokens=T_PAD, max_regions=V_CAP)
    ref, got = run_dense()[0], run_packed()[0]
    torch.cuda.synchronize()
    parity = float((got[:4] - ref[:4]).abs().max())
    if not parity <= 1e-5:
        raise SystemExit(f"packed VQA logits differ from dense: {parity}")

    with harness.sampled_clock() as clock:
        ms = harness.alternate({"dense": run_dense, "packed": run_packed}, args.rounds, args.steps, args.warmup)
    secs = {k: [t * args.steps / 1e3 for t in v] for k, v in ms.items()}          # whole windows, in seconds
    card = harness.card(clock)

    def path(name, issued):
        t = statistics.median(secs[name])
        return {"pairs_per_s": B * args.steps / t, "ms_per_step": 1e3 * t / args.steps, "flops_useful": useful,
                "flops_issued": issued, "windows_s": secs[name]}
    dense, packed = path("dense", dense_issued), path("packed", useful)
    print(json.dumps({"workload": f"batch {B} VQA, text padded to {T_PAD} (U{{5..28}} words + 2), 1 + U{{10..100}} regions, "
                                  f"seed {args.seed}, {args.dtype}",
                      "dense": dense, "packed": packed, "speedup": packed["pairs_per_s"] / dense["pairs_per_s"],
                      "flops_ratio_packed_vs_dense": useful / dense_issued, "vqa_parity_max_abs": parity,
                      "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
