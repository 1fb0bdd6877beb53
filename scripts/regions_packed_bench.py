"""Packed detector-output batches vs dense padded ones, from the detector's output to the VQA logits (one JSON line).

Workload (seeded): batch 64 of VQA rows with questions of U{5..28} words + [CLS] / [SEP] and the detector's box features, pixel boxes
and image sizes.  Two workloads:
  (a) 100 boxes per image, as the reference detector keeps (num_features = 100);
  (b) U{10..100} boxes per image.
Two paths over the same rows, timed with CUDA events in alternating windows after every plan they use is warm (median of --rounds):
  dense  -- forward_regions at 37 tokens (input_mask) and the batch's largest box count (num_boxes masks): what custom_prediction does;
  packed -- forward_regions_packed on the real rows, fixed capacities 37 tokens / 100 boxes (one plan for the batch size).
Reported per path: pairs/s, the useful algorithmic FLOPs (sum over rows of plan_info(1, Tin_i, n_i + 1)) and the FLOPs as issued
(dense: plan_info of the padded batch; packed: the useful FLOPs -- GEMM tiles past the row totals are skipped; the at most 127 rows
that fill the last 128-row tile of each stream are not counted), and the VQA-logit max |dense - packed| over 4 rows (the dense text
padding changes the accumulation, so this is small, not zero).

Worker section: 64 single-image VQA messages with 100 boxes each, submitted at once, through MicroBatchWorker(packed=False) (host-side
build_inputs + prediction_batch) and MicroBatchWorker(packed=True) (custom_prediction_packed); messages/s from the first submit to the
last result, host-side input construction included.  The card name, power limit and SM clock are read through NVML in the same run.

    python scripts/regions_packed_bench.py [--batch 64] [--steps 200] [--dtype bf16]
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

T_PAD, BOX_CAP = 37, 100


def detector_rows(batch, seed, F, vocab, boxes):
    """`batch` VQA rows: (token ids with [CLS] / [SEP], box features [n, F], pixel boxes [n, 4], (w, h)); `boxes` is "100" or "10..100"."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sizes = ((640, 480), (500, 375), (800, 600), (480, 640))
    rows = []
    for i in range(batch):
        t = int(torch.randint(5, 29, (1,), generator=g)) + 2
        n = BOX_CAP if boxes == "100" else int(torch.randint(10, 101, (1,), generator=g))
        q = torch.randint(1000, vocab, (t,), generator=g)
        q[0], q[-1] = 101, 102
        f = torch.relu(torch.randn(n, F, generator=g)) * 1.5
        w, h = sizes[i % len(sizes)]
        xy = torch.rand(n, 2, generator=g) * torch.tensor([0.7 * w, 0.7 * h])
        wh_box = (0.05 + 0.25 * torch.rand(n, 2, generator=g)) * torch.tensor([float(w), float(h)])
        bx = torch.cat([xy, torch.minimum(xy + wh_box, torch.tensor([float(w), float(h)]))], 1)
        rows.append((q, f, bx, (float(w), float(h))))
    return rows


def compare_paths(model, rows, sel, args):
    import torch
    B, F = len(rows), model._dims["v_feature_size"]
    tin, nb = [len(r[0]) for r in rows], [r[1].shape[0] for r in rows]
    n_max = max(nb)
    per = {}
    for t, n in set(zip(tin, nb)):                    # plan_info builds the plans it is asked about: before any timing
        per[(t, n)] = model.plan_info(1, t, n + 1, sel)[1]
    useful = sum(per[(t, n)] for t, n in zip(tin, nb))
    dense_issued = model.plan_info(B, T_PAD, n_max + 1, sel)[1]

    dev = torch.device("cuda", 0)
    q, im = torch.zeros(B, T_PAD, dtype=torch.long), torch.zeros(B, T_PAD, dtype=torch.long)
    f, bx = torch.zeros(B, n_max, F), torch.zeros(B, n_max, 4)
    for b, (qq, ff, bb, _) in enumerate(rows):
        q[b, :len(qq)], im[b, :len(qq)] = qq, 1
        f[b, :ff.shape[0]], bx[b, :ff.shape[0]] = ff, bb
    wh = torch.tensor([list(r[3]) for r in rows])
    task = torch.ones(B, 1, dtype=torch.long)
    nbox = None if min(nb) == n_max else torch.tensor(nb, dtype=torch.int32).to(dev)
    dense_in = [t.to(dev) for t in (q, torch.zeros_like(q), im, task, f, bx, wh)]
    pq = torch.cat([r[0] for r in rows]).to(dev)
    packed_in = (pq, torch.zeros_like(pq), task.to(dev), torch.cat([r[1] for r in rows]).to(dev), torch.cat([r[2] for r in rows]).to(dev),
                 wh.to(dev), tin, nb)
    run_dense = lambda: model.forward_regions(*dense_in, num_boxes=nbox, select=sel, return_spatials=False)
    run_packed = lambda: model.forward_regions_packed(*packed_in, select=sel, max_tokens=T_PAD, max_boxes=BOX_CAP, return_spatials=False)
    ref, got = run_dense()[0][0], run_packed()[0][0]
    torch.cuda.synchronize()
    parity = float((got[:4] - ref[:4]).abs().max())
    if parity != parity:
        raise SystemExit("packed VQA logits are NaN")

    ms = harness.alternate({"dense": run_dense, "packed": run_packed}, args.rounds, args.steps, args.warmup)
    secs = {k: [t * args.steps / 1e3 for t in v] for k, v in ms.items()}          # whole windows, in seconds

    def path(name, issued):
        t = statistics.median(secs[name])
        return {"pairs_per_s": B * args.steps / t, "ms_per_step": 1e3 * t / args.steps, "flops_useful": useful,
                "flops_issued": issued, "windows_s": secs[name]}
    dense, packed = path("dense", dense_issued), path("packed", useful)
    return {"dense": dense, "packed": packed, "speedup": packed["pairs_per_s"] / dense["pairs_per_s"],
            "flops_ratio_packed_vs_dense": useful / dense_issued, "vqa_parity_max_abs": parity, "box_range": [min(nb), n_max],
            "mean_tin": sum(tin) / B}


def compare_workers(model, n_msgs, seed, F, args):
    import torch
    from vilbert_b200 import worker_api as W
    g = torch.Generator().manual_seed(seed)
    words = [f"w{i}" for i in range(500)]
    W.tokenizer = W.WordpieceTokenizer({t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + words)})
    W.model = model
    W.label_maps.update(vqa=None, gqa=None)
    msgs = []
    for k in range(n_msgs):
        n_words = int(torch.randint(5, 29, (1,), generator=g))
        question = " ".join(words[int(i)] for i in torch.randint(0, len(words), (n_words,), generator=g))
        f = torch.relu(torch.randn(BOX_CAP, F, generator=g)) * 1.5
        xy = torch.rand(BOX_CAP, 2, generator=g) * 400
        bbox = torch.cat([xy, xy + 20 + torch.rand(BOX_CAP, 2, generator=g) * 200], 1).numpy()
        msgs.append(({"image_path": [f"/m/demo/i{k}.jpg"], "question": question, "socket_id": f"s{k}", "task_id": "1"},
                     [f], [{"image_width": 640, "image_height": 480, "bbox": bbox}]))
    workers = {"dense": W.MicroBatchWorker(max_rows=n_msgs, max_wait_ms=1000.0, packed=False),
               "packed": W.MicroBatchWorker(max_rows=n_msgs, max_wait_ms=1000.0, packed=True)}

    def one(worker):
        t0 = time.perf_counter()
        futs = [worker.submit(*m) for m in msgs]
        res = [fu.result(timeout=300) for fu in futs]
        return time.perf_counter() - t0, res

    answers = {}
    for name, w in workers.items():                  # warm-up: plans, graphs, allocator
        for _ in range(2):
            _, answers[name] = one(w)
    agree = sum(a["result"]["result"][0]["answer"] == b["result"]["result"][0]["answer"]
                for a, b in zip(answers["dense"], answers["packed"]))
    secs = {"dense": [], "packed": []}
    for _ in range(args.rounds):
        for name, w in workers.items():
            secs[name].append(one(w)[0])
    batches = {name: w.batches[-1] for name, w in workers.items()}
    for w in workers.values():
        w.close()
    out = {name: {"messages_per_s": n_msgs / statistics.median(s), "windows_s": s, "rows_last_forward": batches[name]}
           for name, s in secs.items()}
    out["speedup"] = out["packed"]["messages_per_s"] / out["dense"]["messages_per_s"]
    out["top1_agree"] = f"{agree}/{n_msgs}"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternating dense / packed timing windows; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import vilbert_b200 as vb

    harness.require_gpu("regions_packed_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    sel = vb.OUT_VIL_PREDICTION
    with harness.sampled_clock() as clock:
        result = {}
        for key, boxes in (("a_100_boxes", "100"), ("b_10_100_boxes", "10..100")):
            rows = detector_rows(args.batch, args.seed, cfg.v_feature_size, cfg.vocab_size, boxes)
            result[key] = compare_paths(model, rows, sel, args)
        result["worker_64_messages_100_boxes"] = compare_workers(model, args.batch, args.seed + 1, cfg.v_feature_size, args)
    card = harness.card(clock)
    print(json.dumps({"workload": f"batch {args.batch} VQA rows, text padded to {T_PAD} (U{{5..28}} words + 2), detector boxes "
                                  f"(a) 100 / (b) U{{10..100}} per image, seed {args.seed}, {args.dtype}",
                      **result, "steps": args.steps, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
