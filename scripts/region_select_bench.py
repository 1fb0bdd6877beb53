"""Detector-region selection on the device vs the reference's per-class loop, and the 64-message VQA window from detector heads to
logits (one JSON line).

Workload (seeded, `synthetic.synthetic_detections` with N(0, 2) logits): 1000 proposals, 1601 score columns, 2048 features per image.
  (a) `select_regions` for 1, 8 and 64 images: CUDA events around --reps calls, median of --rounds windows.
  (b) the reference loop (worker.py:123-176) restated with torch ops on the device and torchvision.ops.nms on +1-shifted boxes
      (the legacy IoU), for 1 and 8 images, when torchvision imports: CUDA events around one pass, median of --rounds.
  (c) 64 single-image VQA messages: custom_prediction_packed on features already selected on the host (the path the worker has
      today: numpy box features and boxes per message), split into pack_region_requests and forward_regions_packed, vs
      custom_prediction_detections from the raw heads on the device (selection into the packed rows, one forward).  Wall time of
      each call ending in a device synchronise, host decode included, median of --rounds alternating windows.
The card name, power limit and SM clock are read through NVML in the same run.

    python scripts/region_select_bench.py [--rounds 5] [--reps 10] [--dtype bf16]
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


def _events_ms(fn, reps):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def device_selection(model, args):
    import torch
    from vilbert_b200 import synthetic as S
    res = {}
    for n in (1, 8, 64):
        dets = [tuple(t.cuda() if torch.is_tensor(t) else t for t in d) for d in S.synthetic_detections(n, 1000, seed=args.seed)]
        model.select_regions(dets)
        torch.cuda.synchronize()
        res[f"{n}_images_ms"] = statistics.median(_events_ms(lambda: model.select_regions(dets), args.reps)
                                                  for _ in range(args.rounds))
    return res


def reference_loop(args):
    import torch
    try:
        import torchvision
    except Exception as e:                # noqa: BLE001 -- reported, not timed
        return {"skipped": repr(e)}
    from vilbert_b200 import synthetic as S

    def run(dets):
        for prop, sc, ft, scale in dets:
            p = torch.softmax(sc, -1)
            boxes = prop / scale
            shifted = torch.cat([boxes[:, :2], boxes[:, 2:] + 1], 1)
            max_conf = torch.zeros(p.shape[0], device=p.device)
            for c in range(1, p.shape[1]):
                keep = torchvision.ops.nms(shifted, p[:, c], 0.5)
                s = p[keep, c]
                max_conf[keep] = torch.where((s > max_conf[keep]) & (s > 0.0), s, max_conf[keep])
            _, idx = torch.sort(max_conf, descending=True)
            keep = idx[:100]
            (ft[keep], boxes[keep], torch.argmax(p[keep][1:], dim=1), p[keep])
    res = {}
    for n in (1, 8):
        dets = [tuple(t.cuda() if torch.is_tensor(t) else t for t in d) for d in S.synthetic_detections(n, 1000, seed=args.seed)]
        run(dets[:1])
        torch.cuda.synchronize()
        res[f"{n}_images_ms"] = statistics.median(_events_ms(lambda: run(dets), 1) for _ in range(args.rounds))
    return res


def worker_window(model, args):
    import numpy as np
    import torch
    from vilbert_b200 import synthetic as S
    from vilbert_b200 import worker_api as W
    W.model = model
    W.tokenizer = W.WordpieceTokenizer({t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man",
                                                                      "holding", "?", "color", "of", "dog"])})
    dets = S.synthetic_detections(64, 1000, seed=args.seed + 1)
    infos = [{"image_width": 640.0, "image_height": 480.0}] * 64
    sel = model.select_regions(dets)                  # the host path's inputs: what the detector step hands over today
    torch.cuda.synchronize()
    host_reqs, det_reqs = [], []
    for i in range(64):
        lo, k = sel["dst_rows"][i], sel["n_boxes"][i]
        info = dict(infos[i], bbox=sel["boxes"][lo:lo + k].cpu().numpy())
        host_reqs.append(("what is the man holding?", [1], [sel["box_features"][lo:lo + k].cpu().numpy()], [info], "1"))
        det_reqs.append(("what is the man holding?", [1], [tuple(t.cuda() if torch.is_tensor(t) else t for t in dets[i])],
                         [infos[i]], "1"))              # the detector's heads are on the device already

    def host_split():
        t0 = time.perf_counter()
        p = W.pack_region_requests(host_reqs)
        t1 = time.perf_counter()
        model.forward_regions_packed(p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"], p["image_wh"],
                                     p["n_tokens"], p["n_boxes"], select=p["select"], max_tokens=p["max_tokens"],
                                     max_boxes=p["max_boxes"])
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return {"pack_ms": 1e3 * (t1 - t0), "forward_ms": 1e3 * (t2 - t1)}

    def call(fn, reqs):
        def run():
            t0 = time.perf_counter()
            fn(reqs)
            torch.cuda.synchronize()
            return {"call_ms": 1e3 * (time.perf_counter() - t0)}
        return run

    paths = {"host_selected_split": host_split, "host_selected": call(W.custom_prediction_packed, host_reqs),
             "device_selected": call(W.custom_prediction_detections, det_reqs)}
    agree = W.custom_prediction_detections(det_reqs) == W.custom_prediction_packed(host_reqs)
    runs = {name: [] for name in paths}
    for name, fn in paths.items():
        fn()
    for _ in range(args.rounds):
        for name, fn in paths.items():
            runs[name].append(fn())
    out = {name: {k: statistics.median(r[k] for r in rs) for k in rs[0]} for name, rs in runs.items()}
    out["note"] = ("call_ms: custom_prediction_packed on host-selected features vs custom_prediction_detections on device heads, "
                   "both with host decode")
    out["answers_equal"] = bool(agree)
    out["host_selected_rows_bytes"] = int(sum(np.asarray(r[2][0]).nbytes for r in host_reqs))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10, help="select_regions calls per window in (a)")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import vilbert_b200 as vb

    harness.require_gpu("region_select_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    with harness.sampled_clock() as clock:
        result = {"a_device_selection": device_selection(model, args), "b_reference_loop": reference_loop(args),
                  "c_worker_64_vqa": worker_window(model, args)}
    card = harness.card(clock)
    print(json.dumps({"workload": f"1000 proposals x 1601 classes x 2048 features per image, seed {args.seed}, {args.dtype}",
                      **result, "rounds": args.rounds, "reps": args.reps, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
