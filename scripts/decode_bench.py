"""Answer decode on the host (`worker_api._decode` per message) vs on the device (one `decode_answers` kernel), one JSON line.

(a) Decode only.  64 mixed messages -- 16 VQA, 16 GQA, 12 NLVR2 pairs, 12 grounding images with 100 boxes (101 vision rows) and 8
    retrievals over 10 images -- packed into one `forward_regions_packed` call, run once.  Then, alternating, the per-message
    `_decode` loop of `custom_prediction_packed` and one device decode of the same outputs (`worker_api._answer_regions` with
    decode="host" and "device"); both end in a host synchronisation.  Wall time on the host thread, median over --rounds windows
    of --reps calls each.
(b) The worker window of scripts/regions_packed_bench.py: 64 single-image VQA messages with 100 boxes.  First the real
    `MicroBatchWorker(packed=True)` with decode="host" and decode="device", alternating (messages/s from the first submit to the last
    result).  Then the same steps inline on this thread, split into pack (`pack_region_requests`), forward (`forward_regions_packed`
    followed by a device synchronisation, so the forward's device time is counted here), decode and result shaping (`shape_result`),
    median per step.
The card name, power limit and SM clock are read through NVML in the same run.

    python scripts/decode_bench.py [--rounds 7] [--reps 20] [--dtype bf16]
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

BOXES = 100


def setup_worker(model, seed):
    import torch
    from vilbert_b200 import worker_api as W
    words = [f"w{i}" for i in range(500)]
    W.tokenizer = W.WordpieceTokenizer({t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + words)})
    W.model = model
    W.label_maps.update(vqa=None, gqa=None)
    return words, torch.Generator().manual_seed(seed)


def detector(g, n_images, F, n=BOXES):
    import torch
    feats, infos = [], []
    for _ in range(n_images):
        feats.append(torch.relu(torch.randn(n, F, generator=g)) * 1.5)
        xy = torch.rand(n, 2, generator=g) * 400
        infos.append({"image_width": 640, "image_height": 480,
                      "bbox": torch.cat([xy, xy + 20 + torch.rand(n, 2, generator=g) * 200], 1).numpy()})
    return feats, infos


def question(g, words):
    import torch
    n_words = int(torch.randint(5, 29, (1,), generator=g))
    return " ".join(words[int(i)] for i in torch.randint(0, len(words), (n_words,), generator=g))


def decode_only(model, F, args):
    """(a): the per-message host loop vs one device decode over one packed forward's outputs."""
    from vilbert_b200 import worker_api as W
    words, g = setup_worker(model, args.seed)
    mix = ["1"] * 16 + ["15"] * 16 + ["12"] * 12 + ["11"] * 12 + ["7"] * 8
    images = {"12": 2, "7": 10}
    reqs = []
    for k, task_id in enumerate(mix):
        feats, infos = detector(g, images.get(task_id, 1), F)
        reqs.append((question(g, words), [int(task_id)], feats, infos, task_id))
    p = W.pack_region_requests(reqs)
    out, spatials = model.forward_regions_packed(p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"],
                                                 p["image_wh"], p["n_tokens"], p["n_boxes"], select=p["select"],
                                                 max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
    import torch
    torch.cuda.synchronize()

    def host():
        return W._answer_regions({}, reqs, out, spatials, p["spans"], p["n_tokens"], p["n_boxes"], "host")

    def device():
        return W._answer_regions({}, reqs, out, spatials, p["spans"], p["n_tokens"], p["n_boxes"], "device")

    a, b = host(), device()
    same_idx = 0
    for i in a:
        if isinstance(a[i], list):
            same_idx += [(x["x1"], x["y1"]) for x in a[i]] == [(x["x1"], x["y1"]) for x in b[i]]
        else:
            same_idx += a[i]["top3_answer"] == b[i]["top3_answer"]
    secs = {"host": [], "device": []}
    for _ in range(args.rounds):
        for name, fn in (("host", host), ("device", device)):
            t0 = time.perf_counter()
            for _ in range(args.reps):
                fn()
            secs[name].append((time.perf_counter() - t0) / args.reps)
    res = {name: {"ms_per_batch": 1e3 * statistics.median(s), "windows_ms": [1e3 * x for x in s]} for name, s in secs.items()}
    res["speedup"] = res["host"]["ms_per_batch"] / res["device"]["ms_per_batch"]
    res["answers_agree"] = f"{same_idx}/{len(a)}"
    res["messages"], res["forward_rows"], res["vision_rows"] = len(reqs), len(p["n_boxes"]), sum(p["n_boxes"]) + len(p["n_boxes"])
    return res


def worker_window(model, F, args):
    """(b): MicroBatchWorker(packed=True) end to end per decode mode, then the same window split into its steps."""
    import torch
    from vilbert_b200 import worker_api as W
    words, g = setup_worker(model, args.seed + 1)
    msgs = []
    for k in range(64):
        feats, infos = detector(g, 1, F)
        msgs.append(({"image_path": [f"/m/demo/i{k}.jpg"], "question": question(g, words), "socket_id": f"s{k}", "task_id": "1"},
                     feats, infos))
    workers = {m: W.MicroBatchWorker(max_rows=64, max_wait_ms=1000.0, packed=True, decode=m) for m in ("host", "device")}

    def one(worker):
        t0 = time.perf_counter()
        futs = [worker.submit(*m) for m in msgs]
        res = [fu.result(timeout=300) for fu in futs]
        return time.perf_counter() - t0, res

    answers = {}
    for name, w in workers.items():
        for _ in range(2):
            _, answers[name] = one(w)
    agree = sum(a["result"]["result"] == b["result"]["result"] for a, b in zip(answers["host"], answers["device"]))
    secs = {"host": [], "device": []}
    for _ in range(args.rounds):
        for name, w in workers.items():
            secs[name].append(one(w)[0])
    for w in workers.values():
        w.close()
    result = {"end_to_end": {name: {"messages_per_s": 64 / statistics.median(s), "windows_s": s} for name, s in secs.items()},
              "answers_identical": f"{agree}/64"}

    reqs = [(b["question"], [int(b["task_id"])], f, i, b["task_id"]) for b, f, i in msgs]

    def split(decode):
        t = [time.perf_counter()]
        p = W.pack_region_requests(reqs)
        t.append(time.perf_counter())
        out, spatials = model.forward_regions_packed(p["question"], p["segment_ids"], p["task_tokens"], p["box_features"], p["boxes"],
                                                     p["image_wh"], p["n_tokens"], p["n_boxes"], select=p["select"],
                                                     max_tokens=p["max_tokens"], max_boxes=p["max_boxes"])
        torch.cuda.synchronize()
        t.append(time.perf_counter())
        dec = W._answer_regions({}, reqs, out, spatials, p["spans"], p["n_tokens"], p["n_boxes"], decode)
        t.append(time.perf_counter())
        for i, (b, _, _) in enumerate(msgs):
            W.shape_result(b["task_id"], dec[i], b["image_path"])
        t.append(time.perf_counter())
        return [t[k + 1] - t[k] for k in range(4)]

    steps = {"host": [], "device": []}
    for name in steps:
        split(name)
    for _ in range(args.rounds):
        for name in steps:
            steps[name].append(split(name))
    names = ("pack", "forward", "decode", "shape")
    result["split_ms"] = {name: {n: 1e3 * statistics.median(r[k] for r in rows) for k, n in enumerate(names)} for name, rows in steps.items()}
    for name, d in result["split_ms"].items():
        d["total"] = sum(d[n] for n in names)
        d["decode_share"] = d["decode"] / d["total"]
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7, help="alternating host / device windows; the median is reported")
    ap.add_argument("--reps", type=int, default=20, help="decode calls per window in (a)")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import vilbert_b200 as vb

    harness.require_gpu("decode_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    with harness.sampled_clock() as clock:
        result = {"a_decode_only_64_mixed": decode_only(model, cfg.v_feature_size, args),
                  "b_worker_64_vqa_100_boxes": worker_window(model, cfg.v_feature_size, args)}
    card = harness.card(clock)
    print(json.dumps({"workload": f"(a) 64 mixed messages from one packed forward, (b) 64 VQA messages with {BOXES} boxes through "
                                  f"MicroBatchWorker(packed=True); seed {args.seed}, {args.dtype}",
                      **result, "rounds": args.rounds, "reps": args.reps, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
