"""The queue worker from detector heads to answers: selection per message on the host's side of the queue vs one selection per
micro-batch inside the worker (one JSON line).

Workload (seeded): 64 single-image VQA messages of 5..28 words, each with the raw heads of its image on the device
(`synthetic.synthetic_detections` with N(0, 2) logits): 1000 proposals x 1601 score columns x 2048 features.  All 64 are submitted
at once; a window runs from the first submit (or, for (a), the first feature extraction) to the last future's result.
  (a) `process_feature_extraction` per message (one selection and one host synchronisation each), then
      `MicroBatchWorker(packed=True)` on the selected features as that function returns them;
  (b) `MicroBatchWorker(source="detections")`: the worker selects the regions of its whole micro-batch in one call.
Each with decode="host" and decode="device": the four windows alternate, two warm-up windows each, the median of --rounds is
reported as messages/s.  The answers of (a) and (b) are compared message by message.  The card name, power limit and SM clock are
read through NVML in the same run.

    python scripts/worker_detections_bench.py [--rounds 7] [--dtype bf16]
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

N_MSGS = 64


def messages(model, seed):
    import torch
    from vilbert_b200 import synthetic as S
    from vilbert_b200 import worker_api as W
    words = [f"w{i}" for i in range(500)]
    W.tokenizer = W.WordpieceTokenizer({t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + words)})
    W.model = model
    W.label_maps.update(vqa=None, gqa=None)
    g = torch.Generator().manual_seed(seed)
    heads = S.synthetic_detections(N_MSGS, 1000, seed=seed)
    msgs = []
    for k in range(N_MSGS):
        n_words = int(torch.randint(5, 29, (1,), generator=g))
        q = " ".join(words[int(i)] for i in torch.randint(0, len(words), (n_words,), generator=g))
        det = tuple(t.cuda() if torch.is_tensor(t) else t for t in heads[k])      # the detector's outputs are on the device
        msgs.append(({"image_path": [f"/m/demo/i{k}.jpg"], "question": q, "socket_id": f"s{k}", "task_id": "1"}, [det],
                     [{"image_width": 640.0, "image_height": 480.0}]))
    torch.cuda.synchronize()
    return msgs


def host_selected(W, worker, msgs):
    """(a): the worker's caller selects each message's regions, then submits the selected features."""
    futs = []
    for body, dets, infos in msgs:
        props, scores, feats, scales = zip(*dets)
        f, inf = W.process_feature_extraction(props, scores, feats, scales, [{"width": i["image_width"], "height": i["image_height"]}
                                                                            for i in infos])
        futs.append(worker.submit(body, f, inf))
    return [fu.result(timeout=300) for fu in futs]


def device_selected(W, worker, msgs):
    """(b): the heads go to the worker as they are."""
    futs = [worker.submit(*m) for m in msgs]
    return [fu.result(timeout=300) for fu in futs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7, help="alternating windows per path; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import vilbert_b200 as vb
    from vilbert_b200 import worker_api as W

    harness.require_gpu("worker_detections_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    msgs = messages(model, args.seed)
    paths = {}
    for decode in ("host", "device"):
        paths[f"a_host_selected_{decode}"] = (host_selected, W.MicroBatchWorker(max_rows=N_MSGS, max_wait_ms=1000.0, packed=True,
                                                                                decode=decode))
        paths[f"b_device_selected_{decode}"] = (device_selected, W.MicroBatchWorker(max_rows=N_MSGS, max_wait_ms=1000.0,
                                                                                    source="detections", decode=decode))

    def window(name):
        fn, worker = paths[name]
        t0 = time.perf_counter()
        res = fn(W, worker, msgs)
        return time.perf_counter() - t0, res

    with harness.sampled_clock() as clock:
        answers = {}
        for name in paths:
            for _ in range(2):
                _, answers[name] = window(name)
        secs = {name: [] for name in paths}
        for _ in range(args.rounds):
            for name in paths:
                secs[name].append(window(name)[0])
    for _, worker in paths.values():
        worker.close()
    result = {name: {"messages_per_s": N_MSGS / statistics.median(s), "windows_s": s} for name, s in secs.items()}
    for decode in ("host", "device"):
        a, b = answers[f"a_host_selected_{decode}"], answers[f"b_device_selected_{decode}"]
        result[f"answers_equal_{decode}"] = f"{sum(x == y for x, y in zip(a, b))}/{N_MSGS}"
        result[f"speedup_{decode}"] = result[f"b_device_selected_{decode}"]["messages_per_s"] / \
            result[f"a_host_selected_{decode}"]["messages_per_s"]
    card = harness.card(clock)
    print(json.dumps({"workload": f"{N_MSGS} single-image VQA messages, device heads of 1000 proposals x 1601 classes x 2048 "
                                  f"features, submitted at once; seed {args.seed}, {args.dtype}",
                      **result, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
