"""Retrieval galleries from raw detector heads: host-side construction vs encode_detections_packed on one GPU (one JSON line).

Workload (seeded): one rank's block of a 1000 x 1000 retrieval, 125 captions x 1000 images, bf16.  Captions as oracle.make_inputs
draws them (7..30 real tokens).  Every gallery image has detector heads of 1000 proposals x 1601 classes x 2048 features
(`synthetic.synthetic_detections`, N(0, 2) logits); to keep host-side generation short the 1000 images cycle through --pool distinct
seeded heads, resident on the device.  Each image keeps its top 100 boxes.  Two ways to turn the heads into cached gallery states:
  (a) host -- worker_api.process_feature_extraction (the selection, with the per-image lists the reference returns), then
      custom_prediction's construction (mean row, normalised boxes and area, the [0,0,1,1,1] row) with torch ops on the device over
      all images at once, then model.encode_image_packed;
  (b) device -- model.encode_detections_packed: one select_regions into packed rows, one encode_regions_packed.
Each encode is timed with a host clock around the call and a device synchronise, in alternating runs after one warm-up each; the
median is reported.  The caption states are encoded once, and the block's 125 000 pairs are scored from each gallery in chunks of
--pair-batch with forward_cached_packed (CUDA events, alternating; pairs/s of the median run).  Reported: max |score difference|
between (a) and (b) (the torch mean row is summed in another order), and for (b) the max |difference| against forward_regions_packed
of --sample random pairs, which is 0.0 when the reuse path is bit-identical to the forward.  The card name, power limit and SM clock
are read in the same run.

    python scripts/retrieval_regions_bench.py [--captions 125] [--images 1000] [--pool 100] [--pair-batch 256] [--rounds 3]
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

IMAGE_W, IMAGE_H = 1333.0, 800.0                  # the synthetic heads' original image (proposals are at im_scale times it)


def host_gallery(model, W, heads, max_boxes):
    """Path (a): process_feature_extraction, custom_prediction's construction with torch ops on the device, encode_image_packed."""
    import numpy as np
    import torch
    props, scores, feats, scales = zip(*heads)
    infos = [{"width": IMAGE_W, "height": IMAGE_H}] * len(heads)
    feat_list, info_list = W.process_feature_extraction(props, scores, feats, scales, infos, num_features=max_boxes)
    dev = feat_list[0].device
    k = torch.tensor([f.shape[0] for f in feat_list], device=dev)
    bf = torch.cat(feat_list)
    bx = torch.from_numpy(np.concatenate([i["bbox"] for i in info_list])).to(dev)
    n = len(feat_list)
    img = torch.repeat_interleave(torch.arange(n, device=dev), k)
    mean = torch.zeros(n, bf.shape[1], device=dev).index_add_(0, img, bf) / k[:, None].float()     # worker.py:432-434
    loc = torch.zeros(bx.shape[0], 5, device=dev)
    loc[:, :4] = bx
    loc[:, 4] = (loc[:, 3] - loc[:, 1]) * (loc[:, 2] - loc[:, 0]) / (IMAGE_W * IMAGE_H)
    loc[:, [0, 2]] /= IMAGE_W
    loc[:, [1, 3]] /= IMAGE_H
    rows = k + 1
    first = torch.cumsum(rows, 0) - rows                                                # each image's mean row
    is_box = torch.ones(int(rows.sum()), dtype=torch.bool, device=dev)
    is_box[first] = False
    f = torch.empty(is_box.numel(), bf.shape[1], device=dev)
    s = torch.empty(is_box.numel(), 5, device=dev)
    f[first], f[is_box] = mean, bf
    s[first], s[is_box] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0], device=dev), loc    # worker.py:443-444
    return model.encode_image_packed(f, s, rows.tolist(), max_regions=max_boxes + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--captions", type=int, default=125)
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--pool", type=int, default=100, help="distinct seeded detector heads the gallery cycles through")
    ap.add_argument("--proposals", type=int, default=1000)
    ap.add_argument("--max-boxes", type=int, default=100)
    ap.add_argument("--pair-batch", type=int, default=256)
    ap.add_argument("--sample", type=int, default=64, help="pairs of (b) checked against forward_regions_packed")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import parallel as P
    from vilbert_b200 import synthetic as S
    from vilbert_b200 import worker_api as W
    from oracle import vilbert_ref as R

    harness.require_gpu("retrieval_regions_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    W.model = model
    dev = torch.device("cuda", 0)
    n_cap, n_img, K = args.captions, args.images, args.max_boxes
    q, _, _, seg, im, _, _, _ = R.make_inputs(n_cap, 30, 1, seed=args.seed, vocab_size=cfg.vocab_size)
    t_lens = im.sum(dim=1).tolist()
    q_rows, seg_rows = P.pack_rows(q, t_lens).to(dev), P.pack_rows(seg, t_lens).to(dev)
    ts = model.encode_text_packed(q_rows, seg_rows, torch.full((n_cap, 1), 7, dtype=torch.long, device=dev), t_lens)
    pool = [tuple(t.to(dev) if torch.is_tensor(t) else t for t in d)
            for d in S.synthetic_detections(min(args.pool, n_img), args.proposals, seed=args.seed + 1)]
    heads = [pool[i % len(pool)] for i in range(n_img)]
    image_wh = torch.tensor([[IMAGE_W, IMAGE_H]] * n_img)

    encode = {"host": lambda: host_gallery(model, W, heads, K),
              "device": lambda: model.encode_detections_packed(heads, image_wh, max_boxes=K)}
    ci, ii, total = P.retrieval_pairs(n_cap, n_img, args.pair_batch)

    def score(vs):
        out = torch.empty(ci.numel(), dtype=torch.float32, device=dev)
        for s0 in range(0, ci.numel(), args.pair_batch):
            out[s0:s0 + args.pair_batch] = model.forward_cached_packed(ts, ci[s0:s0 + args.pair_batch], vs,
                                                                       ii[s0:s0 + args.pair_batch])[2].view(-1)
        return out[:total].view(n_cap, n_img)

    with harness.sampled_clock() as clock:
        states = {k: fn() for k, fn in encode.items()}                # warm-up: every plan either path uses
        scores = {k: score(v) for k, v in states.items()}
        torch.cuda.synchronize()
        enc_s, pair_s = {k: [] for k in encode}, {k: [] for k in encode}
        for _ in range(args.rounds):
            for k in encode:
                del states[k]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                states[k] = encode[k]()
                torch.cuda.synchronize()
                enc_s[k].append(time.perf_counter() - t0)
                pair_s[k].append(harness.timed(lambda: scores.update({k: score(states[k])}), 1, 0) / 1e3)
        diff = float((scores["host"] - scores["device"]).abs().max())

        # (b) against the worker's forward of the same pairs: one selection of the sampled images, then forward_regions_packed
        g = torch.Generator().manual_seed(args.seed + 3)
        pc = torch.randint(0, n_cap, (args.sample,), generator=g).tolist()
        pi = torch.randint(0, n_img, (args.sample,), generator=g).tolist()
        r = model.select_regions([heads[i] for i in pi], K)
        t_offs = [0] + list(torch.cumsum(torch.tensor(t_lens), 0).tolist())
        rows = lambda x: torch.cat([x[t_offs[c]:t_offs[c + 1]] for c in pc])
        fwd, _ = model.forward_regions_packed(rows(q_rows), rows(seg_rows), torch.full((args.sample, 1), 7, dtype=torch.long, device=dev),
                                              r["box_features"], r["boxes"], image_wh[pi], [t_lens[c] for c in pc], r["n_boxes"],
                                              select=vb.OUT_VIL_LOGIT, return_spatials=False)
        torch.cuda.synchronize()
        fwd_diff = float((fwd[2].view(-1) - scores["device"][pc, pi]).abs().max())

    card = harness.card(clock)
    med = lambda xs: statistics.median(xs)
    print(json.dumps({
        "workload": f"{n_cap} captions x {n_img} images, heads {args.proposals} x 1601 x 2048 ({len(pool)} distinct), top {K} boxes, "
                    f"pair batch {args.pair_batch}, seed {args.seed}, {args.dtype}",
        "encode_s": {k: med(v) for k, v in enc_s.items()}, "encode_runs_s": enc_s,
        "encode_speedup_device_vs_host": med(enc_s["host"]) / med(enc_s["device"]),
        "pairs_per_s": {k: total / med(v) for k, v in pair_s.items()}, "pair_runs_s": pair_s,
        "mean_boxes": int(states["device"]["offsets"][-1]) / n_img - 1,
        "max_abs_score_diff_host_vs_device": diff, "sampled_pairs": args.sample,
        "max_abs_diff_device_vs_forward_regions_packed": fwd_diff, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
