"""Packed vs dense caption-image retrieval on one GPU (one JSON line).

Workload (seeded): one rank's block of a 1000 x 1000 retrieval, 125 captions x 1000 images (125 000 pairs).  Captions as
oracle.make_inputs draws them (7..30 real tokens, padded to 30); two region workloads:
  fixed    -- 36 regions per image (no padding);
  detector -- 1 + U{9..100} regions per image (V uniform in 10..101, what the detector returns plus the global row), padded to 101.
Per workload, parallel.retrieval_scores_cached (dense: every pair at the padded shape) and parallel.retrieval_scores_packed (every
caption and image at its own length) score the whole block, in alternating timed runs after one warm-up run each; each run is
timed with CUDA events around the whole call (padding strip, encodes, pair chunks).  Reported per path: pairs/s (median run), and
the pair-suffix FLOPs from shapes -- useful (every pair at its real lengths) and issued (dense: every pair at the padded lengths;
packed: the real lengths, since GEMM tiles past the row totals are skipped; the rows that fill the last 128-row tile of a chunk are
not counted).  The encodes run once per caption / image and are left out of the FLOP counts.  max |score difference| between the
two matrices is reported per workload, and the card name, power limit and SM clock are read in the same run.

    python scripts/retrieval_packed_bench.py [--captions 125] [--images 1000] [--pair-batch 256] [--rounds 2] [--dtype bf16]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402


def suffix_flops(cfg, T, V):
    """Algorithmic FLOPs of one pair's suffix (connection layers, the text / image layers scheduled after the first connection
    layer, poolers, vil_logit) at T text rows and V image rows."""
    H, Hv, Hb, I, Iv = cfg.hidden_size, cfg.v_hidden_size, cfg.bi_hidden_size, cfg.intermediate_size, cfg.v_intermediate_size
    n_c = len(cfg.t_biattention_id)
    n_t = cfg.num_hidden_layers - cfg.t_biattention_id[0]          # text layers after the first connection layer
    n_v = cfg.v_num_hidden_layers                                  # every image layer runs after it (v_biattention_id[0] = 0)
    text_row = n_c * (3 * Hb * H + H * Hb + 2 * I * H) + n_t * (4 * H * H + 2 * I * H)
    image_row = n_c * (3 * Hb * Hv + Hv * Hb + 2 * Iv * Hv) + n_v * (4 * Hv * Hv + 2 * Iv * Hv)
    attention = n_t * 2 * T * T * H + n_v * 2 * V * V * Hv + n_c * 4 * T * V * Hb
    heads = H * Hb + Hv * Hb + Hb
    return 2.0 * (T * text_row + V * image_row + attention + heads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--captions", type=int, default=125)
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--pair-batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2, help="alternating dense / packed timed runs per workload; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import parallel as P
    from oracle import vilbert_ref as R

    harness.require_gpu("retrieval_packed_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    dev = torch.device("cuda", 0)
    n_cap, n_img, T_PAD = args.captions, args.images, 30
    q, _, _, seg, im, _, _, _ = R.make_inputs(n_cap, T_PAD, 1, seed=args.seed, vocab_size=cfg.vocab_size)
    captions = tuple(t.to(dev) for t in (q, seg, im))
    t_lens = im.sum(dim=1).tolist()

    def images(kind):
        V = 36 if kind == "fixed" else 101
        _, f, s, _, _, vm, _, _ = R.make_inputs(n_img, 3, V, seed=args.seed + 1, vocab_size=cfg.vocab_size)   # text unused
        if kind == "detector":
            g = torch.Generator().manual_seed(args.seed + 2)
            v_lens = torch.randint(10, 102, (n_img,), generator=g)
            vm = (torch.arange(V)[None, :] < v_lens[:, None]).to(torch.uint8)
        return tuple(t.to(dev) for t in (f, s, vm)), vm.sum(dim=1).tolist(), V

    pairs = n_cap * n_img
    padded_pairs = -(-pairs // args.pair_batch) * args.pair_batch
    results = {}
    with harness.sampled_clock() as clock:
        for kind in ("fixed", "detector"):
            imgs, v_lens, V_PAD = images(kind)
            run = {"dense": lambda: P.retrieval_scores_cached(model, captions, imgs, pair_batch=args.pair_batch),
                   "packed": lambda: P.retrieval_scores_packed(model, captions, imgs, pair_batch=args.pair_batch)}
            scores = {k: fn() for k, fn in run.items()}              # warm-up: every plan either path uses
            torch.cuda.synchronize()
            secs = {"dense": [], "packed": []}
            for _ in range(args.rounds):
                for k in ("dense", "packed"):
                    secs[k].append(harness.timed(lambda: scores.update({k: run[k]()}), 1, 0) / 1e3)
            diff = float((scores["packed"] - scores["dense"]).abs().max())
            useful = sum(suffix_flops(cfg, t + 1, v) for t in t_lens for v in v_lens)
            dense_issued = padded_pairs * suffix_flops(cfg, T_PAD + 1, V_PAD)
            packed_issued = useful + (padded_pairs - pairs) * suffix_flops(cfg, t_lens[0] + 1, v_lens[0])
            path = lambda k, issued: {"pairs_per_s": pairs / statistics.median(secs[k]), "s_per_block": statistics.median(secs[k]),
                                      "runs_s": secs[k], "flops_useful": useful, "flops_issued": issued}
            results[kind] = {"regions": "36" if kind == "fixed" else f"U{{10..101}} padded to {V_PAD}",
                             "mean_regions": sum(v_lens) / n_img, "mean_tokens": sum(t_lens) / n_cap,
                             "dense": path("dense", dense_issued), "packed": path("packed", packed_issued),
                             "speedup": statistics.median(secs["dense"]) / statistics.median(secs["packed"]),
                             "issued_flops_ratio_packed_vs_dense": packed_issued / dense_issued, "max_abs_score_diff": diff}
            del imgs, scores
            torch.cuda.empty_cache()

    card = harness.card(clock)
    print(json.dumps({"workload": f"{n_cap} captions x {n_img} images (make_inputs captions, 7..30 tokens padded to {T_PAD}), "
                                  f"pair batch {args.pair_batch}, seed {args.seed}, {args.dtype}",
                      "results": results, "rounds": args.rounds, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
