"""Pre-training losses from full-row logits in torch vs on the device at the masked rows, one JSON line.

Batch 64 at Conceptual-Captions-like shapes -- 36 tokens, 36 boxes plus the global row (V = 37), about 15 % of the tokens and regions
masked (synthetic.synthetic_masked_batch) -- on the full synthetic pre-training model (no task heads, task_specific_tokens off):
(a) one forward with both full-row pre-training heads (prediction_scores_t [64, 36, 30522], prediction_scores_v [64, 37, 1601]) and
    the alignment head on the pooled taps, then torch's cross_entropy(ignore_index=-1) / kl_div on the device, as upstream computes
    the losses;
(b) one forward with the final-state taps, then one vb200_pretraining_objectives call at the rows the labels pick.
The two paths alternate, --reps calls per window, each window ending in a device synchronisation; the median and spread over
--rounds windows of the whole-call time per batch are reported, with the bytes each path writes (computed from the shapes) and the
largest difference between the two paths' losses.  The card name, power limit and SM clock are read in the same run.

    python scripts/pretraining_objectives_bench.py [--rounds 9] [--reps 10] [--dtype bf16]
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

B, TIN, V = 64, 36, 37


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--dtype", default="bf16", choices=("fp16", "bf16"))
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    from vilbert_b200 import synthetic as S

    harness.require_gpu("pretraining_objectives_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=False)
    model = vb.BertForMultiModalPreTraining.from_pretrained(S.synthetic_pretraining_state_dict(cfg, seed=42), config=cfg,
                                                            compute_dtype=args.dtype).eval().cuda(0)
    vocab, vt = cfg.vocab_size, cfg.v_target_size
    batch = S.synthetic_masked_batch(B, TIN, V, seed=args.seed, vocab_size=vocab, v_feature_size=cfg.v_feature_size, v_target_size=vt)
    keys = ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")
    inp = [batch[k].cuda() for k in keys]
    lm, il, tgt, nsp = (batch[k].cuda() for k in ("masked_lm_labels", "image_label", "image_target", "next_sentence_label"))
    labels = [lm, il, tgt, nsp]                          # on the device, as (a) has them; the forward reads the small ones to the host
    n_t, n_v, n_p = int((lm != -1).sum()), int((il == 1).sum()), int((nsp != -1).sum())

    def path_a():
        out, taps = vb.VILBertForVLTasks.forward(model, *inp, None, None, select=L.OUT_LINGUISIC_PREDICTION | L.OUT_VISION_PREDICTION,
                                                 debug_taps=True)
        align = model.pretraining_heads(taps, pair_rows=range(B))["alignment"]
        t, v = out[7], out[5]
        lm_loss = F.cross_entropy(t.reshape(-1, vocab), lm.reshape(-1), ignore_index=-1)
        kl = F.kl_div(F.log_softmax(v[:, 1:], dim=2), tgt, reduction="none")
        picked = (il == 1)
        img_loss = torch.sum(kl * picked.unsqueeze(2).float()) / picked.sum()
        nsp_loss = F.cross_entropy(align, nsp, ignore_index=-1)
        return torch.stack([lm_loss, img_loss, nsp_loss])

    def path_b():
        return torch.cat(model(*inp, *labels))

    a, b = path_a(), path_b()                            # plans and row buckets are built here
    torch.cuda.synchronize()
    max_diff = float((a - b).abs().max())
    max_rel = float(((a - b).abs() / a.abs()).max())

    def window(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.reps

    with harness.sampled_clock() as clock:
        for _ in range(2):                               # warm-up windows
            window(path_a)
            window(path_b)
        ms = {"a": [], "b": []}
        for _ in range(args.rounds):
            ms["a"].append(window(path_a))
            ms["b"].append(window(path_b))

    H, Hv, Hb = cfg.hidden_size, cfg.v_hidden_size, cfg.bi_hidden_size
    taps_bytes = 4 * (B * TIN * H + B * V * Hv + B * Hb)
    bytes_a = taps_bytes + 4 * (B * TIN * vocab + B * V * vt) + 4 * B * 2          # logits written by the forward and the alignment
    bytes_b = taps_bytes + 4 * (n_t + n_v + n_p + 3)                                # per-row losses and the three reduced values

    def summary(xs):
        return {"median_ms": round(statistics.median(xs), 3), "min_ms": round(min(xs), 3), "max_ms": round(max(xs), 3)}
    card = harness.card(clock)
    print(json.dumps({
        "workload": f"batch {B}, {TIN} tokens, V {V}, {args.dtype}; {n_t} masked tokens, {n_v} masked regions, {n_p} labelled pairs",
        "a_full_rows_torch": {**summary(ms["a"]), "bytes_written": bytes_a},
        "b_device_objectives": {**summary(ms["b"]), "bytes_written": bytes_b},
        "losses_a": [round(float(x), 6) for x in a], "losses_b": [round(float(x), 6) for x in b],
        "max_abs_diff": max_diff, "max_rel_diff": max_rel, "rounds": args.rounds, "reps": args.reps, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
