"""Pre-training heads on every row vs at chosen rows, one JSON line.

Batch 64 at (Tin, V) = (37, 101), full model, synthetic weights:
(a) one forward with the task heads and both pre-training heads on every row (select = OUT_ALL): linguisic_prediction [64, 38, 30522]
    and vision_prediction [64, 101, 1601] come back whole;
(b) one forward with the task heads and the final-state taps, then one `pretraining_heads` call on 15 % of the text rows and 15 % of the
    region rows (seeded random choice) with top_k = 5: the logits of those rows and their softmax top 5, ranked on the device.
The two paths alternate, --reps calls per window, each window ending in a device synchronisation; the median and spread over
--rounds windows of the whole-call time per batch are reported.  Bytes written to caller buffers and issued FLOPs are computed from the
shapes (GEMMs at 128-row tile granularity, as the kernels issue them).  (b)'s logits are checked bit for bit against (a)'s rows.
The card name, power limit and SM clock are read in the same run.

    python scripts/pretraining_rows_bench.py [--rounds 9] [--reps 10] [--dtype bf16]
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

B, TIN, V = 64, 37, 101
SHARE = 0.15
TOP_K = 5


def tiles(rows):
    return -(-rows // 128) * 128


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--dtype", default="bf16", choices=("fp16", "bf16"))
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    from vilbert_b200 import synthetic as S

    harness.require_gpu("pretraining_rows_bench.py")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)
    model = harness.synthetic_model(cfg, args.dtype)
    inp = [t.cuda() for t in S.synthetic_request(B, TIN, V, seed=args.seed)]
    T = TIN + 1
    H, Hv, Hb, vocab, vt = cfg.hidden_size, cfg.v_hidden_size, cfg.bi_hidden_size, cfg.vocab_size, cfg.v_target_size
    g = torch.Generator().manual_seed(args.seed)
    n_t, n_v = round(SHARE * B * T), round(SHARE * B * V)
    text_rows = torch.randperm(B * T, generator=g)[:n_t].tolist()
    image_rows = torch.randperm(B * V, generator=g)[:n_v].tolist()

    def path_a():
        return model(*inp, select=L.OUT_ALL)

    def path_b():
        out, taps = model(*inp, select=L.OUT_TASK_HEADS, debug_taps=True)
        return out, model.pretraining_heads(taps, text_rows=text_rows, image_rows=image_rows, top_k=TOP_K)

    a, (_, b) = path_a(), path_b()                       # plans, buckets and descriptors are built here
    torch.cuda.synchronize()
    identical = bool(torch.equal(b["token_logits"], a[7].reshape(-1, vocab)[torch.tensor(text_rows)]) and
                     torch.equal(b["region_logits"], a[5].reshape(-1, vt)[torch.tensor(image_rows)]))
    del a, b

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

    _, flops_a = model.plan_info(B, TIN, V, L.OUT_ALL)
    _, flops_task = model.plan_info(B, TIN, V, L.OUT_TASK_HEADS)
    heads_b = 2.0 * tiles(n_t) * (H * H + H * vocab) + 2.0 * tiles(n_v) * (Hv * Hv + Hv * vt)
    heads_a = 2.0 * tiles(B * T) * (H * H + H * vocab) + 2.0 * tiles(B * V) * (Hv * Hv + Hv * vt)
    task_bytes = 4 * B * (3129 + 1533 + 1 + 2 + 3) + 4 * B * V + 4 * B * T
    bytes_a = task_bytes + 4 * B * T * vocab + 4 * B * V * vt
    taps_bytes = 4 * (B * T * H + B * V * Hv + B * Hb)
    bytes_b = task_bytes + taps_bytes + 4 * (n_t * vocab + n_v * vt) + (n_t + n_v) * 244

    def summary(xs):
        return {"median_ms": round(statistics.median(xs), 3), "min_ms": round(min(xs), 3), "max_ms": round(max(xs), 3)}
    card = harness.card(clock)
    print(json.dumps({
        "workload": f"batch {B}, Tin {TIN} (T {T}), V {V}, {args.dtype}; (b) {n_t} text rows and {n_v} region rows, top_k {TOP_K}",
        "a_all_rows": {**summary(ms["a"]), "bytes_written": bytes_a, "issued_gflop": round(flops_a / 1e9, 1),
                       "pretraining_heads_gflop": round(heads_a / 1e9, 1)},
        "b_chosen_rows": {**summary(ms["b"]), "bytes_written": bytes_b, "issued_gflop": round((flops_task + heads_b) / 1e9, 1),
                          "pretraining_heads_gflop": round(heads_b / 1e9, 1)},
        "logits_bit_identical": identical, "rounds": args.rounds, "reps": args.reps, "card": card}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
