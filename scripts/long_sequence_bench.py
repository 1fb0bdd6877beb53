"""Long sequences: the staged and the streaming attention kernels side by side, and whole forwards past 256 rows (one JSON line).

Op level: CUDA-event time per launch of vb200_self_attention / vb200_co_attention (staged: a (sample, head) per CTA, staged whole in
shared memory) and of the streaming hooks (64 query rows per CTA, K / V streamed in 64-key blocks), batch 64, D = 64 (12 heads,
the text stream) and D = 128 (8 heads, image and co-attention), at L in {31, 36, 101, 256} where both run (co-attention: T = V = L),
and the streaming kernels alone at L in {512, 1024}.  Algorithmic FLOPs (4 B heads L^2 D per self-attention, 8 B heads T V D per
co-attention) beside each time.
Model level: pairs/s of forwards of the full 12/6/6 model (seeded weights, bf16, max_rows_per_sample 1024) at (Tin, V) in
{(30, 36), (511, 36), (30, 1000), (511, 1000)}, batch --batch.
The card's name, power limit and SM clock are read in the same run.

    python scripts/long_sequence_bench.py [--batch 8] [--iters 20]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import harness  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8, help="model-level batch")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    from oracle import vilbert_ref as R

    lib = L.load()
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def timed(fn):
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    with harness.sampled_clock() as clock:
        ops = []
        B = 64
        for d, heads in ((64, 12), (128, 8)):
            H = heads * d
            for L_ in (31, 36, 101, 256, 512, 1024):
                qkv = torch.randn(B * L_, 3 * H, device="cuda").half()
                mask = torch.zeros(B * L_, device="cuda")
                ctx = torch.empty(B * L_, H, device="cuda").half()
                ct, ci = torch.empty_like(ctx), torch.empty_like(ctx)
                row = {"D": d, "heads": heads, "B": B, "L": L_, "self_flops": 4.0 * B * heads * L_ * L_ * d,
                       "co_flops": 8.0 * B * heads * L_ * L_ * d}

                def self_(name, offs=()):
                    return lambda: L.check(getattr(lib, name)(qkv.data_ptr(), 3 * H, H, mask.data_ptr(), ctx.data_ptr(), H, B, L_,
                                                              heads, d, 1, *offs, st()))

                def co_(name, offs=()):
                    return lambda: L.check(getattr(lib, name)(qkv.data_ptr(), 3 * H, qkv.data_ptr(), 3 * H, H, mask.data_ptr(),
                                                              mask.data_ptr(), ct.data_ptr(), H, ci.data_ptr(), H, B, L_, L_, heads,
                                                              d, 1, *offs, st()))
                row["stream_self_ms"] = timed(self_("vb200_self_attention_stream", (None,)))
                row["stream_co_ms"] = timed(co_("vb200_co_attention_stream", (None, None)))
                if L_ <= 256:
                    row["staged_self_ms"] = timed(self_("vb200_self_attention"))
                    row["staged_co_ms"] = timed(co_("vb200_co_attention"))
                ops.append(row)
                del qkv, mask, ctx, ct, ci

        oracle = R.build(seed=42)
        cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
        model = vb.VILBertForVLTasks.from_pretrained(oracle.state_dict(), config=cfg, num_labels=oracle.num_labels,
                                                     compute_dtype="bf16", max_rows_per_sample=1024).eval().cuda(0)
        del oracle
        shapes = []
        for tin, v in ((30, 36), (511, 36), (30, 1000), (511, 1000)):
            inp = [t.cuda() for t in R.make_inputs(args.batch, tin, v, seed=1, full_masks=True)]
            ms = timed(lambda: model(*inp))
            n, fl = model.plan_info(args.batch, tin, v)
            shapes.append({"Tin": tin, "V": v, "batch": args.batch, "ms": ms, "pairs_per_s": args.batch / ms * 1e3, "launches": n,
                           "flops": fl})
        model.close()
    card = harness.card(clock)
    print(json.dumps({"card": card, "ops": ops, "model": shapes}))


if __name__ == "__main__":
    main()
