"""Per-kernel timing through the C ABI (CUDA events on the launching stream, after warm-up), at the shapes one
B=64 forward launches.  Used to pick optimisation targets and, under `ncu --set full`, to read stall reasons.

    python scripts/kernel_bench.py [--only NAME] [--reps 50] [--batch 64] [--variant 0,5] [--bn 64]
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vilbert_b200 import _lib as L


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def time_graph(run, reps, n_in_graph=20):
    """True GPU time per launch: the launches are captured once into a CUDA graph and replayed, so neither Python, ctypes,
    cuTensorMapEncode nor cudaFuncSetAttribute sit between kernels (an eager loop of ~7 us kernels is host-bound)."""
    for i in range(3):
        run(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(n_in_graph):
            run(i)
    g.replay()
    torch.cuda.synchronize()
    n = max(1, reps // n_in_graph)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (n * n_in_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--act", default="fp16")
    ap.add_argument("--sets", type=int, default=4, help="operand sets cycled through per kernel")
    ap.add_argument("--stamps", action="store_true", help="print clock64 phase stamps of the persistent kernel")
    ap.add_argument("--bn", type=int, default=0, help="override block_n of every plain GEMM")
    ap.add_argument("--variant", default="0", help="vb200_linear variant of the plain GEMMs (comma list, each timed in turn): "
                                                   "0 cooperative persistent kernel, 5 ping-pong")
    ap.add_argument("--debug", default="0", help="VB200_DEBUG timing decomposition (comma list, each timed in turn): "
                                                 "1 no MMA, 2 no stores, 4 no operand loads")
    a = ap.parse_args()
    debug_modes = [int(x) for x in str(a.debug).split(",")]
    variants = [int(x) for x in str(a.variant).split(",")]
    only = [x for x in a.only.split(",") if x]
    lib = L.load()
    B, T, V = a.batch, 31, 36
    Mt, Mv = B * T, B * V
    act = torch.float16 if a.act == "fp16" else torch.bfloat16
    f16 = 1 if a.act == "fp16" else 0
    cur = lambda: torch.cuda.current_stream().cuda_stream      # the capture stream while a graph is being recorded
    g = torch.Generator(device="cuda").manual_seed(0)
    # name, M, N, K, act, fp32 output only (the GEMMs a row LayerNorm follows), block_n
    gemms = [
        ("text_qkv", Mt, 2304, 768, 0, False, 0), ("text_attn_out_f32", Mt, 768, 768, 0, True, 0),
        ("text_ffn_in_gelu", Mt, 3072, 768, 1, False, 0), ("text_ffn_out_f32", Mt, 768, 3072, 0, True, 0),
        ("img_qkv", Mv, 3072, 1024, 0, False, 0), ("img_attn_out_f32", Mv, 1024, 1024, 0, True, 0),
        ("img_ffn_in_gelu", Mv, 1024, 1024, 1, False, 0), ("img_embed_f32", Mv, 1024, 2112, 0, True, 0),
        ("co_txt_qkv", Mt, 3072, 768, 0, False, 0), ("co_dense2_f32", Mt, 768, 1024, 0, True, 0),
        ("text_ffn_in_gelu_bn256", Mt, 3072, 768, 1, False, 256), ("pool_t", B, 1024, 768, 2, False, 0),
        ("vqa_fc0_gelu_f32", B, 2048, 1024, 1, True, 0), ("vqa_fc3", B, 3129, 2048, 0, False, 0),
        ("plain_text_ffn_out", Mt, 768, 3072, 0, False, 0), ("plain_img_out", Mv, 1024, 1024, 0, False, 0),
        ("plain_text_attn_out", Mt, 768, 768, 0, False, 0),
        # the pruned tails of the last text and image layer: one row per sample
        ("tail_text_attn_out_f32", B, 768, 768, 0, True, 0), ("tail_text_ffn_in_gelu", B, 3072, 768, 1, False, 0),
        ("tail_text_ffn_out_f32", B, 768, 3072, 0, True, 0), ("tail_img_attn_out_f32", B, 1024, 1024, 0, True, 0),
        ("tail_img_ffn_in_gelu", B, 1024, 1024, 1, False, 0), ("tail_img_ffn_out_f32", B, 1024, 1024, 0, True, 0),
    ]
    res = []
    for name, M, N, K, actf, f32, bn in gemms:
        if only and not any(o == name or (o.endswith("*") and o[:-1] in name) for o in only):
            continue
        if a.bn:
            bn = a.bn
        sets = []
        for _ in range(a.sets):
            x = torch.randn(M, K, generator=g, device="cuda").to(act)
            w = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).to(act)
            b = torch.randn(N, generator=g, device="cuda")
            ldf = (N + 3) // 4 * 4
            yb = torch.empty(M, N, dtype=act, device="cuda") if N % 8 == 0 and not f32 else None
            yf = torch.empty(M, ldf, device="cuda") if (f32 or N % 8) else None
            sets.append((x, w, b, yb, yf, ldf))

        def run(i):
            x, w, b, yb, yf, ldf = sets[i % a.sets]
            rc = lib.vb200_linear(ptr(x), K, ptr(w), K, ptr(b), None, 0, None, None, 1e-12, actf,
                                  ptr(yb), N, ptr(yf), ldf, M, N, K, bn, 0, f16, variant, None, C.c_void_p(cur()))
            L.check(rc, None)
        plain_pp = N % (bn if bn in (64, 128) else 128) == 0 and bn != 256
        for variant, dbg in [(v, d) for v in variants for d in debug_modes if v == 0 or plain_pp]:
            os.environ["VB200_DEBUG"] = str(dbg)
            us = time_graph(run, a.reps)
            fl = 2.0 * M * N * K
            res.append(dict(kernel=name, M=M, N=N, K=K, bn=bn, variant=variant, debug=dbg, us=round(us, 2), tflops=round(fl / us / 1e6, 1)))
            print(json.dumps(res[-1]), flush=True)
            if a.stamps:
                tb = torch.zeros(16 * 4096, dtype=torch.int64, device="cuda")
                x, w, b, yb, yf, ldf = sets[0]
                rc = lib.vb200_linear(ptr(x), K, ptr(w), K, ptr(b), None, 0, None, None, 1e-12, actf,
                                      ptr(yb), N, ptr(yf), ldf, M, N, K, bn, 0, f16, variant, ptr(tb), C.c_void_p(cur()))
                L.check(rc, None)
                torch.cuda.synchronize()
                t = tb.view(-1, 16).cpu()
                t = t[t[:, 0] != 0]
                d = (t - t[:, :1]).double()
                names = ["entry", "setup", "first_kblock", "mma_issued", "acc_ready", "epi_pass1", "producer_waited", "epi_done",
                         "c0_ld", "c0_res", "c0_math", "c0_store", "c1_ld", "c1_res", "c1_math", "c1_store"]
                print("   stamps (SM cycles since CTA entry, median over %d CTAs): " % len(t) +
                      ", ".join(f"{n}={int(d[:, i].median())}" for i, n in enumerate(names[:8]) if (t[:, i] != 0).any()), flush=True)
                lead = t[t[:, 11] != 0]
                if len(lead):
                    nkb = (K + 63) // 64
                    per = ((lead[:, 10] - lead[:, 2]).double() / (lead[:, 11].double() * nkb))
                    print(f"   steady state: {len(lead)} MMA-issuing CTAs, tiles/CTA median {int(lead[:, 11].median())}, "
                          f"cycles per k-block median {per.median():.0f} (min {per.min():.0f} max {per.max():.0f}); "
                          f"producer done {int((t[:, 12] - t[:, 0]).double().median())}, mma done {int((lead[:, 10] - lead[:, 0]).double().median())}, "
                          f"epilogue done {int((t[:, 13] - t[:, 0]).double().median())}", flush=True)
                if (t[:, 14] != 0).any():
                    print(f"   epilogue of warp 2: acc_ready -> first chunk loaded {int((t[:, 14] - t[:, 4]).double().median())}, "
                          f"-> first chunk stored {int((t[:, 15] - t[:, 4]).double().median())}, -> done {int((t[:, 7] - t[:, 4]).double().median())}", flush=True)
                g0, g1 = t[:, 8].double(), t[:, 9].double()
                print(f"   globaltimer: kernel span {(g1.max() - g0.min()) / 1e3:.2f} us, CTA start spread {(g0.max() - g0.min()) / 1e3:.2f} us, "
                      f"CTA lifetime median {(g1 - g0).median() / 1e3:.2f} us max {(g1 - g0).max() / 1e3:.2f} us, "
                      f"end spread {(g1.max() - g1.min()) / 1e3:.2f} us", flush=True)

    attn = [("self_attn_text", 12, 64, T), ("self_attn_img", 8, 128, V)]
    for name, heads, d, Lq in attn:
        if only and name not in only:
            continue
        H = heads * d
        qkv = torch.randn(B * Lq, 3 * H, generator=g, device="cuda").to(act)
        mask = torch.zeros(B, Lq, device="cuda")
        ctx = torch.empty(B * Lq, H, dtype=act, device="cuda")

        def run(i):
            L.check(lib.vb200_self_attention(ptr(qkv), 3 * H, H, ptr(mask), ptr(ctx), H, B, Lq, heads, d, f16, C.c_void_p(cur())), None)
        us = time_graph(run, a.reps)
        print(json.dumps(dict(kernel=name, us=round(us, 2))), flush=True)
    if not only or "co_attn" in only:
        H = 1024
        qi = torch.randn(Mv, 3 * H, generator=g, device="cuda").to(act)
        qt = torch.randn(Mt, 3 * H, generator=g, device="cuda").to(act)
        mi, mt = torch.zeros(B, V, device="cuda"), torch.zeros(B, T, device="cuda")
        ct, ci = torch.empty(Mt, H, dtype=act, device="cuda"), torch.empty(Mv, H, dtype=act, device="cuda")

        def run(i):
            L.check(lib.vb200_co_attention(ptr(qi), 3 * H, ptr(qt), 3 * H, H, ptr(mi), ptr(mt), ptr(ct), H, ptr(ci), H,
                                           B, T, V, 8, 128, f16, C.c_void_p(cur())), None)
        print(json.dumps(dict(kernel="co_attn", us=round(time_graph(run, a.reps), 2))), flush=True)


if __name__ == "__main__":
    main()
