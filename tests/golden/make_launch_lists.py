"""Generate launch_lists.json: the launch list of every case tests/test_gpu_launch_list.py pins (run on an H100, commit the .json).

    python tests/golden/make_launch_lists.py

Per case: vb200_profile_ops' kind, dims and FLOPs of every launch-list entry, vb200_plan_info's launch count and FLOPs and
vb200_timeline's {M, N, K, stream} of every GEMM.  No time is recorded.  bench.py groups its per-kernel table by these kinds and
dims, so a change to them is a change to that table.
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

POOLED = 0x1F                   # the heads that read pooled_output only: both tails are pruned
ROW_HEADS = (1 << 6) | (1 << 8)   # VISION_LOGIT | LINGUISIC_LOGIT: every final row of both streams is read
OUT_ALL = 0x1FF

# name -> (model, compute dtype, (batch, n_tokens, n_regions), select, gemm_kernel)
CASES = {
    "tiny_fp16": ("tiny", "fp16", (4, 30, 36), OUT_ALL, 1),
    "tiny_bf16": ("tiny", "bf16", (4, 30, 36), OUT_ALL, 1),
    "tiny_fp32x": ("tiny", "fp32x", (4, 30, 36), OUT_ALL, 1),
    "full_b1": ("full", "bf16", (1, 30, 36), 1, 1),
    "full_b8": ("full", "bf16", (8, 30, 36), 1, 1),            # lone-rows 64-wide tiles
    "full_b64": ("full", "bf16", (64, 30, 36), 1, 1),
    "full_b512": ("full", "bf16", (512, 30, 36), 1, 1),
    "full_b64_pooled": ("full", "bf16", (64, 30, 36), POOLED, 1),
    "full_b64_row_heads": ("full", "bf16", (64, 30, 36), POOLED | ROW_HEADS, 1),
    "full_b64_cooperative": ("full", "bf16", (64, 30, 36), 1, 0),
}


def engine(oracle, dtype):
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    return vb.VILBertForVLTasks.from_pretrained(oracle.state_dict(), config=cfg, num_labels=oracle.num_labels,
                                                compute_dtype=dtype, max_plans=64).eval().cuda(0)


def record(model, shape, select, gemm_kernel):
    """The case's launch list on `model`; leaves the engine at gemm_kernel 1 with the timeline off."""
    from vilbert_b200 import _lib as L
    lib, h = L.load(), model._handle
    B, Tin, V = shape
    model.set_option("gemm_kernel", gemm_kernel)
    launches, flops = model.plan_info(B, Tin, V, select)
    cap = 4096
    n = C.c_int32()
    kinds, ms, fl, dims = (C.c_int32 * cap)(), (C.c_double * cap)(), (C.c_double * cap)(), (C.c_int32 * (4 * cap))()
    L.check(lib.vb200_profile_ops(h, B, Tin, V, select, 1, cap, C.byref(n), kinds, ms, fl, dims), h)
    ops = [[kinds[i], *dims[4 * i:4 * i + 4], fl[i]] for i in range(n.value)]
    model.set_option("timeline", 1)
    try:
        L.check(lib.vb200_timeline(h, B, Tin, V, select, 0, cap, C.byref(n), dims, None), h)
        timeline = [list(dims[4 * i:4 * i + 4]) for i in range(n.value)]
    finally:
        model.set_option("timeline", 0)
        model.set_option("gemm_kernel", 1)
    return {"launches": launches, "flops": flops, "ops": ops, "timeline": timeline}


def main():
    from oracle import vilbert_ref as R
    oracles = {"tiny": R.build(R.tiny_config(), seed=7, num_labels=200), "full": R.build(seed=42)}
    out = {}
    for (kind, dtype) in sorted({(c[0], c[1]) for c in CASES.values()}):
        m = engine(oracles[kind], dtype)
        for name, (k, d, shape, select, gk) in CASES.items():
            if (k, d) == (kind, dtype):
                out[name] = record(m, shape, select, gk)
                print(name, out[name]["launches"], out[name]["flops"])
        m.close()
    fn = os.path.join(os.path.dirname(os.path.abspath(__file__)), "launch_lists.json")
    with open(fn, "w") as f:
        json.dump({name: out[name] for name in CASES}, f, separators=(",", ":"))
        f.write("\n")
    print("wrote", fn)


if __name__ == "__main__":
    main()
