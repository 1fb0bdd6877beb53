"""BASELINE.json configs[4]: sequence-length sweep at batch 256 -- text 16..128 tokens x regions 10..100 --
pairs/s, TFLOP/s and fraction of the tensor roofline per point (CUDA-event timed, CUDA-graph replay).

    python scripts/sweep.py [--batch 256] > sweep.jsonl
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import vilbert_b200 as vb
from vilbert_b200 import synthetic as S
from vilbert_b200 import _lib as L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    peak = 1405.4
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["bf16_tflops_sustained"]
    except Exception:
        pass
    cfg = vb.BertConfig(task_specific_tokens=True)
    model = vb.VILBertForVLTasks.from_pretrained(S.synthetic_state_dict(cfg, seed=42), config=cfg, num_labels=3129).eval().cuda(0)
    for tin in (16, 32, 64, 128):
        for v in (10, 36, 64, 100):
            req = [t.cuda() for t in S.synthetic_request(a.batch, tin, v, seed=7)]
            _, flops = model.plan_info(a.batch, tin, v, L.OUT_VIL_PREDICTION)
            for _ in range(3):
                model(*req, select=L.OUT_VIL_PREDICTION)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                model(*req, select=L.OUT_VIL_PREDICTION)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
            tf = flops / (ms * 1e-3) / 1e12
            print(json.dumps(dict(batch=a.batch, n_tokens=tin, n_regions=v, ms_per_step=round(ms, 3), pairs_per_s=round(a.batch / ms * 1e3),
                                  gflop_per_pair=round(flops / a.batch / 1e9, 2), tflops=round(tf, 1), frac_of_sustained_peak=round(tf / peak, 3))),
                  flush=True)
    model.close()


if __name__ == "__main__":
    main()
