"""Where the SMs spend a step: per-SM occupancy by persistent GEMM CTAs while `--inflight` batches run concurrently.

Needs a -DVB200_STAMPS build for the "first k-block landed" stamp (`make -C vilbert-multi-task_b200/csrc EXTRA=-DVB200_STAMPS`).
Every GEMM CTA of the LAST forward of each workspace slot leaves (SM id, %globaltimer at entry / exit, clock64 at entry, first
operand tile landed, last tile accumulated, exit) -- include/vilbert_b200.h vb200_timeline.  Inside the window in which all slots'
last forwards overlap, for every SM:

  resident k   fraction of the window with exactly k GEMM CTAs resident (k = 0: the SM runs LayerNorm / attention CTAs or nothing)
  mma k        fraction with exactly k resident CTAs between "first k-block landed" and "last tile accumulated" (their main loop)

and per launch family the mean CTA lifetime split into prologue (entry -> first k-block), main loop, tail (last tile accumulated -> exit).
Prints one JSON object; `--out` also saves it.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--n-tokens", type=int, default=30)
    ap.add_argument("--n-regions", type=int, default=36)
    ap.add_argument("--inflight", type=int, default=2)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    from vilbert_b200 import synthetic as S

    dev = torch.device("cuda:0")
    cfg = vb.BertConfig(task_specific_tokens=True, visualization=True)       # worker.py:509-522
    sd = S.synthetic_state_dict(cfg, seed=42)
    model = vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=3129, compute_dtype=args.dtype).eval().cuda(0)
    model.set_option("timeline", 1)
    B, Tin, V = args.batch, args.n_tokens, args.n_regions
    sel = L.OUT_VIL_PREDICTION
    reqs = [[t.to(dev) for t in S.synthetic_request(B, Tin, V, seed=1234 + i)] for i in range(4)]
    nfl = args.inflight
    streams = [torch.cuda.Stream(device=dev) for _ in range(nfl)]
    for i in range(args.steps + 3 * nfl):
        with torch.cuda.stream(streams[i % nfl]):
            model(*reqs[i % 4], select=sel, slot=i % nfl)
    torch.cuda.synchronize()

    lib = L.load()
    cap, ctas = 256, 304
    recs = []                                               # (slot, op, dims, stamps[ctas, 16])
    for slot in range(nfl):
        n = C.c_int32()
        dims = (C.c_int32 * (4 * cap))()
        st = np.zeros((cap, ctas, 16), dtype=np.int64)
        L.check(lib.vb200_timeline(model._handle, B, Tin, V, sel, slot, cap, C.byref(n), dims, st.ctypes.data_as(C.POINTER(C.c_int64))),
                model._handle)
        for o in range(min(n.value, cap)):
            recs.append((slot, o, tuple(dims[4 * o:4 * o + 4]), st[o]))

    # ---- intervals in ns (globaltimer); clock64 differences scaled by the CTA's own (exit - entry) ratio
    iv_owner = []
    iv = []                                                 # slot, dims, sm, t_in, t_first, t_mma_end, t_out
    for slot, o, d, st in recs:
        live = st[:, 9] > 0
        for c in np.nonzero(live)[0]:
            s = st[c]
            t_in, t_out = float(s[8]), float(s[9])
            cyc = float(s[13] - s[0])
            ns_per_cyc = (t_out - t_in) / cyc if cyc > 0 else 0.0
            first = t_in + (s[2] - s[0]) * ns_per_cyc if s[2] > 0 else t_in
            mma_end = t_in + (s[10] - s[0]) * ns_per_cyc if s[10] > 0 else t_out
            iv.append((slot, d, int(s[12]), t_in, first, mma_end, t_out, int(s[11])))
            iv_owner.append((slot, o))
    if not iv:
        raise SystemExit("no stamps: was the library built with -DVB200_STAMPS and the timeline option set?")
    per_slot = {}
    for r in iv:
        a = per_slot.setdefault(r[0], [np.inf, -np.inf])
        a[0] = min(a[0], r[3]); a[1] = max(a[1], r[6])
    w0 = max(a[0] for a in per_slot.values())
    w1 = min(a[1] for a in per_slot.values())
    out = {"config": vars(args), "forward_ns": {str(k): v[1] - v[0] for k, v in per_slot.items()}, "window_ns": w1 - w0}
    if w1 <= w0:
        out["error"] = "the slots' last forwards do not overlap"
        print(json.dumps(out)); return

    def occupancy(key_lo, key_hi):
        """Fractions of the window with exactly k intervals [lo, hi) open, averaged over the SMs."""
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        frac = np.zeros(4)
        for sm in range(n_sm):
            ev = []
            for r in iv:
                if r[2] != sm: continue
                lo, hi = max(r[key_lo], w0), min(r[key_hi], w1)
                if hi > lo: ev += [(lo, 1), (hi, -1)]
            ev.sort()
            t, k = w0, 0
            for tt, dlt in ev:
                frac[min(k, 3)] += tt - t
                t, k = tt, k + dlt
            frac[min(k, 3)] += w1 - t
        return (frac / (n_sm * (w1 - w0))).round(4).tolist()

    out["resident_fraction_by_count"] = occupancy(3, 6)       # [0 CTAs, 1, 2, >= 3]
    out["main_loop_fraction_by_count"] = occupancy(4, 5)
    fam = {}
    for r in iv:
        f = fam.setdefault(r[1][:3], [0, 0.0, 0.0, 0.0, 0])
        f[0] += 1; f[1] += r[4] - r[3]; f[2] += r[5] - r[4]; f[3] += r[6] - r[5]; f[4] += r[7]
    out["families"] = [dict(M=k[0], N=k[1], K=k[2], ctas=v[0], tiles_per_cta=round(v[4] / v[0], 2), prologue_us=round(v[1] / v[0] / 1e3, 2),
                            main_us=round(v[2] / v[0] / 1e3, 2), tail_us=round(v[3] / v[0] / 1e3, 2)) for k, v in sorted(fam.items(), key=lambda kv: -kv[1][0])]
    # one-tile CTAs: where prologue and tail go (clock64 stamps of the first = only tile, in cycles)
    #   0 entry | 1 setup done | 6 producer past griddepcontrol.wait | 2 first k-block landed | 10 last MMA committed | 4 accumulator ready
    #   14 first 32-column chunk in registers | 15 first chunk stored | 5 all chunks stored (+ TMA store read) | 13 exit
    br = {}
    for slot, o, d, st in recs:
        for c in np.nonzero((st[:, 9] > 0) & (st[:, 11] == 1) & (st[:, 2] > 0) & (st[:, 4] > 0))[0]:
            x = st[c]
            b = br.setdefault(tuple(d[:3]), [0] + [0.0] * 9)
            b[0] += 1
            for i, (lo, hi) in enumerate([(0, 1), (1, 6), (6, 2), (2, 10), (10, 4), (4, 14), (14, 15), (15, 5), (5, 13)]):
                b[1 + i] += float(x[hi] - x[lo])
    names = ["setup", "setup_to_pdl_wait_done", "pdl_to_first_kblock", "main_loop", "mma_drain", "first_acc_read", "first_chunk_store",
             "other_chunks_and_tma_store", "teardown"]
    out["one_tile_cta_cycles"] = [dict(M=k[0], N=k[1], K=k[2], ctas=v[0], **{n: round(v[1 + i] / v[0]) for i, n in enumerate(names)})
                                  for k, v in sorted(br.items(), key=lambda kv: -kv[1][0])]
    # how many distinct GEMM launches (slot, op) have a CTA resident / in their main loop at a time, GPU-wide (time-weighted histogram)
    def launches_active(key_lo, key_hi):
        ev = []
        # one interval per (slot, op): from its first CTA's key_lo to its last CTA's key_hi
        agg = {}
        for r, (slot, o) in zip(iv, iv_owner):
            a = agg.setdefault((slot, o), [np.inf, -np.inf])
            a[0] = min(a[0], r[key_lo]); a[1] = max(a[1], r[key_hi])
        for lo, hi in agg.values():
            lo, hi = max(lo, w0), min(hi, w1)
            if hi > lo: ev += [(lo, 1), (hi, -1)]
        ev.sort()
        hist = np.zeros(8)
        t, k = w0, 0
        for tt, dlt in ev:
            hist[min(k, 7)] += tt - t
            t, k = tt, k + dlt
        hist[min(k, 7)] += w1 - t
        return (hist / (w1 - w0)).round(4).tolist()

    out["gemm_launches_resident_hist"] = launches_active(3, 6)      # index = number of GEMM launches with a resident CTA (7 = 7 or more)
    out["gemm_launches_in_main_loop_hist"] = launches_active(4, 5)
    # CTAs resident GPU-wide (of one slot per SM), time-weighted mean and the share of them that are still waiting for their producer kernel
    res_ns = sum(min(r[6], w1) - max(r[3], w0) for r in iv if min(r[6], w1) > max(r[3], w0))
    out["mean_gemm_ctas_resident"] = round(res_ns / (w1 - w0), 1)
    tot = sum(r[6] - r[3] for r in iv if r[3] >= w0 and r[6] <= w1)
    out["gemm_cta_ns_in_window"] = tot
    out["slot_capacity_ns"] = torch.cuda.get_device_properties(0).multi_processor_count * (w1 - w0)
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
