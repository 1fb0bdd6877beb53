"""Worst step-parity values over many seeds: the measurement behind oracle/step_ref.py STEP_BOUNDS.

Runs the cases of tests/test_gpu_step_parity.py (reduced-width dense shapes, packed, detector-output, past 256 rows, the 268 M model
at B = 2 and at the bench shape B = 64) in fp16 and bf16 for --seeds seeds each (the 268 M model and the long cases for fewer,
--heavy-seeds), and prints one JSON line per mode and family with the worst value, its case, step and row, the worst value per step,
and the card's name, power limit and maximum SM clock read in the same run.

    python scripts/step_parity_sweep.py [--seeds 20] [--heavy-seeds 3] [--weights synthetic|trained] [--out FILE]

--out appends the lines to FILE too.  --weights trained runs every case on oracle/trained_like.py's checkpoint-like weights (seed
trained_like.SEED), the measurement behind step_ref.STEP_BOUNDS_TRAINED; the default is the seeded synthetic checkpoint of STEP_BOUNDS.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _cases_module():
    spec = importlib.util.spec_from_file_location("step_parity_cases", os.path.join(ROOT, "tests", "test_gpu_step_parity.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _card():
    import torch
    card = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in out.split(","))
        card.update(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:          # nvidia-smi missing: report it
        card["nvidia_smi_error"] = repr(e)
    return card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=20)
    ap.add_argument("--heavy-seeds", type=int, default=3, help="seeds of the long-sequence and 268 M model cases")
    ap.add_argument("--weights", choices=("synthetic", "trained"), default="synthetic")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()

    from oracle import vilbert_ref as R
    T = _cases_module()
    worst = {}       # (mode, family) -> {"max": (err, case, label, where), "steps": {label: err}}

    failed = []

    def record(case, mode, run, *a, **kw):
        try:
            result = run(*a, **kw)
        except Exception:           # a case that cannot run is reported, and the sweep goes on to the others
            failed.append((case, mode, traceback.format_exc()))
            print(f"case {case} {mode} failed:\n{failed[-1][2]}", file=sys.stderr, flush=True)
            return
        for fam, errs in result.items():
            w = worst.setdefault((mode, T.family(fam)), {"max": (0.0, "", "", ""), "steps": {}})
            for label, e, where in errs:
                w["steps"][label] = max(w["steps"].get(label, 0.0), e)
                if e > w["max"][0]:
                    w["max"] = (e, case, label, where)

    tiny_oracle = R.build(R.tiny_config(), seed=7, num_labels=200)
    long_oracle = T.long_oracle()
    full_oracle = R.build(seed=42)
    if args.weights == "trained":
        from oracle import trained_like as TL
        tiny_oracle, long_oracle, full_oracle = (TL.trained_like(o, TL.SEED) for o in (tiny_oracle, long_oracle, full_oracle))
    for mode in T.MODES:
        model = T.engine(tiny_oracle, mode)
        for s in range(args.seeds):
            for B, Tin, V, pad in T.TINY_DENSE:
                inp = T.tiny_inputs(tiny_oracle, B, Tin, V, seed=5000 + 97 * s + 7 * B + Tin, pad=pad)
                record(f"tiny_B{B}_T{Tin}_V{V}_pad{pad}", mode, T.run_dense, model, tiny_oracle, mode, inp)
            record("tiny_packed", mode, T.run_packed, model, tiny_oracle, mode, T.packed_samples(model, T.PACKED_LENS, 6000 + 31 * s))
            imgs = T.region_images(model, T.REGION_LENS, 7000 + 31 * s) + T.region_images(model, [T.REGION_LENS[0]], 7500 + 31 * s)
            record("tiny_regions", mode, T.run_regions, model, tiny_oracle, mode, imgs)
        model.close()
        model = T.engine(long_oracle, mode, max_rows_per_sample=1024)
        for s in range(args.heavy_seeds):
            for Tin, V in T.LONG:
                record(f"long_T{Tin}_V{V}", mode, T.run_dense, model, long_oracle, mode, T.tiny_inputs(long_oracle, 2, Tin, V, 8000 + s, pad=5))
        model.close()
        model = T.engine(full_oracle, mode)
        for s in range(args.heavy_seeds):
            record("full_B2", mode, T.run_dense, model, full_oracle, mode, R.make_inputs(2, 30, 36, seed=9000 + s, pad_regions=4))
            record("full_B64", mode, T.run_dense, model, full_oracle, mode, R.make_inputs(64, 30, 36, seed=9100 + s), every=8)
        model.close()

    card = _card()
    lines = [json.dumps({"mode": mode, "family": fam, "worst": w["max"][0], "case": w["max"][1], "step": w["max"][2],
                         "where": w["max"][3], "weights": args.weights, "seeds": args.seeds, "heavy_seeds": args.heavy_seeds, "per_step": w["steps"],
                         "card": card}) for (mode, fam), w in sorted(worst.items())]
    for line in lines:
        print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write("".join(line + "\n" for line in lines))
    if failed:
        sys.exit(f"{len(failed)} case(s) failed: " + ", ".join(f"{c} {m}" for c, m, _ in failed))


if __name__ == "__main__":
    main()
