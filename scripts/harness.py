"""Measurement plumbing shared by the benchmark scripts.

The scripts measure one way: warm up, synchronise, time a loop of whole calls with CUDA events, alternate the compared paths window
by window, and read the card's name, its power limit and the SM clock sampled while the windows ran in the same run.  A script run
as `python scripts/<name>.py` imports this module as `harness`, after putting the repository root on sys.path (for bench.py).
torch is imported inside the functions, so a script's --help needs neither torch nor a GPU.
"""
import contextlib

from bench import ClockSampler


def require_gpu(name):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit(f"{name} needs an H100: there is no CPU path")


def synthetic_model(cfg, dtype, **kw):
    """The full synthetic VILBertForVLTasks (seed-42 weights, 3129 VQA labels) in `dtype` on cuda:0."""
    import vilbert_b200 as vb
    from vilbert_b200 import synthetic as S
    return vb.VILBertForVLTasks.from_pretrained(S.synthetic_state_dict(cfg, seed=42), config=cfg, num_labels=3129,
                                                compute_dtype=dtype, **kw).eval().cuda(0)


def timed(fn, steps, warmup):
    """ms per call of fn: `warmup` calls, a device synchronise, then CUDA events around `steps` calls."""
    import torch
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def alternate(paths, rounds, steps, warmup):
    """{name: [ms per call of each window]}: every round times each of the named callables once, in the mapping's order."""
    ms = {name: [] for name in paths}
    for _ in range(rounds):
        for name, fn in paths.items():
            ms[name].append(timed(fn, steps, warmup))
    return ms


@contextlib.contextmanager
def sampled_clock():
    """Samples the SM clock of cuda:0 (bench.ClockSampler) while the block runs; pass the sampler to card() afterwards."""
    clock = ClockSampler(0)
    clock.start()
    try:
        yield clock
    finally:
        clock.stop_flag = True
        clock.join()


def card(clock):
    """cuda:0's name and power limit through NVML (or the name and the NVML error), with the clock sampled by `clock`."""
    import torch
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(0)
        name = nv.nvmlDeviceGetName(h)
        out = {"name": name.decode() if isinstance(name, bytes) else name,
               "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception as e:          # NVML missing: report it
        out = {"name": torch.cuda.get_device_name(0), "nvml_error": repr(e)}
    out.update(clock.result())
    return out


def pixel_boxes(g, n):
    """n seeded pixel boxes [n, 4] (x1, y1, x2, y2) in a 640 x 480 image: corners in the top-left 448 x 336, sides 40..160 clipped
    to the image.  Two torch.rand calls on g."""
    import torch
    xy = torch.rand(n, 2, generator=g) * torch.tensor([448.0, 336.0])
    return torch.cat([xy, torch.minimum(xy + 40 + 120 * torch.rand(n, 2, generator=g), torch.tensor([640.0, 480.0]))], 1)
