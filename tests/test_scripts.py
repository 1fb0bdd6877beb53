"""The benchmark scripts on their shared harness (scripts/harness.py), checked without a GPU: every script that imports the harness
parses --help (each parses its arguments before importing torch or touching a device, so this catches a broken import), and the card
record keeps its keys when NVML is missing."""
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = ["ablation", "attention_maps", "decode", "head_ablation", "head_mask", "interaction", "layer_states", "long_sequence",
           "message_ablation", "packed_attention", "packed", "pretraining_objectives", "pretraining_rows", "region_select",
           "regions_packed", "relevance", "retrieval_packed", "retrieval_regions", "shapley", "worker_detections"]


@pytest.mark.parametrize("name", SCRIPTS)
def test_help(name):
    r = subprocess.run([sys.executable, os.path.join("scripts", f"{name}_bench.py"), "--help"], capture_output=True, text=True,
                       timeout=120, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout


def test_card_without_nvml(monkeypatch):
    import torch
    spec = importlib.util.spec_from_file_location("harness", os.path.join(ROOT, "scripts", "harness.py"))
    harness = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(harness)

    class Clock:
        def result(self):
            return {"sm_mhz": 1755.0, "sm_max_mhz": 1980, "reasons": ["sw_power_cap"], "samples": 12}

    monkeypatch.setitem(sys.modules, "pynvml", None)          # `import pynvml` raises ModuleNotFoundError
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda index=None: f"card {index}")
    card = harness.card(Clock())
    assert list(card) == ["name", "nvml_error", "sm_mhz", "sm_max_mhz", "reasons", "samples"]
    assert card["name"] == "card 0" and card["nvml_error"].startswith("ModuleNotFoundError")
    assert {k: card[k] for k in ("sm_mhz", "sm_max_mhz", "reasons", "samples")} == Clock().result()
