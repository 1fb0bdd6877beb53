import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `-m gpu`)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container (run under gpurun)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


PARITY_LOG = os.path.join(ROOT, "gpurun_out", "parity.jsonl")


@pytest.fixture(scope="session")
def parity_log():
    """Append measured parity numbers (max abs err, logit std) so they can be copied into profiles/."""
    os.makedirs(os.path.dirname(PARITY_LOG), exist_ok=True)

    def log(**kw):
        with open(PARITY_LOG, "a") as f:
            f.write(json.dumps(kw) + "\n")
        print("PARITY", json.dumps(kw))
    return log


@pytest.fixture(scope="session")
def full_oracle():
    """Full-size (268 M parameter) oracle with the seeded synthetic checkpoint (seed 42)."""
    from oracle import vilbert_ref as R
    return R.build(seed=42)


@pytest.fixture(scope="session")
def tiny_oracle():
    from oracle import vilbert_ref as R
    return R.build(R.tiny_config(), seed=7, num_labels=200)
