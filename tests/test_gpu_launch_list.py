"""The engine's launch lists, pinned: per case, vb200_profile_ops' kind, dims and FLOPs of every entry, vb200_plan_info's launch count
and FLOPs and vb200_timeline's {M, N, K, stream} of every GEMM, against tests/golden/launch_lists.json (written by
tests/golden/make_launch_lists.py).  bench.py groups its per-kernel table by these kinds and dims.  Times are not compared.
`-m gpu` only.
"""
import json
import os
import sys

import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLDEN)
import make_launch_lists as G  # noqa: E402
sys.path.remove(GOLDEN)

with open(os.path.join(GOLDEN, "launch_lists.json")) as f:
    WANT = json.load(f)


@pytest.fixture(scope="module")
def engines(tiny_oracle, full_oracle):
    oracles = {"tiny": tiny_oracle, "full": full_oracle}
    made = {}

    def get(kind, dtype):
        if (kind, dtype) not in made:
            made[kind, dtype] = G.engine(oracles[kind], dtype)
        return made[kind, dtype]
    yield get
    for m in made.values():
        m.close()


def test_every_case_is_pinned():
    assert sorted(WANT) == sorted(G.CASES)


@pytest.mark.parametrize("name", list(G.CASES))
def test_launch_list(engines, name):
    kind, dtype, shape, select, gemm_kernel = G.CASES[name]
    got = G.record(engines(kind, dtype), shape, select, gemm_kernel)
    want = WANT[name]
    assert got["launches"] == want["launches"]
    assert got["flops"] == want["flops"]
    assert len(got["ops"]) == len(want["ops"])
    for i, (g, w) in enumerate(zip(got["ops"], want["ops"])):
        assert g == w, f"launch-list entry {i}: [kind, dims, flops] {g} != {w}"
    assert got["timeline"] == want["timeline"]
    assert sum(op[5] for op in got["ops"]) == got["flops"]
