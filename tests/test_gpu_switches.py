"""Every A/B launch switch against the default path.  `-m gpu` only.

The VB200_* switches of the README's "A/B switches" list change how a kernel is launched -- the persistent GEMM grid, the tile
width of small forwards, warps per attention CTA, rows per LayerNorm CTA, the default GEMM kernel, programmatic dependent launch --
and are documented to give the same bits.  Each is read once per process, so every setting runs tests/switch_child.py in a fresh
process: the child checks each kernel against its oracle at the shapes where the setting moves work around (exact GEMMs at tile
counts around the setting's grid, LayerNorm at ragged row counts, attention at every edge mask) and digests every output.  The test
then requires the digests it shares with a run without any VB200_* variable to be equal: a setting may not change a single bit.
"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHILD = os.path.join(HERE, "switch_child.py")
TIMEOUT = 600

ALL_AT_ONCE = {"GRID_PCT": "37", "GRID_BALANCE": "0", "LN_ROWS": "3", "ATTN_SPLIT_WARPS": "1", "LONE_ROWS": "0", "GEMM": "coop",
               "PDL": "off"}
# (setting, sections): each setting runs the sections whose launches it changes
SETTINGS = [
    ({"GRID_PCT": "10"}, "gemm,fwd"),
    ({"GRID_PCT": "37"}, "gemm,fwd,full"),
    ({"GRID_BALANCE": "0"}, "gemm,fwd"),
    ({"GRID_PCT": "37", "GRID_BALANCE": "0"}, "gemm"),
    ({"LN_ROWS": "1"}, "ln,fwd"),
    ({"LN_ROWS": "3"}, "ln,fwd"),
    ({"LN_ROWS": "8"}, "ln,fwd"),
    ({"ATTN_SPLIT_WARPS": "1"}, "attn,fwd"),
    ({"LONE_ROWS": "0"}, "fwd,full"),
    ({"LONE_ROWS": "100000"}, "fwd,full"),
    ({"GEMM": "coop"}, "gemm_rows,fwd"),
    ({"PDL": "off"}, "fwd"),
    (ALL_AT_ONCE, "gemm,ln,attn,fwd,full"),
    # out of range: the code maps each back to its default (100 %, 2 rows per CTA, lone rows off); the grid-stamp cases check that
    # the grid is the full one
    ({"GRID_PCT": "5", "LN_ROWS": "9", "LONE_ROWS": "-1"}, "gemm_grid,ln,fwd"),
]


def _id(setting):
    return "all" if setting is ALL_AT_ONCE else "+".join(f"{k}={v}" for k, v in setting.items())


def _clean_env():
    """os.environ without any VB200_* variable: a developer's shell settings stay out of the baseline."""
    return {k: v for k, v in os.environ.items() if not k.startswith("VB200_")}


def _run_child(env, sections, out):
    """One child process; (exit code, stderr tail, digests or None).  subprocess.run kills the child on timeout."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [CHILD, "--sections", sections, "--out", str(out)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=TIMEOUT)
    digests = None
    if r.returncode == 0:
        with open(out) as f:
            digests = json.load(f)
    return r.returncode, (r.stdout + r.stderr)[-4000:], digests


@pytest.fixture(scope="module")
def baseline(tmp_path_factory):
    rc, tail, digests = _run_child(_clean_env(), "gemm,ln,attn,fwd,full", tmp_path_factory.mktemp("switches") / "baseline.json")
    assert rc == 0, f"the child failed without any VB200_* setting:\n{tail}"
    return digests


@pytest.mark.parametrize("setting,sections", SETTINGS, ids=[_id(s) for s, _ in SETTINGS])
def test_switch_same_bits(setting, sections, baseline, tmp_path):
    """The child passes its checks under the setting, and every output it shares with the baseline has the baseline's bits.  The
    tile-count cases are named by their tile count, which follows the grid, so most of them exist under one setting only: for them
    the in-child exact check is the oracle."""
    env = _clean_env()
    env.update({"VB200_" + k: v for k, v in setting.items()})
    rc, tail, digests = _run_child(env, sections, tmp_path / "digests.json")
    assert rc == 0, f"the child failed under {_id(setting)}:\n{tail}"
    missing = [k for k in digests if k not in baseline and not k.startswith("gemm/tiles")]
    assert not missing, f"outputs without a baseline: {missing[:20]}"
    shared = sorted(set(digests) & set(baseline))
    differ = [k for k in shared if digests[k] != baseline[k]]
    assert not differ, f"{len(differ)} of {len(shared)} outputs differ from the baseline under {_id(setting)}: {differ[:40]}"
