"""Coalition ablation and Shapley values without a GPU: the C structs against the header, units and their validation, seeded
permutations, coalition bitmaps and chain order, the split of a layout at the engine's sample cap, the numpy restatement of the
device estimator, and argument errors raised before any engine is needed."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import vilbert_b200  # noqa: F401
from vilbert_b200 import _lib as L
from vilbert_b200 import model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6


def test_header_declares_and_library_exports_the_entry_points():
    hdr = open(HEADER).read()
    for fn in ("vb200_coalition_ablation_layout", "vb200_coalition_ablation", "vb200_shapley_values"):
        assert fn in set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
        assert fn in L.EXPORTS and hasattr(L.load(), fn)
    assert f"#define VB200_COALITION_MAX_UNITS {L.COALITION_MAX_UNITS}" in hdr


def test_structs_match_the_c_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    structs = {"vb200_coalition_message": L.CoalitionMessage, "vb200_shapley_message": L.ShapleyMessage}
    body = "".join(f'  printf("%zu' + " %zu" * len(c._fields_) + '\\n", sizeof(' + name + ")"
                   + "".join(f", offsetof({name}, {f})" for f, _ in c._fields_) + ");\n" for name, c in structs.items())
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    for line, c in zip(lines, structs.values()):
        assert [int(x) for x in line.split()] == [C.sizeof(c)] + [getattr(c, f).offset for f, _ in c._fields_]


def test_default_and_custom_units():
    # positions 1 .. Tin - 2, then every box of the message (one-box images included)
    assert M.coalition_units(None, 5, 3) == [((1,), ()), ((2,), ()), ((3,), ()), ((), (0,)), ((), (1,)), ((), (2,))]
    assert M.coalition_units(None, 2, 1) == [((), (0,))]
    assert M.coalition_units([([1, 2], []), ([], [0, 4]), ((3,), (1,))], 5, 6) == [((1, 2), ()), ((), (0, 4)), ((3,), (1,))]


@pytest.mark.parametrize("units, match", [
    ([((), ())], "unit 0 is empty"),
    ([((5,), ())], "position 5 outside"),
    ([((-1,), ())], "position -1 outside"),
    ([((), (6,))], "box 6 outside"),
    ([((1,), ()), ((1,), (2,))], "unit 1 has position 1, which unit 0"),
    ([((), (2, 2))], "unit 0 has box 2, which unit 0"),
    ([((1,),)], "needs \\(positions, boxes\\)"),
    ([], "0 units"),
    ([((), (j,)) for j in range(6)] * 200, "1200 units"),
])
def test_unit_errors(units, match):
    with pytest.raises(ValueError, match=match):
        M.coalition_units(units, 5, 6)


def test_seeded_permutations():
    a = M.shapley_permutations(9, 6, torch.Generator().manual_seed(3))
    b = M.shapley_permutations(9, 6, torch.Generator().manual_seed(3))
    assert torch.equal(a, b) and a.shape == (6, 9)
    for i in range(0, 6, 2):
        assert sorted(a[i].tolist()) == list(range(9))
        assert torch.equal(a[i + 1], a[i].flip(0))
    c = M.shapley_permutations(9, 3, torch.Generator().manual_seed(3), antithetic=False)
    assert c.shape == (3, 9) and not torch.equal(c[1], c[0].flip(0))
    with pytest.raises(ValueError, match="even number"):
        M.shapley_permutations(9, 5, torch.Generator(), antithetic=True)
    with pytest.raises(ValueError, match=">= 1"):
        M.shapley_permutations(9, 0, torch.Generator(), antithetic=False)


def test_chain_order_and_bitmaps():
    perm = torch.tensor([[2, 0, 1], [1, 2, 0]])
    ch = M.shapley_chain(perm)
    # v(empty) first (v(all) is the full input), then S^p_1 .. S^p_{n-1} per row: no duplicate of either end
    assert ch.int().tolist() == [[0, 0, 0], [0, 0, 1], [1, 0, 1], [0, 1, 0], [0, 1, 1]]
    assert M.coalition_bitmaps(ch, 3).reshape(-1).tolist() == [0, 4, 5, 2, 6]
    wide = np.zeros((2, 130), dtype=bool)
    wide[0, [0, 63, 64, 129]] = True
    wide[1, 128] = True
    bm = M.coalition_bitmaps(wide, 130)
    assert bm.dtype == np.uint64 and bm.shape == (2, 3)
    assert bm[0].tolist() == [1 | 1 << 63, 1, 2] and bm[1].tolist() == [0, 0, 1]
    with pytest.raises(ValueError, match="shape"):
        M.coalition_bitmaps(np.zeros((2, 4), dtype=bool), 5)


def test_calls_split_at_the_cap_with_their_full_input():
    recs = [(0, 0, -1, 1)] + [(0, 4, i, 1) for i in range(2500)] + [(1, 0, -1, 2)] + [(1, 4, i, 2) for i in range(10)] \
        + [(2, 0, -1, 3)] + [(2, 4, i, 3) for i in range(400)]
    calls = M.coalition_calls(recs)
    assert calls == [[(0, (0, 1023))], [(0, (1023, 2046))], [(0, (2046, 2500)), (1, (0, 10))], [(2, (0, 340))], [(2, (340, 400))]]
    base = {0: 1, 1: 2, 2: 3}
    for call in calls:
        assert sum(base[m] * (1 + c1 - c0) for m, (c0, c1) in call) <= L.ABLATION_MAX_VARIANTS
    assert M.coalition_calls([(0, 0, -1, 600)]) == [[(0, (0, 0))]]
    with pytest.raises(ValueError, match="too many"):
        M.coalition_calls([(0, 0, -1, 600), (0, 4, 0, 600)])


def test_estimator_reference():
    rng = np.random.default_rng(0)
    n, P = 5, 6
    perm = np.stack([rng.permutation(n) for _ in range(P)])
    v = rng.random(2 + P * (n - 1)).astype(np.float32)
    for g in (1, 2):
        phi, se = M.shapley_reference(v, perm, g)
        c = np.concatenate([np.full((P, 1), v[0]), v[2:].reshape(P, n - 1), np.full((P, 1), v[1])], axis=1).astype(np.float64)
        d = np.zeros((P, n))
        for p in range(P):
            d[p, perm[p]] = np.diff(c[p])
        assert np.allclose(phi, d.mean(0), atol=1e-7)
        gm = d.reshape(P // g, g, n).mean(1)
        assert np.allclose(se, gm.std(0, ddof=1) / math.sqrt(P // g), atol=1e-7)
        # efficiency: every row's marginals telescope to v(all) - v(empty)
        assert abs(float(phi.astype(np.float64).sum()) - (float(v[1]) - float(v[0]))) < 1e-6
    phi, se = M.shapley_reference(v[:2 + 2 * (n - 1)], perm[:2], 2)
    assert np.isnan(se).all()
    # a unit whose marginals are all 0: phi and stderr exactly 0
    flat = np.full(2 + P * (n - 1), 0.25, dtype=np.float32)
    phi, se = M.shapley_reference(flat, perm, 2)
    assert (phi == 0).all() and (se == 0).all()


@pytest.mark.parametrize("msg, match", [
    (("grounding", 0, 1), "grounding message"),
    (("16", 0, 1), "grounding message"),
    (("vqa", 0, 2), "n_images 2"),
    (("12", 0, 1), "n_images 1"),
    (("7", 0, 0), "n_images 0"),
    (("7", 4, 3), "outside the batch"),
    (("vqa", 0, 1, -2), "answer -2"),
    (("vqa", 0, 1, None, 5), "fields"),
    (("bogus", 0, 1), "unknown family"),
])
def test_message_errors_need_no_engine(msg, match):
    with pytest.raises(ValueError, match=match):
        M.coalition_messages([msg], 5)


def test_messages_resolve_families():
    assert M.coalition_messages([("vqa", 0, 1), ("12", 1, 2, 1), (RET, 3, 2), ("13", 4, 1)], 5) == \
        [(VQA, 0, 1, -1), (NLVR2, 1, 2, 1), (RET, 3, 2, -1), (SNLI, 4, 1, -1)]
