"""Shapley-Taylor pair indices without a GPU: the C struct against the header, cross pairs and the pair coalitions on a hand-worked
example, the numpy restatement of the device estimator against the exact index from its subset formula and against efficiency,
pair and message errors raised before any engine is needed, and the split of a layout whose pair coalitions cross the engine's
sample cap."""
import ctypes as C
import itertools
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")


def test_header_declares_and_library_exports_the_entry_point():
    hdr = open(HEADER).read()
    assert "vb200_interaction_values" in set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    assert "vb200_interaction_values" in L.EXPORTS and hasattr(L.load(), "vb200_interaction_values")
    assert f"#define VB200_INTERACTION_MAX_PAIRS {L.INTERACTION_MAX_PAIRS}" in hdr


def test_struct_matches_the_c_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    c, name = L.InteractionMessage, "vb200_interaction_message"
    body = (f'  printf("%zu' + " %zu" * len(c._fields_) + '\\n", sizeof(' + name + ")"
            + "".join(f", offsetof({name}, {f})" for f, _ in c._fields_) + ");\n")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    line = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in line] == [C.sizeof(c)] + [getattr(c, f).offset for f, _ in c._fields_]


def test_cross_pairs():
    units = [((1,), ()), ((), (0,)), ((2, 3), ()), ((4,), (1,)), ((), (2, 5))]
    # word units 0 and 2, box units 1 and 4; unit 3 has both and is in no pair
    assert M.cross_pairs(units) == [(0, 1), (0, 4), (2, 1), (2, 4)]
    assert M.cross_pairs([((1,), ()), ((2,), ())]) == []


def test_pair_coalitions_by_hand():
    """4 units, 2 permutations, pairs (0, 2) and (3, 1): S + {second} then S + {a, b} per permutation and pair."""
    perm = torch.tensor([[2, 0, 3, 1], [1, 3, 0, 2]])
    got = M.interaction_coalitions(perm, [(0, 2), (3, 1)])
    assert got.dtype == torch.bool and got.shape == (8, 4)
    assert got.int().tolist() == [
        [1, 0, 0, 0], [1, 0, 1, 0],      # row 0, pair (0, 2): S = {}, first 2, second 0
        [1, 1, 1, 0], [1, 1, 1, 1],      # row 0, pair (3, 1): S = {2, 0}, first 3, second 1
        [0, 1, 1, 1], [1, 1, 1, 1],      # row 1, pair (0, 2): S = {1, 3}, first 0, second 2
        [0, 0, 0, 1], [0, 1, 0, 1],      # row 1, pair (3, 1): S = {}, first 1, second 3
    ]
    # the order within a pair changes nothing
    assert torch.equal(M.interaction_coalitions(perm, [(2, 0), (1, 3)]), got)


def _table(n, seed):
    """A synthetic fp32 value for every subset (bit u of the index: unit u present)."""
    return np.random.default_rng(seed).random(1 << n).astype(np.float32)


def _values(v, perm, pairs):
    """The call's value layout from a subset table: v(empty), v(all), the chains, then x1, x2 per permutation and pair."""
    n = perm.shape[1]
    full = (1 << n) - 1
    out = [v[0], v[full]]
    for p in perm:
        s = 0
        for j in range(n - 1):
            s |= 1 << int(p[j])
            out.append(v[s])
    for row in M.interaction_coalitions(torch.from_numpy(perm), pairs).int().numpy():
        out.append(v[int(sum(int(b) << u for u, b in enumerate(row)))])
    return np.float32(out)


def _exact(v, n, a, b):
    """The Shapley-Taylor index of {a, b} from its subset formula: weight 2 t! (n - 1 - t)! / n! for |T| = t."""
    total = 0.0
    v = v.astype(np.float64)
    for T in range(1 << n):
        if T >> a & 1 or T >> b & 1:
            continue
        t = bin(T).count("1")
        d = v[T | 1 << a | 1 << b] - v[T | 1 << a] - v[T | 1 << b] + v[T]
        total += 2 * math.factorial(t) * math.factorial(n - 1 - t) / math.factorial(n) * d
    return total


def test_reference_is_exact_with_every_permutation_and_efficient():
    n = 5
    v = _table(n, 0)
    perm = np.array(list(itertools.permutations(range(n))), dtype=np.int64)
    pairs = np.array(list(itertools.combinations(range(n), 2)), dtype=np.int64)
    vals = _values(v, perm, pairs)
    assert len(vals) == 2 + len(perm) * (n - 1) + 2 * len(perm) * len(pairs)
    inter, se = M.interaction_reference(vals, perm, pairs, 1, dtype=np.float64)
    exact = np.array([_exact(v, n, a, b) for a, b in pairs])
    assert np.abs(inter - exact).max() <= 1e-12
    # efficiency: the singletons' first differences and every pair's index add up to v(N) - v(empty)
    v64 = v.astype(np.float64)
    total = sum(v64[1 << i] - v64[0] for i in range(n)) + inter.sum()
    assert abs(total - (v64[-1] - v64[0])) <= 1e-12
    assert se.shape == (len(pairs),) and np.isfinite(se).all()
    # the prefix is a valid Shapley input at the same offset
    phi, _ = M.shapley_reference(vals[:2 + len(perm) * (n - 1)], perm, 1, dtype=np.float64)
    assert abs(phi.sum() - (v64[-1] - v64[0])) <= 1e-12
    # (a, b) and (b, a): the same bits
    swapped = pairs[:, ::-1].copy()
    assert np.array_equal(M.interaction_reference(_values(v, perm, swapped), perm, swapped, 1)[0],
                          M.interaction_reference(vals, perm, pairs, 1)[0])


def test_reference_groups_and_dummy():
    rng = np.random.default_rng(1)
    n, P = 6, 6
    v = _table(n, 2)
    perm = np.stack([rng.permutation(n) for _ in range(P)])
    pairs = np.array([(0, 3), (5, 1), (2, 4)])
    vals = _values(v, perm, pairs)
    for g in (1, 2):
        inter, se = M.interaction_reference(vals, perm, pairs, g)
        # the header's arithmetic, restated with numpy reductions: the same values up to summation order
        x = vals[2 + P * (n - 1):].astype(np.float64).reshape(P, len(pairs), 2)
        c = np.concatenate([np.full((P, 1), vals[0]), vals[2:2 + P * (n - 1)].reshape(P, n - 1), np.full((P, 1), vals[1])], 1)
        rank = np.argsort(perm, 1)
        d = np.empty((P, len(pairs)))
        for p in range(P):
            for q, (a, b) in enumerate(pairs):
                r = min(rank[p, a], rank[p, b])
                d[p, q] = x[p, q, 1] - c[p, r + 1] - x[p, q, 0] + c[p, r]
        assert np.allclose(inter, d.mean(0), atol=1e-7)
        gm = d.reshape(P // g, g, -1).mean(1)
        assert np.allclose(se, gm.std(0, ddof=1) / math.sqrt(P // g), atol=1e-7)
    assert np.isnan(M.interaction_reference(_values(v, perm[:2], pairs), perm[:2], pairs, 2)[1]).all()
    # unit 0 changes no value: every pair with it is exactly 0, and so is its standard error
    dummy = v.copy()
    for s in range(1 << n):
        dummy[s] = dummy[s & ~1]
    inter, se = M.interaction_reference(_values(dummy, perm, pairs), perm, pairs, 2)
    assert inter[0] == 0.0 and se[0] == 0.0


@pytest.mark.parametrize("pairs, n_units, match", [
    ([[(0, 0)]], [3], "message 0 pair 0 pairs unit 0 with itself"),
    ([[(0, 1), (1, 3)]], [3], "message 0 pair 1 \\(1, 3\\) has a unit outside \\[0, 3\\)"),
    ([[(-1, 1)]], [3], "outside"),
    ([[]], [3], "message 0 has no pairs"),
    ([[(0, 1)], "cross"], [3, 3], "message 1 has no pairs"),
    ([[(0, 1)], "all"], [3, 3], "a list of \\(a, b\\) or \"cross\""),
    ([[(0, 1)]], [1], "message 0 has 1 unit"),
    ([[(0, 1)]], [3, 3], "one entry per message"),
    ([[(0, 1)] * 40000, [(1, 2)] * 30000], [3, 3], "messages 0..1 have 70000 pairs, above 65536"),
])
def test_pair_errors(pairs, n_units, match):
    units = [[((1 + u,), ()) for u in range(n)] for n in n_units]
    with pytest.raises(ValueError, match=match):
        M.interaction_pairs(pairs, units)


def test_pairs_resolve():
    units = [((1,), ()), ((2,), ()), ((), (0,))]
    got = M.interaction_pairs(["cross", [(2, 0), (1, 2)]], [units, units])
    assert [g.dtype for g in got] == [np.int32, np.int32]
    assert got[0].tolist() == [[0, 2], [1, 2]] and got[1].tolist() == [[2, 0], [1, 2]]


@pytest.fixture(scope="module")
def cpu_model(tiny_oracle):
    cfg = vb.BertConfig.from_dict(tiny_oracle.config.to_dict())
    return vb.VILBertForVLTasks.from_pretrained(tiny_oracle.state_dict(), config=cfg, num_labels=200).eval()


@pytest.mark.parametrize("messages, pairs, match", [
    ([("vqa", 0, 1)], [[(0, 0)]], "pairs unit 0 with itself"),
    ([("vqa", 0, 1)], [[(0, 9)]], "outside \\[0, 9\\)"),
    ([("grounding", 0, 1)], ["cross"], "grounding message"),
    ([("vqa", 0, 1), ("vqa", 0, 1)], ["cross"], "one entry per message"),
])
def test_message_and_pair_errors_need_no_engine(cpu_model, messages, pairs, match, monkeypatch):
    def no_library():
        raise AssertionError("reached the library")
    monkeypatch.setattr(L, "load", no_library)
    F = cpu_model.config.v_feature_size
    args = (torch.ones(7, dtype=torch.int64), None, None, torch.zeros(4, F), torch.zeros(4, 4), torch.ones(1, 2), [7], [4])
    with pytest.raises(ValueError, match=match):
        cpu_model.shapley_interactions(*args, messages, pairs)


def _samples(calls, base):
    """Forward samples of the calls: each piece runs its full input and its coalitions, every variant ``base`` samples."""
    return sum(base * (1 + c1 - c0) for call in calls for _, (c0, c1) in call)


def test_calls_split_where_the_pair_coalitions_cross_the_cap():
    # one VQA message at the default units of 37 tokens and 100 boxes: n = 135, P = 8, Q = 128
    n, P, Q = 135, 8, 128
    chain, extra = 1 + P * (n - 1), 2 * P * Q
    recs = [(0, 0, -1, 1)] + [(0, 4, c, 1) for c in range(chain + extra)]
    calls = M.coalition_calls(recs)
    assert [piece for call in calls for piece in call] == [(0, (0, 1023)), (0, (1023, 2046)), (0, (2046, 3069)), (0, (3069, 3121))]
    assert _samples(calls, 1) == 2 + P * (n - 1) + 2 * P * Q + 3 == 3125
    assert _samples(M.coalition_calls(recs[:1 + chain]), 1) == 2 + P * (n - 1) + 1 == 1075
    # an NLVR2 message (2 samples per variant) after it: every call within the cap, every coalition once, in order
    recs += [(1, 0, -1, 2)] + [(1, 4, c, 2) for c in range(1 + 4 * 9 + 2 * 4 * 20)]
    calls = M.coalition_calls(recs)
    base = {0: 1, 1: 2}
    for call in calls:
        assert sum(base[m] * (1 + c1 - c0) for m, (c0, c1) in call) <= L.ABLATION_MAX_VARIANTS
    for m, total in ((0, chain + extra), (1, 1 + 4 * 9 + 2 * 4 * 20)):
        spans = [s for call in calls for mm, s in call if mm == m]
        assert spans[0][0] == 0 and spans[-1][1] == total and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
