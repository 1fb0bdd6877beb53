"""Head ablation without a GPU: the C struct against the header, the engine messages built from Python's, the split of a layout at
the engine's sample cap at entry boundaries, and argument errors raised before any engine is needed."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6


def test_header_declares_and_library_exports_head_ablation():
    hdr = open(HEADER).read()
    for fn in ("vb200_head_ablation_layout", "vb200_head_ablation"):
        assert fn in set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
        assert fn in L.EXPORTS and hasattr(L.load(), fn)


def test_message_struct_matches_the_c_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    c, name = L.HeadAblationMessage, "vb200_head_ablation_message"
    body = f'  printf("%zu' + " %zu" * len(c._fields_) + '\\n", sizeof(' + name + ")" + \
        "".join(f", offsetof({name}, {f})" for f, _ in c._fields_) + ");\n"
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [C.sizeof(c)] + [getattr(c, f).offset for f, _ in c._fields_] == [24, 0, 4, 8, 12, 16, 20]


def test_messages_defaults_and_rules():
    assert M.head_messages([("vqa", 0, 1), ("12", 1, 2, 3, (2, 5)), (RET, 3, 4, None, [0, 0])], 7, 30) == \
        [(VQA, 0, 1, -1, 0, 30), (NLVR2, 1, 2, 3, 2, 5), (RET, 3, 4, -1, 0, 0)]
    bad = [((VQA, 0, 2), "n_images"), ((NLVR2, 0, 1), "n_images"), ((RET, 5, 3), "outside the batch"), ((VQA, 0, 1, -2), "answer"),
           ((VQA, 0, 1, None, (3, 2)), "entry range"), ((VQA, 0, 1, None, (0, 31)), "entry range"), ((VQA, 0), "fields"),
           (("x", 0, 1), "unknown family")]
    for msg, needle in bad:
        with pytest.raises(ValueError, match=needle):
            M.head_messages([msg], 7, 30)


def _records(msgs, heads, K):
    """The layout records vb200_head_ablation_layout writes for messages (index, entry range) with per-entry heads and K samples."""
    H = max(heads)
    out = []
    for m, (eb, ee) in msgs:
        out.append((m, 0, -1, K[m]))
        out += [(m, 3, e * H + h, K[m]) for e in range(eb, ee) for h in range(heads[e])]
    return out


# T0..T5, C0 (two directions), then five times T, V, C (two directions), then V5 and T11
HEADS_12_6_6 = [12] * 6 + [8, 8] + [12, 8, 8, 8] * 5 + [8, 12]


def test_every_head_counts():
    """One message over every head of 12/6/6: 1 + 288 variants, 289 samples (578 for NLVR2); three single-image messages fit a call."""
    assert len(HEADS_12_6_6) == 30 and sum(HEADS_12_6_6) == 288
    recs = _records([(0, (0, 30)), (1, (0, 30)), (2, (0, 30))], HEADS_12_6_6, [1, 1, 1])
    assert len(recs) == 3 * 289
    assert M.head_calls(recs, 12) == [[(0, (0, 30)), (1, (0, 30)), (2, (0, 30))]]
    nlvr2 = _records([(0, (0, 30))], HEADS_12_6_6, [2])
    assert sum(r[3] for r in nlvr2) == 578 and M.head_calls(nlvr2, 12) == [[(0, (0, 30))]]


def test_splitter_cuts_at_entry_boundaries():
    """A retrieval message of K = 4 over every head (1,156 samples) splits into pieces of whole entries, each with its own
    unablated variant; every piece stays within the cap and together they cover every entry once."""
    recs = _records([(0, (0, 30)), (1, (4, 6))], HEADS_12_6_6, [4, 1])
    calls = M.head_calls(recs, 12)
    pieces = [p for c in calls for p in c]
    covered = [e for m, (b, e_) in pieces if m == 0 for e in range(b, e_)]
    assert covered == list(range(30))
    for c in calls:
        assert sum(4 * (1 + sum(HEADS_12_6_6[b:e])) if m == 0 else 1 + sum(HEADS_12_6_6[b:e]) for m, (b, e) in c) <= L.ABLATION_MAX_VARIANTS
    assert (1, (4, 6)) in pieces
    # an entry whose variants alone exceed the cap cannot run
    with pytest.raises(ValueError, match="too many"):
        M.head_calls(_records([(0, (0, 1))], [12], [100]), 12)


def test_no_engine_raises():
    model = vb.VILBertForVLTasks(vb.BertConfig(), num_labels=10)
    with pytest.raises(vb.VilbertB200Error, match="cuda"):
        model.head_ablation([1], [0], [[1]], [[0.0]], [[0.0, 0, 1, 1]], [[10.0, 10.0]], [1], [1], [(VQA, 0, 1)])
