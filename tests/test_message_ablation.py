"""Message ablation without a GPU: the C structs against the header, the engine messages built from Python's, the split of a layout
at the engine's sample cap, argument errors raised before any engine is needed, and the worker's spans as messages."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import model as M
from vilbert_b200 import worker_api as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")
VQA, GQA, NLVR2, SNLI, RET, GRD = 1, 2, 3, 4, 5, 6


def test_header_declares_and_library_exports_message_ablation():
    hdr = open(HEADER).read()
    for fn in ("vb200_message_ablation_layout", "vb200_message_ablation"):
        assert fn in set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
        assert fn in L.EXPORTS and hasattr(L.load(), fn)


def test_message_structs_match_the_c_layout(tmp_path):
    """sizeof / offsetof of vb200_ablation_message and vb200_ablation_variant as a C compiler lays them out, against ctypes."""
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    structs = {"vb200_ablation_message": L.AblationMessage, "vb200_ablation_variant": L.AblationVariant}
    body = "".join(f'  printf("%zu' + " %zu" * len(c._fields_) + '\\n", sizeof(' + name + ")"
                   + "".join(f", offsetof({name}, {f})" for f, _ in c._fields_) + ");\n" for name, c in structs.items())
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    for line, c in zip(lines, structs.values()):
        assert [int(x) for x in line.split()] == [C.sizeof(c)] + [getattr(c, f).offset for f, _ in c._fields_]
    assert C.sizeof(L.AblationVariant) == 32


def test_families_by_name_task_id_or_value():
    assert [M.message_family(f) for f in ("vqa", "nlvr2", "retrieval", "grounding", "12", "7", "16", "15", 4)] == \
        [VQA, NLVR2, RET, GRD, NLVR2, RET, GRD, GQA, SNLI]
    with pytest.raises(ValueError, match="unknown family"):
        M.message_family("3")


def test_pieces_defaults_and_explicit_ranges():
    nt, nb = [5, 6, 6, 6, 9, 4], [3, 4, 1, 6, 8, 2]
    got = M.message_pieces([("vqa", 0, 1), ("7", 1, 3, 2, (0, 3)), (GRD, 4, 1, None, None, (2, 5)), (NLVR2, 4, 2, 1)], nt, nb)
    assert got == [((VQA, 0, 1, -1, 1, 4, 0, 3), 0),
                   ((RET, 1, 3, 2, 0, 3, 0, 4), 1), ((RET, 1, 3, 2, 0, 0, 5, 11), 1),     # the one-box image splits the boxes
                   ((GRD, 4, 1, -1, 1, 8, 2, 5), 2),
                   ((NLVR2, 4, 2, 1, 1, 8, 0, 10), 3)]
    # a one-box image alone: no box run, one piece
    assert M.message_pieces([(VQA, 2, 1)], nt, nb) == [((VQA, 2, 1, -1, 1, 5, 0, 0), 0)]


@pytest.mark.parametrize("msg, match", [
    (("vqa", 0, 2), "n_images 2"),
    (("12", 0, 1), "n_images 1"),
    (("7", 0, 0), "n_images 0"),
    (("7", 4, 3), "outside the batch"),
    (("vqa", -1, 1), "outside the batch"),
    (("vqa", 0, 1, -2), "answer -2"),
    (("vqa", 0, 1, None, (3, 2)), "token range"),
    (("vqa", 0, 1, None, (0, 6)), "token range"),
    (("7", 1, 3, None, None, (0, 12)), "box range"),
    (("7", 1, 3, None, None, (3, 5)), "drops a box of its image 1"),
    (("bogus", 0, 1), "unknown family"),
    (("vqa", 0, 1, None, None, None, 7), "fields"),
])
def test_python_argument_errors_need_no_engine(msg, match):
    with pytest.raises(ValueError, match=match):
        M.message_pieces([msg], [5, 6, 6, 6, 9], [3, 4, 1, 6, 8])


def test_message_ablation_errors_before_the_engine():
    m = vb.VILBertForVLTasks.__new__(vb.VILBertForVLTasks)
    with pytest.raises(ValueError, match="same, positive length"):
        m.message_ablation(None, None, None, None, None, None, [3, 4], [2], [("vqa", 0, 1)])
    with pytest.raises(ValueError, match="no messages"):
        m.message_ablation(None, None, None, None, None, None, [3], [2], [])
    with pytest.raises(ValueError, match="n_images"):
        m.message_ablation(None, None, None, None, None, None, [3], [2], [("12", 0, 1)])


def _recs(spec):
    """Layout records from (message, base samples, [(kind, samples)...])."""
    out = []
    for m, base, units in spec:
        out.append((m, 0, -1, base))
        count = {1: 0, 2: 0}
        for kind, s in units:
            out.append((m, kind, count[kind], s))
            count[kind] += 1
    return out


def test_split_keeps_messages_whole_where_they_fit():
    recs = _recs([(0, 2, [(1, 2)] * 3 + [(2, 2)] * 2), (1, 1, [(1, 1)] * 4), (2, 3, [(1, 3), (2, 1)])])
    # 12, 5, 7 samples
    assert M.message_calls(recs, cap=17) == [[(0, (0, 3, 0, 2)), (1, (0, 4, 0, 0))], [(2, (0, 1, 0, 1))]]
    assert M.message_calls(recs, cap=24) == [[(0, (0, 3, 0, 2)), (1, (0, 4, 0, 0)), (2, (0, 1, 0, 1))]]


def test_split_an_oversized_message_into_pieces():
    """Each piece repeats the unablated variant's samples; units stay in order, tokens then boxes, and no call passes the cap."""
    recs = _recs([(0, 3, [(1, 3)] * 5 + [(2, 1)] * 7), (1, 1, [(2, 1)] * 2)])     # 3 + 15 + 7 = 25 samples
    calls = M.message_calls(recs, cap=10)
    assert calls == [[(0, (0, 2, 0, 0))], [(0, (2, 4, 0, 0))], [(0, (4, 5, 0, 4))], [(0, (0, 0, 4, 7)), (1, (0, 0, 0, 2))]]
    for call in calls:
        n = 0
        for m, (tb, te, bb, be) in call:
            base = 3 if m == 0 else 1
            n += base + (te - tb) * (3 if m == 0 else 1) + (be - bb)
        assert n <= 10
    with pytest.raises(ValueError, match="too many"):
        M.message_calls(_recs([(0, 6, [(1, 6)])]), cap=10)


def test_split_at_the_engine_cap():
    """A 10-image retrieval message at 37 tokens and 100 boxes per image: 10 + 35 * 10 + 1000 = 1360 samples, two calls."""
    recs = _recs([(0, 10, [(1, 10)] * 35 + [(2, 1)] * 1000)])
    calls = M.message_calls(recs)
    assert calls == [[(0, (0, 35, 0, 664))], [(0, (0, 0, 664, 1000))]]
    assert 10 + 350 + 664 == L.ABLATION_MAX_VARIANTS


def test_worker_spans_map_to_messages():
    reqs = [("q", [1], None, [{}], "1"), ("q", [12], None, [{}, {}], "12"), ("q", [7], None, [{}] * 4, "7"),
            ("q", [11], None, [{}], "11")]
    spans = {0: (0, 1), 1: (2, 4), 2: (4, 8), 3: (8, 9)}           # request 1: a filler row in front of the pair
    msgs = W.ablation_messages(reqs, spans, tokens=(1, 3))
    assert msgs == {0: ("1", 0, 1, None, (1, 3), None), 1: ("12", 2, 2, None, (1, 3), None), 2: ("7", 4, 4, None, (1, 3), None),
                    3: ("11", 8, 1, None, (1, 3), None)}
    nt, nb = [5] * 9, [3, 1, 2, 2, 4, 1, 3, 3, 6]
    pieces = M.message_pieces(list(msgs.values()), nt, nb)
    assert [p for p, _ in pieces] == [(VQA, 0, 1, -1, 1, 3, 0, 3), (NLVR2, 2, 2, -1, 1, 3, 0, 4), (RET, 4, 4, -1, 1, 3, 0, 4),
                                      (RET, 4, 4, -1, 0, 0, 5, 11), (GRD, 8, 1, -1, 1, 3, 0, 6)]
    assert W._pixel_box({"image_width": 640, "image_height": 480, "bbox": [[1, 2, 3, 4], [5, 6, 7, 8]]}, 2) == [5.0, 6.0, 7.0, 8.0]
    assert W._pixel_box({"image_width": 640, "image_height": 480}, 0) == [0.0, 0.0, 640.0, 480.0]
