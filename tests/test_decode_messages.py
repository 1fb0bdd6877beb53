"""CPU checks of the answer decode's host side: the descriptors worker_api.decode_messages builds from a batch's spans, the C
declarations of vb200_decode_answers[_host] against the library and the ctypes binding, and the decode="host" | "device" argument."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vilbert_b200 import _lib as L
from vilbert_b200 import worker_api as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "a", "dog"])}


def _info(w=640, h=480):
    return {"image_width": w, "image_height": h}


def test_dense_spans_with_nlvr2_filler_and_retrieval():
    """prediction_batch's layout: VQA on row 0, a filler row 1, the NLVR2 pair on rows 2-3, retrieval over rows 4-8, grounding on
    row 9 of a dense batch with V = 37 regions, SNLI-VE and GQA after it."""
    tasks = {0: ("1", [_info()]), 1: ("12", [_info(), _info()]), 2: ("7", [_info()] * 5), 3: ("4", [_info(500, 375)]),
             4: ("13", [_info()]), 5: ("15", [_info()])}
    spans = {0: (0, 1), 1: (2, 4), 2: (4, 9), 3: (9, 10), 4: (10, 11), 5: (11, 12)}
    V = 37
    got = W.decode_messages(tasks, spans, [k * V for k in range(17)])
    assert got == [(0, ("1", 0, 1, 3, None)), (1, ("12", 1, 1, 2, None)), (2, ("7", 4, 5, 5, None)),
                   (3, ("4", 9 * V, V, 3, (500, 375))), (4, ("13", 10, 1, 3, None)), (5, ("15", 11, 1, 3, None))]


def test_second_nlvr2_pair_and_odd_rows():
    """A pair starting on row 6 reads pair row 3; the message order follows the spans, not the request numbers."""
    tasks = {4: ("12", [_info(), _info()]), 1: ("2", [_info()])}
    got = W.decode_messages(tasks, {4: (6, 8), 1: (5, 6)}, list(range(9)))
    assert got == [(4, ("12", 3, 1, 2, None)), (1, ("2", 5, 1, 3, None))]


def test_packed_grounding_rows_with_mixed_box_counts():
    """custom_prediction_packed's layout: pack_region_requests' spans and box counts -> each grounding image's packed vision rows
    (its global row, then its boxes), whatever the box counts of the rows before it."""
    rng = np.random.default_rng(0)
    tok = W.WordpieceTokenizer(VOCAB)

    def req(task_id, counts, w=640, h=480):
        feats = [rng.random((n, 8), dtype=np.float32) for n in counts]
        infos = [{"image_width": w, "image_height": h, "bbox": rng.random((n, 4), dtype=np.float32) * 100} for n in counts]
        return ("what is the man", [int(task_id)], feats, infos, task_id)

    reqs = [req("11", [7]), req("12", [3, 9]), req("7", [5, 2, 11]), req("4", [100], 333, 517), req("16", [1]), req("1", [40])]
    p = W.pack_region_requests(reqs, bucket=8, tok=tok)
    # rows: 11 -> 0, filler 1, pair 2-3, retrieval 4-6, 4 -> 7, 16 -> 8, 1 -> 9, then fillers to 16
    assert p["spans"] == {0: (0, 1), 1: (2, 4), 2: (4, 7), 3: (7, 8), 4: (8, 9), 5: (9, 10)}
    v_off = np.concatenate([[0], np.cumsum([n + 1 for n in p["n_boxes"]])])
    got = dict(W.decode_messages({i: (r[4], r[3]) for i, r in enumerate(reqs)}, p["spans"], v_off))
    # vision rows per batch row: 8, 2 (filler), 4, 10, 6, 3, 12, 101, 2, 41
    assert got[0] == ("11", 0, 8, 3, (640, 480))
    assert got[1] == ("12", 1, 1, 2, None)
    assert got[2] == ("7", 4, 3, 3, None)
    assert got[3] == ("4", 8 + 2 + 4 + 10 + 6 + 3 + 12, 101, 3, (333, 517))
    assert got[4] == ("16", 8 + 2 + 4 + 10 + 6 + 3 + 12 + 101, 2, 3, (640, 480))
    assert got[5] == ("1", 9, 1, 3, None)


def test_header_declares_and_library_exports_decode():
    hdr = open(HEADER).read()
    declared = set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    lib = L.load()
    for name in ("vb200_decode_answers", "vb200_decode_answers_host"):
        assert name in declared and name in L.EXPORTS and hasattr(lib, name)
    fams = dict(re.findall(r"VB200_DECODE_([A-Z_0-9]+) = (\d+)", hdr))
    assert {k: int(v) for k, v in fams.items()} == {"VQA": L.DECODE_VQA, "GQA": L.DECODE_GQA, "NLVR2": L.DECODE_NLVR2,
                                                    "SNLI_VE": L.DECODE_SNLI_VE, "RETRIEVAL": L.DECODE_RETRIEVAL,
                                                    "GROUNDING": L.DECODE_GROUNDING}
    assert re.search(r"#define VB200_DECODE_MAX_TOP (\d+)", hdr).group(1) == str(L.DECODE_MAX_TOP)


def test_decode_structs_match_the_c_layout(tmp_path):
    """sizeof / offsetof of vb200_decode_msg and vb200_answer as a C compiler lays them out from the header, against ctypes."""
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(vb200_decode_msg), offsetof(vb200_decode_msg, top_n),'
                   ' offsetof(vb200_decode_msg, image_w), offsetof(vb200_decode_msg, image_h));\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(vb200_answer), offsetof(vb200_answer, index), offsetof(vb200_answer, prob),'
                   ' offsetof(vb200_answer, box));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    msg = [int(x) for x in lines[0].split()]
    ans = [int(x) for x in lines[1].split()]
    assert msg == [C.sizeof(L.DecodeMsg), L.DecodeMsg.top_n.offset, L.DecodeMsg.image_w.offset, L.DecodeMsg.image_h.offset]
    assert ans == [C.sizeof(L.Answer), L.Answer.index.offset, L.Answer.prob.offset, L.Answer.box.offset]
    assert C.sizeof(L.Answer) == 4 + 10 * 4 + 10 * 4 + 10 * 16


def test_task_families_cover_every_task():
    assert set(L.TASK_DECODE_FAMILY) == set(W.TASK_OUTPUT)
    assert all(L.TASK_DECODE_FAMILY[t] == L.DECODE_GROUNDING for t in W.GROUNDING_TASKS)


def test_decode_mode_is_checked_before_any_work():
    with pytest.raises(ValueError, match="decode must be"):
        W.prediction_batch([], decode="gpu")
    with pytest.raises(ValueError, match="decode must be"):
        W.prediction_packed([], decode="cuda")
    with pytest.raises(ValueError, match="decode must be"):
        W.custom_prediction_packed([], decode=None)
    with pytest.raises(ValueError, match="decode must be"):
        W.MicroBatchWorker(decode="both")
    assert W.prediction_batch([]) == [] and W.prediction_batch([], decode="device") == []
