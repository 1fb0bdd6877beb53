"""Packed detector-output batches on CPU: worker_api.pack_region_requests / _split_outputs / custom_prediction_packed and
MicroBatchWorker(packed=True) with a stub in place of the engine, plus the C ABI surface of vb200_forward_regions_packed
(vb200_packed_region_inputs layout, export, NULL handle).  The engine call itself is covered by tests/test_gpu_regions_packed.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from vilbert_b200 import _lib as L
from vilbert_b200 import worker_api as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "a", "dog", "on", "grass"])}
TOK = W.WordpieceTokenizer(VOCAB)


def _det(n_boxes, F=8, seed=0, wh=(640, 480)):
    """Detector output for images with the given box counts: box features [n, F] and infos with pixel boxes."""
    g = torch.Generator().manual_seed(seed)
    feats, infos = [], []
    for n in n_boxes:
        feats.append(torch.rand(n, F, generator=g))
        xy = torch.rand(n, 2, generator=g) * 300
        infos.append({"image_width": wh[0], "image_height": wh[1],
                      "bbox": torch.cat([xy, xy + 20 + torch.rand(n, 2, generator=g) * 100], 1).numpy().astype(np.float32)})
    return feats, infos


class StubRegionModel:
    """forward_regions_packed with the engine's output layout (per-image outputs [B, ...], per-row outputs and spatials packed over
    sum V_i / sum T_i rows).  Every output row carries its row index, so a split that picks the wrong rows is visible."""
    _device = 0

    def __init__(self):
        self.calls = []

    def forward_regions_packed(self, question, segment_ids, task_tokens, box_features, boxes, image_wh, n_tokens, n_boxes, select=None,
                               max_tokens=0, max_boxes=0):
        self.calls.append(dict(question=question.clone(), segment_ids=segment_ids.clone(), task=task_tokens.clone(),
                               box_features=box_features.clone(), boxes=boxes.clone(), image_wh=image_wh.clone(),
                               n_tokens=list(n_tokens), n_boxes=list(n_boxes), select=select, max_tokens=max_tokens, max_boxes=max_boxes))
        B, rv, rt = len(n_tokens), sum(n_boxes) + len(n_boxes), sum(n_tokens) + len(n_tokens)
        idx = lambda n, w: (torch.arange(n, dtype=torch.float32)[:, None] * 0.01 + torch.arange(w, dtype=torch.float32)[None] * 1e-4)
        sp = torch.rand(rv, 5, generator=torch.Generator().manual_seed(rv))
        return (idx(B, 3129), idx(B, 1533), idx(B, 1), idx(B // 2, 2) if B % 2 == 0 else idx(B, 2), idx(B, 3), None, idx(rv, 1), None,
                idx(rt, 1), []), sp


@pytest.fixture(autouse=True)
def _tokenizer():
    W.tokenizer = TOK
    W.label_maps.update(vqa=None, gqa=None)
    yield
    W.tokenizer = None


def test_real_tokens_strip_the_padding():
    toks, segs = W.real_tokens("what is the man holding?")
    assert toks == [2, 4, 5, 6, 7, 8, 9, 10, 3] and segs == [0] * 9
    full, mask, _ = W.tokenize_query("what is the man holding?")
    assert len(full) == W.MAX_LENGTH and toks == full[:sum(mask)]
    long_q = " ".join(["what"] * 50)
    assert len(W.real_tokens(long_q)[0]) == 52                      # never truncated, like tokenize_query


def test_packing_expands_text_per_image_and_keeps_box_counts():
    f1, i1 = _det([5], seed=1)
    f7, i7 = _det([4, 9, 3], seed=2)
    p = W.pack_region_requests([("what is the man holding?", [1], f1, i1, "1"), ("a dog", [7], f7, i7, "7")], bucket=8)
    # VQA: 9 tokens, 5 boxes; retrieval: "[CLS] a dog [SEP]" repeated per image, each image its own box count; fillers 1 / 1
    assert p["n_tokens"] == [9, 4, 4, 4, 1, 1, 1, 1]
    assert p["n_boxes"] == [5, 4, 9, 3, 1, 1, 1, 1]
    assert p["spans"] == {0: (0, 1), 1: (1, 4)}
    q = p["question"]
    assert q.numel() == sum(p["n_tokens"]) and p["segment_ids"].numel() == q.numel()
    assert q[:9].tolist() == [2, 4, 5, 6, 7, 8, 9, 10, 3]
    assert q[9:13].tolist() == q[13:17].tolist() == q[17:21].tolist() == [2, 13, 14, 3]
    assert q[21:].tolist() == [0, 0, 0, 0]
    assert p["task_tokens"].view(-1).tolist() == [1, 7, 7, 7, 0, 0, 0, 0]
    bf, bx = p["box_features"], p["boxes"]
    assert bf.shape == (sum(p["n_boxes"]), 8) and bx.shape == (sum(p["n_boxes"]), 4)
    assert torch.equal(bf[:5], f1[0]) and torch.equal(bf[5:9], f7[0]) and torch.equal(bf[9:18], f7[1]) and torch.equal(bf[18:21], f7[2])
    assert torch.equal(bx[9:18], torch.from_numpy(i7[1]["bbox"]))
    assert bool((bf[21:] == 0).all()) and bool((bx[21:] == 0).all())
    assert p["image_wh"].tolist() == [[640, 480]] * 4 + [[1, 1]] * 4
    assert p["max_tokens"] == W.MAX_LENGTH and p["max_boxes"] == 100


def test_capacities_grow_with_the_longest_request():
    f, i = _det([120], seed=3)
    p = W.pack_region_requests([(" ".join(["what"] * 50), [1], f, i, "1")], bucket=1, max_boxes=100)
    assert p["max_tokens"] == 52 and p["max_boxes"] == 120


def test_nlvr2_pairs_on_even_rows_after_an_odd_request():
    f1, i1 = _det([5], seed=1)
    f12, i12 = _det([6, 7], seed=2)
    p = W.pack_region_requests([("what is the man holding?", [1], f1, i1, "1"), ("a dog on the grass", [12], f12, i12, "12")], bucket=1)
    assert p["n_boxes"] == [5, 1, 6, 7]                               # one filler row so that the pair starts on row 2
    assert p["n_tokens"] == [9, 1, 7, 7]
    assert p["spans"][1] == (2, 4)


def test_odd_bucket_made_even_for_the_pair_head():
    f, i = _det([4], seed=1)
    p = W.pack_region_requests([("what", [1], f, i, "1")], bucket=3)
    assert len(p["n_tokens"]) == 4
    p = W.pack_region_requests([("what", [1], f, i, "1")], bucket=3, select=L.OUT_VIL_PREDICTION)
    assert len(p["n_tokens"]) == 3                                    # no pair head: the odd bucket stands


def test_offsets_and_filler_rows_through_custom_prediction_packed():
    W.model = StubRegionModel()
    f1, i1 = _det([5], seed=1)
    f11, i11 = _det([6], seed=2)
    f7, i7 = _det([4, 9, 3], seed=3)
    reqs = [("what is the man holding?", [1], f1, i1, "1"), ("the man", [11], f11, i11, "11"), ("a dog", [7], f7, i7, "7")]
    ans = W.custom_prediction_packed(reqs, bucket=8)
    assert len(W.model.calls) == 1
    c = W.model.calls[0]
    out, sp = StubRegionModel().forward_regions_packed(c["question"], c["segment_ids"], c["task"], c["box_features"], c["boxes"],
                                                        c["image_wh"], c["n_tokens"], c["n_boxes"])
    conf, idx = torch.topk(torch.softmax(out[0][0], dim=0), 3)
    assert ans[0]["top3_answer"] == [f"<vqa:{k}>" for k in idx.tolist()]
    assert ans[0]["top3_confidence"] == pytest.approx(conf.tolist())
    # grounding reads ITS OWN regions: packed rows 6..12 (image 0 has 5 boxes + its global row) of vision_logit and spatials
    v = out[6][6:13].view(-1)
    conf, idx = torch.topk(torch.softmax(v, dim=0), 3)
    assert [a["confidence"] for a in ans[1]] == pytest.approx([x * 100 for x in conf.tolist()])
    assert [a["x1"] for a in ans[1]] == [int(b[0] * 640) for b in sp[6:13][idx][:, :4].tolist()]
    # retrieval: rows 2..4 of vil_logit
    conf, idx = torch.topk(torch.softmax(out[2][2:5].view(-1), dim=0), 3)
    assert ans[2]["top3_answer"] == idx.tolist()
    assert np.allclose(ans[2]["top3_confidence"], conf.tolist())


def test_split_outputs_layout():
    out, sp = StubRegionModel().forward_regions_packed(torch.zeros(12, dtype=torch.long), torch.zeros(12, dtype=torch.long),
                                                       torch.zeros(4, 1, dtype=torch.long), torch.zeros(14, 8), torch.zeros(14, 4),
                                                       torch.ones(4, 2), [3, 2, 2, 5], [1, 4, 6, 3])
    v_off = [0, 2, 7, 14, 18]                                         # boxes [1, 4, 6, 3], each with its global row
    t_off = [0, 4, 7, 10, 16]                                         # tokens [3, 2, 2, 5], each with its task token
    sl, s = W._split_outputs(out, sp, 1, 3, v_off, t_off, "12")
    assert torch.equal(sl[0], out[0][1:3]) and torch.equal(sl[3], out[3][0:1])
    assert torch.equal(sl[6], out[6][2:14]) and torch.equal(sl[8], out[8][4:10]) and torch.equal(s, sp[2:14])
    sl, s = W._split_outputs(out, sp, 3, 4, v_off, t_off, "11")
    assert sl[6].shape == (1, 4, 1) and torch.equal(sl[6][0], out[6][14:18]) and s.shape == (1, 4, 5)
    assert sl[3].numel() == 0


def test_rejections_are_per_request():
    W.model = StubRegionModel()
    f1, i1 = _det([5], seed=1)
    f2, i2 = _det([5, 6], seed=2)
    too_many, tm_i = _det([256], seed=3)
    bad_width, bw_i = _det([4], F=16, seed=4)
    short_bbox = [dict(i1[0], bbox=i1[0]["bbox"][:3])]
    good, good_i = _det([6], seed=5)
    reqs = [("what", [1], f1, i1, "1"),
            ("what", [1], f2, i2, "1"),                   # VQA with two images
            ("what", [1], too_many, tm_i, "1"),           # 256 boxes: V = 257
            ("what", [1], bad_width, bw_i, "1"),          # feature width differs from the batch's
            ("what", [1], f1, short_bbox, "1"),           # fewer boxes than features
            ("what", [99], good, good_i, "99"),           # unknown task
            ("a dog", [13], good, good_i, "13")]
    ans = W.custom_prediction_packed(reqs, bucket=2)
    assert isinstance(ans[0], dict) and isinstance(ans[6], dict)
    assert isinstance(ans[1], AssertionError)
    assert isinstance(ans[2], ValueError) and "255" in str(ans[2])
    assert isinstance(ans[3], ValueError) and "F = 8" in str(ans[3])
    assert isinstance(ans[4], ValueError) and "bbox" in str(ans[4])
    assert isinstance(ans[5], ValueError)
    assert W.model.calls[0]["n_boxes"] == [5, 6]
    assert isinstance(W.custom_prediction_packed([reqs[1]])[0], AssertionError)      # nothing left: no model call
    assert len(W.model.calls) == 1


def test_micro_batch_worker_packed_round_trip_with_stub():
    """MicroBatchWorker(packed=True): raw detector output in, one packed call for every pending message (a retrieval message whose
    images have different box counts included), result dicts out."""
    W.model = StubRegionModel()
    msgs = []
    for k, (task_id, counts, q) in enumerate([("1", [5], "what is the man holding?"), ("7", [4, 9, 3], "a dog"), ("13", [7], "a dog")]):
        feats, infos = _det(counts, seed=10 + k)
        msgs.append(({"image_path": [f"/m/demo/i{j}.jpg" for j in range(len(counts))], "question": q, "socket_id": f"s{k}",
                      "task_id": task_id}, feats, infos))
    worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=300.0, packed=True)
    futs = [worker.submit(*m) for m in msgs]
    res = [f.result(timeout=60) for f in futs]
    worker.close()
    assert len(W.model.calls) == 1 and worker.batches == [5]
    assert W.model.calls[0]["n_boxes"][:5] == [5, 4, 9, 3, 7]
    assert [r["socket_id"] for r in res] == ["s0", "s1", "s2"]
    assert res[1]["result"]["task_id"] == "7" and len(res[1]["result"]["image_name_list"]) == 3
    assert W.MicroBatchWorker.__init__.__defaults__[-1] is False         # dense stays the default


def test_regions_packed_symbol_in_header_and_exports():
    hdr = open(os.path.join(ROOT, "include", "vilbert_b200.h")).read()
    declared = set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    assert "vb200_forward_regions_packed" in declared and "vb200_forward_regions_packed" in L.EXPORTS
    assert "vb200_packed_region_inputs;" in hdr
    assert re.search(r"#define VB200_ABI_VERSION 2\b", hdr)


def test_packed_region_inputs_layout_matches_header(tmp_path):
    """ctypes PackedRegionInputs against the C compiler's view of vb200_packed_region_inputs (size and every field offset, LP64)."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in L.PackedRegionInputs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n'
                   '    printf("%zu", sizeof(vb200_packed_region_inputs));\n'
                   + "".join(f'    printf(" %zu", offsetof(vb200_packed_region_inputs, {f}));\n' for f in fields)
                   + '    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[0] == C.sizeof(L.PackedRegionInputs) == 88
    assert got[1:] == [getattr(L.PackedRegionInputs, f).offset for f in fields]


def test_forward_regions_packed_rejects_null_handle():
    lib = L.load()
    inp = L.PackedRegionInputs()
    assert lib.vb200_forward_regions_packed(None, C.byref(inp), None, L.OUT_TASK_HEADS, 0, None) == -1
