"""CPU checks of the region-selection oracle (oracle/detections_ref.py) against an independent per-class formulation on
torchvision's NMS, its tie and threshold edge cases, and the C layout of the vb200_select_regions structs."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import detections_ref as D
from vilbert_b200 import _lib as L
from vilbert_b200 import synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _integer_heads(n, C, seed, scale=2.0):
    """Integer pixel boxes (so the legacy +1 IoU is exact after a +1 shift) in clusters, distinct random logits."""
    g = torch.Generator().manual_seed(seed)
    centre = torch.randint(40, 200, (4, 2), generator=g)[torch.randint(0, 4, (n,), generator=g)]
    half = torch.randint(5, 40, (n, 2), generator=g)
    x1y1 = (centre - half + torch.randint(-6, 7, (n, 2), generator=g)).clamp(min=0)
    x2y2 = x1y1 + 2 * half
    proposals = (torch.cat([x1y1, x2y2], dim=1) * 2).float()        # even coordinates: / 2.0 is exact
    scores = torch.randn(n, C, generator=g) * 3
    feats = torch.relu(torch.randn(n, 8, generator=g))
    return proposals, scores, feats, scale


def _torchvision_select(proposals, scores, scale, K, conf_thresh, background, iou=0.5):
    tv = pytest.importorskip("torchvision")
    p = torch.softmax(scores, -1)
    dets = proposals / scale
    shifted = dets.clone()
    shifted[:, 2:] += 1                       # torchvision: w = x2 - x1; legacy: w = x2 - x1 + 1
    start = 0 if background else 1
    max_conf = torch.zeros(p.shape[0])
    for c in range(start, p.shape[1]):
        keep = tv.ops.nms(shifted, p[:, c], iou)
        s = p[keep, c]
        max_conf[keep] = torch.where((s > max_conf[keep]) & (s > conf_thresh), s, max_conf[keep])
    srt, idx = torch.sort(max_conf, descending=True, stable=True)
    keep = idx[:K]
    return dict(keep=keep.numpy(), max_conf=srt[:K].numpy(), num_boxes=int((srt[:K] != 0).sum()), bbox=dets[keep].numpy(),
                objects=torch.argmax(p[keep][start:], dim=1).numpy())


@pytest.mark.parametrize("n,C,K,thr,background,seed", [(60, 31, 20, 0.0, False, 1), (90, 17, 100, 0.0, True, 2),
                                                       (75, 40, 30, 0.2, False, 3), (1, 5, 10, 0.0, False, 4)])
def test_oracle_matches_torchvision_formulation(n, C, K, thr, background, seed):
    prop, sc, ft, scale = _integer_heads(n, C, seed)
    ref = _torchvision_select(prop, sc, scale, K, thr, background)
    got = D.select_image(prop, sc, ft, scale, K, thr, background)
    np.testing.assert_array_equal(got["keep"], ref["keep"])
    np.testing.assert_array_equal(got["max_conf"], ref["max_conf"])
    assert got["num_boxes"] == ref["num_boxes"]
    np.testing.assert_array_equal(got["bbox"], ref["bbox"])
    np.testing.assert_array_equal(got["objects"], ref["objects"])
    np.testing.assert_array_equal(got["features"], ft.numpy()[ref["keep"]])


def test_fewer_proposals_than_max_boxes():
    prop, sc, ft, scale = _integer_heads(7, 9, 5)
    r = D.select_image(prop, sc, ft, scale, max_boxes=100)
    assert r["keep"].shape == (7,) and r["features"].shape == (7, 8) and r["cls_prob"].shape == (7, 9)
    assert sorted(r["keep"].tolist()) == list(range(7))
    assert r["objects"].shape == (6,)              # the reference's row slice: k - start entries


def test_threshold_leaves_zeros_ranked_by_index():
    prop, sc, ft, scale = _integer_heads(40, 12, 6)
    r = D.select_image(prop, sc, ft, scale, max_boxes=30, conf_thresh=0.9)
    nz = r["num_boxes"]
    assert nz < 30
    assert (r["max_conf"][:nz] > 0.9).all() and (r["max_conf"][nz:] == 0).all()
    zeros = r["keep"][nz:]
    assert zeros.tolist() == sorted(zeros.tolist())
    assert zeros.tolist() == [i for i in range(40) if r["max_conf_all"][i] == 0][:len(zeros)]


def test_background_takes_part_and_keeps_every_object_row():
    prop, sc, ft, scale = _integer_heads(30, 6, 7)
    sc[:, 0] += 30.0                               # background dominates every row
    fg = D.select_image(prop, sc, ft, scale, max_boxes=10)
    bg = D.select_image(prop, sc, ft, scale, max_boxes=10, background=True)
    assert fg["objects"].shape == (9,) and bg["objects"].shape == (10,)
    assert (bg["objects"] == 0).all() and (fg["objects"] == 0).all()    # argmax over every column, background included
    assert bg["max_conf"][0] > 0.9 > fg["max_conf"][0]


def _two_box_heads(second):
    proposals = torch.tensor([[0.0, 0.0, 9.0, 9.0], second])
    scores = torch.tensor([[0.0, 2.0, 0.0], [0.0, 1.0, 0.0]])
    return proposals, scores, torch.eye(2, 4), 1.0


def test_iou_equal_to_threshold_is_not_suppressed():
    # legacy IoU of [0,0,9,9] and [0,0,9,4]: inter 10 * 5 = 50, areas 100 and 50 -> 50 / 100 = 0.5 exactly
    assert D.iou_matrix(np.array([[0, 0, 9, 9], [0, 0, 9, 4]], np.float32))[0, 1] == np.float32(0.5)
    at = D.select_image(*_two_box_heads([0.0, 0.0, 9.0, 4.0]), max_boxes=2)
    assert at["max_conf_all"][1] > 0                  # kept by class 1: IoU 0.5 is not > 0.5
    above = D.select_image(*_two_box_heads([0.0, 0.0, 9.0, 5.0]), max_boxes=2)   # IoU 0.6
    np.testing.assert_array_equal(above["max_conf_all"][1] > 0, True)    # class 2 (scores equal) still keeps it first...
    assert above["max_conf_all"][1] < at["max_conf_all"][1]             # ...but class 1's higher score is suppressed


def test_duplicate_boxes_with_equal_scores_keep_the_lower_index():
    proposals = torch.tensor([[10.0, 10.0, 50.0, 50.0]] * 3)
    scores = torch.tensor([[0.0, 3.0, 1.0]] * 3)
    r = D.select_image(proposals, scores, torch.arange(12.0).view(3, 4), 1.0, max_boxes=3)
    assert r["keep"].tolist() == [0, 1, 2]
    assert r["max_conf_all"][0] > 0 and (r["max_conf_all"][1:] == 0).all()
    assert r["num_boxes"] == 1


def test_synthetic_margin_heads_sum_to_one_exactly():
    (prop, sc, ft, scale), = synthetic.synthetic_detections(1, 50, n_classes=1601, feature_size=16, seed=3, margin=0.05)
    e = np.exp(sc.double().numpy())
    assert (e.sum(1) - 1.0 < 2.0 ** -26).all()        # below half an ulp of 1.0f: fp32 sums are exactly 1
    assert (prop[:, 2:] > prop[:, :2]).all() and ft.min() >= 0


def test_select_structs_match_the_c_layout(tmp_path):
    assert (C.sizeof(L.Detections), C.sizeof(L.SelectParams), C.sizeof(L.Selected)) == (40, 28, 56)
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(vb200_detections), offsetof(vb200_detections, im_scale),'
                   ' offsetof(vb200_detections, proposals), offsetof(vb200_detections, features));\n'
                   '  printf("%zu %zu %zu\\n", sizeof(vb200_select_params), offsetof(vb200_select_params, conf_thresh),'
                   ' offsetof(vb200_select_params, out_rows));\n'
                   '  printf("%zu %zu\\n", sizeof(vb200_selected), offsetof(vb200_selected, objects));\n  return 0;\n}\n')
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [int(x) for x in lines[0].split()] == [C.sizeof(L.Detections), L.Detections.im_scale.offset,
                                                  L.Detections.proposals.offset, L.Detections.features.offset]
    assert [int(x) for x in lines[1].split()] == [C.sizeof(L.SelectParams), L.SelectParams.conf_thresh.offset,
                                                  L.SelectParams.out_rows.offset]
    assert [int(x) for x in lines[2].split()] == [C.sizeof(L.Selected), L.Selected.objects.offset]
