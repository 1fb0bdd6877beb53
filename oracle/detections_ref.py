"""CPU restatement of the detector's feature extraction step (the reference worker's `_process_feature_extraction`,
worker.py:123-176): the per-image region selection that `vb200_select_regions` runs on the device.

For image i with proposals [n, 4] at the detector's input scale, class logits [n, C] (column 0 background) and features [n, F]:
  p = softmax(logits) per row (fp32); dets = proposals / im_scale (fp32);
  max_conf[b] = the largest p[b, c] over the classes c >= start whose greedy NMS keeps b and with p[b, c] > conf_thresh, else 0;
  keep = the first k = min(K, n) indices of max_conf, descending;
  outputs: features[keep], bbox = dets[keep], num_boxes = nonzero scores among the k, cls_prob = p[keep],
  objects = argmax(p[keep][start:], axis=1) -- rows start.. of the kept rows, every column (the reference's row slice, kept as is).

The NMS is upstream maskrcnn_benchmark's, which is not in this tree; what this module assumes of it is DETECTOR_ASSUMPTIONS.
"""
from __future__ import annotations

import numpy as np
import torch

DETECTOR_ASSUMPTIONS = {
    "nms_order": "greedy: boxes in descending score order; a box is kept unless a kept box suppresses it",
    "nms_iou": "legacy +1 IoU on the divided boxes, each step in fp32 in this order: w = max(min(x2) - max(x1) + 1, 0), the same "
               "for h, inter = w * h, areas (x2 - x1 + 1) * (y2 - y1 + 1), IoU = inter / (Sa + Sb - inter)",
    "nms_suppress": "a box is suppressed when IoU > threshold (strict): an IoU of exactly the threshold survives",
    "ties": "equal scores rank the lower proposal index first, in each class's NMS order and in the final ranking (torch.sort "
            "leaves that order open)",
    "argmax": "ties go to the lower column, as torch.argmax documents",
    "box_division": "fp32 x / float32(im_scale); torch on CUDA may compute it as a multiply by the reciprocal, which can differ "
                    "by 1 ulp",
}


def softmax_rows(scores) -> np.ndarray:
    """fp32 softmax over each row (torch's CPU kernel)."""
    return torch.softmax(torch.as_tensor(np.asarray(scores, dtype=np.float32)), dim=-1).numpy()


def divide_boxes(proposals, im_scale) -> np.ndarray:
    return np.asarray(proposals, dtype=np.float32) / np.float32(im_scale)


def iou_matrix(dets) -> np.ndarray:
    """[n, n] legacy IoU of every pair, each operation rounded in fp32."""
    d = np.asarray(dets, dtype=np.float32)
    one, zero = np.float32(1), np.float32(0)
    x1, y1, x2, y2 = (d[:, k] for k in range(4))
    w = np.maximum(np.minimum(x2[:, None], x2[None, :]) - np.maximum(x1[:, None], x1[None, :]) + one, zero)
    h = np.maximum(np.minimum(y2[:, None], y2[None, :]) - np.maximum(y1[:, None], y1[None, :]) + one, zero)
    inter = w * h
    area = (x2 - x1 + one) * (y2 - y1 + one)
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / (area[:, None] + area[None, :] - inter)


def ranked(scores) -> np.ndarray:
    """Indices by descending score, equal scores by ascending index."""
    s = np.asarray(scores)
    return np.lexsort((np.arange(s.shape[0]), -s))


def suppression_rows(over) -> list:
    """The [n, n] bool suppression matrix (IoU > threshold) as one int bitset per row."""
    return [int.from_bytes(np.packbits(r, bitorder="little").tobytes(), "little") for r in np.asarray(over, dtype=bool)]


def greedy_nms(rows, scores) -> list:
    """Kept indices of a greedy NMS, in score order; ``rows`` from `suppression_rows`."""
    removed, keep = 0, []
    for j in ranked(scores):
        j = int(j)
        if removed >> j & 1:
            continue
        keep.append(j)
        removed |= rows[j]
    return keep


def select_image(proposals, scores, features, im_scale, max_boxes=100, conf_thresh=0.0, background=False, nms_iou=0.5):
    """One image's selection.  Returns a dict: keep (int64 [k]), max_conf (the sorted scores [k]), num_boxes, bbox [k, 4],
    features [k, F], cls_prob [k, C], argmax (per kept row, every column) and objects (the reference's argmax(p[keep][start:]))."""
    p = softmax_rows(scores)
    dets = divide_boxes(proposals, im_scale)
    n, C = p.shape
    start = 0 if background else 1
    thr = np.float32(conf_thresh)
    rows = suppression_rows(iou_matrix(dets) > np.float32(nms_iou))
    max_conf = np.zeros(n, dtype=np.float32)
    for c in range(start, C):
        keep = np.asarray(greedy_nms(rows, p[:, c]), dtype=np.int64)
        s = p[keep, c]
        upd = (s > max_conf[keep]) & (s > thr)
        max_conf[keep] = np.where(upd, s, max_conf[keep])
    k = min(int(max_boxes), n)
    keep = ranked(max_conf)[:k].astype(np.int64)
    sorted_conf = max_conf[keep]
    cls_prob = p[keep]
    argmax = np.argmax(cls_prob, axis=1).astype(np.int64)       # numpy: first maximum, the lower column
    return dict(keep=keep, max_conf=sorted_conf, num_boxes=int((sorted_conf != 0).sum()), bbox=dets[keep],
                features=np.asarray(features, dtype=np.float32)[keep], cls_prob=cls_prob, argmax=argmax,
                objects=argmax[start:], max_conf_all=max_conf)


def process_feature_extraction(proposals, scores, feats, im_scales, im_infos, conf_thresh=0.0, background=False, num_features=100,
                               nms_iou=0.5):
    """`(feat_list, info_list)` of the reference's method for per-image heads: feat_list holds the kept feature rows, info_list
    dicts with bbox, num_boxes, objects, image_width, image_height and cls_prob (numpy, the reference's dtypes)."""
    feat_list, info_list = [], []
    for prop, sc, ft, scale, info in zip(proposals, scores, feats, im_scales, im_infos):
        r = select_image(prop, sc, ft, scale, num_features, conf_thresh, background, nms_iou)
        feat_list.append(torch.from_numpy(r["features"]))
        info_list.append({"bbox": r["bbox"], "num_boxes": r["num_boxes"], "objects": r["objects"],
                          "image_width": info["width"], "image_height": info["height"], "cls_prob": r["cls_prob"]})
    return feat_list, info_list
