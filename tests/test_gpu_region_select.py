"""Detector-region selection on the device (vb200_select_regions / VILBertForVLTasks.select_regions /
worker_api.process_feature_extraction / worker_api.custom_prediction_detections).  `-m gpu` only.

The heads come from `synthetic_detections(margin=...)`: every softmax sum is exactly 1 and different logits give probabilities a
factor exp(margin) apart, so the selection is unambiguous and the device must reproduce the oracle's indices exactly; equal logits
give equal probabilities on both sides and exercise the index tie rule.  Boxes and feature rows are gathers with the same fp32
expression as the oracle's, so they are compared bit for bit; probabilities within 1e-6 relative.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import detections_ref as D
import support

pytestmark = pytest.mark.gpu

VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "a", "dog", "on", "grass"])}


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16"))


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="bf16")


def _heads(counts, seed, F=2048, Cn=1601):
    from vilbert_b200 import synthetic as S
    return S.synthetic_detections(len(counts), counts, n_classes=Cn, feature_size=F, seed=seed, margin=0.05)


def _device(m, dets, **kw):
    r = m.select_regions(dets, cls_prob=True, objects=True, **kw)
    torch.cuda.synchronize()
    return r


def _check_image(r, i, ref, log=None, tag=""):
    lo, k = r["dst_rows"][i], r["n_boxes"][i]
    assert k == ref["keep"].shape[0]
    np.testing.assert_array_equal(r["keep_index"][lo:lo + k].cpu().numpy(), ref["keep"])
    assert int(r["num_boxes"][i]) == ref["num_boxes"]
    np.testing.assert_array_equal(r["objects"][lo:lo + k].cpu().numpy(), ref["argmax"])
    assert torch.equal(r["boxes"][lo:lo + k].cpu(), torch.from_numpy(ref["bbox"]))
    assert torch.equal(r["box_features"][lo:lo + k].cpu(), torch.from_numpy(ref["features"]))
    mc, cp = r["max_conf"][lo:lo + k].cpu().numpy(), r["cls_prob"][lo:lo + k].cpu().numpy()
    np.testing.assert_allclose(mc, ref["max_conf"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(cp, ref["cls_prob"], rtol=1e-6, atol=1e-30)
    if log is not None:
        rel = float(np.max(np.abs(cp - ref["cls_prob"]) / np.maximum(np.abs(ref["cls_prob"]), 1e-30)))
        log(test="region_select", case=tag, image=i, n=int(ref["max_conf_all"].shape[0]), max_rel_err_cls_prob=rel)


@pytest.mark.parametrize("counts", [[1000], [1, 37, 2048], [100, 1000, 37, 1, 2048, 100, 1000, 37]], ids=["1img", "3img", "8img"])
def test_parity_with_oracle(tiny, counts, parity_log):
    dets = _heads(counts, seed=len(counts))
    r = _device(tiny["bf16"], dets)
    for i, d in enumerate(dets):
        _check_image(r, i, D.select_image(*d), parity_log, f"{len(counts)}img")


def _small(proposals, scores, F=4, scale=1.0):
    n = len(proposals)
    return (torch.tensor(proposals, dtype=torch.float32), torch.tensor(scores, dtype=torch.float32),
            torch.arange(n * F, dtype=torch.float32).view(n, F), scale)


@pytest.mark.parametrize("case", ["duplicates", "iou_at_threshold", "iou_above_threshold", "threshold_zeros", "background",
                                  "fewer_than_k"])
def test_ties_and_thresholds(tiny, case):
    from vilbert_b200 import synthetic as S
    kw, ref_kw = {}, {}
    if case == "duplicates":
        d = _small([[10.0, 10.0, 50.0, 50.0]] * 3, [[0.0, 3.0, 1.0]] * 3)
    elif case.startswith("iou"):
        second = [0.0, 0.0, 9.0, 4.0] if case == "iou_at_threshold" else [0.0, 0.0, 9.0, 5.0]
        d = _small([[0.0, 0.0, 9.0, 9.0], second], [[0.0, 2.0, 0.0], [0.0, 1.0, 0.0]])
    elif case == "threshold_zeros":
        d = S.synthetic_detections(1, 300, n_classes=50, feature_size=8, seed=5, margin=0.5, n_clusters=2, n_dominant=2)[0]
        kw = ref_kw = dict(conf_thresh=0.5)
    elif case == "background":
        d = S.synthetic_detections(1, 200, n_classes=30, feature_size=8, seed=6, margin=0.5)[0]
        kw = ref_kw = dict(background=True)
    else:
        d = S.synthetic_detections(1, 7, n_classes=9, feature_size=8, seed=7, margin=0.5)[0]
    ref = D.select_image(*d, max_boxes=100, **ref_kw)
    r = _device(tiny["fp16"], [d], max_boxes=100, **kw)
    _check_image(r, 0, ref)
    if case == "threshold_zeros":
        assert 0 < ref["num_boxes"] < 100


def _bits(r, i):
    lo, k = r["dst_rows"][i], r["n_boxes"][i]
    return [r[n][lo:lo + k].cpu() for n in ("keep_index", "max_conf", "boxes", "box_features", "cls_prob", "objects")] + \
        [r["num_boxes"][i].cpu()]


def test_images_are_independent_and_calls_deterministic(tiny):
    m = tiny["bf16"]
    dets = _heads([300, 1000, 64], seed=21)
    batched = _device(m, dets)
    again = _device(m, dets)
    for i, d in enumerate(dets):
        alone = _device(m, [d])
        for a, b, c in zip(_bits(batched, i), _bits(alone, 0), _bits(again, i)):
            assert torch.equal(a, b) and torch.equal(a, c)


def test_back_to_back_calls_need_no_synchronisation(tiny):
    m = tiny["bf16"]
    small, big = _heads([50, 80], seed=31), _heads([2048, 1500, 900, 2000], seed=32)
    want = [_device(m, small), _device(m, big)]
    got = [m.select_regions(small, cls_prob=True, objects=True), m.select_regions(big, cls_prob=True, objects=True),
           m.select_regions(small, cls_prob=True, objects=True)]
    torch.cuda.synchronize()
    for r, w in zip(got, want + want[:1]):
        for i in range(len(w["n_boxes"])):
            for a, b in zip(_bits(r, i), _bits(w, i)):
                assert torch.equal(a, b)


def _composition(m, counts, seed):
    """select_regions -> forward_regions_packed vs forward_regions_packed on the oracle's selection uploaded from the host."""
    F = m._dims["v_feature_size"]
    dets = _heads(counts, seed=seed, F=F)
    g = torch.Generator().manual_seed(seed)
    n_tokens = [int(x) for x in torch.randint(3, 20, (len(counts),), generator=g)]
    question = torch.randint(5, 200, (sum(n_tokens),), generator=g)
    seg = torch.zeros_like(question)
    task = torch.ones(len(counts), 1, dtype=torch.long)
    wh = torch.tensor([[640.0, 480.0]] * len(counts))
    r = m.select_regions(dets, max_boxes=100)
    refs = [D.select_image(*d, max_boxes=100) for d in dets]
    host_feats = torch.cat([torch.from_numpy(x["features"]) for x in refs])
    host_boxes = torch.cat([torch.from_numpy(x["bbox"]) for x in refs])
    nb = r["n_boxes"]
    a, sa = m.forward_regions_packed(question, seg, task, r["box_features"], r["boxes"], wh, n_tokens, nb, max_boxes=100)
    b, sb = m.forward_regions_packed(question, seg, task, host_feats, host_boxes, wh, n_tokens, nb, max_boxes=100)
    torch.cuda.synchronize()
    assert torch.equal(sa, sb)
    for x, y in zip(a[:9], b[:9]):
        assert (x is None) == (y is None)
        if x is not None:
            assert torch.equal(x, y)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_composition_tiny(tiny, dtype):
    _composition(tiny[dtype], [37, 1000, 1, 100], seed=41)


def test_composition_full(full):
    _composition(full, [1000, 37, 250], seed=42)


def _worker(m):
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = m
    return W


def test_process_feature_extraction_matches_oracle(full):
    W = _worker(full)
    counts = [1000, 37, 1]
    dets = _heads(counts, seed=51)
    props, scores, feats, scales = zip(*dets)
    infos = [{"width": 640 + i, "height": 480 - i} for i in range(len(counts))]
    for background in (False, True):
        got_f, got_i = W.process_feature_extraction(props, torch.cat(scores).cuda(), torch.cat(feats).cuda(), scales, infos,
                                                    background=background)
        ref_f, ref_i = D.process_feature_extraction(props, scores, feats, scales, infos, background=background)
        for gf, rf, gi, ri in zip(got_f, ref_f, got_i, ref_i):
            assert torch.equal(gf.cpu(), rf)
            assert set(gi) == set(ri)
            for k in ri:
                if isinstance(ri[k], np.ndarray):
                    assert gi[k].dtype == ri[k].dtype and gi[k].shape == ri[k].shape, k
                    if k == "cls_prob":
                        np.testing.assert_allclose(gi[k], ri[k], rtol=1e-6, atol=1e-30)
                    else:
                        np.testing.assert_array_equal(gi[k], ri[k])
                else:
                    assert type(gi[k]) is type(ri[k]) and gi[k] == ri[k], k


@pytest.mark.parametrize("decode", ["host", "device"])
def test_custom_prediction_detections_matches_host_selection(full, decode):
    """VQA, NLVR2, retrieval over three images, RefCOCO grounding and GQA in one call, against custom_prediction_packed fed with
    the features and boxes process_feature_extraction selected (copied to the host)."""
    W = _worker(full)
    F = full._dims["v_feature_size"]
    det_reqs, host_reqs = [], []
    for k, (task_id, counts, q) in enumerate([("1", [1000], "what is the man holding?"), ("12", [300, 80], "the man is holding a dog"),
                                               ("7", [60, 1000, 40], "a dog on the grass"), ("11", [500], "the man"),
                                               ("15", [90], "what is the color of the dog")]):
        dets = _heads(counts, seed=600 + k, F=F)
        infos = [{"image_width": 640.0 + j, "image_height": 480.0} for j in range(len(counts))]
        det_reqs.append((q, [int(task_id)], dets, infos, task_id))
        props, scores, feats, scales = zip(*dets)
        f, inf = W.process_feature_extraction(props, scores, feats, scales, [{"width": i["image_width"], "height": i["image_height"]}
                                                                              for i in infos])
        host_infos = [dict(i, image_width=h["image_width"], image_height=h["image_height"]) for i, h in zip(inf, infos)]
        host_reqs.append((q, [int(task_id)], [x.cpu() for x in f], host_infos, task_id))
    got = W.custom_prediction_detections(det_reqs, decode=decode)
    want = W.custom_prediction_packed(host_reqs, decode=decode)
    assert got == want


def _call(m, imgs, params, out):
    from vilbert_b200 import _lib as L
    arr = (L.Detections * max(1, len(imgs)))(*imgs)
    rc = L.load().vb200_select_regions(m._handle, arr, len(imgs), C.byref(params), C.byref(out), None)
    return rc, (L.load().vb200_last_error(m._handle) or b"").decode()


def test_rejections_name_the_image_and_enqueue_nothing(tiny):
    from vilbert_b200 import _lib as L
    m = tiny["fp16"]
    dets = _heads([40, 40], seed=71, F=8, Cn=11)
    dev = [tuple(t.cuda() if torch.is_tensor(t) else t for t in d) for d in dets]
    bf = torch.full((40, 8), 7.0, device="cuda")
    bx = torch.full((40, 4), 7.0, device="cuda")
    nb = torch.full((2,), 7, dtype=torch.int32, device="cuda")

    def img(i, **kw):
        p, s, f, sc = dev[i]
        a = dict(n_proposals=40, dst_row=20 * i, im_scale=sc, proposals=p.data_ptr(), scores=s.data_ptr(), features=f.data_ptr())
        a.update(kw)
        return L.Detections(**a)

    def params(**kw):
        a = dict(n_classes=11, feature_size=8, max_boxes=20, conf_thresh=0.0, nms_iou=0.5, background=0, out_rows=40)
        a.update(kw)
        return L.SelectParams(**a)
    out = L.Selected(bf.data_ptr(), bx.data_ptr(), nb.data_ptr(), None, None, None, None)
    rc, _ = _call(m, [img(0), img(1)], params(), out)        # the valid call: writes every row
    assert rc == 0
    torch.cuda.synchronize()
    bf.fill_(7.0), bx.fill_(7.0), nb.fill_(7)
    cases = [([img(0), img(1, n_proposals=0)], params(), out, "image 1"),
             ([img(0), img(1, n_proposals=2049)], params(), out, "image 1"),
             ([img(0), img(1, scores=None)], params(), out, "image 1"),
             ([img(0), img(1, features=dev[1][2].data_ptr() + 4)], params(), out, "image 1"),
             ([img(0), img(1, im_scale=0.0)], params(), out, "image 1"),
             ([img(0), img(1, dst_row=10)], params(), out, "image 1"),
             ([img(0), img(1, dst_row=21)], params(), out, "image 1"),
             ([img(0, dst_row=-1), img(1)], params(), out, "image 0"),
             ([img(0), img(1)], params(n_classes=1), out, "n_classes"),
             ([img(0), img(1)], params(n_classes=2049), out, "n_classes"),
             ([img(0), img(1)], params(feature_size=6), out, "feature_size"),
             ([img(0), img(1)], params(max_boxes=0), out, "max_boxes"),
             ([img(0), img(1)], params(max_boxes=256), out, "max_boxes"),
             ([img(0), img(1)], params(nms_iou=0.0), out, "nms_iou"),
             ([img(0), img(1)], params(nms_iou=1.5), out, "nms_iou"),
             ([img(0), img(1)], params(background=2), out, "background"),
             ([img(0), img(1)], params(out_rows=39), out, "image 1"),
             ([img(0), img(1)], params(), L.Selected(None, bx.data_ptr(), nb.data_ptr(), None, None, None, None), "required"),
             ([img(0), img(1)], params(), L.Selected(bf.data_ptr(), bx.data_ptr(), None, None, None, None, None), "required"),
             ([], params(), out, "n = 0")]
    for imgs, p, o, needle in cases:
        rc, msg = _call(m, imgs, p, o)
        assert rc == -1, (needle, rc, msg)                  # VB200_ERR_INVALID
        assert needle in msg, (needle, msg)
    torch.cuda.synchronize()
    assert (bf == 7.0).all() and (bx == 7.0).all() and (nb == 7).all()
