"""Round-2 paths on the GPU engine against the fp32 CPU oracle.  `-m gpu`.

* fp32-parity mode (compute_dtype="fp32x": fp16 hi/lo split operands, three tensor-core products per k-step, fp32
  attention): <= 1e-3 per logit, the north_star's fp32 tolerance, on BASELINE.json configs[0] (one pair, 36 regions x 30
  tokens, full 268 M model) and on every output of the reduced-width model;
* attn_data_list (element 9 of the reference's tuple, worker.py:287-288): structure and values vs the oracle's list;
* custom_prediction()'s tensor construction on the device (forward_regions, worker.py:422-455) vs the host construction;
* retrieval reuse (encode_text / encode_image / forward_cached): bit-identical to the full forward of the same pairs;
* plan-cache bound; custom_prediction / handle_request / a real MicroBatchWorker round trip on the engine.
"""
import os

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL_FP32X = 1e-3            # north_star: "within 1e-3 fp32 ... per logit"
NAMES = ["vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction",
         "vision_prediction", "vision_logit", "linguisic_prediction", "linguisic_logit"]


def _max_err(ref, out):
    worst = {}
    for i, name in enumerate(NAMES):
        if ref[i] is None:
            continue
        r, o = ref[i], out[i].cpu()
        assert tuple(r.shape) == tuple(o.shape), name
        small = r.abs() < 1000
        worst[name] = (float((o - r).abs()[small].max()), float(r[small].std()) if small.sum() > 1 else 0.0)
    return worst


@pytest.fixture(scope="module")
def tiny_x(tiny_oracle):
    yield from support.one_engine(tiny_oracle, compute_dtype="fp32x", return_attention=True)


@pytest.fixture(scope="module")
def full_x(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="fp32x")


@pytest.fixture(scope="module")
def full_h(full_oracle):
    yield from support.one_engine(full_oracle, return_attention=True)


@pytest.fixture(scope="module")
def tiny_h(tiny_oracle):
    yield from support.one_engine(tiny_oracle, return_attention=True)


# ----------------------------------------------------------------------------------------------- fp32-parity mode
@pytest.mark.parametrize("B,Tin,V,pad", [(2, 30, 36, 0), (3, 16, 10, 3), (1, 12, 37, 0), (4, 37, 101, 7), (2, 70, 100, 0)])
def test_fp32x_tiny_all_outputs(tiny_oracle, tiny_x, parity_log, B, Tin, V, pad):
    inp = support.tiny_inputs(tiny_oracle, B, Tin, V, 500 + B, pad)
    ref = tiny_oracle(*inp, compute_pretraining_heads=True)
    out = tiny_x(*[t.cuda() for t in inp], compute_pretraining_heads=True)
    torch.cuda.synchronize()
    for name, (err, std) in _max_err(ref, out).items():
        parity_log(test=f"fp32x_tiny_B{B}_T{Tin}_V{V}", output=name, err_vs_fp32=err, ref_std=std)
        assert err < TOL_FP32X, (name, err)


def test_fp32x_full_model_configs0(full_oracle, full_x, parity_log):
    """BASELINE.json configs[0]: one pair, 36 regions x 30 tokens, full model; <= 1e-3 per logit on every task head, and on the
    committed fixture of that shape."""
    from oracle import vilbert_ref as R
    for B, seed, pad in ((1, 1235, 0), (2, 1236, 0), (3, 99, 4)):
        inp = R.make_inputs(B, 30, 36, seed=seed, pad_regions=pad)
        ref = full_oracle(*inp, compute_pretraining_heads=False)
        out = full_x(*[t.cuda() for t in inp])
        torch.cuda.synchronize()
        for name, (err, std) in _max_err(ref, out).items():
            parity_log(test=f"fp32x_full_B{B}", output=name, err_vs_fp32=err, ref_std=std)
            assert err < TOL_FP32X, (name, err)
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "full_B1_T30_V36.npz"))
    B, Tin, V, seed, pad = (int(z[k]) for k in ("B", "Tin", "V", "seed", "pad"))
    inp = R.make_inputs(B, Tin, V, seed=seed, pad_regions=pad)
    out = full_x(*[t.cuda() for t in inp])
    err = float((out[0].cpu() - torch.from_numpy(z["vil_prediction"])).abs().max())
    parity_log(test="fp32x_golden_full_B1_T30_V36", output="vil_prediction", max_abs_err=err)
    assert err < TOL_FP32X


def test_fp32x_pretraining_heads_and_shards(full_oracle, full_x, parity_log):
    from oracle import vilbert_ref as R
    inp = R.make_inputs(4, 30, 36, seed=314)
    ref = full_oracle(*inp, compute_pretraining_heads=True)
    dev = [t.cuda() for t in inp]
    out = full_x(*dev, compute_pretraining_heads=True)
    torch.cuda.synchronize()
    for name, (err, std) in _max_err(ref, out).items():
        parity_log(test="fp32x_full_pretraining", output=name, err_vs_fp32=err, ref_std=std)
        assert err < TOL_FP32X * max(1.0, std), (name, err)
    halves = [full_x(*[t[i:i + 2] for t in dev], compute_pretraining_heads=True) for i in (0, 2)]
    assert torch.equal(torch.cat([h[0] for h in halves]), out[0])            # batch sharding stays bit-exact in this mode too


# ----------------------------------------------------------------------------------------------- attention probabilities
def _check_attn(attn, ref_attn, tol, tag, parity_log):
    assert len(attn) == len(ref_attn) == 24
    worst = 0.0
    for a, r in zip(attn, ref_attn):
        if isinstance(r, tuple):
            assert isinstance(a, tuple) and len(a) == 2
            pairs = list(zip(a, r))
        else:
            pairs = [(a, r)]
        for x, y in pairs:
            assert tuple(x.shape) == tuple(y.shape)
            worst = max(worst, float((x.cpu() - y).abs().max()))
            assert float((x.sum(-1) - 1).abs().max()) < 1e-4
    parity_log(test=tag, max_abs_err=worst)
    assert worst < tol, worst


def test_attention_probabilities_tiny(tiny_oracle, tiny_h, tiny_x, parity_log):
    inp = support.tiny_inputs(tiny_oracle, 3, 20, 12, 61, pad=2)
    ref = tiny_oracle(*inp, output_all_attention_masks=True)
    dev = [t.cuda() for t in inp]
    out = tiny_h(*dev, output_all_attention_masks=True)
    _check_attn(out[9], ref[9], 5e-3, "attn_probs_tiny_fp16", parity_log)
    outx = tiny_x(*dev, output_all_attention_masks=True)
    _check_attn(outx[9], ref[9], 1e-4, "attn_probs_tiny_fp32x", parity_log)
    # asking for the probabilities does not change the logits; not asking returns []
    plain = tiny_h(*dev, output_all_attention_masks=False)
    assert plain[9] == []
    for x, y in zip(out[:9], plain[:9]):
        if x is not None:
            assert torch.equal(x, y)
    tiny_h.return_attention = False
    assert tiny_h(*dev, output_all_attention_masks=True)[9] == []
    tiny_h.return_attention = True


def test_attention_probabilities_full(full_oracle, full_h, parity_log):
    from oracle import vilbert_ref as R
    inp = R.make_inputs(2, 30, 36, seed=808, pad_regions=3)
    ref = full_oracle(*inp, output_all_attention_masks=True, compute_pretraining_heads=False)
    out = full_h(*[t.cuda() for t in inp], output_all_attention_masks=True)
    _check_attn(out[9], ref[9], 5e-3, "attn_probs_full_fp16", parity_log)
    assert out[9][0].shape == (2, 12, 31, 31) and out[9][6][0].shape == (2, 8, 31, 36) and out[9][6][1].shape == (2, 8, 36, 31)


# ----------------------------------------------------------------------------------------------- device-side input builder
VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "un", "##aff", "##able", ",", "a", "dog", "on", "grass"])}


def test_forward_regions_matches_host_construction(full_oracle, full_x, full_h, parity_log):
    """One region-pack kernel == worker.py:422-455 on the host (build_inputs) followed by the ordinary forward."""
    from vilbert_b200 import worker_api as W
    tok = W.WordpieceTokenizer(VOCAB)
    feats, infos = support.detector_output_features_first(3, 20, 2048, seed=12)
    text, f, s, seg, im, vm, co, task = W.build_inputs("what is the man holding?", [7], feats, infos, torch.device("cuda", 0), tok)
    rep = lambda t: t.repeat(3, 1)
    boxes = torch.stack([torch.from_numpy(i["bbox"]) for i in infos])
    wh = torch.tensor([[i["image_width"], i["image_height"]] for i in infos], dtype=torch.float32)
    for eng, tol, tag in ((full_x, 2e-4, "fp32x"), (full_h, 5e-3, "fp16")):
        ref = eng(rep(text), f, s, rep(seg), rep(im), vm, None, rep(task))
        out, sp = eng.forward_regions(rep(text), rep(seg), rep(im), rep(task), torch.stack(feats), boxes, wh)
        torch.cuda.synchronize()
        assert float((sp - s).abs().max()) < 1e-6                     # the spatials tensor the reference would have built
        for i in (0, 2, 6):
            err = float((out[i] - ref[i]).abs().max())
            parity_log(test="forward_regions_vs_host_" + tag, output=NAMES[i], max_abs_diff=err)
            assert err < tol, (tag, NAMES[i], err)
    # padded boxes: image 1 has only 13 valid boxes -> same as the forward with those regions masked and a 13-box mean row
    nb = torch.tensor([20, 13, 20], dtype=torch.int32)
    f2, vm2 = f.clone(), vm.clone()
    f2[1, 0] = feats[1][:13].sum(0) / 13
    f2[1, 14:] = 0
    vm2[1, 14:] = 0
    s2 = s.clone()
    s2[1, 14:] = 0
    ref = full_x(rep(text), f2, s2, rep(seg), rep(im), vm2, None, rep(task))
    out, sp = full_x.forward_regions(rep(text), rep(seg), rep(im), rep(task), torch.stack(feats), boxes, wh, num_boxes=nb)
    assert float((out[2] - ref[2]).abs().max()) < 2e-4
    assert float((sp - s2).abs().max()) < 1e-6


# ----------------------------------------------------------------------------------------------- retrieval reuse
@pytest.mark.parametrize("which", ["tiny_fp16", "full_fp16", "tiny_fp32x"])
def test_cached_states_are_bit_identical(which, request, tiny_oracle, full_oracle, parity_log):
    from oracle import vilbert_ref as R
    from vilbert_b200 import _lib as L
    if which.startswith("tiny"):
        eng = request.getfixturevalue("tiny_h" if which == "tiny_fp16" else "tiny_x")
        cap, img = support.tiny_inputs(tiny_oracle, 5, 22, 14, 71), support.tiny_inputs(tiny_oracle, 4, 22, 14, 72, pad=2)
    else:
        eng = request.getfixturevalue("full_h")
        cap, img = R.make_inputs(5, 30, 36, seed=71), R.make_inputs(4, 30, 36, seed=72, pad_regions=2)
    q, seg, im = (cap[i].cuda() for i in (0, 3, 4))
    f, s, vm = (img[i].cuda() for i in (1, 2, 5))
    task = torch.full((5, 1), 7, dtype=torch.long).cuda()
    ts = eng.encode_text(q, seg, im, task)
    vs = eng.encode_image(f, s, vm)
    ci = torch.tensor([0, 0, 1, 2, 3, 4, 4, 2, 1], dtype=torch.int32)
    ii = torch.tensor([0, 3, 1, 2, 0, 3, 1, 1, 2], dtype=torch.int32)
    sel = L.OUT_VIL_LOGIT | L.OUT_VIL_PREDICTION | L.OUT_VISION_LOGIT
    got = eng.forward_cached(ts, ci, vs, ii, select=sel)
    cl, il = ci.long().cuda(), ii.long().cuda()
    want = eng(q[cl], f[il], s[il], seg[cl], im[cl], vm[il], None, task[cl], select=sel)
    torch.cuda.synchronize()
    for i in (0, 2, 6):
        assert torch.equal(got[i], want[i]), (which, NAMES[i], float((got[i] - want[i]).abs().max()))
    parity_log(test="cached_states_bit_identical_" + which, pairs=int(ci.numel()))


def test_plan_cache_is_bounded(tiny_oracle):
    import ctypes as C
    from vilbert_b200 import _lib as L
    eng = support.engine(tiny_oracle, max_plans=3)
    first = None
    for k, B in enumerate([1, 2, 3, 4, 5, 1]):
        inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, B, 20, 12, 31)]
        out = eng(*inp)[0].clone()
        if k == 0:
            first = out
        n = C.c_int64()
        L.check(L.load().vb200_model_dim(eng._handle, b"n_plans", C.byref(n)), eng._handle)
        assert n.value <= 3
    assert torch.equal(out, first)                 # the evicted B=1 plan was rebuilt and gives the same logits
    eng.close()


# ----------------------------------------------------------------------------------------------- host API on the engine
class _OracleAsModel:
    _device = 0

    def __init__(self, oracle):
        self.oracle = oracle

    def __call__(self, *a, **kw):
        kw.pop("select", None)
        a = [t.cpu() if torch.is_tensor(t) else t for t in a]
        return self.oracle(*a, compute_pretraining_heads=False)


def _same_answer(a, b):
    if isinstance(a, list):
        assert [(x["x1"], x["y1"], x["x2"], x["y2"]) for x in a] == [(x["x1"], x["y1"], x["x2"], x["y2"]) for x in b]
        assert [x["confidence"] for x in a] == pytest.approx([x["confidence"] for x in b], abs=0.5)
    else:
        assert a["top3_answer"] == b["top3_answer"]
        assert a["top3_confidence"] == pytest.approx(b["top3_confidence"], abs=5e-3)


@pytest.mark.parametrize("task_id,n_img", [("1", 1), ("12", 2), ("7", 4), ("11", 1), ("13", 1), ("15", 1)])
def test_custom_prediction_on_engine(full_oracle, full_h, task_id, n_img):
    """custom_prediction (tokenise, device-side region pack, forward, decode) on the engine == the reference's host-side tensor
    construction (build_inputs) + the oracle's forward + the same decode."""
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    feats, infos = support.detector_output_features_first(n_img, 20, 2048, seed=40 + n_img)
    W.model = full_h
    ans = W.custom_prediction("what is the man holding?", [int(task_id)], feats, infos, task_id)
    W.model = _OracleAsModel(full_oracle)
    args = W.build_inputs("what is the man holding?", [int(task_id)], feats, infos, torch.device("cpu"))
    ref = W.prediction(*args, task_id, infos)
    W.model = full_h
    _same_answer(ans, ref)
    body = {"image_path": [f"/m/demo/i{k}.jpg" for k in range(n_img)], "question": "what is the man holding?", "socket_id": "s",
            "task_id": task_id}
    res = W.handle_request(body, feats, infos)                      # callback() minus transport (worker.py:556-649)
    assert res["task_id"] == task_id and res == W.shape_result(task_id, ans, body["image_path"])


def test_custom_prediction_unequal_box_counts(full_oracle, full_h):
    """Images with different box counts (torch.stack at worker.py:452 cannot take them): padded, masked, left out of the mean."""
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = full_h
    feats, infos = support.detector_output_features_first(3, 20, 2048, seed=9)
    feats[1] = feats[1][:11]
    infos[1] = dict(infos[1], bbox=infos[1]["bbox"][:11])
    ans = W.custom_prediction("a dog on the grass", [7], feats, infos, "7")
    # image 1 alone (11 boxes, no padding) must score the same as inside the padded batch
    probs = []
    for k in range(3):
        out, _ = full_h.forward_regions(*[t.cuda() for t in (torch.tensor([W.tokenize_query("a dog on the grass")[0]]),
                                                              torch.zeros(1, 37, dtype=torch.long),
                                                              torch.tensor([W.tokenize_query("a dog on the grass")[1]]),
                                                              torch.tensor([[7]]))],
                                        feats[k][None], torch.from_numpy(infos[k]["bbox"])[None],
                                        torch.tensor([[float(infos[k]["image_width"]), float(infos[k]["image_height"])]]))
        probs.append(float(out[2].view(-1)[0]))
    order = sorted(range(3), key=lambda k: -probs[k])
    assert ans["top3_answer"] == order


def test_micro_batch_worker_on_engine(full_oracle, full_h):
    """A real MicroBatchWorker round trip: JSON messages in, WebSocket result dicts out, concurrent messages share one forward,
    and every answer equals handle_request() of that message alone."""
    from vilbert_b200 import worker_api as W
    W.label_maps.update(vqa=None, gqa=None)
    W.tokenizer = W.WordpieceTokenizer(VOCAB)
    W.model = full_h
    msgs = []
    for k, (task_id, n_img, q) in enumerate([("1", 1, "what is the man holding?"), ("12", 2, "the man is holding a dog"),
                                              ("7", 3, "a dog on the grass"), ("11", 1, "the man"), ("13", 1, "a dog"),
                                              ("12", 2, "what color"), ("15", 1, "what is the color of the dog")]):
        feats, infos = support.detector_output_features_first(n_img, 20, 2048, seed=600 + k)
        body = {"image_path": [f"/m/demo/i{j}.jpg" for j in range(n_img)], "question": q, "socket_id": f"s{k}", "task_id": task_id}
        msgs.append((body, feats, infos))
    want = [W.handle_request(*m) for m in msgs]
    worker = W.MicroBatchWorker(max_rows=64, max_wait_ms=500.0)
    futs = [worker.submit(*m) for m in msgs]
    res = [f.result(timeout=120) for f in futs]
    worker.close()
    assert len(worker.batches) == 1 and worker.batches[0] == 11          # all seven messages shared one forward (11 image rows)
    for r, w, m in zip(res, want, msgs):
        assert r["socket_id"] == m[0]["socket_id"] and r["result"]["task_id"] == w["task_id"]
        if "result" in w:
            assert [x["answer"] for x in r["result"]["result"]] == [x["answer"] for x in w["result"]]
            assert [x["confidence"] for x in r["result"]["result"]] == pytest.approx([x["confidence"] for x in w["result"]], abs=0.3)
        else:
            assert r["result"]["image_name_list"] == w["image_name_list"]
            assert r["result"]["confidence_list"] == pytest.approx(w["confidence_list"], abs=0.3)


# ----------------------------------------------------------------------------------------------- step timeline (profiling hook)
def test_timeline_records_every_gemm_cta(tiny_oracle):
    """set_option("timeline", 1): every plain persistent GEMM launch of a forward leaves per-CTA stamps (entry / exit %globaltimer, SM id);
    the logits are the same bits as without the hook."""
    import ctypes as C
    import numpy as np
    from vilbert_b200 import _lib as L
    inp = support.tiny_inputs(tiny_oracle, 4, 30, 36, 94)
    dev = [t.cuda() for t in inp]
    eng = support.engine(tiny_oracle)
    sel = L.OUT_VIL_PREDICTION
    plain = eng(*dev, select=sel)[0].clone()
    eng.set_option("timeline", 1)
    out = eng(*dev, select=sel)[0]
    torch.cuda.synchronize()
    assert torch.equal(plain, out)
    cap, ctas = 256, 304
    n = C.c_int32()
    dims = (C.c_int32 * (4 * cap))()
    st = np.zeros((cap, ctas, 16), dtype=np.int64)
    L.check(L.load().vb200_timeline(eng._handle, 4, 30, 36, sel, 0, cap, C.byref(n), dims, st.ctypes.data_as(C.POINTER(C.c_int64))), eng._handle)
    assert 100 <= n.value <= cap                                   # 125 GEMM launches minus whatever runs on the LN variant
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    for o in range(n.value):
        M, N, K = dims[4 * o], dims[4 * o + 1], dims[4 * o + 2]
        live = st[o][:, 9] > 0
        tiles = ((M + 127) // 128) * ((N + 63) // 64)                              # 64-wide tiles at most
        assert 1 <= live.sum() <= min(tiles, n_sms), (o, M, N, K, int(live.sum()))        # one CTA per SM
        s = st[o][live]
        assert (s[:, 9] >= s[:, 8]).all() and (s[:, 13] > s[:, 0]).all()          # exit after entry (globaltimer and clock64)
        assert (s[:, 12] >= 0).all() and (s[:, 12] < n_sms).all()                    # SM id
    eng.set_option("timeline", 0)
    assert torch.equal(eng(*dev, select=sel)[0], plain)
    eng.close()
