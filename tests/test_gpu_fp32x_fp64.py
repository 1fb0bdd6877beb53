"""The fp32-parity mode (compute_dtype="fp32x") against an fp64 run of the oracle, at the accuracy the mode has.  `-m gpu` only.

tests/test_gpu_round2.py holds this mode to 1e-3 per logit against the fp32 oracle, which is ~1000x what it achieves: a 16-bit
rounding where a hi/lo split belongs, or the polynomial GELU epilogue in place of erf, passes that.  Here every fp32x path runs against
the fp64 oracle (oracle.fp64) on the same inputs, and each check family has one bound in oracle/fp64.py, set from measurement and
kept under the smallest such defect the family must catch (tests/test_fp64_oracle.py enforces that on CPU):

* the nine outputs (and pretraining_heads' logits, the pre-training scores): max |o - r| / max(1, |r|), so the -10000 rows of masked
  regions count on a relative scale;
* the final-state taps (debug_taps=True): sequence_output_t / _v against the oracle's final states, pooled_output against the product
  the alignment head reads;
* with return_attention=True, all 24 attention maps, max |o - r|; a failure names the first layer and map over the bound;
* the three pre-training losses, max |o - r| / max(1, |r|).

Every path, the 268 M model included, is held to ``BOUNDS``.  The split GEMM itself is checked against fp64 at K = 256 ... 3072: its
error must not grow with the contraction length (the wgmma accumulator's own fp32 sums over K' = 3K did).

Every measured error goes to the parity log before anything is asserted.
"""
import pytest
import torch

from oracle import fp64 as X
import support

pytestmark = pytest.mark.gpu

VOCAB = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "what", "is", "the", "man", "hold", "##ing",
                                     "?", "color", "of", "un", "##aff", "##able", ",", "a", "dog", "on", "grass"])}


def _check(tag, parity_log, logits=None, states=None, attention=None, losses=None):
    """Log every error of a case, then hold each family to its bound in ``X.BOUNDS``.  ``attention`` is attention_errs' list in execution order."""
    bound = X.BOUNDS
    fams = {"logits": logits or {}, "states": states or {}, "losses": losses or {}, "attention": dict(attention or [])}
    for fam, errs in fams.items():
        for name, e in errs.items():
            parity_log(test="fp32x_vs_fp64_" + tag, family=fam, output=name, err_vs_fp64=e, bound=bound[fam])
    over = {fam: {n: e for n, e in errs.items() if not e < bound[fam]} for fam, errs in fams.items() if fam != "attention"}
    over = {fam: v for fam, v in over.items() if v}
    first = X.first_over(attention or [], bound["attention"])
    assert not over and first is None, \
        f"{tag}: over the bound: {over}" + (f"; first attention map over {bound['attention']}: {first[0]} ({first[1]:.3e})" if first else "")


def _forward(o64, eng, inp, tag, parity_log, pretraining=True, attention=True):
    """One dense forward: the nine outputs, the final-state taps and (``attention``) the 24 maps against the fp64 oracle."""
    collect = {}
    ref = o64(*inp, compute_pretraining_heads=pretraining, output_all_attention_masks=attention, collect=collect)
    out, taps = eng(*[t.cuda() for t in inp], compute_pretraining_heads=pretraining, output_all_attention_masks=attention,
                    debug_taps=True)
    torch.cuda.synchronize()
    attn = X.attention_errs(out[9], ref[9], o64.bert.encoder.schedule()) if attention else None
    if not attention:
        assert out[9] == []
    _check(tag, parity_log, logits=X.output_errs(out, ref), states=X.state_errs(taps, collect["final"]), attention=attn)
    return out, taps


@pytest.fixture(scope="module")
def tiny64(tiny_oracle):
    return X.fp64(tiny_oracle)


@pytest.fixture(scope="module")
def full64(full_oracle):
    return X.fp64(full_oracle)


@pytest.fixture(scope="module")
def tiny_x(tiny_oracle):
    yield from support.one_engine(tiny_oracle, compute_dtype="fp32x", return_attention=True)


@pytest.fixture(scope="module")
def full_x(full_oracle):
    yield from support.one_engine(full_oracle, compute_dtype="fp32x", return_attention=True)


# ------------------------------------------------------------------ the split GEMM
# max |y - r| / (|x| |w|^T), r = the documented hi.hi + lo.hi + hi.lo in fp64; ~4x the worst measured on an H100 80GB HBM3 (700 W):
# 9.1e-8 / 7.3e-8 / 7.4e-8 at K = 256 / 768 / 3072
SPLIT_GEMM_BOUND = 4e-7


@pytest.mark.parametrize("K", [256, 768, 3072])
def test_split_gemm_error_does_not_grow_with_k(K, parity_log):
    """vb200_linear_split (the engine's fp32-parity GEMM) against the documented contraction in fp64, at the reduced-width model's
    K and the 268 M model's: the error, relative to sum_k |x_k w_k|, stays at fp32 rounding whatever K."""
    import ctypes as C
    from oracle import kernel_refs as KR
    from vilbert_b200 import _lib as L
    g = torch.Generator().manual_seed(K)
    M, N = 256, 384
    x, w = torch.randn(M, K, generator=g) * 1.7, torch.randn(N, K, generator=g) * 0.02
    xh, wh = x.half().double(), w.half().double()
    xl, wl = (x - x.half().float()).half().double(), (w - w.half().float()).half().double()
    ref = xh @ wh.t() + xl @ wh.t() + xh @ wl.t()
    scale = x.double().abs() @ w.double().abs().t()
    x3, w3, b = KR.split16(x).cuda(), KR.split16_w(w).cuda(), torch.zeros(N, device="cuda")
    y = torch.full((M, N), float("nan"), device="cuda")
    L.check(L.load().vb200_linear_split(x3.data_ptr(), 3 * K, w3.data_ptr(), 3 * K, b.data_ptr(), 0, None, 0, y.data_ptr(), N, M, N,
                                        3 * K, C.c_void_p(torch.cuda.current_stream().cuda_stream)), None)
    torch.cuda.synchronize()
    err = float(((y.cpu().double() - ref).abs() / scale).max())
    parity_log(test=f"fp32x_vs_fp64_split_gemm_K{K}", family="split_gemm", output="y", err_vs_fp64=err, bound=SPLIT_GEMM_BOUND)
    assert err < SPLIT_GEMM_BOUND, (K, err)


# ------------------------------------------------------------------ dense forwards
@pytest.mark.parametrize("B,Tin,V,pad", [(2, 30, 36, 0), (3, 16, 10, 3), (1, 12, 37, 0), (4, 37, 101, 7), (2, 70, 100, 0),
                                         (1, 3, 1, 0), (1, 155, 256, 11), (5, 3, 7, 2)])
def test_tiny_dense(tiny_oracle, tiny64, tiny_x, parity_log, B, Tin, V, pad):
    """The shapes of test_fp32x_tiny_all_outputs and the corners of test_tiny_model_all_outputs, with the pre-training heads."""
    _forward(tiny64, tiny_x, support.tiny_inputs(tiny_oracle, B, Tin, V, 500 + B, pad), f"tiny_B{B}_T{Tin}_V{V}", parity_log)


@pytest.mark.parametrize("B,seed,pad,pretraining", [(1, 1235, 0, False), (2, 1236, 0, False), (3, 99, 4, False), (4, 314, 0, True)])
def test_full_model(full64, full_x, parity_log, B, seed, pad, pretraining):
    """The 268 M model at 30 tokens x 36 regions: the cases of test_fp32x_full_model_configs0, and B = 4 with the pre-training heads."""
    from oracle import vilbert_ref as R
    _forward(full64, full_x, R.make_inputs(B, 30, 36, seed=seed, pad_regions=pad), f"full_B{B}", parity_log, pretraining=pretraining)


def test_full_model_without_attention_output(full64, full_x, parity_log):
    """The same engine when the call does not ask for the maps (the plan every serving call runs)."""
    from oracle import vilbert_ref as R
    _forward(full64, full_x, R.make_inputs(2, 30, 36, seed=808, pad_regions=3), "full_B2_no_maps", parity_log, pretraining=False,
             attention=False)


# ------------------------------------------------------------------ detector output in (forward_regions)
def test_forward_regions(tiny_oracle, tiny64, tiny_x, parity_log):
    """vb200_forward_regions against the fp64 oracle on the host construction of the same detector output (build_inputs), with all
    boxes valid and with image 1 holding 13 valid boxes of 20 (padded boxes zero, masked, left out of the mean row)."""
    from vilbert_b200 import worker_api as W
    tok = W.WordpieceTokenizer(VOCAB)
    feats, infos = support.detector_output_features_first(3, 20, tiny_oracle.config.v_feature_size, seed=12)
    text, f, s, seg, im, vm, _, task = W.build_inputs("what is the man holding?", [7], feats, infos, torch.device("cpu"), tok)
    rep = lambda t: t.repeat(3, 1)
    boxes = torch.stack([torch.from_numpy(i["bbox"]) for i in infos])
    wh = torch.tensor([[i["image_width"], i["image_height"]] for i in infos], dtype=torch.float32)
    args = [t.cuda() for t in (rep(text), rep(seg), rep(im), rep(task), torch.stack(feats), boxes, wh)]
    sched = tiny64.bert.encoder.schedule()
    ref = tiny64(rep(text), f, s, rep(seg), rep(im), vm, None, rep(task), compute_pretraining_heads=False, output_all_attention_masks=True)
    out, _ = tiny_x.forward_regions(*args, output_all_attention_masks=True)
    torch.cuda.synchronize()
    _check("forward_regions", parity_log, logits=X.output_errs(out, ref), attention=X.attention_errs(out[9], ref[9], sched))
    f2, vm2, s2 = f.clone(), vm.clone(), s.clone()
    f2[1, 0] = feats[1][:13].sum(0) / 13
    f2[1, 14:] = 0
    vm2[1, 14:] = 0
    s2[1, 14:] = 0
    ref = tiny64(rep(text), f2, s2, rep(seg), rep(im), vm2, None, rep(task), compute_pretraining_heads=False,
                 output_all_attention_masks=True)
    out, _ = tiny_x.forward_regions(*args, num_boxes=torch.tensor([20, 13, 20], dtype=torch.int32), output_all_attention_masks=True)
    torch.cuda.synchronize()
    _check("forward_regions_num_boxes", parity_log, logits=X.output_errs(out, ref), attention=X.attention_errs(out[9], ref[9], sched))


# ------------------------------------------------------------------ retrieval reuse
def test_cached_states(tiny_oracle, tiny64, tiny_x, parity_log):
    """encode_text / encode_image once, forward_cached on nine pairs (repeats included) against the fp64 oracle on those pairs."""
    from vilbert_b200 import _lib as L
    cap, img = support.tiny_inputs(tiny_oracle, 5, 22, 14, 71), support.tiny_inputs(tiny_oracle, 4, 22, 14, 72, pad=2)
    q, seg, im = (cap[i] for i in (0, 3, 4))
    f, s, vm = (img[i] for i in (1, 2, 5))
    task = torch.full((5, 1), 7, dtype=torch.long)
    ts = tiny_x.encode_text(q.cuda(), seg.cuda(), im.cuda(), task.cuda())
    vs = tiny_x.encode_image(f.cuda(), s.cuda(), vm.cuda())
    ci = torch.tensor([0, 0, 1, 2, 3, 4, 4, 2, 1], dtype=torch.int32)
    ii = torch.tensor([0, 3, 1, 2, 0, 3, 1, 1, 2], dtype=torch.int32)
    out = tiny_x.forward_cached(ts, ci, vs, ii, select=L.OUT_TASK_HEADS)
    torch.cuda.synchronize()
    cl, il = ci.long(), ii.long()
    ref = tiny64(q[cl], f[il], s[il], seg[cl], im[cl], vm[il], None, task[cl], compute_pretraining_heads=False)
    _check("cached_states", parity_log, logits=X.output_errs(out, ref))


# ------------------------------------------------------------------ sequences past 256 rows
def test_long_sequences(parity_log):
    """The tiny model with 1024 positions on an engine bounded at 1024 rows: the streaming fp32 attention kernel past 256 rows."""
    from oracle import vilbert_ref as R
    oracle = R.build(R.tiny_config(max_position_embeddings=1024), seed=7, num_labels=200)
    o64 = X.fp64(oracle)
    m = support.engine(oracle, compute_dtype="fp32x", max_rows_per_sample=1024, return_attention=True)
    try:
        for Tin, V in [(300, 36), (511, 257), (30, 1000)]:
            _forward(o64, m, support.tiny_inputs(oracle, 1, Tin, V, Tin + V), f"long_T{Tin}_V{V}", parity_log)
    finally:
        m.close()


# ------------------------------------------------------------------ pre-training
def test_pretraining_heads_at_rows(tiny64, tiny_x, parity_log):
    """pretraining_heads on an fp32x forward's taps, at listed rows (the 128-row bucket edges, the last row, duplicates), against the
    fp64 cls heads on the fp64 final states."""
    B, Tin, V = 3, 60, 50
    inp = support.tiny_inputs(tiny64, B, Tin, V, 103, pad=2)
    _, taps = tiny_x(*[t.cuda() for t in inp], select=0, debug_taps=True)
    last_t, last_v = B * (Tin + 1) - 1, B * V - 1
    tr, vr, pr = [0, 127, 128, last_t, 5, 5, last_t], [0, 127, 128, last_v, 3, 3], [2, 0, 1, 1]
    res = tiny_x.pretraining_heads(taps, text_rows=tr, image_rows=vr, pair_rows=pr)
    torch.cuda.synchronize()
    collect = {}
    tiny64(*inp, compute_pretraining_heads=False, collect=collect)
    t, v, pt, pv = collect["final"]
    cls = tiny64.cls
    with torch.no_grad():
        ref = {"token_logits": cls.predictions(t.reshape(-1, t.shape[-1])[tr]),
               "region_logits": cls.imagePredictions(v.reshape(-1, v.shape[-1])[vr]),
               "alignment": cls.bi_seq_relationship((pt * pv)[pr])}
    _check("pretraining_heads_rows", parity_log, logits={k: X.rel_err(res[k], r) for k, r in ref.items()},
           states=X.state_errs(taps, collect["final"]))


@pytest.fixture(scope="module")
def pt():
    from oracle import pretraining_ref as P
    import vilbert_b200 as vb
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    m = support.engine(oracle, vb.BertForMultiModalPreTraining, return_attention=True, compute_dtype="fp32x")
    yield X.fp64(oracle), m
    m.close()


KEYS = ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")
LABELS = ("masked_lm_labels", "image_label", "image_target", "next_sentence_label")


def _masked_batch(model, B, Tin, V, seed):
    from vilbert_b200 import synthetic as S
    d = model._dims
    return S.synthetic_masked_batch(B, Tin, V, seed=seed, vocab_size=d["vocab_size"], v_feature_size=d["v_feature_size"],
                                    v_target_size=d["v_target_size"])


def test_pretraining_model_scores(pt, parity_log):
    """BertForMultiModalPreTraining without labels: the token and region scores, the alignment score, the 24 maps and the final
    states against the fp64 pre-training oracle."""
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    o64, model = pt
    b = _masked_batch(model, 3, 24, 11, seed=1)
    inp = [b[k] for k in KEYS]
    dev = [x.cuda() for x in inp]
    t, v, align, attn = model(*dev, output_all_attention_masks=True)
    _, taps = vb.VILBertForVLTasks.forward(model, *dev, None, None, select=L.OUT_LINGUISIC_PREDICTION | L.OUT_VISION_PREDICTION,
                                           debug_taps=True)
    torch.cuda.synchronize()
    collect = {}
    rt, rv, ralign, rattn = o64(*inp, collect=collect)
    _check("pretraining_model_scores", parity_log,
           logits={"prediction_scores_t": X.rel_err(t, rt), "prediction_scores_v": X.rel_err(v, rv),
                   "seq_relationship_score": X.rel_err(align, ralign)},
           states=X.state_errs(taps, collect["final"]), attention=X.attention_errs(attn, rattn, o64.bert.encoder.schedule()))


def test_pretraining_model_losses(pt, parity_log):
    """The three losses of BertForMultiModalPreTraining with labels against oracle/pretraining_ref.py in fp64."""
    o64, model = pt
    b = _masked_batch(model, 4, 36, 37, seed=9)
    got = model(*[b[k].cuda() for k in KEYS], *[b[k].cuda() for k in LABELS])
    torch.cuda.synchronize()
    labels = [b[k] for k in LABELS]
    labels[2] = labels[2].double()
    ref = o64(*[b[k] for k in KEYS], *labels)
    _check("pretraining_model_losses", parity_log,
           losses={n: X.rel_err(g, r) for n, g, r in zip(("masked_lm_loss", "masked_img_loss", "next_sentence_loss"), got, ref)})
