"""Packed variable-length batches (vb200_forward_packed / VILBertForVLTasks.forward_packed / worker_api.prediction_packed) and the
GEMM's device row count.  `-m gpu` only.

A packed batch computes, per sample, exactly what a forward of that sample alone computes: every kernel is row- or sample-local
with a fixed k-order, the tile width does not change bits (DESIGN.md section 4.1), and attention runs each sample at its own length.
So the packed outputs are compared with single-sample dense forwards bit for bit, and with the fp32 oracle on the equivalent padded
batch at the tolerances of test_gpu_model.py.
"""
import ctypes as C

import pytest
import torch

import support

pytestmark = pytest.mark.gpu

TOL = 1e-2                 # fp16 mode vs the fp32 oracle (test_gpu_model.py)
TOL_BF16_VS_FP32 = 3.5e-2  # bf16 mode vs the fp32 oracle, x max(1, logit std) (test_gpu_model.py)
DT = ("fp16", "bf16")
ROW_OUT = {5: "regions", 6: "regions", 7: "tokens", 8: "tokens"}    # per-row outputs of the 10-tuple


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, DT)


@pytest.fixture(scope="module")
def full(full_oracle):
    yield from support.one_engine(full_oracle)


def _packed(model, samples, select, **kw):
    out = model.forward_packed(*support.packed_sample_args(samples), select=select, debug_taps=True, **kw)
    torch.cuda.synchronize()
    return out


def _check_bitwise(model, samples, packed):
    import vilbert_b200 as vb
    (out, taps) = packed
    B = len(samples)
    t_rows = [len(s[0]) + model._dims["task_specific_tokens"] for s in samples]
    v_rows = [s[2].shape[0] for s in samples]
    for i, smp in enumerate(samples):
        ref, rtaps = support.dense_alone(model, smp, select=vb.OUT_ALL, debug_taps=True)
        for k in range(9):
            if k in ROW_OUT:
                got = support.split_rows(out[k], v_rows if ROW_OUT[k] == "regions" else t_rows)[i]
                want = ref[k][0]
            elif k == 3:
                if B % 2 == 0:
                    continue            # the pair head reads two samples: covered by pooled_output below and the oracle test
                got, want = out[3][i], ref[3][0]
            else:
                got, want = out[k][i], ref[k][0]
            assert torch.equal(got, want), f"sample {i}: output {k} differs from the sample's own dense forward"
        assert torch.equal(support.split_rows(taps["sequence_output_t"], t_rows)[i], rtaps["sequence_output_t"][0]), f"sample {i}: text tap"
        assert torch.equal(support.split_rows(taps["sequence_output_v"], v_rows)[i], rtaps["sequence_output_v"][0]), f"sample {i}: image tap"
        assert torch.equal(taps["pooled_output"][i], rtaps["pooled_output"][0]), f"sample {i}: pooled tap"


CORNERS = [(1, 101), (3, 1), (12, 256), (37, 7), (155, 36), (37, 256), (1, 1)]


@pytest.mark.parametrize("mode", DT)
@pytest.mark.parametrize("B", [7, 6])
def test_packed_bitwise_equals_dense_per_sample(tiny, mode, B):
    """Tin in {1, 3, 12, 37, 155} and V in {1, 7, 36, 101, 256} mixed in one batch, odd and even B: all nine outputs and the three
    taps of every sample equal the dense forward of that sample alone, bit for bit."""
    import vilbert_b200 as vb
    model = tiny[mode]
    samples = support.batch(model, CORNERS[:B], seed=40 + B)
    _check_bitwise(model, samples, _packed(model, samples, vb.OUT_ALL))


def test_packed_bitwise_full_model(full):
    """The 268 M model with an 8-sample mix of worker-like lengths (VQA head plus the per-row heads)."""
    import vilbert_b200 as vb
    lens = [(9, 37), (30, 101), (14, 11), (37, 64), (7, 100), (22, 18), (5, 2), (28, 73)]
    samples = support.batch(full, lens, seed=7)
    _check_bitwise(full, samples, _packed(full, samples, vb.OUT_ALL))


@pytest.mark.parametrize("mode", DT)
def test_packed_matches_oracle_on_padded_batch(tiny_oracle, tiny, mode):
    """Packed outputs vs the fp32 oracle on the same samples padded to a common shape with input_mask / image_mask = 1 on the real
    rows, restricted to the real rows."""
    import vilbert_b200 as vb
    model = tiny[mode]
    lens = [(5, 36), (30, 10), (12, 101), (1, 1), (37, 7), (20, 64)]
    samples = support.batch(model, lens, seed=3)
    out, _ = _packed(model, samples, vb.OUT_ALL)
    B, Tm, Vm = len(samples), max(t for t, _ in lens), max(v for _, v in lens)
    F = model._dims["v_feature_size"]
    q, seg, im = (torch.zeros(B, Tm, dtype=torch.long) for _ in range(3))
    f, s, vm = torch.zeros(B, Vm, F), torch.zeros(B, Vm, 5), torch.zeros(B, Vm, dtype=torch.uint8)
    for b, (qq, sg, ff, ss, _) in enumerate(samples):
        q[b, :len(qq)], seg[b, :len(qq)], im[b, :len(qq)] = qq, sg, 1
        f[b, :ff.shape[0]], s[b, :ff.shape[0]], vm[b, :ff.shape[0]] = ff, ss, 1
    task = torch.tensor([[smp[4]] for smp in samples])
    ref = tiny_oracle(q, f, s, seg, im, vm, None, task, compute_pretraining_heads=True)
    for k in range(9):
        if k in ROW_OUT:
            per = [r[:(t + 1) if ROW_OUT[k] == "tokens" else v] for r, (t, v) in zip(ref[k], lens)]
            want = torch.cat(per, dim=0).reshape(out[k].shape)
        else:
            want = ref[k]
        err = float((out[k].cpu() - want).abs().max())
        tol = TOL if mode == "fp16" else TOL_BF16_VS_FP32 * max(1.0, float(want.std()))
        assert err < tol, f"{mode}: output {k} vs fp32 oracle: {err} >= {tol}"


def test_packed_plan_reuse_and_capacity(tiny):
    """Lengths in one 16-row bucket share a plan; fixed capacities share one plan across quite different maxima, and capacity
    changes no bit."""
    import vilbert_b200 as vb
    model = tiny["fp16"]
    sel = vb.OUT_TASK_HEADS
    a = support.batch(model, [(20, 40), (3, 33), (25, 12), (8, 47)], seed=11)       # maxima T = 26, V = 47 -> bucket (32, 48)
    b = support.batch(model, [(30, 35), (30, 48), (2, 5), (17, 20)], seed=12)       # maxima T = 31, V = 48 -> the same bucket
    _packed(model, a, sel)
    n = support.n_plans(model)
    _packed(model, b, sel)
    assert support.n_plans(model) == n
    cap = dict(max_tokens=37, max_regions=101)
    small = support.batch(model, [(2, 3), (5, 1), (4, 9), (1, 2)], seed=13)
    large = support.batch(model, [(37, 101), (12, 60), (30, 7), (36, 100)], seed=14)
    ref_small, ref_large = _packed(model, small, sel), _packed(model, large, sel)
    got_small = _packed(model, small, sel, **cap)
    n = support.n_plans(model)
    got_large = _packed(model, large, sel, **cap)
    assert support.n_plans(model) == n
    for got, ref in ((got_small, ref_small), (got_large, ref_large)):
        for k in range(9):
            assert (got[0][k] is None) == (ref[0][k] is None)
            if got[0][k] is not None:
                assert torch.equal(got[0][k], ref[0][k]), f"output {k} depends on the plan capacity"
        for k in got[1]:
            assert torch.equal(got[1][k], ref[1][k]), k


def test_packed_rejections(tiny_oracle, tiny):
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    model = tiny["fp16"]
    ok = support.batch(model, [(5, 3), (4, 2)], seed=21)
    with pytest.raises(L.VilbertB200Error, match=r"error -1: .*VB200_OUT_ATTENTION"):
        _packed(model, ok, L.OUT_TASK_HEADS | L.OUT_ATTENTION)
    with pytest.raises(L.VilbertB200Error, match=r"error -1: .*n_tokens 0"):
        model.forward_packed(torch.zeros(4, dtype=torch.long).cuda(), torch.zeros(5, model._dims["v_feature_size"]).cuda(),
                             torch.zeros(5, 5).cuda(), None, torch.zeros(2, 1, dtype=torch.long).cuda(), [0, 4], [3, 2])
    with pytest.raises(L.VilbertB200Error, match=r"error -1: .*T=257"):
        _packed(model, support.batch(model, [(256, 3)], seed=22), vb.OUT_TASK_HEADS)
    with pytest.raises(L.VilbertB200Error, match=r"error -1: .*capacity"):
        _packed(model, ok, vb.OUT_TASK_HEADS, max_tokens=4)
    x = support.engine(tiny_oracle, compute_dtype="fp32x")
    try:
        with pytest.raises(L.VilbertB200Error, match=r"error -1: .*fp32x"):
            _packed(x, ok, vb.OUT_TASK_HEADS)
    finally:
        x.close()


@pytest.mark.parametrize("block_n", [64, 128])
def test_linear_device_row_count(block_n):
    """vb200_linear_rows at capacity M = 1024 with m_rows = 300: rows < 300 equal vb200_linear at M = 300 bit for bit, and every
    tile that starts at or past row 300 (rows >= 384) is skipped -- those rows keep the sentinel."""
    from vilbert_b200 import _lib as L
    lib = L.load()
    M, N, K, m = 1024, 256, 192, 300
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, K, generator=g, device="cuda").half()
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.05).half()
    b = torch.randn(N, generator=g, device="cuda")
    rows = torch.tensor([m], dtype=torch.int32, device="cuda")
    y = torch.full((M, N), 12345.0, device="cuda")
    ref = torch.empty(m, N, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.vb200_linear_rows(x.data_ptr(), K, w.data_ptr(), K, b.data_ptr(), 1, None, 0, y.data_ptr(), N, M, N, K, block_n, 1,
                                  rows.data_ptr(), st), None)
    L.check(lib.vb200_linear(x.data_ptr(), K, w.data_ptr(), K, b.data_ptr(), None, 0, None, None, 1e-12, 1, None, 0, ref.data_ptr(), N,
                             m, N, K, block_n, 0, 1, 0, None, st), None)
    torch.cuda.synchronize()
    assert torch.equal(y[:m], ref)
    assert bool((y[384:] == 12345.0).all())


def _worker_requests(model):
    """One request each of VQA, GQA, SNLI-VE, retrieval, NLVR2 and grounding, text padded to 37 like the worker's tokenizer."""
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    reqs = []
    for j, (task, n_img, V, words) in enumerate([("1", 1, 37, 7), ("15", 1, 101, 20), ("13", 1, 12, 35), ("7", 3, 50, 11),
                                                  ("12", 2, 80, 15), ("11", 1, 23, 4)]):
        g = torch.Generator().manual_seed(100 + j)
        q = torch.zeros(1, 37, dtype=torch.long)
        q[0, :words] = torch.randint(1000, vocab, (words,), generator=g)
        im = torch.zeros(1, 37, dtype=torch.long)
        im[0, :words] = 1
        f = torch.relu(torch.randn(n_img, V, F, generator=g)) * 1.5
        x1, y1 = torch.rand(n_img, V, generator=g) * 0.7, torch.rand(n_img, V, generator=g) * 0.7
        s = torch.stack([x1, y1, x1 + 0.2, y1 + 0.2, torch.full_like(x1, 0.04)], dim=-1)
        infos = [{"image_width": 640, "image_height": 480}] * n_img
        reqs.append((q.cuda(), f.cuda(), s.cuda(), torch.zeros(1, 37, dtype=torch.long).cuda(), im.cuda(),
                     torch.ones(n_img, V, dtype=torch.uint8).cuda(), None, torch.tensor([[int(task)]]).cuda(), task, infos))
    return reqs


def test_prediction_packed_matches_prediction(full):
    """One engine call for six tasks with different text lengths and region counts; every answer equals prediction()'s for that
    request alone (labels / boxes in the same order, confidences within 1e-4)."""
    from vilbert_b200 import worker_api as W
    W.model = full
    reqs = _worker_requests(full)
    calls = []
    orig = full.forward_packed

    def counted(*a, **kw):
        calls.append(1)
        return orig(*a, **kw)
    full.forward_packed = counted
    try:
        got = W.prediction_packed(reqs)
    finally:
        del full.forward_packed
    assert len(calls) == 1
    for r, ans in zip(reqs, got):
        want = W.prediction(*r)
        if isinstance(want, list):           # grounding: boxes
            assert [{k: v for k, v in a.items() if k != "confidence"} for a in ans] == \
                   [{k: v for k, v in a.items() if k != "confidence"} for a in want]
            assert [a["confidence"] for a in ans] == pytest.approx([a["confidence"] for a in want], abs=1e-2)
        else:
            assert ans["top3_answer"] == want["top3_answer"], r[8]
            assert ans["top3_confidence"] == pytest.approx(want["top3_confidence"], abs=1e-4), r[8]
