"""Attention maps by selection (vb200_set_option "attention_entries" / "attention_heads", from_pretrained(attention_entries=...,
attention_heads=...)).  `-m gpu` only.

A selected entry is the probability output of a forward with every map, bit for bit; a head-mean entry is the float32 left-to-right
sum of that forward's per-head maps divided by the head count, bit for bit; every packed sample equals a dense forward of that sample
alone.  Logits, taps and the launch list are unchanged apart from the probability launches of the selected entries.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16", "fp32x")
TOL_ATTN = 5e-3            # engine (fp16) vs the fp32 oracle's attention probabilities (tests/test_gpu_round2.py)
NAN = float("nan")


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, MODES, return_attention=True)


class _Selected:
    """The model's map selection set to (entries, heads) inside the block, back to every entry / every head after it."""

    def __init__(self, model, entries=None, heads="all"):
        from vilbert_b200 import model as M
        self.model, self.heads = model, heads
        self.mask = None if entries is None else M.attention_mask_bits(entries)

    def __enter__(self):
        if self.mask is not None:
            self.model.set_option("attention_entries", self.mask)
        self.model.set_option("attention_heads", 1 if self.heads == "mean" else 0)
        return self.model

    def __exit__(self, *exc):
        n = len(self.model.attention_selection()[0])
        self.model.set_option("attention_entries", (1 << n) - 1)
        self.model.set_option("attention_heads", 0)


def _kinds(model):
    return model.attention_selection()[0]


def _selections(model):
    """Named entry lists: single entries, the first and last, the connection-layer directions only, one direction of a layer."""
    kinds = _kinds(model)
    n = len(kinds)
    conn = [e for e, k in enumerate(kinds) if k >= 2]
    t2i = [e for e, k in enumerate(kinds) if k == 2]
    i2t = [e for e, k in enumerate(kinds) if k == 3]
    return {"first": [0], "middle": [n // 2], "first_last": [0, n - 1], "connection": conn, "one_t2i": [t2i[1]],
            "one_i2t": [i2t[-1]], "all": list(range(n))}


def _positions(kinds):
    """(position, direction or None) of every full-list entry in element 9."""
    out, pos, e = [], 0, 0
    while e < len(kinds):
        if kinds[e] == 2:
            out += [(pos, 0), (pos, 1)]
            e += 2
        else:
            out.append((pos, None))
            e += 1
        pos += 1
    return out


def _entry(attn, where):
    pos, d = where
    return attn[pos] if d is None else attn[pos][d]


def _dense(model, inp, maps=True):
    out = model(*inp, output_all_attention_masks=maps, debug_taps=True)
    torch.cuda.synchronize()
    return out


def _same_outputs(a, b):
    """Logits and taps of two (10-tuple, taps) results are bit-identical."""
    for x, y in zip(a[0][:9], b[0][:9]):
        assert (x is None) == (y is None)
        if x is not None:
            assert torch.equal(x, y)
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), k


def _np_mean(maps, axis):
    """float32 sum over the head axis, left to right, divided by the head count -- the head-mean kernel's definition."""
    m = np.ascontiguousarray(np.moveaxis(maps.cpu().numpy(), axis, 0))
    s = m[0].copy()
    for h in range(1, m.shape[0]):
        s = (s + m[h]).astype(np.float32)
    return np.expand_dims(s / np.float32(m.shape[0]), axis)


def _check_selected(attn, full, kinds, entries, mean, axis=1):
    """attn (element 9 under a selection) against full (every entry, every head): None where not selected, the full entry (or its
    head mean) where selected."""
    assert len(attn) == len(full) == sum(1 for k in kinds if k != 3)
    for e, where in enumerate(_positions(kinds)):
        got, ref = _entry(attn, where), _entry(full, where)
        if e not in entries:
            assert got is None, e
            continue
        pairs = list(zip(got, ref)) if isinstance(ref, list) else [(got, ref)]
        for g, r in pairs:
            if mean:
                assert g.shape[axis] == 1
                assert np.array_equal(g.cpu().numpy(), _np_mean(r, axis)), e
            else:
                assert torch.equal(g, r), e


# ------------------------------------------------------------------------------------------------------------ dense, per head
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,pad", [(2, 0), (3, 2)])
def test_dense_selected_entries_bitwise(tiny, tiny_oracle, mode, B, pad):
    L = support.lib()
    model = tiny[mode]
    inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, B, 14, 11, seed=300 + B, pad=pad)]
    full = _dense(model, inp)
    plain = _dense(model, inp, maps=False)
    _same_outputs(full, plain)
    kinds = _kinds(model)
    n_plain = model.plan_info(B, 14, 11, L.OUT_TASK_HEADS)[0]
    for name, entries in _selections(model).items():
        with _Selected(model, entries):
            out = _dense(model, inp)
            _check_selected(out[0][9], full[0][9], kinds, entries, mean=False)
            _same_outputs(out, plain)
            # 16-bit modes: one probability launch per selected entry; fp32x: the context launches write them
            n = model.plan_info(B, 14, 11, L.OUT_TASK_HEADS | L.OUT_ATTENTION)[0]
            assert n == n_plain + (len(entries) if mode != "fp32x" else 0), name


# ------------------------------------------------------------------------------------------------------------ dense, head mean
@pytest.mark.parametrize("mode", MODES)
def test_dense_head_mean_bitwise(tiny, tiny_oracle, mode):
    L = support.lib()
    model = tiny[mode]
    inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 3, 20, 12, seed=61, pad=2)]
    full = _dense(model, inp)
    plain = _dense(model, inp, maps=False)
    kinds = _kinds(model)
    n_plain = model.plan_info(3, 20, 12, L.OUT_TASK_HEADS)[0]
    for entries in (list(range(len(kinds))), _selections(model)["connection"], [0, len(kinds) - 1]):
        with _Selected(model, entries, "mean"):
            out = _dense(model, inp)
            _check_selected(out[0][9], full[0][9], kinds, entries, mean=True)
            _same_outputs(out, plain)
            n = model.plan_info(3, 20, 12, L.OUT_TASK_HEADS | L.OUT_ATTENTION)[0]
            # one head-mean launch per selected entry (in fp32x on top of the context launches)
            assert n == n_plain + len(entries)


def test_head_mean_vs_oracle(tiny, tiny_oracle, parity_log):
    """The fp32 oracle's maps averaged over heads, at the tolerance of the per-head maps."""
    inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 3, 20, 12, seed=61, pad=2)]
    ref = tiny_oracle(*[t.cpu() for t in inp], output_all_attention_masks=True)[9]
    model = tiny["fp16"]
    with _Selected(model, None, "mean"):
        attn = _dense(model, inp)[0][9]
    worst = 0.0
    for a, r in zip(attn, ref):
        for x, y in (zip(a, r) if isinstance(r, tuple) else [(a, r)]):
            assert tuple(x.shape) == (y.shape[0], 1) + tuple(y.shape[2:])
            worst = max(worst, float((x.cpu() - y.mean(1, keepdim=True)).abs().max()))
            assert float((x.sum(-1) - 1).abs().max()) < 1e-4
    parity_log(test="attn_probs_head_mean_tiny_fp16", max_abs_err=worst)
    assert worst < TOL_ATTN, worst


# ------------------------------------------------------------------------------------------------------------ packed
def _packed(model, samples, maps=True, sync=True):
    L = support.lib()
    out = model.forward_packed(*support.packed_sample_args(samples), select=L.OUT_TASK_HEADS, debug_taps=True, output_all_attention_masks=maps)
    if sync:
        torch.cuda.synchronize()
    return out


def _alone(model, smp):
    return support.dense_alone(model, smp, select=support.lib().OUT_TASK_HEADS, output_all_attention_masks=True)[9]


def _check_packed_vs_alone(attn, alone, kinds, entries):
    """Each packed sample's selected maps == the dense forward of that sample alone under the same selection."""
    for e, where in enumerate(_positions(kinds)):
        got = _entry(attn, where)
        if e not in entries:
            assert got is None
            continue
        for b, ref in enumerate(alone):
            assert torch.equal(got[b], _entry(ref, where)[0]), (e, b)


LENS = [(1, 40), (31, 1), (12, 64), (5, 17)]


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_packed_selection(tiny, mode):
    model = tiny[mode]
    samples = support.batch(model, LENS, seed=900)
    full = _packed(model, samples)
    plain = _packed(model, samples, maps=False)
    kinds = _kinds(model)
    for heads in ("all", "mean"):
        for name in ("first_last", "connection", "one_i2t"):
            entries = _selections(model)[name]
            with _Selected(model, entries, heads):
                out = _packed(model, samples)
                _check_selected(out[0][9], full[0][9], kinds, entries, mean=heads == "mean", axis=0)
                _same_outputs(out, plain)
                if heads == "mean":
                    _check_packed_vs_alone(out[0][9], [_alone(model, s) for s in samples], kinds, entries)


def test_regions_packed_selection(tiny):
    L = support.lib()
    model = tiny["bf16"]
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = []
    for i, (tin, n) in enumerate([(7, 3), (1, 30), (20, 9)]):
        g = torch.Generator().manual_seed(70 + i)
        q, seg = torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g)
        f = torch.relu(torch.randn(n, F, generator=g))
        x1, y1 = torch.rand(n, generator=g) * 400, torch.rand(n, generator=g) * 300
        bx = torch.stack([x1, y1, x1 + 100, y1 + 80], 1)
        imgs.append((q, seg, f, bx, torch.tensor([640.0, 480.0]), i + 1))
    cat = lambda k: torch.cat([im[k] for im in imgs], dim=0).cuda()

    def run(maps=True):
        (out, _) = model.forward_regions_packed(cat(0), cat(1), torch.tensor([[im[5]] for im in imgs]).cuda(), cat(2), cat(3),
                                                torch.stack([im[4] for im in imgs]).cuda(), [len(im[0]) for im in imgs],
                                                [im[2].shape[0] for im in imgs], select=L.OUT_TASK_HEADS,
                                                output_all_attention_masks=maps)
        torch.cuda.synchronize()
        return out

    full = run()
    kinds = _kinds(model)
    for heads in ("all", "mean"):
        entries = _selections(model)["first_last"] + _selections(model)["one_t2i"]
        with _Selected(model, entries, heads):
            out = run()
            _check_selected(out[9], full[9], kinds, entries, mean=heads == "mean", axis=0)
            for x, y in zip(out[:9], run(maps=False)[:9]):
                assert (x is None and y is None) or torch.equal(x, y)


def test_long_rows_head_mean(tiny_oracle):
    """Rows past 256 (max_rows_per_sample 1024): the context comes from the streaming kernels, the maps from the fp32 kernel with
    1024-key accumulators; each packed sample equals its dense forward alone, and the dense mean equals the per-head maps' mean."""
    from oracle import vilbert_ref as R
    oracle = R.build(R.tiny_config(max_position_embeddings=1024), seed=7, num_labels=200)
    model = support.engine(oracle, compute_dtype="bf16", max_rows_per_sample=1024, return_attention=True)
    try:
        kinds = _kinds(model)
        samples = support.batch(model, [(300, 20), (10, 1024), (3, 3)], seed=50)
        full_alone = [_alone(model, s) for s in samples]
        entries = list(range(len(kinds)))
        with _Selected(model, entries, "mean"):
            out = _packed(model, samples)
            alone = [_alone(model, s) for s in samples]
            _check_packed_vs_alone(out[0][9], alone, kinds, entries)
            for a, f in zip(alone, full_alone):
                _check_selected(a, f, kinds, entries, mean=True)
    finally:
        model.close()


def test_full_model_bf16_selection(full_oracle):
    from oracle import vilbert_ref as R
    model = support.engine(full_oracle, compute_dtype="bf16", return_attention=True)
    try:
        inp = [t.cuda() for t in R.make_inputs(2, 30, 36, seed=808, pad_regions=3)]
        full = _dense(model, inp)
        kinds = _kinds(model)
        assert len(kinds) == 30
        for name in ("connection", "one_t2i", "first_last"):
            entries = _selections(model)[name]
            with _Selected(model, entries):
                _check_selected(_dense(model, inp)[0][9], full[0][9], kinds, entries, mean=False)
        with _Selected(model, _selections(model)["connection"], "mean"):
            out = _dense(model, inp)[0][9]
            _check_selected(out, full[0][9], kinds, _selections(model)["connection"], mean=True)
            assert out[6][0].shape == (2, 1, 31, 36) and out[6][1].shape == (2, 1, 36, 31) and out[0] is None
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------------ layouts, sentinel
def test_layouts_follow_selection(tiny):
    model = tiny["fp16"]
    kinds = _kinds(model)
    full, full_total = model.attention_layout(2, 9, 7)
    full_p, _ = model.attention_layout_packed([3, 9], [7, 2])
    for heads in ("all", "mean"):
        entries = _selections(model)["first_last"] + _selections(model)["connection"][:3]
        entries = sorted(set(entries))
        with _Selected(model, entries, heads):
            k, where = model.attention_selection()
            assert k == kinds and [w for w in where if w >= 0] == list(range(len(entries)))
            assert [e for e, w in enumerate(where) if w >= 0] == entries
            lay, total = model.attention_layout(2, 9, 7)
            assert len(lay) == len(entries)
            off = 0
            for (h, lq, lk, kind, o), e in zip(lay, entries):
                fh, flq, flk, fkind, _ = full[e]
                assert (lq, lk, kind) == (flq, flk, fkind) and h == (1 if heads == "mean" else fh) and o == off
                off += 2 * h * lq * lk
            assert total == off
            lay_p, total_p = model.attention_layout_packed([3, 9], [7, 2])
            assert len(lay_p) == len(entries)
            T, V = [4, 10], [7, 2]
            off = 0
            for (h, kind, o), e in zip(lay_p, entries):
                assert kind == full_p[e][1] and h == (1 if heads == "mean" else full_p[e][0]) and o == off
                lq, lk = {0: (T, T), 1: (V, V), 2: (T, V), 3: (V, T)}[kind]
                off += h * sum(a * b for a, b in zip(lq, lk))
            assert total_p == off
            v = C.c_int64()
            L = support.lib()
            L.check(L.load().vb200_model_dim(model._handle, b"attention_entries", C.byref(v)), model._handle)
            assert v.value == sum(1 << e for e in entries)
            L.check(L.load().vb200_model_dim(model._handle, b"attention_heads", C.byref(v)), model._handle)
            assert v.value == (1 if heads == "mean" else 0)
    assert model.attention_layout(2, 9, 7) == (full, full_total)


def test_every_float_written(tiny, tiny_oracle):
    """A NaN-filled buffer has no NaN left after a dense or packed forward under a selection."""
    L = support.lib()
    model = tiny["bf16"]
    dev = torch.device("cuda", 0)
    entries = _selections(model)["first_last"] + _selections(model)["one_t2i"]
    for heads in ("all", "mean"):
        with _Selected(model, entries, heads):
            q, f, s, seg, im, vm, co, tk = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 3, 9, 7, seed=5, pad=2)]
            outs, o, select = model._alloc_outputs(3, 9, 7, L.OUT_TASK_HEADS, False, True, dev)
            outs["attention_probs"].fill_(NAN)
            inp = L.Inputs(3, 9, 7, q.data_ptr(), f.data_ptr(), s.data_ptr(), seg.data_ptr(), im.data_ptr(), vm.data_ptr(), None,
                           tk.data_ptr())
            model._call("vb200_forward_slot", C.byref(inp), C.byref(o), select, 0)
            torch.cuda.synchronize()
            assert not torch.isnan(outs["attention_probs"]).any()

            samples = support.batch(model, LENS, seed=11)
            qp, fp, sp, segp, tkp, nt, nv = support.packed_sample_args(samples)
            _, total = model.attention_layout_packed(nt, nv)
            flat = torch.full((total,), NAN, device=dev)
            rows_t = sum(nt) + len(nt)
            pouts, po = model._alloc_packed_outputs(len(nt), rows_t, sum(nv), L.OUT_TASK_HEADS, False, dev)
            po.attention_probs = flat.data_ptr()
            from vilbert_b200 import model as M
            pin = L.PackedInputs(len(nt), 0, 0, M._int32s(nt), M._int32s(nv), qp.data_ptr(), segp.data_ptr(), fp.data_ptr(),
                                 sp.data_ptr(), tkp.data_ptr())
            model._call("vb200_forward_packed", C.byref(pin), C.byref(po), L.OUT_TASK_HEADS | L.OUT_ATTENTION_PACKED, 0)
            torch.cuda.synchronize()
            assert not torch.isnan(flat).any()


# ------------------------------------------------------------------------------------------------------------ changing the selection
def test_change_selection_between_calls(tiny_oracle):
    model = support.engine(tiny_oracle, compute_dtype="fp16", return_attention=True)
    try:
        inp = [t.cuda() for t in support.tiny_inputs(tiny_oracle, 2, 8, 6, seed=3)]
        kinds = _kinds(model)
        full = _dense(model, inp)[0][9]
        plans = support.n_plans(model)
        sel = _selections(model)
        with _Selected(model, sel["connection"]):
            _check_selected(_dense(model, inp)[0][9], full, kinds, sel["connection"], mean=False)
        assert support.n_plans(model) == plans + 1
        _check_selected(_dense(model, inp)[0][9], full, kinds, list(range(len(kinds))), mean=False)
        assert support.n_plans(model) == plans + 1                   # the default selection's plan is reused
        with _Selected(model, sel["connection"], "mean"):
            _check_selected(_dense(model, inp)[0][9], full, kinds, sel["connection"], mean=True)
        assert support.n_plans(model) == plans + 2
        with _Selected(model, sel["connection"]):
            _dense(model, inp)
        assert support.n_plans(model) == plans + 2                   # and so is the first selection's

        # unsynchronised back-to-back packed calls under different selections, each into its own buffer
        samples = support.batch(model, LENS, seed=21)
        pfull = _packed(model, samples)[0][9]
        a = model.forward_packed(*support.packed_sample_args(samples), debug_taps=True, output_all_attention_masks=True)
        model.set_option("attention_entries", 1 << 3)
        b = model.forward_packed(*support.packed_sample_args(samples), debug_taps=True, output_all_attention_masks=True)
        model.set_option("attention_heads", 1)
        c = model.forward_packed(*support.packed_sample_args(samples), debug_taps=True, output_all_attention_masks=True)
        torch.cuda.synchronize()
        _check_selected(a[0][9], pfull, kinds, list(range(len(kinds))), mean=False, axis=0)
        _check_selected(b[0][9], pfull, kinds, [3], mean=False, axis=0)
        _check_selected(c[0][9], pfull, kinds, [3], mean=True, axis=0)
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------------ rejections
def test_rejections(tiny):
    L = support.lib()
    model = tiny["fp16"]
    n = len(_kinds(model))
    for key, value, msg in (("attention_entries", 0, "attention_entries"), ("attention_entries", 1 << n, "attention_entries"),
                            ("attention_entries", (1 << n) | 1, "attention_entries"), ("attention_entries", -1, "attention_entries"),
                            ("attention_heads", 2, "attention_heads"), ("attention_heads", -1, "attention_heads")):
        rc = L.load().vb200_set_option(model._handle, key.encode(), value)
        assert rc == -1, (key, value)                          # VB200_ERR_INVALID
        assert msg in L.load().vb200_last_error(model._handle).decode(), (key, value)
    v = C.c_int64()
    L.check(L.load().vb200_model_dim(model._handle, b"attention_entries", C.byref(v)), model._handle)
    assert v.value == (1 << n) - 1
    L.check(L.load().vb200_model_dim(model._handle, b"attention_heads", C.byref(v)), model._handle)
    assert v.value == 0


def test_pretraining_engine_accepts_selection():
    import vilbert_b200 as vb
    from oracle import pretraining_ref as P
    from oracle import vilbert_ref as R
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    full = vb.BertForMultiModalPreTraining.from_pretrained(oracle.state_dict(), config=cfg, return_attention=True).eval().cuda(0)
    n = len(full.attention_selection()[0])
    sel = vb.BertForMultiModalPreTraining.from_pretrained(oracle.state_dict(), config=cfg, return_attention=True,
                                                          attention_entries=[0, n - 1], attention_heads="mean").eval().cuda(0)
    try:
        inp = list(R.make_inputs(2, 10, 6, seed=4, vocab_size=cfg.vocab_size))
        inp[1] = inp[1][..., :cfg.v_feature_size].contiguous()
        args = [t.cuda() for t in inp[:6]]
        a = full(*args, output_all_attention_masks=True)
        b = sel(*args, output_all_attention_masks=True)
        torch.cuda.synchronize()
        for x, y in zip(a[:3], b[:3]):
            assert torch.equal(x, y)
        kinds = _kinds(sel)
        _check_selected(b[3], a[3], kinds, [0, n - 1], mean=True)
    finally:
        full.close()
        sel.close()
