"""Layer states by selection (VB200_OUT_LAYER_STATES, from_pretrained(state_entries=..., state_rows=...), output_layer_states=True).
`-m gpu` only.

Every entry is the fp32 residual-stream state after a step that writes a stream, so it matches the oracle's ``collect`` states; the
last text / image entries are the sequence_output taps bit for bit; first and mean are exact functions of the rows; each packed sample
equals a dense forward of that sample alone; and nothing else a forward computes changes.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import support

pytestmark = pytest.mark.gpu

ROWS = {"all": 0, "first": 1, "mean": 2}
TOL = {"fp16": 1e-2, "bf16": 3.5e-2}     # rel_err of oracle/fp64.py against the fp32 oracle, the model tests' logit tolerances


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    yield from support.engines(tiny_oracle, ("fp16", "bf16", "fp32x"), return_attention=True)


class _States:
    """The model's state selection set inside the block, back to every entry, every row after it."""

    def __init__(self, model, entries=None, rows="all"):
        from vilbert_b200 import model as M
        self.model, self.rows = model, rows
        self.mask = None if entries is None else M.entry_mask_bits(entries, "state_entries")

    def __enter__(self):
        if self.mask is not None:
            self.model.set_option("state_entries", self.mask)
        self.model.set_option("state_rows", ROWS[self.rows])
        return self.model

    def __exit__(self, *exc):
        self.model.set_option("state_entries", (1 << len(self.model.state_selection()[0])) - 1)
        self.model.set_option("state_rows", 0)


def _oracle_entries(oracle, inp):
    """The full state list from the oracle's collect: embeddings, then per step its text state (T, C) before its image state (V, C)."""
    collect = {}
    with torch.no_grad():
        oracle(*inp, compute_pretraining_heads=False, collect=collect)
    t, v = collect["emb"]
    out = [t, v]
    for step in oracle.bert.encoder.schedule():
        t, v = collect[step]
        if step[0] != "V":
            out.append(t)
        if step[0] != "T":
            out.append(v)
    return out


def _dense(model, inp, states=True, **kw):
    out = model(*[t.cuda() for t in inp], debug_taps=True, output_layer_states=states, **kw)
    torch.cuda.synchronize()
    return out


def _last(model):
    kinds = model.state_selection()[0]
    return max(e for e, k in enumerate(kinds) if k == 0), max(e for e, k in enumerate(kinds) if k == 1)


def _np_mean(rows):
    """float32 sum of the rows in increasing order, one rounding per add, divided once by the count (NaN without a row)."""
    if len(rows) == 0:
        return np.full(rows.shape[1], np.nan, np.float32)
    acc = np.zeros(rows.shape[1], np.float32)
    for r in rows:
        acc = np.add(acc, r, dtype=np.float32)
    return np.divide(acc, np.float32(len(rows)), dtype=np.float32)


def _eq(a, b):
    assert torch.equal(torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu())


def _eq_nan(a, b):
    a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
    assert torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))


# ------------------------------------------------------------------------------------------------------------ oracle parity
@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_oracle_parity_tiny(tiny, tiny_oracle, mode, parity_log):
    from oracle import fp64 as X
    model = tiny[mode]
    inp = support.tiny_inputs(tiny_oracle, 3, 14, 20, seed=31, pad=4)
    _, states = _dense(model, inp)
    ref = _oracle_entries(tiny_oracle, inp)
    assert len(states) == len(ref) == 32
    errs = [X.rel_err(s, r) for s, r in zip(states, ref)]
    parity_log(test=f"layer_states_tiny_{mode}", max_rel_err=max(errs))
    assert max(errs) < TOL[mode], errs


def test_oracle_parity_fp32x_vs_fp64(tiny, tiny_oracle, parity_log):
    from oracle import fp64 as X
    inp = support.tiny_inputs(tiny_oracle, 2, 12, 17, seed=32, pad=3)
    _, states = _dense(tiny["fp32x"], inp)
    ref = _oracle_entries(X.fp64(tiny_oracle), inp)
    errs = [X.rel_err(s, r) for s, r in zip(states, ref)]
    parity_log(test="layer_states_fp32x_vs_fp64", max_rel_err=max(errs), bound=X.BOUNDS["states"])
    assert max(errs) < X.BOUNDS["states"], errs


def test_oracle_parity_full_model_bf16(full_oracle, parity_log):
    from oracle import fp64 as X
    from oracle import vilbert_ref as R
    model = support.engine(full_oracle, compute_dtype="bf16", return_attention=True)
    try:
        inp = list(R.make_inputs(2, 20, 36, seed=33, pad_regions=5))
        _, states = _dense(model, inp)
        ref = _oracle_entries(full_oracle, inp)
        errs = [X.rel_err(s, r) for s, r in zip(states, ref)]
        parity_log(test="layer_states_full_bf16", max_rel_err=max(errs))
        assert max(errs) < TOL["bf16"], errs
        # per-sample identity on the full model: packed regions of each sample vs that sample alone
        samples = support.batch(model, [(9, 30), (20, 12)], seed=34)
        for rows in ROWS:
            with _States(model, rows=rows):
                _check_packed_vs_alone(model, samples, rows)
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------------ exact reductions
@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_reductions_dense_exact(tiny, tiny_oracle, mode):
    model = tiny[mode]
    inp = support.tiny_inputs(tiny_oracle, 3, 14, 20, seed=41, pad=6)
    (_, taps), rows = _dense(model, inp)
    lt, lv = _last(model)
    _eq(rows[lt], taps["sequence_output_t"])
    _eq(rows[lv], taps["sequence_output_v"])
    with _States(model, rows="first"):
        (_, _), first = _dense(model, inp)
    with _States(model, rows="mean"):
        (_, _), mean = _dense(model, inp)
    task = torch.ones(3, model._dims["task_specific_tokens"], dtype=torch.long)
    t_real = torch.cat([task, inp[4].long()], 1).bool()                                # task token + input_mask
    v_real = inp[5].bool()
    kinds = model.state_selection()[0]
    for e, k in enumerate(kinds):
        _eq(first[e], rows[e][:, 0])
        real = t_real if k == 0 else v_real
        r = rows[e].cpu().numpy()
        ref = np.stack([_np_mean(r[b][real[b].numpy()]) for b in range(3)])
        _eq(mean[e], ref)


def _packed(model, samples, states=True, sync=True, **kw):
    L = support.lib()
    out = model.forward_packed(*support.packed_sample_args(samples), select=L.OUT_TASK_HEADS, debug_taps=True, output_layer_states=states, **kw)
    if sync:
        torch.cuda.synchronize()
    return out


def _check_packed_vs_alone(model, samples, rows, regions=False):
    """Every reduction of every packed sample == the dense forward of that sample alone (forward_packed, or with ``regions`` the
    detector-output pair forward_regions_packed / forward_regions)."""
    if regions:
        got, alone = _regions(model, samples)
    else:
        (_, got) = _packed(model, samples)
        alone = [support.dense_alone(model, s, select=support.lib().OUT_TASK_HEADS, output_layer_states=True)[1] for s in samples]
    for e, entry in enumerate(got):
        for b, ref in enumerate(alone):
            _eq_nan(entry[b], ref[e][0])      # rows: sample b's [L_b, H] view vs [1, L_b, H]; first / mean: [H] vs [1, H]


LENS = [(1, 40), (31, 1), (12, 64), (5, 17)]


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
def test_reductions_packed_exact(tiny, mode):
    model = tiny[mode]
    samples = support.batch(model, LENS, seed=500)
    (_, taps), rows = _packed(model, samples)
    lt, lv = _last(model)
    _eq(torch.cat(rows[lt]), taps["sequence_output_t"])
    _eq(torch.cat(rows[lv]), taps["sequence_output_v"])
    with _States(model, rows="first"):
        (_, first) = _packed(model, samples)
    with _States(model, rows="mean"):
        (_, mean) = _packed(model, samples)
    for e in range(len(rows)):
        _eq(first[e], torch.stack([x[0] for x in rows[e]]))
        _eq(mean[e], np.stack([_np_mean(x.cpu().numpy()) for x in rows[e]]))


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("rows", tuple(ROWS))
def test_packed_per_sample_identity(tiny, mode, rows):
    model = tiny[mode]
    with _States(model, rows=rows):
        _check_packed_vs_alone(model, support.batch(model, LENS, seed=600), rows)


def test_packed_per_sample_identity_past_256_rows(tiny):
    model = tiny["bf16"]
    model.set_option("max_rows_per_sample", 512)
    try:
        for rows in ROWS:
            with _States(model, rows=rows):
                _check_packed_vs_alone(model, support.batch(model, [(150, 300), (3, 512), (40, 20)], seed=650), rows)
    finally:
        model.set_option("max_rows_per_sample", 256)


def _regions(model, imgs_lens):
    L = support.lib()
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = []
    for i, (tin, n) in enumerate(imgs_lens):
        g = torch.Generator().manual_seed(70 + i)
        q, seg = torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g)
        f = torch.relu(torch.randn(n, F, generator=g))
        x1, y1 = torch.rand(n, generator=g) * 400, torch.rand(n, generator=g) * 300
        imgs.append((q, seg, f, torch.stack([x1, y1, x1 + 100, y1 + 80], 1), torch.tensor([640.0, 480.0]), i + 1))
    cat = lambda k: torch.cat([im[k] for im in imgs], dim=0).cuda()
    (_, got) = model.forward_regions_packed(cat(0), cat(1), torch.tensor([[im[5]] for im in imgs]).cuda(), cat(2), cat(3),
                                            torch.stack([im[4] for im in imgs]).cuda(), [len(im[0]) for im in imgs],
                                            [im[2].shape[0] for im in imgs], select=L.OUT_TASK_HEADS, output_layer_states=True)
    alone = []
    for q, seg, f, bx, wh, task in imgs:
        (_, st) = model.forward_regions(q[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
                                        torch.tensor([[task]]).cuda(), f[None].cuda(), bx[None].cuda(), wh[None].cuda(),
                                        select=L.OUT_TASK_HEADS, output_layer_states=True)
        alone.append(st)
    torch.cuda.synchronize()
    return got, alone


@pytest.mark.parametrize("mode", ("fp16", "bf16"))
@pytest.mark.parametrize("rows", tuple(ROWS))
def test_regions_packed_per_sample_identity(tiny, mode, rows):
    model = tiny[mode]
    with _States(model, rows=rows):
        _check_packed_vs_alone(model, [(7, 3), (1, 30), (20, 9)], rows, regions=True)


# ------------------------------------------------------------------------------------------------------------ no side effects
def _same(a, b):
    for x, y in zip(a[0][:9], b[0][:9]):
        assert (x is None) == (y is None)
        if x is not None:
            _eq(x, y)
    for k in a[1]:
        _eq(a[1][k], b[1][k])


@pytest.mark.parametrize("mode", ("fp16", "bf16", "fp32x"))
def test_selection_and_no_side_effects_dense(tiny, tiny_oracle, mode):
    model = tiny[mode]
    inp = support.tiny_inputs(tiny_oracle, 2, 10, 15, seed=51, pad=2)
    plain = _dense(model, inp, states=False, output_all_attention_masks=True)
    res, every = _dense(model, inp, output_all_attention_masks=True)
    _same(res, plain)
    for a, b in zip(res[0][9], plain[0][9]):
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            _eq(x, y)
    lt, lv = _last(model)
    for sel in ([0, 1], [3, 17], [lt], [lv], [0, lt, lv]):
        with _States(model, sel):
            r, s = _dense(model, inp)
            _same(r, plain)
            for e, x in enumerate(s):
                assert (x is None) == (e not in sel)
                if x is not None:
                    _eq(x, every[e])


def test_no_side_effects_packed(tiny):
    model = tiny["fp16"]
    samples = support.batch(model, LENS, seed=700)
    plain = _packed(model, samples, states=False, output_all_attention_masks=True)
    res, every = _packed(model, samples, output_all_attention_masks=True)
    _same(res, plain)
    with _States(model, [2, 9, 30]):
        r, s = _packed(model, samples)
        _same(r, _packed(model, samples, states=False))
        for e, x in enumerate(s):
            assert (x is None) == (e not in (2, 9, 30))
            if x is not None:
                for a, b in zip(x, every[e]):
                    _eq(a, b)


# ------------------------------------------------------------------------------------------------------------ pruning
def test_pruning(tiny):
    L = support.lib()
    model = tiny["fp16"]
    lt, lv = _last(model)
    base_n, base_f = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION)
    tap_n, tap_f = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LINGUISIC_LOGIT)   # a per-row text head un-prunes text
    for sel in ([0], [1, 5, 20], [lv - 1, lv - 2]):   # lv - 1, lv - 2: the last connection layer's image and text states
        with _States(model, sel):
            n, f = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LAYER_STATES)
            assert n == base_n + len(sel) and f == base_f, sel
    kinds = model.state_selection()[0]
    with _States(model, rows="mean"):
        n_all, f_all = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LAYER_STATES)
    with _States(model, [lt]):
        n_t, f_t = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LAYER_STATES)
    with _States(model, [lv]):
        n_v, f_v = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LAYER_STATES)
    with _States(model, [lt, lv]):
        n_b, f_b = model.plan_info(4, 12, 20, L.OUT_VIL_PREDICTION | L.OUT_LAYER_STATES)
    # un-pruning a stream adds FLOPs; each last entry only un-prunes its own stream, both together add both
    assert f_t > base_f and f_v > base_f and f_b > max(f_t, f_v)
    assert abs((f_b - base_f) - ((f_t - base_f) + (f_v - base_f))) < 1e-6 * f_b
    # the text tail un-pruned by its last entry costs what a per-row text head's un-pruning costs (minus that head's own FLOPs)
    assert f_t - base_f <= tap_f - base_f
    # every entry: both tails un-pruned as by the two last entries, one launch per entry
    assert f_all == f_b and n_all == n_b + len(kinds) - 2


# ------------------------------------------------------------------------------------------------------------ plans and buffers
def test_plans_and_buffers(tiny, tiny_oracle):
    L = support.lib()
    model = tiny["bf16"]
    model.set_option("max_plans", 1024)           # no eviction hides a plan built or reused below
    samples = support.batch(model, LENS, seed=800)
    _packed(model, samples)
    n0 = support.n_plans(model)
    _packed(model, samples)
    assert support.n_plans(model) == n0                      # same selection: the plan is reused
    with _States(model, [4, 6]):
        _packed(model, samples)
        assert support.n_plans(model) == n0 + 1              # changed selection: a plan of its own
    ref = _packed(model, samples)[1]
    # unsynchronised back-to-back calls into different buffers each get their own states
    other = support.batch(model, [(3, 5), (20, 33), (7, 7), (2, 60)], seed=801)
    a = _packed(model, samples, sync=False)[1]
    b = _packed(model, other, sync=False)[1]
    c = _packed(model, samples, sync=False)[1]
    torch.cuda.synchronize()
    ref_b = _packed(model, other)[1]
    for e in range(len(ref)):
        for x, y, z, rb, w in zip(a[e], c[e], ref[e], ref_b[e], b[e]):
            _eq(x, z)
            _eq(y, z)
            _eq(w, rb)
    # every one of total_floats is written, dense and packed, for every reduction
    nt, nr = [len(s[0]) for s in samples], [s[2].shape[0] for s in samples]
    for rows in ROWS:
        with _States(model, [0, 7, 31], rows=rows):
            layout, total = model.state_layout_packed(nt, nr)
            flat = torch.full((total,), float("nan"), device="cuda")
            o = L.StateOutputs()
            o.layer_states = flat.data_ptr()
            q, f, s, seg, task, _, _ = support.packed_sample_args(samples)
            pin = L.PackedInputs(len(samples), 0, 0, C.cast((C.c_int32 * 4)(*nt), C.c_void_p), C.cast((C.c_int32 * 4)(*nr), C.c_void_p),
                                 q.data_ptr(), seg.data_ptr(), f.data_ptr(), s.data_ptr(), task.data_ptr())
            model._call("vb200_forward_packed", C.byref(pin), C.byref(o), L.OUT_TASK_HEADS | L.OUT_LAYER_STATES, 0)
            torch.cuda.synchronize()
            assert not torch.isnan(flat).any(), rows
            _, total_d = model.state_layout(2, 9, 13)
            flat_d = torch.full((total_d,), float("nan"), device="cuda")
            assert _dense_raw(model, support.tiny_inputs(tiny_oracle, 2, 9, 13, seed=802, pad=3), flat_d.data_ptr()) == 0
            torch.cuda.synchronize()
            assert not torch.isnan(flat_d).any(), rows


def _dense_raw(model, inp, states_ptr, select=None, fn="vb200_forward"):
    """vb200_forward (or the host-buffer ``fn``) of make_inputs tensors with vb200_outputs.layer_states = states_ptr; the status."""
    L = support.lib()
    q, f, s, seg, im, vm = inp[:6]
    B, Tin = q.shape
    dev = "cpu" if fn.startswith("vb200_forward_host") else "cuda"
    keep = [q.long(), f.float(), s.float(), seg.long(), im.long(), vm.to(torch.uint8), inp[7].long().reshape(B, -1)[:, :1]]
    keep = [t.contiguous().to(dev) for t in keep]
    di = L.Inputs(B, Tin, f.shape[1], *(t.data_ptr() for t in keep[:6]), None, keep[6].data_ptr())
    o = L.StateOutputs()
    o.layer_states = states_ptr
    lib = L.load()
    sel = L.OUT_LAYER_STATES if select is None else select
    if fn == "vb200_forward_host_slot":
        return lib.vb200_forward_host_slot(model._handle, C.byref(di), C.byref(o), sel, 0, 1, None)
    return getattr(lib, fn)(model._handle, C.byref(di), C.byref(o), sel, None)


# ------------------------------------------------------------------------------------------------------------ options and rejections
def test_options_read_back_and_validation(tiny, tiny_oracle):
    L = support.lib()
    model = tiny["fp16"]
    # the engine's full list is the specified one: embeddings, then per step its text state before its image state
    spec = [0, 1]
    for step in tiny_oracle.bert.encoder.schedule():
        spec += ([0] if step[0] != "V" else []) + ([1] if step[0] != "T" else [])
    assert model.state_selection()[0] == spec
    lib = L.load()
    v = C.c_int64()
    assert lib.vb200_model_dim(model._handle, b"state_entries", C.byref(v)) == 0 and v.value == (1 << 32) - 1
    assert lib.vb200_model_dim(model._handle, b"state_rows", C.byref(v)) == 0 and v.value == 0
    for key, bad in ((b"state_entries", 0), (b"state_entries", 1 << 32), (b"state_rows", 3), (b"state_rows", -1)):
        assert lib.vb200_set_option(model._handle, key, bad) == -1
    with _States(model, [3, 5], rows="mean"):
        assert lib.vb200_model_dim(model._handle, b"state_entries", C.byref(v)) == 0 and v.value == 40
        assert lib.vb200_model_dim(model._handle, b"state_rows", C.byref(v)) == 0 and v.value == 2
        kinds, where = model.state_selection()
        assert where[3] == 0 and where[5] == 1 and where.count(-1) == 30
        layout, total = model.state_layout(2, 9, 13)
        assert [(k, r) for k, r, w, o in layout] == [(kinds[3], 2), (kinds[5], 2)]


def test_rejections(tiny, tiny_oracle):
    L = support.lib()
    model = tiny["fp16"]
    lib = L.load()
    h = model._handle
    flat = torch.full((64,), -7.0, device="cuda")
    inp = support.tiny_inputs(tiny_oracle, 1, 6, 5, seed=90)
    bit = L.OUT_VIL_LOGIT | L.OUT_LAYER_STATES

    def rejects(rc, name):
        assert rc == -1
        assert name in lib.vb200_last_error(h).decode()
        torch.cuda.synchronize()
        assert bool((flat == -7.0).all())

    rejects(_dense_raw(model, inp, flat.data_ptr(), bit, "vb200_forward_host"), "vb200_forward_host")
    rejects(_dense_raw(model, inp, flat.data_ptr(), bit, "vb200_forward_host_slot"), "vb200_forward_host")
    o = L.StateOutputs()
    o.layer_states = flat.data_ptr()
    idx = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = torch.zeros(4096, device="cuda")
    rejects(lib.vb200_forward_cached(h, 1, 6, 5, idx.data_ptr(), 1, st.data_ptr(), st.data_ptr(), st.data_ptr(), idx.data_ptr(), 1,
                                     st.data_ptr(), st.data_ptr(), st.data_ptr(), C.byref(o), bit, 0, None), "vb200_forward_cached")
    # the packed pair suffix: host index / offset arrays, device states (never read before the rejection)
    zero = (C.c_int32 * 1)(0)
    t_offs, v_offs = (C.c_int32 * 2)(0, 7), (C.c_int32 * 2)(0, 5)
    pairs = L.PackedPairs(1, 0, 0, C.cast(zero, C.c_void_p), C.cast(zero, C.c_void_p), 1, C.cast(t_offs, C.c_void_p), st.data_ptr(),
                          st.data_ptr(), 1, C.cast(v_offs, C.c_void_p), st.data_ptr(), st.data_ptr())
    rejects(lib.vb200_forward_cached_packed(h, C.byref(pairs), C.byref(o), bit, 0, None), "vb200_forward_cached_packed")
    # the bit without a buffer, or with one the 16-byte state stores cannot write: dense and packed
    rejects(_dense_raw(model, inp, None, bit), "layer_states (NULL)")
    rejects(_dense_raw(model, inp, flat[1:].data_ptr(), bit), "vb200_forward: vb200_outputs.layer_states is not 16-byte aligned")
    samples = support.batch(model, [(3, 4), (5, 2)], seed=92)
    q, f, s, seg, task, nt, nr = support.packed_sample_args(samples)
    pin = L.PackedInputs(2, 0, 0, C.cast((C.c_int32 * 2)(*nt), C.c_void_p), C.cast((C.c_int32 * 2)(*nr), C.c_void_p),
                         q.data_ptr(), seg.data_ptr(), f.data_ptr(), s.data_ptr(), task.data_ptr())
    o.layer_states = flat[2:].data_ptr()
    rejects(lib.vb200_forward_packed(h, C.byref(pin), C.byref(o), bit, 0, None),
            "vb200_forward_packed: vb200_outputs.layer_states is not 16-byte aligned")
    # fp32x keeps rejecting packed calls as before
    x = tiny["fp32x"]
    with pytest.raises(L.VilbertB200Error, match="split_fp32"):
        x.forward_packed(*support.packed_sample_args(support.batch(model, [(3, 4)], seed=91)), output_layer_states=True)


def test_pretraining_engine_accepts_states():
    """A pre-training engine (no task heads) writes the states of dense and packed forwards; the last entries are its taps."""
    import vilbert_b200 as vb
    from oracle import pretraining_ref as P
    oracle = P.build(P.tiny_pretraining_config(), seed=7)
    model = vb.BertForMultiModalPreTraining.from_pretrained(oracle.state_dict(), config=vb.BertConfig.from_dict(oracle.config.to_dict()),
                                                           compute_dtype="bf16").eval().cuda(0)
    try:
        lt, lv = _last(model)
        samples = support.batch(model, [(4, 9), (11, 3)], seed=93)
        (_, taps), states = model.forward_packed(*support.packed_sample_args(samples), select=0, debug_taps=True, output_layer_states=True)
        _eq(torch.cat(states[lt]), taps["sequence_output_t"])
        _eq(torch.cat(states[lv]), taps["sequence_output_v"])
        q, seg, f, s, task = samples[0]
        (_, taps_d), states_d = vb.VILBertForVLTasks.forward(
            model, q[None].cuda(), f[None].cuda(), s[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
            torch.ones(1, f.shape[0], dtype=torch.uint8).cuda(), None, torch.tensor([[task]]).cuda(),
            select=support.lib().OUT_LINGUISIC_PREDICTION | support.lib().OUT_VISION_PREDICTION, debug_taps=True, output_layer_states=True)
        torch.cuda.synchronize()
        _eq(states_d[lt], taps_d["sequence_output_t"])
        _eq(states_d[lv], taps_d["sequence_output_v"])
        for e in range(len(states)):
            _eq(states[e][0], states_d[e][0])          # the packed sample equals the dense forward of it alone
    finally:
        model.close()
