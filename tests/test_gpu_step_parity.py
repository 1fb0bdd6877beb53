"""Step-by-step parity of the fp16 and bf16 forwards: every layer state against oracle/step_ref.py run on the engine's own previous
states (teacher forcing).  `-m gpu` only.

End to end, tests/test_gpu_model.py can only hold a 16-bit forward to the format floor against the fp32 oracle.  Here every entry of
the full layer-state list (``output_layer_states``, every row) is compared with ``StepRef`` fed the engine's previous entries and the
engine's masks, so engine and reference differ by one step's last-bit disagreements only, and a failure names the first step, stream,
sample and row over the bound.  Families (``step_ref.STEP_BOUNDS``):

* states: every entry, embeddings included (oracle.fp64.rel_err);
* maps: every step's attention probabilities against the fp64 softmax of the reference's 16-bit Q and K (max abs);
* pooled: the ``pooled_output`` tap against the poolers run on the final entries;
* logits: the nine outputs, pre-training heads included, against the heads run on the ``pooled_output`` and final-state taps.

The forwards here select per-row outputs and taps, so no stream's last layer is pruned; the pruned plans' taps and states are the
unpruned ones bit for bit (tests/test_gpu_pruned_tail.py, tests/test_gpu_layer_states.py), which these tests rely on.  The reference
runs in fp64 on the GPU.  Each case logs one line per mode and family with its worst step (the ``parity_log`` fixture);
scripts/step_parity_sweep.py runs the same cases over many seeds.
"""
import pytest
import torch

from oracle import fp64 as X
from oracle import step_ref as S

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16")
TINY_DENSE = [(2, 30, 36, 0), (3, 16, 10, 3), (4, 37, 101, 7), (1, 3, 1, 0), (1, 155, 256, 11), (5, 3, 7, 2)]
LONG = [(300, 36), (30, 1000)]
PACKED_LENS = [(1, 40), (31, 1), (12, 64), (5, 17), (99, 100), (60, 3), (7, 77)]
REGION_LENS = [(7, 3), (1, 30), (20, 9), (45, 99)]


# ------------------------------------------------------------------------------------------------------------ engines
def engine(oracle, mode, **kw):
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    return vb.VILBertForVLTasks.from_pretrained(oracle.state_dict(), config=cfg, num_labels=oracle.num_labels, compute_dtype=mode,
                                                return_attention=True, **kw).eval().cuda(0)


def long_oracle():
    from oracle import vilbert_ref as R
    return R.build(R.tiny_config(max_position_embeddings=1024), seed=7, num_labels=200)


@pytest.fixture(scope="module")
def tiny(tiny_oracle):
    e = {m: engine(tiny_oracle, m) for m in MODES}
    yield e
    for m in e.values():
        m.close()


# ------------------------------------------------------------------------------------------------------------ cases
def _OUT_ALL():
    from vilbert_b200 import _lib as L
    return L.OUT_ALL


def tiny_inputs(oracle, B, Tin, V, seed, pad=0):
    from oracle import vilbert_ref as R
    inp = list(R.make_inputs(B, Tin, V, seed=seed, vocab_size=oracle.config.vocab_size, pad_regions=pad))
    inp[1] = inp[1][..., :oracle.config.v_feature_size].contiguous()
    return inp


def _last(schedule):
    labels = S.entry_labels(schedule)
    return (max(i for i, x in enumerate(labels) if x.endswith("text")), max(i for i, x in enumerate(labels) if x.endswith("image")))


def _heads(ref, res, taps, v_mask_rows):
    """pooled and logits families from the taps (the reference heads on the engine's pooled product and final states)."""
    out = ref.outputs(taps["pooled_output"], taps["sequence_output_t"], taps["sequence_output_v"], v_mask_rows)
    return [(name,) + S.row_err(res[i], out[i]) for i, name in enumerate(X.OUTPUT_NAMES)]


def run_dense(model, oracle, mode, inp, every=1):
    """A dense forward against StepRef, teacher-forced on its states: {family: [(label, err, where)]}.  ``every``: the reference runs
    on every ``every``-th sample (every step is sample-local); the per-sample heads run on all of them."""
    (res, taps), states = model(*[t.cuda() for t in inp], select=_OUT_ALL(), debug_taps=True, output_all_attention_masks=True,
                                output_layer_states=True)
    torch.cuda.synchronize()
    ref = S.StepRef(oracle, mode, device="cuda")
    tm, vm = (m.cuda() for m in S.key_masks(inp[4], inp[5], oracle.config.task_specific_tokens))
    sl = slice(None, None, every)
    maps = [tuple(x[sl] for x in m) if isinstance(m, tuple) else m[sl] for m in res[9]]
    out = S.teacher_forced(ref, [s[sl] for s in states], ref.text_embed(inp[0][sl], inp[3][sl], inp[7][sl]),
                           ref.image_embed(inp[1][sl], inp[2][sl]), tm[sl], vm[sl], maps)
    lt, lv = _last(ref.schedule)
    out["pooled"] = [("pooled_output",) + S.row_err(taps["pooled_output"], ref.pooled(states[lt][:, 0], states[lv][:, 0]))]
    out["logits"] = _heads(ref, res, taps, vm)
    return out


def _merge(per_sample):
    """Per-sample result dicts -> one: per label the worst sample, named in ``where``."""
    res = {}
    for b, r in enumerate(per_sample):
        for fam, errs in r.items():
            cur = res.setdefault(fam, [None] * len(errs))
            for i, (lab, e, where) in enumerate(errs):
                if cur[i] is None or e > cur[i][1]:
                    cur[i] = (lab, e, where.replace("sample 0", f"sample {b}", 1))
    return res


def _packed_sample(ref, states, maps, b, emb_t, emb_v):
    """Sample b of a packed forward: its states and maps at its own lengths, all rows real."""
    st = [s[b][None] for s in states]
    mp = [tuple(x[b][None] for x in m) if isinstance(m, tuple) else m[b][None] for m in maps]
    tm = torch.zeros(1, st[0].shape[1], dtype=torch.float64, device="cuda")
    vm = torch.zeros(1, st[1].shape[1], dtype=torch.float64, device="cuda")
    return S.teacher_forced(ref, st, emb_t, emb_v, tm, vm, mp)


def _packed_heads(ref, res, taps, states, n_rows_v):
    lt, lv = _last(ref.schedule)
    t_first = torch.stack([x[0] for x in states[lt]])
    v_first = torch.stack([x[0] for x in states[lv]])
    pooled = [("pooled_output",) + S.row_err(taps["pooled_output"], ref.pooled(t_first, v_first))]
    return pooled, _heads(ref, res, taps, torch.zeros(n_rows_v, dtype=torch.float64, device="cuda"))


def packed_samples(model, lens, seed):
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    out = []
    for i, (tin, v) in enumerate(lens):
        g = torch.Generator().manual_seed(seed + i)
        q = torch.randint(1, vocab, (tin,), generator=g)
        f = torch.relu(torch.randn(v, F, generator=g)) * 1.5
        x1, y1 = torch.rand(v, generator=g) * 0.7, torch.rand(v, generator=g) * 0.7
        x2, y2 = x1 + 0.05 + torch.rand(v, generator=g) * 0.25, y1 + 0.05 + torch.rand(v, generator=g) * 0.25
        s = torch.stack([x1, y1, x2.clamp(max=1.0), y2.clamp(max=1.0), (x2 - x1) * (y2 - y1)], dim=-1)
        s[0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
        seg = torch.randint(0, 2, (tin,), generator=g)
        out.append((q, seg, f, s, int(torch.randint(0, 20, (1,), generator=g))))
    return out


def run_packed(model, oracle, mode, samples):
    """forward_packed: every sample teacher-forced at its own lengths."""
    cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda()
    task = torch.tensor([[s[4]] for s in samples]).cuda()
    nt, nv = [len(s[0]) for s in samples], [s[2].shape[0] for s in samples]
    (res, taps), states = model.forward_packed(cat(0), cat(2), cat(3), cat(1), task, nt, nv, select=_OUT_ALL(), debug_taps=True,
                                               output_all_attention_masks=True, output_layer_states=True)
    torch.cuda.synchronize()
    ref = S.StepRef(oracle, mode, device="cuda")
    per = []
    for b, (q, seg, f, sp, tk) in enumerate(samples):
        per.append(_packed_sample(ref, states, res[9], b, ref.text_embed(q[None], seg[None], torch.tensor([[tk]])),
                                  ref.image_embed(f[None], sp[None])))
    out = _merge(per)
    out["pooled"], out["logits"] = _packed_heads(ref, res, taps, states, sum(nv))
    return out


def region_images(model, lens, seed):
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    imgs = []
    for i, (tin, n) in enumerate(lens):
        g = torch.Generator().manual_seed(seed + i)
        q, seg = torch.randint(1, vocab, (tin,), generator=g), torch.randint(0, 2, (tin,), generator=g)
        f = torch.relu(torch.randn(n, F, generator=g))
        x1, y1 = torch.rand(n, generator=g) * 400, torch.rand(n, generator=g) * 300
        bx = torch.stack([x1, y1, x1 + 20 + torch.rand(n, generator=g) * 200, y1 + 20 + torch.rand(n, generator=g) * 150], 1)
        imgs.append((q, seg, f, bx, torch.tensor([640.0, 480.0]), i + 1))
    return imgs


def _region_embed(ref, f, bx, wh):
    from oracle import kernel_refs as K
    rows, loc, _ = K.region_rows(f.numpy(), bx.numpy(), float(wh[0]), float(wh[1]), f.shape[0])
    return ref.image_embed(torch.from_numpy(rows)[None], torch.from_numpy(loc)[None])


def run_regions(model, oracle, mode, imgs):
    """forward_regions (one dense batch of images with the same text length and box count) and forward_regions_packed (the same
    images at their own lengths).  Dense: states and maps (forward_regions has no taps); packed: every family."""
    from vilbert_b200 import _lib as L
    ref = S.StepRef(oracle, mode, device="cuda")
    q, seg, f, bx, wh, tk = imgs[0]
    dense = [im for im in imgs if im[0].shape == q.shape and im[2].shape == f.shape]
    st = lambda k: torch.stack([im[k] for im in dense])
    ((res, _), states) = model.forward_regions(st(0).cuda(), st(1).cuda(), torch.ones(len(dense), len(q), dtype=torch.long).cuda(),
                                               torch.tensor([[im[5]] for im in dense]).cuda(), st(2).cuda(), st(3).cuda(),
                                               st(4).cuda(), select=L.OUT_ALL, output_all_attention_masks=True,
                                               output_layer_states=True)
    torch.cuda.synchronize()
    emb_v = torch.cat([_region_embed(ref, im[2], im[3], im[4]) for im in dense])
    tm = torch.zeros(len(dense), len(q) + 1, dtype=torch.float64, device="cuda")
    vm = torch.zeros(len(dense), f.shape[0] + 1, dtype=torch.float64, device="cuda")
    out = {"regions " + k: v for k, v in S.teacher_forced(ref, states, ref.text_embed(st(0), st(1), torch.tensor([[im[5]] for im in dense])),
                                                          emb_v, tm, vm, res[9]).items()}
    cat = lambda k: torch.cat([im[k] for im in imgs], dim=0).cuda()
    nt, nb = [len(im[0]) for im in imgs], [im[2].shape[0] for im in imgs]
    (((res, taps), _), states) = model.forward_regions_packed(cat(0), cat(1), torch.tensor([[im[5]] for im in imgs]).cuda(), cat(2),
                                                              cat(3), torch.stack([im[4] for im in imgs]).cuda(), nt, nb,
                                                              select=L.OUT_ALL, debug_taps=True, output_all_attention_masks=True,
                                                              output_layer_states=True)
    torch.cuda.synchronize()
    per = [_packed_sample(ref, states, res[9], b, ref.text_embed(im[0][None], im[1][None], torch.tensor([[im[5]]])),
                          _region_embed(ref, im[2], im[3], im[4])) for b, im in enumerate(imgs)]
    out.update(_merge(per))
    out["pooled"], out["logits"] = _packed_heads(ref, res, taps, states, sum(n + 1 for n in nb))
    return out


# ------------------------------------------------------------------------------------------------------------ checks
def family(name):
    return name.split(" ")[-1]


def report(tag, mode, result, log=None):
    """Log one line per family with its worst entry; return the failures [(family, (label, err, where), bound)]: each family's
    first entry in execution order at or over its bound."""
    fails = []
    for fam, errs in result.items():
        if not errs:
            continue
        bound = S.STEP_BOUNDS[mode][family(fam)]
        w = S.worst(errs)
        if log is not None:
            log(test=f"step_parity_{tag}_{mode}", family=fam, max_err=w[1], worst_step=w[0], where=w[2], bound=bound)
        first = S.first_over(errs, bound)
        if first is not None:
            fails.append((fam, first, bound))
    return fails


def _assert(tag, mode, result, parity_log):
    fails = report(tag, mode, result, parity_log)
    assert not fails, "; ".join(f"{fam}: first over {bound:g} at {lab} ({where}): {e:.3e}" for fam, (lab, e, where), bound in fails)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,Tin,V,pad", TINY_DENSE)
def test_tiny_dense(tiny, tiny_oracle, mode, B, Tin, V, pad, parity_log):
    inp = tiny_inputs(tiny_oracle, B, Tin, V, seed=1000 + 7 * B + Tin, pad=pad)
    _assert(f"tiny_B{B}_T{Tin}_V{V}_pad{pad}", mode, run_dense(tiny[mode], tiny_oracle, mode, inp), parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_tiny_packed(tiny, tiny_oracle, mode, parity_log):
    model = tiny[mode]
    _assert("tiny_packed", mode, run_packed(model, tiny_oracle, mode, packed_samples(model, PACKED_LENS, 1100)), parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_tiny_regions(tiny, tiny_oracle, mode, parity_log):
    model = tiny[mode]
    imgs = region_images(model, REGION_LENS, 1200) + region_images(model, [REGION_LENS[0]], 1250)
    _assert("tiny_regions", mode, run_regions(model, tiny_oracle, mode, imgs), parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_past_256_rows(mode, parity_log):
    """The streaming attention kernels: a tiny model with the 1024-position table, as tests/test_gpu_long_sequences.py builds it."""
    oracle = long_oracle()
    model = engine(oracle, mode, max_rows_per_sample=1024)
    try:
        for Tin, V in LONG:
            inp = tiny_inputs(oracle, 2, Tin, V, seed=1300 + Tin, pad=5)
            _assert(f"long_T{Tin}_V{V}", mode, run_dense(model, oracle, mode, inp), parity_log)
        _assert("long_packed", mode, run_packed(model, oracle, mode, packed_samples(model, [(300, 20), (17, 700), (80, 257)], 1350)),
                parity_log)
    finally:
        model.close()


@pytest.mark.parametrize("mode", MODES)
def test_full_model(full_oracle, mode, parity_log):
    """The 268 M model at B = 2 (64-wide small-forward GEMM tiles) and at the bench shape B = 64, 30 tokens x 36 regions (128-wide
    tiles; the reference on every 8th sample)."""
    from oracle import vilbert_ref as R
    model = engine(full_oracle, mode)
    try:
        _assert("full_B2", mode, run_dense(model, full_oracle, mode, R.make_inputs(2, 30, 36, seed=1400, pad_regions=4)), parity_log)
        _assert("full_B64", mode, run_dense(model, full_oracle, mode, R.make_inputs(64, 30, 36, seed=1401), every=8), parity_log)
    finally:
        model.close()
