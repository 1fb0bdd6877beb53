"""Every configuration of the matrix (support.CONFIGS) on the engine.  `-m gpu` only.

The other suites build two model shapes that share one layer schedule, the head sizes, bi_hidden == v_hidden, widths of 1, 2 or an
even number of 128-column tiles and task tokens on.  The plan builder has code that only other configurations reach: image layers
ahead of the first connection layer, an empty text prefix, a stream that ends in a connection layer (its tail stays unpruned),
connection layers back to back or none at all, head sizes swapped between the streams, connection heads outnumbering the stream
heads (padded head-gate slots), bi_hidden != v_hidden (the QKV and context buffers sized by the wider of the two), widths of three
and five tiles, an image-embedding K that is not a multiple of 64 and the multi-task heads without the task row.  For each entry:

* the fp32x forward against the fp64 oracle at ``oracle.fp64.BOUNDS``: the nine outputs, the final-state taps, every map;
* the fp16 and bf16 forwards step by step against ``oracle.step_ref.StepRef`` at ``STEP_BOUNDS``;
* the bits the engine promises: packed = each sample alone, packed regions = each image alone, the retrieval split (dense and packed)
  = the forward of the same pairs, the pruned plan = the unpruned one, an all-ones head mask = no mask;
* the attention-map and layer-state layouts, dense and packed, and the head-mask shape against the schedule;
* without task tokens, the coalition and message ablations, whose variant offsets subtract the task rows of the samples before.

Every case is small (B <= 4, <= 40 tokens, <= 40 regions); each entry builds three engines.
"""
import pytest
import torch

from oracle import fp64 as X
from oracle import step_ref as S
import support
from test_gpu_fp32x_fp64 import _forward
from test_gpu_head_mask import _bit_equal, _packed as _packed_gated_outputs, _shape
from test_gpu_packed import _check_bitwise as _packed_equals_alone
from test_gpu_regions_packed import _check_bitwise as _regions_equal_alone, _images as _region_images
from test_gpu_retrieval_packed import _assert_same, _captions, _encode, _forward_packed_pairs, _images as _gallery
from test_gpu_step_parity import _assert as _step_assert, engine as _step_engine, run_dense

pytestmark = pytest.mark.gpu

MODES = ("fp16", "bf16")
POOLED = 0x1F               # the heads that read pooled_output only: a plan selecting nothing else prunes both stream tails
ROW_HEADS = (1 << 6) | (1 << 8)   # VISION_LOGIT | LINGUISIC_LOGIT: every final row of both streams is read
DENSE = (3, 16, 10, 3)      # B, Tin, V, padded regions
PACKED_LENS = [(1, 40), (17, 3), (33, 21)]       # (Tin, V) per sample, odd B
REGION_LENS = [(1, 39), (12, 1), (30, 9)]        # (Tin, boxes) per image; V = boxes + 1


@pytest.fixture(scope="module", params=sorted(support.CONFIGS))
def entry(request):
    """(name, fp32 oracle, {"fp16", "bf16", "fp32x": engine with return_attention}) of one matrix entry."""
    name = request.param
    oracle = support.config_oracle(name)
    engines = {}
    try:
        for m in MODES:
            engines[m] = _step_engine(oracle, m)
        engines["fp32x"] = support.engine(oracle, compute_dtype="fp32x", return_attention=True)
        yield name, oracle, engines
    finally:
        for m in engines.values():
            m.close()


def _dense(oracle, seed, shape=DENSE):
    B, Tin, V, pad = shape
    return support.tiny_inputs(oracle, B, Tin, V, seed, pad)


# ------------------------------------------------------------------------------------------------------------ against the oracles
def test_fp32x_against_fp64(entry, parity_log):
    name, oracle, eng = entry
    _forward(X.fp64(oracle), eng["fp32x"], _dense(oracle, 61), f"config_{name}", parity_log)


@pytest.mark.parametrize("mode", MODES)
def test_step_parity(entry, mode, parity_log):
    name, oracle, eng = entry
    _step_assert(f"config_{name}", mode, run_dense(eng[mode], oracle, mode, _dense(oracle, 62)), parity_log)


# ------------------------------------------------------------------------------------------------------------ same bits
@pytest.mark.parametrize("mode", MODES)
def test_packed_equals_each_sample_alone(entry, mode):
    import vilbert_b200 as vb
    _, _, eng = entry
    model = eng[mode]
    samples = support.batch(model, PACKED_LENS, seed=63)
    out = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_ALL, debug_taps=True)
    torch.cuda.synchronize()
    _packed_equals_alone(model, samples, out)


@pytest.mark.parametrize("mode", MODES)
def test_regions_packed_equals_each_image_alone(entry, mode):
    import vilbert_b200 as vb
    _, _, eng = entry
    model = eng[mode]
    imgs = _region_images(model, REGION_LENS, seed=64)
    out = model.forward_regions_packed(*support.packed_image_args(imgs), select=vb.OUT_ALL, debug_taps=True)
    torch.cuda.synchronize()
    _regions_equal_alone(model, imgs, out)


@pytest.mark.parametrize("mode", MODES)
def test_retrieval_split_equals_forward(entry, mode):
    """encode_text / encode_image -> forward_cached against forward on the same padded batch, and encode_text_packed /
    encode_image_packed -> forward_cached_packed against forward_packed of the same pairs (captions and images repeated)."""
    import vilbert_b200 as vb
    _, oracle, eng = entry
    model = eng[mode]
    q, f, s, seg, im, vm, _, task = [t.cuda() for t in _dense(oracle, 65)]
    ts, vs = model.encode_text(q, seg, im, task), model.encode_image(f, s, vm)
    idx = torch.arange(q.shape[0], dtype=torch.int32).cuda()
    got = model.forward_cached(ts, idx, vs, idx, select=vb.OUT_ALL)
    want = model(q, f, s, seg, im, vm, None, task, select=vb.OUT_ALL)
    torch.cuda.synchronize()
    for k in range(9):
        assert torch.equal(got[k], want[k]), f"forward_cached: output {k} differs from forward"
    caps, imgs = _captions(model, [1, 20, 38], seed=66), _gallery(model, [1, 17, 40], seed=66)
    ts, vs = _encode(model, caps, imgs)
    ti, ii = [2, 0, 1, 2], [0, 2, 2, 1]
    got = model.forward_cached_packed(ts, torch.tensor(ti), vs, torch.tensor(ii).cuda(), select=vb.OUT_ALL, debug_taps=True)
    torch.cuda.synchronize()
    _assert_same(got, _forward_packed_pairs(model, caps, imgs, ti, ii, vb.OUT_ALL), f"forward_cached_packed {mode}")


def _last_writer(schedule, stream):
    """The kind ("T", "V" or "C") of the last schedule step that writes ``stream`` ("T" text, "V" image)."""
    return next(s[0] for s in reversed(schedule) if s[0] in (stream, "C"))


@pytest.mark.parametrize("mode", MODES)
def test_pruned_plan_equals_unpruned(entry, mode):
    """vil_prediction alone prunes each stream whose last step is a stream layer; a stream that ends in a connection layer keeps
    its rows.  The pruned plans' vil_prediction equals the OUT_ALL plan's, dense and packed, and the pruned plan drops exactly the
    pruned streams' row-local GEMMs past each sample's first row."""
    import vilbert_b200 as vb
    _, oracle, eng = entry
    model = eng[mode]
    inp = [t.cuda() for t in _dense(oracle, 67)]
    pruned, full = model(*inp, select=vb.OUT_VIL_PREDICTION), model(*inp, select=vb.OUT_ALL)
    samples = support.batch(model, PACKED_LENS, seed=68)
    p_packed = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_VIL_PREDICTION)
    f_packed = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_ALL)
    torch.cuda.synchronize()
    assert torch.equal(pruned[0], full[0]), "dense: vil_prediction differs with the pruned tail"
    assert torch.equal(p_packed[0], f_packed[0]), "packed: vil_prediction differs with the pruned tail"
    c, schedule = oracle.config, oracle.bert.encoder.schedule()
    B, Tin, V, _ = DENSE
    T = Tin + (1 if c.task_specific_tokens else 0)
    removed = 0
    if _last_writer(schedule, "T") == "T":
        removed += 2 * B * (T - 1) * (c.hidden_size ** 2 + 2 * c.hidden_size * c.intermediate_size)
    if _last_writer(schedule, "V") == "V":
        removed += 2 * B * (V - 1) * (c.v_hidden_size ** 2 + 2 * c.v_hidden_size * c.v_intermediate_size)
    row_heads = 2 * B * T * c.hidden_size + 2 * B * V * c.v_hidden_size
    _, f_pruned = model.plan_info(B, Tin, V, POOLED)
    _, f_kept = model.plan_info(B, Tin, V, POOLED | ROW_HEADS)
    assert f_kept - f_pruned == removed + row_heads


@pytest.mark.parametrize("mode", MODES)
def test_all_ones_head_mask_is_ungated(entry, mode):
    """Every output, tap, map and layer state of a packed forward with an all-ones head mask, bit for bit, with the gate table
    sized for the configuration's widest attention."""
    _, _, eng = entry
    model = eng[mode]
    samples = support.batch(model, PACKED_LENS, seed=69)
    _bit_equal(_packed_gated_outputs(model, samples, head_mask=torch.ones(_shape(model))), _packed_gated_outputs(model, samples))


# ------------------------------------------------------------------------------------------------------------ layouts
def _map_shape(label, c, B, T, V):
    if label[0] == "T":
        return (B, c.num_attention_heads, T, T)
    if label[0] == "V":
        return (B, c.v_num_attention_heads, V, V)
    return (B, c.bi_num_attention_heads) + ((T, V) if label.endswith("text->image") else (V, T))


def test_layouts_follow_the_schedule(entry):
    """The maps and layer states of a dense and a packed forward, the selection kinds and the head-mask shape, against the
    oracle's labels of the entry's schedule."""
    import ctypes as C
    import vilbert_b200 as vb
    _, oracle, eng = entry
    model, c = eng["bf16"], oracle.config
    schedule = oracle.bert.encoder.schedule()
    maps, entries = S.map_labels(schedule), S.entry_labels(schedule)
    kinds = [0 if m[0] == "T" else 1 if m[0] == "V" else 2 if m.endswith("text->image") else 3 for m in maps]
    assert model.attention_selection()[0] == kinds
    assert model.state_selection()[0] == [0 if e.endswith("text") else 1 for e in entries]
    L = support.lib()
    for key, want in zip(("head_mask_entries", "head_mask_heads"), _shape(model)):
        v = C.c_int64()
        L.check(L.load().vb200_model_dim(model._handle, key.encode(), C.byref(v)), model._handle)
        assert v.value == want == (len(maps) if key == "head_mask_entries" else
                                   max(c.num_attention_heads, c.v_num_attention_heads, c.bi_num_attention_heads)), key
    B, Tin, V, _ = DENSE
    T = Tin + (1 if c.task_specific_tokens else 0)
    res, states = model(*[t.cuda() for t in _dense(oracle, 70)], select=vb.OUT_ALL, output_all_attention_masks=True,
                        output_layer_states=True)
    torch.cuda.synchronize()
    got = S.flat_maps(res[9])
    assert len(got) == len(maps)
    for lab, m in zip(maps, got):
        assert tuple(m.shape) == _map_shape(lab, c, B, T, V), lab
    assert len(states) == len(entries)
    for lab, st in zip(entries, states):
        assert tuple(st.shape) == ((B, T, c.hidden_size) if lab.endswith("text") else (B, V, c.v_hidden_size)), lab
    samples = support.batch(model, PACKED_LENS, seed=71)
    res, states = model.forward_packed(*support.packed_sample_args(samples), select=vb.OUT_ALL, output_all_attention_masks=True,
                                       output_layer_states=True)
    torch.cuda.synchronize()
    got = S.flat_maps(res[9])
    assert len(got) == len(maps) and len(states) == len(entries)
    for b, (tin, v) in enumerate(PACKED_LENS):
        t = tin + (1 if c.task_specific_tokens else 0)
        for lab, m in zip(maps, got):
            assert tuple(m[b].shape) == _map_shape(lab, c, 1, t, v)[1:], (lab, b)
        for lab, st in zip(entries, states):
            assert tuple(st[b].shape) == ((t, c.hidden_size) if lab.endswith("text") else (v, c.v_hidden_size)), (lab, b)


# ------------------------------------------------------------------------------------------------------------ no task tokens
MASK = 103
VQA, NLVR2 = 1, 3


@pytest.fixture(scope="module")
def untasked():
    oracle = support.config_oracle("no_task_tokens")
    yield from support.one_engine(oracle, compute_dtype="bf16")


def test_ablations_without_task_tokens(untasked):
    """With no task row, a sample's text rows start at the sum of the earlier samples' lengths alone.  One coalition per question
    position (that position absent) gives message ablation's token variants bit for bit, for messages on the first and on later
    samples; and a VQA token variant is forward_regions of that image alone with the token replaced by the mask token."""
    import vilbert_b200 as vb
    model = untasked
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    lens = [(7, 4), (9, 6), (5, 3), (5, 8)]
    imgs = [support.image(t, n, 72 + i, F, vocab) for i, (t, n) in enumerate(lens)]
    imgs[3] = imgs[2][:2] + imgs[3][2:5] + (imgs[2][5],)            # an NLVR2 pair: one question on two images
    args = support.packed_image_args(imgs)
    msgs = [(VQA, 0, 1), (VQA, 1, 1), (NLVR2, 2, 2)]
    ab = model.message_ablation(*args, [m + (None, (0, lens[m[1]][0]), (0, 0)) for m in msgs], mask_token=MASK, return_logits=True)
    units = [[((p,), ()) for p in range(lens[m[1]][0])] for m in msgs]
    coal = [(~torch.eye(len(u), dtype=torch.bool)).tolist() for u in units]
    res = model.coalition_ablation(*args, msgs, units, coal, mask_token=MASK, return_logits=True)
    torch.cuda.synchronize()
    for i, (a, r) in enumerate(zip(ab, res)):
        assert a["tokens"] == list(range(lens[msgs[i][1]][0])) and not a["boxes"]
        assert len(a["logits"]) == len(r["logits"]) == 1 + len(a["tokens"])
        for k, (x, y) in enumerate(zip(a["logits"], r["logits"])):
            assert torch.equal(x, y), f"message {i}: variant {k}"
        assert r["prob"] == a["prob"] and torch.equal(r["coalition_prob"], torch.cat([a["token_prob"], a["box_prob"]]))
    for i in (0, 1):
        for p in (0, 3, lens[i][0] - 1):
            q = imgs[i][0].clone()
            q[p] = MASK
            out, _ = support.regions_alone(model, (q,) + imgs[i][1:], vb.OUT_VIL_PREDICTION)
            assert torch.equal(ab[i]["logits"][1 + p], out[0][0]), f"sample {i} position {p}"
