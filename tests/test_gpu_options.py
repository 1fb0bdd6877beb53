"""Every engine option against the default path, on every call family.  `-m gpu` only.

The header promises that the engine options -- use_cuda_graph, use_pdl, vb200_set_option's "gemm_kernel", the plan-cache bound
max_plans and the validation bound "max_rows_per_sample" -- change scheduling only, never bits.  Each call family stages its own
per-call layout (packed rows, maps and states destinations, gates, ablation variants, decode and pre-training descriptors) through
pinned staging into a plan's metadata or an engine workspace, and those copies interleave differently with the launches in eager
mode, without PDL, on the cooperative GEMM and in a plan rebuilt after an eviction.  So here:

* one seeded workload per family on the tiny model, with ragged packed layouts whose row totals are not multiples of 128 and a
  sample past 256 rows (the streaming attention kernels);
* a baseline of every family on a default engine per compute dtype, the fp32x one also held to the fp64 oracle at ``BOUNDS``;
* every row of ``ROWS`` on a fresh engine of the same dtype: each family's first call, its replay, and its call after every plan was
  evicted and rebuilt, bit for bit against the baseline.  Every buffer the model allocates is filled with 0xFF bytes (a NaN in every
  float format) before the engine sees it, so an element an option leaves unwritten fails the comparison; the baseline itself has
  none left, and rows a layout leaves unwritten (the free rows past a region selection's images) keep them;
* concurrency made deterministic with torch.cuda._sleep: calls queued behind a sleeping stream on other slots and streams, and back
  to back on one slot, with and without evictions, each equal to the same call run alone.

fp32x engines accept only the dense, cached, decode, selection, relevance and pre-training families (every packed entry point,
and so the gated forwards and the ablations, refuses split_fp32); their rows cover those.
"""
import contextlib
import struct

import numpy as np
import pytest
import torch

from oracle import fp64 as X
import support

pytestmark = pytest.mark.gpu

DTYPES = ("fp16", "bf16", "fp32x")
# Engine options of each row: constructor keywords, and "gemm_kernel" through vb200_set_option.
ROWS = {
    "eager": dict(use_cuda_graph=False),
    "no_pdl": dict(use_pdl=False),
    "pdl_on": dict(use_pdl=True),
    "eager_no_pdl": dict(use_cuda_graph=False, use_pdl=False),
    "coop_gemm": dict(gemm_kernel=0),
    "max_plans_1": dict(max_plans=1),
    "rows_1024": dict(max_rows_per_sample=1024),
    "all": dict(use_cuda_graph=False, use_pdl=False, gemm_kernel=0, max_plans=1, max_rows_per_sample=1024),
}
POISON = 0xFF              # every byte of a fresh buffer: NaN in fp32 / fp16 / bf16, -1 in every integer type
LONG_V = 300               # image rows of the long samples (past the 256 rows the staged attention kernels hold)


# ------------------------------------------------------------------------------------------------------------ poisoned buffers
class _PoisonedTorch:
    """The torch module as model.py sees it, with ``empty`` returning buffers filled with POISON bytes."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def empty(*args, **kw):
        t = torch.empty(*args, **kw)
        if t.numel():
            t.view(-1).view(torch.uint8).fill_(POISON)
        return t


@contextlib.contextmanager
def _poisoned():
    from vilbert_b200 import model as M
    saved, M.torch = M.torch, _PoisonedTorch()
    try:
        yield
    finally:
        M.torch = saved


def _flat(obj, name, out):
    """Every tensor, array and number of a family's result under a path name, tensors copied to the host."""
    if obj is None:
        return out
    if torch.is_tensor(obj):
        out[name] = obj.detach().contiguous().cpu().clone()
    elif isinstance(obj, np.ndarray):
        out[name] = torch.from_numpy(np.ascontiguousarray(obj)).clone()
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _flat(v, f"{name}.{k}", out)
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _flat(v, f"{name}[{i}]", out)
    elif isinstance(obj, float):
        out[name] = struct.pack("<d", obj)
    else:
        out[name] = obj
    return out


def _bytes(t):
    return t.view(-1).view(torch.uint8) if t.numel() else t.view(torch.uint8)


def _same(a, b):
    """Bit equality: tensors byte for byte (NaN positions and payloads included), everything else by value."""
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bytes(a), _bytes(b))
    return a == b


def _compare(tag, got, want):
    assert got.keys() == want.keys(), f"{tag}: outputs {sorted(set(got) ^ set(want))[:5]} differ in presence"
    bad = [k for k in want if not _same(got[k], want[k])]
    assert not bad, f"{tag}: {len(bad)} of {len(want)} outputs differ from the default path, first {bad[:4]}"


def _poison_left(t):
    """Elements of a float32 tensor that still hold the POISON pattern (never a value a kernel writes)."""
    return t.dtype == torch.float32 and bool((t.view(torch.int32) == -1).any())


# ------------------------------------------------------------------------------------------------------------ workloads
def _pinned(t):
    return t.contiguous().pin_memory()


@pytest.fixture(scope="module")
def work(tiny_oracle):
    """Host tensors of every family's seeded workload (drawn once, the same for every engine)."""
    cfg = tiny_oracle.config
    F, vocab = cfg.v_feature_size, cfg.vocab_size
    w = {}
    # dense: an odd batch with two padded regions, and one sample past 256 image rows
    w["dense"] = support.tiny_inputs(tiny_oracle, 3, 20, 13, 901, pad=2)
    w["dense_long"] = support.tiny_inputs(tiny_oracle, 1, 30, LONG_V, 902)
    # packed: 54 text rows and 66 image rows; one layout with a 300-row image
    w["packed"] = [support.sample(t, v, 910 + i, F, vocab) for i, (t, v) in enumerate([(7, 20), (30, 5), (1, 1), (12, 40)])]
    w["packed_b"] = [support.sample(t, v, 920 + i, F, vocab) for i, (t, v) in enumerate([(16, 3), (2, 33), (25, 9), (5, 11)])]
    w["packed_long"] = [support.sample(t, v, 930 + i, F, vocab) for i, (t, v) in enumerate([(9, LONG_V), (4, 3)])]
    # detector output: dense with one image at 4 valid boxes of 9, packed at its own box counts, one image of 299 boxes
    w["regions"] = [support.image(11, 9, 940 + i, F, vocab) for i in range(3)]
    w["regions_packed"] = [support.image(t, n, 950 + i, F, vocab) for i, (t, n) in enumerate([(9, 12), (20, 3), (5, 1), (14, 30)])]
    w["regions_long"] = [support.image(6, LONG_V - 1, 960, F, vocab), support.image(3, 2, 961, F, vocab)]
    # head gates: zeros, halves, ones and a gain, per sample
    E, H = _gate_shape(cfg)
    g = torch.Generator().manual_seed(970)
    levels = torch.tensor([0.0, 0.5, 1.0, 1.25])
    w["gate"] = levels[torch.randint(0, 4, (4, E, H), generator=g)]
    w["gate_b"] = levels[torch.randint(0, 4, (4, E, H), generator=g)]
    # retrieval: captions, a padded image gallery, and the same at packed lengths
    w["captions"] = support.tiny_inputs(tiny_oracle, 3, 22, 14, 980)
    w["gallery"] = support.tiny_inputs(tiny_oracle, 2, 22, 14, 981, pad=3)
    w["gallery_long"] = support.tiny_inputs(tiny_oracle, 1, 22, LONG_V, 982)
    # ablations: an NLVR2 pair, a VQA image and a retrieval message over two images
    w["ablation"] = [support.image(8, n, 990 + i, F, vocab) for i, n in enumerate([4, 5, 3, 6])]
    w["coalitions"] = torch.rand(6, 6 + 3, generator=torch.Generator().manual_seed(991)) < 0.5
    # region selection: raw heads of three images (9 classes), 10 boxes kept per image, 5 free rows after them
    g = torch.Generator().manual_seed(995)
    dets = []
    for n in (40, 7, 25):
        xy = torch.rand(n, 2, generator=g) * 400
        prop = torch.cat([xy, xy + 20 + torch.rand(n, 2, generator=g) * 150], 1)
        dets.append((prop, torch.randn(n, 9, generator=g) * 2, torch.relu(torch.randn(n, F, generator=g)), 1.25))
    w["detections"] = dets
    w["select_text"] = [support.image(t, 1, 996 + i, F, vocab)[:2] + (7,) for i, t in enumerate([6, 13, 2])]
    return w


def _gate_shape(cfg):
    from vilbert_b200.model import head_mask_shape
    return head_mask_shape(cfg)


def _dev(ts):
    return [t.cuda() if torch.is_tensor(t) else t for t in ts]


# ------------------------------------------------------------------------------------------------------------ families
# Each family runs its calls on an engine and returns its outputs as a nested structure.  ``x3``: the engine is fp32x, so only the
# dense parts run.  ``long_rows``: the family's cases past 256 rows run with max_rows_per_sample raised to 1024 for their duration.
@contextlib.contextmanager
def _rows(m, n):
    was = m.max_rows_per_sample
    if n > was:
        m.set_option("max_rows_per_sample", n)
    try:
        yield
    finally:
        if n > was:
            m.set_option("max_rows_per_sample", was)


def _packed_args(samples):
    return support.packed_sample_args(samples)


def fam_forward(m, w, x3):
    from vilbert_b200 import _lib as L
    res = [m(*_dev(w["dense"]), select=L.OUT_ALL, debug_taps=True)]
    with _rows(m, 1024):
        res.append(m(*_dev(w["dense_long"]), select=L.OUT_ALL, debug_taps=True))
    return res


def fam_forward_host(m, w, x3):
    from vilbert_b200 import _lib as L
    res = []
    for key in ("dense", "dense_long"):
        inp = w[key]
        B, Tin, V = inp[0].shape[0], inp[0].shape[1], inp[1].shape[1]
        hin = [_pinned(t) for i, t in enumerate(inp) if i != 6]
        out = {"vil_prediction": torch.full((B, m.num_labels), float("nan")).pin_memory(),
               "vision_logit": torch.full((B, V, 1), float("nan")).pin_memory(),
               "vil_binary_prediction": torch.full((B, 2), float("nan")).pin_memory()}
        sel = L.OUT_VIL_PREDICTION | L.OUT_VISION_LOGIT | L.OUT_VIL_BINARY_PREDICTION
        with _rows(m, 1024 if V > 256 else 0):
            m.forward_host(*hin, out, select=sel, synchronize=False)
            torch.cuda.current_stream().synchronize()
        res.append(out)
    return res


def _regions_dense_args(imgs, num_boxes):
    q, seg = torch.stack([im[0] for im in imgs]), torch.stack([im[1] for im in imgs])
    return (q.cuda(), seg.cuda(), torch.ones_like(q).cuda(), torch.tensor([[im[5]] for im in imgs]).cuda(),
            torch.stack([im[2] for im in imgs]).cuda(), torch.stack([im[3] for im in imgs]).cuda(),
            torch.stack([im[4] for im in imgs]).cuda()), (torch.tensor(num_boxes, dtype=torch.int32) if num_boxes else None)


def fam_forward_regions(m, w, x3):
    from vilbert_b200 import _lib as L
    args, nb = _regions_dense_args(w["regions"], [9, 4, 9])
    res = [m.forward_regions(*args, num_boxes=nb, select=L.OUT_ALL)]
    args, _ = _regions_dense_args(w["regions_long"][:1], None)
    with _rows(m, 1024):
        res.append(m.forward_regions(*args, select=L.OUT_TASK_HEADS))
    return res


def fam_forward_packed(m, w, x3):
    from vilbert_b200 import _lib as L
    if x3:
        return None
    res = [m.forward_packed(*_packed_args(w["packed"]), select=L.OUT_ALL, debug_taps=True),
           m.forward_packed(*_packed_args(w["packed_b"]), select=L.OUT_ALL, max_tokens=30, max_regions=40)]
    with _rows(m, 1024):
        res.append(m.forward_packed(*_packed_args(w["packed_long"]), select=L.OUT_TASK_HEADS, debug_taps=True))
    return res


def fam_forward_regions_packed(m, w, x3):
    from vilbert_b200 import _lib as L
    if x3:
        return None
    res = [m.forward_regions_packed(*support.packed_image_args(w["regions_packed"]), select=L.OUT_ALL, debug_taps=True)]
    with _rows(m, 1024):
        res.append(m.forward_regions_packed(*support.packed_image_args(w["regions_long"]), select=L.OUT_TASK_HEADS))
    return res


def fam_gated(m, w, x3):
    from vilbert_b200 import _lib as L
    if x3:
        return None
    gate, gate_b = w["gate"].cuda(), w["gate_b"].cuda()
    res = [m.forward_packed(*_packed_args(w["packed"]), select=L.OUT_TASK_HEADS, debug_taps=True, head_mask=gate),
           m.forward_packed(*_packed_args(w["packed"]), select=L.OUT_TASK_HEADS, debug_taps=True, head_mask=gate_b),
           m.forward_regions_packed(*support.packed_image_args(w["regions_packed"]), select=L.OUT_TASK_HEADS, head_mask=gate)]
    with _rows(m, 1024):               # the streaming attention kernels with gates
        res.append(m.forward_packed(*_packed_args(w["packed_long"]), select=L.OUT_TASK_HEADS, debug_taps=True, head_mask=gate[:2]))
        res.append(m.forward_regions_packed(*support.packed_image_args(w["regions_long"]), select=L.OUT_TASK_HEADS,
                                            head_mask=gate_b[:2]))
    return res


def fam_cached(m, w, x3):
    from vilbert_b200 import _lib as L
    cap, gal = w["captions"], w["gallery"]
    task = torch.full((3, 1), 7, dtype=torch.long).cuda()
    ts = m.encode_text(cap[0].cuda(), cap[3].cuda(), cap[4].cuda(), task)
    vs = m.encode_image(gal[1].cuda(), gal[2].cuda(), gal[5].cuda())
    ti, ii = torch.tensor([0, 1, 2, 2, 0], dtype=torch.int32), torch.tensor([1, 0, 1, 0, 0], dtype=torch.int32)
    res = [ts, vs, m.forward_cached(ts, ti, vs, ii, select=L.OUT_TASK_HEADS)]
    long = w["gallery_long"]
    with _rows(m, 1024):
        vl = m.encode_image(long[1].cuda(), long[2].cuda(), long[5].cuda())
        res += [vl, m.forward_cached(ts, torch.tensor([2], dtype=torch.int32), vl, torch.tensor([0], dtype=torch.int32),
                                     select=L.OUT_TASK_HEADS)]
    return res


def fam_cached_packed(m, w, x3):
    from vilbert_b200 import _lib as L
    if x3:
        return None
    caps, imgs = w["packed"], w["packed_b"]
    q, f, s, seg, task, nt, nv = _packed_args(caps)
    ts = m.encode_text_packed(q, seg, task, nt)
    q, f, s, seg, task, nt, nv = _packed_args(imgs)
    vs = m.encode_image_packed(f, s, nv)
    rq, rseg, rtask, bf, bx, wh, rnt, rnb = support.packed_image_args(w["regions_packed"])
    rs = m.encode_regions_packed(bf, bx, wh, rnb)
    ti, ii = [0, 1, 2, 3, 3, 0], [3, 2, 0, 1, 1, 3]
    res = [ts, vs, rs, m.forward_cached_packed(ts, ti, vs, ii, select=L.OUT_TASK_HEADS, debug_taps=True),
           m.forward_cached_packed(ts, ti[:4], rs, ii[:4], select=L.OUT_TASK_HEADS)]
    with _rows(m, 1024):
        q, f, s, seg, task, nt, nv = _packed_args(w["packed_long"])
        vl = m.encode_image_packed(f, s, nv)
        res += [vl, m.forward_cached_packed(ts, [1, 2], vl, [0, 1], select=L.OUT_TASK_HEADS)]
    return res


def _selection(m, key, entries, mode):
    """Sets a map or state selection (mask over ``entries`` of the full list, ``mode``) and returns what restores the default."""
    kinds = (m.attention_selection if key == "attention" else m.state_selection)()[0]
    m.set_option(f"{key}_entries", sum(1 << e for e in entries))
    m.set_option(f"{key}_heads" if key == "attention" else "state_rows", mode)
    return lambda: (m.set_option(f"{key}_entries", (1 << len(kinds)) - 1),
                    m.set_option(f"{key}_heads" if key == "attention" else "state_rows", 0))


def fam_attention(m, w, x3):
    n = len(m.attention_selection()[0])
    res = []
    for heads in (0, 1):
        restore = _selection(m, "attention", [0, 3, n - 3, n - 2, n - 1], heads)
        try:
            res.append(m(*_dev(w["dense"]), output_all_attention_masks=True)[9])
            if not x3:
                res.append(m.forward_packed(*_packed_args(w["packed"]), output_all_attention_masks=True)[9])
                with _rows(m, 1024):
                    res.append(m.forward_regions_packed(*support.packed_image_args(w["regions_long"]),
                                                        output_all_attention_masks=True)[0][9])
        finally:
            restore()
    return res


def fam_states(m, w, x3):
    n = len(m.state_selection()[0])
    res = []
    for rows in (0, 1, 2):
        restore = _selection(m, "state", [0, 1, 4, n - 2, n - 1], rows)
        try:
            res.append(m(*_dev(w["dense"]), output_layer_states=True)[1])
            if not x3:
                res.append(m.forward_packed(*_packed_args(w["packed"]), output_layer_states=True)[1])
                with _rows(m, 1024):
                    res.append(m.forward_packed(*_packed_args(w["packed_long"]), output_layer_states=True)[1])
        finally:
            restore()
    return res


def fam_decode(m, w, x3):
    from vilbert_b200 import _lib as L
    inp = _dev(w["dense"])
    out = m(*inp, select=L.OUT_TASK_HEADS)
    msgs = [("1", 0, 1, 5, None), ("15", 1, 2, 10, None), ("12", 0, 3, 2, None), ("13", 2, 1, 3, None), ("7", 0, 3, 3, None),
            ("4", 13, 13, 4, (640, 480))]
    return [out, m.decode_answers(out, msgs, spatials=inp[2].contiguous())]


def _abl_args(imgs):
    return support.packed_image_args(imgs)


def fam_ablation(m, w, x3):
    if x3:
        return None
    a = _abl_args(w["ablation"])
    msgs = [("nlvr2", 0, 2), ("vqa", 2, 1), ("retrieval", 2, 2, None, (1, 3), (0, 2))]
    res = [m.message_ablation(*a, msgs, return_logits=True),
           m.head_ablation(*a, [("vqa", 2, 1, None, (0, 3)), ("snli_ve", 3, 1, 1, (5, 7))], return_logits=True)]
    n_units = 6 + 3                                  # positions 1 .. Tin - 2 of image 2 and its three boxes
    assert w["coalitions"].shape[1] == n_units
    res.append(m.coalition_ablation(*a, [("vqa", 2, 1)], [None], [w["coalitions"].numpy()], return_logits=True))
    res.append(m.shapley(*a, [("vqa", 2, 1), ("nlvr2", 0, 2)], permutations=4, seed=3))
    res.append(m.shapley_interactions(*a, [("vqa", 2, 1)], ["cross"], permutations=2, seed=4))
    with _rows(m, 1024):
        res.append(m.message_ablation(*_abl_args(w["regions_long"][:1]), [("vqa", 0, 1, None, (1, 3), (0, 2))], return_logits=True))
    return res


def fam_select_regions(m, w, x3):
    r = m.select_regions(w["detections"], max_boxes=10, out_rows=10 + 7 + 10 + 5, cls_prob=True, objects=True)
    res = [r]
    if not x3:
        rows = sum(r["n_boxes"])
        text = w["select_text"]
        q, seg = torch.cat([t[0] for t in text]).cuda(), torch.cat([t[1] for t in text]).cuda()
        task = torch.tensor([[t[2]] for t in text]).cuda()
        wh = torch.tensor([[640.0, 480.0], [500.0, 375.0], [320.0, 240.0]]).cuda()
        res.append(m.forward_regions_packed(q, seg, task, r["box_features"][:rows], r["boxes"][:rows], wh, [len(t[0]) for t in text],
                                            r["n_boxes"]))
    return res


def fam_relevance(m, w, x3):
    out = m(*_dev(w["dense"]), output_all_attention_masks=True)
    res = [out[9], m.attention_relevance(out[9])]
    with _rows(m, 1024):
        res.append(m.attention_relevance(m(*_dev(w["dense_long"]), output_all_attention_masks=True)[9]))
        if not x3:
            res.append(m.attention_relevance(m.forward_packed(*_packed_args(w["packed_long"]), output_all_attention_masks=True)[9]))
    if not x3:
        res.append(m.attention_relevance(m.forward_packed(*_packed_args(w["packed"]), output_all_attention_masks=True)[9]))
    return res


FAMILIES = {
    "forward": fam_forward, "forward_host": fam_forward_host, "forward_regions": fam_forward_regions,
    "forward_packed": fam_forward_packed, "forward_regions_packed": fam_forward_regions_packed, "gated": fam_gated,
    "cached": fam_cached, "cached_packed": fam_cached_packed, "attention": fam_attention, "states": fam_states,
    "decode": fam_decode, "ablation": fam_ablation, "select_regions": fam_select_regions, "relevance": fam_relevance,
}
# Outputs a layout leaves unwritten: the rows of a region selection past its images (select_regions' out_rows = 32, 27 used).
TAILS = {"select_regions[0].box_features": 27, "select_regions[0].boxes": 27, "select_regions[0].keep_index": 27,
         "select_regions[0].max_conf": 27, "select_regions[0].cls_prob": 27, "select_regions[0].objects": 27}


PT_KEYS = ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")
PT_LABELS = ("masked_lm_labels", "image_label", "image_target", "next_sentence_label")


def fam_pretraining(m, w, x3):
    """pretraining_heads (with a ranking) and pretraining_objectives (one empty list: NaN, as upstream) on the taps of a dense
    forward, and the model's own scores and losses."""
    import vilbert_b200 as vb
    from vilbert_b200 import _lib as L
    b = w
    dev = [b[k].cuda() for k in PT_KEYS]
    scores = m(*dev, output_all_attention_masks=True)
    losses = m(*dev, *[b[k].cuda() for k in PT_LABELS])
    _, taps = vb.VILBertForVLTasks.forward(m, *dev, None, None, select=0, debug_taps=True)
    heads = m.pretraining_heads(taps, text_rows=[0, 5, 71, 5], image_rows=[1, 32, 0], pair_rows=[2, 0], top_k=4)
    obj = m.pretraining_objectives(taps, text_rows=[3, 40], token_labels=[17, 4], image_rows=[2],
                                   image_targets=torch.softmax(torch.randn(1, m._dims["v_target_size"],
                                                                           generator=torch.Generator().manual_seed(6)), -1),
                                   pair_rows=[], pair_labels=[])
    return [scores, losses, taps, heads, obj]


def run_families(m, w, x3, pt=None, pt_batch=None):
    """Every family once on ``m`` (and the pre-training families on ``pt``), outputs flattened; every buffer poisoned first."""
    out = {}
    with _poisoned():
        for name, fn in FAMILIES.items():
            _flat(fn(m, w, x3), name, out)
        if pt is not None:
            _flat(fam_pretraining(pt, pt_batch, x3), "pretraining", out)
        torch.cuda.synchronize()
    return out


def check_written(tag, out):
    """No float32 output keeps a poisoned element, except the documented tails, which keep all of theirs."""
    for k, t in out.items():
        if not torch.is_tensor(t):
            continue
        if k in TAILS:
            assert torch.equal(_bytes(t[TAILS[k]:]), torch.full_like(_bytes(t[TAILS[k]:]), POISON)), f"{tag}: {k} wrote past its rows"
            t = t[:TAILS[k]]
        assert not _poison_left(t), f"{tag}: {k} has elements no kernel wrote"


# ------------------------------------------------------------------------------------------------------------ engines
def _make(oracle, dtype, opts, cls=None):
    kw = {k: v for k, v in opts.items() if k != "gemm_kernel"}
    m = support.engine(oracle, cls, compute_dtype=dtype, return_attention=True, **kw)
    if "gemm_kernel" in opts:
        m.set_option("gemm_kernel", opts["gemm_kernel"])
    return m


@pytest.fixture(scope="module")
def pt_oracle():
    from oracle import pretraining_ref as P
    return P.build(P.tiny_pretraining_config(), seed=7)


@pytest.fixture(scope="module")
def pt_batch(pt_oracle):
    from vilbert_b200 import synthetic as S
    c = pt_oracle.config
    return S.synthetic_masked_batch(3, 24, 11, seed=5, vocab_size=c.vocab_size, v_feature_size=c.v_feature_size,
                                    v_target_size=c.v_target_size)


@pytest.fixture(scope="module")
def baseline(tiny_oracle, pt_oracle, work, pt_batch):
    """Every family's outputs on a default engine, per compute dtype."""
    import vilbert_b200 as vb
    res = {}
    for dt in DTYPES:
        m, pt = _make(tiny_oracle, dt, {}), _make(pt_oracle, dt, {}, vb.BertForMultiModalPreTraining)
        try:
            res[dt] = run_families(m, work, dt == "fp32x", pt, pt_batch)
        finally:
            m.close()
            pt.close()
        check_written(f"baseline {dt}", res[dt])
    return res


def test_baseline_covers_the_families(baseline):
    """The baseline ran every family in fp16 / bf16 and the dense ones in fp32x, and the fp32x run refuses nothing it was given."""
    for dt in DTYPES:
        got = {k.split("[")[0].split(".")[0] for k in baseline[dt]}
        want = set(FAMILIES) | {"pretraining"}
        if dt == "fp32x":
            want -= {"forward_packed", "forward_regions_packed", "gated", "cached_packed", "ablation"}
        assert got == want, (dt, got ^ want)


def test_fp32x_baseline_against_fp64(tiny_oracle, pt_oracle, baseline, work, pt_batch, parity_log):
    """The fp32x baseline's dense forwards (nine outputs, final states, every map), cached scores and pre-training scores and
    losses against the fp64 oracles at BOUNDS.  Every fp32x row equals this baseline bit for bit, so it holds for them too."""
    from test_gpu_fp32x_fp64 import _check
    b = baseline["fp32x"]
    o64, p64 = X.fp64(tiny_oracle), X.fp64(pt_oracle)
    worst = {}

    def check(tag, **fams):
        _check(tag, parity_log, **fams)
        for fam, errs in fams.items():
            for e in (errs.values() if isinstance(errs, dict) else [e for _, e in errs]):
                worst[fam] = max(worst.get(fam, 0.0), e / X.BOUNDS[fam])

    sched = o64.bert.encoder.schedule()
    for i, key in enumerate(("dense", "dense_long")):
        collect = {}
        ref = o64(*work[key], compute_pretraining_heads=True, output_all_attention_masks=False, collect=collect)
        out = [b.get(f"forward[{i}][0][{j}]") for j in range(9)]
        taps = {k: b[f"forward[{i}][1].{k}"] for k in ("sequence_output_t", "sequence_output_v", "pooled_output")}
        check(f"options_{key}", logits=X.output_errs(out, ref), states=X.state_errs(taps, collect["final"]))
    ref = o64(*work["dense"], compute_pretraining_heads=False, output_all_attention_masks=True)
    check("options_dense_maps", attention=X.attention_errs([_unflat_map(b, "relevance[0]", k, r) for k, r in enumerate(ref[9])], ref[9],
                                                           sched))
    cap, gal = work["captions"], work["gallery"]
    ci, ii = torch.tensor([0, 1, 2, 2, 0]), torch.tensor([1, 0, 1, 0, 0])
    task = torch.full((5, 1), 7, dtype=torch.long)
    ref = o64(cap[0][ci], gal[1][ii], gal[2][ii], cap[3][ci], cap[4][ci], gal[5][ii], None, task, compute_pretraining_heads=False)
    out = [b.get(f"cached[2][{j}]") for j in range(9)]
    check("options_cached", logits=X.output_errs(out, ref))
    inp = [pt_batch[k] for k in PT_KEYS]
    rt, rv, ralign, rattn = p64(*inp)
    check("options_pretraining_scores", logits={"prediction_scores_t": X.rel_err(b["pretraining[0][0]"], rt),
                                                "prediction_scores_v": X.rel_err(b["pretraining[0][1]"], rv),
                                                "seq_relationship_score": X.rel_err(b["pretraining[0][2]"], ralign)},
          attention=X.attention_errs([_unflat_map(b, "pretraining[0][3]", k, r) for k, r in enumerate(rattn)], rattn,
                                     p64.bert.encoder.schedule()))
    labels = [pt_batch[k] for k in PT_LABELS]
    labels[2] = labels[2].double()
    ref = p64(*inp, *labels)
    check("options_pretraining_losses", losses={n: X.rel_err(b[f"pretraining[1][{i}]"], r) for i, (n, r) in
                                                enumerate(zip(("masked_lm_loss", "masked_img_loss", "next_sentence_loss"), ref))})
    parity_log(test="options_fp32x_worst_fraction_of_bound", **worst)
    print("fp32x worst error / bound:", worst)


def _unflat_map(b, name, k, ref):
    """Attention map k of a flattened element 9 (a connection layer: its two directions)."""
    if isinstance(ref, tuple):
        return b[f"{name}[{k}][0]"], b[f"{name}[{k}][1]"]
    return b[f"{name}[{k}]"]


def _evict_all(m, oracle, bound):
    """A plan of a new shape under max_plans = 1 drops every other plan; the bound is then restored."""
    m.set_option("max_plans", 1)
    m(*[t.cuda() for t in support.tiny_inputs(oracle, 1, 5, 5, 1)])
    torch.cuda.synchronize()
    assert support.n_plans(m) == 1
    m.set_option("max_plans", bound)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("row", list(ROWS))
def test_option_row_equals_default(tiny_oracle, pt_oracle, work, pt_batch, baseline, dtype, row):
    """A fresh engine with the row's options: every family's first calls (plan builds: the eager validation pass, then the capture),
    their replays, and their calls after every plan was evicted and rebuilt equal the default engine's bits."""
    import vilbert_b200 as vb
    opts = ROWS[row]
    m, pt = _make(tiny_oracle, dtype, opts), _make(pt_oracle, dtype, opts, vb.BertForMultiModalPreTraining)
    bound = opts.get("max_plans", 24)
    try:
        for attempt in ("first call", "replay", "after eviction"):
            if attempt == "after eviction":
                _evict_all(m, tiny_oracle, bound)
            got = run_families(m, work, dtype == "fp32x", pt, pt_batch)
            assert support.n_plans(m) <= bound
            _compare(f"{row}/{dtype}/{attempt}", got, baseline[dtype])
    finally:
        m.close()
        pt.close()


# ------------------------------------------------------------------------------------------------------------ concurrency
SLEEP_CYCLES = 200_000_000         # ~0.1 s at the H100's 1.98 GHz boost clock


MASK_TOKEN = 103               # [MASK], message_ablation's default
_IN_FLIGHT = []                # what an enqueued call's inputs point at, kept until the test has synchronised the device


def _ablation_enqueued(m, args, msgs, slot):
    """One vb200_message_ablation call that returns as soon as it is enqueued (message_ablation waits for its scores): the segments
    and scores, complete once the stream gets there.  Its segment descriptors sit in the engine's ablation workspace until the gather
    after its forward reads them.  The batch and the message structs stay alive in _IN_FLIGHT."""
    import ctypes as C
    from vilbert_b200 import model as M
    q, seg, task, bf, bx, wh, nt, nb = args
    batch = M.PackedRegionBatch("message_ablation", bf.device, m._dims["v_feature_size"], q, seg, task, bf, bx, wh, nt, nb)
    inp = batch.inputs(0, 0)
    recs, n_floats, arr = m._message_layout(nt, nb, [p for p, _ in M.message_pieces(msgs, nt, nb)])
    logits = M.torch.empty(n_floats, dtype=torch.float32, device=bf.device)
    scores = M.torch.empty(len(recs), 4, dtype=torch.int32, device=bf.device)
    _IN_FLIGHT.append((batch, inp, arr))
    m._call("vb200_message_ablation", C.byref(inp), arr, len(arr), MASK_TOKEN, logits.data_ptr(), scores.data_ptr(), slot)
    return logits, scores


def _concurrent_calls(m, w, eager):
    """(name, stream index, call) of the concurrency workload.  Graph mode: on stream A a packed call on slot 0 and a message ablation
    on slot 5 that does not wait for its scores; then on stream B a packed call of another layout at the same capacities on slot 1, a
    regions-packed call on slot 2, a gated call with another mask on slot 3 and a message ablation of other messages on slot 4, whose
    descriptors go to the workspace the queued ablation's gather is still to read; stream A then gets a second packed layout back to
    back on slot 0.  Eager mode has one slot, and the header's one stream per handle: every call back to back on stream A, slot 0."""
    from vilbert_b200 import _lib as L
    cap = dict(max_tokens=30, max_regions=40)
    slot = (lambda s: 0) if eager else (lambda s: s)
    pa, pb = _packed_args(w["packed"]), _packed_args(w["packed_b"])
    ra, ab = support.packed_image_args(w["regions_packed"]), _abl_args(w["ablation"])
    gate_b = w["gate_b"].cuda()       # every input is on the device before the sleep: a pageable copy would wait for it
    B = 0 if eager else 1
    return [
        ("packed_a", 0, lambda: m.forward_packed(*pa, select=L.OUT_TASK_HEADS, debug_taps=True, slot=slot(0), **cap)),
        ("ablation_a", 0, lambda: _ablation_enqueued(m, ab, [("vqa", 2, 1), ("retrieval", 2, 2)], slot(5))),
        ("packed_b", B, lambda: m.forward_packed(*pb, select=L.OUT_TASK_HEADS, debug_taps=True, slot=slot(1), **cap)),
        ("regions", B, lambda: m.forward_regions_packed(*ra, select=L.OUT_TASK_HEADS, slot=slot(2))),
        ("gated", B, lambda: m.forward_packed(*pa, select=L.OUT_TASK_HEADS, head_mask=gate_b, slot=slot(3), **cap)),
        ("ablation", B, lambda: m.message_ablation(*ab, [("nlvr2", 0, 2), ("vqa", 2, 1)], return_logits=True, slot=slot(4))),
        ("packed_a2", 0, lambda: m.forward_packed(*pb, select=L.OUT_TASK_HEADS, debug_taps=True, slot=slot(0), **cap)),
    ]


@pytest.mark.parametrize("eager", [False, True], ids=["graph", "eager"])
@pytest.mark.parametrize("evict", [False, True], ids=["cached", "evicting"])
def test_calls_behind_a_sleeping_stream(tiny_oracle, work, eager, evict):
    """Calls queued behind ~0.1 s of sleep on stream A, on their own slots and stream B (graph mode) or back to back on stream A
    (eager mode), each equal to the same call run alone.  ``evicting``: max_plans is one below the plans the calls use, so calls
    rebuild plans and evict another slot's plan while its work is still queued; n_plans never exceeds the bound.  The evicting runs
    build plans while stream A still sleeps: the regression case for a build whose zero fills were not ordered before its
    validation pass."""
    m = support.engine(tiny_oracle, compute_dtype="fp16", use_cuda_graph=not eager)
    try:
        calls = _concurrent_calls(m, work, eager)
        with _poisoned():
            alone = {}
            for name, _, fn in calls:
                alone[name] = _flat(fn(), name, {})
                torch.cuda.synchronize()
                _IN_FLIGHT.clear()
        used = support.n_plans(m)
        bound = used - 1 if evict else 24
        if evict:                      # every plan is rebuilt below, and each build past the bound evicts the oldest
            _evict_all(m, tiny_oracle, bound)
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        results = {}
        with _poisoned():
            with torch.cuda.stream(streams[0]):
                torch.cuda._sleep(SLEEP_CYCLES)
            for name, s, fn in calls:
                with torch.cuda.stream(streams[s]):
                    results[name] = fn()
                assert support.n_plans(m) <= bound, name
            torch.cuda.synchronize()
            _IN_FLIGHT.clear()
        for name, _, _ in calls:
            _compare(f"{'eager' if eager else 'graph'}/{name}", _flat(results[name], name, {}), alone[name])
        if eager:
            with pytest.raises(RuntimeError, match="concurrent slots need CUDA-graph plans"):
                m.forward_packed(*_packed_args(work["packed"]), slot=1)
    finally:
        m.close()
