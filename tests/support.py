"""Shared support for the test suites: engine construction, engine queries, seeded input builders and batch-1 reference forwards.

Not a test module: pytest does not collect it.  It holds no checks, because pytest explains a failed check in detail only in test
modules and conftest.py; every check stays in the test file that makes it.  Importing it neither loads libvilbert_b200.so nor
initialises CUDA: vilbert_b200 is imported inside the functions that need it.  Every builder draws from its own seeded generator in a fixed order; where two suites draw in
different orders, both orders are kept as separately named functions so that no suite's inputs change.
"""
import ctypes as C
import socket

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------------------ engines
def engine(oracle, cls=None, **kw):
    """The oracle's weights on cuda:0 in eval mode: VILBertForVLTasks with the oracle's num_labels, or ``cls`` (e.g.
    BertForMultiModalPreTraining) without num_labels.  Every engine option is the caller's keyword."""
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(oracle.config.to_dict())
    if cls is None:
        return vb.VILBertForVLTasks.from_pretrained(oracle.state_dict(), config=cfg, num_labels=oracle.num_labels, **kw).eval().cuda(0)
    return cls.from_pretrained(oracle.state_dict(), config=cfg, **kw).eval().cuda(0)


def engines(oracle, modes, cls=None, **kw):
    """Fixture body: yields {compute_dtype: engine} for ``modes`` and closes every engine afterwards."""
    e = {}
    try:
        for k in modes:
            e[k] = engine(oracle, cls, compute_dtype=k, **kw)
        yield e
    finally:
        for m in e.values():
            m.close()


def one_engine(oracle, cls=None, **kw):
    """Fixture body: yields one engine and closes it afterwards."""
    m = engine(oracle, cls, **kw)
    try:
        yield m
    finally:
        m.close()


def lib():
    """The vilbert_b200._lib module, imported on first use."""
    from vilbert_b200 import _lib as L
    return L


def n_plans(model):
    """The number of plans the engine holds."""
    L = lib()
    v = C.c_int64()
    L.check(L.load().vb200_model_dim(model._handle, b"n_plans", C.byref(v)), model._handle)
    return v.value


def call(name, *args):
    """Call a C-ABI hook on the current stream.  Tensors are passed as themselves and turned into pointers here, so that every
    temporary stays alive until its launch is enqueued (later allocations are then ordered after the kernel on the stream)."""
    L = lib()
    ptrs = [a.data_ptr() if torch.is_tensor(a) else a for a in args]
    L.check(getattr(L.load(), name)(*ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream)), None)


def eq16(a, b):
    """Bit equality of two 16-bit tensors."""
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def eq32(a, b):
    """Bit equality of two 32-bit tensors."""
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def tiny_cfg(**kw):
    """A small BertConfig with the worker's layout (task tokens on), updated by ``kw``."""
    import vilbert_b200 as vb
    d = dict(hidden_size=128, num_attention_heads=2, intermediate_size=256, v_hidden_size=256,
             v_num_attention_heads=2, v_intermediate_size=256, bi_hidden_size=256, bi_num_attention_heads=2,
             bi_intermediate_size=256, vocab_size=512, v_feature_size=64, v_target_size=32,
             max_position_embeddings=64, task_specific_tokens=True)
    d.update(kw)
    return vb.BertConfig(**d)


# Configurations the engine accepts beyond the two model shapes the other suites build (tiny_config and the 268 M model share one
# layer schedule, head sizes 64 / 128 / 128, bi_hidden == v_hidden, widths of 1, 2 or a multiple of 2 column tiles of 128 and task
# tokens on).  Each entry overrides oracle.vilbert_ref.tiny_config; CONFIG_LABELS is the number of answer labels of every entry (a
# ragged N).  tests/test_config_matrix.py pins each entry's schedule and the property it exists for; tests/test_gpu_configs.py runs
# them on the engine.
CONFIG_LABELS = 129
CONFIGS = {
    # connection heads (8 x 64) outnumber the stream heads (text 2 x 128, image 4 x 64); bi_hidden_size != v_hidden_size
    "heads_swapped": dict(hidden_size=256, num_attention_heads=2, v_hidden_size=256, v_num_attention_heads=4, bi_hidden_size=512,
                          bi_num_attention_heads=8),
    # widths of 3 and 5 column tiles; image-embedding K = 200 + 64 = 264
    "odd_widths": dict(hidden_size=384, num_attention_heads=6, intermediate_size=640, v_hidden_size=640, v_num_attention_heads=5,
                       v_intermediate_size=384, bi_hidden_size=384, bi_num_attention_heads=3, v_feature_size=200, v_target_size=37),
    # an image layer ahead of C0, connection layers back to back, both streams ending in a connection layer
    "back_to_back": dict(num_hidden_layers=6, v_num_hidden_layers=4, t_biattention_id=[1, 3, 3, 6], v_biattention_id=[1, 1, 1, 4]),
    # the text stream ends in a connection layer (its tail cannot be pruned), the image stream in an image layer
    "text_ends_in_c": dict(num_hidden_layers=4, v_num_hidden_layers=3, t_biattention_id=[2, 4], v_biattention_id=[0, 1]),
    # no connection layer: the retrieval suffix is the heads alone
    "no_coattention": dict(num_hidden_layers=3, v_num_hidden_layers=2, t_biattention_id=[], v_biattention_id=[]),
    # the multi-task heads without the task row
    "no_task_tokens": dict(task_specific_tokens=False),
    # the text embedding at its 1024-wide limit, 8 x 128 text heads
    "wide_text": dict(hidden_size=1024, num_attention_heads=8, intermediate_size=1024, num_hidden_layers=2, v_num_hidden_layers=2,
                      t_biattention_id=[1], v_biattention_id=[1]),
}


def config_oracle(name):
    """The fp32 oracle of CONFIGS[name] with seeded synthetic weights (seed 7, CONFIG_LABELS answer labels)."""
    from oracle import vilbert_ref as R
    return R.build(R.tiny_config(**CONFIGS[name]), seed=7, num_labels=CONFIG_LABELS)


def free_port():
    """A free TCP port on 127.0.0.1 for a gloo process group."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# ------------------------------------------------------------------------------------------------------------ inputs
def tiny_inputs(oracle, B, Tin, V, seed, pad=0):
    """oracle.vilbert_ref.make_inputs on the host, with the features cut to the oracle's v_feature_size."""
    from oracle import vilbert_ref as R
    inp = list(R.make_inputs(B, Tin, V, seed=seed, vocab_size=oracle.config.vocab_size, pad_regions=pad))
    inp[1] = inp[1][..., :oracle.config.v_feature_size].contiguous()
    return inp


def sample(tin, v, seed, F, vocab):
    """One packed request's real rows: (token ids [tin], segments [tin], features [v, F], spatials [v, 5], task id): relu features,
    boxes in [0, 1], the global box first."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(1, vocab, (tin,), generator=g)
    f = torch.relu(torch.randn(v, F, generator=g)) * 1.5
    x1, y1 = torch.rand(v, generator=g) * 0.7, torch.rand(v, generator=g) * 0.7
    x2, y2 = x1 + 0.05 + torch.rand(v, generator=g) * 0.25, y1 + 0.05 + torch.rand(v, generator=g) * 0.25
    s = torch.stack([x1, y1, x2.clamp(max=1.0), y2.clamp(max=1.0), (x2 - x1) * (y2 - y1)], dim=-1)
    s[0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
    seg = torch.randint(0, 2, (tin,), generator=g)
    task = int(torch.randint(0, 20, (1,), generator=g))
    return q, seg, f, s, task


def batch(model, lens, seed):
    """sample() for every (tin, v) in ``lens``, seeds seed, seed + 1, ..., at the engine's feature size and vocabulary."""
    F, vocab = model._dims["v_feature_size"], model._dims["vocab_size"]
    return [sample(t, v, seed + i, F, vocab) for i, (t, v) in enumerate(lens)]


def image(tin, n, seed, F, vocab, wh=(640, 480)):
    """One detector-output sample: (token ids [tin], segments [tin], box features [n, F], pixel boxes [n, 4] inside the image,
    image size [2], task id)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(1, vocab, (tin,), generator=g)
    seg = torch.randint(0, 2, (tin,), generator=g)
    f = torch.relu(torch.randn(n, F, generator=g)) * 1.5
    w, h = wh
    x1, y1 = torch.rand(n, generator=g) * 0.7 * w, torch.rand(n, generator=g) * 0.7 * h
    x2 = torch.minimum(x1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * w, torch.tensor(float(w)))
    y2 = torch.minimum(y1 + (0.05 + 0.25 * torch.rand(n, generator=g)) * h, torch.tensor(float(h)))
    task = int(torch.randint(0, 20, (1,), generator=g))
    return q, seg, f, torch.stack([x1, y1, x2, y2], 1), torch.tensor([float(w), float(h)]), task


def packed_sample_args(samples):
    """forward_packed's positional arguments for sample() rows, on the device."""
    cat = lambda k: torch.cat([s[k] for s in samples], dim=0).cuda()
    task = torch.tensor([[s[4]] for s in samples]).cuda()
    return cat(0), cat(2), cat(3), cat(1), task, [len(s[0]) for s in samples], [s[2].shape[0] for s in samples]


def packed_image_args(imgs):
    """forward_regions_packed's positional arguments for image() rows, on the device."""
    cat = lambda k: torch.cat([im[k] for im in imgs], dim=0).cuda()
    return (cat(0), cat(1), torch.tensor([[im[5]] for im in imgs]).cuda(), cat(2), cat(3), torch.stack([im[4] for im in imgs]).cuda(),
            [len(im[0]) for im in imgs], [im[2].shape[0] for im in imgs])


def _pixel_boxes(g, n, w, h):
    x1, y1 = torch.rand(n, generator=g) * 0.7 * w, torch.rand(n, generator=g) * 0.7 * h
    bw, bh = (0.05 + 0.25 * torch.rand(n, generator=g)) * w, (0.05 + 0.25 * torch.rand(n, generator=g)) * h
    bbox = torch.stack([x1, y1, torch.minimum(x1 + bw, torch.tensor(float(w))), torch.minimum(y1 + bh, torch.tensor(float(h)))], 1)
    return {"image_width": w, "image_height": h, "bbox": bbox.numpy().astype(np.float32)}


def detector_output(n_boxes, F, seed, wh=((640, 480), (500, 375), (320, 240))):
    """Detector output of len(n_boxes) images, (features, infos with pixel boxes), drawn image by image: its features, then its
    boxes."""
    g = torch.Generator().manual_seed(seed)
    feats, infos = [], []
    for i, n in enumerate(n_boxes):
        w, h = wh[i % len(wh)]
        feats.append(torch.relu(torch.randn(n, F, generator=g)) * 1.5)
        infos.append(_pixel_boxes(g, n, w, h))
    return feats, infos


def detector_output_features_first(n_img, n, F, seed, wh=((640, 480), (500, 375), (320, 240))):
    """Detector output of n_img images of n boxes each, (features, infos with pixel boxes), drawn as every image's features first,
    then every image's boxes."""
    g = torch.Generator().manual_seed(seed)
    feats = [torch.relu(torch.randn(n, F, generator=g)) * 1.5 for _ in range(n_img)]
    return feats, [_pixel_boxes(g, n, *wh[i % len(wh)]) for i in range(n_img)]


def split_rows(t, counts):
    """The per-sample blocks of a packed row tensor."""
    offs = np.concatenate([[0], np.cumsum(counts)])
    return [t[offs[i]:offs[i + 1]] for i in range(len(counts))]


def padded_gallery(n_img, F, v_pad=5):
    """A padded image gallery ((features, spatials, image_mask), real box counts): image i has 1 + 7i mod v_pad real rows of value i."""
    lens = [1 + (7 * i) % v_pad for i in range(n_img)]
    f, s, vm = torch.zeros(n_img, v_pad, F), torch.rand(n_img, v_pad, 5), torch.zeros(n_img, v_pad, dtype=torch.uint8)
    for i, k in enumerate(lens):
        f[i, :k], vm[i, :k] = float(i), 1
    return (f, s, vm), lens


# ------------------------------------------------------------------------------------------------------------ batch-1 references
def dense_alone(model, smp, **kw):
    """The dense forward of one sample() as its own batch of one, no padding, with the forward's keywords; synchronised."""
    q, seg, f, s, task = smp
    out = model(q[None].cuda(), f[None].cuda(), s[None].cuda(), seg[None].cuda(), torch.ones(1, len(q), dtype=torch.long).cuda(),
                torch.ones(1, f.shape[0], dtype=torch.uint8).cuda(), None, torch.tensor([[task]]).cuda(), **kw)
    torch.cuda.synchronize()
    return out


def regions_alone(model, im, select, debug_taps=False):
    """vb200_forward_regions of one image() (batch 1, its own Tin and box count, no padding); synchronised.  Returns (the model's
    result, spatials [1, V, 5]); the result is (10-tuple, taps) with ``debug_taps``."""
    L = lib()
    q, seg, f, bx, wh, task = im
    dev = lambda t, dt: torch.as_tensor(t).to(device="cuda", dtype=dt).contiguous()
    q, seg, ones = dev(q[None], torch.int64), dev(seg[None], torch.int64), torch.ones(1, len(q), dtype=torch.int64, device="cuda")
    tk, f, bx = dev([[task]], torch.int64), dev(f[None], torch.float32), dev(bx[None], torch.float32)
    wh = dev(torch.as_tensor(wh)[None], torch.float32)
    n = f.shape[1]
    sp = torch.empty(1, n + 1, 5, device="cuda")
    inp = L.RegionInputs(1, q.shape[1], n, q.data_ptr(), seg.data_ptr(), ones.data_ptr(), tk.data_ptr(), f.data_ptr(), bx.data_ptr(),
                         wh.data_ptr(), None, sp.data_ptr())
    outs, o, select = model._alloc_outputs(1, q.shape[1], n + 1, select, debug_taps, False, torch.device("cuda", 0))
    L.check(L.load().vb200_forward_regions(model._handle, C.byref(inp), C.byref(o), select, 0,
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)), model._handle)
    torch.cuda.synchronize()
    return model._result(outs, 1, q.shape[1], n + 1, debug_taps), sp
