"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  Checkpoint-like weights from a seed: an oracle at the statistics of a trained model.

``init_weights`` (oracle/vilbert_ref.py) draws N(0, 0.02) matrices and LayerNorms near the identity.  At those weights attention is
almost uniform, no FFN leaves the GELU's linear region and every 16-bit operand has magnitude about 1, so a kernel or wiring mistake
that only shows where a trained checkpoint runs passes every model-level check.  ``trained_like(oracle, seed)`` returns a copy of an
oracle (reduced-width or 268 M) whose state_dict keeps the key names, shapes and dtypes and has these statistics instead:

* peaked attention: Q and K read the ordinary channels only (the outlier channels below would put single Q / K elements in the
  thousands), queries and keys are centred on the calibration rows, and every head's Q and K rows are scaled so that the non-sink
  heads' median row maximum reaches ``SHARP``, from the first head at SHARP[0] to the mildest at SHARP[1], with no Q or K element past
  OPERAND_CAP (64) on the calibration batch: the sharpness comes from how queries and keys align.  The argmax of a sharp head lands
  on any key, so past 64 keys the running max rises mid-row;
* sink heads: in every other schedule step the last head of each direction is made to put ``SINK`` of its mass (median over query
  rows) on key 0, the [CLS] row or the image global row.  The [CLS] word embedding and position 0 get a direction, and so does the
  area column of the image location embedding (1 on the global row, under 0.1 on a box).  The head's key weight gains a rank-one
  term along the direction separating key 0 from the other keys in the calibration states (which the other heads' keys no longer
  see), and its query bias a matching constant, scaled until the target is met; where no scale under OPERAND_CAP meets it the head
  becomes a mild head instead;
* GELU past saturation: in every FFN, 3 % of the intermediate units get a bias of 5 to 12 in magnitude (one of 14) and 3x their
  weight row, so at least 1 % of pre-activations exceed the polynomial GELU's saturation at |x| = 4.3 and the largest passes 10;
* outlier channels: per stream, three channels carry |beta| in [5, 20] in every LayerNorm of that stream, and one channel gets an
  FFN output-dense bias of 100 to 130 in two FFNs of the stream, so the fp32 sum before those LayerNorms reaches |x| >= 100.  Every
  LayerNorm's gamma on the ordinary channels is then scaled, as it first runs on the calibration batch, so that they leave it with
  unit rms: otherwise the outliers' share of the variance would shrink the rows' differences at every LayerNorm.

Every calibration runs in fp64, one schedule step at a time on the previous steps' calibrated states; every scale is chosen from a
fixed grid of powers of 2^(1/4), and the build runs on one thread, so the same seed gives the same state_dict bit for bit (DIGESTS).  Linear weights are finally rounded to
bf16-representable values, as ``init_weights`` leaves them.  ``attention_regime`` and ``activation_regime`` measure the targets (tests/test_trained_like.py on the
fp32 oracle, tests/test_gpu_trained_like.py on the engine's own maps).
"""
from __future__ import annotations

import copy
import math

import torch
from torch import nn

from oracle import vilbert_ref as R

SEED = 1                     # the seed every test and scripts/step_parity_sweep.py --weights trained use
SHARP = (0.95, 0.3)           # median row-max of the sharpest and the mildest non-sink head of a layer (linear in between)
SINK = 0.75                  # median mass of a sink head on key 0
GRID = [2.0 ** (i / 4) for i in range(-8, 100)]
CLS_ID = 101
FFN_SAT_SHARE = 0.03         # share of an FFN's intermediate units pushed past the GELU saturation
LN_OUTLIERS = 3              # LayerNorm channels per stream with |beta| in [5, 20]
KEY_BLOCK = 64
OPERAND_CAP = 64.0         # no calibrated Q or K element past this on the calibration batch

# digest() of trained_like(..., SEED) for the reduced-width oracle of tests/conftest.py, its 1024-position variant and the 268 M
# oracle: the weights the bounds of oracle/step_ref.py STEP_BOUNDS_TRAINED and oracle/fp64.py BOUNDS_TRAINED were measured on
DIGESTS = {"tiny": "7e8443f4587e929b4cde68fb02942a2d12ea55c4fc9c047f40385336929cf3a6",
           "long": "9bd14aaf7ea412f69de1289ad03ba92bbd56a1158c139af0a95e18793e8a8e5e",
           "full": "a9727760b160cbbf0dc9063dfa09464d09f8870f8f31bd698540912848c460e4"}

# targets regime() is checked against (tests/test_trained_like.py, tests/test_gpu_trained_like.py)
TARGETS = {"sharpest_head_rowmax": 0.8, "model_rowmax": 0.4, "late_winner": 0.10, "sink_mass": 0.5, "gelu_sat_share": 0.01,
           "gelu_max": 10.0, "gelu_sat": 4.3, "ln_outlier": (5.0, 20.0), "operand_outlier": 16.0, "residual_outlier": 100.0,
           "operand_max": 4096.0}


def calibration_inputs(config, seed):
    """The calibration batch: two samples, 80 tokens (81 text rows with the task token) and 101 regions, 5 of them padded, so both
    streams have keys past the first 64-key block."""
    inp = list(R.make_inputs(2, 80, 101, seed=seed, vocab_size=config.vocab_size, pad_regions=5))
    inp[1] = inp[1][..., :config.v_feature_size].contiguous()
    return inp


def _stream_layernorms(model, text):
    enc, n = model.bert.encoder, len(model.bert.encoder.c_layer)
    if text:
        out = [model.bert.embeddings.LayerNorm]
        out += [m for lay in enc.layer for m in (lay.attention.output.LayerNorm, lay.output.LayerNorm)]
        out += [m for c in enc.c_layer for m in (c.biOutput.LayerNorm2, c.t_output.LayerNorm)]
    else:
        out = [model.bert.v_embeddings.LayerNorm]
        out += [m for lay in enc.v_layer for m in (lay.attention.output.LayerNorm, lay.output.LayerNorm)]
        out += [m for c in enc.c_layer for m in (c.biOutput.LayerNorm1, c.v_output.LayerNorm)]
    assert n == len(enc.c_layer)
    return out


def _ffns(model, text):
    """(intermediate dense, output dense) of every FFN of a stream."""
    enc = model.bert.encoder
    if text:
        return [(l.intermediate.dense, l.output.dense) for l in enc.layer] + [(c.t_intermediate.dense, c.t_output.dense) for c in enc.c_layer]
    return [(l.intermediate.dense, l.output.dense) for l in enc.v_layer] + [(c.v_intermediate.dense, c.v_output.dense) for c in enc.c_layer]


def _uniform(g, n, lo, hi):
    return lo + (hi - lo) * torch.rand(n, generator=g, dtype=torch.float64)


def _signs(g, n):
    return torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()


def _unit(g, n):
    u = torch.randn(n, generator=g, dtype=torch.float64)
    return u / u.norm()


def _outliers(model, g):
    """LayerNorm outlier channels, residual outlier channels and saturating FFN units: fixed rules, no calibration needed.  Returns
    each stream's outlier channels {True: text, False: image}."""
    chosen = {}
    for text, H in ((True, model.config.hidden_size), (False, model.config.v_hidden_size)):
        chans = torch.randperm(H, generator=g)[:LN_OUTLIERS + 1]
        ln_ch, res_ch = chans[:LN_OUTLIERS], int(chans[LN_OUTLIERS])
        chosen[text] = chans
        for ln in _stream_layernorms(model, text):
            # beta, not gamma: a gamma outlier feeds back through the residual (the next LayerNorm sees gamma z, normalises it to
            # ~sqrt(H) and multiplies by gamma again), until its channel sets every LayerNorm's variance and the ordinary channels
            # shrink by ~gamma; a beta outlier adds the same offset each time and settles
            ln.bias.data[ln_ch] = _signs(g, len(ln_ch)) * _uniform(g, len(ln_ch), 5.0, 20.0)
        ffns = _ffns(model, text)
        for i, (inter, out) in enumerate(ffns):
            n = max(2, math.ceil(FFN_SAT_SHARE * inter.out_features))
            units = torch.randperm(inter.out_features, generator=g)[:n]
            mag = _uniform(g, n, 5.0, 12.0)
            mag[0] = 14.0
            inter.bias.data[units] = _signs(g, n) * mag
            inter.weight.data[units] *= 3.0
            if i in (0, len(ffns) // 2):        # a few residual outliers: each one sets its own LayerNorm's variance
                out.bias.data[res_ch] = float(_signs(g, 1) * _uniform(g, 1, 100.0, 130.0))
    return chosen


def _heads(y, nh):
    B, L, H = y.shape
    return y.view(B, L, nh, H // nh).transpose(1, 2)


def _median_over(x, rows):
    """Median of x [B, h, Lq] over the real query rows ``rows`` [B, Lq] (bool), per head -> [h]."""
    return torch.stack([x[:, h][rows].median() for h in range(x.shape[1])])


def _calibrate_attention(q_lin, k_lin, v_lin, xq, xk, mask, q_rows, k_rows, nh, g, q_out, k_out, sink=True):
    """Scale the heads of one attention (queries from xq through q_lin, keys from xk through k_lin, additive key mask [B, Lk]) to
    their sharpness targets, and (``sink``) turn the last head into a sink on key 0.  q_out / k_out: the outlier channels of the query and key
    streams, which Q and K do not read."""
    d = q_lin.out_features // nh
    with torch.no_grad():
        # Q and K read the ordinary channels only.  An outlier channel (|x| up to ~500) through a scaled Q / K row would put single
        # elements in the thousands, where one 16-bit ulp moves a score by O(10^2); without them the heads get their sharpness from
        # how queries and keys align, with Q and K elements of O(10) as in a trained checkpoint
        q_lin.weight.data[:, q_out] = 0.0
        k_lin.weight.data[:, k_out] = 0.0
        # the direction that sets key 0 apart from the other keys, over the channels K reads
        others = k_rows.clone()
        others[:, 0] = False
        xo = xk.clone()
        xo[..., k_out] = 0.0
        rest = xo[others]
        cov = torch.cov(rest.t())
        cov = cov + 1e-3 * cov.diagonal().mean() * torch.eye(cov.shape[0], dtype=cov.dtype)
        dirn = torch.linalg.solve(cov, xo[:, 0].mean(0) - rest.mean(0))       # the direction separating key 0 best (Fisher)
        dirn = dirn / dirn.norm()
        # what sets key 0 apart is left to the sink head: the other heads' keys do not see it, so their winners fall anywhere
        for h in range(nh - 1 if sink else nh):
            sl = slice(h * d, (h + 1) * d)
            k_lin.weight.data[sl] -= (k_lin.weight.data[sl] @ dirn)[:, None] * dirn[None, :]
        # queries and keys centred on their mean over the real rows.  For the keys that is a per-query constant in every score, so
        # no map moves; for the queries it removes the query-independent score q_mean . k_j, which would otherwise send every
        # query of a scaled head to the same key on this batch only
        k_lin.bias.data -= k_lin(xk)[k_rows].mean(0)
        q_lin.bias.data -= q_lin(xq)[q_rows].mean(0)
        q, k = _heads(q_lin(xq), nh), _heads(k_lin(xk), nh)
        s0 = q @ k.transpose(-1, -2) / math.sqrt(d)
        m = mask[:, None, None, :]
        targets = torch.linspace(SHARP[0], SHARP[1], max(nh - 1, 1), dtype=torch.float64).tolist()
        for h in range(nh - 1):
            _sharpen(q_lin, k_lin, q, k, s0, m, q_rows, h, d, targets[h])
        # the sink: key 0's state differs from the other keys along dirn; the head's keys gain sigma a (dirn . x) and its queries
        # sigma a, so key 0's score rises by ~sigma^2 (dirn . (x_0 - x_j)) / sqrt(d) over every other key's
        h = nh - 1
        if not sink:
            _sharpen(q_lin, k_lin, q, k, s0, m, q_rows, h, d, SHARP[1])
            return False
        sl = slice(h * d, (h + 1) * d)
        a = _unit(g, d)
        proj = xo @ dirn - float((rest @ dirn).mean())                          # [B, Lk], 0 on the mean other key
        qh, kh = q[:, h], k[:, h]
        sigma = None
        for sg in GRID:
            qs, ks = qh + sg * a, kh + sg * proj[..., None] * a
            if max(float(qs.abs().max()), float(ks.abs().max())) > OPERAND_CAP:
                break
            p = torch.softmax(qs @ ks.transpose(-1, -2) / math.sqrt(d) + mask[:, None, :], -1)
            if p[..., 0][q_rows].median() >= SINK:
                sigma = sg
                break
        if sigma is None:          # key 0 not separable enough on these states: a mild head instead
            _sharpen(q_lin, k_lin, q, k, s0, m, q_rows, h, d, SHARP[1])
            return False
        q_lin.bias.data[sl] += sigma * a
        k_lin.weight.data[sl] += sigma * torch.outer(a, dirn)
        k_lin.bias.data[sl] -= sigma * float((rest @ dirn).mean()) * a
        # what the sink passes on: its values without the row-0 direction, so the rows attending to key 0 do not take on what sets
        # key 0 apart (as a trained sink head's values carry little)
        v_lin.weight.data[sl] -= (v_lin.weight.data[sl] @ dirn)[:, None] * dirn[None, :]
    return True


def _sharpen(q_lin, k_lin, q, k, s0, m, q_rows, h, d, target):
    """Scale head h's Q and K rows (weights and biases, sqrt(alpha) each, so its scores scale by alpha) to the smallest grid alpha
    whose median row max reaches ``target``, with no Q or K element past OPERAND_CAP."""
    alpha, big = GRID[0], max(float(q[:, h].abs().max()), float(k[:, h].abs().max()))
    for a in GRID:
        if math.sqrt(a) * big > OPERAND_CAP:
            break
        alpha = a
        p = torch.softmax(a * s0[:, h:h + 1] + m, -1)
        if p.amax(-1)[:, 0][q_rows].median() >= target:
            break
    sl = slice(h * d, (h + 1) * d)
    for lin in (q_lin, k_lin):
        lin.weight.data[sl] *= math.sqrt(alpha)
        lin.bias.data[sl] *= math.sqrt(alpha)


def _unit_rms(keep):
    """A pre-hook that, on its LayerNorm's first call, divides the gamma of the ``keep`` channels by the rms of their normalised
    input, so that they leave with about unit rms whatever the outlier channels do to the variance."""
    def hook(ln, args):
        if getattr(ln, "_calibrated", False):
            return
        x = args[0]
        u = x.mean(-1, keepdim=True)
        z = (x - u) / torch.sqrt((x - u).pow(2).mean(-1, keepdim=True) + ln.variance_epsilon)
        ln.weight.data[keep] /= float(z[..., keep].pow(2).mean().sqrt())
        ln._calibrated = True
    return hook


def trained_like(oracle, seed: int = 0):
    """A copy of ``oracle`` (fp32, left unchanged) with trained-model statistics (module docstring); deterministic in ``seed``."""
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # one summation order for every reduction, whatever the host's core count
    try:
        return _trained_like(oracle, seed)
    finally:
        torch.set_num_threads(threads)


def _trained_like(oracle, seed):
    cfg = oracle.config
    g = torch.Generator().manual_seed(seed)
    m = copy.deepcopy(oracle).double().eval()
    emb, vemb = m.bert.embeddings, m.bert.v_embeddings
    with torch.no_grad():
        u_t, u_v = _unit(g, cfg.hidden_size), _unit(g, cfg.v_hidden_size)
        row = emb.word_embeddings.weight[CLS_ID].norm() + emb.position_embeddings.weight[0].norm()
        emb.word_embeddings.weight.data[CLS_ID] += 0.75 * row * u_t
        emb.position_embeddings.weight.data[0] += 0.75 * row * u_t
        vemb.image_location_embeddings.weight.data[:, 4] += 4.0 * u_v
        out_ch = _outliers(m, g)

        # every LayerNorm's ordinary channels scaled back to unit rms on the calibration batch, as it first runs: the outlier
        # channels set the LayerNorm's variance, and without a matching gamma the rows' differences would shrink by that factor at
        # every LayerNorm until all rows of a sample were alike
        hooks = []
        for text in (True, False):
            keep = torch.ones(cfg.hidden_size if text else cfg.v_hidden_size, dtype=torch.bool)
            keep[out_ch[text]] = False
            for ln in _stream_layernorms(m, text):
                hooks.append(ln.register_forward_pre_hook(_unit_rms(keep)))
        inp = calibration_inputs(cfg, seed + 1)
        txt, feat, loc, seg, in_mask, im_mask, _, task = inp
        t_real = torch.cat([torch.ones_like(in_mask[:, :1]), in_mask], 1).bool() if cfg.task_specific_tokens else in_mask.bool()
        v_real = im_mask.bool()
        t_add, v_add = (~t_real).double() * -10000.0, (~v_real).double() * -10000.0
        t = emb(txt, seg, task)
        v = vemb(feat.double(), loc.double())
        enc = m.bert.encoder
        for i, step in enumerate(enc.schedule()):
            kind, idx = step[0], int(step[1:])
            sink = i % 2 == 0                   # sinks in every other step: the sharp heads keep winners past key 63
            if kind in "TV":
                lay = (enc.layer if kind == "T" else enc.v_layer)[idx]
                x, add, real = (t, t_add, t_real) if kind == "T" else (v, v_add, v_real)
                sa = lay.attention.self
                oc = out_ch[kind == "T"]
                _calibrate_attention(sa.query, sa.key, sa.value, x, x, add, real, real, sa.num_attention_heads, g, oc, oc, sink)
                x = lay(x, add[:, None, None, :])[0]
                if kind == "T":
                    t = x
                else:
                    v = x
            else:
                c = enc.c_layer[idx]
                ba = c.biattention
                _calibrate_attention(ba.query2, ba.key1, ba.value1, t, v, v_add, t_real, v_real, ba.num_attention_heads, g,
                                     out_ch[True], out_ch[False], sink)   # text -> image
                _calibrate_attention(ba.query1, ba.key2, ba.value2, v, t, t_add, v_real, t_real, ba.num_attention_heads, g,
                                     out_ch[False], out_ch[True], sink)   # image -> text
                v, t, _ = c(v, v_add[:, None, None, :], t, t_add[:, None, None, :])
        for h in hooks:
            h.remove()
        for mod in m.modules():
            if isinstance(mod, nn.Linear):
                mod.weight.data = mod.weight.data.to(torch.bfloat16).double()
    return m.float().eval()


# ---------------------------------------------------------------------------------------------------------------- measurement
def map_labels(schedule):
    return [x for s in schedule for x in ((f"{s} text->image", f"{s} image->text") if s[0] == "C" else (s,))]


def attention_regime(maps, schedule, t_real, v_real):
    """Attention statistics of a forward's maps (element 9, fp32 oracle or engine; [B, heads, Lq, Lk] each) over the real query
    rows (t_real [B, T], v_real [B, V] bool): {label: {"rowmax": per-head median row max, "sink": per-head median mass on key 0,
    "late": share of rows whose largest probability is past key 63, over the samples with more than 64 real keys (None
    without one)}}, "model_rowmax": the median row max over
    every real row of every head and map, "late": the share of such rows over every map with more than 64 keys}."""
    flat = [x for mp in maps for x in (mp if isinstance(mp, tuple) else (mp,))]
    labels = map_labels(schedule)
    assert len(flat) == len(labels), (len(flat), len(labels))
    out, all_max, late_n, late_k = {}, [], 0, 0
    for lab, p in zip(labels, flat):
        p = p.detach().double().cpu()
        qk = {"T": (t_real, t_real), "V": (v_real, v_real)}.get(lab[0]) or \
            ((t_real, v_real) if lab.endswith("text->image") else (v_real, t_real))
        rows = qk[0]
        rm = p.amax(-1)
        ent = {"rowmax": _median_over(rm, rows).tolist(), "sink": _median_over(p[..., 0], rows).tolist(), "late": None}
        all_max.append(rm.transpose(0, 1)[:, rows].reshape(-1))
        long_rows = rows & (qk[1].sum(1, keepdim=True) > KEY_BLOCK)        # samples with more than 64 real keys
        if long_rows.any():
            am = p.argmax(-1).transpose(0, 1)[:, long_rows]
            ent["late"] = float((am >= KEY_BLOCK).double().mean())
            late_n += int((am >= KEY_BLOCK).sum())
            late_k += am.numel()
        out[lab] = ent
    return {"maps": out, "model_rowmax": float(torch.cat(all_max).median()), "late": late_n / late_k if late_k else None}


def activation_regime(oracle, inp):
    """The fp32 oracle's activations on ``inp``: per FFN the share of pre-activations past the GELU saturation and the largest
    |pre-activation|; per stream the largest |state| and the largest |fp32 sum| entering a LayerNorm; the largest 16-bit operand
    (every tensor-core GEMM input and every Q / K / V, as oracle/vilbert_ref.py emulate_activation_rounding lists them)."""
    res = {"ffn": {}, "ln_in": {"text": 0.0, "image": 0.0}, "operand_max": 0.0}
    hooks = []
    text_ln = {id(x) for x in _stream_layernorms(oracle, True)}
    sat = TARGETS["gelu_sat"]

    def ffn_hook(name):
        def f(_m, _a, y):
            y = y.detach().abs()
            res["ffn"][name] = (float((y > sat).double().mean()), float(y.max()))
        return f

    def ln_hook(mod, a):
        k = "text" if id(mod) in text_ln else "image"
        res["ln_in"][k] = max(res["ln_in"][k], float(a[0].detach().abs().max()))

    def lin_in(_m, a):
        res["operand_max"] = max(res["operand_max"], float(a[0].detach().abs().max()))

    def lin_out(_m, _a, y):
        res["operand_max"] = max(res["operand_max"], float(y.detach().abs().max()))

    narrow = R.emulate_activation_rounding.NARROW
    for name, mod in oracle.named_modules():
        if name.endswith("intermediate.dense"):
            hooks.append(mod.register_forward_hook(ffn_hook(name)))
        if isinstance(mod, R.BertLayerNorm) and name.startswith("bert.encoder"):
            hooks.append(mod.register_forward_pre_hook(ln_hook))
        if isinstance(mod, nn.Linear) and name not in narrow:
            hooks.append(mod.register_forward_pre_hook(lin_in))
            if name.rsplit(".", 1)[-1] in R.emulate_activation_rounding.QKV:
                hooks.append(mod.register_forward_hook(lin_out))
    collect = {}
    try:
        with torch.no_grad():
            out = oracle(*inp, compute_pretraining_heads=True, output_all_attention_masks=True, collect=collect)
    finally:
        for h in hooks:
            h.remove()
    t_max = max(float(collect[k][0].abs().max()) for k in collect if k != "final")
    v_max = max(float(collect[k][1].abs().max()) for k in collect if k != "final")
    res["state_max"] = {"text": t_max, "image": v_max}
    return res, out


def real_rows(inp, task_tokens=True):
    """(text real rows [B, T], image real rows [B, V]) of make_inputs-style inputs, the task token's row real."""
    m = inp[4].bool()
    if task_tokens:
        m = torch.cat([torch.ones_like(m[:, :1]), m], 1)
    return m, inp[5].bool()


def assert_attention_targets(reg):
    """The attention targets on an ``attention_regime`` result: a head with median row max >= 0.8 in every layer and direction, the
    model's median row max >= 0.4, >= 10 % of rows over more than 64 keys won past key 63, and for each stream's keys (text: text
    layers and image->text; image: image layers and text->image) a head with >= 0.5 of its mass on key 0 for most rows."""
    tg = TARGETS
    flat = [(lab, max(e["rowmax"])) for lab, e in reg["maps"].items()]
    low = [x for x in flat if x[1] < tg["sharpest_head_rowmax"]]
    assert not low, f"layers without a head at median row max {tg['sharpest_head_rowmax']}: {low}"
    assert reg["model_rowmax"] >= tg["model_rowmax"], reg["model_rowmax"]
    assert reg["late"] is not None and reg["late"] >= tg["late_winner"], reg["late"]
    for keys, pick in (("text", lambda l: l[0] == "T" or l.endswith("image->text")),
                       ("image", lambda l: l[0] == "V" or l.endswith("text->image"))):
        best = max((max(e["sink"]), lab) for lab, e in reg["maps"].items() if pick(lab))
        assert best[0] >= tg["sink_mass"], f"no sink head on the {keys} keys' key 0: best {best}"


def digest(model):
    """sha256 of a model's state_dict (names and bytes, in name order): what tests/test_gpu_trained_like.py checks the weights its
    bounds were measured on against."""
    import hashlib
    h = hashlib.sha256()
    sd = model.state_dict()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()
