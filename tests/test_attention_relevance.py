"""Attention relevance without a GPU: the references of tests/relevance_ref.py against the definition and each other, the Python
buffer lookup of model.attention_relevance, and the C ABI's NULL-handle rejection."""
import ctypes as C

import numpy as np
import pytest
import torch

from relevance_ref import (attention_relevance_f32, attention_relevance_f64, rollout_vector, sample_maps, step_matrix, steps)

# The 12/6/6 configuration's entry kinds in execution order ("T0-5 C0 (T6 V0 C1) ... (T10 V4 C5) V5 T11"): 30 entries
KINDS = [0] * 6 + [2, 3] + [0, 1, 2, 3] * 5 + [1, 0]


def _dims(kind, T, V):
    return {0: (T, T), 1: (V, V), 2: (T, V), 3: (V, T)}[kind]


def _random_maps(kinds, T, V, heads, seed, t_real=None, v_real=None):
    """Row-stochastic maps per entry, [heads, Lq, Lk]; keys past t_real / v_real get probability 0 (a padded dense forward)."""
    g = np.random.default_rng(seed)
    t_real, v_real = t_real or T, v_real or V
    maps = []
    for k in kinds:
        lq, lk = _dims(k, T, V)
        s = g.standard_normal((heads, lq, lk)) * 2
        real = t_real if k in (0, 3) else v_real
        s[..., real:] = -np.inf
        p = np.exp(s - s.max(-1, keepdims=True))
        maps.append((p / p.sum(-1, keepdims=True)).astype(np.float32))
    return maps


def test_kinds_are_the_schedule():
    assert len(KINDS) == 30 and len(steps(KINDS)) == 24


def test_identity_self_attention_leaves_rows():
    T, V = 5, 7
    kinds = [0, 1, 0, 1]
    maps = [np.eye(T if k == 0 else V, dtype=np.float32)[None].repeat(3, 0) for k in kinds]
    r = attention_relevance_f32(maps, kinds, T, V)
    expect = np.zeros((2, T + V), dtype=np.float32)
    expect[0, 0] = expect[1, T] = 1
    assert np.array_equal(r, expect)


def test_connection_one_key_moves_half():
    """A connection step whose maps put all weight on one key moves exactly half of each row's mass to that key."""
    T, V, kt, kv = 4, 6, 2, 3
    a_tv = np.zeros((1, T, V), dtype=np.float32)
    a_tv[..., kv] = 1
    a_vt = np.zeros((1, V, T), dtype=np.float32)
    a_vt[..., kt] = 1
    r = attention_relevance_f32([a_tv, a_vt], [2, 3], T, V)
    expect = np.zeros((2, T + V), dtype=np.float32)
    expect[0, 0] = expect[0, T + kv] = 0.5           # CLS: half stays, half to the image key its text query reads
    expect[1, T] = expect[1, kt] = 0.5               # image global row: half stays, half to the text key
    assert np.array_equal(r, expect)


def _sequential_f64(maps, kinds, T, V):
    """The wrong reading: each direction of a connection layer as a step of its own, text->image first."""
    R = np.eye(T + V)
    for e in range(len(kinds)):
        R = step_matrix(maps, kinds, (e,), T, V) @ R
    return R[[0, T]]


def test_connection_is_one_step():
    """Hand-built: text queries all read image key 1, image queries all read text key 0 (T = V = 2).  As one step the image global
    row is [0.5, 0, 0.5, 0]; as two sequential steps it would be [0.25, 0, 0.5, 0.25].  Two such layers in a row differ for CLS too."""
    T = V = 2
    a_tv = np.array([[[0, 1], [0, 1]]], dtype=np.float32)
    a_vt = np.array([[[1, 0], [1, 0]]], dtype=np.float32)
    one = attention_relevance_f64([a_tv, a_vt], [2, 3], T, V)
    assert np.array_equal(one[1], [0.5, 0, 0.5, 0])
    assert np.array_equal(_sequential_f64([a_tv, a_vt], [2, 3], T, V)[1], [0.25, 0, 0.5, 0.25])
    assert np.array_equal(attention_relevance_f32([a_tv, a_vt], [2, 3], T, V), one.astype(np.float32))
    two = attention_relevance_f64([a_tv, a_vt] * 2, [2, 3, 2, 3], T, V)
    seq = _sequential_f64([a_tv, a_vt] * 2, [2, 3, 2, 3], T, V)
    assert not np.allclose(two[0], seq[0]) and not np.allclose(two[1], seq[1])
    assert np.array_equal(attention_relevance_f32([a_tv, a_vt] * 2, [2, 3, 2, 3], T, V), two.astype(np.float32))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_vector_order_equals_matrix_product_f64(seed):
    T, V = 9, 13
    maps = _random_maps(KINDS, T, V, heads=3, seed=seed)
    assert np.abs(rollout_vector(maps, KINDS, T, V, np.float64) - attention_relevance_f64(maps, KINDS, T, V)).max() < 1e-14


@pytest.mark.parametrize("heads", [1, 8])
def test_f32_within_1e6_of_f64_at_demo_shape(heads):
    """T = 38 (37 tokens + task token), V = 101 (100 boxes + the global row): the demo's largest shape."""
    T, V = 38, 101
    maps = _random_maps(KINDS, T, V, heads=heads, seed=5 + heads)
    r32 = attention_relevance_f32(maps, KINDS, T, V)
    r64 = attention_relevance_f64(maps, KINDS, T, V)
    assert r32.dtype == np.float32
    assert np.abs(r32 - r64).max() < 1e-6
    assert np.abs(r32.astype(np.float64).sum(1) - 1).max() < 1e-5
    assert np.abs(r64.sum(1) - 1).max() < 1e-6       # the float32 maps' rows sum to 1 within their rounding only
    assert (r32 >= 0).all() and (r32 <= 1).all()


def test_rows_sum_to_one_small_shapes():
    for T, V, seed in ((1, 1, 0), (2, 1, 1), (1, 5, 2), (17, 3, 3)):
        r = attention_relevance_f32(_random_maps(KINDS, T, V, heads=2, seed=seed), KINDS, T, V)
        assert np.abs(r.astype(np.float64).sum(1) - 1).max() < 1e-5, (T, V)


def test_padding_invariance():
    """Maps of a padded dense forward (padded keys at probability 0, padded query rows arbitrary) give the unpadded sample's bits on
    its real columns and exactly 0 on the padded ones."""
    T, V, t_real, v_real = 12, 20, 7, 13
    padded = _random_maps(KINDS, T, V, heads=2, seed=9, t_real=t_real, v_real=v_real)
    real = []
    for k, m in zip(KINDS, padded):
        lq, lk = _dims(k, t_real, v_real)
        real.append(np.ascontiguousarray(m[:, :lq, :lk]))
    rp = attention_relevance_f32(padded, KINDS, T, V)
    rr = attention_relevance_f32(real, KINDS, t_real, v_real)
    cols = np.r_[0:t_real, T:T + v_real]
    assert np.array_equal(rp[:, cols], rr)
    assert np.array_equal(np.delete(rp, cols, axis=1), np.zeros((2, T + V - len(cols)), dtype=np.float32))


def test_head_mean_maps_give_the_same_bits():
    T, V = 6, 9
    maps = _random_maps(KINDS, T, V, heads=4, seed=3)
    from relevance_ref import head_mean
    mean = [head_mean(m)[None] for m in maps]
    assert np.array_equal(attention_relevance_f32(maps, KINDS, T, V), attention_relevance_f32(mean, KINDS, T, V))


# ------------------------------------------------------------------------------------------------------------ Python lookup
def _model():
    from vilbert_b200 import model as M
    return M


def _dense_attn(flat, B, T, V, heads):
    """Element 9 of a dense forward with every entry: views of ``flat`` at the vb200_attention_layout offsets; and the layout."""
    M = _model()
    entries, layout, off = [], [], 0
    for k in KINDS:
        lq, lk = _dims(k, T, V)
        entries.append(flat[off:off + B * heads * lq * lk].view(B, heads, lq, lk))
        layout.append((heads, off))
        off += B * heads * lq * lk
    return M.attention_list(KINDS, list(range(len(KINDS))), entries), layout, off


def test_dense_buffer_lookup():
    M = _model()
    B, T, V, heads = 3, 5, 8, 2
    flat = torch.arange(200000, dtype=torch.float32)
    attn, layout, total = _dense_attn(flat, B, T, V, heads)
    entries, packed, t_rows, v_rows = M.relevance_entries(attn, KINDS)
    assert not packed and t_rows == [T] * B and v_rows == [V] * B
    assert M.maps_pointer(entries, packed, layout) == flat.data_ptr()
    # a buffer that starts inside a larger allocation is found as well
    attn2, layout2, _ = _dense_attn(flat[100:], B, T, V, heads)
    assert M.maps_pointer(M.relevance_entries(attn2, KINDS)[0], False, layout2) == flat.data_ptr() + 400
    # the maps of another layout (a wrong head count) are refused
    with pytest.raises(ValueError, match="not where"):
        M.maps_pointer(entries, packed, [(1, off) for _, off in layout])


def test_packed_buffer_lookup():
    M = _model()
    T_b, V_b, heads = [3, 7], [5, 2], 2
    layout, off = [], 0
    for k in KINDS:
        layout.append((heads, k, off))
        off += heads * sum(lq * lk for lq, lk in (_dims(k, t, v) for t, v in zip(T_b, V_b)))
    flat = torch.zeros(off, dtype=torch.float32)
    attn = M.split_packed_attention(flat, layout, T_b, V_b)
    entries, packed, t_rows, v_rows = M.relevance_entries(attn, KINDS)
    assert packed and t_rows == T_b and v_rows == V_b
    assert M.maps_pointer(entries, packed, [(h, o) for h, _, o in layout]) == flat.data_ptr()
    maps = sample_maps(attn, 1)
    assert [m.shape for m in maps[6:8]] == [(heads, 7, 2), (heads, 2, 7)]


def test_none_entry_is_rejected():
    M = _model()
    flat = torch.zeros(100000, dtype=torch.float32)
    attn, _, _ = _dense_attn(flat, 2, 4, 3, 1)
    attn[6] = (attn[6][0], None)
    with pytest.raises(ValueError, match="entry 7 is None"):
        M.relevance_entries(attn, KINDS)
    attn[0] = None
    with pytest.raises(ValueError, match="entry 0 is None"):
        M.relevance_entries(attn, KINDS)
    with pytest.raises(ValueError, match="attention entries"):
        M.relevance_entries([], KINDS)


def test_null_handle_rejected_without_device():
    from vilbert_b200 import _lib as L
    lib = L.load()
    n = (C.c_int32 * 1)(4)
    out = torch.zeros(4)
    assert lib.vb200_attention_relevance(None, C.c_void_p(out.data_ptr()), 1, C.cast(n, C.c_void_p), C.cast(n, C.c_void_p), 0,
                                         C.c_void_p(out.data_ptr()), None) == -1          # VB200_ERR_INVALID
