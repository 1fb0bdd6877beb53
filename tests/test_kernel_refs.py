"""CPU checks of the references the op-level kernel tests rely on (oracle/kernel_refs.py): exact 16-bit rounding, the fp16 hi / lo
split, the float32 region-pack restatement against worker_api.build_inputs, and the attention rounding floor the GPU bounds rest on."""
import numpy as np
import pytest
import torch

from oracle import kernel_refs as R
from vilbert_b200 import worker_api as W


def _edge_values():
    one = np.float32(1.0)
    ulp_f16, ulp_bf16 = np.float32(2.0 ** -10), np.float32(2.0 ** -7)
    v = [0.0, -0.0, 1.0, -1.0, 65504.0, -65504.0, 65519.0, 65519.996, 65520.0, -65520.0, 65536.0, 1e5, -1e5, 3.0e38, -3.0e38,
         6.1e-5, 5.96e-8, 2.98e-8, 8.9e-8, 1e-40,
         one + ulp_f16 / 2, one + 3 * ulp_f16 / 2, one + ulp_bf16 / 2, one + 3 * ulp_bf16 / 2,   # ties: to the even neighbour
         -(one + ulp_f16 / 2), -(one + 3 * ulp_bf16 / 2), 2049.0, 2051.0, 4097.0, 257.0, 259.0]
    return np.array(v, dtype=np.float32)


@pytest.mark.parametrize("f16", [True, False], ids=["fp16", "bf16"])
def test_sat_rn_matches_independent_rounding(f16):
    """sat_rn (torch) == the numpy / integer implementation bit for bit: ties, +-65504, 65520 (the fp16 tie that rounds to inf
    without the clamp), huge values, subnormals, and a million random values over many binades."""
    g = np.random.default_rng(0)
    rnd = (g.standard_normal(1 << 20) * np.exp2(g.integers(-30, 30, 1 << 20))).astype(np.float32)
    x = np.concatenate([_edge_values(), rnd])
    got = R.bits16(R.sat_rn(torch.from_numpy(x), f16)).numpy().view(np.uint16)
    assert np.array_equal(got, R.sat_rn_bits_np(x, f16))


def test_sat_rn_edges():
    t = torch.tensor([65504.0, 65519.0, 65520.0, 1e5, -1e5, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11])
    h = R.sat_rn(t, True).float().tolist()
    assert h == [65504.0, 65504.0, 65504.0, 65504.0, -65504.0, 1.0, 1.0 + 2.0 ** -9]
    assert torch.isinf(torch.tensor([65520.0]).half()).all()          # what a store without the clamp would write
    b = R.sat_rn(torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1e5]), False).float().tolist()
    assert b == [1.0, 1.0 + 2.0 ** -6, 99840.0]


def test_split16_matches_gemm_test_helper():
    """The hi / lo split helper equals the one the fp32-parity GEMM tests build their operands with, and hi + lo carries x to
    2^-22 relative."""
    from test_gpu_ops import _split_act
    g = torch.Generator().manual_seed(3)
    x = torch.randn(37, 256, generator=g) * torch.exp2(torch.randint(-12, 12, (37, 256), generator=g).float())
    x[0, :4] = torch.tensor([7e4, -7e4, 65504.0, 1e-9])
    got = R.split16(x)
    assert torch.equal(R.bits16(got), R.bits16(_split_act(x)))
    far = R.split16(torch.full((1, 64), 1e6)).view(3, 64).float()         # past 2 x 65504 the lo part saturates too
    assert far[0].eq(65504).all() and far[1].eq(65504).all()
    v = got.view(37, 4, 3, 64)
    assert torch.equal(R.bits16(v[:, :, 0]), R.bits16(v[:, :, 2]))
    back = (v[:, :, 0].float() + v[:, :, 1].float()).reshape(37, 256)
    ok = x.abs() <= 65504
    assert ((back - x).abs()[ok] <= x.abs()[ok] * 2.0 ** -21 + 2.0 ** -24).all()


class _Tok:
    def encode(self, s):
        return [5, 6, 7]

    def add_special_tokens_single_sentence(self, ids):
        return [2] + ids + [3]


@pytest.mark.parametrize("n,F", [(7, 2048), (36, 2048), (1, 64), (100, 40)])
def test_region_restatement_matches_build_inputs(n, F):
    """The float32 region-pack restatement against the host input builder: box rows and spatials bit for bit; the mean row (torch.sum
    adds in its own order) within one unit in the last place of the 16-bit formats."""
    g = np.random.default_rng(n * F)
    feats = (g.random((n, F), dtype=np.float32) * g.choice([0.01, 1.0, 300.0], size=(n, F))).astype(np.float32)
    x1 = g.integers(0, 300, n).astype(np.float32)
    y1 = g.integers(0, 200, n).astype(np.float32)
    boxes = np.stack([x1, y1, x1 + g.integers(1, 300, n), y1 + g.integers(1, 250, n)], axis=1).astype(np.float32)
    w, h = 640.0, 427.0
    info = {"image_width": w, "image_height": h, "bbox": boxes}
    _, f, s, *_ = W.build_inputs("q", [1], [torch.from_numpy(feats)], [info], torch.device("cpu"), _Tok())
    rows, loc, real = R.region_rows(feats, boxes, w, h, n)
    assert real.all()
    assert np.array_equal(rows[1:], f[0, 1:].numpy())
    assert np.array_equal(loc.view(np.uint32), s[0].numpy().view(np.uint32))
    mean_bi = f[0, 0].numpy()
    for f16 in (True, False):
        ulp = np.float32(2.0 ** (-10 if f16 else -7)) * np.exp2(np.floor(np.log2(np.maximum(np.abs(rows[0]), 2.0 ** -14))))
        assert (np.abs(rows[0] - mean_bi) <= ulp).all()


def test_region_restatement_padding():
    """nb < n: the mean over the valid boxes only, zero rows and zero locations for the padded ones; nb = 0: a zero mean row."""
    g = np.random.default_rng(1)
    feats = g.random((6, 16), dtype=np.float32)
    boxes = np.tile(np.array([[1, 2, 30, 40]], dtype=np.float32), (6, 1))
    rows, loc, real = R.region_rows(feats, boxes, 100.0, 50.0, 3)
    assert np.array_equal(rows[0], ((feats[0] + feats[1]) + feats[2]) / np.float32(3))
    assert not rows[4:].any() and not loc[4:].any() and real.tolist() == [True] * 4 + [False] * 3
    rows, loc, real = R.region_rows(feats, boxes, 100.0, 50.0, 0)
    assert not rows.any() and loc[0].tolist() == [0, 0, 1, 1, 1] and real.tolist() == [True] + [False] * 6


@pytest.mark.parametrize("L,d", [(16, 64), (17, 128), (31, 64), (65, 128), (129, 128), (256, 64)])
def test_attention_rounding_floor(L, d):
    """The CPU emulation of the tensor-core attention's rounding points (16-bit P before P V, 16-bit context) against fp64, at inputs
    like the GPU tests' (N(0, 1) Q / K / V in the 16-bit format, per-sample masks with interior masked keys), as the error over
    max(1, |reference|).  Measured at these shapes: at most 4.4e-3 (bf16) and 6.2e-4 (fp16).  The GPU attention tests bound the
    kernels at 1.2e-2 and 1.5e-3 of the same measure, about twice this floor."""
    heads = 2
    H = heads * d
    g = torch.Generator().manual_seed(L + d)
    for f16, bound in ((False, 1.2e-2), (True, 1.5e-3)):
        dt = torch.float16 if f16 else torch.bfloat16
        qkv = torch.randn(2, L, 3 * H, generator=g).to(dt)
        mask = torch.zeros(2, L)
        mask[0, 1:L:3] = -10000.0
        mask[1, L // 2 + 1:] = -10000.0
        q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
        ref = R.attention_fp64(q, k, v, mask, heads)
        err = ((R.attention_emulated(q, k, v, mask, heads, f16) - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
        assert err < bound / 2, (f16, err)
