"""Plain references for the op-level kernel tests (tests/test_gpu_kernel_parity.py): the exact 16-bit conversions the kernels apply,
the fp16 hi / lo split of the fp32-parity mode, a float32 restatement of the detector-output input builder in the region-pack
kernel's order, and an emulation of the tensor-core attention's rounding points.  CPU only; checked by tests/test_kernel_refs.py."""
from __future__ import annotations

import math

import numpy as np
import torch

F16_MAX = 65504.0


# ---------------------------------------------------------------------------------------------------------------- 16-bit rounding
def sat_rn(x: torch.Tensor, f16: bool) -> torch.Tensor:
    """The 16-bit value every saturating kernel store writes for the fp32 value x (common.cuh pack16x2_rt): fp16 clamps to +-65504
    and then rounds to nearest even; bf16 rounds to nearest even."""
    x = x.float()
    if f16:
        return x.clamp(-F16_MAX, F16_MAX).to(torch.float16)
    return x.to(torch.bfloat16)


def sat_rn_bits_np(x: np.ndarray, f16: bool) -> np.ndarray:
    """sat_rn as raw uint16 bits, computed without torch (numpy's fp16 cast; bf16 by integer round-to-nearest-even on the fp32
    bits), so the torch helper above can be checked against an independent implementation.  Finite inputs only."""
    x = np.asarray(x, dtype=np.float32)
    if f16:
        return np.clip(x, -F16_MAX, F16_MAX).astype(np.float16).view(np.uint16)
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bits16(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16)


def split16(x: torch.Tensor) -> torch.Tensor:
    """fp32 [M, K] (K % 64 == 0) -> the fp32-parity operand, fp16 [M, 3K]: per 64 columns hi | lo | hi with hi = sat_rn_fp16(x),
    lo = sat_rn_fp16(x - hi) (common.cuh split_col / split_lo; lo goes through the same saturating store as hi, which only matters
    past 2 x 65504, where x - hi itself leaves the fp16 range)."""
    x = x.float()
    hi = sat_rn(x, True)
    lo = sat_rn(x - hi.float(), True)
    M, K = x.shape
    g = K // 64
    return torch.stack([hi.view(M, g, 64), lo.view(M, g, 64), hi.view(M, g, 64)], dim=2).reshape(M, 3 * K).contiguous()


# ---------------------------------------------------------------------------------------------------------------- region pack
def region_rows(box_feats: np.ndarray, boxes: np.ndarray, w: float, h: float, nb: int):
    """One image of the region-pack kernel in float32, in the kernel's order of operations (worker.py:422-455 restated):
    box_feats [n, F], boxes [n, 4] pixel x1 y1 x2 y2, nb <= n valid boxes.  Returns (operand rows [n + 1, F] fp32, locations
    [n + 1, 5] fp32, real-row flags [n + 1]).  Row 0 is the mean of the valid boxes -- a sequential fp32 sum divided by max(nb, 1),
    so nb = 0 gives a zero row --, padded boxes are zero rows; the area (y2 - y1)(x2 - x1) / float(w h) is taken before the
    coordinates are divided by w and h."""
    box_feats = np.asarray(box_feats, dtype=np.float32)
    boxes = np.asarray(boxes, dtype=np.float32)
    n, F = box_feats.shape
    rows = np.zeros((n + 1, F), dtype=np.float32)
    s = np.zeros(F, dtype=np.float32)
    for r in range(nb):
        s = s + box_feats[r]                                     # float32 + float32, one box at a time
    rows[0] = s / np.float32(max(nb, 1))
    rows[1:nb + 1] = box_feats[:nb]
    w32, h32 = np.float32(w), np.float32(h)
    wh = np.float32(float(w32) * float(h32))
    loc = np.zeros((n + 1, 5), dtype=np.float32)
    loc[0] = [0, 0, 1, 1, 1]
    b = boxes[:nb]
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    loc[1:nb + 1, 4] = (y2 - y1) * (x2 - x1) / wh
    loc[1:nb + 1, 0] = x1 / w32
    loc[1:nb + 1, 1] = y1 / h32
    loc[1:nb + 1, 2] = x2 / w32
    loc[1:nb + 1, 3] = y2 / h32
    real = np.zeros(n + 1, dtype=bool)
    real[:nb + 1] = True
    return rows, loc, real


def operand_rows(feat: np.ndarray, loc: np.ndarray, Kp: int) -> np.ndarray:
    """[feat | loc | 0 ...] rows, Kp wide, fp32 (the image operand before its 16-bit conversion)."""
    R, F = feat.shape
    out = np.zeros((R, Kp), dtype=np.float32)
    out[:, :F] = feat
    out[:, F:F + 5] = loc
    return out


# ---------------------------------------------------------------------------------------------------------------- attention
def attention_fp64(q, k, v, mask_add, heads):
    """softmax(Q K^T / sqrt(d) + mask) V in fp64; q [B, Lq, H], k / v [B, Lk, H], mask_add [B, Lk] -> [B, Lq, H] fp64."""
    B, Lq, H = q.shape
    Lk = k.shape[1]
    d = H // heads
    qh = q.double().reshape(B, Lq, heads, d).permute(0, 2, 1, 3)
    kh = k.double().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    vh = v.double().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(d) + mask_add.double()[:, None, None, :]
    return (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(B, Lq, H)


def attention_emulated(q, k, v, mask_add, heads, f16: bool):
    """The tensor-core attention's rounding points on the CPU: fp32 scores and softmax numerators p = exp2(s - max) (log2 domain,
    as attention.cu), the denominator summed from the fp32 p, P rounded to the 16-bit format before P V, the context rounded to the
    16-bit format.  One key block (the kernel's online softmax over 64-key blocks only rescales by exact powers of the running
    max, which this ignores).  Returns the 16-bit context as fp64 [B, Lq, H]."""
    B, Lq, H = q.shape
    Lk = k.shape[1]
    d = H // heads
    dt = torch.float16 if f16 else torch.bfloat16
    qh = q.float().reshape(B, Lq, heads, d).permute(0, 2, 1, 3)
    kh = k.float().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    vh = v.float().reshape(B, Lk, heads, d).permute(0, 2, 1, 3)
    log2e = 1.4426950408889634
    s = (qh.double() @ kh.double().transpose(-1, -2)).float() * (log2e / math.sqrt(d)) + (mask_add.float() * log2e)[:, None, None, :]
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = (p.to(dt).double() @ vh.double()).float() * (1.0 / l)
    return o.to(dt).double().permute(0, 2, 1, 3).reshape(B, Lq, H)
