"""References for the attention relevance (vb200_attention_relevance, model.attention_relevance): the residual-weighted attention
rollout (Abnar & Zuidema 2020) through both ViLBERT streams, for one sample's maps.  CPU only; checked by
tests/test_attention_relevance.py and used by tests/test_gpu_attention_relevance.py.

One sample has T text rows (task token included) and V image rows, positions 0..T-1 text and T..T+V-1 image.  ``maps`` is the list
of the sample's entries in execution order, entry e a ``[heads, Lq, Lk]`` array of kind ``kinds[e]``: 0 text layer [T, T], 1 image
layer [V, V], 2 / 3 the two directions of a connection layer ([T, V] text queries over image keys, then [V, T]), always adjacent.
A step is one text layer, one image layer or one connection layer (both directions: they read the same pre-layer streams).  Step l
maps a row i it writes to 0.5 (e_i + M_l[i, :]) and leaves the others e_i, M_l its head-mean map in its block; the result is rows
0 (text CLS) and T (image global row) of R = W_n ... W_1, [2, T + V].
"""
from __future__ import annotations

import numpy as np


def steps(kinds):
    """The steps of a kind list: tuples of entry indices, (e,) for a text or image layer, (e, e + 1) for a connection layer."""
    out, e = [], 0
    while e < len(kinds):
        if kinds[e] == 2:
            assert kinds[e + 1] == 3, "a kind-2 entry is followed by its kind-3 direction"
            out.append((e, e + 1))
            e += 2
        else:
            assert kinds[e] in (0, 1), kinds[e]
            out.append((e,))
            e += 1
    return out


def head_mean(p, dtype=np.float32):
    """[heads, Lq, Lk] -> [Lq, Lk]: the heads summed left to right from 0 in ``dtype``, then divided once by the head count (the
    engine's head mean; the identity for one head)."""
    p = np.asarray(p, dtype=dtype)
    s = np.zeros(p.shape[1:], dtype=dtype)
    for h in range(p.shape[0]):
        s = s + p[h]
    return s / dtype(p.shape[0])


def _blocks(kind, T, V):
    """(query position offset, key position offset) of an entry's map among the T + V positions."""
    return {0: (0, 0), 1: (T, T), 2: (0, T), 3: (T, 0)}[kind]


def rollout_vector(maps, kinds, T, V, dtype=np.float32):
    """The normative evaluation: r = e_0 and e_T, multiplied by W_l from the last step to the first.  For every column j a step's
    map covers, acc_j = sum over its query rows i in increasing order of r_i * Abar[i, j] (each product and each add one rounding
    in ``dtype``, from 0), then r_j = 0.5 * (r_j + acc_j); other columns keep r_j.  Both directions of a connection step read the
    old r."""
    N = T + V
    r = np.zeros((2, N), dtype=dtype)
    r[0, 0] = 1
    r[1, T] = 1
    half = dtype(0.5)
    for step in reversed(steps(kinds)):
        acc = np.zeros((2, N), dtype=dtype)
        covered = np.zeros(N, dtype=bool)
        for e in step:
            a = head_mean(maps[e], dtype)
            q0, k0 = _blocks(kinds[e], T, V)
            lq, lk = a.shape
            for i in range(lq):
                acc[:, k0:k0 + lk] = acc[:, k0:k0 + lk] + r[:, q0 + i:q0 + i + 1] * a[i][None, :]
            covered[k0:k0 + lk] = True
        r[:, covered] = half * (r[:, covered] + acc[:, covered])
    return r


def attention_relevance_f32(maps, kinds, T, V):
    """The kernel's result, bit for bit: ``rollout_vector`` in float32."""
    return rollout_vector(maps, kinds, T, V, np.float32)


def step_matrix(maps, kinds, step, T, V):
    """W of one step in float64, [T + V, T + V]."""
    N = T + V
    M = np.zeros((N, N))
    written = np.zeros(N, dtype=bool)
    for e in step:
        a = head_mean(maps[e], np.float64)
        q0, k0 = _blocks(kinds[e], T, V)
        M[q0:q0 + a.shape[0], k0:k0 + a.shape[1]] = a
        written[q0:q0 + a.shape[0]] = True
    W = np.eye(N)
    W[written] = 0.5 * (W[written] + M[written])
    return W


def attention_relevance_f64(maps, kinds, T, V):
    """The definition as a matrix product in float64: rows 0 and T of R = W_n ... W_1."""
    R = np.eye(T + V)
    for step in steps(kinds):
        R = step_matrix(maps, kinds, step, T, V) @ R
    return R[[0, T]]


def sample_maps(attn, b):
    """Sample b's entries in execution order from element 9 (every entry present): numpy float32 ``[heads, Lq, Lk]`` each."""
    out = []
    for pos in attn:
        for x in (pos if isinstance(pos, tuple) else (pos,)):
            m = x[b]
            out.append(np.asarray(m.detach().cpu().numpy() if hasattr(m, "detach") else m, dtype=np.float32))
    return out
