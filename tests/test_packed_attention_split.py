"""CPU checks of split_packed_attention: the flat packed attention buffer (VB200_OUT_ATTENTION_PACKED) as the reference's
attn_data_list, one view per layer and sample at the sample's own lengths."""
import torch

from vilbert_b200 import model as M


def _layout(schedule, heads, t_rows, v_rows):
    """The layout vb200_attention_layout_packed documents, built on the host: entries in execution order, each entry's samples back to
    back at heads * Lq_b * Lk_b floats."""
    tt = sum(t * t for t in t_rows)
    vv = sum(v * v for v in v_rows)
    tv = sum(t * v for t, v in zip(t_rows, v_rows))
    out, off = [], 0
    for step in schedule:
        for kind, n in ({"T": [(0, tt)], "V": [(1, vv)], "C": [(2, tv), (3, tv)]}[step]):
            out.append((heads[kind], kind, off))
            off += heads[kind] * n
    return out, off


def test_split_packed_attention_views_cover_the_buffer_in_order():
    schedule = ["T", "V", "C", "T", "C", "V"]
    heads = {0: 3, 1: 2, 2: 4, 3: 4}
    t_rows, v_rows = [2, 33, 1], [1, 5, 64]
    layout, total = _layout(schedule, heads, t_rows, v_rows)
    flat = torch.arange(total, dtype=torch.float32)
    attn = M.split_packed_attention(flat, layout, t_rows, v_rows)
    assert len(attn) == len(schedule)
    pos = 0
    for step, a in zip(schedule, attn):
        if step == "C":
            assert isinstance(a, tuple) and len(a) == 2
            parts = [(a[0], 2), (a[1], 3)]
        else:
            assert isinstance(a, list)
            parts = [(a, 0 if step == "T" else 1)]
        for per, kind in parts:
            assert len(per) == len(t_rows)
            lq_rows = t_rows if kind in (0, 2) else v_rows
            lk_rows = t_rows if kind in (0, 3) else v_rows
            for b, x in enumerate(per):
                assert tuple(x.shape) == (heads[kind], lq_rows[b], lk_rows[b])
                assert x.is_contiguous() and x.data_ptr() == flat.data_ptr() + 4 * pos    # a view, at the next float
                assert float(x.reshape(-1)[0]) == pos
                pos += x.numel()
    assert pos == total


def test_split_packed_attention_one_sample_one_layer():
    layout, total = _layout(["T"], {0: 2}, [3], [4])
    flat = torch.arange(total, dtype=torch.float32)
    (per,) = M.split_packed_attention(flat, layout, [3], [4])
    assert len(per) == 1 and torch.equal(per[0], flat.view(2, 3, 3))
