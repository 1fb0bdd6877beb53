"""CPU checks of attention maps by selection: element 9 assembled from fabricated layouts (None positions, connection-layer tuple
halves, the kept head axis of a head-mean entry) and the Python-side validation of attention_entries / attention_heads."""
import pytest
import torch

from vilbert_b200 import model as M

# a schedule T, C, V, C: entries 0 text, 1 / 2 the first connection layer, 3 image, 4 / 5 the second connection layer
KINDS = [0, 2, 3, 1, 2, 3]


def _where(selected):
    where, n = [], 0
    for e in range(len(KINDS)):
        where.append(n if e in selected else -1)
        n += e in selected
    return where


def test_attention_list_positions():
    entries = ["e1", "e3", "e4"]
    attn = M.attention_list(KINDS, _where([1, 3, 4]), entries)
    assert attn == [None, ("e1", None), "e3", ("e4", None)]
    assert M.attention_list(KINDS, _where([2, 5]), ["a", "b"]) == [None, (None, "a"), None, (None, "b")]
    assert M.attention_list(KINDS, list(range(6)), list("abcdef")) == ["a", ("b", "c"), "d", ("e", "f")]


def test_split_packed_attention_selection_head_mean():
    """Selected entries 1 (text->image) and 3 (image) at heads 1: [1, Lq_b, Lk_b] views back to back."""
    t_rows, v_rows = [2, 3], [4, 1]
    tv = sum(t * v for t, v in zip(t_rows, v_rows))
    vv = sum(v * v for v in v_rows)
    layout = [(1, 2, 0), (1, 1, tv)]
    flat = torch.arange(tv + vv, dtype=torch.float32)
    attn = M.split_packed_attention(flat, layout, t_rows, v_rows, (KINDS, _where([1, 3])))
    assert len(attn) == 4 and attn[0] is None and attn[3] == (None, None)
    t2i, img = attn[1][0], attn[2]
    assert attn[1][1] is None
    assert [tuple(x.shape) for x in t2i] == [(1, 2, 4), (1, 3, 1)]
    assert [tuple(x.shape) for x in img] == [(1, 4, 4), (1, 1, 1)]
    assert float(t2i[1].reshape(-1)[0]) == 8 and float(img[0].reshape(-1)[0]) == tv
    assert img[1].data_ptr() == flat.data_ptr() + 4 * (tv + 16)


def test_split_packed_attention_without_selection_is_unchanged():
    layout = [(2, 0, 0), (2, 2, 18), (2, 3, 42)]
    flat = torch.arange(66, dtype=torch.float32)
    a, (b, c) = M.split_packed_attention(flat, layout, [3], [4])
    assert torch.equal(a[0], flat[:18].view(2, 3, 3))
    assert torch.equal(b[0], flat[18:42].view(2, 3, 4)) and torch.equal(c[0], flat[42:].view(2, 4, 3))


def test_mask_bits():
    assert M.attention_mask_bits([0, 5, 29]) == (1 | 1 << 5 | 1 << 29)
    assert M.attention_mask_bits(range(3)) == 7
    assert M.attention_mask_bits((4, 4)) == 16
    for bad, err in (([], ValueError), ([63], ValueError), ([-1], ValueError), (["1"], TypeError), ([True], TypeError),
                     ([1.0], TypeError), ("01", TypeError), (5, TypeError)):
        with pytest.raises(err):
            M.attention_mask_bits(bad)


def test_constructor_validates_selection():
    from oracle import vilbert_ref as R
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(R.tiny_config().to_dict())
    with pytest.raises(ValueError, match="attention_heads"):
        vb.VILBertForVLTasks(cfg, attention_heads="max")
    with pytest.raises(ValueError, match="attention_entries"):
        vb.VILBertForVLTasks(cfg, attention_entries=[])
    with pytest.raises(TypeError, match="attention_entries"):
        vb.VILBertForVLTasks(cfg, attention_entries="0")
    m = vb.VILBertForVLTasks(cfg, attention_entries=[1, 2], attention_heads="mean")
    assert m._opts["attention_entries"] == 6 and m._opts["attention_heads"] == 1
    d = vb.VILBertForVLTasks(cfg)
    assert d._opts["attention_entries"] is None and d._opts["attention_heads"] == 0
