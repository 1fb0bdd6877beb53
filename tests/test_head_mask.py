"""Head masks on the CPU: the mask's shape per configuration, its broadcast rules, and the argument errors raised before any engine
call (the GPU behaviour is in test_gpu_head_mask.py)."""
import pytest
import torch

import support


def test_shape_12_6_6():
    import vilbert_b200 as vb
    from vilbert_b200.model import head_mask_shape
    assert head_mask_shape(vb.BertConfig()) == (30, 12)         # 12 text + 6 image layers, 6 connection layers x 2 directions


def test_shape_follows_config():
    from vilbert_b200.model import head_mask_shape
    cfg = support.tiny_cfg(num_hidden_layers=4, v_num_hidden_layers=3, v_biattention_id=[0, 2], t_biattention_id=[1, 3],
                           num_attention_heads=2, v_num_attention_heads=4, bi_num_attention_heads=8)
    assert head_mask_shape(cfg) == (4 + 3 + 2 * 2, 8)


def test_broadcast_and_per_sample():
    from vilbert_b200.model import head_mask_rows
    shape = (30, 12)
    m = torch.rand(shape)
    r = head_mask_rows(m, 3, shape, torch.device("cpu"))
    assert r.shape == (3, 30, 12) and r.dtype == torch.float32 and r.is_contiguous()
    assert all(torch.equal(r[b], m) for b in range(3))
    per = torch.rand(3, *shape, dtype=torch.float64)
    r = head_mask_rows(per, 3, shape, torch.device("cpu"))
    assert r.dtype == torch.float32 and torch.equal(r, per.float())
    r = head_mask_rows(m.tolist(), 2, shape, torch.device("cpu"))           # any array-like
    assert torch.equal(r[1], m)


@pytest.mark.parametrize("bad", [(12, 30), (30,), (2, 30, 12), (3, 30, 11), (1, 3, 30, 12)])
def test_wrong_shapes_rejected(bad):
    from vilbert_b200.model import head_mask_rows
    with pytest.raises(ValueError, match="head_mask has shape"):
        head_mask_rows(torch.ones(bad), 3, (30, 12), torch.device("cpu"))


def test_forward_without_engine_raises():
    import vilbert_b200 as vb
    model = vb.VILBertForVLTasks(support.tiny_cfg(), num_labels=10)
    for fn in (model.forward_packed, model.forward_regions_packed):
        with pytest.raises(vb.VilbertB200Error, match="cuda"):
            fn(*([None] * 8), head_mask=torch.ones(30, 2))
