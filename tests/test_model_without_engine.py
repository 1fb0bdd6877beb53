"""Every engine-backed method of a model without an engine (no .cuda(i) yet) raises VilbertB200Error asking for .cuda(i),
before it creates a CUDA tensor or reaches the library (CPU only)."""
import pytest
import torch

import vilbert_b200 as vb
from vilbert_b200 import _lib as L

F = 256         # v_feature_size of the tiny config
B, TIN, V = 2, 5, 4


def _text():
    return torch.ones(B, TIN, dtype=torch.int64), torch.zeros(B, TIN, dtype=torch.int64), torch.ones(B, TIN, dtype=torch.int64)


def _dense():
    q, seg, im = _text()
    return q, torch.zeros(B, V, F), torch.zeros(B, V, 5), seg, im, torch.ones(B, V, dtype=torch.uint8), torch.zeros(B, 1, dtype=torch.int64)


_DET = [(torch.zeros(8, 4), torch.zeros(8, 3), torch.zeros(8, F), 1.0)]
_TEXT_STATE = dict(kind="text", n=1, Tin=TIN, offsets=torch.tensor([0, TIN + 1], dtype=torch.int32), max_len=TIN)
_IMAGE_STATE = dict(kind="image", n=1, V=V, offsets=torch.tensor([0, V], dtype=torch.int32), max_len=V)

CALLS = {
    "plan_info": lambda m: m.plan_info(1, TIN, V),
    "set_option": lambda m: m.set_option("max_plans", 4),
    "profile_ops": lambda m: m.profile_ops(1, TIN, V),
    "attention_layout": lambda m: m.attention_layout(1, TIN, V),
    "attention_layout_packed": lambda m: m.attention_layout_packed([TIN], [V]),
    "forward": lambda m: m(*_dense()),
    "forward_host": lambda m: m.forward_host(*_dense(), out={"vil_prediction": torch.empty(B, 200)}),
    "forward_regions": lambda m: m.forward_regions(*_text(), torch.zeros(B, 1, dtype=torch.int64), torch.zeros(B, V, F),
                                                   torch.zeros(B, V, 4), torch.ones(B, 2)),
    "forward_packed": lambda m: m.forward_packed(torch.ones(TIN, dtype=torch.int64), torch.zeros(V, F), torch.zeros(V, 5), None,
                                                 None, [TIN], [V]),
    "forward_regions_packed": lambda m: m.forward_regions_packed(torch.ones(TIN, dtype=torch.int64), None, None, torch.zeros(V, F),
                                                                 torch.zeros(V, 4), torch.ones(1, 2), [TIN], [V]),
    "decode_answers": lambda m: m.decode_answers((None,) * 10, [("1", 0, 1, 1, None)]),
    "select_regions": lambda m: m.select_regions(_DET),
    "encode_text": lambda m: m.encode_text(*_text(), torch.zeros(B, 1, dtype=torch.int64)),
    "encode_image": lambda m: m.encode_image(torch.zeros(B, V, F), torch.zeros(B, V, 5), torch.ones(B, V, dtype=torch.uint8)),
    "encode_text_packed": lambda m: m.encode_text_packed(torch.ones(TIN, dtype=torch.int64), torch.zeros(TIN, dtype=torch.int64),
                                                         torch.zeros(1, 1, dtype=torch.int64), [TIN]),
    "encode_image_packed": lambda m: m.encode_image_packed(torch.zeros(V, F), torch.zeros(V, 5), [V]),
    "encode_regions_packed": lambda m: m.encode_regions_packed(torch.zeros(V, F), torch.zeros(V, 4), torch.ones(1, 2), [V]),
    "encode_detections_packed": lambda m: m.encode_detections_packed(_DET, torch.ones(1, 2)),
    "forward_cached": lambda m: m.forward_cached(_TEXT_STATE, torch.zeros(1, dtype=torch.int32), _IMAGE_STATE,
                                                 torch.zeros(1, dtype=torch.int32)),
    "forward_cached_packed": lambda m: m.forward_cached_packed(_TEXT_STATE, [0], _IMAGE_STATE, [0]),
}


@pytest.fixture(scope="module")
def model(tiny_oracle):
    cfg = vb.BertConfig.from_dict(tiny_oracle.config.to_dict())
    assert cfg.v_feature_size == F
    return vb.VILBertForVLTasks.from_pretrained(tiny_oracle.state_dict(), config=cfg, num_labels=200).eval()


@pytest.mark.parametrize("name", sorted(CALLS))
def test_method_without_engine_asks_for_cuda(model, name, monkeypatch):
    def no_library():
        raise AssertionError(f"{name} reached the library without an engine")
    monkeypatch.setattr(L, "load", no_library)
    with pytest.raises(L.VilbertB200Error, match=r"call model\.cuda\(i\) first"):
        CALLS[name](model)
