"""CPU checks of layer states by selection: the vb200_outputs layout against the C compiler, the specified entry list of the 12/6/6
and reduced-width schedules, the Python mask and split helpers, and the errors of a model without an engine."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from vilbert_b200 import _lib as L
from vilbert_b200 import model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cc():
    for name in ("cc", "gcc", "clang"):
        if shutil.which(name):
            return name
    pytest.skip("no C compiler")


def test_outputs_struct_matches_header(tmp_path):
    """vb200_outputs in the header and L.StateOutputs agree on the new last field's offset and the struct size, and the field
    follows every field of L.Outputs, the struct of hosts built before it."""
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "vilbert_b200.h"\n'
                   'int main(void) { printf("%zu %zu %d\\n", offsetof(vb200_outputs, layer_states), sizeof(vb200_outputs), '
                   '(int)VB200_OUT_LAYER_STATES); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([_cc(), "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    off, size, bit = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert off == L.StateOutputs.layer_states.offset == C.sizeof(L.Outputs)
    assert size == C.sizeof(L.StateOutputs)
    assert bit == L.OUT_LAYER_STATES == 1 << 11
    # a free public bit: no overlap with the other select bits or the internal pruning bits (1 << 30, 1 << 31)
    assert not bit & (L.OUT_ALL | L.OUT_ATTENTION | L.OUT_ATTENTION_PACKED | (3 << 30))
    assert L.OUTPUT_FIELDS[-1] == "attention_probs"


def _state_kinds(schedule):
    """The full layer-state list as the engine builds it: text and image embeddings, then per step its text state before its image
    state."""
    kinds = [0, 1]
    for step in schedule:
        if step[0] != "V":
            kinds.append(0)
        if step[0] != "T":
            kinds.append(1)
    return kinds


@pytest.mark.parametrize("cfg", ("full", "tiny"))
def test_entry_list_spec(cfg):
    """The entry list the issue specifies, restated from the schedule; the GPU tests hold the engine's list
    (vb200_state_selection) to this same restatement."""
    from oracle import vilbert_ref as R
    c = R.RefConfig() if cfg == "full" else R.tiny_config()
    schedule = _schedule(c)
    kinds = _state_kinds(schedule)
    assert len(kinds) == 32 and kinds.count(0) == 19 and kinds.count(1) == 13
    # 12/6/6: the last text entry is the last (T11), the last image entry the one of V5, the step before it
    assert schedule[-2:] == ["V5", "T11"]
    assert kinds[-1] == 0 and kinds[-2] == 1
    # a connection layer's two entries are adjacent, text first
    pos = 2
    for step in schedule:
        if step[0] == "C":
            assert kinds[pos:pos + 2] == [0, 1]
        pos += 2 if step[0] == "C" else 1


def _schedule(c):
    order, v_start, t_start = [], 0, 0
    for count, (v_end, t_end) in enumerate(zip(c.v_biattention_id, c.t_biattention_id)):
        order += [f"T{i}" for i in range(t_start, t_end)] + [f"V{i}" for i in range(v_start, v_end)] + [f"C{count}"]
        v_start, t_start = v_end, t_end
    return order + [f"V{i}" for i in range(v_start, c.v_num_hidden_layers)] + [f"T{i}" for i in range(t_start, c.num_hidden_layers)]


def test_state_mask_bits():
    assert M.entry_mask_bits([0, 31], "state_entries") == 1 | 1 << 31
    for bad, err in (([], ValueError), ([63], ValueError), ([-1], ValueError), ([True], TypeError), ("3", TypeError)):
        with pytest.raises(err, match="state_entries"):
            M.entry_mask_bits(bad, "state_entries")
    # the attention wrapper keeps its name in messages
    with pytest.raises(ValueError, match="attention_entries"):
        M.attention_mask_bits([])


def test_state_list_positions():
    assert M.state_list([-1, 0, -1, 1], ["a", "b"]) == [None, "a", None, "b"]
    assert M.state_list([0, 1, 2], list("xyz")) == list("xyz")


def test_split_packed_states():
    t_rows, v_rows = [2, 3], [4, 1]
    # entry 0: text rows (5 x 2), entry 1: image rows (5 x 3)
    layout = [(0, 5, 2, 0), (1, 5, 3, 10)]
    flat = torch.arange(25, dtype=torch.float32)
    t, v = M.split_packed_states(flat, layout, t_rows, v_rows, 0)
    assert [tuple(x.shape) for x in t] == [(2, 2), (3, 2)] and [tuple(x.shape) for x in v] == [(4, 3), (1, 3)]
    assert float(t[1][0, 0]) == 4 and float(v[1][0, 0]) == 22
    assert v[0].data_ptr() == flat.data_ptr() + 4 * 10
    # first / mean: one [B, width] view per entry
    first = M.split_packed_states(flat[:10], [(0, 2, 2, 0), (1, 2, 3, 4)], t_rows, v_rows, 1)
    assert tuple(first[0].shape) == (2, 2) and tuple(first[1].shape) == (2, 3) and float(first[1][1, 0]) == 7


def test_constructor_validates_state_selection():
    from oracle import vilbert_ref as R
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(R.tiny_config().to_dict())
    with pytest.raises(ValueError, match="state_rows"):
        vb.VILBertForVLTasks(cfg, state_rows="max")
    with pytest.raises(ValueError, match="state_entries"):
        vb.VILBertForVLTasks(cfg, state_entries=[])
    m = vb.VILBertForVLTasks(cfg, state_entries=[0, 31], state_rows="mean")
    assert m._opts["state_entries"] == 1 | 1 << 31 and m._opts["state_rows"] == 2
    d = vb.VILBertForVLTasks(cfg)
    assert d._opts["state_entries"] is None and d._opts["state_rows"] == 0


def test_no_engine_errors():
    from oracle import vilbert_ref as R
    import vilbert_b200 as vb
    cfg = vb.BertConfig.from_dict(R.tiny_config().to_dict())
    m = vb.VILBertForVLTasks(cfg)
    for call in (m.state_selection, lambda: m.state_layout(1, 4, 4), lambda: m.state_layout_packed([3], [4])):
        with pytest.raises(L.VilbertB200Error, match="cuda"):
            call()
    with pytest.raises(L.VilbertB200Error, match="cuda"):
        m.forward_packed(torch.zeros(3, dtype=torch.long), torch.zeros(4, 256), torch.zeros(4, 5), None, None, [3], [4],
                         output_layer_states=True)
