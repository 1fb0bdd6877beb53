"""Answer ablation without a GPU: the C structs against the header, the Python variant order, default ranges and the split of a batch
at the engine's variant cap, and argument errors raised before any engine is needed."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vilbert_b200.h")


def test_header_declares_and_library_exports_ablation():
    hdr = open(HEADER).read()
    assert "vb200_answer_ablation" in set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    assert "vb200_answer_ablation" in L.EXPORTS and hasattr(L.load(), "vb200_answer_ablation")
    assert re.search(r"#define VB200_ABLATION_MAX_VARIANTS (\d+)", hdr).group(1) == str(L.ABLATION_MAX_VARIANTS)


def test_ablation_structs_match_the_c_layout(tmp_path):
    """sizeof / offsetof of vb200_ablation_msg and vb200_ablation_score as a C compiler lays them out from the header, against ctypes."""
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(vb200_ablation_msg), offsetof(vb200_ablation_msg, answer),'
                   ' offsetof(vb200_ablation_msg, token_begin), offsetof(vb200_ablation_msg, token_end),'
                   ' offsetof(vb200_ablation_msg, box_begin), offsetof(vb200_ablation_msg, box_end));\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(vb200_ablation_score), offsetof(vb200_ablation_score, answer),'
                   ' offsetof(vb200_ablation_score, prob), offsetof(vb200_ablation_score, top1), offsetof(vb200_ablation_score, top1_prob));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    msg = [int(x) for x in lines[0].split()]
    score = [int(x) for x in lines[1].split()]
    m, s = L.AblationMsg, L.AblationScore
    assert msg == [C.sizeof(m), m.answer.offset, m.token_begin.offset, m.token_end.offset, m.box_begin.offset, m.box_end.offset]
    assert score == [C.sizeof(s), s.answer.offset, s.prob.offset, s.top1.offset, s.top1_prob.offset]
    assert C.sizeof(s) == 16          # model.answer_ablation reads the scores as an int32 [n, 4] tensor


def test_default_ranges_keep_cls_and_sep_and_drop_every_box():
    assert M.ablation_ranges([37, 3, 2, 1], [100, 2, 1, 36]) == [(1, 36, 0, 100), (1, 2, 0, 2), (1, 1, 0, 0), (1, 1, 0, 36)]


def test_ranges_for_every_sample_or_per_sample():
    assert M.ablation_ranges([10, 12], [5, 6], tokens=(2, 4)) == [(2, 4, 0, 5), (2, 4, 0, 6)]
    assert M.ablation_ranges([10, 12], [5, 6], tokens=[(0, 10), None], boxes_range=[None, (3, 3)]) == [(0, 10, 0, 5), (1, 11, 3, 3)]
    assert M.ablation_ranges([10], [1], boxes_range=(0, 0)) == [(1, 9, 0, 0)]


@pytest.mark.parametrize("kw, match", [
    (dict(tokens=(3, 2)), "token range"),
    (dict(tokens=(0, 11)), "token range"),
    (dict(boxes_range=(-1, 2)), "box range"),
    (dict(boxes_range=(0, 6)), "box range"),
    (dict(tokens=[(0, 1)]), "one per sample"),
])
def test_bad_ranges_are_rejected(kw, match):
    with pytest.raises(ValueError, match=match):
        M.ablation_ranges([10, 10], [5, 5], **kw)


def test_box_ablation_needs_two_boxes():
    with pytest.raises(ValueError, match="needs >= 2"):
        M.ablation_ranges([5], [1], boxes_range=(0, 1))


def test_variant_order_is_base_tokens_boxes_per_sample():
    call = [(0, (1, 3, 0, 2)), (1, (0, 0, 1, 2))]
    assert M.ablation_variants(call) == [(0, "base", None), (0, "token", 1), (0, "token", 2), (0, "box", 0), (0, "box", 1),
                                         (1, "base", None), (1, "box", 1)]


def test_a_batch_within_the_cap_is_one_call():
    ranges = M.ablation_ranges([37] * 7, [100] * 7)            # 7 x 136 = 952 variants
    calls = M.ablation_calls(ranges)
    assert len(calls) == 1 and [i for i, _ in calls[0]] == list(range(7))
    assert len(M.ablation_variants(calls[0])) == 952


def test_batches_split_at_sample_boundaries():
    ranges = M.ablation_ranges([37] * 8, [100] * 8)            # 8 x 136 = 1088 > 1024
    calls = M.ablation_calls(ranges)
    assert [[i for i, _ in c] for c in calls] == [list(range(7)), [7]]
    assert all(len(M.ablation_variants(c)) <= L.ABLATION_MAX_VARIANTS for c in calls)
    assert [r for c in calls for _, r in c] == ranges


def test_a_sample_above_the_cap_is_split_into_pieces():
    ranges = [(1, 9, 0, 10), (0, 2, 0, 0)]                      # 19 and 3 variants
    calls = M.ablation_calls(ranges, cap=8)
    assert calls == [[(0, (1, 8, 0, 0))], [(0, (8, 9, 0, 6))], [(0, (0, 0, 6, 10)), (1, (0, 2, 0, 0))]]
    units = [(i, k, u) for c in calls for i, k, u in M.ablation_variants(c) if k != "base"]
    assert units == [(0, "token", p) for p in range(1, 9)] + [(0, "box", j) for j in range(10)] + [(1, "token", 0), (1, "token", 1)]
    assert all(len(M.ablation_variants(c)) <= 8 for c in calls)


def _model():
    cfg = vb.BertConfig(hidden_size=128, num_attention_heads=2, intermediate_size=256, v_hidden_size=256, v_num_attention_heads=2,
                        v_intermediate_size=256, bi_hidden_size=256, bi_num_attention_heads=2, bi_intermediate_size=256, vocab_size=512,
                        v_feature_size=64, v_target_size=32, max_position_embeddings=64, task_specific_tokens=True)
    return vb.VILBertForVLTasks(cfg, num_labels=40)


def _args(nt=(6, 4), nb=(3, 2)):
    return (None, None, None, None, None, None, list(nt), list(nb))


@pytest.mark.parametrize("kw, match", [
    (dict(family="nlvr2"), "not one of"),
    (dict(family=L.DECODE_GROUNDING), "not one of"),
    (dict(family=L.DECODE_RETRIEVAL), "not one of"),
    (dict(answer=[1]), "2 samples"),
    (dict(answer=-2), ">= 0"),
    (dict(tokens=(0, 7)), "token range"),
])
def test_argument_errors_without_an_engine(kw, match):
    with pytest.raises(ValueError, match=match):
        _model().answer_ablation(*_args(), **kw)


def test_lengths_must_match():
    with pytest.raises(ValueError, match="same, positive length"):
        _model().answer_ablation(*_args(nt=(6,), nb=(3, 2)))


def test_valid_arguments_need_an_engine():
    with pytest.raises(vb.VilbertB200Error, match="cuda"):
        _model().answer_ablation(*_args(), family="snli_ve", answer=[None, 2])


def test_null_handle_is_invalid():
    assert L.load().vb200_answer_ablation(None, None, None, L.DECODE_VQA, 103, None, None, 0, None) == -1
