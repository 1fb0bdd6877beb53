"""CPU-side checks of packed caption-image retrieval: padding strip, row packing and offsets, the pair layout, and the C ABI surface
(vb200_encode_text_packed / vb200_encode_image_packed / vb200_forward_cached_packed and vb200_packed_pairs).  The engine calls
themselves are covered on the GPU by tests/test_gpu_retrieval_packed.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import parallel as P
from vilbert_b200.model import packed_offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("vb200_encode_text_packed", "vb200_encode_image_packed", "vb200_forward_cached_packed")


def test_strip_padding_prefix_masks():
    m = torch.tensor([[1, 1, 1, 0, 0], [1, 0, 0, 0, 0], [1, 1, 1, 1, 1]])
    assert P.strip_padding(m) == [3, 1, 5]
    assert P.strip_padding(m.to(torch.uint8)) == [3, 1, 5]


@pytest.mark.parametrize("row", [[1, 0, 1, 0], [0, 1, 1, 0], [0, 0, 0, 0], [1, 2, 0, 0]])
def test_strip_padding_rejects_non_prefix(row):
    m = torch.tensor([[1, 1, 0, 0], row])
    with pytest.raises(ValueError, match="image_mask row 1 is not a prefix of ones"):
        P.strip_padding(m, "image_mask")


def test_pack_rows_and_offsets():
    x = torch.arange(3 * 4 * 2).reshape(3, 4, 2)
    lens = [2, 4, 1]
    got = P.pack_rows(x, lens)
    want = torch.cat([x[0, :2], x[1, :4], x[2, :1]])
    assert torch.equal(got, want)
    assert P.pack_rows(torch.arange(12).reshape(3, 4), lens).tolist() == [0, 1, 4, 5, 6, 7, 8]
    # caption states carry one task-token row per caption, image states none
    assert packed_offsets(lens, 1) == [0, 3, 8, 10]
    assert packed_offsets(lens) == [0, 2, 6, 7]
    offs = packed_offsets(lens)
    for i, k in enumerate(lens):
        assert torch.equal(got[offs[i]:offs[i + 1]], x[i, :k])


def test_retrieval_pairs_layout():
    ci, ii, total = P.retrieval_pairs(3, 5, 4)
    assert total == 15 and ci.dtype == torch.int32 and ii.dtype == torch.int32
    assert ci.numel() == 16 and ci.device.type == "cpu"
    assert ci[:15].tolist() == [c for c in range(3) for _ in range(5)]
    assert ii[:15].tolist() == [i for _ in range(3) for i in range(5)]
    assert (ci[15].item(), ii[15].item()) == (0, 0)          # padding repeats pair 0
    ci, ii, total = P.retrieval_pairs(2, 4, 8)
    assert total == 8 and ci.numel() == 8


def test_packed_retrieval_symbols_in_header_and_exports():
    hdr = open(os.path.join(ROOT, "include", "vilbert_b200.h")).read()
    declared = set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    for name in NEW_SYMBOLS:
        assert name in declared and name in L.EXPORTS, name
    assert "vb200_packed_pairs;" in hdr
    assert re.search(r"#define VB200_ABI_VERSION 2\b", hdr)


def test_packed_pairs_layout_matches_header(tmp_path):
    """ctypes PackedPairs against the C compiler's view of vb200_packed_pairs (size and every field offset, LP64)."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in L.PackedPairs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vilbert_b200.h"\nint main(void) {\n'
                   '    printf("%zu", sizeof(vb200_packed_pairs));\n'
                   + "".join(f'    printf(" %zu", offsetof(vb200_packed_pairs, {f}));\n' for f in fields)
                   + '    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[0] == C.sizeof(L.PackedPairs) == 96
    assert got[1:] == [getattr(L.PackedPairs, f).offset for f in fields]


def test_forward_cached_packed_rejects_dense_states():
    model = vb.VILBertForVLTasks(vb.BertConfig())
    dense_text, dense_image = dict(kind="text", n=1, Tin=5), dict(kind="image", n=1, V=3)
    with pytest.raises(ValueError, match="encode_text_packed and encode_image_packed"):
        model.forward_cached_packed(dense_text, torch.zeros(1), dense_image, torch.zeros(1))


def test_engine_entry_points_reject_null_handle():
    lib = L.load()
    pairs = L.PackedPairs()
    assert lib.vb200_forward_cached_packed(None, C.byref(pairs), None, L.OUT_VIL_LOGIT, 0, None) == -1
    assert lib.vb200_encode_text_packed(None, 1, 0, None, None, None, None, None, None, None) == -1
    assert lib.vb200_encode_image_packed(None, 1, 0, None, None, None, None, None, None) == -1
