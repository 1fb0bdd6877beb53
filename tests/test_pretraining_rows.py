"""Host side of the pre-training heads at chosen rows (vb200_pretraining_heads, VILBertForVLTasks.pretraining_heads) and of the
score="alignment" routing of parallel.retrieval_scores_packed / retrieval_scores_regions, on a stub model under a gloo world of 2.
The engine call itself is covered on the GPU by tests/test_gpu_pretraining_rows.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vilbert_b200 import _lib as L
from vilbert_b200 import parallel as P
from vilbert_b200.model import packed_offsets
import support

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 8

ROWS_FIELDS = ["text_state", "image_state", "pooled_state", "t_rows", "v_rows", "p_rows", "n_t", "n_v", "n_p", "text_rows",
               "image_rows", "pair_rows", "top_k"]
OUT_FIELDS = ["token_logits", "region_logits", "alignment", "token_top", "region_top"]


# ------------------------------------------------------------------ C ABI
def test_ctypes_structs_match_header_layout():
    assert [f for f, _ in L.PretrainRows._fields_] == ROWS_FIELDS
    assert [f for f, _ in L.PretrainOut._fields_] == OUT_FIELDS
    assert C.sizeof(L.PretrainRows) == 80 and C.sizeof(L.PretrainOut) == 40
    assert [getattr(L.PretrainRows, f).offset for f in ROWS_FIELDS] == [0, 8, 16, 24, 28, 32, 36, 40, 44, 48, 56, 64, 72]


def test_struct_layout_from_the_c_compiler(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vilbert_b200.h"', "int main(void) {"]
    lines.append('printf("%zu %zu\\n", sizeof(vb200_pretrain_rows), sizeof(vb200_pretrain_out));')
    for s, fields in (("vb200_pretrain_rows", ROWS_FIELDS), ("vb200_pretrain_out", OUT_FIELDS)):
        lines += [f'printf("%zu\\n", offsetof({s}, {f}));' for f in fields]
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    want = [C.sizeof(L.PretrainRows), C.sizeof(L.PretrainOut)] + [getattr(L.PretrainRows, f).offset for f in ROWS_FIELDS] + \
        [getattr(L.PretrainOut, f).offset for f in OUT_FIELDS]
    assert [int(x) for x in got] == want


def test_symbol_in_header_and_exports():
    hdr = open(os.path.join(ROOT, "include", "vilbert_b200.h")).read()
    m = re.search(r"int vb200_pretraining_heads\(([^;]*)\);", hdr)
    assert m and "vb200_pretraining_heads" in L.EXPORTS
    params = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")
    assert len(params) == len(L.load().vb200_pretraining_heads.argtypes) == 4


def test_null_handle_rejected():
    assert L.load().vb200_pretraining_heads(None, None, None, None) == -1


def test_pretraining_heads_needs_an_engine(monkeypatch):
    import vilbert_b200 as vb
    model = vb.VILBertForVLTasks(vb.BertConfig())

    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(L, "load", no_library)
    monkeypatch.setattr(torch, "empty", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a tensor was created")))
    taps = {"sequence_output_t": torch.zeros(3, 768)}
    with pytest.raises(L.VilbertB200Error, match=r"call model\.cuda\(i\) first"):
        model.pretraining_heads(taps, text_rows=[0, 2], top_k=5)


# ------------------------------------------------------------------ score= routing of the packed retrieval calls
class StubModel:
    """Records every engine call.  A caption's first token is its index and every feature row of image i holds i; a pair's vil_logit is
    table[caption, image] and its pooled tap row is (caption, image), from which the stub's alignment head reads align[caption, image]."""

    def __init__(self, table, align):
        self.table, self.align, self.calls = table, align, []

    def encode_text_packed(self, question, segment_ids, task_tokens, n_tokens, max_tokens=0):
        offs = packed_offsets(n_tokens)
        self.calls.append(("encode_text_packed", list(n_tokens), question[offs[:-1]].tolist(), task_tokens.tolist()))
        return dict(kind="text", ids=question[offs[:-1]])

    def encode_image_packed(self, features, spatials, n_regions, max_regions=0):
        offs = packed_offsets(n_regions)
        self.calls.append(("encode_image_packed", list(n_regions)))
        return dict(kind="image", ids=features[offs[:-1], 0].long())

    def encode_regions_packed(self, box_features, boxes, image_wh, n_boxes, max_boxes=0):
        offs = packed_offsets(n_boxes)
        self.calls.append(("encode_regions_packed", list(n_boxes), max_boxes))
        return dict(kind="image", ids=box_features[offs[:-1], 0].long())

    def forward_cached_packed(self, ts, text_index, vs, image_index, select=0, debug_taps=False):
        self.calls.append(("forward_cached_packed", text_index.tolist(), image_index.tolist(), select) + ((True,) if debug_taps else ()))
        c, i = ts["ids"][text_index.long()], vs["ids"][image_index.long()]
        out = (None, None, self.table[c, i].unsqueeze(1)) + (None,) * 7
        if not debug_taps:
            return out
        return out, {"pooled_output": torch.stack([c, i], 1).float()}

    def pretraining_heads(self, taps, text_rows=None, image_rows=None, pair_rows=None, top_k=0):
        rows = list(pair_rows)
        self.calls.append(("pretraining_heads", rows, text_rows, image_rows, top_k))
        p = taps["pooled_output"][rows].long()
        return {"alignment": self.align[p[:, 0], p[:, 1]]}


def _captions(n_cap, t_pad=6):
    lens = [1 + (3 * c) % t_pad for c in range(n_cap)]
    q, seg, im = (torch.zeros(n_cap, t_pad, dtype=torch.long) for _ in range(3))
    for c, k in enumerate(lens):
        q[c, :k], im[c, :k] = torch.arange(c, c + k), 1
    return (q, seg, im), lens


def _gallery(n_img):
    n_boxes = [1 + (7 * i) % 5 for i in range(n_img)]
    bf = torch.cat([torch.full((k, F), float(i)) for i, k in enumerate(n_boxes)])
    return (bf, torch.rand(sum(n_boxes), 4), torch.full((n_img, 2), 100.0), n_boxes)


def _check(rank, world, n_cap, n_img, pair_batch):
    g = torch.Generator().manual_seed(5)
    table, align = torch.randn(n_cap, n_img, generator=g), torch.randn(n_cap, n_img, 2, generator=g)
    caps, t_lens = _captions(n_cap)
    lo, hi = P.shard_range(n_cap, rank, world)
    text_call = ("encode_text_packed", t_lens[lo:hi], list(range(lo, hi)), [[7]] * (hi - lo))
    ci, ii, _ = P.retrieval_pairs(hi - lo, n_img, pair_batch)
    chunks = [(ci[s:s + pair_batch].tolist(), ii[s:s + pair_batch].tolist()) for s in range(0, ci.numel(), pair_batch)]
    default = [("forward_cached_packed", c, i, L.OUT_VIL_LOGIT) for c, i in chunks]
    aligned = []
    for c, i in chunks:
        aligned += [("forward_cached_packed", c, i, 0, True), ("pretraining_heads", list(range(pair_batch)), None, None, 0)]
    images, v_lens = support.padded_gallery(n_img, F)
    gallery = _gallery(n_img)
    for score, expect, calls in ((None, table, default), ("vil_logit", table, default), ("alignment", align, aligned)):
        kw = {} if score is None else {"score": score}
        m = StubModel(table, align)
        full = P.retrieval_scores_packed(m, caps, images, pair_batch=pair_batch, **kw)
        assert torch.equal(full, expect), score
        assert m.calls == [("encode_image_packed", v_lens), text_call] + calls, score
        m = StubModel(table, align)
        full = P.retrieval_scores_regions(m, caps, gallery, pair_batch=pair_batch, max_boxes=6, **kw)
        assert torch.equal(full, expect), score
        assert m.calls == [("encode_regions_packed", gallery[3], 6), text_call] + calls, score
    return True


def _worker(rank, world, port, n_cap, n_img, pair_batch, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        try:
            ok = _check(rank, world, n_cap, n_img, pair_batch)
        except AssertionError as e:
            ok = repr(e)
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_cap,n_img,pair_batch", [(5, 6, 4), (3, 7, 5)])
def test_score_routing_gloo_world2(n_cap, n_img, pair_batch):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = support.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n_cap, n_img, pair_batch, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]


def test_score_routing_single_process():
    assert _check(0, 1, 4, 5, 6)


def test_unknown_score_rejected():
    caps, _ = _captions(2)
    m = StubModel(torch.zeros(2, 2), torch.zeros(2, 2, 2))
    with pytest.raises(ValueError, match="score must be"):
        P.retrieval_scores_regions(m, caps, _gallery(2), score="probability")
    assert m.calls == []
