"""Host side of BertForMultiModalPreTraining (vb200_create_pretraining) and of the pre-training objectives
(vb200_pretraining_objectives): struct layouts, the no-engine errors, the checkpoint audit before any device is touched (from Python
and from plain C), the oracle's losses against a direct torch formulation, and score="alignment" retrieval routing for a pre-training
model under a gloo world of 2.  The engine calls themselves are covered on the GPU by tests/test_gpu_pretraining_model.py."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import parallel as P
from vilbert_b200 import synthetic as S
from vilbert_b200.model import packed_offsets
import support

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TARGET_FIELDS = ["token_labels", "image_targets", "pair_labels"]
LOSS_FIELDS = ["token_loss", "region_loss", "pair_loss", "reduced"]


def _cfg(**kw):
    d = dict(hidden_size=128, num_attention_heads=2, intermediate_size=256, v_hidden_size=256, v_num_attention_heads=2,
             v_intermediate_size=256, bi_hidden_size=256, bi_num_attention_heads=2, bi_intermediate_size=256, vocab_size=2048,
             v_feature_size=64, v_target_size=32, max_position_embeddings=64, task_specific_tokens=False)
    d.update(kw)
    return vb.BertConfig(**d)


# ------------------------------------------------------------------ C ABI
def test_ctypes_structs_match_header_layout():
    assert [f for f, _ in L.PretrainTargets._fields_] == TARGET_FIELDS
    assert [f for f, _ in L.PretrainLosses._fields_] == LOSS_FIELDS
    assert C.sizeof(L.PretrainTargets) == 24 and C.sizeof(L.PretrainLosses) == 32


def test_struct_layout_from_the_c_compiler(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vilbert_b200.h"', "int main(void) {",
             'printf("%zu %zu\\n", sizeof(vb200_pretrain_targets), sizeof(vb200_pretrain_losses));']
    for s, fields in (("vb200_pretrain_targets", TARGET_FIELDS), ("vb200_pretrain_losses", LOSS_FIELDS)):
        lines += [f'printf("%zu\\n", offsetof({s}, {f}));' for f in fields]
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    want = [C.sizeof(L.PretrainTargets), C.sizeof(L.PretrainLosses)] + [getattr(L.PretrainTargets, f).offset for f in TARGET_FIELDS] + \
        [getattr(L.PretrainLosses, f).offset for f in LOSS_FIELDS]
    assert [int(x) for x in got] == want


def test_null_handle_rejected():
    assert L.load().vb200_pretraining_objectives(None, None, None, None, None) == -1


# ------------------------------------------------------------------ no engine
def _no_library(monkeypatch):
    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(L, "load", no_library)


@pytest.mark.parametrize("cls", ["VILBertForVLTasks", "BertForMultiModalPreTraining"])
def test_objectives_need_an_engine(monkeypatch, cls):
    model = getattr(vb, cls)(_cfg())
    _no_library(monkeypatch)
    taps = {"sequence_output_t": torch.zeros(3, 128)}
    with pytest.raises(L.VilbertB200Error, match=r"call model\.cuda\(i\) first"):
        model.pretraining_objectives(taps, text_rows=[0], token_labels=[1])


def test_pretraining_model_needs_an_engine(monkeypatch):
    model = vb.BertForMultiModalPreTraining(_cfg())
    _no_library(monkeypatch)
    b = S.synthetic_masked_batch(2, 10, 5, seed=1, vocab_size=2048, v_feature_size=64, v_target_size=32)
    keys = ("input_ids", "image_feat", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")
    for labels in ({}, {k: b[k] for k in ("masked_lm_labels", "image_label", "image_target", "next_sentence_label")}):
        with pytest.raises(L.VilbertB200Error, match=r"call model\.cuda\(i\) first"):
            model(*[b[k] for k in keys], **labels)
    with pytest.raises(L.VilbertB200Error, match=r"call model\.cuda\(i\) first"):
        model.pretraining_heads(taps={}, pair_rows=[0])
    with pytest.raises(ValueError, match="together"):
        model(*[b[k] for k in keys], masked_lm_labels=b["masked_lm_labels"])
    with pytest.raises(L.VilbertB200Error, match="train"):
        model.train()


# ------------------------------------------------------------------ the audit, before any device is touched
def _create(cfg, sd, strict=True, num_labels=0, fn="vb200_create_pretraining"):
    lib = L.load()
    m = vb.BertForMultiModalPreTraining(cfg, state_dict=sd, strict=strict)
    names = [k.encode() for k in m._sd]
    arr = (L.Tensor * len(m._sd))()
    for i, (k, v) in enumerate(m._sd.items()):
        arr[i].name, arr[i].dtype, arr[i].ndim = names[i], 0, v.dim()
        arr[i].shape[0], arr[i].shape[1] = v.shape[0], (v.shape[1] if v.dim() == 2 else 0)
        arr[i].data = v.data_ptr()
    o = L.Options()
    o.num_labels = num_labels
    o.strict = 1 if strict else -1
    h = C.c_void_p()
    rc = getattr(lib, fn)(m._config_json(), len(m._sd), arr, C.byref(o), C.byref(h))
    msg = lib.vb200_last_error(None).decode()
    if rc == 0:
        lib.vb200_destroy(h)
    return rc, msg


needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device failure path")


@needs_no_gpu
def test_good_pretraining_checkpoint_passes_the_audit():
    cfg = _cfg()
    rc, msg = _create(cfg, S.synthetic_pretraining_state_dict(cfg, seed=1))
    assert rc == -5 and "no CPU fallback" in msg, msg          # audit passed, then VB200_ERR_NO_DEVICE
    with pytest.raises(vb.VilbertB200Error):
        vb.BertForMultiModalPreTraining.from_pretrained(S.synthetic_pretraining_state_dict(cfg, seed=1), config=cfg).cuda(0)


@pytest.mark.parametrize("key", ["cls.predictions.bias", "cls.imagePredictions.decoder.weight", "cls.bi_seq_relationship.bias",
                                 "cls.predictions.transform.LayerNorm.weight"])
def test_audit_missing_cls_key(key):
    cfg = _cfg()
    sd = S.synthetic_pretraining_state_dict(cfg, seed=1)
    del sd[key]
    rc, msg = _create(cfg, sd)
    assert rc == -3 and f'missing key "{key}"' in msg, msg


def test_audit_task_head_keys_are_extra_keys():
    cfg = _cfg()
    sd = S.synthetic_pretraining_state_dict(cfg, seed=1)
    full = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    sd.update({k: v for k, v in full.items() if k.startswith("vil_logit.")})
    rc, msg = _create(cfg, sd)
    assert rc == -3 and "unexpected" in msg and "vil_logit.weight" in msg, msg
    rc, msg = _create(cfg, sd, strict=False)
    assert rc != -3, msg
    # the multi-task constructor still asks for the task heads, with the same message as before
    rc, msg = _create(cfg, S.synthetic_pretraining_state_dict(cfg, seed=1), fn="vb200_create")
    assert rc == -3 and msg == 'checkpoint is missing key "vil_prediction.logit_fc.3.weight"', msg


def test_audit_legacy_names_and_prefix():
    cfg = _cfg()
    sd = {("module." + k).replace("LayerNorm.weight", "LayerNorm.gamma").replace("LayerNorm.bias", "LayerNorm.beta"): v
          for k, v in S.synthetic_pretraining_state_dict(cfg, seed=1).items()}
    rc, msg = _create(cfg, sd)
    assert rc not in (-2, -3), msg


@pytest.mark.parametrize("kw, rc_want, needle", [
    (dict(visual_target=1), -2, "visual_target=1 is not supported"),
    (dict(visual_target=2), -2, "visual_target=2 is not supported"),
    (dict(predict_feature=True), -2, "predict_feature=true is not supported"),
])
def test_config_rejections(kw, rc_want, needle):
    cfg = _cfg(**kw)
    rc, msg = _create(cfg, S.synthetic_pretraining_state_dict(_cfg(), seed=1))
    assert rc == rc_want and needle in msg, msg


def test_num_labels_rejected():
    cfg = _cfg()
    rc, msg = _create(cfg, S.synthetic_pretraining_state_dict(cfg, seed=1), num_labels=3129)
    assert rc == -1 and "num_labels must be 0" in msg, msg


def test_c_host_audit(tmp_path):
    """A plain C host reaches vb200_create_pretraining through the header alone and gets the audit's status and message."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "pt.c"
    src.write_text(r'''
#include <dlfcn.h>
#include <stdio.h>
#include "vilbert_b200.h"
typedef int (*create_fn)(const char*, int64_t, const vb200_tensor*, const vb200_options*, vb200_handle*);
typedef const char* (*err_fn)(vb200_handle);
int main(int argc, char** argv) {
    void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
    if (!lib) return 2;
    create_fn create = (create_fn)dlsym(lib, "vb200_create_pretraining");
    err_fn last_error = (err_fn)dlsym(lib, "vb200_last_error");
    if (!create || !last_error) return 2;
    float w[4] = {0};
    vb200_tensor t = {"cls.predictions.bias", VB200_F32, 1, {4, 0}, w};
    vb200_handle h = NULL;
    int rc = create("{\"visual_target\": 1}", 1, &t, NULL, &h);
    printf("%d|%s\n", rc, last_error(NULL));
    rc = create("{\"task_specific_tokens\": false}", 1, &t, NULL, &h);
    printf("%d|%s\n", rc, last_error(NULL));
    return h == NULL ? 0 : 1;
}
''')
    exe = tmp_path / "pt"
    subprocess.run([cc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-ldl"], check=True)
    out = subprocess.run([str(exe), L.LIB_PATH], check=True, capture_output=True, text=True).stdout.splitlines()
    assert out[0].startswith("-2|visual_target=1 is not supported"), out
    assert out[1].startswith("-3|checkpoint is missing key"), out


# ------------------------------------------------------------------ the oracle's losses
def test_oracle_losses_against_direct_torch():
    from oracle import pretraining_ref as PR
    g = torch.Generator().manual_seed(3)
    B, T, V, vocab, vt = 3, 9, 6, 50, 12
    st, sv, sr = torch.randn(B, T, vocab, generator=g), torch.randn(B, V, vt, generator=g), torch.randn(B, 2, generator=g)
    lm = torch.full((B, T), -1)
    lm[0, 2], lm[1, 5], lm[2, 0], lm[2, 8] = 7, 0, vocab - 1, 3
    il = torch.full((B, V - 1), -1)
    il[0, 0], il[1, 3], il[2, 4] = 1, 1, 1
    tgt = torch.softmax(torch.randn(B, V - 1, vt, generator=g), -1)
    tgt[0, 0] = 0.0
    tgt[0, 0, 3] = 1.0                                                    # one-hot: exact zeros elsewhere
    nsp = torch.tensor([1, -1, 0])
    got = PR.pretraining_losses(st, sv, sr, lm, il, tgt, nsp)
    m = lm != -1
    want_lm = torch.stack([torch.logsumexp(st[m][i], 0) - st[m][i][lm[m][i]] for i in range(int(m.sum()))]).mean()
    rows = [(b, j) for b in range(B) for j in range(V - 1) if il[b, j] == 1]
    kl = []
    for b, j in rows:
        t, ls = tgt[b, j], torch.log_softmax(sv[b, j + 1], 0)
        kl.append(sum(float(t[c]) * (float(torch.log(t[c])) - float(ls[c])) for c in range(vt) if t[c] > 0))
    want_img = sum(kl) / len(rows)
    want_nsp = torch.stack([torch.logsumexp(sr[b], 0) - sr[b, nsp[b]] for b in (0, 2)]).mean()
    assert all(x.shape == (1,) for x in got)
    assert torch.allclose(got[0], want_lm.reshape(1), rtol=1e-5)
    assert abs(float(got[1]) - want_img) < 1e-5 * abs(want_img)
    assert torch.allclose(got[2], want_nsp.reshape(1), rtol=1e-5)
    # nothing to score: 0 / 0
    empty = PR.pretraining_losses(st, sv, sr, torch.full((B, T), -1), torch.full((B, V - 1), -1), tgt, torch.full((B,), -1))
    assert all(torch.isnan(x).all() for x in empty)
    assert PR.PRETRAINING_ASSUMPTIONS["ignore_index"] == -1 and PR.PRETRAINING_ASSUMPTIONS["matched_alignment_column"] is None
    assert F.kl_div(torch.zeros(1), torch.zeros(1), reduction="sum") == 0


def test_synthetic_masked_batch():
    b = S.synthetic_masked_batch(8, 36, 37, seed=4, vocab_size=30522, v_feature_size=64, v_target_size=1601)
    lm, il, t = b["masked_lm_labels"], b["image_label"], b["image_target"]
    masked = lm != -1
    assert bool((b["input_ids"][masked] == 103).all()) and 0.05 < float(masked.float().mean()) < 0.25
    assert il.shape == (8, 36) and t.shape == (8, 36, 1601) and bool((b["image_feat"][:, 1:][il == 1] == 0).all())
    assert torch.allclose(t.sum(-1), torch.ones(8, 36)) and bool((t == 0).any())
    assert set(b["next_sentence_label"].tolist()) <= {-1, 0, 1}
    sd = S.synthetic_pretraining_state_dict(_cfg(), seed=1)
    assert all(k.startswith(("bert.", "cls.")) for k in sd) and "bert.embeddings.task_embeddings.weight" not in sd
    with pytest.raises(ValueError, match="task_specific_tokens"):
        S.synthetic_pretraining_state_dict(_cfg(task_specific_tokens=True))


# ------------------------------------------------------------------ score="alignment" on a pre-training model, gloo world of 2
class StubPretraining(vb.BertForMultiModalPreTraining):
    """A pre-training model whose engine calls are recorded; a pair's pooled tap row is (caption, image) and its alignment is
    align[caption, image].  Captions carry no task-token row (task_specific_tokens off)."""

    def __init__(self, align):
        super().__init__(_cfg())
        self.align, self.calls = align, []

    def encode_text_packed(self, question, segment_ids, task_tokens, n_tokens, max_tokens=0):
        offs = packed_offsets(n_tokens)
        self.calls.append(("encode_text_packed", list(n_tokens)))
        return dict(kind="text", ids=question[offs[:-1]])

    def encode_image_packed(self, features, spatials, n_regions, max_regions=0):
        offs = packed_offsets(n_regions)
        self.calls.append(("encode_image_packed", list(n_regions)))
        return dict(kind="image", ids=features[offs[:-1], 0].long())

    def forward_cached_packed(self, ts, text_index, vs, image_index, select=0, debug_taps=False):
        self.calls.append(("forward_cached_packed", select, debug_taps))
        c, i = ts["ids"][text_index.long()], vs["ids"][image_index.long()]
        return (None,) * 10, {"pooled_output": torch.stack([c, i], 1).float()}

    def pretraining_heads(self, taps, text_rows=None, image_rows=None, pair_rows=None, top_k=0):
        rows = list(pair_rows)
        self.calls.append(("pretraining_heads", len(rows)))
        p = taps["pooled_output"][rows].long()
        return {"alignment": self.align[p[:, 0], p[:, 1]]}


def _check(rank, world, n_cap, n_img, pair_batch):
    g = torch.Generator().manual_seed(5)
    align = torch.randn(n_cap, n_img, 2, generator=g)
    lens = [1 + (3 * c) % 6 for c in range(n_cap)]
    q, seg, im = (torch.zeros(n_cap, 6, dtype=torch.long) for _ in range(3))
    for c, k in enumerate(lens):
        q[c, :k], im[c, :k] = torch.arange(c, c + k), 1
    v_lens = [1 + (7 * i) % 5 for i in range(n_img)]
    f, s, vm = torch.zeros(n_img, 5, 8), torch.rand(n_img, 5, 5), torch.zeros(n_img, 5, dtype=torch.uint8)
    for i, k in enumerate(v_lens):
        f[i, :k], vm[i, :k] = float(i), 1
    m = StubPretraining(align)
    full = P.retrieval_scores_packed(m, (q, seg, im), (f, s, vm), pair_batch=pair_batch, score="alignment")
    assert torch.equal(full, align)
    assert all(c[0] != "forward_cached_packed" or c[1:] == (0, True) for c in m.calls)     # no task head is asked for
    assert any(c[0] == "pretraining_heads" for c in m.calls)
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


def test_alignment_routing_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = support.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, 5, 6, 4, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]
