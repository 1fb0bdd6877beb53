"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the header declares,
audits configs / checkpoints before touching a device, and fails loudly (no CPU fallback) without a GPU."""
import ctypes as C
import os
import re

import pytest
import torch

import vilbert_b200 as vb
from vilbert_b200 import _lib as L
from vilbert_b200 import synthetic as S
import support

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_all_exported():
    hdr = open(os.path.join(ROOT, "include", "vilbert_b200.h")).read()
    declared = set(re.findall(r"\b(vb200_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(L.EXPORTS), declared ^ set(L.EXPORTS)
    lib = L.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.vb200_abi_version() == 2


def test_ctypes_structs_match_header_layout():
    # field order / sizes the header fixes (LP64)
    assert C.sizeof(L.Tensor) == 8 + 4 + 4 + 16 + 8
    assert C.sizeof(L.Inputs) == 16 + 8 * 8
    assert C.sizeof(L.Outputs) == 13 * 8
    assert C.sizeof(L.Options) == 40
    assert C.sizeof(L.RegionInputs) == 16 + 9 * 8


def _create(cfg, sd, ln_fold=0, fused_layernorm=0, split_fp32=0, **opt):
    m = vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=opt.pop("num_labels", 40), **opt)
    lib = L.load()
    names = [k.encode() for k in m._sd]
    arr = (L.Tensor * len(m._sd))()
    for i, (k, v) in enumerate(m._sd.items()):
        arr[i].name, arr[i].dtype, arr[i].ndim = names[i], 0, v.dim()
        arr[i].shape[0], arr[i].shape[1] = v.shape[0], (v.shape[1] if v.dim() == 2 else 0)
        arr[i].data = v.data_ptr()
    o = L.Options()
    o.num_labels = m.num_labels
    o.strict = 1 if m._opts["strict"] else -1
    o.ln_fold = ln_fold
    o.fused_layernorm = fused_layernorm
    o.split_fp32 = split_fp32
    h = C.c_void_p()
    rc = lib.vb200_create(m._config_json(), len(m._sd), arr, C.byref(o), C.byref(h))
    msg = lib.vb200_last_error(None).decode()
    if rc == 0:
        lib.vb200_destroy(h)
    return rc, msg


needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device failure path")


@needs_no_gpu
def test_good_checkpoint_fails_loudly_without_gpu():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    rc, msg = _create(cfg, sd)
    assert rc == -5 and "no CPU fallback" in msg          # audit passed, then VB200_ERR_NO_DEVICE
    with pytest.raises(vb.VilbertB200Error):
        vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=40).cuda(0)


def test_checkpoint_audit_missing_key():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    del sd["bert.encoder.c_layer.3.biattention.query2.weight"]
    rc, msg = _create(cfg, sd)
    assert rc == -3 and "c_layer.3.biattention.query2.weight" in msg


def test_checkpoint_audit_wrong_shape():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    sd["bert.encoder.v_layer.0.output.dense.weight"] = torch.zeros(256, 128)
    rc, msg = _create(cfg, sd)
    assert rc == -3 and "v_layer.0.output.dense.weight" in msg and "expected" in msg


def test_checkpoint_audit_unexpected_key_strict_and_lenient():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    sd["bert.encoder.layer.0.some_new_thing.weight"] = torch.zeros(4, 4)
    rc, msg = _create(cfg, sd)
    assert rc == -3 and "unexpected" in msg and "some_new_thing" in msg
    rc, msg = _create(cfg, sd, strict=False)
    assert rc != -3


def test_checkpoint_audit_num_labels_mismatch():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    rc, msg = _create(cfg, sd, num_labels=3129)
    assert rc == -3 and "num_labels" in msg


def test_reserved_ln_fold_option_rejected():
    """vb200_options::ln_fold is reserved since the LayerNorm fold was removed: a non-zero value is refused before the checkpoint
    audit, so with or without a device."""
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    rc, msg = _create(cfg, sd, ln_fold=1)
    assert rc == -1 and "LayerNorm fold was removed" in msg, (rc, msg)


@pytest.mark.parametrize("split_fp32", [0, 1])
def test_reserved_fused_layernorm_option_rejected(split_fp32):
    """vb200_options::fused_layernorm is reserved since the cluster-LayerNorm GEMM epilogue was removed: a positive value is
    refused before the checkpoint audit, so with or without a device, and in fp32-parity mode too."""
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    rc, msg = _create(cfg, sd, fused_layernorm=1, split_fp32=split_fp32)
    assert rc == -1 and "cluster-LayerNorm GEMM epilogue was removed" in msg, (rc, msg)


@pytest.mark.parametrize("value", [0, -1])
def test_fused_layernorm_off_values_accepted(value):
    """0 and negative fused_layernorm values ("off" in the tri-state convention) get past the option check: the checkpoint
    audit, which needs no device, then reports the missing key."""
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    del sd["bert.encoder.c_layer.3.biattention.query2.weight"]
    rc, msg = _create(cfg, sd, fused_layernorm=value)
    assert rc == -3 and "c_layer.3.biattention.query2.weight" in msg, (rc, msg)


@pytest.mark.parametrize("arg", ["residual", "gamma", "beta"])
def test_linear_rejects_layernorm_arguments(arg):
    """vb200_linear has no LayerNorm epilogue: a non-null residual, gamma or beta is an invalid argument, refused before any
    CUDA call (so also without a device)."""
    lib = L.load()
    buf = torch.zeros(64)
    p = C.c_void_p(buf.data_ptr())
    ptrs = {k: (p if k == arg else None) for k in ("residual", "gamma", "beta")}
    rc = lib.vb200_linear(p, 64, p, 64, None, ptrs["residual"], 64, ptrs["gamma"], ptrs["beta"], 1e-12, 0,
                          None, 0, p, 64, 1, 8, 64, 0, 0, 0, 0, None, None)
    assert rc == -1
    assert "residual, gamma and beta must be NULL" in lib.vb200_last_error(None).decode()


def test_model_rejects_fused_layernorm():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    with pytest.raises(ValueError, match="cluster-LayerNorm GEMM epilogue was removed"):
        vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=40, fused_layernorm=True)


@pytest.mark.parametrize("kw,want", [
    ({}, dict(use_cuda_graph=1, use_pdl=0, strict=1, act_fp16=1, split_fp32=0, max_plans=0)),
    (dict(use_cuda_graph=False, use_pdl=False, strict=False), dict(use_cuda_graph=-1, use_pdl=-1, strict=-1)),
    (dict(use_pdl=True, max_plans=3), dict(use_pdl=1, max_plans=3)),
    (dict(compute_dtype="bf16"), dict(act_fp16=-1, split_fp32=0)),
    (dict(compute_dtype="fp32x", use_cuda_graph=True), dict(use_cuda_graph=1, act_fp16=1, split_fp32=1)),
])
def test_model_options_reach_the_engine(kw, want):
    """The model's keywords become vb200_options in the tri-state convention (1 on, -1 off, 0 the engine default): use_pdl=None
    leaves the engine's default, False is -1 and not 0; the reserved fields stay 0."""
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    o = vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=40, **kw)._options(2)
    assert (o.device, o.num_labels, o.fused_layernorm, o.ln_fold) == (2, 40, 0, 0)
    for field, value in want.items():
        assert getattr(o, field) == value, (field, getattr(o, field), value)


def test_checkpoint_legacy_names_accepted():
    """`module.` prefixes (DataParallel) and gamma/beta LayerNorm names ([UPSTREAM] from_pretrained fix-ups)."""
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    legacy = {}
    for k, v in sd.items():
        if "LayerNorm.weight" in k:
            k = k.replace("LayerNorm.weight", "LayerNorm.gamma")
        elif "LayerNorm.bias" in k:
            k = k.replace("LayerNorm.bias", "LayerNorm.beta")
        legacy["module." + k] = v
    rc, msg = _create(cfg, legacy)
    assert rc != -3, msg


@pytest.mark.parametrize("kw,needle", [
    (dict(dynamic_attention=True), "dynamic_attention"),
    (dict(hidden_act="relu"), "gelu"),
    (dict(num_attention_heads=4), "head size"),
    (dict(hidden_size=100, num_attention_heads=1), "head size"),
    (dict(fusion_method="sum"), "fusion_method"),
    # connection-layer ids outside the layer counts, negative or decreasing
    (dict(num_hidden_layers=4), "t_biattention_id[0] = 6 is outside [0, num_hidden_layers = 4]"),
    (dict(v_num_hidden_layers=2), "v_biattention_id[3] = 3 is outside [0, v_num_hidden_layers = 2]"),
    (dict(t_biattention_id=[6, 7, 8, 9, 10, 13]), "t_biattention_id[5] = 13 is outside [0, num_hidden_layers = 12]"),
    (dict(v_biattention_id=[-1, 1, 2, 3, 4, 5]), "v_biattention_id[0] = -1 is outside"),
    (dict(t_biattention_id=[6, 7, 8, 10, 9, 11]), "t_biattention_id[4] = 9 is below t_biattention_id[3] = 10"),
    (dict(v_biattention_id=[0, 1, 2, 3, 5, 4]), "v_biattention_id[5] = 4 is below v_biattention_id[4] = 5"),
])
def test_config_rejections(kw, needle):
    cfg = support.tiny_cfg(**kw)
    sd = S.synthetic_state_dict(support.tiny_cfg(), num_labels=40, gqa_labels=24, seed=1)
    rc, msg = _create(cfg, sd)
    assert rc == -2 and needle in msg, (rc, msg)


def test_config_json_garbage():
    lib = L.load()
    h = C.c_void_p()
    t = (L.Tensor * 1)()
    x = torch.zeros(1)
    t[0].name, t[0].ndim, t[0].data = b"x", 1, x.data_ptr()
    t[0].shape[0] = 1
    assert lib.vb200_create(b"{ not json", 1, t, None, C.byref(h)) == -2
    assert lib.vb200_create(None, 1, t, None, C.byref(h)) == -2
    assert lib.vb200_create(b"{}", 0, None, None, C.byref(h)) == -3


def test_config_json_string_escapes():
    """The engine's JSON reader decodes escape sequences (RFC 8259 section 7): "g\\u0065lu" is "gelu"; a broken \\u escape and an
    escaped value that is NOT gelu are configuration errors, not silently accepted strings."""
    lib = L.load()
    h = C.c_void_p()
    t = (L.Tensor * 1)()
    x = torch.zeros(1)
    t[0].name, t[0].ndim, t[0].data = b"x", 1, x.data_ptr()
    t[0].shape[0] = 1
    ok = b'{"hidden_act": "g\\u0065lu", "v_hidden_act": "gel\\u0075", "note": "a \\"quoted\\" \\\\ path\\n"}'
    assert lib.vb200_create(ok, 1, t, None, C.byref(h)) == -3                     # config accepted; the 1-tensor checkpoint is what fails
    assert "x" in lib.vb200_last_error(None).decode() or "missing" in lib.vb200_last_error(None).decode()
    assert lib.vb200_create(b'{"hidden_act": "g\\u00zzlu"}', 1, t, None, C.byref(h)) == -2
    assert lib.vb200_create(b'{"hidden_act": "r\\u0065lu"}', 1, t, None, C.byref(h)) == -2
    assert "gelu" in lib.vb200_last_error(None).decode()


def test_bertconfig_protocol(tmp_path):
    """worker.py:495-522: from_json_file, attribute mutation, to_dict round trip."""
    p = tmp_path / "bert_base_6layer_6conect.json"
    p.write_text('{"hidden_size": 768, "v_biattention_id": [0, 1], "t_biattention_id": [10, 11], "bi_hidden_size": 1024}')
    c = vb.BertConfig.from_json_file(str(p))
    c.v_target_size = 1601
    c.predict_feature = False
    c.task_specific_tokens = True
    c.visualization = True
    assert c.v_biattention_id == [0, 1] and c.to_dict()["task_specific_tokens"] is True
    assert vb.BertConfig.from_dict(c.to_dict()).to_dict() == c.to_dict()


def test_model_protocol_without_engine():
    cfg = support.tiny_cfg()
    sd = S.synthetic_state_dict(cfg, num_labels=40, gqa_labels=24, seed=1)
    m = vb.VILBertForVLTasks.from_pretrained(sd, config=cfg, num_labels=40)
    assert m.eval() is m
    with pytest.raises(vb.VilbertB200Error):
        m.to("cpu")
    with pytest.raises(vb.VilbertB200Error):
        m(torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 3, 64), torch.zeros(1, 3, 5))   # no .cuda() -> no CPU path
    with pytest.raises(ValueError):
        vb.VILBertForVLTasks.from_pretrained(sd)


def test_product_path_never_imports_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may touch oracle/."""
    pkg = os.path.join(ROOT, "vilbert-multi-task_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith(".py"):
                src = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), fn


def test_c_host_example_builds_and_runs(tmp_path):
    """examples/host_min.c: a plain C program binds the library with nothing but include/vilbert_b200.h (dlopen), checks the ABI
    version and gets status + message for a bad config and an incomplete checkpoint -- all before any device is touched."""
    import shutil
    import subprocess
    from vilbert_b200 import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    exe = tmp_path / "host_min"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "host_min.c"), "-o", str(exe), "-ldl"], check=True)
    r = subprocess.run([str(exe), L.LIB_PATH], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "bad config       -> -2" in r.stdout and "empty checkpoint -> -3" in r.stdout and r.stdout.strip().endswith("ok")
