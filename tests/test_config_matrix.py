"""The configuration matrix (support.CONFIGS) on CPU: each entry's schedule and the property it exists for, pinned as literals so that
an edit of the matrix cannot quietly drop what tests/test_gpu_configs.py runs on the engine; the fp32 oracle runs every entry, the
step reference restates its fp64 copy on every schedule, and the engine's config and checkpoint audit accepts every entry.
"""
import pytest
import torch

import support
from test_cabi import _create, needs_no_gpu
from test_step_ref import _check_restatement

# name -> the schedule (BertEncoder.schedule()) and the facts _facts reads off the config
EXPECTED = {
    "heads_swapped": dict(schedule="T0 T1 T2 T3 T4 T5 C0 T6 V0 C1 T7 V1 C2 T8 V2 C3 T9 V3 C4 T10 V4 C5 V5 T11",
                          head_sizes=(128, 64, 64), bi_heads_most=True, bi_hidden_is_v_hidden=False, odd_tile_widths=(),
                          v_feature_mod_64=0, image_prefix_layers=0, adjacent_c=False, ends=("T", "V"), task_tokens=True),
    "odd_widths": dict(schedule="T0 T1 T2 T3 T4 T5 C0 T6 V0 C1 T7 V1 C2 T8 V2 C3 T9 V3 C4 T10 V4 C5 V5 T11",
                       head_sizes=(64, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=False, odd_tile_widths=(384, 640),
                       v_feature_mod_64=8, image_prefix_layers=0, adjacent_c=False, ends=("T", "V"), task_tokens=True),
    "back_to_back": dict(schedule="T0 V0 C0 T1 T2 C1 C2 T3 T4 T5 V1 V2 V3 C3",
                         head_sizes=(64, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=True, odd_tile_widths=(),
                         v_feature_mod_64=0, image_prefix_layers=1, adjacent_c=True, ends=("C", "C"), task_tokens=True),
    "text_ends_in_c": dict(schedule="T0 T1 C0 T2 T3 V0 C1 V1 V2",
                           head_sizes=(64, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=True, odd_tile_widths=(),
                           v_feature_mod_64=0, image_prefix_layers=0, adjacent_c=False, ends=("C", "V"), task_tokens=True),
    "no_coattention": dict(schedule="V0 V1 T0 T1 T2",
                           head_sizes=(64, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=True, odd_tile_widths=(),
                           v_feature_mod_64=0, image_prefix_layers=2, adjacent_c=False, ends=("T", "V"), task_tokens=True),
    "no_task_tokens": dict(schedule="T0 T1 T2 T3 T4 T5 C0 T6 V0 C1 T7 V1 C2 T8 V2 C3 T9 V3 C4 T10 V4 C5 V5 T11",
                           head_sizes=(64, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=True, odd_tile_widths=(),
                           v_feature_mod_64=0, image_prefix_layers=0, adjacent_c=False, ends=("T", "V"), task_tokens=False),
    "wide_text": dict(schedule="T0 V0 C0 V1 T1",
                      head_sizes=(128, 128, 128), bi_heads_most=False, bi_hidden_is_v_hidden=True, odd_tile_widths=(),
                      v_feature_mod_64=0, image_prefix_layers=1, adjacent_c=False, ends=("T", "V"), task_tokens=True),
}


def _facts(c, schedule):
    """What a configuration reaches in a plan, read off the config and its schedule."""
    first_c = schedule.index("C0") if "C0" in schedule else len(schedule)
    widths = (c.hidden_size, c.intermediate_size, c.v_hidden_size, c.v_intermediate_size, c.bi_hidden_size)
    last = lambda skip: next(s[0] for s in reversed(schedule) if s[0] != skip)
    return dict(schedule=" ".join(schedule),
                head_sizes=(c.hidden_size // c.num_attention_heads, c.v_hidden_size // c.v_num_attention_heads,
                            c.bi_hidden_size // c.bi_num_attention_heads),
                bi_heads_most=c.bi_num_attention_heads > max(c.num_attention_heads, c.v_num_attention_heads),
                bi_hidden_is_v_hidden=c.bi_hidden_size == c.v_hidden_size,
                odd_tile_widths=tuple(sorted({w for w in widths if w > 128 and w % 128 == 0 and (w // 128) % 2 == 1})),
                v_feature_mod_64=c.v_feature_size % 64,
                image_prefix_layers=sum(s[0] == "V" for s in schedule[:first_c]),
                adjacent_c=any(a[0] == b[0] == "C" for a, b in zip(schedule, schedule[1:])),
                ends=(last("V"), last("T")),
                task_tokens=bool(c.task_specific_tokens))


def test_matrix_is_pinned():
    assert sorted(support.CONFIGS) == sorted(EXPECTED)
    assert support.CONFIG_LABELS == 129


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_schedule_and_property(name):
    oracle = support.config_oracle(name)
    assert _facts(oracle.config, oracle.bert.encoder.schedule()) == EXPECTED[name]


def test_matrix_reaches_every_property():
    """Every plan property the matrix exists for is reached by at least one entry."""
    f = EXPECTED
    assert any(x["head_sizes"][0] == 128 for x in f.values()) and any(x["head_sizes"][1:] == (64, 64) for x in f.values())
    assert any(x["bi_heads_most"] for x in f.values()) and any(not x["bi_hidden_is_v_hidden"] for x in f.values())
    assert {384, 640} <= {w for x in f.values() for w in x["odd_tile_widths"]}
    assert any(x["v_feature_mod_64"] for x in f.values())
    assert any(x["image_prefix_layers"] for x in f.values()) and any(x["adjacent_c"] for x in f.values())
    assert any(x["ends"] == ("C", "C") for x in f.values()) and any(x["ends"] == ("C", "V") for x in f.values())
    assert any("C" not in x["schedule"] for x in f.values()) and any(x["schedule"].startswith("T0 V0 C0") for x in f.values())
    assert any(not x["task_tokens"] for x in f.values())
    assert any(c.get("hidden_size") == 1024 for c in support.CONFIGS.values())


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_oracle_runs(name):
    """The fp32 oracle of each entry on a padded batch: one map per schedule step (a pair per connection layer), nine outputs."""
    oracle = support.config_oracle(name)
    inp = support.tiny_inputs(oracle, 2, 9, 6, seed=3, pad=2)
    out = oracle(*inp, output_all_attention_masks=True)
    schedule = oracle.bert.encoder.schedule()
    assert len(out[9]) == len(schedule)
    T = 9 + (1 if oracle.config.task_specific_tokens else 0)
    for step, p in zip(schedule, out[9]):
        assert isinstance(p, tuple) == (step[0] == "C"), step
    assert out[0].shape == (2, support.CONFIG_LABELS) and out[8].shape == (2, T, 1)
    assert all(torch.isfinite(o).all() for o in out[:9])


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_step_reference_restates_oracle(name):
    """oracle.step_ref without rounding is the fp64 oracle on each entry's schedule, head sizes and task-token layout."""
    oracle = support.config_oracle(name)
    _check_restatement(oracle, support.tiny_inputs(oracle, 3, 12, 9, seed=5, pad=2), name)


@needs_no_gpu
@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_engine_audit_accepts(name):
    """vb200_create's config and checkpoint audit passes every entry: the call gets as far as the missing device."""
    import vilbert_b200 as vb
    oracle = support.config_oracle(name)
    rc, msg = _create(vb.BertConfig.from_dict(oracle.config.to_dict()), oracle.state_dict(), num_labels=support.CONFIG_LABELS)
    assert rc == -5 and "no CPU fallback" in msg, (rc, msg)
