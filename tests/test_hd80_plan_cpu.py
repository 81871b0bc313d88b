"""Launch plans of models with 80-wide attention heads (FasterViT-5 / -6: dim 320, heads [4, 8, 16, 32]), built on the
CPU: every attention runs on the tensor-core kernels at padded head dim 80 (the tile kernels up to 63 tokens, the
key-loop kernels from 64 on in training), head dims 65 .. 79 are padded to 80, every GEMM lands on a variant that
tests/test_gemm_variants_gpu.py covers, and the plans of the existing reduced models contain no hdp-80 launch."""
import pytest
import torch

import fastervit_b200 as F
from fastervit_b200 import lib as L

import _attn_geometry
import _gemm_variants as V
from test_gemm_variants_cpu import plan_gemms, plans as existing_plans, signature

# reduced FasterViT-5: 80-wide heads at levels 2 (320 / 4) and 3 (640 / 8); channel counts that are multiples of 16
HD80 = dict(dim=80, in_dim=16, num_heads=[1, 2, 4, 8], depths=[1, 1, 2, 2], layer_scale=1e-5)
AR80 = dict(HD80, resolution=[384, 576], window_size=[7, 7, 12, 6], ct_size=2)


def attention_launches(plan):
    """(entry point, S, padded head dim) of every attention-core launch in the plan's launch lists (for the SIMT
    forward the last field is the unpadded head dim, its only head-width argument)"""
    for a in _attn_geometry.attention_launches(plan):
        yield a.entry, a.S, a.hdp


def _plans(name, kw, res, drop_path_rate=0.1):
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    m = F.create_model(name, drop_path_rate=drop_path_rate, **kw)
    h, w = (res, res) if isinstance(res, int) else res
    yield "eval", Plan(m.eval(), 2, h, w, False, cpu)
    yield "train", TrainPlan(m.train(), 2, h, w, cpu)
    yield "eval-gradient", TrainPlan(m.eval(), 2, h, w, cpu, spec=dict(kind=None, eval=True))


def hd80_plans():
    for desc, plan in _plans("faster_vit_5_224", HD80, 224):
        yield f"fv5-like 224 {desc}", plan
    for desc, plan in _plans("faster_vit_5_any_res", AR80, AR80["resolution"]):
        yield f"fv5-like any-res {desc}", plan


@pytest.fixture(scope="module")
def hd80():
    return [(desc, plan, sorted(set(attention_launches(plan)))) for desc, plan in hd80_plans()]


def test_every_attention_of_the_hd80_models_runs_on_tensor_cores(hd80):
    for desc, plan, launches in hd80:
        assert launches, desc
        names = {n for n, _, _ in launches}
        assert not names & {"fvit_attn_core_fwd", "fvit_attn_core_bwd"}, (desc, launches)
        assert "fvit_hat_attn_fwd" not in names, desc       # the fused kernel is 64 only
        assert all(d == 80 for _, _, d in launches), (desc, launches)
        if "train" in desc or "gradient" in desc:
            assert any(n.endswith("_bwd") or n.endswith("_bwd_long") for n in names), desc


def test_hd80_window_shapes_reach_the_kernels_fv5_runs(hd80):
    got = {desc: launches for desc, _, launches in hd80}
    # 224: level-2 windows of 49 + 4 carrier tokens, 16 carriers, level-3 windows of 49 tokens
    for mode in ("eval", "train"):
        assert {("fvit_attn_tc_fwd", S, 80) for S in (53, 16, 49)} <= set(got[f"fv5-like 224 {mode}"])
    assert {("fvit_attn_tc_bwd", S, 80) for S in (53, 16, 49)} <= set(got["fv5-like 224 train"])
    # any-res, window 12 at level 2: S = 144 + 4 = 148 trains through the key-loop kernels
    assert ("fvit_attn_loop_fwd", 148, 80) in got["fv5-like any-res eval"]
    for mode in ("train", "eval-gradient"):
        assert {("fvit_attn_loop_fwd", 148, 80), ("fvit_attn_loop_bwd_long", 148, 80)} <= set(got[f"fv5-like any-res {mode}"])


def test_a_64_token_window_at_hdp_80_trains_through_the_key_loop():
    """fvit_attn_tc_bwd's shared memory holds S <= 63 at hdp 80: a 64-token window (level 3, window 8, no carriers)
    takes the key-loop forward and backward in training, and stays on the tile forward in inference"""
    kw = dict(AR80, window_size=[7, 7, 12, 8])
    got = {desc: set(attention_launches(plan)) for desc, plan in _plans("faster_vit_5_any_res", kw, kw["resolution"])}
    assert ("fvit_attn_tc_fwd", 64, 80) in got["eval"]
    for mode in ("train", "eval-gradient"):
        assert {("fvit_attn_loop_fwd", 64, 80), ("fvit_attn_loop_bwd_long", 64, 80)} <= got[mode], got[mode]
        assert not any(S == 64 and n in ("fvit_attn_tc_fwd", "fvit_attn_tc_bwd") for n, S, _ in got[mode])


@pytest.mark.parametrize("hd,hdp", [(32, 32), (49, 64), (64, 64), (65, 80), (72, 80), (80, 80), (81, 81), (96, 96)])
def test_head_pad(hd, hdp):
    from fastervit_b200.engine import Plan
    assert Plan._head_pad(hd) == hdp
    assert (Plan._attn_kind(49, hdp) == "simt") == (hdp > 80)


def test_hd72_heads_are_padded_to_80():
    """dim 72: 72-wide heads at level 2 (288 / 4) and 3 (576 / 8), zero-padded to 80 through the head-padding kernels"""
    kw = dict(HD80, dim=72)
    for desc, plan in _plans("faster_vit_5_224", kw, 224):
        launches = set(attention_launches(plan))
        assert launches and all(d == 80 for _, _, d in launches), (desc, launches)
        names = {op[2] for lst in vars(plan).values() if isinstance(lst, list) for op in lst
                 if isinstance(op, tuple) and len(op) == 3 and isinstance(op[2], str)}
        assert "fvit_cast_headpad_f16" in names, desc


def test_hd80_gemms_take_covered_variants():
    covered = V.covered_triples()
    missing, n = [], 0
    for desc, plan in hd80_plans():
        for g in plan_gemms(plan):
            n += 1
            key = (L.gemm_args_variant(g), signature(g), V.vec_ok(g))
            assert key[0] != L.GEMM_F_GENERIC, (desc, g.m, g.n, g.kc)
            if key not in covered:
                missing.append((desc, V.name(key[0]), key[1], key[2], g.m, g.n, g.kc))
    assert n > 100
    assert not missing, missing[:10]


def test_existing_models_have_no_hdp80_launch():
    for desc, plan in existing_plans():
        bad = [a for a in attention_launches(plan) if a[2] == 80]
        assert not bad, (desc, bad)
