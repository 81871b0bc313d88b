"""FasterViT-5 and -6 at full width (dim 320: level 3 is 2560 channels wide, every transformer head 80 wide), on the CPU:
the oracle against the fv5 golden of the unmodified reference (tests/make_golden_fv5.py), the state_dict schema, and
the eval, train and eval-gradient launch plans of the four entrypoints at full size (batch 2), built without a GPU. A
model whose LayerNorm rows are wider than the LayerNorm kernels take raises FvitError when its plan is built."""
import gc

import pytest
import torch

import fastervit_b200 as F
from fastervit_b200 import lib as L
from fastervit_b200.engine import LN_MAX_C

import _gemm_variants as V
import test_oracle_golden as golden
import test_product_cpu as product
from test_gemm_variants_cpu import plan_gemms, signature
from test_hd80_plan_cpu import attention_launches

ENTRIES = ["faster_vit_5_224", "faster_vit_6_224", "faster_vit_5_any_res", "faster_vit_6_any_res"]
# argument position of C per LayerNorm entry point (include/fvit.h)
_LN = {"fvit_ln_fwd": 4, "fvit_ln_bwd": 8, "fvit_ln_dgrad": 8}


def ln_widths(plan):
    """(entry point, C) of every LayerNorm launch in the plan's launch lists"""
    for lst in (v for v in vars(plan).values() if isinstance(v, list)):
        for op in lst:
            if isinstance(op, tuple) and len(op) == 3 and isinstance(op[2], str) and op[2] in _LN:
                args = op[1][2] if op[0] == "unless_deploy" else op[1]
                yield op[2], args[_LN[op[2]]]


def test_oracle_matches_the_fv5_golden():
    golden.test_oracle_eval_matches_reference_fp64("fv5")


def test_fv5_state_dict_schema_equals_reference():
    product.test_state_dict_schema_equals_reference("fv5")


@pytest.mark.parametrize("entry", ENTRIES)
def test_full_size_plans_build(entry):
    """eval, train and eval-gradient plans at batch 2 and the entrypoint's own resolution: every GEMM on a covered,
    non-generic fvit_gemm variant, every attention on the tensor-core kernels at padded head dim 80, and LayerNorm
    rows up to 2560 channels on the kernels that take them"""
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    covered = V.covered_triples()
    m = F.create_model(entry)
    res = m.cfg["resolution"]
    h, w = (res, res) if isinstance(res, int) else res
    builders = {"eval": lambda: Plan(m.eval(), 2, h, w, False, cpu),
                "train": lambda: TrainPlan(m.train(), 2, h, w, cpu),
                "eval-gradient": lambda: TrainPlan(m.eval(), 2, h, w, cpu, spec=dict(kind=None, eval=True))}
    for mode, build in builders.items():
        plan = build()
        missing = []
        for g in plan_gemms(plan):
            key = (L.gemm_args_variant(g), signature(g), V.vec_ok(g))
            assert key[0] != L.GEMM_F_GENERIC, (mode, g.m, g.n, g.kc)
            if key not in covered:
                missing.append((V.name(key[0]), key[1], key[2], g.m, g.n, g.kc))
        assert not missing, (mode, missing[:10])
        launches = set(attention_launches(plan))
        assert launches and all(d == 80 for _, _, d in launches), (mode, launches)
        assert not any(n.startswith("fvit_attn_core_") for n, _, _ in launches), (mode, launches)
        widths = set(ln_widths(plan))
        assert max(c for _, c in widths) == LN_MAX_C == 2560, (mode, widths)
        want = {"fvit_ln_fwd"} if mode == "eval" else {"fvit_ln_fwd", "fvit_ln_bwd"}
        assert {n for n, c in widths if c == 2560} == want, (mode, widths)
        del plan
        gc.collect()


@pytest.mark.parametrize("mode", ["eval", "train", "eval-gradient"])
def test_too_wide_layernorm_rows_raise_at_plan_build(mode):
    """dim 336: level 3 is 2688 channels wide, past the 2560 of the LayerNorm kernels"""
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    m = F.create_model("faster_vit_6_224", dim=336, depths=[1, 1, 1, 1])
    with pytest.raises(L.FvitError, match="level 3: 2688-channel LayerNorm rows.* at most 2560 channels"):
        if mode == "eval":
            Plan(m.eval(), 2, 224, 224, False, cpu)
        elif mode == "train":
            TrainPlan(m.train(), 2, 224, 224, cpu)
        else:
            TrainPlan(m.eval(), 2, 224, 224, cpu, spec=dict(kind=None, eval=True))
