"""Host-side checks of the fvit_gemm kernel-variant table: every compiled variant has a recipe in _gemm_variants.py
(so tests/test_gemm_variants_gpu.py runs it), every GEMM launch of the plans the package builds lands on a variant,
optional-input signature and store path that the GPU file exercises, and none falls through to the generic kernel.
The plans are built on the CPU; nothing is launched. Also the comparator's self-test."""
import pytest
import torch

import fastervit_b200 as F
from fastervit_b200 import lib as L

import _gemm_variants as V

_SMALL = dict(depths=[1, 1, 2, 1], in_dim=16, num_classes=10)


def _classification(name, dim):
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    m = F.create_model(name, drop_path_rate=0.1, dim=dim, **_SMALL)
    yield f"{name} eval", Plan(m.eval(), 2, 224, 224, False, cpu)
    yield f"{name} train", TrainPlan(m.train(), 2, 224, 224, cpu)
    yield f"{name} eval-gradient", TrainPlan(m.eval(), 2, 224, 224, cpu, spec=dict(kind=None, eval=True))


def plans():
    """(description, plan) of the reduced fv0 (no layer scale), fv4 and 21k (layer scale) models in inference,
    training with stochastic depth and eval-gradient mode, the detection backbone in levels-mode training at a DETR
    size, and the tracking backbone's frozen-BatchNorm / LayerNorm2d recipe in training."""
    from fastervit_b200.engine_train import TrainPlan
    yield from _classification("faster_vit_0_224", 32)
    yield from _classification("faster_vit_4_224", 64)
    yield from _classification("faster_vit_4_21k_224", 64)
    cpu = torch.device("cpu")
    from fastervit_b200.detection import build_fastervit as det_build
    det = det_build("faster_vit_0_224", out_indices=(0, 1, 2, 3), drop_path_rate=0.1, dim=16, in_dim=16,
                    depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]).train()
    outs = tuple((i, getattr(det, f"norm{i}")) for i in range(4))
    yield "detection levels train 160x224", TrainPlan(det, 2, 160, 224, cpu, dict(kind="levels", outs=outs, frozen=-1))
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit as trk_build
    from test_tracking_cpu import _layernorm2d
    trk = trk_build("faster_vit_0_224", FrozenBatchNorm2d, _layernorm2d(), out_indices=(0, 1, 2, 3), drop_path_rate=0.1,
                    frozen_stages=0, dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]).train()
    outs = tuple((i, trk._level_norm(i)) for i in range(4))
    yield "tracking frozen/LN train 96x160", TrainPlan(trk, 2, 96, 160, cpu, spec=dict(kind="levels", outs=outs, frozen=0))


def plan_gemms(plan):
    """The GemmArgs of every fvit_gemm launch in the plan's launch lists."""
    for lst in (v for v in vars(plan).values() if isinstance(v, list)):
        for op in lst:
            if isinstance(op, tuple) and len(op) == 3 and op[2] == "fvit_gemm":
                args = op[1][2] if op[0] == "unless_deploy" else op[1]
                yield args[0]._obj


def signature(g) -> tuple:
    return V.signature_of(**{f: bool(getattr(g, f)) for f in ("col_scale", "col_shift", "aux_scale", "row_map")},
                          taps=g.ntaps > 1, b_taps=g.b_ntaps > 1)


def test_every_variant_has_a_recipe():
    got = L.gemm_variants()
    assert len(got) == len(set(got)) == 30
    assert set(V.RECIPES) == set(got), sorted(hex(v) for v in set(V.RECIPES) ^ set(got))
    assert L.GEMM_F_GENERIC not in got


def test_recipes_record_their_signature():
    for variant, r in V.RECIPES.items():
        assert r.variant == variant
        assert isinstance(r.sig, tuple) and set(r.sig) <= set(V.SIG_FIELDS)


@pytest.fixture(scope="module")
def launches():
    out = {}
    for desc, plan in plans():
        for g in plan_gemms(plan):
            out.setdefault((L.gemm_args_variant(g), signature(g), V.vec_ok(g)), []).append((desc, g.m, g.n, g.kc))
    return out


def test_plans_launch_only_covered_variants(launches):
    covered = V.covered_triples()
    missing = {k: v[0] for k, v in launches.items() if k not in covered}
    assert not missing, "\n".join(f"{V.name(k[0])} sig={k[1]} vec_ok={k[2]} e.g. {v}" for k, v in missing.items())


def test_no_plan_launch_takes_the_generic_kernel(launches):
    generic = [v[0] for k, v in launches.items() if k[0] == L.GEMM_F_GENERIC]
    assert not generic, generic
    # every plan kind contributes launches, and the train plans reach the split-K weight gradient
    assert sum(len(v) for v in launches.values()) > 300
    assert any(k[0] == V.SPLITK_WGRAD for k in launches)


def test_variant_query_validates_like_the_launcher():
    a = torch.zeros(256, 64, dtype=torch.float16)
    b = torch.zeros(64, 64, dtype=torch.float16)
    o16 = torch.zeros(256, 64, dtype=torch.float16)
    assert L.gemm_variant(a, b, out_f16=o16) == L.GEMM_F_DIRECT | L.GEMM_F_O16
    assert L.gemm_variant(a, b, n=56, out_f16=o16[:, :56]) == L.GEMM_F_O16            # n % 16 != 0: staged
    assert L.gemm_variant(a.bfloat16(), b.bfloat16(), out_f16=o16) == L.GEMM_F_GENERIC  # bf16: generic only
    with pytest.raises(L.FvitError, match="no output"):
        L.gemm_variant(a, b)
    with pytest.raises(L.FvitError, match="backward activation needs aux"):
        L.gemm_variant(a, b, out_f16=o16, act=L.ACT_GELU_BWD)


def test_comparator_rejects_one_planted_element():
    """A GEMM result that meets the per-element bound everywhere passes; the same result with one element off by 1e-3
    relative, in a column whose magnitude is 1 % of the matrix maximum, fails."""
    g = torch.Generator().manual_seed(0)
    m, n, k = 96, 40, 784
    a = torch.randn(m, k, generator=g).half()
    b = torch.randn(n, k, generator=g)
    b[7] *= 0.01
    b = b.half()
    ref = a.double() @ b.double().t()
    bound = V.acc_bound(a.double().abs() @ b.double().abs().t(), k) + V.U32 * ref.abs()
    got = (a.float() @ b.float().t()).double()
    V.assert_within(got, ref, bound, "clean")
    assert ref[:, 7].abs().max() < 0.02 * ref.abs().max()
    i = int(ref[:, 7].abs().argmax())
    bad = got.clone()
    bad[i, 7] = ref[i, 7] * (1 + 1e-3)
    with pytest.raises(AssertionError, match="planted"):
        V.assert_within(bad, ref, bound, "planted")
    # the same element with fp16 output rounding allowed
    bound16 = bound + V.U16 * ref.abs() + 2.0 ** -25
    bad16 = ref.half().double()
    bad16[i, 7] = ref[i, 7] * (1 + 1e-3)
    with pytest.raises(AssertionError):
        V.assert_within(bad16, ref, bound16, "planted16")
