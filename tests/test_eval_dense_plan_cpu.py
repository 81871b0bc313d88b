"""Host-side checks of the eval levels plan, the backward of grad-enabled eval()-mode dense outputs (forward_levels,
forward_features, FasterViTBackbone; built on the CPU, nothing launched): running-statistics BatchNorms without
accumulators, the eval backward kernels, the image gradient, the stop level; and the train levels plan as before."""
import pytest
import torch

KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[2, 2, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7])


def _backbone(out_indices, fs=-1, train=False):
    from fastervit_b200.backbone import FasterViTBackbone
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=out_indices, frozen_stages=fs, drop_path_rate=0.3, **KW)
    return bb.train() if train else bb.eval()


def _plan(out_indices, fs=-1, eval_=True, normed=True):
    from fastervit_b200.engine_train import TrainPlan
    bb = _backbone(out_indices, fs, train=not eval_)
    norms = [getattr(bb, f"norm{i}") if normed else None for i in out_indices]
    spec = dict(kind="levels", outs=tuple(zip(out_indices, norms)), frozen=fs)
    if eval_:
        spec["eval"] = True
    return bb, TrainPlan(bb.body, 2, 160, 224, torch.device("cpu"), spec=spec)


def _names(ops):
    return [op[2] for op in ops]


@pytest.mark.parametrize("out_indices", [(0, 1, 2, 3), (1,), (2,), (0, 3)])
@pytest.mark.parametrize("normed", [True, False])
def test_eval_levels_plan_uses_running_statistics_and_the_eval_kernels(out_indices, normed):
    bb, plan = _plan(out_indices, normed=normed)
    fwd = _names(plan.ops)
    assert not [n for n in fwd + _names(plan._scale_ops) if n.startswith(("fvit_colstats", "fvit_bn_finalize"))]
    assert not plan.drop_specs and not plan.fwd_zero and not plan._bn_modules
    assert not [op for op in plan.ops if op[2] == "fvit_gemm" and (op[1][0]._obj.col_sum or op[1][0]._obj.col_sumsq)]
    assert "fvit_feature_map_fwd" not in fwd and not plan.outputs     # (the outputs come from the inference launch list)
    bwd = _names(plan.bwd_ops)
    assert "fvit_feature_map_bwd" not in bwd and "fvit_bn_bwd" not in bwd
    assert bwd.count("fvit_feature_map_eval_bwd") == len(out_indices)
    n_bn = sum(isinstance(mod, torch.nn.BatchNorm2d) for lv in bb.body.levels[:max(out_indices) + 1] if lv.conv
               for mod in lv.modules()) + 2                          # (+ the stem's two)
    assert bwd.count("fvit_bn_eval_bwd") == n_bn
    assert _names(plan._scale_ops).count("fvit_feature_map_bwd_stats") == len(out_indices)
    # the normed outputs: running mean / rstd in the stats pass and the apply; dw / dbeta into the norm's slices
    for (i, bn), d in zip(plan.spec["outs"], plan.dense):
        apply = [op[1] for op in plan.bwd_ops if op[2] == "fvit_feature_map_eval_bwd" and op[1][0] == d["dy"].data_ptr()]
        assert len(apply) == 1
        if normed:
            assert d["mu"] is bn.running_mean and apply[0][5] == d["rs"].data_ptr()
            assert apply[0][13] == plan.G(bn.weight) and apply[0][14] == plan.G(bn.bias)
        else:
            assert apply[0][5] is None and apply[0][13] is None
    # the image gradient, and a forward / backward that stop at the highest requested level
    assert tuple(plan.dx.shape) == (2, 3, 160, 224)
    assert "fvit_stem_conv_dgrad" in bwd
    assert plan.stop_level == max(out_indices)
    assert max(lv["level_index"] for lv in plan.conv_lv + plan.lv) == max(out_indices)


def test_eval_levels_plan_with_a_frozen_prefix():
    """x without a gradient: the backbone's frozen prefix gets no backward; its norm gradients still come out"""
    _, full = _plan((1, 2, 3), fs=-1)
    _, fs2 = _plan((1, 2, 3), fs=2)
    assert not hasattr(fs2, "dx") and "fvit_stem_conv_dgrad" not in _names(fs2.bwd_ops)
    assert len(fs2.bwd_ops) < len(full.bwd_ops)
    _, fs4 = _plan((1, 2), fs=4)          # both outputs inside the prefix: only the norms' dw / dbeta
    fmb = [a for fn, a, name in fs4.bwd_ops if name == "fvit_feature_map_eval_bwd"]
    assert len(fmb) == 2 and all(a[11] is None for a in fmb)
    assert not [op for op in fs4.bwd_ops if op[2] == "fvit_gemm"]


def test_eval_levels_plan_param_order_matches_the_engine():
    """the autograd node hands the plan's gradient views to the parameters it was given, in the same order"""
    from fastervit_b200.engine import Engine
    bb, plan = _plan((1, 2, 3))
    eng = Engine(bb.body)
    eng._check_weights()
    assert [id(p) for p in eng._dense_params(plan.spec["outs"])] == [id(p) for p in plan.params]


def test_train_levels_plan_keeps_its_launch_list():
    """batch statistics: pivoted column statistics + finalize per norm, the map forward, fvit_feature_map_bwd; no eval
    kernels and no image gradient"""
    out_indices = (0, 1, 2, 3)
    bb, plan = _plan(out_indices, eval_=False)
    fwd, bwd = _names(plan.ops), _names(plan.bwd_ops)
    assert fwd.count("fvit_colstats_pivot_f32") == len(out_indices)
    assert fwd.count("fvit_feature_map_fwd") == len(out_indices) and len(plan.outputs) == len(out_indices)
    assert bwd.count("fvit_feature_map_bwd") == len(out_indices)
    assert not [n for n in bwd if n in ("fvit_feature_map_eval_bwd", "fvit_bn_eval_bwd", "fvit_stem_conv_dgrad")]
    assert plan.drop_specs and plan.fwd_zero and not hasattr(plan, "dx")
    assert set(map(id, plan._bn_modules)) >= {id(getattr(bb, f"norm{i}")) for i in out_indices}
