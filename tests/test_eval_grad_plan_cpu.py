"""Host-side checks of the eval-grad plan, the backward of a grad-enabled eval()-mode forward (built on the CPU, nothing
launched): running-statistics BatchNorms without accumulators, the eval backward kernels, the conv-bias gradients, the
image gradient, and the side-branch hazards of its backward list."""
import pytest
import torch

import fastervit_b200 as F


def _reduced(name: str) -> dict:
    spec = F.configs.MODEL_SPECS[name]["defaults"]
    dim = spec["num_heads"][0] * 4 * 2
    kw = dict(dim=dim, in_dim=16, num_classes=10)
    if name.endswith("any_res"):
        kw["resolution"] = [160, 224]
    return kw


def _plan(name: str, monkeypatch=None, kind=None):
    from fastervit_b200.engine_train import TrainPlan
    kw = _reduced(name)
    if kind == "pooled":
        kw["num_classes"] = 0
    m = F.create_model(name, drop_path_rate=0.3, **kw).eval()
    res = kw.get("resolution", m.cfg["resolution"])
    H, W = (res if isinstance(res, (list, tuple)) else (res, res))
    return m, TrainPlan(m, 2, H, W, torch.device("cpu"), spec=dict(kind=kind, eval=True))


def _names(ops):
    return [op[2] for op in ops]


@pytest.mark.parametrize("kind", [None, "pooled"])
@pytest.mark.parametrize("name", ["faster_vit_0_224", "faster_vit_0_any_res"])
def test_eval_grad_plan_uses_running_statistics_and_the_eval_backward_kernels(name, kind):
    m, plan = _plan(name, kind=kind)
    fwd = _names(plan.ops)
    assert not [n for n in fwd if n.startswith(("fvit_colstats", "fvit_bn_finalize"))]
    assert not plan.drop_specs and not plan.fwd_zero and not plan._bn_modules
    # the convolution GEMMs accumulate no statistics either
    assert not [op for op in plan.ops if op[2] == "fvit_gemm" and (op[1][0]._obj.col_sum or op[1][0]._obj.col_sumsq)]
    bwd = _names(plan.bwd_ops)
    n_bn2d = sum(isinstance(mod, torch.nn.BatchNorm2d) for mod in m.modules())
    assert "fvit_bn_bwd" not in bwd and "fvit_pool_bn_bwd" not in bwd
    assert bwd.count("fvit_bn_eval_bwd") == n_bn2d - 1          # (the head norm is the pooled one)
    assert bwd.count("fvit_pool_bn_eval_bwd") == 1
    assert bwd.count("fvit_stem_conv_dgrad") == 1
    assert tuple(plan.dx.shape) == (2, 3, plan.H, plan.W)
    # one column sum per ConvBlock convolution bias, into that bias' gradient slice
    biases = [conv.bias for lv in m.levels if lv.conv for blk in lv.blocks for conv in (blk.conv1, blk.conv2)]
    assert biases
    for b in biases:
        hits = [op for op in plan.bwd_ops if op[2] == "fvit_colsum" and plan.G(b) in op[1]]
        assert len(hits) == 1


def test_train_plans_keep_their_launch_lists():
    """the classification train plan has no eval kernels, and its conv-bias gradients stay identically zero"""
    from fastervit_b200.engine_train import TrainPlan
    kw = _reduced("faster_vit_0_224")
    m = F.create_model("faster_vit_0_224", drop_path_rate=0.3, **kw).train()
    plan = TrainPlan(m, 2, 224, 224, torch.device("cpu"))
    bwd = _names(plan.bwd_ops)
    assert "fvit_bn_eval_bwd" not in bwd and "fvit_pool_bn_eval_bwd" not in bwd and "fvit_stem_conv_dgrad" not in bwd
    assert bwd.count("fvit_bn_bwd") == sum(isinstance(mod, torch.nn.BatchNorm2d) for mod in m.modules()) - 1
    assert plan.drop_specs and plan.fwd_zero


@pytest.mark.parametrize("name", ["faster_vit_0_224", "faster_vit_0_any_res"])
def test_eval_grad_side_branch_weight_gradients_never_race_a_buffer_rewrite(name):
    """the hazard walk of the train plan's side-branch weight gradients (test_product_cpu.py), on the eval-grad
    backward, whose conv-bias column sums join the side branch"""
    _, plan = _plan(name)
    assert any(o[0] == "wait_side" for o in plan.bwd_ops)
    side_all = plan._bwd_side | plan._bwd_side_wgrad
    assert plan._side_set() is None         # (no launch graphs on the host: every marker is inert)
    pure_readers = {"fvit_colsum"}          # main-branch launches that only read the activation gradient they are handed
    outstanding: dict[int, int] = {}        # buffer -> index of the side launch still reading it
    n_side_gemm = n_wgrad = 0
    for i, (fn, args, nm) in enumerate(plan.bwd_ops):
        if fn == "wait_side":
            for k in args:
                outstanding.pop(k, None)
            continue
        if fn == "bucket":
            outstanding.clear()             # bucket points join the side branch
            continue
        gemm = nm == "fvit_gemm"
        g = args[0]._obj if gemm else None
        if gemm and g.a_mn_major and g.b_mn_major:   # dW = dZ^T X: both operands read along the token dimension
            n_wgrad += 1
            big = g.m * g.n * g.kc >= 64 * 64 * 1024
            assert (i in side_all) or not big or g.m <= 64, (i, g.m, g.n, g.kc)
        if i in side_all:
            n_side_gemm += gemm
            for k in plan._side_reads.get(i, ()):
                outstanding[k] = i
            continue
        if gemm:
            writes = {int(p) for p in (g.out_f16, g.out_f32, g.out_pre16) if p}
        elif nm in pure_readers:
            writes = set()
        else:
            writes = {a for a in args if isinstance(a, int) and a in outstanding}
        clash = writes & set(outstanding)
        assert not clash, (i, nm, [outstanding[c] for c in clash])
    assert n_side_gemm >= 0.8 * n_wgrad > 0
