"""Host-side checks of the train-mode image gradient and the data-only backward stages (plans built on the CPU, nothing
launched): the stage mask, plan-key separation, which parameters get flat-buffer slices, the launch lists, and the new
entry points in include/fvit.h and lib.py."""
import collections
import contextlib
import re
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[2, 2, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7])
NEW = ("fvit_bn_eval_dgrad", "fvit_ln_dgrad", "fvit_token_init_dgrad")
PARAM_OPS = ("fvit_colsum", "fvit_cpb_mlp_bwd", "fvit_attn_bias_bwd", "fvit_bn_eval_bwd", "fvit_bn_bwd", "fvit_ln_bwd",
             "fvit_branch_grad", "fvit_group_sum", "fvit_unpack_conv_grad", "fvit_token_init_bwd", "fvit_unpad_heads_f32")


def _names(ops):
    return collections.Counter(op[2] for op in ops)


def _wgrads(ops):
    return sum(1 for op in ops if op[2] == "fvit_gemm" and op[1][0]._obj.a_mn_major and op[1][0]._obj.b_mn_major)


def _backbone_plan(fs, train, **spec):
    from fastervit_b200.backbone import FasterViTBackbone
    from fastervit_b200.engine_train import TrainPlan
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=fs, drop_path_rate=0.3, **KW)
    bb = bb.train() if train else bb.eval()
    outs = tuple((i, getattr(bb, f"norm{i}")) for i in (1, 2, 3))
    full = dict(kind="levels", outs=outs, frozen=fs, **spec)
    if not train:
        full["eval"] = True
    return bb, TrainPlan(bb.body, 2, 160, 224, torch.device("cpu"), spec=full)


def test_stage_mask_from_requires_grad_and_from_frozen_stages():
    from fastervit_b200.engine_train import stage_mask
    bb, plan = _backbone_plan(2, True)
    assert stage_mask(bb.body, lambda p: p.requires_grad) == (True, True, False, False, False)
    assert plan.data_only == (True, True, False, False, False) and not plan.want_dx
    for fs, want in ((-1, 0), (0, 1), (1, 1), (3, 3)):
        assert sum(_backbone_plan(fs, True)[1].data_only) == want
    bb.body.levels[3].blocks[0].norm1.weight.requires_grad_(False)    # one frozen tensor does not make a stage data-only
    assert stage_mask(bb.body, lambda p: p.requires_grad)[4] is False


def test_train_plan_without_dx_keeps_its_launch_list_and_dx_adds_the_prefix():
    for fs in (-1, 0, 2, 3):
        _, p0 = _backbone_plan(fs, True)
        _, p1 = _backbone_plan(fs, True, want_dx=True)
        n0, n1 = _names(p0.bwd_ops), _names(p1.bwd_ops)
        assert not hasattr(p0, "dx") and not any(n0[k] for k in NEW + ("fvit_stem_conv_dgrad", "fvit_stem_col2im"))
        assert tuple(p1.dx.shape) == (2, 3, 160, 224) and n1["fvit_stem_conv_dgrad"] == 1
        # the image gradient costs no weight-gradient GEMM and no parameter reduction: the prefix is data-only
        assert _wgrads(p1.bwd_ops) == _wgrads(p0.bwd_ops)
        for k in PARAM_OPS:
            assert n1[k] == n0[k], (fs, k)
        if fs < 0:
            assert len(p1.bwd_ops) == len(p0.bwd_ops) + 1 and not any(n1[k] for k in NEW)
        else:
            assert n1["fvit_bn_eval_dgrad"] == 2 + 4 * p1.n_frozen_lv and n1["fvit_ln_dgrad"] == p1.n_frozen_lv
        # a train plan keeps one flat-buffer layout whatever the input asks for
        assert len(p0._goff) == len(p1._goff) == len(p1.params) and p0.gflat.numel() == p1.gflat.numel()
        frozen = {id(p) for s, mod in enumerate([p1.model.patch_embed, *p1.model.levels]) if p1.data_only[s]
                  for p in mod.parameters()}
        views = p1.grad_views_on_path()
        assert all((v is None) for p, v in zip(p1.params, views) if id(p) in frozen)


def test_eval_plan_all_stages_data_only():
    _, full = _backbone_plan(-1, False)
    bb, do = _backbone_plan(-1, False, want_dx=True, data_only=(True,) * 5)
    n = _names(do.bwd_ops)
    assert _wgrads(full.bwd_ops) > 30 and _wgrads(do.bwd_ops) == 0
    assert not any(n[k] for k in PARAM_OPS)
    assert n["fvit_stem_conv_dgrad"] == 1 and n["fvit_token_init_dgrad"] == 1
    assert n["fvit_bn_eval_dgrad"] == _names(full.bwd_ops)["fvit_bn_eval_bwd"]
    assert n["fvit_ln_dgrad"] == _names(full.bwd_ops)["fvit_ln_bwd"]
    launches = lambda ops: sum(1 for op in ops if op[0] not in ("wait_side", "bucket"))
    assert launches(do.bwd_ops) < 0.7 * launches(full.bwd_ops)
    # the attention backward runs without its bias-gradient accumulator
    attn = [op[1] for op in do.bwd_ops if op[2].startswith("fvit_attn_")]
    assert attn and all(a[-1] is None for a in attn if len(a) == 14)
    # slices: only the level norms' and the final norm's (they are no stage's parameters)
    with_slice = {id(p) for p in do.params if id(p) in do._goff}
    assert with_slice == {id(p) for n in ("norm1", "norm2", "norm3") for p in getattr(bb, n).parameters()} | {
        id(p) for p in bb.body.norm.parameters()}
    assert do.gflat.numel() < full.gflat.numel() // 100
    views = do.grad_views()
    assert [v is None for v in views] == [id(p) not in with_slice for p in do.params]


def test_eval_plan_mixed_mask_and_no_dx():
    """only levels[3] takes gradients and x none: the backward ends below level 3; with x it crosses the rest data-only"""
    mask = (True, True, True, True, False)
    _, top = _backbone_plan(-1, False, want_dx=False, data_only=mask)
    _, dx = _backbone_plan(-1, False, want_dx=True, data_only=mask)
    assert not hasattr(top, "dx") and not any(_names(top.bwd_ops)[k] for k in NEW)
    assert _wgrads(top.bwd_ops) == _wgrads(dx.bwd_ops) == 4
    assert len(dx.bwd_ops) > len(top.bwd_ops) and _names(dx.bwd_ops)["fvit_stem_conv_dgrad"] == 1
    lvl3 = {id(p) for p in dx.model.levels[3].parameters()}
    assert lvl3 <= dx._goff.keys() and not ({id(p) for p in dx.model.levels[2].parameters()} & dx._goff.keys())
    # a trained stage below a data-only one keeps the gradient flowing through it
    _, stem = _backbone_plan(-1, False, want_dx=False, data_only=(False, True, True, True, True))
    n = _names(stem.bwd_ops)
    assert n["fvit_bn_eval_bwd"] == 2 and n["fvit_bn_eval_dgrad"] == 8 and "fvit_stem_conv_dgrad" not in n


def test_plan_keys_separate_dx_and_masks(monkeypatch):
    from fastervit_b200 import engine as E
    from fastervit_b200.registry import create_model
    m = create_model("faster_vit_0_any_res", **KW).eval()
    eng = E.Engine(m)
    built = []

    class FakePlan:
        def __init__(self, model, B, H, W, device, spec=None):
            built.append(spec)

    import fastervit_b200.engine_train as ET
    monkeypatch.setattr(ET, "TrainPlan", FakePlan)
    monkeypatch.setattr(E.Engine, "_check_weights", lambda self: ())
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())

    class X:   # a CUDA-looking input: only its metadata is read
        is_cuda, dtype, shape = True, torch.float32, torch.Size((2, 3, 160, 224))
        device = next(m.parameters()).device

        def dim(self):
            return 4
    x = X()
    a = eng.eval_grad_plan(x)
    assert eng.eval_grad_plan(x, True, (False,) * 5) is a              # nothing data-only, dx wanted: today's plan
    b = eng.eval_grad_plan(x, True, (True,) * 5)
    c = eng.eval_grad_plan(x, False, (True,) * 5)
    d = eng.eval_grad_plan(x, True, (True, True, False, False, False))
    assert len({id(p) for p in (a, b, c, d)}) == 4 and eng.eval_grad_plan(x, True, (True,) * 5) is b
    assert built[0] == dict(kind=None, eval=True) and built[1]["data_only"] == (True,) * 5 and built[2]["want_dx"] is False
    outs = ((1, None),)
    e = eng.eval_dense_plan(x, outs, 2)
    f = eng.eval_dense_plan(x, outs, 2, True, (True, True, False, False, False))
    assert e is not f and eng.eval_dense_plan(x, outs, 2) is e


def test_new_entry_points_are_declared_and_bound():
    from fastervit_b200 import lib
    header = (ROOT / "include" / "fvit.h").read_text()
    cdll = lib.load()
    for name in NEW:
        decl = re.search(name + r"\s*\(([^;]*)\);", header)
        assert decl, name
        nargs = len([a for a in decl.group(1).split(",") if a.strip()])
        assert len(lib._OP_SIGS[name]) == nargs, name      # (the stream included)
        assert getattr(cdll, name).argtypes == lib._OP_SIGS[name]
