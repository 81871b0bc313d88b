"""Host-side checks of the stem launches for in_chans != 3 (plans built on the CPU, nothing launched): the im2col row
width stem_ld = round_up(9 * in_chans, 32), the conv1 GEMM's K, the weight-gradient width, the image-gradient GEMM and
col2im of the eval-grad plan, the RGB launches kept as they were, and the in_chans limit."""
import pytest
import torch

import fastervit_b200 as F
from fastervit_b200 import lib as L
from fastervit_b200.engine import Plan


def _model(name: str, cin: int):
    kw = dict(dim=16, in_dim=16, num_classes=10, in_chans=cin)
    if name.endswith("any_res"):
        kw["resolution"] = [160, 224]
    m = F.create_model(name, **kw).eval()
    res = kw.get("resolution", m.cfg["resolution"])
    return m, (res if isinstance(res, (list, tuple)) else (res, res))


def _gemms(ops):
    return [op[1][0]._obj for op in ops if op[2] == "fvit_gemm"]


def _stem(plan, m):
    """(im2col args, conv1 weight cast args, conv1 GEMM) of a plan's forward"""
    w = m.patch_embed.conv_down[0].weight.data_ptr()
    cast = [op[1] for op in plan.prep_ops if op[2] == "fvit_cast_pad_f16" and op[1][0] == w]
    assert len(cast) == 1
    im2col = [op for op in plan.ops if op[0] == "im2col"]
    assert len(im2col) == 1 and plan.ops[0] is im2col[0]
    col = plan._x_args[im2col[0][1]]
    conv1 = [g for g in _gemms(plan.ops) if g.a == col["out"]]
    assert len(conv1) == 1
    return col, cast[0], conv1[0]


def _eval_grad_plan(m, H, W):
    from fastervit_b200.engine_train import TrainPlan
    return TrainPlan(m, 2, H, W, torch.device("cpu"), spec=dict(kind=None, eval=True))


@pytest.mark.parametrize("name", ["faster_vit_0_224", "faster_vit_0_any_res"])
@pytest.mark.parametrize("cin,sld", [(1, 32), (4, 64), (13, 128), (64, 576)])
def test_stem_launches_follow_in_chans(name, cin, sld):
    m, (H, W) = _model(name, cin)
    k1 = 9 * cin
    npix1 = 2 * ((H + 1) // 2) * ((W + 1) // 2)
    for plan in (Plan(m, 2, H, W, False, torch.device("cpu")), _eval_grad_plan(m, H, W)):
        assert plan.stem_cols() == (k1, sld)
        col, cast, g = _stem(plan, m)
        assert (col["cin"], col["ldo"], col["H"], col["W"]) == (cin, sld, H, W)
        assert plan.bufs.named["stem.col16"].shape == (npix1, sld)
        assert cast[1:] == (k1, plan.bufs.named["stem.conv1.w16"].data_ptr(), sld, 16, k1, sld)
        assert (g.kc, g.lda, g.ldb, g.n, g.m, g.ntaps) == (sld, sld, sld, 16, npix1, 1)
        assert plan.op_flops[[i for i, op in enumerate(plan.ops) if op[2] == "fvit_gemm"][0]] == 2.0 * npix1 * 16 * k1
    # eval-grad backward: conv1 weight gradient of width 9 * cin, the image gradient as GEMM + col2im
    bwd = _gemms(plan.bwd_ops)
    col16, w1 = plan.bufs.named["stem.col16"].data_ptr(), plan.bufs.named["stem.conv1.w16"].data_ptr()
    wg = [x for x in bwd if x.b == col16]
    assert len(wg) == 1
    wg = wg[0]
    assert (wg.a_mn_major, wg.b_mn_major, wg.m, wg.n, wg.kc, wg.ldb, wg.ld_out_f32) == (1, 1, 16, k1, npix1, sld, k1)
    assert wg.out_f32 == plan.G(m.patch_embed.conv_down[0].weight)
    ldc = (k1 + 3) // 4 * 4
    dcol = plan.bufs.named["stem.dcol"]
    assert dcol.shape == (npix1, ldc) and dcol.dtype == torch.float32
    dg = [x for x in bwd if x.b == w1]
    assert len(dg) == 1
    dg = dg[0]
    assert (dg.a_mn_major, dg.b_mn_major, dg.m, dg.n, dg.kc, dg.b_rows, dg.ldb) == (0, 1, npix1, k1, 16, 16, sld)
    assert (dg.out_f32, dg.ld_out_f32, dg.alpha_ptr) == (dcol.data_ptr(), ldc, plan.scal.data_ptr() + 4)
    names = [op[2] for op in plan.bwd_ops]
    assert "fvit_stem_conv_dgrad" not in names and names.count("fvit_stem_col2im") == 1
    c2i = plan.bwd_ops[names.index("fvit_stem_col2im")][1]
    assert c2i == (dcol.data_ptr(), ldc, 2, cin, H, W, plan.dx.data_ptr())
    assert tuple(plan.dx.shape) == (2, cin, H, W)
    assert names.index("fvit_stem_col2im") > max(i for i, op in enumerate(plan.bwd_ops) if op[1] and op[2] == "fvit_gemm"
                                                 and op[1][0]._obj.b == w1)


@pytest.mark.parametrize("name", ["faster_vit_0_224", "faster_vit_0_any_res"])
def test_rgb_stem_launches_are_unchanged(name):
    """in_chans = 3 keeps the launches it had before other channel counts were supported: STEM_LD = 32 rows, a single
    32-deep K block, a 27-wide weight gradient and the fused image-gradient gather"""
    m, (H, W) = _model(name, 3)
    npix1 = 2 * ((H + 1) // 2) * ((W + 1) // 2)
    assert Plan.STEM_LD == 32
    from fastervit_b200.engine_train import TrainPlan
    plans = [Plan(m, 2, H, W, False, torch.device("cpu")), _eval_grad_plan(m, H, W),
             TrainPlan(m.train(), 2, H, W, torch.device("cpu"))]
    for plan in plans:
        col, cast, g = _stem(plan, m)
        assert (col["cin"], col["ldo"]) == (3, 32)
        assert cast[1:] == (27, plan.bufs.named["stem.conv1.w16"].data_ptr(), 32, 16, 27, 32)
        assert (g.kc, g.lda, g.ldb, g.n) == (32, 32, 32, 16)
        assert plan.op_flops[[i for i, op in enumerate(plan.ops) if op[2] == "fvit_gemm"][0]] == 2.0 * npix1 * 16 * 27
    for plan in plans[1:]:
        col16 = plan.bufs.named["stem.col16"].data_ptr()
        wg = [x for x in _gemms(plan.bwd_ops) if x.b == col16]
        assert len(wg) == 1 and (wg[0].n, wg[0].ld_out_f32, wg[0].ldb) == (27, 27, 32)
        assert wg[0].split_k == plan._split_k(16, 27, npix1)
        assert "stem.dcol" not in plan.bufs.named
        assert "fvit_stem_col2im" not in [op[2] for op in plan.bwd_ops]
    names = [op[2] for op in plans[1].bwd_ops]
    assert names.count("fvit_stem_conv_dgrad") == 1
    dz1 = plans[1].bufs.named["stem.dz1"].data_ptr()
    assert plans[1].bwd_ops[names.index("fvit_stem_conv_dgrad")][1][:5] == (dz1, 16, 2, H, W)
    assert "fvit_stem_conv_dgrad" not in [op[2] for op in plans[2].bwd_ops]


@pytest.mark.parametrize("cin", [0, 65])
def test_in_chans_outside_the_stem_kernels_raises_at_plan_build(cin):
    m, (H, W) = _model("faster_vit_0_224", cin)
    with pytest.raises(L.FvitError, match="1 <= in_chans <= 64"):
        Plan(m, 2, H, W, False, torch.device("cpu"))
    with pytest.raises(L.FvitError, match="1 <= in_chans <= 64"):
        _eval_grad_plan(m, H, W)
    from fastervit_b200.engine_train import TrainPlan
    with pytest.raises(L.FvitError, match="1 <= in_chans <= 64"):
        TrainPlan(m.train(), 2, H, W, torch.device("cpu"))


def test_in_chans_state_dict_matches_the_conv_weight():
    m, _ = _model("faster_vit_0_224", 4)
    assert tuple(m.state_dict()["patch_embed.conv_down.0.weight"].shape) == (16, 4, 3, 3)
    assert m.cfg["in_chans"] == 4
