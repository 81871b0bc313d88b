"""Data-only backward stages on the device: the eval-mode input gradient with frozen parameters against the full
backward of the same build and the fp64 oracle, mixed masks, the backbone's frozen prefix, and the new kernels against
fp64 torch. The data-only path still adds dQ partials (key-loop attention) and carrier-row gradients
(fvit_propagate_bwd) with fp32 atomics, so two runs agree to rounding, not bitwise: determinism is tested to 1e-5."""
from pathlib import Path

import pytest
import torch

from test_eval_grad_gpu import _oracle_grads, _rel_l2, _setup

pytestmark = pytest.mark.gpu
DX_BAR = 3e-2


def _lib():
    from fastervit_b200 import lib as L
    L.load()
    return L


def _names(plan):
    return [op[2] for op in plan.bwd_ops]


def _wgrads(plan):
    return sum(1 for op in plan.bwd_ops if op[2] == "fvit_gemm" and op[1][0]._obj.a_mn_major and op[1][0]._obj.b_mn_major)


def _dx(model, x, target):
    xg = x.cuda().requires_grad_(True)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    return xg.grad


@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar148", "fv0"])
def test_frozen_parameters_input_gradient(case):
    L = _lib()
    g, model, sd, x = _setup(case)
    target = g["train"]["target"]
    L.reset_launch_count()
    full = _dx(model, x, target)
    torch.cuda.synchronize()
    n_full = L.launch_count()
    model.zero_grad(set_to_none=True)
    for p in model.parameters():
        p.requires_grad_(False)
    L.reset_launch_count()
    got = _dx(model, x, target)
    torch.cuda.synchronize()
    n_do = L.launch_count()
    again = _dx(model, x, target)
    assert all(p.grad is None for p in model.parameters())
    assert _rel_l2(got.double(), full.double(), 0.0) <= 1e-3
    assert _rel_l2(again.double(), got.double(), 0.0) <= 1e-5
    _, _, ref_dx = _oracle_grads(sd, g["cfg"], x, target)
    assert _rel_l2(got.double().cpu(), ref_dx, 0.0) <= DX_BAR
    plans = model._get_engine().eval_grad_plans()
    do = next(p for p in plans if all(p.data_only))
    fullp = next(p for p in plans if not any(p.data_only))
    banned = {"fvit_cpb_mlp_bwd", "fvit_attn_bias_bwd", "fvit_bn_eval_bwd", "fvit_ln_bwd", "fvit_branch_grad",
              "fvit_unpack_conv_grad", "fvit_token_init_bwd", "fvit_group_sum"}
    assert not banned & set(_names(do))
    # what is left belongs to the head, which is no stage: its Linear's weight gradient and bias column sum
    assert _wgrads(do) == 1 and _names(do).count("fvit_colsum") == 1 and _wgrads(fullp) > 20
    assert n_do < n_full, (n_do, n_full)


def test_mixed_mask_last_level_and_head():
    g, model, sd, x = _setup("tiny_a")
    target = g["train"]["target"]
    full_dx = _dx(model, x, target)
    full = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    keep = ("levels.3.", "head.")
    for k, p in model.named_parameters():
        p.requires_grad_(k.startswith(keep))
    got_dx = _dx(model, x, target)
    assert _rel_l2(got_dx.double(), full_dx.double(), 0.0) <= 1e-3
    for k, p in model.named_parameters():
        if k.startswith(keep):
            assert _rel_l2(p.grad.double(), full[k].double(), 1e-12) <= 2e-3, k
        else:
            assert p.grad is None, k
    plan = next(p for p in model._get_engine().eval_grad_plans() if any(p.data_only))
    assert plan.data_only == (True, True, True, True, False)


def test_eval_backbone_frozen_prefix_is_data_only():
    import sys
    sys.path.insert(0, str(Path(__file__).resolve().parent))
    import _dense_oracle as DO
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    from test_train_image_grad_gpu import ANY_RES_CFG, ANY_RES_KW
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=2, **ANY_RES_KW)
    O.synth_fill_(bb.state_dict(), 11)
    sd = {k: v.detach().clone() for k, v in bb.state_dict().items()}
    x = O.synth_input(2, [160, 224], 3, torch.float32)
    bb = bb.cuda().eval()
    xg = x.cuda().requires_grad_(True)
    outs = bb.forward_raw(xg)
    gen = torch.Generator().manual_seed(8)
    w = [torch.randn(o.shape, generator=gen, dtype=torch.float64) for o in outs]
    torch.autograd.backward(outs, [wi.float().cuda() for wi in w])
    frozen = ["patch_embed.", "levels.0."]
    body_sd = {k[len("body."):]: v for k, v in sd.items() if k.startswith("body.")}
    body_sd.update({k: v for k, v in sd.items() if not k.startswith("body.")})
    leaf = DO.leaves(body_sd, frozen)
    xl = x.double().clone().requires_grad_(True)
    fw = DO.dense_forward(leaf, ANY_RES_CFG, xl, stop_level=3, training=False)
    loss = sum((O._bn(fw["levels"][i], leaf, f"norm{i}", 1e-5, False, None) * wi).sum() for i, wi in zip((1, 2, 3), w))
    names = [k for k, v in leaf.items() if torch.is_tensor(v) and v.requires_grad and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names] + [xl], allow_unused=True)
    assert _rel_l2(xg.grad.double().cpu(), grads[-1], 0.0) <= DX_BAR
    ref = {k: gr for k, gr in zip(names, grads[:-1]) if gr is not None}
    l2s = []
    for k, p in bb.named_parameters():
        k = k[len("body."):] if k.startswith("body.") else k
        if k.startswith(tuple(frozen)):
            assert p.grad is None, k
        elif k in ref:
            l2s.append(_rel_l2(p.grad.double().cpu(), ref[k], 1e-12))
    assert l2s and sorted(l2s)[len(l2s) // 2] <= 4e-3
    plan = next(p for p in bb.body._get_engine().eval_grad_plans())
    assert plan.data_only == (True, True, False, False, False) and plan.want_dx
    assert _names(plan).count("fvit_bn_eval_dgrad") == 2 + 2 and "fvit_bn_eval_bwd" in _names(plan)


# ---------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("C,ld,g16,act,colmul", [(196, 200, True, 1, False), (196, 200, False, 0, True), (64, 64, True, 0, False),
                                                 (64, 64, False, 1, True), (30, 30, True, 1, True), (30, 30, False, 0, False)])
def test_bn_eval_dgrad_matches_fp64(C, ld, g16, act, colmul):
    """C = 196 (fv4's level 0: a 4-channel tail vector), C = 30 (the element-wise kernel), -1 entries in every row map"""
    L = _lib()
    torch.manual_seed(C + act)
    nrows, total = 300, 420
    raw = torch.zeros(total, ld, dtype=torch.float16)
    raw[:, :C] = torch.randn(total, C).half()
    gin = torch.randn(total, ld, dtype=torch.float64)
    g_rows, r_rows, o_rows = (torch.randperm(total)[:nrows] for _ in range(3))
    skip = torch.zeros(nrows, dtype=torch.bool)
    skip[::7] = True
    scale, shift = torch.randn(C, dtype=torch.float64), torch.randn(C, dtype=torch.float64) * 0.3
    pre = raw.double()[r_rows, :C] * scale.float().double() + shift.float().double()
    gin[g_rows[:, None], torch.arange(C)] *= (pre.abs() > 1e-3)       # (no gradient where fp32 / fp64 may disagree on the sign)
    cm = torch.rand(C, dtype=torch.float64) + 0.5 if colmul else None
    scalar = 0.25
    gin_dev = (gin.half() if g16 else gin.float()).cuda()
    want = gin_dev.double().cpu()[g_rows, :C] * scale.float().double() * scalar * (cm.float().double() if colmul else 1.0)
    if act == 1:
        want = want * (pre > 0)
    out = torch.full((total, ld), 7.0, dtype=torch.float16, device="cuda")
    dev = lambda t: t.float().cuda()
    keep = [dev(scale), dev(shift), dev(cm) if colmul else None, torch.tensor([scalar], device="cuda"), raw.cuda()]
    gr = torch.where(skip, -1, g_rows).int().cuda()
    rr, orr = r_rows.int().cuda(), torch.where(skip, -1, o_rows).int().cuda()
    L.call("fvit_bn_eval_dgrad", gin_dev.data_ptr(), int(g16), ld, gr.data_ptr(), keep[4].data_ptr(), ld, rr.data_ptr(), nrows,
           C, keep[0].data_ptr(), keep[1].data_ptr(), act, L.ptr(keep[2]), keep[3].data_ptr(), out.data_ptr(), ld, orr.data_ptr())
    torch.cuda.synchronize()
    got = out.double().cpu()
    live = ~skip
    err = (got[o_rows[live], :C] - want[live]).abs().max().item() / want.abs().max().item()
    assert err < 2e-3, err
    untouched = torch.ones(total, dtype=torch.bool)
    untouched[o_rows[live]] = False
    assert (got[untouched] == 7.0).all()
    if C % 4 == 0 and ld > C:
        assert (got[o_rows[live], C:] == 0).all()       # padding columns of a written row are zeroed


@pytest.mark.parametrize("C", [196, 392, 40])
@pytest.mark.parametrize("routed", [False, True])
def test_ln_dgrad_equals_the_dx_of_ln_bwd(C, routed):
    """the same g as fvit_ln_bwd, bitwise on the vectorised path (one kernel) and to rounding on the generic one; dy_map
    with -1 rows; in_map + clear_moved as the carrier-token rows use them"""
    L = _lib()
    torch.manual_seed(C)
    rows, extra = 200, 40
    dy = torch.randn(rows, C, device="cuda").half()
    xh = torch.randn(rows, C, device="cuda").half()
    rstd = torch.rand(rows, device="cuda") + 0.5
    gamma = torch.randn(C, device="cuda")
    dy_map = torch.randperm(rows, device="cuda").int()
    dy_map[::9] = -1
    g0 = torch.randn(rows + extra, C, device="cuda")
    in_map = None
    if routed:
        in_map = torch.arange(rows, device="cuda").int()
        in_map[:extra] = torch.arange(rows, rows + extra, device="cuda").int()   # the first rows move to the tail
    one = torch.ones(1, device="cuda")
    ga, gb = g0.clone(), g0.clone()
    dgam, dbet = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    args = (dy.data_ptr(), C, dy_map.data_ptr(), xh.data_ptr(), C, rstd.data_ptr(), gamma.data_ptr(), rows, C)
    tail = (C, L.ptr(in_map), 1, int(routed))
    L.call("fvit_ln_bwd", *args, ga.data_ptr(), *tail, one.data_ptr(), dgam.data_ptr(), dbet.data_ptr())
    L.call("fvit_ln_dgrad", *args, gb.data_ptr(), *tail)
    torch.cuda.synchronize()
    if C % 8 == 0:
        assert torch.equal(ga, gb)
    else:
        assert (ga - gb).abs().max().item() <= 1e-5 * ga.abs().max().item()
    d = dy.double() * gamma.double()
    want = rstd.double()[:, None] * (d - d.mean(1, keepdim=True) - xh.double() * (d * xh.double()).mean(1, keepdim=True))
    ref = g0.double().clone()
    src = dy_map.long()
    live = src >= 0
    upd = torch.zeros(rows, C, dtype=torch.float64, device="cuda")
    dq = dy.double()[src.clamp(min=0)] * gamma.double()
    upd = rstd.double()[:, None] * (dq - dq.mean(1, keepdim=True) - xh.double() * (dq * xh.double()).mean(1, keepdim=True))
    dst = in_map.long() if routed else torch.arange(rows, device="cuda")
    r = torch.arange(rows, device="cuda")[live]
    vals = g0.double()[r] + upd[r]
    if routed:
        moved = r[dst[r] != r]
        ref[moved] = 0.0
    ref[dst[r]] = vals
    assert (gb.double() - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


def test_token_init_dgrad_equals_the_gx_of_token_init_bwd():
    L = _lib()
    torch.manual_seed(0)
    B, Hp, Wp, C, oh, ow = 2, 14, 14, 40, 2, 2
    kh = kw = sh = sw = 7
    npix = B * Hp * Wp
    pix_map = torch.randperm(npix + 8, device="cuda")[:npix].int()
    ct_rows = torch.arange(npix + 8, npix + 8 + B * oh * ow, device="cuda").int()
    g0 = torch.randn(npix + 8 + B * oh * ow, C, device="cuda")
    x16 = torch.randn(npix + 8, C, device="cuda").half()
    w = torch.randn(C, 9, device="cuda")
    one = torch.ones(1, device="cuda")
    ga, gb = g0.clone(), g0.clone()
    dw, db = torch.zeros(C, 9, device="cuda"), torch.zeros(C, device="cuda")
    L.call("fvit_token_init_bwd", ga.data_ptr(), C, x16.data_ptr(), C, pix_map.data_ptr(), ct_rows.data_ptr(), B, Hp, Wp, C,
           w.data_ptr(), kh, kw, sh, sw, oh, ow, one.data_ptr(), ga.data_ptr(), C, dw.data_ptr(), db.data_ptr())
    L.call("fvit_token_init_dgrad", gb.data_ptr(), C, pix_map.data_ptr(), ct_rows.data_ptr(), B, Hp, Wp, C, w.data_ptr(), kh,
           kw, sh, sw, oh, ow, gb.data_ptr(), C)
    torch.cuda.synchronize()
    assert torch.equal(ga, gb) and not torch.equal(gb, g0)
