"""GPU tests of the dense-prediction outputs in training: forward_levels / forward_features / num_classes = 0 pooled
features / FasterViTBackbone under .train(), against fp64 autograd of the oracle (tests/_dense_oracle.py), and the
fvit_feature_map_bwd kernels against torch autograd of F.batch_norm(training=True).

Tolerances follow tests/test_train_gpu.py: outputs 3e-3 max-relative, parameter gradients relative L2 <= 4e-2
(6e-2 for patch_embed.*) with a median <= 4e-3, BatchNorm running statistics 1e-3."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_dense_oracle.py
import _dense_oracle as DO  # noqa: E402

pytestmark = pytest.mark.gpu

ANY_RES_KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8],
                  window_size=[7, 7, 5, 7])
ANY_RES_CFG = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7], ct_size=2,
                   mlp_ratio=4, resolution=[160, 224], hat=[False, False, True, False], do_propagation=False, any_res=True)


def _model(case, **extra):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES, cfg_of
    entry, kw, _ = CASES[case]
    model = F.create_model(entry, drop_path_rate=0.0, **kw, **extra)
    O.synth_fill_(model.state_dict(), 1234)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    res = cfg_of(case)["resolution"]
    x = O.synth_input(2, res, 56, torch.float32)
    return model.cuda().train(), sd, cfg_of(case), x


def _weights(shapes: dict, seed: int = 3) -> dict:
    """fixed random output-gradient weights, one decade of scale apart per level (1e3 between the extremes)"""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(s, generator=g, dtype=torch.float64) * 10.0 ** (n % 4) for n, (k, s) in enumerate(shapes.items())}


def _rel(a, b) -> float:
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


def _check_grads(named, ref: dict, prefix: str = "") -> None:
    gmax = max(v.abs().max().item() for v in ref.values())
    bad, l2s = [], []
    for k, p in named:
        want = ref.get(prefix + k)
        if want is None:
            continue
        assert p.grad is not None, k
        err = (p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5)
        l2s.append(err)
        if err > (6e-2 if (prefix + k).startswith("patch_embed.") else 4e-2):
            bad.append((k, err))
    assert l2s and not bad, bad[:10]
    med = sorted(l2s)[len(l2s) // 2]
    assert med <= 4e-3, med


# ------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("bn", [True, False])
def test_feature_map_bwd_kernel_matches_autograd(bn):
    from fastervit_b200 import lib as L
    torch.manual_seed(0)
    B, H, W, C, extra = 3, 5, 9, 40, 23          # T = 45 and C = 40: neither a multiple of 32
    T = H * W
    nrows = B * T + extra
    xs = torch.randn(nrows, C, device="cuda") * 1.5 + 0.3
    row_map = torch.randperm(nrows, device="cuda")[:B * T].to(torch.int32)   # the other rows play padding / carriers
    xmap = xs[row_map.long()].view(B, H, W, C).permute(0, 3, 1, 2).contiguous()
    w = torch.rand(C, device="cuda") + 0.5
    beta = torch.randn(C, device="cuda") * 0.1
    dy = torch.randn(B, C, H, W, device="cuda")
    g0 = torch.randn(nrows + 1, C, device="cuda")
    g = g0.clone()
    S = 4.0
    gs = torch.tensor([S, 1 / S], device="cuda")
    acc = torch.zeros(1 + 2 * C, device="cuda")
    amax, s1, s2 = acc[0:1], acc[1:1 + C], acc[1 + C:]
    dw0, db0 = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    dw, db = dw0.clone(), dw0.clone() * 0 + db0
    if bn:
        mean = xmap.mean(dim=(0, 2, 3))
        rstd = torch.rsqrt(xmap.var(dim=(0, 2, 3), unbiased=False) + 1e-5)
        L.call("fvit_feature_map_bwd_stats", dy.data_ptr(), xs.data_ptr(), C, row_map.data_ptr(), B, T, C,
               mean.data_ptr(), rstd.data_ptr(), s1.data_ptr(), s2.data_ptr(), amax.data_ptr())
        L.call("fvit_feature_map_bwd", dy.data_ptr(), xs.data_ptr(), C, row_map.data_ptr(), B, T, C, mean.data_ptr(),
               rstd.data_ptr(), w.data_ptr(), s1.data_ptr(), s2.data_ptr(), gs.data_ptr(), None, g.data_ptr(), C,
               dw.data_ptr(), db.data_ptr())
        xr = xmap.double().requires_grad_(True)
        wr, br = w.double().requires_grad_(True), beta.double().requires_grad_(True)
        y = torch.nn.functional.batch_norm(xr, None, None, wr, br, training=True, eps=1e-5)
        y.backward(dy.double())
        dx, dwr, dbr = xr.grad, wr.grad, br.grad
        assert (dw.double() - dw0.double() - dwr).abs().max().item() <= 1e-4 * dwr.abs().max().item()
        assert (db.double() - db0.double() - dbr).abs().max().item() <= 1e-4 * dbr.abs().max().item()
    else:
        L.call("fvit_feature_map_bwd_stats", dy.data_ptr(), None, C, row_map.data_ptr(), B, T, C, None, None, None, None,
               amax.data_ptr())
        L.call("fvit_feature_map_bwd", dy.data_ptr(), None, C, row_map.data_ptr(), B, T, C, None, None, None, None, None,
               gs.data_ptr(), None, g.data_ptr(), C, None, None)
        dx = dy.double()
    torch.cuda.synchronize()
    assert amax.item() == dy.abs().max().item()
    want = g0.double().clone()
    want[row_map.long()] += S * dx.permute(0, 2, 3, 1).reshape(B * T, C)
    got = g.double()
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    untouched = torch.ones(nrows + 1, dtype=torch.bool, device="cuda")
    untouched[row_map.long()] = False
    assert torch.equal(g[untouched], g0[untouched])     # padding / carrier / zero rows bitwise as they were


def test_gradient_scale_over_several_outputs():
    """S = 2^floor(log2(64 / max)) over the |dy| maxima of every output (one stats pass each, one finalize)."""
    from fastervit_b200 import lib as L
    torch.manual_seed(1)
    amax = torch.zeros(1, device="cuda")
    maxima = []
    for B, C, T, scale in ((2, 33, 70, 1e-3), (2, 64, 17, 2.5), (2, 8, 5, 0.1)):
        dy = torch.randn(B, C, T, device="cuda") * scale
        maxima.append(dy.abs().max().item())
        L.call("fvit_feature_map_bwd_stats", dy.data_ptr(), None, C, None, B, T, C, None, None, None, None, amax.data_ptr())
    gs = torch.zeros(2, device="cuda")
    L.call("fvit_grad_scale_finalize", amax.data_ptr(), 64.0, gs.data_ptr())
    torch.cuda.synchronize()
    m = max(maxima)
    assert amax.item() == m
    S = 2.0 ** torch.floor(torch.log2(torch.tensor(64.0 / m))).item()
    assert gs[0].item() == S and gs[1].item() == 1.0 / S


# ------------------------------------------------------------------------------------------------------- forward_levels
@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar"])
@pytest.mark.parametrize("idx", [(0, 1, 2, 3), (1, 2, 3), (2,), (0, 1), (0,)])   # (0, 1) / (0,): a conv top level
def test_forward_levels_train_matches_oracle(case, idx):
    model, sd, cfg, x = _model(case)
    feats = model.forward_levels(x.cuda(), idx)
    assert all(f.grad_fn is not None for f in feats)
    w = _weights({i: tuple(f.shape) for i, f in zip(idx, feats)})
    torch.autograd.backward(feats, [w[i].float().cuda() for i in idx])
    ref_out, ref_g, _ = DO.levels_loss_and_grads(sd, cfg, x, w)
    for i, f in zip(idx, feats):
        assert tuple(f.shape) == tuple(ref_out[i].shape)
        assert _rel(f, ref_out[i]) < 3e-3, (i, _rel(f, ref_out[i]))
    top = max(idx)
    for k, p in model.named_parameters():
        off = (k.startswith(("norm.", "head.")) or (k.startswith("levels.") and int(k.split(".")[1]) > top)
               or k.startswith(f"levels.{top}.downsample."))
        if off:
            assert p.grad is None, k
        else:
            assert k in ref_g, k
    _check_grads(model.named_parameters(), ref_g)


def test_forward_features_train_matches_oracle():
    model, sd, cfg, x = _model("tiny_a")
    rm0, rv0 = model.norm.running_mean.clone(), model.norm.running_var.clone()
    f = model.forward_features(x.cuda())
    w = _weights({"norm": tuple(f.shape)})
    (f * w["norm"].float().cuda()).sum().backward()
    ref_out, ref_g, stats = DO.levels_loss_and_grads(sd, cfg, x, w, final="norm")
    assert _rel(f, ref_out["norm"]) < 3e-3
    assert model.norm.weight.grad is not None and model.norm.bias.grad is not None
    assert model.head.weight.grad is None
    _check_grads(model.named_parameters(), ref_g)
    mean, var = stats["norm"]
    m = model.norm.momentum
    for got, want in ((model.norm.running_mean, (1 - m) * rm0.double().cpu() + m * mean),
                      (model.norm.running_var, (1 - m) * rv0.double().cpu() + m * var)):
        assert (got.double().cpu() - want).abs().max().item() <= 1e-3 * want.abs().max().item()


def test_pooled_features_train_num_classes_0():
    model, sd, cfg, x = _model("tiny_a", num_classes=0)
    out = model(x.cuda())
    assert out.shape == (2, model.num_features) and out.grad_fn is not None
    w = _weights({"pooled": tuple(out.shape)})
    (out * w["pooled"].float().cuda()).sum().backward()
    ref_out, ref_g, _ = DO.levels_loss_and_grads(sd, cfg, x, w, final="pooled")
    assert _rel(out, ref_out["pooled"]) < 3e-3
    _check_grads(model.named_parameters(), ref_g)


# ------------------------------------------------------------------------------------------------------- backbone
def _backbone(fs):
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=fs, drop_path_rate=0.0,
                           **ANY_RES_KW)
    O.synth_fill_(bb.state_dict(), 11)
    sd = {k: v.detach().clone() for k, v in bb.state_dict().items()}
    x = O.synth_input(2, [160, 224], 3, torch.float32)
    return bb.cuda().train(), sd, x


@pytest.mark.parametrize("fs", [-1, 1, 2])
def test_backbone_train_matches_oracle(fs):
    bb, sd, x = _backbone(fs)
    frozen = (["patch_embed."] if fs >= 0 else []) + [f"levels.{i}." for i in range(max(fs - 1, 0))]
    before = {k: v.clone() for k, v in bb.state_dict().items()}
    outs = bb.forward_raw(x.cuda())
    w = _weights({i: tuple(o.shape) for i, o in zip((1, 2, 3), outs)}, seed=8)
    torch.autograd.backward(outs, [w[i].float().cuda() for i in (1, 2, 3)])
    body_sd = {k[len("body."):]: v for k, v in sd.items() if k.startswith("body.")}
    body_sd.update({k: v for k, v in sd.items() if not k.startswith("body.")})
    ref_out, ref_g, _ = DO.levels_loss_and_grads(body_sd, ANY_RES_CFG, x, w, level_norms={i: f"norm{i}" for i in (1, 2, 3)},
                                                 frozen_prefixes=frozen)
    # outputs and norm{i} running statistics against torch BatchNorm2d (train mode) on the oracle's level maps
    with torch.no_grad():
        maps = DO.dense_forward(DO.leaves(body_sd), ANY_RES_CFG, x.double(), stop_level=3, eval_bn_prefixes=frozen)
    for i, o in zip((1, 2, 3), outs):
        tbn = torch.nn.BatchNorm2d(o.shape[1]).double()
        tbn.load_state_dict({k[len(f"norm{i}."):]: v for k, v in sd.items() if k.startswith(f"norm{i}.")})
        want = tbn.train()(maps["levels"][i].detach())
        assert _rel(o, want) < 3e-3, (i, _rel(o, want))
        assert _rel(o, ref_out[i]) < 3e-3
        bn = getattr(bb, f"norm{i}")
        for got, ref in ((bn.running_mean, tbn.running_mean), (bn.running_var, tbn.running_var)):
            assert (got.double().cpu() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item(), i
        assert bn.num_batches_tracked.item() == 1
    named = [(k[len("body."):] if k.startswith("body.") else k, p) for k, p in bb.named_parameters()]
    for k, p in named:
        if any(k.startswith(f) for f in frozen):
            assert p.grad is None, k
    _check_grads(named, ref_g)
    after = bb.state_dict()
    for k, v in before.items():
        body_k = k[len("body."):]
        if any(body_k.startswith(f) for f in frozen) and k.endswith(("running_mean", "running_var", "num_batches_tracked")):
            assert torch.equal(after[k], v), k     # frozen BatchNorms: running statistics bitwise unchanged


def test_backbone_frozen_plan_is_shorter_and_buckets_tile():
    lens = {}
    for fs in (-1, 2):
        bb, sd, x = _backbone(fs)
        outs = bb.forward_raw(x.cuda())
        sum(o.sum() for o in outs).backward()
        plan = next(p for p in bb.body._get_engine().plans.values() if p.training)
        lens[fs] = len(plan.bwd_ops)
        total = plan.gflat.numel()
        covered = sorted(plan.grad_buckets)
        assert covered[0][0] == 0 and covered[-1][1] == total
        assert all(a[1] == b[0] for a, b in zip(covered, covered[1:]))
        for i in (1, 2, 3):          # the norm{i} slices sit inside the buckets
            bn = getattr(bb, f"norm{i}")
            for p in (bn.weight, bn.bias):
                o = plan._goff[id(p)]
                assert sum(1 for lo, hi in plan.grad_buckets if lo <= o and o + p.numel() <= hi) == 1
    assert lens[2] < lens[-1], lens


# ------------------------------------------------------------------------------------------------------- execution rules
def test_graph_replays_read_each_steps_gradients():
    """Five steps with a fixed input: the third and later backward calls replay CUDA graphs; scaling the injected
    gradients by 2 must scale every parameter gradient by 2 (to the atomics noise of the train-step test)."""
    model, sd, cfg, x = _model("tiny_a")
    x = x.cuda()
    idx = (0, 1, 2, 3)
    w = None
    base = None
    for step, c in enumerate((1.0, 2.0, 1.0, 2.0, 2.0)):
        feats = model.forward_levels(x, idx)
        if w is None:
            w = [torch.randn(f.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(i)) for i, f in enumerate(feats)]
        torch.autograd.backward(feats, [c * wi for wi in w])
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        model.zero_grad(set_to_none=True)
        if base is None:
            base = grads
            gmax = max(v.abs().max().item() for v in base.values())
            continue
        for k, g in grads.items():
            ref = c * base[k]
            tol = 2e-2 * max(ref.abs().max().item(), 1e-2 * gmax * c)
            assert (g - ref).abs().max().item() <= tol, (step, k)


def test_stale_forward_and_input_grad_raise_on_levels_plan():
    from fastervit_b200.lib import FvitError
    model, sd, cfg, x = _model("tiny_a")
    x = x.cuda()
    f1 = model.forward_levels(x, (2, 3))
    f2 = model.forward_levels(x * 0.5, (2, 3))
    with pytest.raises(FvitError):
        sum(f.sum() for f in f1).backward()
    sum(f.sum() for f in f2).backward()
    with pytest.raises(FvitError):
        model.forward_levels(x.clone().requires_grad_(True), (2, 3))
    # only one output of two used: the other's gradient counts as zeros
    model.zero_grad(set_to_none=True)
    f3 = model.forward_levels(x, (2, 3))
    f3[0].sum().backward()
    assert model.levels[2].blocks[0].mlp.fc1.weight.grad is not None
    assert model.levels[3].blocks[0].mlp.fc1.weight.grad.abs().max().item() == 0.0


def test_backbone_frozen_prefix_is_deterministic_under_stochastic_depth():
    """frozen_stages=2 with drop_path_rate > 0: the frozen level-0 blocks draw no stochastic-depth masks (the reference
    eval()s them), so level 1's input is the same from step to step while level 1 itself still drops branches"""
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    kw = dict(ANY_RES_KW, depths=[2, 2, 2, 1])
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(0, 1), frozen_stages=2, drop_path_rate=0.5, **kw)
    O.synth_fill_(bb.state_dict(), 5)
    bb = bb.cuda().train()
    x = O.synth_input(2, [160, 224], 3, torch.float32).cuda()
    torch.manual_seed(0)   # (the masks come from torch's CUDA generator: a fixed draw sequence)
    outs = [bb.forward_raw(x) for _ in range(5)]
    plan = next(p for p in bb.body._get_engine().plans.values() if p.training)
    names = [d["name"] for d in plan.drop_specs]
    assert names and not any(n.startswith("levels.0.") for n in names), names
    # level 0 (frozen, running-statistics BatchNorms, no DropPath) is deterministic; its norm0 runs on batch statistics
    # of identical maps, so the output repeats to the atomics noise of the statistics
    for o in outs[1:]:
        assert _rel(o[0], outs[0][0]) < 1e-5
    assert max(_rel(o[1], outs[0][1]) for o in outs[1:]) > 1e-2     # level 1 trains with its masks


def test_reallocated_level_norm_rebuilds_the_plan():
    """the backbone's norm{i} tensors are read through raw pointers: replacing one (.data = ...) builds a new plan
    instead of reading freed memory"""
    bb, sd, x = _backbone(-1)
    x = x.cuda()
    o1 = bb.forward_raw(x)
    eng = bb.body._get_engine()
    p1 = next(p for p in eng.plans.values() if p.training)
    bn = bb.norm2
    bn.weight.data = bn.weight.data.clone() * 2
    bn.bias.data = bn.bias.data.clone()
    o2 = bb.forward_raw(x)
    p2 = next(p for p in eng.plans.values() if p.training)
    assert p2 is not p1 and len([p for p in eng.plans.values() if p.training]) == 1
    assert p2.G(bn.weight) != 0 and bn.weight.data_ptr() in p2._norm_sig
    # norm2's output is affine in its weight: (o2 - bias) = 2 (o1 - bias)
    b = bn.bias.detach().view(1, -1, 1, 1)
    assert _rel(o2[1] - b, 2 * (o1[1] - b)) < 3e-3
    sum(o.sum() for o in o2).backward()
    assert bn.weight.grad is not None
