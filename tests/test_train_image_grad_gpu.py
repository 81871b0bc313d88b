"""The image gradient of a train-mode step (FasterViT.enable_input_grad): model(x), forward_levels, forward_features, pooled features and
FasterViTBackbone under .train() with x.requires_grad, against fp64 autograd of the oracle with training=True (batch
statistics, leaf x). Bars as in the eval-mode tests: image gradient relative L2 <= 3e-2 (the fp16-operand floor,
measured 1.8e-2 .. 2.3e-2), parameter gradients median relative L2 <= 4e-3."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_dense_oracle.py
import _dense_oracle as DO  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"
DX_BAR = 3e-2
ANY_RES_KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8],
                  window_size=[7, 7, 5, 7])
ANY_RES_CFG = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7], ct_size=2,
                   mlp_ratio=4, resolution=[160, 224], hat=[False, False, True, False], do_propagation=False, any_res=True)


def _rel_l2(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return ((got - want).norm() / want.norm()).item()


def _setup(case, in_chans=None, drop_path_rate=0.0, **extra):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    kw = dict(g["kwargs"], **extra)
    if in_chans is not None:
        kw["in_chans"] = in_chans
    model = F.create_model(g["entry"], drop_path_rate=drop_path_rate, **kw)
    O.synth_fill_(model.state_dict(), g["seeds"]["w"])
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = O.synth_input(2, g["cfg"]["resolution"], g["seeds"]["x"] + 300, torch.float32)
    if in_chans is not None:
        gen = torch.Generator().manual_seed(in_chans)
        x = torch.randn((2, in_chans) + tuple(x.shape[2:]), generator=gen)
    return g, model.cuda().train().enable_input_grad(), sd, x


def _logit_grads(sd, cfg, x, target, drop_masks=None):
    """fp64 autograd of cross_entropy(oracle(x), target) under training=True: ({name: grad}, dx)"""
    from oracle import fastervit_oracle as O
    leaf = DO.leaves(sd)
    xl = x.double().clone().requires_grad_(True)
    logits = O.forward(leaf, cfg, xl, training=True, drop_masks=drop_masks)
    loss = torch.nn.functional.cross_entropy(logits, target)
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names] + [xl], allow_unused=True)
    return {k: g for k, g in zip(names, grads[:-1]) if g is not None}, grads[-1]


def _median_l2(model, ref):
    gmax = max(v.abs().max().item() for v in ref.values())
    l2s = []
    for k, p in model.named_parameters():
        if k in ref:
            assert p.grad is not None, k
            want = ref[k]
            l2s.append((p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5))
    return sorted(l2s)[len(l2s) // 2]


@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar", "tiny_21k224", "fv0"])
def test_logits_image_gradient_matches_fp64(case):
    g, model, sd, x = _setup(case)
    target = g["train"]["target"][:2]
    ref_g, ref_dx = _logit_grads(sd, g["cfg"], x, target)
    xg = x.cuda().requires_grad_(True)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    assert xg.grad.shape == xg.shape and xg.grad.dtype == torch.float32
    err, med = _rel_l2(xg.grad, ref_dx), _median_l2(model, ref_g)
    print(f"{case}: dx rel-L2 {err:.2e}, parameter median rel-L2 {med:.2e}")
    assert err <= DX_BAR and med <= 4e-3, (err, med)
    # the same step with x detached: the parameter gradients do not depend on asking for dx (train-mode statistics are
    # accumulated with atomics, so two runs of one plan already differ in the last bits; 1e-2 of a tensor's norm
    # is a bar on wiring mistakes, not on rounding)
    with_dx = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.load_state_dict(sd)
    model.zero_grad(set_to_none=True)
    torch.nn.functional.cross_entropy(model(x.cuda()), target.cuda()).backward()
    gmax = max(v.abs().max().item() for v in with_dx.values())
    for k, p in model.named_parameters():
        floor = 1e-3 * gmax * p.numel() ** 0.5
        assert (p.grad - with_dx[k]).norm().item() <= 1e-2 * max(with_dx[k].norm().item(), floor), k


@pytest.mark.parametrize("idx", [(0, 1, 2, 3), (1, 3), (0,)])
def test_forward_levels_image_gradient(idx):
    g, model, sd, x = _setup("tiny_ar")
    xg = x.cuda().requires_grad_(True)
    feats = model.forward_levels(xg, idx)
    gen = torch.Generator().manual_seed(5)
    w = {i: torch.randn(f.shape, generator=gen, dtype=torch.float64) for i, f in zip(idx, feats)}
    torch.autograd.backward(feats, [w[i].float().cuda() for i in idx])
    xl = x.double().clone().requires_grad_(True)
    fw = DO.dense_forward(DO.leaves(sd), g["cfg"], xl, stop_level=max(idx))
    sum((fw["levels"][i] * w[i]).sum() for i in idx).backward()
    assert _rel_l2(xg.grad, xl.grad) <= DX_BAR, _rel_l2(xg.grad, xl.grad)
    assert model.patch_embed.conv_down[0].weight.grad is not None


@pytest.mark.parametrize("final", ["norm", "pooled"])
def test_features_and_pooled_image_gradient(final):
    g, model, sd, x = _setup("tiny_a", **(dict(num_classes=0) if final == "pooled" else {}))
    xg = x.cuda().requires_grad_(True)
    out = model(xg) if final == "pooled" else model.forward_features(xg)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    (out * w.float().cuda()).sum().backward()
    xl = x.double().clone().requires_grad_(True)
    fw = DO.dense_forward(DO.leaves(sd), g["cfg"], xl, final=final)
    (fw[final] * w).sum().backward()
    assert _rel_l2(out, fw[final]) < 3e-3
    assert _rel_l2(xg.grad, xl.grad) <= DX_BAR, _rel_l2(xg.grad, xl.grad)


@pytest.mark.parametrize("fs", [-1, 0, 1, 2, 3])
def test_backbone_image_gradient_through_the_frozen_prefix(fs):
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=fs, drop_path_rate=0.0, **ANY_RES_KW)
    O.synth_fill_(bb.state_dict(), 11)
    sd = {k: v.detach().clone() for k, v in bb.state_dict().items()}
    x = O.synth_input(2, [160, 224], 3, torch.float32)
    bb = bb.cuda().train().enable_input_grad()
    frozen = (["patch_embed."] if fs >= 0 else []) + [f"levels.{i}." for i in range(max(fs - 1, 0))]
    before = {k: v.clone() for k, v in bb.state_dict().items()}
    xg = x.cuda().requires_grad_(True)
    outs = bb.forward_raw(xg)
    gen = torch.Generator().manual_seed(8)
    w = [torch.randn(o.shape, generator=gen, dtype=torch.float64) for o in outs]
    torch.autograd.backward(outs, [wi.float().cuda() for wi in w])
    body_sd = {k[len("body."):]: v for k, v in sd.items() if k.startswith("body.")}
    body_sd.update({k: v for k, v in sd.items() if not k.startswith("body.")})
    leaf = DO.leaves(body_sd, frozen)
    xl = x.double().clone().requires_grad_(True)
    fw = DO.dense_forward(leaf, ANY_RES_CFG, xl, stop_level=3, eval_bn_prefixes=frozen)
    loss = sum((O._bn(fw["levels"][i], leaf, f"norm{i}", 1e-5, True, None) * wi).sum() for i, wi in zip((1, 2, 3), w))
    names = [k for k, v in leaf.items() if torch.is_tensor(v) and v.requires_grad and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names] + [xl], allow_unused=True)
    assert _rel_l2(xg.grad, grads[-1]) <= DX_BAR, _rel_l2(xg.grad, grads[-1])
    ref = {k: gr for k, gr in zip(names, grads[:-1]) if gr is not None}
    named = [(k[len("body."):] if k.startswith("body.") else k, p) for k, p in bb.named_parameters()]
    l2s = []
    for k, p in named:
        if any(k.startswith(f) for f in frozen):
            assert p.grad is None, k
        elif k in ref:
            l2s.append(_rel_l2(p.grad, ref[k]))
    assert sorted(l2s)[len(l2s) // 2] <= 4e-3
    after = bb.state_dict()
    moved = 0
    for k, v in before.items():
        if not k.endswith(("running_mean", "running_var")):
            continue
        if any(k[len("body."):].startswith(f) for f in frozen):
            assert torch.equal(after[k], v), k     # the prefix's running statistics: bitwise unchanged
        elif k.startswith(("norm", "body.levels.")) and not k.startswith("body.levels.3.downsample"):
            moved += int(not torch.equal(after[k], v))
    assert moved >= 6      # the norm{i} (and every trained conv-level BatchNorm) were updated


@pytest.mark.parametrize("in_chans,channels_last", [(1, False), (4, False), (13, False), (3, True)])
def test_channel_counts_and_channels_last(in_chans, channels_last):
    g, model, sd, x = _setup("tiny_a", in_chans=None if in_chans == 3 else in_chans)
    target = g["train"]["target"][:2]
    _, ref_dx = _logit_grads(sd, dict(g["cfg"], in_chans=in_chans), x, target)
    xg = x.cuda()
    if channels_last:
        xg = xg.contiguous(memory_format=torch.channels_last)
    xg.requires_grad_(True)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    assert _rel_l2(xg.grad, ref_dx) <= DX_BAR, _rel_l2(xg.grad, ref_dx)


def test_drop_path_masks_reach_the_image_gradient():
    g, model, sd, x = _setup("tiny_a", drop_path_rate=0.3)
    target = g["train"]["target"][:2]
    xg = x.cuda().requires_grad_(True)
    model(xg)     # builds the plan
    plan = next(p for p in model._get_engine().plans.values() if p.training and p.want_dx)
    gen = torch.Generator().manual_seed(0)
    masks = {d["name"]: torch.bernoulli(torch.full((d["groups"],), d["keep"]), generator=gen) / d["keep"]
             for d in plan.drop_specs}
    assert any((m == 0).any() for m in masks.values())
    plan.forced_drop_masks = masks
    model.load_state_dict(sd)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    _, ref_dx = _logit_grads(sd, g["cfg"], x, target, drop_masks={k: v.double() for k, v in masks.items()})
    assert _rel_l2(xg.grad, ref_dx) <= DX_BAR, _rel_l2(xg.grad, ref_dx)


def test_guards_and_plan_reuse():
    from fastervit_b200.lib import FvitError
    g, model, sd, x = _setup("tiny_a")
    xg = x.cuda().requires_grad_(True)
    # the image gradient is asked for per model: without enable_input_grad() such an input raises as before
    model.enable_input_grad(False)
    for call in (model, model.forward_features, lambda t: model.forward_levels(t, (1, 3))):
        with pytest.raises(FvitError, match="enable_input_grad"):
            call(xg)
    assert not model._get_engine().plans      # (refused before anything was built)
    model.enable_input_grad()
    first = model(xg).sum()
    model(xg)
    with pytest.raises(FvitError, match="stale forward"):
        first.backward()
    out = model(xg).sum()
    (dx,) = torch.autograd.grad(out, xg, create_graph=True)
    with pytest.raises(RuntimeError):
        dx.sum().backward()
    with pytest.raises(FvitError, match="CUDA"):
        model(x.clone().requires_grad_(True))
    # a forward of the same shape without an input gradient runs a plan with no image-gradient launch
    model(x.cuda()).sum().backward()
    plans = [p for p in model._get_engine().plans.values() if p.training]
    assert len(plans) == 2
    plain = next(p for p in plans if not p.want_dx)
    names = {op[2] for op in plain.bwd_ops}
    assert not names & {"fvit_stem_conv_dgrad", "fvit_stem_col2im"} and not hasattr(plain, "dx")
    assert "fvit_stem_conv_dgrad" in {op[2] for op in next(p for p in plans if p.want_dx).bwd_ops}
