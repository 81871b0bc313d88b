"""Gradients of the dense-prediction outputs under .eval(): forward_levels, forward_features, forward_head and
FasterViTBackbone, against fp64 autograd of the oracle with training=False (tests/_dense_oracle.dense_forward, leaf
parameters, leaf x, level norms through oracle._bn on running statistics); the two eval backward kernels against fp64
torch; and the invariants and guards of the autograd node.

Bars as in tests/test_eval_grad_gpu.py: per tensor max element error 8e-2 and relative L2 4e-2 (6e-2 for the stem),
median parameter relative L2 1.5e-3, image-gradient relative L2 3e-2. Measured on an H100 80GB HBM3: median parameter
relative L2 2.8e-4 .. 9.2e-4, image gradient 1.8e-2 .. 2.5e-2 over every case below."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_dense_oracle.py
import _dense_oracle as DO  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"
EVAL_MEDIAN_BAR = 1.5e-3
DX_BAR = 3e-2


def _lib():
    from fastervit_b200 import lib as L
    L.load()
    return L


def _rel_l2(got, want, floor):
    return (got - want).norm().item() / max(want.norm().item(), floor * want.numel() ** 0.5)


# ---------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("bn", [True, False])
def test_feature_map_eval_bwd_matches_fp64(bn):
    """a cropped any-res map (5 x 9 pixels of 8 x 14 padded windows), C = 40 (not a multiple of 32); rows outside the
    map keep their sentinel; dw / dbeta from the stats pass on running statistics"""
    L = _lib()
    torch.manual_seed(5)
    B, Hm, Wm, Hc, Wc, C = 3, 8, 14, 5, 9, 40
    T = Hc * Wc
    rows_total = B * Hm * Wm + 7
    bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(Hc), torch.arange(Wc), indexing="ij")
    rmap = (bi * Hm * Wm + yi * Wm + xi).reshape(-1)
    xs = torch.randn(rows_total, C, dtype=torch.float64) * 2 + 30.0
    mean = (xs[rmap].mean(0) + 0.2 * torch.randn(C, dtype=torch.float64)).float()
    var = (xs[rmap].var(0) * (1 + 0.2 * torch.rand(C, dtype=torch.float64))).float()
    eps = 1e-5
    rstd = torch.rsqrt(var + eps)
    w = torch.randn(C) * 0.7
    dy = torch.randn(B, C, Hc, Wc)
    S = 8.0
    g0 = torch.randn(rows_total, C)
    dw0, db0 = torch.randn(C), torch.randn(C)
    dev = lambda t: t.contiguous().cuda()
    d_xs, d_rmap, d_mean, d_rstd, d_w, d_dy = dev(xs.float()), dev(rmap.int()), dev(mean), dev(rstd), dev(w), dev(dy)
    g, dw, db = dev(g0.clone()), dev(dw0.clone()), dev(db0.clone())
    acc = torch.zeros(1 + 2 * C, device="cuda")
    amax, s1, s2 = acc[0:1], acc[1:1 + C], acc[1 + C:]
    gs = torch.tensor([S, 1 / S], device="cuda")
    if bn:
        L.call("fvit_feature_map_bwd_stats", d_dy.data_ptr(), d_xs.data_ptr(), C, d_rmap.data_ptr(), B, T, C,
               d_mean.data_ptr(), d_rstd.data_ptr(), s1.data_ptr(), s2.data_ptr(), amax.data_ptr())
        L.call("fvit_feature_map_eval_bwd", d_dy.data_ptr(), d_rmap.data_ptr(), B, T, C, d_rstd.data_ptr(), d_w.data_ptr(),
               s1.data_ptr(), s2.data_ptr(), gs.data_ptr(), None, g.data_ptr(), C, dw.data_ptr(), db.data_ptr())
    else:
        L.call("fvit_feature_map_eval_bwd", d_dy.data_ptr(), d_rmap.data_ptr(), B, T, C, None, None, None, None,
               gs.data_ptr(), None, g.data_ptr(), C, None, None)
    torch.cuda.synchronize()
    dy_rows = dy.double().permute(0, 2, 3, 1).reshape(B * T, C)
    k = S * (w.double() * rstd.double() if bn else torch.ones(C, dtype=torch.float64))
    want = g0.double().clone()
    want[rmap] += k * dy_rows
    got = g.double().cpu()
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    untouched = torch.ones(rows_total, dtype=torch.bool)
    untouched[rmap] = False
    assert torch.equal(got[untouched], g0.double()[untouched])
    if bn:
        xh = (xs.float().double()[rmap] - mean.double()) * rstd.double()
        for name, got_, want_ in (("dw", dw, dw0.double() + (dy_rows * xh).sum(0)), ("db", db, db0.double() + dy_rows.sum(0))):
            e = (got_.double().cpu() - want_).abs().max().item() / want_.abs().max().item()
            assert e < 1e-4, (name, e)


@pytest.mark.parametrize("mode", ["map", "pooled", "identity"])
def test_head_eval_bwd_matches_fp64(mode):
    L = _lib()
    torch.manual_seed(7)
    B, C, H, W, ncls = 5, 200, 7, 9, 37
    T = 1 if mode == "pooled" else H * W
    if mode == "identity":
        ncls = C
    feats = torch.randn(B, C, H, W) * 2 + 1 if T > 1 else torch.randn(B, C)
    Wt = torch.randn(ncls, C) * 0.1
    dl = torch.randn(B, ncls)
    pooled = feats.double().mean((2, 3)) if T > 1 else feats.double()
    dp = dl.double() @ Wt.double() if mode != "identity" else dl.double()
    want_df = (dp / T)[:, :, None, None].expand(B, C, H, W) if T > 1 else dp
    dW0, db0 = torch.randn(ncls, C), torch.randn(ncls)
    want_dW = dW0.double() + dl.double().t() @ pooled
    want_db = db0.double() + dl.double().sum(0)
    d_f, d_W, d_dl = feats.cuda(), Wt.cuda(), dl.cuda()
    df = torch.full(feats.shape, 7.0, device="cuda")
    lin = mode != "identity"
    dW, db = (dW0.cuda(), db0.cuda()) if lin else (None, None)
    ws = torch.empty(B * C, device="cuda")
    L.call("fvit_head_eval_bwd", d_dl.data_ptr(), ncls, B, ncls, d_f.data_ptr(), C, T, d_W.data_ptr() if lin else None,
           ws.data_ptr(), df.data_ptr(), L.ptr(dW), L.ptr(db))
    torch.cuda.synchronize()
    assert (df.double().cpu() - want_df).abs().max().item() <= 1e-5 * want_df.abs().max().item()
    if lin:
        for name, got_, want_ in (("dW", dW, want_dW), ("db", db, want_db)):
            e = (got_.double().cpu() - want_).abs().max().item() / want_.abs().max().item()
            assert e < 1e-5, (name, e)


# ---------------------------------------------------------------------------------- model
def _setup(case, batch=None):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    model = F.create_model(g["entry"], drop_path_rate=0.0, **g["kwargs"])
    O.synth_fill_(model.state_dict(), g["seeds"]["w"])
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    x = _input(batch or g["train"]["batch"], g["cfg"]["resolution"], model.cfg["in_chans"], g["seeds"]["x"] + 300)
    return g, model.cuda().eval(), sd, x


def _input(b, res, cin, seed):
    gen = torch.Generator().manual_seed(seed)
    res = (res, res) if isinstance(res, int) else tuple(res)
    return torch.randn((b, cin) + res, generator=gen, dtype=torch.float64).float()


def _weights(outs, seed=3):
    gen = torch.Generator().manual_seed(seed)
    return {k: torch.randn(tuple(o.shape), generator=gen, dtype=torch.float64) for k, o in outs.items()}


def _oracle(sd, cfg, x, weights, *, norms=None, frozen=(), final=False, head=False):
    """fp64 autograd of the eval-mode oracle, loss = sum_k <weights[k], out_k>: (outputs, {name: grad}, dx, d loss /
    d norm when final). Level outputs, each through the running-statistics BatchNorm `norms[k]` (a state-dict prefix)
    when given; final: the `norm`-ed last map (forward_features), head: its logits (forward_head)."""
    from oracle import fastervit_oracle as O
    leaf = DO.leaves(sd, frozen)
    xl = x.double().clone().requires_grad_(True)
    stop = len(cfg["depths"]) - 1 if final else max(weights)
    fw = DO.dense_forward(leaf, cfg, xl, stop_level=stop, final="norm" if final else None, training=False)
    loss, outs, fnorm = 0.0, {}, None
    for k, w in weights.items():
        if final:
            o = fnorm = fw["norm"]
            fnorm.retain_grad()
            if head:
                o = fw["pooled"] @ leaf["head.weight"].t() + leaf["head.bias"]
        else:
            o = fw["levels"][k]
            if norms and norms.get(k):
                o = O._bn(o, leaf, norms[k], 1e-5, False)
        outs[k] = o.detach()
        loss = loss + (o * w).sum()
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    loss.backward(inputs=[leaf[k] for k in names] + [xl])
    grads = {k: leaf[k].grad for k in names if leaf[k].grad is not None}
    return outs, grads, xl.grad, (fnorm.grad if fnorm is not None else None)


def _check(named, ref, strip="", zero_ok=()):
    """every parameter with a reference gradient within the bars; the others without a gradient"""
    gmax = max(v.abs().max().item() for v in ref.values())
    bad, l2s = [], []
    for k, p in named:
        k = k[len(strip):] if strip and k.startswith(strip) else k
        want = ref.get(k)
        if want is None:
            assert p.grad is None or (k.startswith(zero_ok) and not p.grad.any()), k
            continue
        assert p.grad is not None and p.grad.shape == want.shape, k
        got = p.grad.double().cpu()
        floor = max(want.abs().max().item(), 1e-3 * gmax)
        emax = (got - want).abs().max().item() / floor
        el2 = _rel_l2(got, want, 1e-3 * gmax)
        l2s.append(el2)
        if emax > 8e-2 or el2 > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, emax, el2))
    assert l2s and not bad, bad[:10]
    med = sorted(l2s)[len(l2s) // 2]
    assert med <= EVAL_MEDIAN_BAR, med
    return med


_LEVEL_CASES = [(c, i) for c in ("tiny_a", "tiny_ar") for i in ((0, 1, 2, 3), (1,), (2,))] + \
               [("tiny_21k224", (0, 1, 2, 3)), ("fv0", (0, 1, 2, 3))]


@pytest.mark.parametrize("case,idx", _LEVEL_CASES)
def test_forward_levels_eval_gradients_match_fp64(case, idx):
    g, model, sd, x = _setup(case)
    xg = x.cuda().requires_grad_(True)
    feats = model.forward_levels(xg, idx)
    assert all(f.grad_fn is not None for f in feats)
    w = _weights(dict(zip(idx, feats)))
    torch.autograd.backward(feats, [w[i].float().cuda() for i in idx])
    torch.cuda.synchronize()
    ref_out, ref_g, ref_dx, _ = _oracle(sd, g["cfg"], x, w)
    for i, f in zip(idx, feats):
        assert ((f.detach().double().cpu() - ref_out[i]).abs().max() / ref_out[i].abs().max()).item() < 3e-3, i
    med = _check(model.named_parameters(), ref_g)
    dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"{case} {idx}: median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
    assert dx_err <= DX_BAR, dx_err


@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar"])
def test_forward_features_and_head_eval_gradients_match_fp64(case):
    g, model, sd, x = _setup(case)
    # forward_features alone
    xg = x.cuda().requires_grad_(True)
    f = model.forward_features(xg)
    assert f.grad_fn is not None
    w = _weights({0: f})
    f.backward(w[0].float().cuda())
    _, ref_g, ref_dx, _ = _oracle(sd, g["cfg"], x, w, final=True)
    _check(model.named_parameters(), ref_g)
    assert _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0) <= DX_BAR
    # timm-style forward_head(forward_features(x)): the head's gradients, the map gradient between the two, the image
    model.zero_grad(set_to_none=True)
    xg = x.cuda().requires_grad_(True)
    f = model.forward_features(xg)
    f.retain_grad()
    logits = model.forward_head(f)
    assert logits.grad_fn is not None
    with torch.no_grad():
        assert torch.equal(logits.detach(), model.forward_head(model.forward_features(x.cuda())))
    wl = _weights({0: logits}, seed=4)
    logits.backward(wl[0].float().cuda())
    ref_out, ref_g, ref_dx, ref_df = _oracle(sd, g["cfg"], x, wl, final=True, head=True)
    assert ((logits.detach().double().cpu() - ref_out[0]).abs().max() / ref_out[0].abs().max()).item() < 3e-3
    med = _check(model.named_parameters(), ref_g)
    assert _rel_l2(f.grad.double().cpu(), ref_df, 0.0) <= 1e-5
    dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"{case} features + head: median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
    assert dx_err <= DX_BAR


def _backbone(case, fs, out_indices=(1, 2, 3)):
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    kw = {k: v for k, v in g["kwargs"].items() if k != "num_classes"}
    bb = FasterViTBackbone(g["entry"], out_indices=out_indices, frozen_stages=fs, drop_path_rate=0.0, **kw)
    O.synth_fill_(bb.state_dict(), 11)       # (the norm{i} affines and running statistics too)
    sd = {k: v.detach().clone() for k, v in bb.state_dict().items()}
    body_sd = {k[len("body."):]: v for k, v in sd.items() if k.startswith("body.")}
    body_sd.update({k: v for k, v in sd.items() if not k.startswith("body.")})
    x = _input(2, g["cfg"]["resolution"], bb.body.cfg["in_chans"], 19)
    frozen = (["patch_embed."] if fs >= 0 else []) + [f"levels.{i}." for i in range(fs - 1)]
    return g, bb.cuda().eval(), body_sd, x, frozen


@pytest.mark.parametrize("fs", [-1, 0, 2])
@pytest.mark.parametrize("xgrad", [True, False])
def test_backbone_eval_gradients_match_fp64(fs, xgrad):
    g, bb, sd, x, frozen = _backbone("tiny_ar", fs)
    xg = x.cuda().requires_grad_(xgrad)
    outs = bb(xg)
    feats = [outs[k][0] for k in sorted(outs)]
    assert all(f.grad_fn is not None for f in feats)
    w = _weights(dict(zip((1, 2, 3), feats)), seed=8)
    torch.autograd.backward(feats, [w[i].float().cuda() for i in (1, 2, 3)])
    torch.cuda.synchronize()
    ref_out, ref_g, ref_dx, _ = _oracle(sd, g["cfg"], x, w, norms={i: f"norm{i}" for i in (1, 2, 3)}, frozen=frozen)
    for i, f in zip((1, 2, 3), feats):
        assert ((f.detach().double().cpu() - ref_out[i]).abs().max() / ref_out[i].abs().max()).item() < 3e-3, i
    for k, p in bb.named_parameters():
        if any(k[len("body."):].startswith(f) for f in frozen):
            assert p.grad is None, k                    # the frozen prefix: requires_grad = False, no gradient
    for i in (1, 2, 3):
        assert getattr(bb, f"norm{i}").weight.grad is not None
    med = _check(bb.named_parameters(), ref_g, strip="body.")
    if xgrad:
        dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
        print(f"backbone fs={fs}: median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
        assert dx_err <= DX_BAR, dx_err


def test_backbone_image_gradient_with_four_channels_and_channels_last():
    g, bb, sd, x, frozen = _backbone("tiny_c4", 0, out_indices=(0, 2, 3))
    xa = x.cuda().requires_grad_(True)
    outs = bb.forward_raw(xa)
    w = _weights(dict(zip((0, 2, 3), outs)), seed=9)
    torch.autograd.backward(outs, [w[i].float().cuda() for i in (0, 2, 3)])
    _, ref_g, ref_dx, _ = _oracle(sd, g["cfg"], x, w, norms={i: f"norm{i}" for i in (0, 2, 3)}, frozen=frozen)
    assert xa.grad.shape == (2, 4) + x.shape[2:]
    assert _rel_l2(xa.grad.double().cpu(), ref_dx, 0.0) <= DX_BAR
    _check(bb.named_parameters(), ref_g, strip="body.")
    bb.zero_grad(set_to_none=True)
    xb = x.cuda().to(memory_format=torch.channels_last).requires_grad_(True)
    torch.autograd.backward(bb.forward_raw(xb), [w[i].float().cuda() for i in (0, 2, 3)])
    assert (xa.grad - xb.grad).abs().max().item() <= 1e-6 * xa.grad.abs().max().item()


# ---------------------------------------------------------------------------------- invariants and guards
def test_outputs_buffers_and_plans():
    """outputs bitwise equal to the no_grad call; nothing built before the first backward; running statistics and
    num_batches_tracked untouched by the backward; release_eval_grad_plans frees the new plans"""
    g, bb, sd, x, _ = _backbone("tiny_ar", -1)
    model = bb.body
    x = x.cuda()
    eng = model._get_engine()
    with torch.no_grad():
        ref_raw = bb.forward_raw(x)
        ref_lv = model.forward_levels(x, (0, 2))
        ref_f = model.forward_features(x)
    raw, lv, f = bb.forward_raw(x), model.forward_levels(x, (0, 2)), model.forward_features(x)
    for a, b in zip(raw + lv + (f,), ref_raw + ref_lv + (ref_f,)):
        assert a.requires_grad and torch.equal(a.detach(), b)
    assert not eng.eval_grad_plans()
    bufs = {k: v.clone() for k, v in bb.named_buffers()}
    (sum(o.sum() for o in raw) + lv[1].mean() + f.sum()).backward()
    torch.cuda.synchronize()
    assert len(eng.eval_grad_plans()) == 3
    for k, v in bb.named_buffers():
        assert torch.equal(v, bufs[k]), k
    with torch.no_grad():
        assert all(torch.equal(a, b) for a, b in zip(bb.forward_raw(x), ref_raw))
    model.release_eval_grad_plans()
    assert not eng.eval_grad_plans()


def test_unused_output_and_two_forwards_one_backward():
    g, model, sd, x = _setup("tiny_a")
    x1 = x.cuda()
    x2 = _input(x.shape[0], g["cfg"]["resolution"], 3, 77).cuda()
    # one of two outputs used: the same gradients as asking for that output alone (levels 2-3 on the path, zero)
    a, _ = model.forward_levels(x1, (1, 3))
    w = torch.randn(a.shape, generator=torch.Generator().manual_seed(2)).cuda()
    (a * w).sum().backward()
    g_two = {k: None if p.grad is None else p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    (model.forward_levels(x1, (1,))[0] * w).sum().backward()
    for k, p in model.named_parameters():
        if p.grad is None:
            assert g_two[k] is None or not g_two[k].any(), k
        else:
            scale = p.grad.abs().max().item()
            assert (g_two[k] - p.grad).abs().max().item() <= 2e-2 * max(scale, 1e-6), k
    # two forwards feeding one backward: the sum of two single backwards
    model.zero_grad(set_to_none=True)
    fl = lambda xx: model.forward_levels(xx, (2, 3))
    loss = lambda o: o[0].pow(2).mean() + o[1].sum()
    loss(fl(x1)).backward()
    g1 = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    loss(fl(x2)).backward()
    g2 = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    (loss(fl(x1)) + loss(fl(x2))).backward()
    gmax = max(v.abs().max().item() for v in g1.values())
    for k, p in model.named_parameters():
        if k not in g1:
            assert p.grad is None, k
            continue
        ref = g1[k] + g2[k]
        assert (p.grad - ref).abs().max().item() <= 2e-2 * max(ref.abs().max().item(), 1e-2 * gmax), k


def test_guards():
    from fastervit_b200.lib import FvitError
    from fastervit_b200.optim import FusedAdamW
    g, model, sd, x = _setup("tiny_a")
    x = x.cuda()
    # an optimizer step between forward and backward (after a first backward: the step skips parameters without .grad)
    opt = FusedAdamW(model.parameters(), lr=1e-3)
    model.forward_head(model.forward_features(x)).sum().backward()
    out = model.forward_levels(x, (1, 2))
    opt.step()
    with pytest.raises(FvitError, match="weight change"):
        torch.autograd.backward(out, [torch.ones_like(o) for o in out])
    f = model.forward_features(x)
    logits = model.forward_head(f)
    opt.step()
    with pytest.raises(FvitError, match="weight change"):
        logits.sum().backward()
    # first order only
    xg = x.clone().requires_grad_(True)
    (f,) = model.forward_levels(xg, (2,))
    (dx,) = torch.autograd.grad(f.pow(2).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable"):
        dx.pow(2).sum().backward()
    # enable_grad_allreduce
    model.enable_grad_allreduce()
    out = model.forward_features(x)
    with pytest.raises(FvitError, match="all-reduce"):
        out.sum().backward()
    model._grad_allreduce = None
    # train mode: the image still may not require grad, and forward_head still raises
    model.train()
    with pytest.raises(FvitError, match="input requires grad"):
        model.forward_levels(x.clone().requires_grad_(True), (2,))
    with pytest.raises(FvitError, match="inference helper"):
        model.forward_head(torch.zeros(2, model.num_features, 7, 7, device="cuda"))
    model.eval()
    # deploy mode
    model.switch_to_deploy()
    out = model.forward_levels(x, (2,))[0]
    with pytest.raises(FvitError, match="deploy"):
        out.sum().backward()
