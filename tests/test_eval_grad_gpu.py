"""Gradients of model(x) under .eval(): the three eval backward kernels against fp64 torch, and the model's parameter
and image gradients against autograd of the fp64 oracle with training=False (leaf parameters, leaf x).

Bars: per tensor max element error 8e-2 and relative L2 4e-2 (6e-2 for the stem), as in the training tests. Measured on
an H100 80GB HBM3 over tiny_a, tiny_b, tiny_qk, tiny_ar, tiny_ar148, tiny_21k224, fv0 and the pooled tiny_ar: median
relative L2 of the parameter gradients 3.5e-4 .. 7.3e-4 (fv0 the largest), bar 1.5e-3; image gradient relative L2
1.8e-2 .. 2.25e-2, bar 3e-2. That is the floor of fp16 tensor-core operands: the oracle's own fp16-operand arithmetic
model (quant="fp16", fp64 backward) differs from fp64 by 1.7e-2 (tiny_a) and 1.95e-2 (tiny_ar) in dx, which
test_image_gradient_sits_at_the_fp16_operand_floor pins. The image gradient is compared element by element, so it shows
what the parameter gradients (sums over pixels) average away."""
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"
EVAL_MEDIAN_BAR = 1.5e-3
DX_BAR = 3e-2


def _lib():
    from fastervit_b200 import lib as L
    L.load()
    return L


# ---------------------------------------------------------------------------------- kernels
def _sentinel16(rows, ld):
    return torch.full((rows, ld), 7.0, dtype=torch.float16, device="cuda")


@pytest.mark.parametrize("C,ld,g16,act,colmul,offset", [
    (196, 200, True, 1, False, 0.0), (196, 200, False, 0, True, 0.0), (64, 64, True, 0, False, 100.0),
    (64, 64, False, 1, True, 100.0), (30, 30, True, 1, True, 0.0), (30, 30, False, 0, False, 100.0)])
def test_bn_eval_bwd_matches_fp64(C, ld, g16, act, colmul, offset):
    L = _lib()
    torch.manual_seed(C + act)
    nrows, total = 300, 420
    std = torch.rand(C, dtype=torch.float64) + 0.5
    mean = torch.randn(C, dtype=torch.float64) * std * offset
    var = std ** 2 * (1 + 0.1 * torch.rand(C, dtype=torch.float64))
    raw = (mean + std * torch.randn(total, C, dtype=torch.float64)).half()
    raw_buf = torch.zeros(total, ld, dtype=torch.float16)
    raw_buf[:, :C] = raw
    gin = torch.randn(total, ld, dtype=torch.float64)
    g_rows, r_rows, o_rows = (torch.randperm(total)[:nrows] for _ in range(3))
    w, b = torch.randn(C, dtype=torch.float64), torch.randn(C, dtype=torch.float64) * 0.3
    # no gradient where the ReLU input is within rounding of 0 (fp32 and fp64 may disagree on its sign)
    pre = (raw.double()[r_rows] - mean.float().double()) / torch.sqrt(var.float().double() + 1e-5) * w + b
    gin[g_rows[:, None], torch.arange(C)] *= (pre.abs() > 1e-3)
    cm = torch.rand(C, dtype=torch.float64) + 0.5 if colmul else None
    eps, scalar = 1e-5, 0.25
    gin_dev = (gin.half() if g16 else gin.float()).cuda()
    dy = gin_dev.double().cpu()[g_rows, :C] * (cm if colmul else 1.0)
    rstd = 1.0 / torch.sqrt(var.float().double() + eps)
    xh = (raw_buf.double()[r_rows, :C] - mean.float().double()) * rstd
    if act == 1:
        dy = dy * (xh * w.float().double() + b.float().double() > 0)
    want_out = w.float().double() * rstd * dy
    dw0, db0 = torch.randn(C), torch.randn(C)
    want_dw = dw0.double() + scalar * (dy * xh).sum(0)
    want_db = db0.double() + scalar * dy.sum(0)
    out = _sentinel16(total, ld)
    dw, db = dw0.cuda(), db0.cuda()
    dev = lambda t: t.float().cuda()
    keep = [dev(mean), dev(var), dev(w), dev(b), dev(cm) if colmul else None, torch.tensor([scalar], device="cuda")]
    gr, rr, orr = (t.int().cuda() for t in (g_rows, r_rows, o_rows))
    raw_dev = raw_buf.cuda()
    L.call("fvit_bn_eval_bwd", gin_dev.data_ptr(), int(g16), ld, gr.data_ptr(), raw_dev.data_ptr(), ld, rr.data_ptr(),
           nrows, C, keep[0].data_ptr(), keep[1].data_ptr(), eps, keep[2].data_ptr(), keep[3].data_ptr(), act,
           L.ptr(keep[4]), keep[5].data_ptr(), out.data_ptr(), ld, orr.data_ptr(), dw.data_ptr(), db.data_ptr())
    torch.cuda.synchronize()
    got = out.double().cpu()
    err = (got[o_rows, :C] - want_out).abs().max().item() / want_out.abs().max().item()
    assert err < 2e-3, err
    untouched = torch.ones(total, dtype=torch.bool)
    untouched[o_rows] = False
    assert (got[untouched] == 7.0).all()
    for name, g_, want in (("dw", dw, want_dw), ("db", db, want_db)):
        e = (g_.double().cpu() - want).abs().max().item() / want.abs().max().item()
        assert e < 1e-4, (name, e)


@pytest.mark.parametrize("B,Hm,Wm,crop", [(3, 7, 7, None), (2, 8, 14, (5, 9))])
def test_pool_bn_eval_bwd_matches_fp64(B, Hm, Wm, crop):
    """T = 49, and a cropped any-res map (5 x 9 pixels inside 8 x 14 padded windows)"""
    L = _lib()
    torch.manual_seed(B)
    C, ld = 200, 208
    Hc, Wc = crop or (Hm, Wm)
    T = Hc * Wc
    rows_total = B * Hm * Wm + 5
    bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(Hc), torch.arange(Wc), indexing="ij")
    rmap = (bi * Hm * Wm + yi * Wm + xi).reshape(-1)
    xs = torch.randn(rows_total, ld, dtype=torch.float64) * 2 + 100.0
    mean = xs[rmap, :C].mean(0) + 0.1
    var = xs[rmap, :C].var(0) * 1.1
    w = torch.randn(C, dtype=torch.float64)
    dpool = torch.randn(B, C, dtype=torch.float64)
    eps, scalar = 1e-5, 0.5
    f = lambda t: t.float()
    rstd = 1.0 / torch.sqrt(f(var).double() + eps)
    xh = (f(xs).double()[rmap, :C] - f(mean).double()) * rstd
    want_g = (f(dpool).double() / T * f(w).double() * rstd).repeat_interleave(T, 0)
    dw0, db0 = torch.randn(C), torch.randn(C)
    want_dw = dw0.double() + scalar * (f(dpool).double() * xh.view(B, T, C).mean(1)).sum(0)
    want_db = db0.double() + scalar * f(dpool).double().sum(0)
    g = torch.full((rows_total, C), 7.0, device="cuda")
    dw, db = dw0.cuda(), db0.cuda()
    d = [t.float().cuda() for t in (xs, mean, var, w, dpool)] + [torch.tensor([scalar], device="cuda"), rmap.int().cuda()]
    L.call("fvit_pool_bn_eval_bwd", d[0].data_ptr(), ld, d[6].data_ptr(), B, T, C, d[1].data_ptr(), d[2].data_ptr(), eps,
           d[3].data_ptr(), d[4].data_ptr(), C, d[5].data_ptr(), g.data_ptr(), C, dw.data_ptr(), db.data_ptr())
    torch.cuda.synchronize()
    got = g.double().cpu()
    assert (got[rmap] - want_g).abs().max().item() <= 1e-5 * want_g.abs().max().item()
    untouched = torch.ones(rows_total, dtype=torch.bool)
    untouched[rmap] = False
    assert (got[untouched] == 7.0).all()
    for name, g_, want in (("dw", dw, want_dw), ("db", db, want_db)):
        e = (g_.double().cpu() - want).abs().max().item() / want.abs().max().item()
        assert e < 1e-4, (name, e)


@pytest.mark.parametrize("B,H,W,cout,ld,k", [(2, 224, 224, 64, 64, 6), (2, 35, 61, 196, 196, 10), (3, 1, 1, 16, 16, 0),
                                             (2, 35, 61, 16, 24, 3), (1, 17, 9, 512, 512, 12)])
def test_stem_conv_dgrad_matches_fp64(B, H, W, cout, ld, k):
    L = _lib()
    torch.manual_seed(H + cout)
    H1, W1 = (H + 1) // 2, (W + 1) // 2
    dz = torch.randn(B * H1 * W1, ld).half()
    wgt = torch.randn(cout, 3, 3, 3)
    scalar = 2.0 ** -k
    dz_nchw = dz[:, :cout].double().view(B, H1, W1, cout).permute(0, 3, 1, 2)
    want = scalar * torch.nn.grad.conv2d_input((B, 3, H, W), wgt.double(), dz_nchw, stride=2, padding=1)
    dx = torch.full((B, 3, H, W), 7.0, device="cuda")
    dzd, wd, sd = dz.cuda(), wgt.cuda(), torch.tensor([scalar], device="cuda")
    L.call("fvit_stem_conv_dgrad", dzd.data_ptr(), ld, B, H, W, wd.data_ptr(), cout, sd.data_ptr(), dx.data_ptr())
    torch.cuda.synchronize()
    err = (dx.double().cpu() - want).abs().max().item() / want.abs().max().item()
    assert err < 1e-5, err


# ---------------------------------------------------------------------------------- model
_BUF = ("running_mean", "running_var", "num_batches_tracked", "relative_coords_table", "relative_position_index",
        "relative_bias")


def _oracle_grads(sd, cfg, x, target, identity_head: int = 0, quant=None):
    """fp64 CPU autograd of the oracle forward with training=False: (logits, {name: grad}, dx). identity_head = n: the
    head is replaced by an n x n identity (the pooled features of a num_classes = 0 model)."""
    from oracle import fastervit_oracle as O
    leaf = {}
    for k, v in sd.items():
        v = v.double() if v.is_floating_point() else v
        leaf[k] = v.clone().requires_grad_(True) if v.is_floating_point() and not k.endswith(_BUF) else v.clone()
    for k in list(leaf):
        if ".global_tokenizer.to_global_feature.pos." in k:
            leaf[k] = leaf[k.replace(".to_global_feature.pos.", ".pos_embed.")]
    if identity_head:
        leaf["head.weight"] = torch.eye(identity_head, dtype=torch.float64)
        leaf["head.bias"] = torch.zeros(identity_head, dtype=torch.float64)
    xl = x.double().clone().requires_grad_(True)
    out = O.forward(leaf, cfg, xl, training=False, quant=quant)
    loss = (out * target).sum() if identity_head else torch.nn.functional.cross_entropy(out, target)
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k and not (identity_head and k.startswith("head."))]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names] + [xl], allow_unused=True)
    return out.detach(), {k: g for k, g in zip(names, grads[:-1]) if g is not None}, grads[-1]


def _setup(case, batch=None, num_classes=None):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    kw = dict(g["kwargs"])
    if num_classes is not None:
        kw["num_classes"] = num_classes
    model = F.create_model(g["entry"], drop_path_rate=0.0, **kw)
    O.synth_fill_(model.state_dict(), g["seeds"]["w"])
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    model = model.cuda().eval()
    b = batch or g["train"]["batch"]
    x = O.synth_input(b, g["cfg"]["resolution"], g["seeds"]["x"] + 200, torch.float32)
    return g, model, sd, x


def _rel_l2(got, want, floor):
    return (got - want).norm().item() / max(want.norm().item(), floor * want.numel() ** 0.5)


def _compare(model, ref_grads, skip=()):
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    bad, l2s = [], []
    for k, p in model.named_parameters():
        if k in skip:
            continue
        want = ref_grads[k]
        assert p.grad is not None and p.grad.shape == want.shape, k
        got = p.grad.double().cpu()
        floor = max(want.abs().max().item(), 1e-3 * gmax)
        emax = (got - want).abs().max().item() / floor
        el2 = _rel_l2(got, want, 1e-3 * gmax)
        l2s.append(el2)
        if emax > 8e-2 or el2 > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, emax, el2))
    assert not bad, bad[:10]
    return sorted(l2s)[len(l2s) // 2]


@pytest.mark.parametrize("case", ["tiny_a", "tiny_b", "tiny_qk", "tiny_ar", "tiny_ar148", "tiny_21k224", "fv0"])
def test_eval_gradients_match_fp64(case):
    g, model, sd, x = _setup(case)
    target = g["train"]["target"]
    ref_logits, ref_grads, ref_dx = _oracle_grads(sd, g["cfg"], x, target)
    xg = x.cuda().requires_grad_(True)
    logits = model(xg)
    assert logits.requires_grad
    torch.nn.functional.cross_entropy(logits, target.cuda()).backward()
    torch.cuda.synchronize()
    assert ((logits.detach().double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 1e-3
    med = _compare(model, ref_grads)
    dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"{case}: median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
    assert med <= EVAL_MEDIAN_BAR, med
    assert dx_err <= DX_BAR, dx_err


@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar"])
def test_image_gradient_sits_at_the_fp16_operand_floor(case):
    """dx's distance from fp64 is that of the fp16-operand arithmetic model alone (measured ratios 1.06 / 1.15)"""
    g, model, sd, x = _setup(case)
    target = g["train"]["target"]
    _, _, dx64 = _oracle_grads(sd, g["cfg"], x, target)
    _, _, dx16 = _oracle_grads(sd, g["cfg"], x, target, quant="fp16")
    floor = _rel_l2(dx16, dx64, 0.0)
    xg = x.cuda().requires_grad_(True)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    err = _rel_l2(xg.grad.double().cpu(), dx64, 0.0)
    print(f"{case}: dx rel-L2 {err:.2e}, fp16-operand model {floor:.2e}")
    assert err <= 1.3 * floor, (err, floor)


def test_eval_forward_is_unchanged_and_nothing_else_moves():
    """the logits equal the no_grad call bitwise; the backward leaves the running statistics and num_batches_tracked
    bitwise as they were; a grad-enabled forward without backward builds no eval-grad plan"""
    g, model, sd, x = _setup("tiny_a")
    x = x.cuda()
    with torch.no_grad():
        ref = model(x)
    out = model(x)
    assert out.requires_grad and torch.equal(out.detach(), ref)
    eng = model._get_engine()
    assert not eng.eval_grad_plans()
    bufs = {k: v.clone() for k, v in model.named_buffers()}
    out.sum().backward()
    torch.cuda.synchronize()
    assert len(eng.eval_grad_plans()) == 1
    for k, v in model.named_buffers():
        assert torch.equal(v, bufs[k]), k
    with torch.no_grad():
        assert torch.equal(model(x), ref)
    model.release_eval_grad_plans()
    assert not eng.eval_grad_plans()
    model(x).sum().backward()       # (built again on demand)
    assert len(eng.eval_grad_plans()) == 1


def test_eval_gradients_are_first_order_only():
    """a double-backprop input-gradient penalty raises instead of training with a constant (graph-less) dx"""
    g, model, sd, x = _setup("tiny_a")
    xg = x.cuda().requires_grad_(True)
    ce = torch.nn.functional.cross_entropy(model(xg), g["train"]["target"].cuda())
    (dx,) = torch.autograd.grad(ce, xg, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable"):
        (ce + dx.pow(2).sum()).backward()


def test_linear_probe_and_input_only_gradients():
    g, model, sd, x = _setup("tiny_a")
    target = g["train"]["target"]
    _, ref_grads, ref_dx = _oracle_grads(sd, g["cfg"], x, target)
    for n, p in model.named_parameters():
        p.requires_grad_(n.startswith("head."))
    torch.nn.functional.cross_entropy(model(x.cuda()), target.cuda()).backward()
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    for n, p in model.named_parameters():
        if n.startswith("head."):
            assert _rel_l2(p.grad.double().cpu(), ref_grads[n], 1e-3 * gmax) < 1e-2, n
        else:
            assert p.grad is None, n
    model.zero_grad(set_to_none=True)
    model.requires_grad_(False)
    xg = x.cuda().requires_grad_(True)
    torch.nn.functional.cross_entropy(model(xg), target.cuda()).backward()
    assert all(p.grad is None for p in model.parameters())
    assert _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0) <= DX_BAR


def test_pooled_feature_gradients_of_a_headless_model():
    g, model, sd, x = _setup("tiny_ar", num_classes=0)
    nf = model.num_features
    tgt = torch.randn(x.shape[0], nf, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    ref_out, ref_grads, ref_dx = _oracle_grads(sd, g["cfg"], x, tgt, identity_head=nf)
    xg = x.cuda().requires_grad_(True)
    out = model(xg)
    assert out.shape == (x.shape[0], nf) and out.requires_grad
    (out * tgt.float().cuda()).sum().backward()
    med = _compare(model, ref_grads)
    dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"tiny_ar pooled: median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
    assert med <= EVAL_MEDIAN_BAR and dx_err <= DX_BAR, (med, dx_err)


def test_several_forwards_one_backward():
    """two eval forwards on different inputs and one summed backward give the sum of two single backwards (to the
    split-K summation-order noise of the training test)"""
    from oracle import fastervit_oracle as O
    g, model, sd, x1 = _setup("tiny_a")
    target = g["train"]["target"].cuda()
    x1 = x1.cuda()
    x2 = O.synth_input(x1.shape[0], g["cfg"]["resolution"], 77, torch.float32).cuda()
    ce = torch.nn.functional.cross_entropy
    ce(model(x1), target).backward()
    g1 = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    ce(model(x2), target).backward()
    g2 = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    (ce(model(x1), target) + ce(model(x2), target)).backward()
    gmax = max(v.abs().max().item() for v in g1.values())
    for k, p in model.named_parameters():
        ref = g1[k] + g2[k]
        tol = 2e-2 * max(ref.abs().max().item(), 1e-2 * gmax)
        assert (p.grad - ref).abs().max().item() <= tol, k


def test_guards_and_channels_last_input():
    from fastervit_b200.lib import FvitError
    from fastervit_b200.optim import FusedAdamW
    g, model, sd, x = _setup("tiny_a")
    x = x.cuda()
    ce = torch.nn.functional.cross_entropy
    target = g["train"]["target"].cuda()
    # channels-last x: the same image gradient
    xa = x.clone().requires_grad_(True)
    ce(model(xa), target).backward()
    xb = x.clone().to(memory_format=torch.channels_last).requires_grad_(True)
    ce(model(xb), target).backward()
    assert (xa.grad - xb.grad).abs().max().item() <= 1e-6 * xa.grad.abs().max().item()
    # an in-place change of x between forward and backward: autograd's version check
    xc = x.clone().requires_grad_(True)
    xi = xc * 1.0
    loss = ce(model(xi), target)
    xi.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()
    # an optimizer step between forward and backward changes the weights the recompute would use
    opt = FusedAdamW(model.parameters(), lr=1e-3)
    loss = ce(model(x), target)
    opt.step()
    with pytest.raises(FvitError):
        loss.backward()
