"""in_chans != 3 on the GPU: fvit_stem_im2col for any channel count and the image-gradient pair (dcol GEMM +
fvit_stem_col2im) against fp64 torch with sentinel-filled outputs, then the model at 1, 4 and 13 channels against the
fp64 oracle / the reference's golden vectors (tests/make_golden_in_chans.py): eval logits, one train step, eval-mode
parameter and image gradients, FasterViTBackbone training with a frozen prefix, and channels-last input.
Bars are those of the RGB tests: eval logits 1e-3 (test_model_gpu.py); a train step as test_train_gpu.py; eval-mode
gradients as test_eval_grad_gpu.py (median parameter rel-L2 1.5e-3, image rel-L2 3e-2)."""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as Fn

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/make_golden_in_chans.py, tests/_dense_oracle.py
from make_golden_in_chans import CASES, synth_input  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"
_BUF = ("running_mean", "running_var", "num_batches_tracked", "relative_coords_table", "relative_position_index",
        "relative_bias")


def _lib():
    from fastervit_b200 import lib as L
    L.load()
    return L


def _stem_ld(cin):
    return (9 * cin + 31) // 32 * 32


# ---------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("cin", [1, 2, 4, 7, 13, 64])
def test_stem_im2col_any_cin_is_exact(cin, channels_last):
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(cin)
    B, H, W = 2, 37, 51
    x = torch.randn(B, cin, H, W, device="cuda", generator=g) * 3
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    npix = B * ((H + 1) // 2) * ((W + 1) // 2)
    ldo = _stem_ld(cin) + 8                               # (a wider row: every padding column is written too)
    out = torch.full((npix + 5, ldo), 7.0, dtype=torch.float16, device="cuda")
    L.call("fvit_stem_im2col", x.data_ptr(), *x.stride(), B, cin, H, W, out.data_ptr(), ldo)
    torch.cuda.synchronize()
    want = Fn.unfold(x.half().float(), 3, padding=1, stride=2).transpose(1, 2).reshape(npix, 9 * cin).half()
    assert torch.equal(out[:npix, :9 * cin], want)
    assert (out[:npix, 9 * cin:] == 0).all()
    assert (out[npix:] == 7.0).all()


def test_stem_kernels_reject_channel_counts_outside_the_limit():
    from fastervit_b200.lib import FvitError
    L = _lib()
    x = torch.zeros(1, 65, 8, 8, device="cuda")
    out = torch.zeros(16, 640, dtype=torch.float16, device="cuda")
    for cin in (0, 65):
        with pytest.raises(FvitError, match="must be in \\[1, 64\\]"):
            L.call("fvit_stem_im2col", x.data_ptr(), *x.stride(), 1, cin, 8, 8, out.data_ptr(), 640)
    with pytest.raises(FvitError, match=">= 128"):
        L.call("fvit_stem_im2col", x.data_ptr(), *x.stride(), 1, 13, 8, 8, out.data_ptr(), 120)
    dcol, dx = torch.zeros(16, 600, device="cuda"), torch.zeros(65 * 64, device="cuda")
    with pytest.raises(FvitError, match="must be in \\[1, 64\\]"):
        L.call("fvit_stem_col2im", dcol.data_ptr(), 600, 1, 65, 8, 8, dx.data_ptr())
    with pytest.raises(FvitError, match="bad arguments"):
        L.call("fvit_stem_col2im", dcol.data_ptr(), 8, 1, 1, 8, 8, dx.data_ptr())


@pytest.mark.parametrize("cin,B,H,W,cout", [(1, 2, 37, 51, 16), (4, 2, 64, 48, 64), (13, 1, 33, 35, 64),
                                            (64, 1, 31, 17, 32), (7, 3, 1, 1, 16)])
def test_stem_image_gradient_gemm_and_col2im_match_fp64(cin, B, H, W, cout):
    """dx = conv2d_input(dz, W1) / S as the plans run it: dcol = dz . W1 (fvit_gemm, fp32 out, scale 1/S), then
    fvit_stem_col2im; dz and W1 are the fp16 operands, so fp32 accumulation is the only difference from fp64"""
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(cin * 100 + H)
    H1, W1 = (H + 1) // 2, (W + 1) // 2
    npix, k1, sld = B * H1 * W1, 9 * cin, _stem_ld(cin)
    ld_in = (cout + 7) // 8 * 8
    dz = torch.zeros(npix, ld_in, dtype=torch.float16, device="cuda")
    dz[:, :cout] = torch.randn(npix, cout, device="cuda", generator=g).half()
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.2
    w16 = torch.zeros(cout, sld, dtype=torch.float16, device="cuda")
    w16[:, :k1] = w.reshape(cout, k1).half()
    inv = torch.tensor([0.25], device="cuda")
    ldc = (k1 + 3) // 4 * 4
    dcol = torch.full((npix, ldc), float("nan"), device="cuda")
    L.gemm(dz, w16, b_mn=True, n=k1, kc=cout, alpha_ptr=inv, out_f32=dcol)
    dx = torch.full((B, cin, H, W), float("nan"), device="cuda")
    L.call("fvit_stem_col2im", dcol.data_ptr(), ldc, B, cin, H, W, dx.data_ptr())
    torch.cuda.synchronize()
    dz4 = dz[:, :cout].double().view(B, H1, W1, cout).permute(0, 3, 1, 2)
    want = torch.nn.grad.conv2d_input((B, cin, H, W), w16[:, :k1].double().view(cout, cin, 3, 3), dz4, stride=2,
                                      padding=1) * 0.25
    err = (dx.double() - want).abs().max().item() / want.abs().max().item()
    assert err < 1e-5, err


# ---------------------------------------------------------------------------------- model
def _build(case, cin=None, train_batch=False, **extra):
    """model (synthetic weights of the golden recipe), its fp64 state_dict, the oracle cfg and an input"""
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    entry, kw, cfg, (b_eval, b_train) = CASES[case]
    kw = dict(kw, **extra)
    if cin is not None:
        kw["in_chans"] = cin
    model = F.create_model(entry, drop_path_rate=0.0, **kw)
    O.synth_fill_(model.state_dict(), 1234)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    b = b_train if train_batch else b_eval
    x = synth_input(b, cfg["resolution"], 1 + (100 if train_batch else 0), kw["in_chans"], torch.float32)
    return model.cuda(), sd, cfg, x


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("cin", [1, 4, 13])
@pytest.mark.parametrize("case", ["tiny_c4", "tiny_ar_c1"])
def test_eval_logits_match_the_oracle(case, cin):
    from oracle import fastervit_oracle as O
    model, sd, cfg, x = _build(case, cin)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    with torch.no_grad():
        ref = O.forward(sd, cfg, x.double())
        out = model.eval()(x.cuda())
        feats = model.forward_features(x.cuda())
    torch.cuda.synchronize()
    err = _rel(out, ref)
    print(f"{case} in_chans={cin}: eval logits max-rel {err:.2e}")
    assert err < 1e-3, err
    cap = {}
    with torch.no_grad():
        O.forward(sd, cfg, x.double(), capture=cap)
    assert _rel(feats, cap["norm"]) < 1e-3


@pytest.mark.parametrize("case", ["tiny_c4", "tiny_ar_c1"])
def test_eval_logits_match_the_reference_golden(case):
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    model, _, cfg, x = _build(case)
    with torch.no_grad():
        out = model.eval()(x.cuda())
    assert _rel(out, g["eval"]["logits"]) < 1e-3


def _sample(t, n=512):
    f = t.detach().flatten()
    return f[::max(1, (f.numel() + n - 1) // n)].float().cpu()


@pytest.mark.parametrize("case", ["tiny_c4", "tiny_ar_c1"])
def test_train_step_matches_reference(case):
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    tr = g["train"]
    model, _, _, x = _build(case, train_batch=True)
    logits = model.train()(x.cuda())
    loss = Fn.cross_entropy(logits, tr["target"].cuda())
    loss.backward()
    torch.cuda.synchronize()
    assert _rel(logits, tr["logits"]) < 3e-3
    assert abs(loss.item() - tr["loss"]) < 1e-4 * abs(tr["loss"]) + 1e-4
    sd = model.state_dict()
    for k, want in tr["bn_after"].items():
        assert (_sample(sd[k]) - want["sample"]).abs().max().item() <= 1e-3 * max(want["amax"], 1e-6) + 1e-6, k
    gmax = max(w["amax"] for w in tr["grads"].values())
    bad, l2s = [], []
    for k, p in model.named_parameters():
        want = tr["grads"][k]
        assert p.grad is not None and tuple(p.grad.shape) == tuple(want["shape"]), k
        smp = _sample(p.grad)
        emax = (smp - want["sample"]).abs().max().item() / max(want["amax"], 1e-3 * gmax)
        el2 = (smp - want["sample"]).norm().item() / max(want["sample"].norm().item(), 1e-3 * gmax * smp.numel() ** 0.5)
        l2s.append(el2)
        if emax > 8e-2 or el2 > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, emax, el2))
    assert not bad, bad[:10]
    med = sorted(l2s)[len(l2s) // 2]
    print(f"{case}: train step median gradient rel-L2 {med:.2e}")
    assert med <= 4e-3, med


def _oracle_eval_grads(sd, cfg, x, target):
    """fp64 CPU autograd of the oracle with training=False: (logits, {name: grad}, dx)"""
    from oracle import fastervit_oracle as O
    leaf = {}
    for k, v in sd.items():
        v = v.double() if v.is_floating_point() else v
        leaf[k] = v.clone().requires_grad_(True) if v.is_floating_point() and not k.endswith(_BUF) else v.clone()
    for k in list(leaf):
        if ".global_tokenizer.to_global_feature.pos." in k:
            leaf[k] = leaf[k.replace(".to_global_feature.pos.", ".pos_embed.")]
    xl = x.double().clone().requires_grad_(True)
    out = O.forward(leaf, cfg, xl, training=False)
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(Fn.cross_entropy(out, target), [leaf[k] for k in names] + [xl], allow_unused=True)
    return out.detach(), {k: g for k, g in zip(names, grads[:-1]) if g is not None}, grads[-1]


def _rel_l2(got, want, floor):
    return (got - want).norm().item() / max(want.norm().item(), floor * want.numel() ** 0.5)


@pytest.mark.parametrize("case,cin", [("tiny_c4", 4), ("tiny_ar_c1", 1), ("tiny_c4", 13)])
def test_eval_gradients_match_fp64(case, cin):
    model, sd, cfg, x = _build(case, cin, train_batch=True)
    target = torch.tensor([1, 5, 7][:x.shape[0]])
    ref_logits, ref_grads, ref_dx = _oracle_eval_grads(sd, cfg, x, target)
    xg = x.cuda().requires_grad_(True)
    logits = model.eval()(xg)
    Fn.cross_entropy(logits, target.cuda()).backward()
    torch.cuda.synchronize()
    assert _rel(logits, ref_logits) < 1e-3
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    bad, l2s = [], []
    for k, p in model.named_parameters():
        want = ref_grads[k]
        assert p.grad is not None and p.grad.shape == want.shape, k
        got = p.grad.double().cpu()
        emax = (got - want).abs().max().item() / max(want.abs().max().item(), 1e-3 * gmax)
        el2 = _rel_l2(got, want, 1e-3 * gmax)
        l2s.append(el2)
        if emax > 8e-2 or el2 > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, emax, el2))
    assert not bad, bad[:10]
    med = sorted(l2s)[len(l2s) // 2]
    assert xg.grad.shape == x.shape
    dx_err = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"{case} in_chans={cin}: eval-grad median rel-L2 {med:.2e}, dx rel-L2 {dx_err:.2e}")
    assert med <= 1.5e-3, med
    assert dx_err <= 3e-2, dx_err


@pytest.mark.parametrize("fs", [-1, 1])
def test_backbone_train_with_frozen_stages(fs):
    import _dense_oracle as DO
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    entry, kw, cfg, _ = CASES["tiny_ar_c1"]
    bb = FasterViTBackbone(entry, out_indices=(1, 2, 3), frozen_stages=fs, drop_path_rate=0.0, **dict(kw, in_chans=4))
    O.synth_fill_(bb.state_dict(), 11)
    sd = {k: v.detach().clone() for k, v in bb.state_dict().items()}
    x = synth_input(2, cfg["resolution"], 3, 4)
    bb = bb.cuda().train()
    frozen = ["patch_embed."] if fs >= 0 else []
    outs = bb.forward_raw(x.cuda())
    gen = torch.Generator().manual_seed(8)
    w = {i: torch.randn(tuple(o.shape), generator=gen, dtype=torch.float64) * 10.0 ** n
         for n, (i, o) in enumerate(zip((1, 2, 3), outs))}
    torch.autograd.backward(outs, [w[i].float().cuda() for i in (1, 2, 3)])
    torch.cuda.synchronize()
    body_sd = {k[len("body."):]: v for k, v in sd.items() if k.startswith("body.")}
    body_sd.update({k: v for k, v in sd.items() if not k.startswith("body.")})
    ref_out, ref_g, _ = DO.levels_loss_and_grads(body_sd, cfg, x, w, level_norms={i: f"norm{i}" for i in (1, 2, 3)},
                                                 frozen_prefixes=frozen)
    for i, o in zip((1, 2, 3), outs):
        assert _rel(o, ref_out[i]) < 3e-3, i
    gmax = max(v.abs().max().item() for v in ref_g.values())
    l2s = []
    for k, p in bb.named_parameters():
        k = k[len("body."):] if k.startswith("body.") else k
        if any(k.startswith(f) for f in frozen):
            assert p.grad is None, k
            continue
        want = ref_g.get(k)
        if want is None:
            continue
        assert p.grad is not None, k
        err = _rel_l2(p.grad.double().cpu(), want, 1e-3 * gmax)
        assert err <= (6e-2 if k.startswith("patch_embed.") else 4e-2), (k, err)
        l2s.append(err)
    assert l2s and sorted(l2s)[len(l2s) // 2] <= 4e-3
    if fs < 0:
        assert bb.body.patch_embed.conv_down[0].weight.grad.shape == (16, 4, 3, 3)


def test_channels_last_input_reads_through_the_strides(monkeypatch):
    """without launch graphs the image is read in place, so channels-last strides reach fvit_stem_im2col: the eval
    logits and the eval-mode gradients equal those of the NCHW copy bitwise"""
    monkeypatch.setenv("FVIT_CUDA_GRAPH", "0")
    model, _, _, x = _build("tiny_c4", 13, train_batch=True)
    model.eval()
    xs = x.cuda()
    xc = xs.to(memory_format=torch.channels_last)
    assert not xc.is_contiguous()
    outs, dxs = [], []
    for inp in (xs, xc):
        inp = inp.detach().requires_grad_(True)
        out = model(inp)
        out.sum().backward()
        outs.append(out.detach())
        dxs.append(inp.grad)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(dxs[0], dxs[1])
    # train mode: the batch statistics are sums of atomics, so two steps agree to rounding, not bitwise
    model.train()
    assert _rel(model(xc), model(xs)) < 1e-3


def test_input_with_the_wrong_channel_count_raises():
    from fastervit_b200.lib import FvitError
    model, _, _, x = _build("tiny_c4")
    with pytest.raises(FvitError, match="4-channel"):
        model.eval()(torch.zeros(2, 3, 224, 224, device="cuda"))
