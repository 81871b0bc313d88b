"""fvit_feature_map_ln_fwd / fvit_feature_map_ln_bwd (the channel-LayerNorm level outputs of the tracking backbone)
against fp64 torch: a per-pixel LayerNorm over C of token rows gathered through a row map from a window-padded buffer,
written as an NCHW map, and its backward into the rows (scaled by S) plus the weight / bias sums (scaled by a device
scalar).

Tolerances: the forward is one fp32 normalisation per element, so the map is within 1e-5 of max |ref| even with
per-channel offsets of about 1e3 on rows whose per-pixel spread is about 3 (the statistics are moments about a per-pixel
pivot; E[x^2] - E[x]^2 would lose every digit there). The backward sums C products
per pixel and B*T products per channel in fp32 (float atomics across blocks): 1e-4 relative to max |ref| for g, dw and
dbeta."""
import pytest
import torch

pytestmark = pytest.mark.gpu
CHANNELS = [16, 24, 100, 196, 1568]


def _problem(C, B=2, H=13, W=19, pad=3, seed=0):
    """rows of a window-padded buffer ((H + pad) x (W + pad) per image plus a spare row), the row map of the real pixels,
    and the map gradient"""
    g = torch.Generator().manual_seed(seed * 7919 + C)
    T = H * W
    Hp, Wp = H + pad, W + pad
    nrows = B * Hp * Wp + 1
    ld = C + 4   # (a row stride wider than C)
    off = 1e3 + 2.0 * torch.randn(C, generator=g, dtype=torch.float64)   # (per-pixel std ~ 3 under a mean ~ 1e3)
    xs = torch.randn(nrows, ld, generator=g, dtype=torch.float64) * 2.0
    xs[:, :C] += off
    xs = xs.float().double()   # (the values the kernel sees: the reference differs by its arithmetic alone)
    b, y, x = torch.meshgrid(torch.arange(B), torch.arange(H), torch.arange(W), indexing="ij")
    rmap = (b * Hp * Wp + (y + 1) * Wp + x + 2).reshape(-1).to(torch.int32)
    w = 1.0 + 0.5 * torch.randn(C, generator=g, dtype=torch.float64)
    bias = 0.3 * torch.randn(C, generator=g, dtype=torch.float64)
    dy = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    g0 = torch.randn(nrows, C, generator=g, dtype=torch.float64)
    return dict(B=B, T=T, C=C, H=H, W=W, ld=ld, xs=xs, rmap=rmap, w=w, b=bias, dy=dy, g0=g0, eps=1e-6)


def _ref(p):
    B, C, H, W = p["B"], p["C"], p["H"], p["W"]
    x = p["xs"][p["rmap"].long(), :C].requires_grad_(True)       # [B*T, C]
    w = p["w"].clone().requires_grad_(True)
    b = p["b"].clone().requires_grad_(True)
    y = torch.nn.functional.layer_norm(x, (C,), w, b, p["eps"])
    out = y.reshape(B, H, W, C).permute(0, 3, 1, 2)
    out.backward(p["dy"])
    mean = x.detach().mean(1)
    rstd = (x.detach().var(1, unbiased=False) + p["eps"]).rsqrt()
    return out.detach(), x.grad, w.grad, b.grad, mean, rstd


def _cuda(p):
    return {k: (v.float().cuda() if v.is_floating_point() else v.cuda()) if isinstance(v, torch.Tensor) else v
            for k, v in p.items()}


def _fwd(q, stats=True):
    from fastervit_b200 import lib as L
    B, T, C = q["B"], q["T"], q["C"]
    out = torch.full((B, C, q["H"], q["W"]), float("nan"), device="cuda")
    mean = torch.empty(B * T, device="cuda") if stats else None
    rstd = torch.empty(B * T, device="cuda") if stats else None
    L.call("fvit_feature_map_ln_fwd", q["xs"].data_ptr(), q["ld"], q["rmap"].data_ptr(), B, T, C, q["w"].data_ptr(),
           q["b"].data_ptr(), q["eps"], out.data_ptr(), L.ptr(mean), L.ptr(rstd))
    return out, mean, rstd


def _rel(a, b):
    return ((a.double().cpu() - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("C", CHANNELS)
def test_forward_matches_fp64(C):
    p = _problem(C)
    q = _cuda(p)
    out_ref, _, _, _, mean_ref, rstd_ref = _ref(p)
    out, mean, rstd = _fwd(q)
    assert _rel(out, out_ref) < 1e-5
    assert _rel(mean, mean_ref) < 1e-6
    assert _rel(rstd, rstd_ref) < 1e-5
    out2, _, _ = _fwd(q, stats=False)   # inference: no statistics, the same map
    assert torch.equal(out, out2)


@pytest.mark.parametrize("C", CHANNELS)
@pytest.mark.parametrize("with_g", [True, False])
def test_backward_matches_fp64(C, with_g):
    from fastervit_b200 import lib as L
    p = _problem(C, seed=1)
    q = _cuda(p)
    _, dx_ref, dw_ref, db_ref, _, _ = _ref(p)
    _, mean, rstd = _fwd(q)
    S = 64.0
    gs = torch.tensor([S, 1.0 / S], device="cuda")
    scalar = torch.tensor([0.25], device="cuda")
    g = q["g0"].clone()
    dw0 = torch.randn(C, device="cuda")
    db0 = torch.randn(C, device="cuda")
    dw, db = dw0.clone(), db0.clone()
    L.call("fvit_feature_map_ln_bwd", q["dy"].data_ptr(), q["xs"].data_ptr(), q["ld"], q["rmap"].data_ptr(), q["B"],
           q["T"], C, mean.data_ptr(), rstd.data_ptr(), q["w"].data_ptr(), gs.data_ptr(), scalar.data_ptr(),
           g.data_ptr() if with_g else None, C, dw.data_ptr(), db.data_ptr())
    torch.cuda.synchronize()
    assert _rel(dw - dw0, 0.25 * dw_ref) < 1e-4
    assert _rel(db - db0, 0.25 * db_ref) < 1e-4
    if not with_g:
        assert torch.equal(g, q["g0"])
        return
    rows = p["rmap"].long()
    assert _rel(g[rows] - q["g0"][rows], S * dx_ref) < 1e-4
    unmapped = torch.ones(g.shape[0], dtype=torch.bool)
    unmapped[rows] = False
    assert torch.equal(g[unmapped.cuda()], q["g0"][unmapped.cuda()])   # rows outside the map are untouched


def test_backward_without_parameter_gradients():
    """dw = dbeta = NULL: the input gradient alone, the same as with them"""
    from fastervit_b200 import lib as L
    p = _problem(196, seed=2)
    q = _cuda(p)
    _, mean, rstd = _fwd(q)
    gs = torch.tensor([2.0, 0.5], device="cuda")
    ga, gb = q["g0"].clone(), q["g0"].clone()
    dw, db = torch.zeros(196, device="cuda"), torch.zeros(196, device="cuda")
    args = (q["dy"].data_ptr(), q["xs"].data_ptr(), q["ld"], q["rmap"].data_ptr(), q["B"], q["T"], 196, mean.data_ptr(),
            rstd.data_ptr(), q["w"].data_ptr(), gs.data_ptr(), None)
    L.call("fvit_feature_map_ln_bwd", *args, ga.data_ptr(), 196, None, None)
    L.call("fvit_feature_map_ln_bwd", *args, gb.data_ptr(), 196, dw.data_ptr(), db.data_ptr())
    assert torch.equal(ga, gb)
