"""fp64 parity of the detection backbone's carrier tokenizer kernels -- fvit_token_init_nchw_fwd, _nchw_bwd and
_nchw_dgrad -- against a torch restatement of the reference operation (dino/models/dino/fastervit.py:569-592):
depthwise 3 x 3 convolution + bias, an average pool whose kernel / stride follow the input side, then
x.reshape(B, oh*ow, C) of the pooled NCHW map, so that pooled value (c, p) of image b is channel (c*oh*ow + p) % C of
token (c*oh*ow + p) / C.

Geometries: the level-2 maps of a seeded sweep of DETR training sizes (35 ... 84 pixels a side, pools of kernel 8 ... 14
with stride 3 that overlap, 100 ... 384 carriers: the fallback data-gradient kernel), the small maps of 224-class inputs
(the shared-memory tile kernel), and two large overlapping pools. Channels below, equal to and above oh*ow, so the
token / channel split crosses rows in each of the three ways. The problem layout is test_glue_kernels_gpu.py's: a
scattered pix_map with -1 padding pixels, a scattered ct_row_map with spare rows, strides larger than C."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_token_init.py
from _token_init import detr_shapes, level_sizes, token_init_problem  # noqa: E402

pytestmark = pytest.mark.gpu
WS, CS = 7, 2   # level-2 window and carrier size of the detection configs


def _pool(r):
    """(kernel, stride, output) of the reference's average pool over a padded side of r pixels (fastervit.py:574-579)"""
    out = int(CS * r / WS)
    stride = int(r / out)
    return r - (out - 1) * stride, stride, out


def _sweep_sides():
    """distinct padded level-2 maps token_geometry gives the fv0-like detection backbone over 40 DETR sizes"""
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import token_geometry
    det = build_fastervit("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    sides = []
    for H, W in detr_shapes(40):
        geo = token_geometry(det, 2, *level_sizes(H, W)[2])
        assert tuple(geo["pool"]) == (_pool(geo["Hp"]), _pool(geo["Wp"])) and geo["tokens"] == "nchw"
        if (geo["Hp"], geo["Wp"]) not in sides:
            sides.append((geo["Hp"], geo["Wp"]))
    return sides


# (7, 7) -> 2 x 2, (7, 14) -> 2 x 4, (14, 14) -> 4 x 4 carriers fit the tile kernel's shared memory; (56, 84) (pool
# 11 x 15), (77, 49) (pool 14 x 10) and the sweep take the fallback kernel
SIDES = [(7, 7), (7, 14), (14, 14), (56, 84), (77, 49)]
SIDES += [s for s in _sweep_sides() if s not in SIDES]
CHANNELS = {"below": lambda n: n // 2 + 1, "equal": lambda n: n, "above": lambda n: 2 * n + 5}


def _L():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _close(got, ref, rel, what=""):
    ref = ref.double()
    d = (got.double().cpu() - ref.cpu()).abs().max().item()
    assert d <= rel * max(ref.abs().max().item(), 1e-6), (what, d, ref.abs().max().item())


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _problem(side, rel, seed):
    Hp, Wp = side
    (kh, sh, oh), (kw, sw, ow) = _pool(Hp), _pool(Wp)
    C = CHANNELS[rel](oh * ow)
    P = token_init_problem(_g(seed * 1000 + Hp * Wp + C), 2, Hp, Wp, C, kh, kw, sh, sw)
    assert (P["oh"], P["ow"]) == (oh, ow)
    return P, (Hp, Wp, C, kh, kw, sh, sw, oh, ow)


def _reference(P, geo, x, w, b):
    """the reference forward on an fp64 B x C x Hp x Wp map: the tokens as [B * oh*ow, C]"""
    Hp, Wp, C, kh, kw, sh, sw, oh, ow = geo
    y = torch.nn.functional.conv2d(x, w, b, padding=1, groups=C)
    y = torch.nn.functional.avg_pool2d(y, (kh, kw), (sh, sw))
    assert y.shape[-2:] == (oh, ow)
    return y.reshape(-1, oh * ow, C).reshape(-1, C)


@pytest.mark.parametrize("rel", list(CHANNELS))
@pytest.mark.parametrize("side", SIDES, ids=[f"{h}x{w}" for h, w in SIDES])
def test_token_init_nchw_fwd(side, rel):
    """ct[ct_row_map[b*oh*ow + t], k] = token t, channel k of the reshaped pooled map; rows outside ct_row_map and
    columns >= C keep their sentinels."""
    L = _L()
    P, geo = _problem(side, rel, 1)
    Hp, Wp, C, kh, kw, sh, sw, oh, ow = geo
    ldo = C + 8
    out = torch.full((P["nct"] + 9, ldo), 7.0, device="cuda")
    L.call("fvit_token_init_nchw_fwd", P["xs"].data_ptr(), C + 4, P["pix_map"].data_ptr(), 2, Hp, Wp, C,
           P["w"].data_ptr(), P["bias"].data_ptr(), kh, kw, sh, sw, oh, ow, P["ct_rows"].data_ptr(), out.data_ptr(),
           ldo)
    torch.cuda.synchronize()
    want = _reference(P, geo, P["xmap"].cpu(), P["w"].double().cpu(), P["bias"].double().cpu())
    _close(out[P["ct_rows"].long(), :C], want, 2e-6, "ct")
    assert (out[:, C:] == 7.0).all()
    untouched = torch.ones(P["nct"] + 9, dtype=torch.bool, device="cuda")
    untouched[P["ct_rows"].long()] = False
    assert (out[untouched] == 7.0).all()


@pytest.mark.parametrize("rel", list(CHANNELS))
@pytest.mark.parametrize("side", SIDES, ids=[f"{h}x{w}" for h, w in SIDES])
def test_token_init_nchw_bwd_and_dgrad(side, rel):
    """_nchw_bwd: gx[pix_map[p]] += d/dx onto non-zero contents (padding pixels and rows outside pix_map untouched),
    dw / dbias += scalar * d/dw, d/dbias, against fp64 autograd of the reference forward. _nchw_dgrad: bitwise the gx of
    _nchw_bwd (the same data-gradient kernel without the parameter sums)."""
    L = _L()
    P, geo = _problem(side, rel, 2)
    Hp, Wp, C, kh, kw, sh, sw, oh, ow = geo
    B, n = 2, oh * ow
    x16 = P["xs"].half()
    keep = ~P["pad"]
    xmap = torch.zeros(P["npix"], C, dtype=torch.float64, device="cuda")
    xmap[keep] = x16[P["pix_map"][keep].long(), :C].double()
    xd = xmap.view(B, Hp, Wp, C).permute(0, 3, 1, 2).cpu().clone().requires_grad_(True)
    wd = P["w"].double().cpu().clone().requires_grad_(True)
    bd = P["bias"].double().cpu().clone().requires_grad_(True)
    gct = torch.randn(B * n, C, device="cuda", generator=_g(3))
    _reference(P, geo, xd, wd, bd).backward(gct.double().cpu())
    ldg, ldgx = C + 8, C + 4
    g = torch.full((P["nct"] + 9, ldg), float("nan"), device="cuda")   # rows / columns no carrier owns are never read
    g[P["ct_rows"].long(), :C] = gct
    gx = torch.randn(P["total"], ldgx, device="cuda", generator=_g(4))
    gx0 = gx.clone()
    dw = torch.randn(C, 9, device="cuda", generator=_g(5))
    db = torch.randn(C, device="cuda", generator=_g(6))
    dw0, db0 = dw.clone(), db.clone()
    sc = torch.tensor([0.375], device="cuda")
    L.call("fvit_token_init_nchw_bwd", g.data_ptr(), ldg, x16.data_ptr(), C + 4, P["pix_map"].data_ptr(),
           P["ct_rows"].data_ptr(), B, Hp, Wp, C, P["w"].data_ptr(), kh, kw, sh, sw, oh, ow, sc.data_ptr(),
           gx.data_ptr(), ldgx, dw.data_ptr(), db.data_ptr())
    gx_d = gx0.clone()
    L.call("fvit_token_init_nchw_dgrad", g.data_ptr(), ldg, P["pix_map"].data_ptr(), P["ct_rows"].data_ptr(), B, Hp, Wp,
           C, P["w"].data_ptr(), kh, kw, sh, sw, oh, ow, gx_d.data_ptr(), ldgx)
    torch.cuda.synchronize()
    rows = P["pix_map"][keep].long()
    want = gx0[:, :C].double().clone()
    want[rows] += xd.grad.permute(0, 2, 3, 1).reshape(-1, C).cuda()[keep]
    _close(gx[:, :C], want, 1e-5, "gx")
    untouched = torch.ones(P["total"], dtype=torch.bool, device="cuda")
    untouched[rows] = False
    assert torch.equal(gx[untouched], gx0[untouched]) and torch.equal(gx[:, C:], gx0[:, C:])
    _close(dw - dw0, 0.375 * wd.grad.view(C, 9), 1e-4, "dw")
    _close(db - db0, 0.375 * bd.grad, 1e-4, "dbias")
    assert torch.equal(gx_d, gx), "dgrad differs from the gx of the full backward"
