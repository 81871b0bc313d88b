"""Stride-1 3x3 convolutions through fvit_gemm's slab mode (the three dx taps of a kernel row read one shared
136-row activation slab) against an fp64 conv2d of the same fp16 operands, with the ConvBlock epilogues of a training
step: the forward's BatchNorm column statistics, the data gradient's GELU' of the re-derived pre-activation, and the
row-mapped fp32 residual accumulation. The cases cover row pitches P = W + 2 of 58, 30 and small odd ones (the first M
tile reads negative slab rows, the last one is partial), channel counts with K tails of 4, 8 and 64 columns and of a
single 16-wide step, tile widths 32 ... 128 with a partial last N tile, and grids with 3+ work units per CTA. Slab mode
takes kc > 128; the kc = 64 and 8 cases check that the shapes left on per-tap boxes stay exact too."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-20)).item()


def _gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# (batch, H = W, cin = kc, cout = n, tile_n, epilogue)
CASES = [
    (3, 56, 196, 196, 32, "stats"),    # P 58, K tail 4 (one 16-wide step), 7 N tiles (last 4 wide), 553 units
    (2, 56, 196, 196, 128, "gelu"),    # P 58, N tiles 128 + 68
    (4, 28, 392, 392, 96, "resid"),    # P 30, K tail 8, 5 N tiles (last 8 wide), last M tile 16 rows
    (2, 28, 392, 392, 64, "stats"),    # P 30
    (5, 9, 64, 80, 48, "gelu"),        # P 11, K 64 (no tail), N tiles 48 + 32, 605 rows
    (7, 9, 8, 40, 32, "resid"),        # P 11, K 8 (one block, one step), N tiles 32 + 8
    (4, 11, 196, 130, 0, "stats"),     # P 13, the library's own tile width
    (6, 13, 136, 112, 112, "gelu"),    # P 15, K tail 8 after two full blocks
]


@pytest.mark.parametrize("bsz,hw,cin,cout,tile_n,epi", CASES)
def test_conv3x3_slab(bsz, hw, cin, cout, tile_n, epi):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(bsz * 1000 + hw * 10 + cin)
    H = W = hw
    P = W + 2
    rows = bsz * (H + 2) * P
    ld = (cin + 7) // 8 * 8
    x = torch.randn(bsz, cin, H, W, device="cuda", generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) / (3 * cin ** 0.5)).half()
    xp = torch.zeros(bsz, H + 2, P, ld, device="cuda", dtype=torch.half)
    xp[:, 1:-1, 1:-1, :cin] = x.permute(0, 2, 3, 1)
    a = xp.view(rows, ld)
    kp = (cin + 63) // 64 * 64
    wp = torch.zeros(cout, 9, kp, device="cuda", dtype=torch.half)
    wp[:, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    wp = wp.view(cout, 9 * kp)
    taps = [((dy - 1) * P + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    inside = torch.zeros(bsz, H + 2, P, dtype=torch.bool, device="cuda")
    inside[:, 1:-1, 1:-1] = True
    inside = inside.view(-1)
    ident = torch.arange(rows, device="cuda", dtype=torch.int32)
    row_map = torch.where(inside, ident, torch.full_like(ident, -1))
    units = -(-rows // 128) * -(-cout // tile_n) if tile_n else None

    conv = torch.nn.functional.conv2d(x.double().cpu(), w.double().cpu(), padding=1)   # [B, cout, H, W]
    ref = conv.permute(0, 2, 3, 1).reshape(-1, cout).cuda()                              # interior rows, in order

    def interior(t):
        return t.view(bsz, H + 2, P, -1)[:, 1:-1, 1:-1].reshape(bsz * H * W, -1)[:, :cout]

    ldo = (cout + 7) // 8 * 8
    if epi == "stats":
        shift = torch.randn(cout, device="cuda", generator=g)
        out = torch.full((rows, ldo), 7.0, device="cuda", dtype=torch.half)
        csum, csq = torch.zeros(cout, device="cuda"), torch.zeros(cout, device="cuda")
        lib.gemm(a, wp, m=rows, n=cout, kc=cin, taps=taps, tile_n=tile_n, col_shift=shift, row_map=row_map,
                 out_f16=out, col_sum=csum, col_sumsq=csq)
        want = ref + shift.double()
        assert _rel(interior(out), want) < 2e-3
        assert (out.view(bsz, H + 2, P, ldo)[:, 0] == 7.0).all()          # border rows untouched
        sref, qref = want.sum(0), (want * want).sum(0)
        assert ((csum.double() - sref).norm() / sref.norm()).item() < 1e-4
        assert ((csq.double() - qref).norm() / qref.norm()).item() < 1e-4
    elif epi == "gelu":
        aux = torch.randn(rows, ldo, device="cuda", generator=g).half()
        sc = torch.rand(cout, device="cuda", generator=g) + 0.5
        sh = torch.randn(cout, device="cuda", generator=g) * 0.5
        out = torch.zeros(rows, ldo, device="cuda", dtype=torch.half)
        lib.gemm(a, wp, m=rows, n=cout, kc=cin, taps=taps, tile_n=tile_n, act=lib.ACT_GELU_BWD, aux=aux,
                 aux_scale=sc, aux_shift=sh, row_map=row_map, out_f16=out)
        pre = interior(aux).double() * sc.double() + sh.double()
        assert _rel(interior(out), ref * _gelu_grad(pre)) < 2e-3
    else:
        resid = torch.randn(rows, cout, device="cuda", generator=g)
        r0 = resid.clone()
        lib.gemm(a, wp, m=rows, n=cout, kc=cin, taps=taps, tile_n=tile_n, resid=resid, out_f32=resid, row_map=row_map)
        assert _rel(interior(resid) - interior(r0), ref) < 2e-5
        assert torch.equal(resid[~inside], r0[~inside])                    # border rows untouched
    if units is not None and bsz == 3:
        assert units >= 3 * torch.cuda.get_device_properties(0).multi_processor_count


def test_conv3x3_slab_matches_unshared_taps():
    """The same 9-tap GEMM with its taps listed in another order is not the slab pattern and loads one A box per tap:
    both paths give the same products."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(11)
    bsz, H, cin, cout = 2, 20, 196, 64
    P = H + 2
    rows = bsz * P * P
    a = torch.randn(rows, cin + 4, device="cuda", generator=g).half()
    wp = (torch.randn(cout, 9, 256, device="cuda", generator=g) * 0.05).half()
    wp[:, :, cin:] = 0
    taps = [((dy - 1) * P + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    slab = torch.zeros(rows, cout, device="cuda")
    lib.gemm(a, wp.view(cout, 9 * 256), m=rows, n=cout, kc=cin, taps=taps, out_f32=slab)
    perm = [4, 0, 1, 2, 3, 5, 6, 7, 8]
    wq = wp[:, perm].reshape(cout, 9 * 256).contiguous()
    plain = torch.zeros(rows, cout, device="cuda")
    lib.gemm(a, wq, m=rows, n=cout, kc=cin, taps=[taps[t] for t in perm], out_f32=plain)
    assert _rel(slab, plain) < 1e-5
