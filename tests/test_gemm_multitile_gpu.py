"""fvit_gemm with several work units per CTA: the persistent kernel hands its shared-memory accumulator tile from
the MMA warpgroups to the epilogue warpgroup once per unit, and the next unit's MMAs run while the epilogue reads
the tile. Every shape here deals at least 3 units to each CTA, so each epilogue feature runs on a tile that was
handed over while the previous unit's epilogue was still in flight. A partial last N tile issues MMAs of its own
width (rounded up to 16): its accumulator columns beyond that width hold an earlier unit's values and must never
reach an output. Checked against torch fp32 math on the same 16-bit operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _tiles_m(tiles_n):
    """M tiles such that tiles_m * tiles_n >= 3 units for every SM."""
    return -(-3 * _sms() // tiles_n) + 1


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-20)).item()


@pytest.mark.parametrize("n,b_mn", [(400, False), (400, True), (208, False), (208, True)])
def test_gemm_partial_last_tile_width(n, b_mn):
    """tile_n 128: the last N tile is 16 (n = 400) or 80 (n = 208) columns wide, K-major and MN-major B."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(n + b_mn)
    tiles_n = -(-n // 128)
    m, k = 128 * _tiles_m(tiles_n) - 37, 200
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = torch.randn(n, k, device="cuda", generator=g).half()
    out = torch.full((m, n), float("nan"), device="cuda")
    lib.gemm(a, b.t().contiguous() if b_mn else b, b_mn=b_mn, tile_n=128, out_f32=out)
    assert _rel(out, a.float() @ b.float().t()) < 2e-5


def test_gemm_multitile_staged_epilogue_inplace():
    """Staged epilogue: scale / shift / GELU / cs2, row-map scatter, residual read and written in place, fp32 and fp16
    outputs; n = 328 has a 72-column last tile (80-wide MMA)."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(21)
    n, k = 328, 256
    m = 128 * _tiles_m(3) - 11
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.2).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.2).half()
    cs = torch.rand(n, device="cuda", generator=g) + 0.5
    sh = torch.randn(n, device="cuda", generator=g)
    cs2 = torch.rand(n, device="cuda", generator=g) + 0.5
    perm = torch.randperm(m, device="cuda", generator=g).int()
    perm[::13] = -1
    x = torch.randn(m, n, device="cuda", generator=g)
    x0 = x.clone()
    o16 = torch.full((m, n), 7.0, device="cuda").half()
    lib.gemm(a, b, alpha=0.5, col_scale=cs, col_shift=sh, act=lib.ACT_GELU, col_scale2=cs2, resid=x, row_map=perm,
             out_f32=x, out_f16=o16, tile_n=128)
    val = torch.nn.functional.gelu((a.float() @ b.float().t()) * 0.5 * cs + sh) * cs2
    keep = perm >= 0
    idx = perm[keep].long()
    ref = x0.clone()
    ref[idx] = val[keep] + x0[idx]
    ref16 = torch.full((m, n), 7.0, device="cuda")
    ref16[idx] = ref[idx]
    assert _rel(x, ref) < 2e-5
    assert _rel(o16, ref16) < 1e-3


@pytest.mark.parametrize("layer_scale,drop_path", [(True, False), (False, True), (True, True)])
def test_gemm_multitile_branch_residual(layer_scale, drop_path):
    """The training forward's branch epilogues (their own compile-time variants): bias, then layer scale (cs2, with
    the pre-scale value saved as fp16) and / or a per-row stochastic-depth factor, added to the fp32 residual stream
    in place; n = 784 with tile_n 128 has a 16-column last tile."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(25 + 2 * layer_scale + drop_path)
    n, k = 784, 320
    m = 128 * _tiles_m(7) - 3
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.2).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.2).half()
    sh = torch.randn(n, device="cuda", generator=g)
    x = torch.randn(m, n, device="cuda", generator=g)
    x0 = x.clone()
    kw = {}
    v = a.float() @ b.float().t() + sh
    pre = v.clone()
    if layer_scale:
        cs2 = torch.rand(n, device="cuda", generator=g) + 0.5
        kw.update(col_scale2=cs2, out_pre16=torch.zeros(m, n, device="cuda").half())
        v = v * cs2
    if drop_path:
        rs = (torch.rand(m, device="cuda", generator=g) > 0.3).float() / 0.7
        kw.update(row_scale=rs)
        v = v * rs[:, None]
    lib.gemm(a, b, col_shift=sh, resid=x, out_f32=x, tile_n=128, **kw)
    assert _rel(x, x0 + v) < 2e-5
    if layer_scale:
        assert _rel(kw["out_pre16"], pre) < 1e-3


def test_gemm_multitile_colstats():
    """BatchNorm statistics (per-CTA shared-memory partials over many units); n = 200 with tile_n 64 has an
    8-column last tile (16-wide MMA)."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(22)
    n, k = 200, 128
    m = 128 * _tiles_m(4) - 5
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    sh = torch.randn(n, device="cuda", generator=g)
    rm = torch.arange(m, device="cuda").int()
    rm[3::7] = -1
    s1 = torch.zeros(n, device="cuda")
    s2 = torch.zeros(n, device="cuda")
    o16 = torch.zeros(m, n, device="cuda").half()
    lib.gemm(a, b, col_shift=sh, row_map=rm, out_f16=o16, col_sum=s1, col_sumsq=s2, tile_n=64)
    v = (a.float() @ b.float().t() + sh)[rm >= 0]
    assert _rel(s1, v.sum(0)) < 1e-4
    assert _rel(s2, (v * v).sum(0)) < 1e-4
    assert _rel(o16[rm >= 0], v) < 1e-3


def test_gemm_multitile_direct_epilogue_colsum():
    """Row-per-thread epilogue with the per-column sum of the rounded output (MUL_AUX, device alpha); n = 784 with
    tile_n 128 has a 16-column last tile, MN-major B as in a data-gradient GEMM."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(23)
    n, k = 784, 192
    m = 128 * _tiles_m(7)
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.1).half()
    aux = torch.randn(m, n, device="cuda", generator=g).half()
    o16 = torch.zeros(m, n, device="cuda").half()
    one = torch.ones(1, device="cuda")
    half = torch.full((1,), 0.5, device="cuda")
    osum = torch.ones(n, device="cuda")
    lib.gemm(a, b, b_mn=True, act=lib.ACT_MUL_AUX, aux=aux, alpha_ptr=one, out_f16=o16, out_colsum=osum,
             out_colsum_alpha=half, tile_n=128)
    assert _rel(o16, (a.float() @ b.float()) * aux.float()) < 1e-3
    ref = 1.0 + 0.5 * o16.double().sum(0)
    assert (osum.double() - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3


def test_gemm_multitile_conv3x3_taps():
    """9-tap 3x3 convolution over a zero-bordered NHWC matrix; cout = 208 with tile_n 128 has an 80-column last
    tile."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(24)
    cin, cout, H, W = 64, 208, 28, 30
    Hp, Wp = H + 2, W + 2
    bsz = -(-_tiles_m(2) * 128 // (Hp * Wp))
    x = torch.randn(bsz, cin, H, W, device="cuda", generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.05).half()
    xp = torch.zeros(bsz, Hp, Wp, cin, device="cuda", dtype=torch.half)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    a = xp.view(-1, cin)
    wp = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    out = torch.zeros(bsz * Hp * Wp, cout, device="cuda")
    lib.gemm(a, wp, kc=cin, taps=taps, out_f32=out, tile_n=128)
    got = out.view(bsz, Hp, Wp, cout)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    # CPU reference: keeps cuDNN (slow to cold-load on a fresh box) out of the test
    ref = torch.nn.functional.conv2d(x.float().cpu(), w.float().cpu(), padding=1).cuda()
    assert _rel(got, ref) < 2e-5
