"""GPU parity tests of fvit_gemm (wgmma GEMM + taps + fused epilogue) against torch fp32 math on the
same 16-bit operands. Tolerances: fp32 accumulation-order noise only (operands are identical)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-20)).item()


@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (1000, 64, 32), (520, 48, 16), (300, 200, 136), (4096, 768, 256), (1000, 1000, 520),
                                   (128 * 200 + 5, 512, 192), (53 * 64, 2352, 784)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gemm_nt_plain(m, n, k, dtype):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n)
    a = torch.randn(m, k, device="cuda", generator=g).to(dtype)
    b = torch.randn(n, k, device="cuda", generator=g).to(dtype)
    out = torch.full((m, n), float("nan"), device="cuda")
    lib.gemm(a, b, out_f32=out)
    ref = a.float() @ b.float().t()
    assert _rel(out, ref) < 2e-5


@pytest.mark.parametrize("tile_n", [16, 48, 64, 112, 208, 256])
def test_gemm_tile_n(tile_n):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(tile_n)
    m, n, k = 777, 400, 264
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = torch.randn(n, k, device="cuda", generator=g).half()
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(a, b, out_f32=out, tile_n=tile_n)
    assert _rel(out, a.float() @ b.float().t()) < 2e-5


def test_gemm_strided_operands():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    m, n, k = 500, 196, 196
    abuf = torch.randn(m, 200, device="cuda", generator=g).half()   # lda = 200 (fv4 C=196 padded)
    bbuf = torch.randn(n, 208, device="cuda", generator=g).half()
    a, b = abuf[:, :k], bbuf[:, :k]
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(a, b, out_f32=out)
    assert _rel(out, a.float() @ b.float().t()) < 2e-5


def test_gemm_epilogue_full():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(11)
    m, n, k = 1000, 328, 256
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.2).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.2).half()
    cs = torch.rand(n, device="cuda", generator=g) + 0.5
    sh = torch.randn(n, device="cuda", generator=g)
    cs2 = torch.rand(n, device="cuda", generator=g) + 0.5
    perm = torch.randperm(m, device="cuda", generator=g).int()
    perm[::17] = -1
    resid = torch.randn(m, n, device="cuda", generator=g)
    o32 = torch.full((m, n), 7.0, device="cuda")
    o16 = torch.full((m, n), 7.0, device="cuda").half()
    lib.gemm(a, b, alpha=0.5, col_scale=cs, col_shift=sh, act=lib.ACT_GELU, col_scale2=cs2,
             resid=resid, row_map=perm, out_f32=o32, out_f16=o16)
    acc = (a.float() @ b.float().t()) * 0.5 * cs + sh
    val = torch.nn.functional.gelu(acc) * cs2
    ref = torch.full((m, n), 7.0, device="cuda")
    keep = perm >= 0
    idx = perm[keep].long()
    ref[idx] = val[keep] + resid[idx]
    assert _rel(o32, ref) < 2e-5
    assert _rel(o16, ref) < 1e-3


def test_gemm_inplace_residual():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(12)
    m, n, k = 640, 256, 128
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = torch.randn(n, k, device="cuda", generator=g).half()
    x = torch.randn(m, n, device="cuda", generator=g)
    ref = x + a.float() @ b.float().t()
    lib.gemm(a, b, resid=x, out_f32=x)
    assert _rel(x, ref) < 2e-5


def test_gemm_colstats():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(13)
    m, n, k = 3000, 200, 128
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    sh = torch.randn(n, device="cuda", generator=g)
    rm = torch.arange(m, device="cuda").int()
    rm[5::9] = -1
    s1 = torch.zeros(n, device="cuda")
    s2 = torch.zeros(n, device="cuda")
    o16 = torch.zeros(m, n, device="cuda").half()
    lib.gemm(a, b, col_shift=sh, row_map=rm, out_f16=o16, col_sum=s1, col_sumsq=s2)
    v = a.float() @ b.float().t() + sh
    v = v[rm >= 0]
    assert _rel(s1, v.sum(0)) < 1e-4
    assert _rel(s2, (v * v).sum(0)) < 1e-4


@pytest.mark.parametrize("a_mn,b_mn", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (520, 392, 1000), (784, 200, 3000)])
def test_gemm_mn_major(a_mn, b_mn, m, n, k):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    A = torch.randn(m, k, device="cuda", generator=g).half()
    B = torch.randn(n, k, device="cuda", generator=g).half()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=out)
    assert _rel(out, A.float() @ B.float().t()) < 2e-5


@pytest.mark.parametrize("tile_n", [16, 80, 208])
def test_gemm_mn_major_b_partial_atom_tiles(tile_n):
    """MN-major B is staged in 64-column atoms; the MMA N (tile_n) may be any multiple of 16."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(tile_n)
    m, n, k = 300, 392, 1000
    A = torch.randn(k, m + 4, device="cuda", generator=g).half()[:, :m]
    B = torch.randn(k, n, device="cuda", generator=g).half()
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(A, B, a_mn=True, b_mn=True, tile_n=tile_n, out_f32=out)
    assert _rel(out, A.float().t() @ B.float()) < 2e-5
    A2 = torch.randn(m, k, device="cuda", generator=g).half()
    lib.gemm(A2, B, b_mn=True, tile_n=tile_n, out_f32=out)
    assert _rel(out, A2.float() @ B.float()) < 2e-5


def test_gemm_split_k_and_row_offsets():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(21)
    m, n, k = 256, 192, 5000
    A = torch.randn(k, m, device="cuda", generator=g).half()  # MN-major [K, M]
    B = torch.randn(k, n, device="cuda", generator=g).half()
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(A, B, a_mn=True, b_mn=True, split_k=16, alpha=0.25, out_f32=out)
    assert _rel(out, 0.25 * (A.float().t() @ B.float())) < 1e-4
    # row offset on B: out[m, n] = sum_r A[r, m] * B[r + off, n], OOB rows are zero
    for off in (-3, 70):
        out.zero_()
        lib.gemm(A, B, a_mn=True, b_mn=True, split_k=8, b_row_off=off, out_f32=out)
        Bs = torch.zeros_like(B)
        if off >= 0:
            Bs[: k - off] = B[off:]
        else:
            Bs[-off:] = B[: k + off]
        assert _rel(out, A.float().t() @ Bs.float()) < 1e-4


@pytest.mark.parametrize("cout,cin,k,sk", [(392, 392, 3000, 4), (196, 196, 9000, 16), (64, 32, 1000, 1), (640, 320, 700, 2)])
def test_gemm_taps_in_n_weight_gradient(cout, cin, k, sk):
    """b_ntaps: out[co][t*cin + ci] = sum_q dz[q][co] * x[q + shift_t][ci] (conv weight gradient in one launch)."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    dz = torch.randn(k, cout, device="cuda", generator=g).half()
    ldx = (cin + 7) // 8 * 8
    x = torch.randn(k, ldx, device="cuda", generator=g).half()[:, :cin]
    dz = torch.randn(k, (cout + 7) // 8 * 8, device="cuda", generator=g).half()[:, :cout]
    shifts = [-31, -30, -29, -1, 0, 1, 29, 30, 31]
    out = torch.zeros(cout, 9 * cin, device="cuda")
    lib.gemm(dz, x, a_mn=True, b_mn=True, b_taps=shifts, split_k=sk, alpha=0.5, out_f32=out)
    ref = torch.zeros_like(out)
    for t, off in enumerate(shifts):
        xs = torch.zeros_like(x)
        if off >= 0:
            xs[: k - off] = x[off:]
        else:
            xs[-off:] = x[: k + off]
        ref[:, t * cin:(t + 1) * cin] = 0.5 * (dz.float().t() @ xs.float())
    assert _rel(out, ref) < 1e-4


@pytest.mark.parametrize("cin,cout,hw", [(64, 64, 14), (196, 208, 9), (128, 256, 28)])
def test_gemm_conv3x3_taps(cin, cout, hw):
    """3x3/s1/p1 conv as 9 shifted-row taps over a zero-bordered NHWC matrix vs F.conv2d."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(cin + hw)
    bsz, H, W = 3, hw, hw + 2
    Hp, Wp = H + 2, W + 2
    ld = (cin + 7) // 8 * 8
    x = torch.randn(bsz, cin, H, W, device="cuda", generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.05).half()
    xp = torch.zeros(bsz, Hp, Wp, ld, device="cuda", dtype=torch.half)
    xp[:, 1:-1, 1:-1, :cin] = x.permute(0, 2, 3, 1)
    a = xp.view(-1, ld)[:, :cin]
    kc_pad = (cin + 63) // 64 * 64
    wp = torch.zeros(cout, 9, kc_pad, device="cuda", dtype=torch.half)
    wp[:, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    out = torch.zeros(bsz * Hp * Wp, cout, device="cuda")
    lib.gemm(a, wp.view(cout, 9 * kc_pad), kc=cin, taps=taps, out_f32=out)
    got = out.view(bsz, Hp, Wp, cout)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    # CPU reference: keeps cuDNN (slow to cold-load on a fresh box) out of the test
    ref = torch.nn.functional.conv2d(x.float().cpu(), w.float().cpu(), padding=1).cuda()
    assert _rel(got, ref) < 2e-5


def test_gemm_planes_stride2_conv():
    """3x3/s2/p1 conv through 4 parity planes (space-to-depth split) and per-tap plane select."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    bsz, cin, cout, H, W = 2, 64, 128, 28, 28
    Ho, Wo = H // 2, W // 2
    x = torch.randn(bsz, cin, H, W, device="cuda", generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.05).half()
    # plane (ph, pw)[b, a+1, c+1] = x[b, 2a+ph, 2c+pw]; row/col 0 are the zero border
    planes = torch.zeros(4, bsz, Ho + 1, Wo + 1, cin, device="cuda", dtype=torch.half)
    xn = x.permute(0, 2, 3, 1)
    for ph in range(2):
        for pw in range(2):
            planes[ph * 2 + pw, :, 1:, 1:] = xn[:, ph::2, pw::2]
    a = planes.view(4, -1, cin)
    wp = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    taps = []
    for r in range(3):
        ph, da = (1, -1) if r == 0 else ((0, 0) if r == 1 else (1, 0))
        for s in range(3):
            pw, db = (1, -1) if s == 0 else ((0, 0) if s == 1 else (1, 0))
            taps.append((da * (Wo + 1) + db, ph * 2 + pw))
    rows = bsz * (Ho + 1) * (Wo + 1)
    out = torch.zeros(rows, cout, device="cuda")
    lib.gemm(a, wp, m=rows, kc=cin, taps=taps, a_planes=4, out_f32=out)
    got = out.view(bsz, Ho + 1, Wo + 1, cout)[:, 1:, 1:].permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(x.float().cpu(), w.float().cpu(), stride=2, padding=1).cuda()
    assert _rel(got, ref) < 2e-5


def test_gemm_gelu_bwd_epilogue():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(31)
    m, n, k = 512, 256, 128
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    pre = torch.randn(m, n, device="cuda", generator=g).half()
    o16 = torch.zeros(m, n, device="cuda").half()
    lib.gemm(a, b, act=lib.ACT_GELU_BWD, aux=pre, out_f16=o16)
    p = pre.float().requires_grad_(True)
    torch.nn.functional.gelu(p).sum().backward()
    ref = (a.float() @ b.float().t()) * p.grad
    assert _rel(o16, ref) < 1e-3


@pytest.mark.parametrize("m,n,k", [(512, 256, 128), (1000, 3136, 200), (130, 200, 72)])
def test_gemm_gelu_saves_derivative_and_mul_aux_consumes_it(m, n, k):
    """Training forward of fc1 (fv.py:401-404): one epilogue emits GELU(z) and gelu'(z) (pre_is_grad); the fc2
    data-gradient GEMM multiplies by the saved derivative (FVIT_ACT_MUL_AUX) and sums the rounded output per
    column (fc1 bias gradient). The GELU output must be bit-identical to the plain GELU epilogue."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n)
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    bias = torch.randn(n, device="cuda", generator=g)
    h16 = torch.zeros(m, n, device="cuda").half()
    g16 = torch.zeros(m, n, device="cuda").half()
    lib.gemm(a, b, act=lib.ACT_GELU, col_shift=bias, out_f16=h16, out_pre16=g16, pre_is_grad=True)
    plain = torch.zeros(m, n, device="cuda").half()
    pre16 = torch.zeros(m, n, device="cuda").half()
    lib.gemm(a, b, act=lib.ACT_GELU, col_shift=bias, out_f16=plain, out_pre16=pre16)
    assert torch.equal(h16, plain)
    z = (a.double() @ b.double().t() + bias.double()).requires_grad_(True)
    torch.nn.functional.gelu(z).sum().backward()
    assert _rel(pre16, z.detach()) < 1e-3          # without the flag out_pre16 still holds the pre-activation
    assert (g16.double() - z.grad).abs().max().item() < 1.5e-3   # |gelu'| <= 1.13, fp16 rounding + A-S erf
    # backward: dH = (dY @ W2) * saved derivative, plus the column sums of the rounded result
    dy = torch.randn(m, 64, device="cuda", generator=g).half()
    w2 = (torch.randn(64, n, device="cuda", generator=g) * 0.1).half()      # [K = 64, n]: MN-major B operand
    dh = torch.zeros(m, n, device="cuda").half()
    one = torch.ones(1, device="cuda")
    colsum = torch.zeros(n, device="cuda")
    lib.gemm(dy, w2, b_mn=True, act=lib.ACT_MUL_AUX, aux=g16, alpha_ptr=one, out_f16=dh, out_colsum=colsum,
             out_colsum_alpha=one)
    ref = (dy.double() @ w2.double()) * g16.double()
    assert _rel(dh, ref) < 1e-3
    want = dh.double().sum(0)
    assert (colsum.double() - want).abs().max().item() <= 2e-3 * want.abs().max().item() + 1e-3


@pytest.mark.parametrize("m,n", [(512, 256), (1000, 3136), (130, 200)])
def test_gemm_output_column_sums(m, n):
    """out_colsum: per-column sum of the rounded fp16 output, scaled by a device scalar (bias gradient of the
    previous Linear taken in the epilogue of the dgrad GEMM)."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n)
    k = 192
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.1).half()   # MN-major B like a dgrad weight
    pre = torch.randn(m, n, device="cuda", generator=g).half()
    o16 = torch.zeros(m, n, device="cuda").half()
    alpha = torch.full((1,), 0.5, device="cuda")
    osum = torch.ones(n, device="cuda")        # accumulates on top of existing content
    one = torch.ones(1, device="cuda")
    lib.gemm(a, b, b_mn=True, act=lib.ACT_GELU_BWD, aux=pre, alpha_ptr=one, out_f16=o16, out_colsum=osum,
             out_colsum_alpha=alpha)
    ref = 1.0 + 0.5 * o16.float().sum(0)
    assert (osum - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3
    p = pre.float().requires_grad_(True)
    torch.nn.functional.gelu(p).sum().backward()
    assert _rel(o16, (a.float() @ b.float()) * p.grad) < 1e-3


# ------------------------------------------------------------------------------------------------------------
# cta_group=2 requests (CTA-pair tiles where the hardware has them; one CTA per 128-row tile on sm_90a): same
# contract and results as the default launch.
@pytest.mark.parametrize("m,n,k", [(256, 64, 64), (300, 200, 136), (1000, 1000, 520), (129, 784, 200), (4096, 768, 256),
                                   (53 * 512, 784, 784), (128 * 37 + 5, 3136, 392)])
def test_gemm_pair_nt_plain(m, n, k):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n)
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = torch.randn(n, k, device="cuda", generator=g).half()
    out = torch.full((m, n), float("nan"), device="cuda")
    lib.gemm(a, b, out_f32=out, cta_group=2)
    assert _rel(out, a.float() @ b.float().t()) < 2e-5


@pytest.mark.parametrize("tile_n", [32, 96, 160, 224, 256])
def test_gemm_pair_tile_n(tile_n):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(tile_n)
    m, n, k = 777, 400, 264
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = torch.randn(n, k, device="cuda", generator=g).half()
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(a, b, out_f32=out, tile_n=tile_n, cta_group=2)
    assert _rel(out, a.float() @ b.float().t()) < 2e-5


@pytest.mark.parametrize("a_mn,b_mn", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("m,n,k,tile_n", [(520, 392, 1000, 0), (784, 200, 3000, 0), (300, 392, 1000, 96), (300, 392, 1000, 224)])
def test_gemm_pair_mn_major(a_mn, b_mn, m, n, k, tile_n):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    A = torch.randn(m, k, device="cuda", generator=g).half()
    B = torch.randn(n, k, device="cuda", generator=g).half()
    pad8 = lambda t: torch.nn.functional.pad(t, (0, (-t.shape[1]) % 8))[:, :t.shape[1]]   # row stride multiple of 8
    a = pad8(A.t().contiguous()) if a_mn else A
    b = pad8(B.t().contiguous()) if b_mn else B
    out = torch.zeros(m, n, device="cuda")
    lib.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=out, tile_n=tile_n, cta_group=2)
    assert _rel(out, A.float() @ B.float().t()) < 2e-5


def test_gemm_pair_epilogue_stats_and_split_k():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(11)
    m, n, k = 1000, 328, 256
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.2).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.2).half()
    cs = torch.rand(n, device="cuda", generator=g) + 0.5
    sh = torch.randn(n, device="cuda", generator=g)
    cs2 = torch.rand(n, device="cuda", generator=g) + 0.5
    perm = torch.randperm(m, device="cuda", generator=g).int()
    perm[::17] = -1
    resid = torch.randn(m, n, device="cuda", generator=g)
    o32 = torch.full((m, n), 7.0, device="cuda")
    o16 = torch.full((m, n), 7.0, device="cuda").half()
    lib.gemm(a, b, alpha=0.5, col_scale=cs, col_shift=sh, act=lib.ACT_GELU, col_scale2=cs2, resid=resid, row_map=perm,
             out_f32=o32, out_f16=o16, cta_group=2)
    val = torch.nn.functional.gelu((a.float() @ b.float().t()) * 0.5 * cs + sh) * cs2
    ref = torch.full((m, n), 7.0, device="cuda")
    keep = perm >= 0
    idx = perm[keep].long()
    ref[idx] = val[keep] + resid[idx]
    assert _rel(o32, ref) < 2e-5 and _rel(o16, ref) < 1e-3
    # BatchNorm statistics in the epilogue
    rm = torch.arange(m, device="cuda").int()
    rm[5::9] = -1
    s1, s2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    lib.gemm(a, b, col_shift=sh, row_map=rm, out_f16=o16, col_sum=s1, col_sumsq=s2, cta_group=2)
    v = (a.float() @ b.float().t() + sh)[rm >= 0]
    assert _rel(s1, v.sum(0)) < 1e-4 and _rel(s2, (v * v).sum(0)) < 1e-4
    # split-K atomics, MN-major operands, B row offset
    kk = 5000
    A = torch.randn(kk, 256, device="cuda", generator=g).half()
    B = torch.randn(kk, 192, device="cuda", generator=g).half()
    out = torch.zeros(256, 192, device="cuda")
    lib.gemm(A, B, a_mn=True, b_mn=True, split_k=16, alpha=0.25, out_f32=out, cta_group=2)
    assert _rel(out, 0.25 * (A.float().t() @ B.float())) < 1e-4


@pytest.mark.parametrize("cout,cin,k,sk", [(392, 392, 3000, 4), (196, 196, 9000, 16), (640, 320, 700, 2)])
def test_gemm_pair_taps_in_n_weight_gradient(cout, cin, k, sk):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(k, (cin + 7) // 8 * 8, device="cuda", generator=g).half()[:, :cin]
    dz = torch.randn(k, (cout + 7) // 8 * 8, device="cuda", generator=g).half()[:, :cout]
    shifts = [-31, -30, -29, -1, 0, 1, 29, 30, 31]
    out = torch.zeros(cout, 9 * cin, device="cuda")
    lib.gemm(dz, x, a_mn=True, b_mn=True, b_taps=shifts, split_k=sk, alpha=0.5, out_f32=out, cta_group=2)
    ref = torch.zeros_like(out)
    for t, off in enumerate(shifts):
        xs = torch.zeros_like(x)
        if off >= 0:
            xs[: k - off] = x[off:]
        else:
            xs[-off:] = x[: k + off]
        ref[:, t * cin:(t + 1) * cin] = 0.5 * (dz.float().t() @ xs.float())
    assert _rel(out, ref) < 1e-4


@pytest.mark.parametrize("cin,cout,hw", [(64, 64, 14), (196, 208, 9), (128, 256, 28)])
def test_gemm_pair_conv3x3_taps(cin, cout, hw):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(cin + hw)
    bsz, H, W = 3, hw, hw + 2
    Hp, Wp = H + 2, W + 2
    ld = (cin + 7) // 8 * 8
    x = torch.randn(bsz, cin, H, W, device="cuda", generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.05).half()
    xp = torch.zeros(bsz, Hp, Wp, ld, device="cuda", dtype=torch.half)
    xp[:, 1:-1, 1:-1, :cin] = x.permute(0, 2, 3, 1)
    a = xp.view(-1, ld)[:, :cin]
    kc_pad = (cin + 63) // 64 * 64
    wp = torch.zeros(cout, 9, kc_pad, device="cuda", dtype=torch.half)
    wp[:, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    out = torch.zeros(bsz * Hp * Wp, cout, device="cuda")
    lib.gemm(a, wp.view(cout, 9 * kc_pad), kc=cin, taps=taps, out_f32=out, cta_group=2)
    got = out.view(bsz, Hp, Wp, cout)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(x.float().cpu(), w.float().cpu(), padding=1).cuda()
    assert _rel(got, ref) < 2e-5


# ------------------------------------------------------------------------------------------------------------
# Row-per-thread epilogue (EF_DIRECT): launches that only write 16-bit outputs take it when every leading dimension
# is a multiple of 16 elements; the same call on 8-element-padded views goes through the staging-tile epilogue. Both
# must produce the same bits (same arithmetic, different data movement).
def _wide(m, n, pad, gen=None, scale=1.0):
    buf = torch.zeros(m, n + pad, device="cuda", dtype=torch.float16)
    if gen is not None:
        buf[:, :n] = (torch.randn(m, n, device="cuda", generator=gen) * scale).half()
    return buf[:, :n]


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("m,n,k,tile_n", [(512, 256, 128, 0), (1000, 3136, 200, 0), (333, 784, 72, 0), (700, 400, 136, 0),
                                          (300, 208, 64, 48), (2050, 1024, 784, 160)])
@pytest.mark.parametrize("variant", ["plain", "bias_gelu", "bias_relu", "gelu_pregrad", "dgrad_alpha", "mul_aux_osum",
                                     "gelu_bwd_aux"])
def test_gemm_direct_epilogue_matches_staged(variant, m, n, k, tile_n, cg):
    lib = _lib()
    if cg == 2 and tile_n % 32:
        tile_n = 0
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    bias = torch.randn(n, device="cuda", generator=g)
    scale = torch.rand(n, device="cuda", generator=g) + 0.5
    alpha = torch.full((1,), 0.75, device="cuda")
    outs = {}
    for pad in (0, 8):   # 0: leading dimensions % 16 == 0 -> direct; 8: staged
        g2 = torch.Generator(device="cuda").manual_seed(99)
        o16 = _wide(m, n, pad)
        kw = dict(out_f16=o16, tile_n=tile_n, cta_group=cg)
        extra = []
        if variant == "bias_gelu":
            kw.update(act=lib.ACT_GELU, col_shift=bias, col_scale=scale)
        elif variant == "bias_relu":   # the eval stem's BatchNorm + ReLU
            kw.update(act=lib.ACT_RELU, col_shift=bias, col_scale=scale)
        elif variant == "gelu_pregrad":
            p16 = _wide(m, n, pad)
            kw.update(act=lib.ACT_GELU, col_shift=bias, out_pre16=p16, pre_is_grad=True)
            extra.append(p16)
        elif variant == "dgrad_alpha":
            kw.update(alpha_ptr=alpha)
        elif variant == "mul_aux_osum":
            osum = torch.zeros(n, device="cuda")
            kw.update(act=lib.ACT_MUL_AUX, aux=_wide(m, n, pad, g2), alpha_ptr=alpha, out_colsum=osum, out_colsum_alpha=alpha)
            extra.append(osum)
        elif variant == "gelu_bwd_aux":
            kw.update(act=lib.ACT_GELU_BWD, aux=_wide(m, n, pad, g2), aux_scale=scale, aux_shift=bias)
        lib.gemm(a, b, **kw)
        torch.cuda.synchronize()
        outs[pad] = [o16.clone()] + [e.clone() for e in extra]
    assert torch.equal(outs[0][0], outs[8][0])
    if variant == "gelu_pregrad":
        assert torch.equal(outs[0][1], outs[8][1])
    if variant == "mul_aux_osum":   # float atomics in a different order
        want = 0.75 * outs[0][0].double().sum(0)
        for o in (outs[0][1], outs[8][1]):
            assert (o.double() - want).abs().max().item() <= 2e-3 * want.abs().max().item() + 1e-3
    ref = a.double() @ b.double().t()
    if variant == "plain":
        assert _rel(outs[0][0], ref) < 1e-3
    if variant == "dgrad_alpha":
        assert _rel(outs[0][0], 0.75 * ref) < 1e-3
    if variant == "bias_gelu":
        assert _rel(outs[0][0], torch.nn.functional.gelu(ref * scale.double() + bias.double())) < 1.5e-3
    if variant == "bias_relu":
        assert _rel(outs[0][0], torch.relu(ref * scale.double() + bias.double())) < 1.5e-3


def test_gemm_direct_epilogue_row_map_scatter():
    """The direct epilogue writes row r of the tile to out[row_map[r]] (window-major -> raster scatter of the conv
    data gradients): permuted and dropped (-1) rows, against the staged path on a padded view."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(4)
    m, n, k = 900, 256, 96
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.1).half()
    perm = torch.randperm(m, device="cuda", generator=g).int()
    perm[::7] = -1
    res = []
    for pad in (0, 8):
        o16 = _wide(m, n, pad)
        lib.gemm(a, b, row_map=perm, out_f16=o16)
        res.append(o16.clone())
    assert torch.equal(res[0], res[1])
    ref = (a.float() @ b.float().t()).half()
    keep = perm >= 0
    assert _rel(res[0][perm[keep].long()], ref[keep]) < 1e-3
    dropped = torch.ones(m, dtype=torch.bool, device="cuda")
    dropped[perm[keep].long()] = False
    assert (res[0][dropped] == 0).all()
