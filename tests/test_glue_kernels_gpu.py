"""fp64 parity of the small "glue" entry points that the model tests reach only end to end: each call is checked
against a plain float64 torch restatement of its contract in include/fvit.h, with NaN / sentinel-filled outputs so
rows and columns outside the contract must stay untouched, at the shape edges the kernels are written around (row
counts that are not multiples of the block or vector width, maps containing -1, strides larger than C). Operands are
the fp32 / fp16 values the launch lists pass, so the tolerances cover fp32 arithmetic only (`_close` as in
test_train_ops_gpu.py)."""
import math
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_token_init.py
from _token_init import token_init_problem  # noqa: E402

pytestmark = pytest.mark.gpu


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


# ------------------------------------------------------------------------------------------ row maps and scatters
def test_scatter_add_rows_skips_minus_one_and_keeps_other_rows():
    """dst[map[r]] += src[r] for an injective map with -1 entries; strides > C; rows outside the map bitwise kept."""
    L = _L()
    g = _g(1)
    rows, C, lds, ldd, ndst = 333, 196, 204, 200, 500
    src = torch.randn(rows, lds, device="cuda", generator=g)
    dst = torch.randn(ndst, ldd, device="cuda", generator=g)
    dst0 = dst.clone()
    mp = torch.randperm(ndst, device="cuda", generator=g)[:rows].int()
    mp[::7] = -1
    L.call("fvit_scatter_add_rows", src.data_ptr(), lds, dst.data_ptr(), ldd, mp.data_ptr(), rows, C)
    torch.cuda.synchronize()
    want = dst0.double().clone()
    keep = mp >= 0
    want[mp[keep].long(), :C] += src[keep][:, :C].double()
    assert torch.equal(dst[:, C:], dst0[:, C:])
    _close(dst, want, 1e-6, "scatter")
    untouched = torch.ones(ndst, dtype=torch.bool, device="cuda")
    untouched[mp[keep].long()] = False
    assert torch.equal(dst[untouched], dst0[untouched])


@pytest.mark.parametrize("gamma", [False, True])
def test_propagate_fwd(gamma):
    """xs[r] += gamma * xs[src_map[r]] (gamma NULL = 1); rows with src_map < 0 are untouched."""
    L = _L()
    g = _g(2 + gamma)
    nW, S, ncw, C, ld = 7, 53, 4, 196, 200
    rows = nW * S
    r = torch.arange(rows, device="cuda")
    t = r % S - ncw
    src = torch.where(t >= 0, (r // S) * S + (t % ncw), torch.full_like(r, -1)).int()
    xs = torch.randn(rows, ld, device="cuda", generator=g)
    x0 = xs.clone()
    gm = torch.rand(C, device="cuda", generator=g) * 0.1 if gamma else None
    L.call("fvit_propagate_fwd", xs.data_ptr(), ld, src.data_ptr(), rows, C, None if gm is None else gm.data_ptr())
    torch.cuda.synchronize()
    want = x0.double().clone()
    v = src >= 0
    want[v, :C] += (gm.double() if gamma else 1.0) * x0[src[v].long(), :C].double()
    _close(xs, want, 1e-6, "propagate")
    assert torch.equal(xs[~v], x0[~v]) and torch.equal(xs[:, C:], x0[:, C:])


@pytest.mark.parametrize("ngroups,skip", [(5, 0), (77, 4), (40, 1)])
def test_group_sum(ngroups, skip):
    """out[t - skip] += *scalar * sum_w a[w*group + t] for skip <= t < group; ngroups > 32 takes the grid-z stride."""
    L = _L()
    g = _g(ngroups)
    group, C, lda = 53, 136, 140
    a = torch.randn(ngroups * group, lda, device="cuda", generator=g)
    out = torch.randn(group - skip, C, device="cuda", generator=g)
    o0 = out.clone()
    sc = torch.tensor([0.75], device="cuda")
    L.call("fvit_group_sum", a.data_ptr(), lda, ngroups, group, skip, C, sc.data_ptr(), out.data_ptr())
    torch.cuda.synchronize()
    want = o0.double() + 0.75 * a[:, :C].double().view(ngroups, group, C)[:, skip:].sum(0)
    _close(out, want, 2e-6, "group_sum")


# ------------------------------------------------------------------------------------------ gradient casts
@pytest.mark.parametrize("colmul,scalar,rows_list,row_scale", [(0, 0, 0, 0), (1, 1, 1, 1), (1, 0, 0, 1), (0, 1, 1, 0)])
def test_cast_scale_f16_optional_pointers(colmul, scalar, rows_list, row_scale):
    """out16[r] = half(x[rows[r]] * colmul * *scalar * row_scale[r]); a zero row_scale row; values past the fp16
    range round to inf as the cast does; padding columns up to ldo are not written."""
    L = _L()
    g = _g(10 + 8 * colmul + 4 * scalar + 2 * rows_list + row_scale)
    n, C, ldx, ldo, total = 301, 196, 200, 200, 320
    x = torch.randn(total, ldx, device="cuda", generator=g)
    rl = torch.randperm(total, device="cuda", generator=g)[:n].int() if rows_list else None
    if rows_list:
        rl[0] = 3
    cm = torch.rand(C, device="cuda", generator=g) + 0.5 if colmul else None
    sc = torch.tensor([0.5], device="cuda") if scalar else None
    rs = (torch.rand(n, device="cuda", generator=g) > 0.2).float() * 1.25 if row_scale else None
    if row_scale:
        rs[1] = 0.0
        rs[0] = 2.0
    if colmul:
        cm[:4] = 4.0
    # output row 0 (source row 3 with a row list): the SCALED values sit on the fp16 range edge (max 65504; 65519
    # rounds to 65504, the midpoint 65520 to inf); the multipliers of these elements are powers of two, so the
    # fp32 products are exact
    mult = (4.0 if colmul else 1.0) * (0.5 if scalar else 1.0) * (2.0 if row_scale else 1.0)
    x[3 if rows_list else 0, :4] = torch.tensor([70000.0, -70000.0, 65519.0, 65520.0]) / mult
    out = torch.full((n, ldo), 7.0, device="cuda").half()
    L.call("fvit_cast_scale_f16", x.data_ptr(), ldx, None if rl is None else rl.data_ptr(), n, C,
           None if cm is None else cm.data_ptr(), None if sc is None else sc.data_ptr(), out.data_ptr(), ldo,
           None if rs is None else rs.data_ptr())
    torch.cuda.synchronize()
    src = x[rl.long()] if rows_list else x[:n]
    v = src[:, :C].double()
    if colmul:
        v = v * cm.double()
    if scalar:
        v = v * 0.5
    if row_scale:
        v = v * rs.double()[:, None]
    want = v.float().half()                    # fp32 product, one rounding to fp16
    got = out[:, :C]
    fin = torch.isfinite(want)
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    _close(got[fin].float(), want[fin].float(), 1e-3, "cast")
    assert (out[:, C:] == 7.0).all()
    assert got[0, :4].tolist() == [float("inf"), float("-inf"), 65504.0, float("inf")]
    if row_scale:
        assert (got[1] == 0).all()


@pytest.mark.parametrize("rs,dbias,dgamma", [(0, 1, 1), (1, 1, 1), (1, 0, 1), (0, 1, 0), (1, 0, 0)])
def test_branch_grad_optional_pointers(rs, dbias, dgamma):
    """dz16 = half(g * colmul * *scalar * row_scale); dbias += *bias_alpha * column sum of the ROUNDED dz16 (the bias
    gradient of the Linear whose operand dz16 is); dgamma += *gamma_alpha * sum g * u16 * row_scale."""
    L = _L()
    g = _g(30 + 4 * rs + 2 * dbias + dgamma)
    rows, C, ldg = 1013, 264, 272
    gg = torch.randn(rows, ldg, device="cuda", generator=g) * 3
    cm = torch.rand(C, device="cuda", generator=g) + 0.5
    sc = torch.tensor([0.25], device="cuda")
    rsv = (torch.rand(rows, device="cuda", generator=g) > 0.3).float() / 0.7 if rs else None
    u16 = torch.randn(rows, C, device="cuda", generator=g).half() if dgamma else None
    ba, ga = torch.tensor([0.5], device="cuda"), torch.tensor([2.0], device="cuda")
    lddz = C + 16
    dz = torch.full((rows, lddz), 7.0, device="cuda").half()
    db0, dg0 = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    db, dg = db0.clone(), dg0.clone()
    L.call("fvit_branch_grad", gg.data_ptr(), ldg, rows, C, cm.data_ptr(), sc.data_ptr(),
           None if rsv is None else rsv.data_ptr(), dz.data_ptr(), lddz, ba.data_ptr(), db.data_ptr() if dbias else None,
           None if u16 is None else u16.data_ptr(), C, ga.data_ptr(), dg.data_ptr() if dgamma else None)
    torch.cuda.synchronize()
    gr = gg[:, :C].double() * (rsv.double()[:, None] if rs else 1.0)
    assert (dz[:, C:] == 7.0).all()
    dz = dz[:, :C]
    _close(dz, gr * cm.double() * 0.25, 1e-3, "dz16")
    if dbias:
        _close(db, db0.double() + 0.5 * dz.double().sum(0), 1e-5, "dbias = colsum(dz16)")
    else:
        assert torch.equal(db, db0)
    if dgamma:
        _close(dg, dg0.double() + 2.0 * (gr * u16.double()).sum(0), 1e-5, "dgamma")
    else:
        assert torch.equal(dg, dg0)


# ------------------------------------------------------------------------------------------ gradient scale scalars
def _pow2_floor(v):
    return 2.0 ** math.floor(math.log2(v))


@pytest.mark.parametrize("case", ["n2000", "zeros", "inf", "nan", "tiny", "huge", "pow2"])
def test_grad_scale_init_and_finalize(case):
    """gs = {S, 1/S}, S = 2^floor(log2(target / max|x|)) clamped to [2^-24, 2^40]; S = 1 for an all-zero or a
    non-finite maximum. fvit_grad_scale_finalize applies the same rule to a device maximum."""
    L = _L()
    n, target = 2000, 64.0
    x = torch.randn(n, device="cuda", generator=_g(7)) * 0.3
    if case == "zeros":
        x.zero_()
    elif case == "inf":
        x[1500] = float("-inf")
    elif case == "nan":
        x[1700] = float("nan")
    elif case == "tiny":
        x = x * 1e-30
    elif case == "huge":
        x = x * 1e30
    elif case == "pow2":
        x = x.clamp(-0.25, 0.25)
        x[1999] = 0.5          # max exactly 2^-1: target / max = 128, S = 128 (on the floor boundary)
    def rule(m):
        return min(max(_pow2_floor(target / m), 2.0 ** -24), 2.0 ** 40) if m > 0 and math.isfinite(m) else 1.0

    m = x.abs().max().item()
    if case == "nan":
        m = float("nan")
    S = rule(m)
    # fvit_grad_scale_init skips NaN elements (fvit.h): its S comes from the maximum of the others
    S_init = rule(x[~torch.isnan(x)].abs().max().item()) if case == "nan" else S
    gs = torch.full((2,), float("nan"), device="cuda")
    L.call("fvit_grad_scale_init", x.data_ptr(), n, target, gs.data_ptr())
    amax = torch.tensor([m], device="cuda")
    gs2 = torch.full((2,), float("nan"), device="cuda")
    L.call("fvit_grad_scale_finalize", amax.data_ptr(), target, gs2.data_ptr())
    torch.cuda.synchronize()
    if case == "pow2":
        assert S == 128.0
    if case == "nan":
        assert S == 1.0 and S_init != 1.0
    assert gs.tolist() == [S_init, 1.0 / S_init], (case, gs.tolist(), S_init)
    assert gs2.tolist() == [S, 1.0 / S], (case, gs2.tolist(), S)


@pytest.mark.parametrize("case", ["n3000", "zeros", "inf", "tiny", "pow2"])
def test_pow2_norm(case):
    """out = {s, 1/s}, s = 2^-floor(log2(max|v|)), s = 1 when the maximum is 0 or not finite; n > blockDim."""
    L = _L()
    v = torch.rand(3000, device="cuda", generator=_g(8)) * 3e-5
    if case == "zeros":
        v.zero_()
    elif case == "inf":
        v[2999] = float("inf")
    elif case == "tiny":
        v = v * 1e-30
    elif case == "pow2":
        v = v.clamp(max=2.0 ** -10)
        v[2500] = 2.0 ** -9
    m = v.abs().max().item()
    s = 2.0 ** -math.floor(math.log2(m)) if m > 0 and math.isfinite(m) else 1.0
    out = torch.full((2,), float("nan"), device="cuda")
    L.call("fvit_pow2_norm", v.data_ptr(), v.numel(), out.data_ptr())
    torch.cuda.synchronize()
    if case == "pow2":
        assert s == 512.0
    assert out.tolist() == [s, 1.0 / s], (case, out.tolist(), s)


def test_vec_mul_strided():
    """out[i] = a[i*a_stride] * b[i*b_stride] over n > one block."""
    L = _L()
    g = _g(9)
    n = 1500
    a = torch.randn(3 * n, device="cuda", generator=g)
    b = torch.randn(2 * n, device="cuda", generator=g)
    out = torch.full((n + 5,), float("nan"), device="cuda")
    L.call("fvit_vec_mul", a.data_ptr(), 3, b.data_ptr(), 2, out.data_ptr(), n)
    torch.cuda.synchronize()
    assert torch.equal(out[:n], a[::3] * b[::2])
    assert torch.isnan(out[n:]).all()


# ------------------------------------------------------------------------------------------ BatchNorm vectors
@pytest.mark.parametrize("bn,bias,ls", [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)])
def test_affine_fold_null_combinations(bn, bias, ls):
    """acc*scale + shift == ls * BN_eval(acc + bias) with any of BN / bias / layer scale NULL."""
    L = _L()
    g = _g(40 + 4 * bn + 2 * bias + ls)
    n = 197
    w, bb = torch.rand(n, device="cuda", generator=g) + 0.5, torch.randn(n, device="cuda", generator=g)
    mu, var = torch.randn(n, device="cuda", generator=g), torch.rand(n, device="cuda", generator=g) + 0.1
    bi, lsv = torch.randn(n, device="cuda", generator=g), torch.rand(n, device="cuda", generator=g) * 0.3
    sc, sh = torch.full((n,), float("nan"), device="cuda"), torch.full((n,), float("nan"), device="cuda")
    P = lambda t, on: t.data_ptr() if on else None
    L.call("fvit_affine_fold", sc.data_ptr(), sh.data_ptr(), n, P(w, bn), P(bb, bn), P(mu, bn), P(var, bn), 1e-5,
           P(bi, bias), P(lsv, ls))
    torch.cuda.synchronize()
    acc = torch.randn(5, n, dtype=torch.float64, device="cuda")
    v = acc + (bi.double() if bias else 0.0)
    if bn:
        v = (v - mu.double()) * (var.double() + 1e-5).rsqrt() * w.double() + bb.double()
    if ls:
        v = v * lsv.double()
    _close(acc * sc.double() + sh.double(), v, 2e-6, "fold")


@pytest.mark.parametrize("count", [1, 2, 4096])
def test_bn_finalize_layer_scale_and_small_counts(count):
    """scale = w*rstd*ls, shift = (b - mean*w*rstd)*ls; count = 1 keeps the unbiased running var at the (zero)
    biased var instead of dividing by zero."""
    L = _L()
    g = _g(50 + count)
    C = 196
    x = torch.randn(count, C, device="cuda", generator=g, dtype=torch.float64) * 2 + 1
    if count <= 2:   # quarter steps: the fp32 sums, squares and var = sumsq/n - mean^2 are exact (0 for count 1)
        x = (x * 4).round() / 4
    s = torch.stack([x.sum(0), (x * x).sum(0)]).float()
    w, b = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
    ls = torch.rand(C, device="cuda", generator=g) * 0.3
    rm0, rv0 = torch.randn(C, device="cuda", generator=g), torch.rand(C, device="cuda", generator=g) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    out = [torch.full((C,), float("nan"), device="cuda") for _ in range(4)]
    L.call("fvit_bn_finalize", s[0].data_ptr(), s[1].data_ptr(), float(count), w.data_ptr(), b.data_ptr(), 1e-5, 0.1,
           rm.data_ptr(), rv.data_ptr(), ls.data_ptr(), *[o.data_ptr() for o in out], C)
    torch.cuda.synchronize()
    mean, var = x.mean(0), x.var(0, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    unb = var * count / (count - 1) if count > 1 else var
    tol = 1e-4
    _close(out[0], w.double() * rstd * ls.double(), tol, "scale")
    _close(out[1], (b.double() - mean * w.double() * rstd) * ls.double(), tol, "shift")
    _close(out[2], mean, 1e-5, "mean")
    _close(out[3], rstd, tol, "rstd")
    _close(rm, 0.9 * rm0.double() + 0.1 * mean, 1e-5, "running_mean")
    _close(rv, 0.9 * rv0.double() + 0.1 * unb, tol, "running_var")


# ------------------------------------------------------------------------------------------ head / feature maps
@pytest.mark.parametrize("B,T,C,ldo", [(3, 49, 196, 200), (2, 144, 1568, 1576), (5, 35, 64, 72)])
def test_pool_affine_feature_map_nchw_pool(B, T, C, ldo):
    """fvit_pool_affine_fwd (fp16 [B, ldo]), fvit_feature_map_fwd (NCHW fp32) and fvit_nchw_pool_f16 over a row map
    into a larger token buffer; columns C..ldo of the pooled operand are not written."""
    L = _L()
    g = _g(B * T + C)
    total = B * T + 37
    xs = torch.randn(total, C, device="cuda", generator=g) * 2 + 0.5
    rmap = torch.randperm(total, device="cuda", generator=g)[:B * T].int()
    sc, sh = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
    tok = xs[rmap.long()].double().view(B, T, C)
    y = tok * sc.double() + sh.double()
    pooled = torch.full((B, ldo), 7.0, device="cuda").half()
    L.call("fvit_pool_affine_fwd", xs.data_ptr(), C, rmap.data_ptr(), B, T, C, sc.data_ptr(), sh.data_ptr(),
           pooled.data_ptr(), ldo)
    fmap = torch.full((B, C, T), float("nan"), device="cuda")
    L.call("fvit_feature_map_fwd", xs.data_ptr(), C, rmap.data_ptr(), B, T, C, sc.data_ptr(), sh.data_ptr(),
           fmap.data_ptr())
    p2 = torch.full((B, ldo), 7.0, device="cuda").half()
    L.call("fvit_nchw_pool_f16", fmap.data_ptr(), B, C, T, p2.data_ptr(), ldo)
    torch.cuda.synchronize()
    _close(pooled[:, :C], y.mean(1), 1e-3, "pool_affine")
    _close(fmap, y.permute(0, 2, 1), 2e-6, "feature_map")
    _close(p2[:, :C], fmap.double().mean(2), 1e-3, "nchw_pool")
    assert (pooled[:, C:] == 7.0).all() and (p2[:, C:] == 7.0).all()


@pytest.mark.parametrize("B", [5, 70])
def test_pool_bn_bwd_matches_autograd(B):
    """Backward of batch-statistics BatchNorm + AdaptiveAvgPool2d(1): g rows, dw, dbeta; B > 64 takes the capped
    grid of the reduce pass."""
    L = _L()
    g = _g(60 + B)
    T, C = 49, 196
    total = B * T + 11
    xs = torch.randn(total, C, device="cuda", generator=g) * 1.5 + 0.7
    rmap = torch.randperm(total, device="cuda", generator=g)[:B * T].int()
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    dpool = torch.randn(B, C, device="cuda", generator=g)
    xr = xs[rmap.long()].double().view(B, T, C).permute(0, 2, 1).reshape(B, C, 7, T // 7).clone().requires_grad_(True)
    wr = w.double().clone().requires_grad_(True)
    br = torch.zeros(C, dtype=torch.float64, device="cuda", requires_grad=True)
    y = torch.nn.functional.batch_norm(xr, None, None, wr, br, training=True, eps=1e-5)
    torch.nn.functional.adaptive_avg_pool2d(y, 1).flatten(1).backward(dpool.double())
    mean = xr.detach().mean((0, 2, 3)).float()     # kept alive until the kernels ran
    rstd = (xr.detach().var((0, 2, 3), unbiased=False) + 1e-5).rsqrt().float()
    s1, s2 = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    gbuf = torch.full((total, C), 3.0, device="cuda")
    dw, db = torch.ones(C, device="cuda"), torch.ones(C, device="cuda")
    sc = torch.tensor([0.5], device="cuda")
    L.call("fvit_pool_bn_bwd", xs.data_ptr(), C, rmap.data_ptr(), B, T, C, mean.data_ptr(), rstd.data_ptr(), w.data_ptr(), dpool.data_ptr(), C, s1.data_ptr(), s2.data_ptr(), sc.data_ptr(),
           gbuf.data_ptr(), C, dw.data_ptr(), db.data_ptr())
    torch.cuda.synchronize()
    gx = xr.grad.reshape(B, C, T).permute(0, 2, 1).reshape(B * T, C)
    _close(gbuf[rmap.long()], gx, 1e-4, "g")
    _close(dw, 1 + 0.5 * wr.grad, 1e-4, "dw")
    _close(db, 1 + 0.5 * br.grad, 1e-4, "dbeta")
    untouched = torch.ones(total, dtype=torch.bool, device="cuda")
    untouched[rmap.long()] = False
    assert (gbuf[untouched] == 3.0).all()


# ------------------------------------------------------------------------------------------ weight layouts
@pytest.mark.parametrize("transpose_io", [0, 1])
def test_pack_conv3x3_and_unpack_conv_grad(transpose_io):
    """[cout][cin][3][3] -> [rows][9][kc_pad] fp16 (transpose_io: [cin][9 flipped][cout]), padding columns zero;
    fvit_unpack_conv_grad accumulates a [cout][9*cin] (row stride ld) gradient back into the conv layout."""
    L = _L()
    g = _g(70 + transpose_io)
    cout, cin = 40, 24
    kc_pad = 64
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g)
    rows, inner = (cin, cout) if transpose_io else (cout, cin)
    dst = torch.full((rows, 9, kc_pad), 7.0, device="cuda").half()
    L.call("fvit_pack_conv3x3_f16", w.data_ptr(), dst.data_ptr(), cout, cin, kc_pad, transpose_io)
    torch.cuda.synchronize()
    if transpose_io:
        want = w.flip(2, 3).permute(1, 2, 3, 0).reshape(cin, 9, cout)
    else:
        want = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    assert torch.equal(dst[:, :, :inner], want.half())
    assert (dst[:, :, inner:] == 0).all()
    ld = 9 * cin + 8
    src = torch.randn(cout, ld, device="cuda", generator=g)
    acc = torch.randn(cout, cin, 3, 3, device="cuda", generator=g)
    a0 = acc.clone()
    L.call("fvit_unpack_conv_grad", src.data_ptr(), ld, acc.data_ptr(), cout, cin)
    torch.cuda.synchronize()
    want = a0.double() + src[:, :9 * cin].double().view(cout, 9, cin).permute(0, 2, 1).reshape(cout, cin, 3, 3)
    _close(acc, want, 1e-6, "unpack")


@pytest.mark.parametrize("transpose_io", [0, 1])
def test_pack_conv3x3_taps_parity_planes(transpose_io):
    """Explicit tap lists (no flip) of the four stride-2 parity planes: dst[r][j] = w[..][taps[j]]; kc_pad > inner."""
    L = _L()
    g = _g(80 + transpose_io)
    cout, cin, kc_pad = 32, 16, 64
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g)
    planes = [[0, 2, 6, 8], [1, 7], [3, 5], [4]]
    for taps in planes:
        rows, inner = (cin, cout) if transpose_io else (cout, cin)
        nt = len(taps)
        dst = torch.full((rows, nt, kc_pad), 7.0, device="cuda").half()
        tl = taps + [0] * (9 - nt)
        L.call("fvit_pack_conv3x3_taps_f16", w.data_ptr(), dst.data_ptr(), cout, cin, kc_pad, transpose_io, nt, *tl)
        torch.cuda.synchronize()
        wf = w.view(cout, cin, 9)[:, :, taps]          # [cout, cin, nt]
        want = wf.permute(1, 2, 0) if transpose_io else wf.permute(0, 2, 1)
        assert torch.equal(dst[:, :, :inner], want.half()), taps
        assert (dst[:, :, inner:] == 0).all()


def test_headpad_vec_and_unpad_heads_round_trip():
    """fvit_vec_headpad_f32 spreads blocks of hd to hdp with zero fill; fvit_unpad_heads_f32 (+)= *scalar * src
    without the padding, rows and columns."""
    L = _L()
    g = _g(90)
    heads, hd, hdp = 3, 49, 64
    src = torch.randn(3 * heads * hd, device="cuda", generator=g)
    dst = torch.full((3 * heads * hdp,), float("nan"), device="cuda")
    L.call("fvit_vec_headpad_f32", src.data_ptr(), dst.data_ptr(), dst.numel(), hd, hdp)
    torch.cuda.synchronize()
    blk = dst.view(-1, hdp)
    assert torch.equal(blk[:, :hd].reshape(-1), src) and (blk[:, hd:] == 0).all()
    # rows padded (qkv weight gradient [3*h*hdp, C]) -> [3*h*hd, C], accumulating with a scalar
    C = 40
    gpad = torch.randn(3 * heads * hdp, C + 4, device="cuda", generator=g)
    acc = torch.randn(3 * heads * hd, C, device="cuda", generator=g)
    a0 = acc.clone()
    sc = torch.tensor([0.5], device="cuda")
    L.call("fvit_unpad_heads_f32", gpad.data_ptr(), C + 4, acc.data_ptr(), C, 3 * heads * hdp, C, hd, hdp, 1, 0,
           sc.data_ptr())
    torch.cuda.synchronize()
    want = a0.double() + 0.5 * gpad[:, :C].double().view(-1, hdp, C)[:, :hd].reshape(-1, C)
    _close(acc, want, 1e-6, "unpad rows")
    # columns padded (proj weight gradient [C, h*hdp]) -> [C, h*hd], no scalar
    gcol = torch.randn(C, heads * hdp, device="cuda", generator=g)
    acc2 = torch.zeros(C, heads * hd + 3, device="cuda")
    L.call("fvit_unpad_heads_f32", gcol.data_ptr(), heads * hdp, acc2.data_ptr(), heads * hd + 3, C, heads * hdp, hd,
           hdp, 0, 1, None)
    torch.cuda.synchronize()
    assert torch.equal(acc2[:, :heads * hd], gcol.view(C, heads, hdp)[:, :, :hd].reshape(C, -1))
    assert (acc2[:, heads * hd:] == 0).all()


# ------------------------------------------------------------------------------------------ attention bias
@pytest.mark.parametrize("S,L_", [(49, 49), (53, 49), (148, 144), (4, 16), (8, 16), (36, 64)])
def test_attn_bias_fwd_bwd(S, L_):
    """bias[h][r][c] = 16 sigmoid(table[index[(r-ng)*L + (c-ng)]][h]) for r, c >= ng = S - L, else 0; the backward
    accumulates repeated index entries with the device scalar, carrier rows / columns contribute nothing. S < L (the
    detection backbone's carrier grid smaller than the table it was built with) is F.pad with negative amounts
    (dino/models/dino/fastervit.py:132): the bottom-right S x S block of the table, the cropped entries get no
    gradient."""
    L = _L()
    g = _g(S + L_)
    heads, ntab = 4, 2 * L_
    table = torch.randn(ntab, heads, device="cuda", generator=g)
    index = torch.randint(0, ntab, (L_ * L_,), device="cuda", generator=g, dtype=torch.int64)
    bias = torch.full((heads, S, S), float("nan"), device="cuda")
    L.call("fvit_attn_bias_fwd", table.data_ptr(), index.data_ptr(), heads, S, L_, bias.data_ptr())
    torch.cuda.synchronize()
    ng = S - L_
    td = table.double().requires_grad_(True)
    inner = 16 * torch.sigmoid(td[index].view(L_, L_, heads).permute(2, 0, 1))
    full = torch.nn.functional.pad(inner, (ng, 0, ng, 0))
    _close(bias, full.detach(), 1e-6, "bias fwd")
    if ng > 0:
        assert (bias[:, :ng] == 0).all() and (bias[:, :, :ng] == 0).all()
    else:
        assert torch.equal(full.detach(), inner.detach()[:, -ng:, -ng:])
    dbias = torch.randn(heads, S, S, device="cuda", generator=g)
    full.backward(dbias.double())
    dt = torch.randn(ntab, heads, device="cuda", generator=g)
    d0 = dt.clone()
    sc = torch.tensor([0.25], device="cuda")
    L.call("fvit_attn_bias_bwd", dbias.data_ptr(), bias.data_ptr(), index.data_ptr(), heads, S, L_, sc.data_ptr(),
           dt.data_ptr())
    torch.cuda.synchronize()
    _close(dt, d0.double() + 0.25 * td.grad, 1e-5, "bias bwd")


# ------------------------------------------------------------------------------------------ LayerNorm forward
@pytest.mark.parametrize("C", [64, 196, 784, 2048])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_ln_fwd_maps_posadd_writeback(C, eps):
    """v = x[in_map[r]] + add[r % group - skip] (carrier rows r % group < skip get no add); wb[r] = v; out[out_map[r]]
    = half(LayerNorm(v)) (out_map -1: no write); mean / rstd / xhat outputs. Some rows carry a mean of 1e3 std, which
    a one-pass variance would lose. Strides are larger than C; rows and columns outside the contract keep their
    sentinels."""
    L = _L()
    g = _g(C + int(eps * 1e7))
    group, skip, nwin = 53, 4, 5
    rows = group * nwin
    total = rows + 29
    ldx, ldo, ldwb, ldxh = C + 4, C + 8, C + 4, C + 8
    x = torch.randn(total, ldx, device="cuda", generator=g, dtype=torch.float64)
    x[::3, :C] += 1000.0                                       # large-mean rows (std ~1)
    x = x.float()
    in_map = torch.randperm(total, device="cuda", generator=g)[:rows].int()
    out_rows = rows + 11
    out_map = torch.randperm(out_rows, device="cuda", generator=g)[:rows].int()
    out_map[7::10] = -1
    add = torch.randn(group - skip, C, device="cuda", generator=g)
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.1
    out = torch.full((out_rows, ldo), 7.0, device="cuda").half()
    wb = torch.full((rows, ldwb), 7.0, device="cuda")
    xh = torch.full((rows, ldxh), 7.0, device="cuda").half()
    mean = torch.full((rows,), float("nan"), device="cuda")
    rstd = torch.full((rows,), float("nan"), device="cuda")
    L.call("fvit_ln_fwd", x.data_ptr(), ldx, in_map.data_ptr(), rows, C, add.data_ptr(), group, skip, wb.data_ptr(),
           ldwb, gamma.data_ptr(), beta.data_ptr(), eps, out.data_ptr(), ldo, out_map.data_ptr(), mean.data_ptr(),
           rstd.data_ptr(), xh.data_ptr(), ldxh)
    torch.cuda.synchronize()
    t = torch.arange(rows, device="cuda") % group
    v = x[in_map.long(), :C].double()
    has = t >= skip
    v[has] += add.double()[t[has] - skip]
    mu, var = v.mean(1), v.var(1, unbiased=False)
    rs = (var + eps).rsqrt()
    xhat = (v - mu[:, None]) * rs[:, None]
    y = xhat * gamma.double() + beta.double()
    assert torch.equal(wb[:, :C], v.float())                   # fp32 add of two fp32 values: exact
    _close(mean, mu, 1e-6, "mean")
    _close(rstd, rs, 2e-5, "rstd")                              # two-pass: exact also for the 1e3-mean rows
    _close(xh[:, :C], xhat, 2e-3, "xhat")
    keep = out_map >= 0
    _close(out[out_map[keep].long(), :C], y[keep], 2e-3, "out")
    assert (wb[:, C:] == 7.0).all() and (xh[:, C:] == 7.0).all() and (out[:, C:] == 7.0).all()
    untouched = torch.ones(out_rows, dtype=torch.bool, device="cuda")
    untouched[out_map[keep].long()] = False
    assert (out[untouched] == 7.0).all()


# ------------------------------------------------------------------------------------------ carrier tokens
# (Hp, Wp, kh, kw, sh, sw): the fv 14 x 14 / ct 2 windowing (k5 s3 -> 4 x 4), a non-square any-res map with
# non-overlapping windows, a map larger than the backward's shared-memory tile (its fallback kernel), and a DETR-size
# level-2 map on the fallback kernel whose pools overlap (one conv pixel feeds up to 3 x 4 pooled outputs)
TOKEN_INIT_CASES = [(14, 14, 5, 5, 3, 3), (10, 21, 5, 7, 5, 7), (24, 30, 6, 6, 6, 6), (35, 56, 8, 11, 3, 3)]


@pytest.mark.parametrize("Hp,Wp,kh,kw,sh,sw", TOKEN_INIT_CASES)
def test_token_init_fwd(Hp, Wp, kh, kw, sh, sw):
    """ct[ct_row_map[b, y, x]] = AvgPool_{kh x kw, sh x sw}(dwconv3x3(map) + bias), the map read through pix_map (-1:
    zero pixel); carrier rows outside ct_row_map keep their sentinels."""
    L = _L()
    B, C = 2, 40
    P = token_init_problem(_g(Hp * Wp + kh), B, Hp, Wp, C, kh, kw, sh, sw)
    ldo = C + 8
    out = torch.full((P["nct"] + 9, ldo), 7.0, device="cuda")
    L.call("fvit_token_init_fwd", P["xs"].data_ptr(), C + 4, P["pix_map"].data_ptr(), B, Hp, Wp, C, P["w"].data_ptr(),
           P["bias"].data_ptr(), kh, kw, sh, sw, P["oh"], P["ow"], P["ct_rows"].data_ptr(), out.data_ptr(), ldo)
    torch.cuda.synchronize()
    y = torch.nn.functional.conv2d(P["xmap"].cpu(), P["w"].double().cpu(), P["bias"].double().cpu(), padding=1,
                                   groups=C)
    y = torch.nn.functional.avg_pool2d(y, (kh, kw), (sh, sw))
    assert y.shape[-2:] == (P["oh"], P["ow"])
    want = y.permute(0, 2, 3, 1).reshape(-1, C)
    _close(out[P["ct_rows"].long(), :C], want, 2e-6, "ct")
    assert (out[:, C:] == 7.0).all()
    untouched = torch.ones(P["nct"] + 9, dtype=torch.bool, device="cuda")
    untouched[P["ct_rows"].long()] = False
    assert (out[untouched] == 7.0).all()


@pytest.mark.parametrize("Hp,Wp,kh,kw,sh,sw", TOKEN_INIT_CASES)
def test_token_init_bwd_non_square_and_padding_pixels(Hp, Wp, kh, kw, sh, sw):
    """TokenInitializer backward on non-square maps with pix_map = -1 pixels: gx[pix_map[p]] += d/dx (padding pixels
    write nothing), dw, dbias against autograd of the forward above."""
    L = _L()
    B, C = 2, 40
    P = token_init_problem(_g(7 * Hp * Wp + kw), B, Hp, Wp, C, kh, kw, sh, sw)
    x16 = P["xs"].half()
    xmap = torch.zeros(P["npix"], C, dtype=torch.float64, device="cuda")
    keep = ~P["pad"]
    xmap[keep] = x16[P["pix_map"][keep].long(), :C].double()
    xd = xmap.view(B, Hp, Wp, C).permute(0, 3, 1, 2).cpu().clone().requires_grad_(True)
    wd = P["w"].double().cpu().clone().requires_grad_(True)
    bd = torch.zeros(C, dtype=torch.float64, requires_grad=True)
    y = torch.nn.functional.avg_pool2d(torch.nn.functional.conv2d(xd, wd, bd, padding=1, groups=C), (kh, kw), (sh, sw))
    gct = torch.randn(B, P["oh"], P["ow"], C, device="cuda", generator=_g(3))
    y.backward(gct.double().cpu().permute(0, 3, 1, 2))
    g = torch.zeros(P["nct"] + 9, C, device="cuda")
    g[P["ct_rows"].long()] = gct.reshape(-1, C)
    gx = torch.randn(P["total"], C, device="cuda", generator=_g(4))
    gx0 = gx.clone()
    dw, db = torch.zeros(C, 9, device="cuda"), torch.zeros(C, device="cuda")
    sc = torch.tensor([0.5], device="cuda")
    L.call("fvit_token_init_bwd", g.data_ptr(), C, x16.data_ptr(), C + 4, P["pix_map"].data_ptr(),
           P["ct_rows"].data_ptr(), B, Hp, Wp, C, P["w"].data_ptr(), kh, kw, sh, sw, P["oh"], P["ow"], sc.data_ptr(),
           gx.data_ptr(), C, dw.data_ptr(), db.data_ptr())
    torch.cuda.synchronize()
    want = gx0.double().clone()
    gpix = xd.grad.permute(0, 2, 3, 1).reshape(-1, C).cuda()
    want[P["pix_map"][keep].long()] += gpix[keep]
    _close(gx, want, 1e-5, "gx")
    untouched = torch.ones(P["total"], dtype=torch.bool, device="cuda")
    untouched[P["pix_map"][keep].long()] = False
    assert torch.equal(gx[untouched], gx0[untouched])
    _close(dw, 0.5 * wd.grad.view(C, 9), 1e-4, "dw")
    _close(db, 0.5 * bd.grad, 1e-4, "dbias")


# ------------------------------------------------------------------------------------------ stem
def _stem_input(g, B, H, W, channels_last):
    x = torch.randn(B, 3, H, W, device="cuda", generator=g) * 60 + 120
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    return x


@pytest.mark.parametrize("H,W,channels_last", [(17, 23, False), (17, 23, True), (224, 224, False), (31, 8, True)])
def test_stem_im2col(H, W, channels_last):
    """out[pixel][c*9 + r*3 + s] = half(x[b][c][2oh+r-1][2ow+s-1]), zero outside the image and in columns 27..ldo;
    odd H / W, NCHW and channels-last strides."""
    L = _L()
    B, ldo = 3, 40
    x = _stem_input(_g(H * W + channels_last), B, H, W, channels_last)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = torch.full((B * Ho * Wo, ldo), 7.0, device="cuda").half()
    sb, sc, sh, sw = x.stride()
    L.call("fvit_stem_im2col", x.data_ptr(), sb, sc, sh, sw, B, 3, H, W, out.data_ptr(), ldo)
    torch.cuda.synchronize()
    cols = torch.nn.functional.unfold(x.float(), 3, padding=1, stride=2)         # [B, 27, Ho*Wo], (c, r, s) order
    want = cols.permute(0, 2, 1).reshape(-1, 27).half()
    assert torch.equal(out[:, :27], want)
    assert (out[:, 27:] == 0).all()


@pytest.mark.parametrize("channels_last,affine", [(False, True), (True, False)])
def test_stem_conv_fwd(channels_last, affine):
    """y = relu?(conv3x3 s2 p1(x) * scale + shift) as fp16 rows at out_row_map (-1: no write), and the per-channel
    sum / sum of squares of the raw convolution (train-mode BatchNorm statistics)."""
    L = _L()
    g = _g(11 + channels_last)
    B, H, W, cout, ldo = 2, 37, 30, 32, 40
    x = _stem_input(g, B, H, W, channels_last)
    w = torch.randn(cout, 3, 3, 3, device="cuda", generator=g) / 27 ** 0.5
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    npix = B * Ho * Wo
    rmap = torch.randperm(npix + 5, device="cuda", generator=g)[:npix].int()
    rmap[::9] = -1
    sc = torch.rand(cout, device="cuda", generator=g) + 0.5 if affine else None
    shf = torch.randn(cout, device="cuda", generator=g) if affine else None
    out = torch.full((npix + 5, ldo), 7.0, device="cuda").half()
    s = torch.zeros(2, cout, device="cuda")
    sb, sc_, sh, sw = x.stride()
    L.call("fvit_stem_conv_fwd", x.data_ptr(), sb, sc_, sh, sw, B, 3, H, W, w.data_ptr(), cout,
           None if sc is None else sc.data_ptr(), None if shf is None else shf.data_ptr(), 1, rmap.data_ptr(),
           out.data_ptr(), ldo, s[0].data_ptr(), s[1].data_ptr())
    torch.cuda.synchronize()
    raw = torch.nn.functional.conv2d(x.double().cpu(), w.double().cpu(), stride=2, padding=1)
    raw = raw.permute(0, 2, 3, 1).reshape(-1, cout).cuda()
    y = raw * sc.double() + shf.double() if affine else raw
    y = torch.relu(y)
    keep = rmap >= 0
    _close(out[rmap[keep].long(), :cout], y[keep], 2e-3, "out")
    _close(s[0], raw.sum(0), 1e-5, "sum")
    _close(s[1], (raw * raw).sum(0), 1e-5, "sumsq")
    assert (out[:, cout:] == 7.0).all()
    untouched = torch.ones(npix + 5, dtype=torch.bool, device="cuda")
    untouched[rmap[keep].long()] = False
    assert (out[untouched] == 7.0).all()
