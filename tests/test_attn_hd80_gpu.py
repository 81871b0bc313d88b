"""The tensor-core attention kernels at padded head dim 80 (FasterViT-5 / -6 heads: 1280 / 16 and 2560 / 32) against
fp32 torch on the same fp16 operands, with the tolerances tests/test_attn_gpu.py uses at 32 / 64: forward 2e-3 max-rel,
log-sum-exp 2e-3, dq / dk / dv / dbias 4e-3.

Every output matrix is a NaN-filled window of a larger one: 16 columns on either side and 3 rows past the last window
must stay bitwise untouched (an 80-column head slice is two TMA boxes and two MMAs wide, and one more 16-column chunk
would reach the next head). Heads of 72 columns are zero-padded to 80; their pad columns must come out zero."""
import pytest
import torch

pytestmark = pytest.mark.gpu

HDP = 80
EDGE = 16   # sentinel columns left and right of the output window
TAIL = 3    # sentinel rows past the last window


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _operands(groups, S, heads, hd, seed, with_bias):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.zeros(groups * S, 3, heads, HDP, device="cuda")
    qkv[..., :hd] = torch.randn(groups * S, 3, heads, hd, device="cuda", generator=g)
    qkv16 = qkv.reshape(groups * S, 3 * heads * HDP).half()
    do = torch.zeros(groups * S, heads, HDP, device="cuda")
    do[..., :hd] = torch.randn(groups * S, heads, hd, device="cuda", generator=g)
    do16 = do.reshape(groups * S, heads * HDP).half()
    bias = (torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4) if with_bias else None
    return qkv16, do16, bias


class Window:
    """a [rows, cols] fp16 output inside a NaN-filled [rows + TAIL, EDGE + cols + EDGE] matrix"""

    def __init__(self, rows, cols):
        self.big = torch.full((rows + TAIL, EDGE + cols + EDGE), float("nan"), device="cuda", dtype=torch.half)
        self.rows, self.cols = rows, cols
        self.t = self.big[:rows, EDGE:EDGE + cols]

    def ptr(self):
        return self.t.data_ptr()

    def ld(self):
        return self.big.stride(0)

    def check_sentinels(self):
        b = self.big.view(torch.int16)
        nan = torch.full((), float("nan"), dtype=torch.half).view(torch.int16).item()
        assert (b[:, :EDGE] == nan).all() and (b[:, EDGE + self.cols:] == nan).all(), "columns outside the window"
        assert (b[self.rows:] == nan).all(), "rows past the last window"


def _fwd_ref(qkv16, groups, S, heads, hd, bias, scale):
    q, k, v = qkv16.float().view(groups, S, 3, heads, HDP)[..., :hd].permute(2, 0, 3, 1, 4)
    att = (q @ k.transpose(-2, -1)) * scale + (bias[None] if bias is not None else 0.0)
    out = torch.zeros(groups, S, heads, HDP, device="cuda")
    out[..., :hd] = (att.softmax(-1) @ v).permute(0, 2, 1, 3)
    lse = torch.logsumexp(att, -1).permute(0, 2, 1).reshape(groups * S, heads) * 1.4426950408889634
    return out.reshape(groups * S, heads * HDP), lse


def _bwd_ref(qkv16, do16, groups, S, heads, hd, bias, scale):
    """dqkv (head-padded) and dbias by fp32 autograd on the fp16 operands, in chunks of windows"""
    ref = torch.zeros(groups, S, 3, heads, HDP, device="cuda")
    b = bias.clone().requires_grad_(True) if bias is not None else None
    dbias = torch.zeros(heads, S, S, device="cuda")
    step = max(1, min(groups, (1 << 27) // (heads * S * S)))
    for g0 in range(0, groups, step):
        x = qkv16.float().view(groups, S, 3, heads, HDP)[g0:g0 + step, ..., :hd].clone().requires_grad_(True)
        q, k, v = x.permute(2, 0, 3, 1, 4)
        att = (q @ k.transpose(-2, -1)) * scale + (b[None] if b is not None else 0.0)
        o = (att.softmax(-1) @ v).permute(0, 2, 1, 3)
        o.backward(do16.float().view(groups, S, heads, HDP)[g0:g0 + step, ..., :hd])
        ref[g0:g0 + step, ..., :hd] = x.grad
        if b is not None:
            dbias += b.grad
            b.grad = None
    return ref.reshape(groups * S, 3 * heads * HDP), dbias


def _rel(got, want):
    return ((got.float() - want).abs().max() / want.abs().max()).item()


def _check_fwd(out, ref, hd, heads):
    assert torch.isfinite(out.t.float()).all()
    assert _rel(out.t, ref) < 2e-3, _rel(out.t, ref)
    if hd < HDP:
        assert (out.t.view(-1, heads, HDP)[..., hd:] == 0).all(), "pad columns of the output"
    out.check_sentinels()


def _check_bwd(dqkv, ref, dbias, dbias_ref, hd, heads):
    assert torch.isfinite(dqkv.t.float()).all()
    for w, nm in enumerate("qkv"):
        sl = slice(w * heads * HDP, (w + 1) * heads * HDP)
        err = _rel(dqkv.t[:, sl], ref[:, sl])
        assert err < 4e-3, (nm, err)
    if hd < HDP:
        assert (dqkv.t.view(-1, 3, heads, HDP)[..., hd:] == 0).all(), "pad columns of dqkv"
    dqkv.check_sentinels()
    if dbias is not None:
        assert _rel(dbias, dbias_ref) < 4e-3, ("dbias", _rel(dbias, dbias_ref))


# fv5 / fv6 at 224: level 2 (53-token windows, 16 heads), level 3 (49, 32 heads), carriers (16, 16 heads); group counts
# that leave a partial 128-row tile; the tile boundaries 63 / 64; heads of 72 padded to 80
TILE_SHAPES = [(53, 16, 80, 37), (49, 32, 80, 13), (16, 16, 80, 11), (63, 4, 80, 5), (64, 4, 80, 5), (53, 4, 72, 7),
               (100, 2, 80, 3), (128, 2, 80, 3)]


@pytest.mark.parametrize("S,heads,hd,groups", TILE_SHAPES)
@pytest.mark.parametrize("with_bias", [True, False])
def test_tile_forward(S, heads, hd, groups, with_bias):
    lib = _lib()
    qkv16, _, bias = _operands(groups, S, heads, hd, S * 131 + heads + hd, with_bias)
    out = Window(groups * S, heads * HDP)
    scale = hd ** -0.5
    lib.call("fvit_attn_tc_fwd", qkv16.data_ptr(), qkv16.stride(0), groups, S, heads, HDP,
             bias.data_ptr() if with_bias else None, scale, out.ptr(), out.ld())
    torch.cuda.synchronize()
    _check_fwd(out, _fwd_ref(qkv16, groups, S, heads, hd, bias, scale)[0], hd, heads)


# "bias": bias and dbias; "no_dbias": bias, dbias = NULL; "no_bias": neither
@pytest.mark.parametrize("S,heads,hd,groups", [s for s in TILE_SHAPES if s[0] <= 63])
@pytest.mark.parametrize("mode", ["bias", "no_dbias", "no_bias"])
def test_tile_backward(S, heads, hd, groups, mode):
    lib = _lib()
    qkv16, do16, bias = _operands(groups, S, heads, hd, S * 17 + heads + hd, mode != "no_bias")
    ref, dbias_ref = _bwd_ref(qkv16, do16, groups, S, heads, hd, bias, hd ** -0.5)
    dqkv = Window(groups * S, 3 * heads * HDP)
    dbias = torch.zeros(heads, S, S, device="cuda") if mode == "bias" else None
    lib.call("fvit_attn_tc_bwd", qkv16.data_ptr(), qkv16.stride(0), do16.data_ptr(), do16.stride(0), groups, S, heads,
             hd, HDP, bias.data_ptr() if bias is not None else None, hd ** -0.5, dqkv.ptr(), dqkv.ld(),
             dbias.data_ptr() if dbias is not None else None)
    torch.cuda.synchronize()
    _check_bwd(dqkv, ref, dbias, dbias_ref, hd, heads)


def test_tile_backward_stops_at_63_tokens():
    """S = 64 at hdp 80 exceeds the tile backward's shared memory: the entry point refuses it (the training plans send
    it to the key-loop kernels), and writes nothing"""
    lib = _lib()
    S, heads, groups = 64, 2, 2
    qkv16, do16, bias = _operands(groups, S, heads, 80, 5, True)
    dqkv = Window(groups * S, 3 * heads * HDP)
    with pytest.raises(lib.FvitError, match="shared memory"):
        lib.call("fvit_attn_tc_bwd", qkv16.data_ptr(), qkv16.stride(0), do16.data_ptr(), do16.stride(0), groups, S,
                 heads, 80, HDP, bias.data_ptr(), 0.1, dqkv.ptr(), dqkv.ld(), None)
    torch.cuda.synchronize()
    assert torch.isnan(dqkv.big.float()).all()


# any-res S = 148 (window 12 + 4 carriers), the 12 x 12 / 14 x 14 / 24 x 24 windows, the single-tile cases training
# plans send here (64 at hdp 80, 65 .. 128), heads of 72
LOOP_SHAPES = [(64, 4, 80, 6), (65, 4, 80, 5), (100, 3, 80, 7), (128, 2, 80, 5), (148, 16, 80, 9), (196, 8, 80, 4),
               (576, 4, 80, 2), (148, 4, 72, 5)]


@pytest.mark.parametrize("S,heads,hd,groups", LOOP_SHAPES)
@pytest.mark.parametrize("with_bias", [True, False])
def test_loop_forward_and_lse(S, heads, hd, groups, with_bias):
    if with_bias and S % 4:
        pytest.skip("the key-loop kernel stages bias rows by TMA: S % 4 == 0")
    lib = _lib()
    qkv16, _, bias = _operands(groups, S, heads, hd, S * 131 + heads + hd, with_bias)
    out = Window(groups * S, heads * HDP)
    lse = torch.full((groups * S, heads), float("nan"), device="cuda")
    scale = hd ** -0.5
    lib.call("fvit_attn_loop_fwd", qkv16.data_ptr(), qkv16.stride(0), groups, S, heads, HDP,
             bias.data_ptr() if with_bias else None, scale, out.ptr(), out.ld(), lse.data_ptr())
    torch.cuda.synchronize()
    ref, lse_ref = _fwd_ref(qkv16, groups, S, heads, hd, bias, scale)
    _check_fwd(out, ref, hd, heads)
    assert (lse - lse_ref).abs().max().item() < 2e-3 * max(1.0, lse_ref.abs().max().item())


@pytest.mark.parametrize("S,heads,hd,groups", [s for s in LOOP_SHAPES if s[0] % 4 == 0])
@pytest.mark.parametrize("mode", ["bias", "no_dbias", "no_bias"])
def test_loop_backward(S, heads, hd, groups, mode):
    """fvit_attn_loop_bwd_long after fvit_attn_loop_fwd (output and log-sum-exp rows); the fp32 dq scratch is
    NaN-filled: the kernel must not depend on its contents"""
    lib = _lib()
    qkv16, do16, bias = _operands(groups, S, heads, hd, S * 19 + heads + hd, mode != "no_bias")
    scale = hd ** -0.5
    ref, dbias_ref = _bwd_ref(qkv16, do16, groups, S, heads, hd, bias, scale)
    bptr = bias.data_ptr() if bias is not None else None
    out16 = torch.zeros(groups * S, heads * HDP, device="cuda", dtype=torch.half)
    lse = torch.zeros(groups * S, heads, device="cuda")
    lib.call("fvit_attn_loop_fwd", qkv16.data_ptr(), qkv16.stride(0), groups, S, heads, HDP, bptr, scale,
             out16.data_ptr(), out16.stride(0), lse.data_ptr())
    dqkv = Window(groups * S, 3 * heads * HDP)
    dbias = torch.zeros(heads, S, S, device="cuda") if mode == "bias" else None
    scratch = torch.full((groups * S, heads * HDP), float("nan"), device="cuda")
    lib.call("fvit_attn_loop_bwd_long", qkv16.data_ptr(), qkv16.stride(0), do16.data_ptr(), do16.stride(0),
             out16.data_ptr(), out16.stride(0), lse.data_ptr(), groups, S, heads, HDP, bptr, scale, dqkv.ptr(), dqkv.ld(),
             dbias.data_ptr() if dbias is not None else None, scratch.data_ptr(), scratch.stride(0))
    torch.cuda.synchronize()
    _check_bwd(dqkv, ref, dbias, dbias_ref, hd, heads)
