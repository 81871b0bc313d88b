"""GPU parity of the attention cores (wgmma fvit_attn_tc_fwd and the generic SIMT fvit_attn_core_fwd)
against fp32 torch math on the same fp16 q, k, v. Tolerance 2e-3 max-rel: P is rounded to fp16 before
the PV product in the tensor-core kernel (same as the reference under fp16 autocast)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv, groups, S, heads, hd, hdp, bias, scale):
    q, k, v = qkv.float().view(groups, S, 3, heads, hdp)[..., :hd].permute(2, 0, 3, 1, 4)
    attn = (q @ k.transpose(-2, -1)) * scale
    if bias is not None:
        attn = attn + bias[None]
    p = attn.softmax(-1)
    o = (p @ v).permute(0, 2, 1, 3)  # groups, S, heads, hd
    out = torch.zeros(groups, S, heads, hdp, device=qkv.device)
    out[..., :hd] = o
    return out.reshape(groups * S, heads * hdp)


@pytest.mark.parametrize("S,heads,hd,groups", [(53, 8, 32, 37), (49, 16, 32, 20), (16, 8, 32, 11), (53, 16, 49, 9),
                                               (60, 8, 32, 5), (36, 16, 32, 31), (128, 2, 64, 3), (64, 4, 24, 6),
                                               (53, 8, 32, 1024),
                                               # detection carrier attention: one sequence per image
                                               (4, 8, 32, 2), (8, 4, 16, 2), (100, 16, 49, 2), (120, 8, 32, 2)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_attn_tc_matches_torch(S, heads, hd, groups, with_bias):
    from fastervit_b200 import lib
    lib.load()
    hdp = 32 if hd <= 32 else 64
    g = torch.Generator(device="cuda").manual_seed(S * 131 + heads)
    qkv = torch.zeros(groups * S, 3, heads, hdp, device="cuda")
    qkv[..., :hd] = torch.randn(groups * S, 3, heads, hd, device="cuda", generator=g)
    qkv = qkv.reshape(groups * S, 3 * heads * hdp).half()
    bias = (torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4) if with_bias else None
    out = torch.full((groups * S, heads * hdp), float("nan"), device="cuda", dtype=torch.half)
    scale = hd ** -0.5
    lib.call("fvit_attn_tc_fwd", qkv.data_ptr(), qkv.stride(0), groups, S, heads, hdp,
             bias.data_ptr() if with_bias else None, scale, out.data_ptr(), out.stride(0))
    ref = _ref(qkv, groups, S, heads, hd, hdp, bias, scale)
    err = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    assert torch.isfinite(out.float()).all()
    assert err < 2e-3, err


@pytest.mark.parametrize("S,heads,hd,groups", [(148, 8, 32, 30), (148, 8, 32, 480), (196, 16, 49, 8), (144, 4, 24, 5),
                                               (256, 2, 64, 3), (576, 4, 49, 2), (1024, 2, 49, 1), (2304, 1, 49, 1),
                                               (132, 3, 32, 7), (68, 4, 16, 12), (104, 8, 32, 300), (128, 2, 64, 5),
                                               # detection carrier attention (one sequence per image): last key tile
                                               # of 120, 12, 124 and 128 rows
                                               (120, 8, 32, 2), (140, 4, 16, 2), (252, 16, 49, 2), (384, 8, 32, 2)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_attn_loop_matches_torch(S, heads, hd, groups, with_bias):
    """Key-loop tensor-core attention: the any-res level-2 geometry (S = 148, BASELINE config 4), the 21k windows and
    the single-tile case training plans use for 65..128-token windows, against fp32 torch on the same fp16 operands;
    also the saved log-sum-exp vector."""
    from fastervit_b200 import lib
    lib.load()
    hdp = 32 if hd <= 32 else 64
    g = torch.Generator(device="cuda").manual_seed(S * 131 + heads)
    qkv = torch.zeros(groups * S, 3, heads, hdp, device="cuda")
    qkv[..., :hd] = torch.randn(groups * S, 3, heads, hd, device="cuda", generator=g)
    qkv = qkv.reshape(groups * S, 3 * heads * hdp).half()
    bias = (torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4) if with_bias else None
    out = torch.full((groups * S, heads * hdp), float("nan"), device="cuda", dtype=torch.half)
    lse = torch.full((groups * S, heads), float("nan"), device="cuda")
    scale = hd ** -0.5
    lib.call("fvit_attn_loop_fwd", qkv.data_ptr(), qkv.stride(0), groups, S, heads, hdp,
             bias.data_ptr() if with_bias else None, scale, out.data_ptr(), out.stride(0), lse.data_ptr())
    torch.cuda.synchronize()
    ref = _ref(qkv, groups, S, heads, hd, hdp, bias, scale)
    assert torch.isfinite(out.float()).all()
    err = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < 2e-3, err
    q, k, _ = qkv.float().view(groups, S, 3, heads, hdp)[..., :hd].permute(2, 0, 3, 1, 4)
    attn = (q @ k.transpose(-2, -1)) * scale + (bias[None] if with_bias else 0.0)
    want = torch.logsumexp(attn, -1).permute(0, 2, 1).reshape(groups * S, heads) * 1.4426950408889634
    assert (lse - want).abs().max().item() < 2e-3 * max(1.0, want.abs().max().item())


# the last four exceed one CTA's shared memory as a full S x S score matrix and take the streaming (key-tiled,
# running max / sum) kernel: the windows of the 21k fine-tuned models (fv.py:1253-1418) and ragged tails
@pytest.mark.parametrize("S,heads,hd,groups", [(53, 8, 32, 7), (148, 8, 32, 3), (53, 4, 49, 5), (196, 16, 49, 2),
                                               (576, 4, 49, 1), (300, 3, 32, 2), (2304, 1, 49, 1)])
def test_attn_simt_matches_torch(S, heads, hd, groups):
    from fastervit_b200 import lib
    lib.load()
    g = torch.Generator(device="cuda").manual_seed(S + hd)
    qkv = torch.randn(groups * S, 3 * heads * hd, device="cuda", generator=g).half()
    bias = torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4
    out = torch.zeros(groups * S, heads * hd, device="cuda", dtype=torch.half)
    scale = hd ** -0.5
    lib.call("fvit_attn_core_fwd", qkv.data_ptr(), qkv.stride(0), groups, S, heads, hd, bias.data_ptr(), scale,
             out.data_ptr(), out.stride(0), None)
    ref = _ref(qkv, groups, S, heads, hd, hd, bias, scale)
    err = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < 1e-3, err


@pytest.mark.parametrize("S,heads,hd,groups", [(53, 8, 32, 37), (49, 16, 32, 20), (16, 8, 32, 11), (53, 16, 49, 9),
                                               (60, 8, 32, 5), (36, 4, 24, 13), (53, 8, 32, 1024),
                                               (4, 8, 32, 2), (8, 16, 49, 2)])   # detection carriers, per image
@pytest.mark.parametrize("tc", [True, False])
def test_attn_backward_matches_autograd(S, heads, hd, groups, tc):
    """dq, dk, dv and dbias of both backward kernels (wgmma / SIMT) vs torch autograd in fp32."""
    from fastervit_b200 import lib
    lib.load()
    hdp = 32 if hd <= 32 else 64
    g = torch.Generator(device="cuda").manual_seed(S * 17 + heads + hd)
    qkv = torch.zeros(groups * S, 3, heads, hdp, device="cuda")
    qkv[..., :hd] = torch.randn(groups * S, 3, heads, hd, device="cuda", generator=g)
    qkv16 = qkv.reshape(groups * S, 3 * heads * hdp).half()
    bias = (torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4).requires_grad_(True)
    do = torch.zeros(groups * S, heads, hdp, device="cuda")
    do[..., :hd] = torch.randn(groups * S, heads, hd, device="cuda", generator=g)
    do16 = do.reshape(groups * S, heads * hdp).half()
    scale = hd ** -0.5
    # autograd reference on the fp16-rounded operands
    x = qkv16.float().view(groups, S, 3, heads, hdp)[..., :hd].clone().requires_grad_(True)
    q, k, v = x.permute(2, 0, 3, 1, 4)
    p = ((q @ k.transpose(-2, -1)) * scale + bias[None]).softmax(-1)
    o = (p @ v).permute(0, 2, 1, 3)
    o.backward(do16.float().view(groups, S, heads, hdp)[..., :hd])
    ref = torch.zeros(groups, S, 3, heads, hdp, device="cuda")
    ref[..., :hd] = x.grad
    ref = ref.reshape(groups * S, 3 * heads * hdp)
    dqkv = torch.full((groups * S, 3 * heads * hdp), float("nan"), device="cuda", dtype=torch.half)
    dbias = torch.zeros(heads, S, S, device="cuda")
    name = "fvit_attn_tc_bwd" if tc else "fvit_attn_core_bwd"
    lib.call(name, qkv16.data_ptr(), qkv16.stride(0), do16.data_ptr(), do16.stride(0), groups, S, heads, hd, hdp,
             bias.data_ptr(), scale, dqkv.data_ptr(), dqkv.stride(0), dbias.data_ptr())
    assert torch.isfinite(dqkv.float()).all()
    for w, nm in enumerate("qkv"):
        sl = slice(w * heads * hdp, (w + 1) * heads * hdp)
        err = ((dqkv[:, sl].float() - ref[:, sl]).abs().max() / ref[:, sl].abs().max()).item()
        assert err < 4e-3, (nm, err)
    err = ((dbias - bias.grad).abs().max() / bias.grad.abs().max()).item()
    assert err < 4e-3, ("dbias", err)


@pytest.mark.parametrize("S,heads,hd,groups", [(576, 4, 24, 3), (260, 2, 32, 5), (384, 3, 49, 2), (1024, 2, 64, 2),
                                               (148, 8, 32, 9), (576, 16, 49, 150), (2304, 1, 32, 1),
                                               (68, 4, 16, 12), (104, 8, 32, 7), (128, 2, 64, 5), (100, 3, 49, 200),
                                               (196, 16, 49, 4), (144, 4, 24, 5), (256, 2, 64, 3), (132, 3, 32, 7),
                                               (148, 8, 32, 200),
                                               # detection carrier attention (one sequence per image)
                                               (120, 8, 32, 2), (140, 4, 16, 2), (252, 16, 49, 2), (384, 8, 32, 2)])
def test_attn_loop_long_backward_matches_autograd(S, heads, hd, groups):
    """fvit_attn_loop_bwd_long (any number of 128-row tiles: the any-res S = 148 windows, the 21k models' 576 / 1024 /
    2304-token windows): dq, dk,
    dv and dbias vs torch autograd in fp32. dq goes through the fp32 scratch matrix (NaN-filled here: the kernel must
    not depend on its contents)."""
    from fastervit_b200 import lib
    lib.load()
    hdp = 32 if hd <= 32 else 64
    g = torch.Generator(device="cuda").manual_seed(S * 19 + heads + hd)
    qkv = torch.zeros(groups * S, 3, heads, hdp, device="cuda")
    qkv[..., :hd] = torch.randn(groups * S, 3, heads, hd, device="cuda", generator=g)
    qkv16 = qkv.reshape(groups * S, 3 * heads * hdp).half()
    bias = (torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4).requires_grad_(True)
    do = torch.zeros(groups * S, heads, hdp, device="cuda")
    do[..., :hd] = torch.randn(groups * S, heads, hd, device="cuda", generator=g)
    do16 = do.reshape(groups * S, heads * hdp).half()
    scale = hd ** -0.5
    ref = torch.zeros(groups, S, 3, heads, hdp, device="cuda")
    dbias_ref = torch.zeros(heads, S, S, device="cuda")
    step = max(1, min(groups, (1 << 27) // (heads * S * S)))   # windows per autograd chunk (bounded score memory)
    for g0 in range(0, groups, step):
        x = qkv16.float().view(groups, S, 3, heads, hdp)[g0:g0 + step, ..., :hd].clone().requires_grad_(True)
        q, k, v = x.permute(2, 0, 3, 1, 4)
        p = ((q @ k.transpose(-2, -1)) * scale + bias[None]).softmax(-1)
        o = (p @ v).permute(0, 2, 1, 3)
        o.backward(do16.float().view(groups, S, heads, hdp)[g0:g0 + step, ..., :hd])
        ref[g0:g0 + step, ..., :hd] = x.grad
        dbias_ref += bias.grad
        bias.grad = None
    ref = ref.reshape(groups * S, 3 * heads * hdp)
    out16 = torch.zeros(groups * S, heads * hdp, device="cuda", dtype=torch.half)
    lse = torch.zeros(groups * S, heads, device="cuda")
    lib.call("fvit_attn_loop_fwd", qkv16.data_ptr(), qkv16.stride(0), groups, S, heads, hdp, bias.data_ptr(), scale,
             out16.data_ptr(), out16.stride(0), lse.data_ptr())
    dqkv = torch.full((groups * S, 3 * heads * hdp), float("nan"), device="cuda", dtype=torch.half)
    dbias = torch.zeros(heads, S, S, device="cuda")
    scratch = torch.full((groups * S, heads * hdp), float("nan"), device="cuda")
    lib.call("fvit_attn_loop_bwd_long", qkv16.data_ptr(), qkv16.stride(0), do16.data_ptr(), do16.stride(0),
             out16.data_ptr(), out16.stride(0), lse.data_ptr(), groups, S, heads, hdp, bias.data_ptr(), scale,
             dqkv.data_ptr(), dqkv.stride(0), dbias.data_ptr(), scratch.data_ptr(), scratch.stride(0))
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    for w, nm in enumerate("qkv"):
        sl = slice(w * heads * hdp, (w + 1) * heads * hdp)
        err = ((dqkv[:, sl].float() - ref[:, sl]).abs().max() / ref[:, sl].abs().max()).item()
        assert err < 4e-3, (nm, err)
    err = ((dbias - dbias_ref).abs().max() / dbias_ref.abs().max()).item()
    assert err < 4e-3, ("dbias", err)


@pytest.mark.parametrize("S,heads,hd,groups,C", [(53, 8, 32, 37, 256), (49, 16, 32, 20, 512), (16, 8, 32, 11, 256),
                                                 (53, 16, 49, 9, 784), (49, 32, 49, 6, 1568), (60, 8, 32, 5, 256),
                                                 (36, 16, 32, 31, 512), (128, 2, 64, 3, 128), (64, 4, 24, 6, 96),
                                                 (53, 8, 32, 1024, 256), (85, 4, 16, 4, 64)])
@pytest.mark.parametrize("save_qkv", [False, True])
def test_fused_hat_attention_matches_unfused_math(S, heads, hd, groups, C, save_qkv):
    """fvit_hat_attn_fwd (QKV projection + softmax(QK^T + bias) + PV in one wgmma kernel) against fp32 torch on
    the same fp16 activations / head-padded weights, with q, k, v rounded to fp16 as the kernel's operand tiles are.
    Every head is zero-padded to the kernel's 64 columns, as fv's 49-wide heads are; other padded widths raise."""
    from fastervit_b200 import lib
    lib.load()
    hdp = 64
    g = torch.Generator(device="cuda").manual_seed(S * 131 + heads + C)
    rows = groups * S
    x = torch.randn(rows, C, device="cuda", generator=g).half()
    w = torch.zeros(3, heads, hdp, C, device="cuda")
    w[:, :, :hd] = torch.randn(3, heads, hd, C, device="cuda", generator=g) * C ** -0.5
    w16 = w.reshape(3 * heads * hdp, C).half()
    qb = torch.zeros(3, heads, hdp, device="cuda")
    qb[:, :, :hd] = torch.randn(3, heads, hd, device="cuda", generator=g) * 0.2
    qb = qb.reshape(-1).contiguous()
    bias = torch.randn(heads, S, S, device="cuda", generator=g) * 2 + 4
    scale = hd ** -0.5
    out = torch.full((rows, heads * hdp), float("nan"), device="cuda", dtype=torch.half)
    qkv_out = torch.full((rows, 3 * heads * hdp), float("nan"), device="cuda", dtype=torch.half) if save_qkv else None
    lib.call("fvit_hat_attn_fwd", x.data_ptr(), x.stride(0), C, w16.data_ptr(), w16.stride(0), qb.data_ptr(), groups, S,
             heads, hdp, bias.data_ptr(), scale, out.data_ptr(), out.stride(0),
             qkv_out.data_ptr() if save_qkv else None, 3 * heads * hdp)
    torch.cuda.synchronize()
    qkv = (x.float() @ w16.float().t() + qb).half()
    ref = _ref(qkv, groups, S, heads, hd, hdp, bias, scale)
    assert torch.isfinite(out.float()).all()
    err = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < 2e-3, err
    if save_qkv:
        assert ((qkv_out.float() - qkv.float()).abs().max() / qkv.float().abs().max()).item() < 1e-3
    with pytest.raises(lib.FvitError, match="padded head dim 32"):
        lib.call("fvit_hat_attn_fwd", x.data_ptr(), x.stride(0), C, w16.data_ptr(), w16.stride(0), qb.data_ptr(), groups,
                 S, heads, 32, bias.data_ptr(), scale, out.data_ptr(), out.stride(0), None, 0)
