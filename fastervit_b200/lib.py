"""ctypes binding of libfvit_sm100.so (see include/fvit.h for the C ABI).

The product path has no fallback: if the library is missing, or a call is made without a CUDA
device, this module raises. PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent
import os as _os

LIB_PATH = Path(_os.environ["FVIT_LIB"]) if _os.environ.get("FVIT_LIB") else _PKG / "libfvit_sm100.so"   # (A/B builds)

ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_BWD, ACT_RELU_BWD, ACT_MUL_AUX = 0, 1, 2, 3, 4, 5


class FvitError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("a_rows", C.c_int64), ("lda", C.c_int64), ("a_plane_stride", C.c_int64),
        ("a_planes", C.c_int32), ("a_mn_major", C.c_int32),
        ("b", C.c_void_p), ("b_rows", C.c_int64), ("ldb", C.c_int64),
        ("b_mn_major", C.c_int32), ("bf16", C.c_int32),
        ("m", C.c_int32), ("n", C.c_int32), ("kc", C.c_int32), ("ntaps", C.c_int32),
        ("tap_shift", C.c_int32 * 16), ("tap_plane", C.c_int32 * 16),
        ("a_row_off", C.c_int32), ("b_row_off", C.c_int32),
        ("split_k", C.c_int32), ("b_ntaps", C.c_int32), ("tile_n", C.c_int32),
        ("alpha", C.c_float), ("act", C.c_int32),
        ("col_scale", C.c_void_p), ("col_shift", C.c_void_p), ("col_scale2", C.c_void_p),
        ("aux", C.c_void_p), ("ld_aux", C.c_int64),
        ("resid", C.c_void_p), ("ld_resid", C.c_int64),
        ("row_map", C.c_void_p),
        ("out_f32", C.c_void_p), ("ld_out_f32", C.c_int64),
        ("out_f16", C.c_void_p), ("ld_out_f16", C.c_int64),
        ("col_sum", C.c_void_p), ("col_sumsq", C.c_void_p),
        ("alpha_ptr", C.c_void_p), ("row_scale", C.c_void_p),
        ("out_pre16", C.c_void_p), ("ld_out_pre16", C.c_int64),
        ("out_colsum", C.c_void_p), ("out_colsum_alpha", C.c_void_p),
        ("aux_scale", C.c_void_p), ("aux_shift", C.c_void_p),
        ("pre_is_grad", C.c_int32), ("cta_group", C.c_int32),
    ]


_lib = None


def load() -> C.CDLL:
    """Load the shared library (once). Raises FvitError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise FvitError(
            f"{LIB_PATH} not found: build it with `python -m fastervit_b200.csrc.build` "
            "(there is no CPU / PyTorch fallback for the FasterViT hot path)")
    lib = C.CDLL(str(LIB_PATH))
    lib.fvit_abi_version.restype = C.c_int
    lib.fvit_last_error.restype = C.c_char_p
    lib.fvit_launch_count.restype = C.c_int64
    lib.fvit_reset_launch_count.restype = None
    lib.fvit_set_sm_limit.restype = None
    lib.fvit_set_sm_limit.argtypes = [C.c_int32]
    lib.fvit_add_launch_count.restype = None
    lib.fvit_add_launch_count.argtypes = [C.c_int64]
    lib.fvit_gemm.argtypes = [C.POINTER(GemmArgs), C.c_void_p]
    lib.fvit_gemm.restype = C.c_int
    _bind_ops(lib)
    if lib.fvit_abi_version() != 1:
        raise FvitError("libfvit_sm100.so ABI version mismatch")
    _lib = lib
    return lib


def _bind_ops(lib) -> None:
    """argtypes for the non-GEMM entry points (all: scalar/pointer args + stream, int return)."""
    for name, argtypes in _OP_SIGS.items():
        fn = getattr(lib, name, None)
        if fn is None:
            raise FvitError(f"libfvit_sm100.so does not export {name}; rebuild the library")
        fn.argtypes = argtypes
        fn.restype = C.c_int


_P, _I, _L, _F, _D = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double
_OP_SIGS: dict[str, list] = {
    "fvit_cast_pad_f16": [_P, _L, _P, _L, _I, _I, _I, _P],
    "fvit_pack_conv3x3_f16": [_P, _P, _I, _I, _I, _I, _P],
    "fvit_pack_conv3x3_taps_f16": [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "fvit_affine_fold": [_P, _P, _I, _P, _P, _P, _P, _F, _P, _P, _P],
    "fvit_stem_conv_fwd": [_P, _L, _L, _L, _L, _I, _I, _I, _I, _P, _I, _P, _P, _I, _P, _P, _L, _P, _P, _P],
    "fvit_stem_im2col": [_P, _L, _L, _L, _L, _I, _I, _I, _I, _P, _I, _P],
    "fvit_ln_fwd": [_P, _L, _P, _I, _I, _P, _I, _I, _P, _L, _P, _P, _F, _P, _L, _P, _P, _P, _P, _L, _P],
    "fvit_attn_core_fwd": [_P, _L, _I, _I, _I, _I, _P, _F, _P, _L, _P, _P],
    "fvit_attn_tc_fwd": [_P, _L, _I, _I, _I, _I, _P, _F, _P, _L, _P],
    "fvit_hat_attn_fwd": [_P, _L, _I, _P, _L, _P, _I, _I, _I, _I, _P, _F, _P, _L, _P, _L, _P],
    "fvit_attn_loop_fwd": [_P, _L, _I, _I, _I, _I, _P, _F, _P, _L, _P, _P],
    "fvit_attn_loop_bwd_long": [_P, _L, _P, _L, _P, _L, _P, _I, _I, _I, _I, _P, _F, _P, _L, _P, _P, _L, _P],
    "fvit_cast_headpad_f16": [_P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _P],
    "fvit_vec_headpad_f32": [_P, _P, _I, _I, _I, _P],
    "fvit_colstats_f32": [_P, _L, _P, _I, _I, _P, _P, _P],
    "fvit_bn_finalize": [_P, _P, _F, _P, _P, _F, _F, _P, _P, _P, _P, _P, _P, _P, _I, _P],
    "fvit_colstats_pivot_f32": [_P, _L, _P, _I, _I, _P, _P, _P, _P],
    "fvit_bn_col_shift": [_P, _P, _I, _P, _P],
    "fvit_bn_finalize_pivot": [_P, _P, _P, _I, _F, _P, _P, _F, _F, _P, _P, _P, _P, _P, _P, _P, _I, _P],
    "fvit_affine_rows": [_P, _L, _P, _I, _I, _P, _P, _I, _P, _L, _P, _L, _P, _L, _P, _P],
    "fvit_grad_scale_init": [_P, _I, _F, _P, _P],
    "fvit_vec_mul": [_P, _I, _P, _I, _P, _I, _P],
    "fvit_pow2_norm": [_P, _I, _P, _P],
    "fvit_cast_scale_f16": [_P, _L, _P, _I, _I, _P, _P, _P, _L, _P, _P],
    "fvit_colsum": [_P, _I, _L, _P, _P, _L, _I, _I, _P, _P, _P, _P, _P],
    "fvit_group_sum": [_P, _L, _I, _I, _I, _I, _P, _P, _P],
    "fvit_branch_grad": [_P, _L, _I, _I, _P, _P, _P, _P, _L, _P, _P, _P, _L, _P, _P, _P],
    "fvit_ln_bwd": [_P, _L, _P, _P, _L, _P, _P, _I, _I, _P, _L, _P, _I, _I, _P, _P, _P, _P],
    "fvit_attn_tc_bwd": [_P, _L, _P, _L, _I, _I, _I, _I, _I, _P, _F, _P, _L, _P, _P],
    "fvit_attn_core_bwd": [_P, _L, _P, _L, _I, _I, _I, _I, _I, _P, _F, _P, _L, _P, _P],
    "fvit_unpad_heads_f32": [_P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _P, _P],
    "fvit_attn_bias_bwd": [_P, _P, _P, _I, _I, _I, _P, _P, _P],
    "fvit_cpb_mlp_bwd": [_P, _I, _P, _P, _P, _I, _P, _P, _P, _P, _P],
    "fvit_pool_bn_bwd": [_P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _L, _P, _P, _P, _P, _L, _P, _P, _P],
    "fvit_scatter_add_rows": [_P, _L, _P, _L, _P, _I, _I, _P],
    "fvit_bn_bwd": [_P, _I, _L, _P, _P, _L, _P, _I, _I, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _L, _P, _P, _P, _P, _P],
    "fvit_unpack_conv_grad": [_P, _I, _P, _I, _I, _P],
    "fvit_token_init_bwd": [_P, _L, _P, _L, _P, _P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _L, _P, _P, _P],
    "fvit_propagate_bwd": [_P, _L, _P, _L, _P, _I, _I, _P, _P, _P, _P],
    "fvit_cpb_mlp_fwd": [_P, _I, _P, _P, _P, _I, _P, _P, _P],
    "fvit_attn_bias_fwd": [_P, _P, _I, _I, _I, _P, _P],
    "fvit_token_init_fwd": [_P, _L, _P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _L, _P],
    "fvit_token_init_nchw_bwd": [_P, _L, _P, _L, _P, _P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _L, _P, _P, _P],
    "fvit_token_init_nchw_dgrad": [_P, _L, _P, _P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _L, _P],
    "fvit_token_init_nchw_fwd": [_P, _L, _P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _L, _P],
    "fvit_propagate_fwd": [_P, _L, _P, _I, _I, _P, _P],
    "fvit_pool_affine_fwd": [_P, _L, _P, _I, _I, _I, _P, _P, _P, _L, _P],
    "fvit_feature_map_fwd": [_P, _L, _P, _I, _I, _I, _P, _P, _P, _P],
    "fvit_nchw_pool_f16": [_P, _I, _I, _I, _P, _L, _P],
    # dense-prediction outputs in training (include/fvit.h "Backward of fvit_feature_map_fwd")
    "fvit_feature_map_bwd_stats": [_P, _P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P],
    "fvit_feature_map_bwd": [_P, _P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _L, _P, _P, _P],
    "fvit_grad_scale_finalize": [_P, _F, _P, _P],
    # dense-prediction outputs and forward_head in eval mode (include/fvit.h "running-statistics BatchNorm2d folded in")
    "fvit_feature_map_eval_bwd": [_P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _L, _P, _P, _P],
    # channel-LayerNorm level outputs (include/fvit.h "channel LayerNorm")
    "fvit_feature_map_ln_fwd": [_P, _L, _P, _I, _I, _I, _P, _P, _F, _P, _P, _P, _P],
    "fvit_feature_map_ln_bwd": [_P, _P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _L, _P, _P, _P],
    "fvit_head_eval_bwd": [_P, _L, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P, _P],
    # eval-mode gradients (include/fvit.h "Eval-mode gradients")
    "fvit_bn_eval_bwd": [_P, _I, _L, _P, _P, _L, _P, _I, _I, _P, _P, _F, _P, _P, _I, _P, _P, _P, _L, _P, _P, _P, _P],
    "fvit_pool_bn_eval_bwd": [_P, _L, _P, _I, _I, _I, _P, _P, _F, _P, _P, _L, _P, _P, _L, _P, _P, _P],
    "fvit_stem_conv_dgrad": [_P, _L, _I, _I, _I, _P, _I, _P, _P, _P],
    "fvit_stem_col2im": [_P, _L, _I, _I, _I, _I, _P, _P],
    # data-only backward stages (include/fvit.h "Data-only backward")
    "fvit_bn_eval_dgrad": [_P, _I, _L, _P, _P, _L, _P, _I, _I, _P, _P, _I, _P, _P, _P, _L, _P, _P],
    "fvit_ln_dgrad": [_P, _L, _P, _P, _L, _P, _P, _I, _I, _P, _L, _P, _I, _I, _P],
    "fvit_token_init_dgrad": [_P, _L, _P, _P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _L, _P],
    # optimizer step (include/fvit.h "optimizer step on the flat gradient buffer")
    "fvit_optim_gather_f32": [_P, _I, _P, _P, _P, _P],
    "fvit_optim_sqnorm": [_P, _I, _P, _P, _P, _P],
    "fvit_optim_prepare": [_P, _I, _P, _P, _F, _F, _D, _D, _P, _P],
    "fvit_optim_adamw": [_P, _I, _P, _P, _P, _P, _P, _P, _F, _F, _F, _P, _P, _F, _P],
    "fvit_optim_lamb_stage1": [_P, _I, _P, _P, _P, _P, _P, _P, _P, _F, _F, _F, _P, _P, _P],
    "fvit_optim_lamb_stage2": [_P, _I, _P, _P, _P, _P, _P, _I, _I, _P, _P, _F, _P],
    "fvit_optim_ema": [_P, _I, _P, _P, _F, _P],
}


_weights_epoch = 0


def weights_epoch() -> int:
    return _weights_epoch


def bump_weights_epoch() -> None:
    """Called by everything that writes parameters / buffers through raw pointers (fused optimizer and EMA steps,
    train-mode BatchNorm running statistics): eval plans re-pack their fp16 operands when the epoch moved."""
    global _weights_epoch
    _weights_epoch += 1


def check(rc: int) -> None:
    if rc != 0:
        raise FvitError(load().fvit_last_error().decode())


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def launch_count() -> int:
    return int(load().fvit_launch_count())


def reset_launch_count() -> None:
    load().fvit_reset_launch_count()


def gemm(a: torch.Tensor, b: torch.Tensor, *, m: int | None = None, n: int | None = None,
         kc: int | None = None, a_mn: bool = False, b_mn: bool = False,
         taps: list[tuple[int, int]] | None = None, a_planes: int = 1, a_plane_stride: int = 0,
         a_row_off: int = 0, b_row_off: int = 0, b_taps: list[int] | None = None, split_k: int = 1,
         tile_n: int = 0,
         alpha: float = 1.0, act: int = ACT_NONE,
         col_scale=None, col_shift=None, col_scale2=None, aux=None, resid=None, row_map=None,
         out_f32=None, out_f16=None, col_sum=None, col_sumsq=None, alpha_ptr=None, row_scale=None,
         out_pre16=None, out_colsum=None, out_colsum_alpha=None, aux_scale=None,
         aux_shift=None, pre_is_grad: bool = False, cta_group: int = 0) -> None:
    """Thin functional wrapper over fvit_gemm for 2-D (strided) torch tensors.

    K-major operands are [rows, K] tensors, MN-major operands are [K, rows] tensors; only the row
    stride is taken from the tensor (the inner dimension must be contiguous).
    """
    lib = load()
    if not a.is_cuda:
        raise FvitError("fvit_gemm needs CUDA tensors (no CPU fallback)")
    assert a.dtype in (torch.float16, torch.bfloat16) and b.dtype == a.dtype
    assert a.stride(-1) == 1 and b.stride(-1) == 1
    g = GemmArgs()
    g.a = a.data_ptr()
    g.b = b.data_ptr()
    g.bf16 = 1 if a.dtype == torch.bfloat16 else 0
    g.a_mn_major = 1 if a_mn else 0
    g.b_mn_major = 1 if b_mn else 0
    a2 = a if a.dim() == 2 else a.reshape(-1, a.shape[-1]) if a_planes == 1 else a
    if a_planes > 1:
        assert a.dim() == 3
        g.a_rows, g.lda, g.a_plane_stride = a.shape[1], a.stride(1), a.stride(0)
        k_from_a, m_from_a = a.shape[2], a.shape[1]
    else:
        g.a_rows, g.lda, g.a_plane_stride = a2.shape[0], a2.stride(0), 0
        k_from_a, m_from_a = (a2.shape[0], a2.shape[1]) if a_mn else (a2.shape[1], a2.shape[0])
    g.a_planes = a_planes
    g.b_rows, g.ldb = b.shape[0], b.stride(0)
    n_from_b = b.shape[1] if b_mn else b.shape[0]
    g.m = m if m is not None else m_from_a
    g.n = n if n is not None else n_from_b
    g.kc = kc if kc is not None else k_from_a
    taps = taps or [(0, 0)]
    g.ntaps = len(taps)
    for i, (sh, pl) in enumerate(taps):
        g.tap_shift[i] = sh
        g.tap_plane[i] = pl
    g.a_row_off, g.b_row_off = a_row_off, b_row_off
    if b_taps is not None:
        g.b_ntaps = len(b_taps)
        for i, sh in enumerate(b_taps):
            g.tap_shift[i] = sh
    g.split_k, g.tile_n = split_k, tile_n
    g.alpha, g.act = alpha, act
    g.col_scale, g.col_shift, g.col_scale2 = ptr(col_scale), ptr(col_shift), ptr(col_scale2)
    if aux is not None:
        g.aux, g.ld_aux = aux.data_ptr(), aux.stride(0)
    if resid is not None:
        g.resid, g.ld_resid = resid.data_ptr(), resid.stride(0)
    g.row_map = ptr(row_map)
    if out_f32 is not None:
        g.out_f32, g.ld_out_f32 = out_f32.data_ptr(), out_f32.stride(0)
    if out_f16 is not None:
        g.out_f16, g.ld_out_f16 = out_f16.data_ptr(), out_f16.stride(0)
    g.col_sum, g.col_sumsq = ptr(col_sum), ptr(col_sumsq)
    g.alpha_ptr, g.row_scale = ptr(alpha_ptr), ptr(row_scale)
    if out_pre16 is not None:
        g.out_pre16, g.ld_out_pre16 = out_pre16.data_ptr(), out_pre16.stride(0)
    g.out_colsum, g.out_colsum_alpha = ptr(out_colsum), ptr(out_colsum_alpha)
    g.aux_scale, g.aux_shift = ptr(aux_scale), ptr(aux_shift)
    g.pre_is_grad = 1 if pre_is_grad else 0
    g.cta_group = cta_group
    check(lib.fvit_gemm(C.byref(g), stream_ptr()))


def call(name: str, *args) -> None:
    """Invoke a non-GEMM entry point; the current torch CUDA stream is appended as last argument."""
    lib = load()
    rc = getattr(lib, name)(*args, stream_ptr())
    if rc != 0:
        raise FvitError(f"{name}: {lib.fvit_last_error().decode()}")
