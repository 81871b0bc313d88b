"""Multi-scale deformable attention (Deformable DETR's MSDeformAttn, as used by DINO and MOTRv2) on sm_90a kernels.

    from fastervit_b200.deform import MSDeformAttn      # in place of models/.../ops/modules

MSDeformAttnFunction is the sampling core (libfvit_sm100.so: fvit_msda_fwd / fvit_msda_bwd), with the calling
convention of the MultiScaleDeformableAttention extension's autograd Function. MSDeformAttn is the module around it:
the same parameters, initialisation, attributes and forward as the detectors' module, the four projections staying
torch nn.Linear layers. Neither synchronises with the host, so both can be captured in a CUDA graph.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib
from .lib import FvitError

_INT32_MAX = 2 ** 31 - 1


def _check_core_args(value, spatial_shapes, level_start_index, sampling_locations, attention_weights):
    """Sizes (N, S, M, D, Lq, L, P) of a core call; raises FvitError for anything the kernel does not take."""
    named = dict(value=value, spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                 sampling_locations=sampling_locations, attention_weights=attention_weights)
    for name, t in named.items():
        if not isinstance(t, torch.Tensor):
            raise FvitError(f"MSDeformAttnFunction: {name} must be a tensor, got {type(t).__name__}")
        if not t.is_contiguous():
            raise FvitError(f"MSDeformAttnFunction: {name} must be contiguous")
    for name in ("value", "sampling_locations", "attention_weights"):
        if named[name].dtype != torch.float32:
            raise FvitError(f"MSDeformAttnFunction: {name} is {named[name].dtype}; the kernel takes float32")
    for name in ("spatial_shapes", "level_start_index"):
        if named[name].dtype != torch.int64:
            raise FvitError(f"MSDeformAttnFunction: {name} is {named[name].dtype}; expected int64")
    if value.dim() != 4:
        raise FvitError(f"MSDeformAttnFunction: value must be [N, S, M, D], got {tuple(value.shape)}")
    N, S, M, D = value.shape
    if spatial_shapes.dim() != 2 or spatial_shapes.shape[1] != 2:
        raise FvitError(f"MSDeformAttnFunction: spatial_shapes must be [L, 2], got {tuple(spatial_shapes.shape)}")
    L = spatial_shapes.shape[0]
    if L > lib.MSDA_MAX_LEVELS:
        raise FvitError(f"MSDeformAttnFunction: {L} feature levels; at most {lib.MSDA_MAX_LEVELS} are supported")
    if L < 1:
        raise FvitError("MSDeformAttnFunction: at least one feature level is needed")
    if tuple(level_start_index.shape) != (L,):
        raise FvitError(f"MSDeformAttnFunction: level_start_index must be [{L}], got {tuple(level_start_index.shape)}")
    sl = sampling_locations.shape
    if len(sl) != 6 or sl[0] != N or sl[2] != M or sl[3] != L or sl[5] != 2:
        raise FvitError(f"MSDeformAttnFunction: sampling_locations must be [N={N}, Lq, M={M}, L={L}, P, 2], "
                        f"got {tuple(sl)}")
    Lq, P = sl[1], sl[4]
    if tuple(attention_weights.shape) != (N, Lq, M, L, P):
        raise FvitError(f"MSDeformAttnFunction: attention_weights must be {(N, Lq, M, L, P)}, "
                        f"got {tuple(attention_weights.shape)}")
    if D < 1 or P < 1:
        raise FvitError(f"MSDeformAttnFunction: D={D} and P={P} must be at least 1")
    if max(N, S, M, D, Lq, P) > _INT32_MAX:
        raise FvitError("MSDeformAttnFunction: a size exceeds 2^31 - 1")
    for name, t in named.items():
        if not t.is_cuda:
            raise FvitError(f"MSDeformAttnFunction: {name} is on {t.device}; the kernel needs CUDA tensors "
                            "(there is no CPU fallback)")
        if t.device != value.device:
            raise FvitError(f"MSDeformAttnFunction: {name} is on {t.device}, value on {value.device}")
    return N, S, M, D, Lq, L, P


def _empty_work(value, sampling_locations) -> bool:
    """Nothing to sample: no query-heads, or no value pixels (every sample then reads zero)."""
    return sampling_locations.numel() == 0 or value.numel() == 0


def deterministic_scratch_sizes(N: int, S: int, M: int, D: int) -> tuple[int, int]:
    """(int64 elements of the fixed-point grad_value scratch, fp32 elements of the bound workspace) that the
    deterministic backward (fvit_msda_bwd_deterministic) of a value [N, S, M, D] takes."""
    return N * S * M * D, lib.MSDA_DET_WORKSPACE


class MSDeformAttnFunction(Function):
    """apply(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step) -> out.

    value [N, S, M, D], spatial_shapes [L, 2] int64 (H, W per level), level_start_index [L] int64,
    sampling_locations [N, Lq, M, L, P, 2] (x, y), attention_weights [N, Lq, M, L, P]; out [N, Lq, M*D]. float32,
    contiguous, CUDA. im2col_step is accepted and ignored: the kernel needs no column buffer, so any batch size works.
    The level geometry is read on the device; levels whose rows do not fit in S read as zero.

    The backward is deterministic under torch.use_deterministic_algorithms(True): grad_value is then summed in int64
    fixed point (fvit_msda_bwd_deterministic, a scratch of twice grad_value's size) instead of by float atomics, and is
    NaN throughout if attention_weights or grad_output holds an inf or NaN. The other two gradients are deterministic
    either way.
    """

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        N, S, M, D, Lq, L, P = _check_core_args(value, value_spatial_shapes, value_level_start_index,
                                                sampling_locations, attention_weights)
        out = torch.empty(N, Lq, M * D, device=value.device, dtype=torch.float32)
        if _empty_work(value, sampling_locations):
            out.zero_()
        else:
            with torch.cuda.device(value.device):
                lib.call("fvit_msda_fwd", value.data_ptr(), value_spatial_shapes.data_ptr(),
                         value_level_start_index.data_ptr(), sampling_locations.data_ptr(),
                         attention_weights.data_ptr(), N, S, M, D, Lq, L, P, out.data_ptr())
        ctx.sizes = (N, S, M, D, Lq, L, P)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                              attention_weights)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, starts, locs, weights = ctx.saved_tensors
        N, S, M, D, Lq, L, P = ctx.sizes
        grad_output = grad_output.contiguous()
        if grad_output.dtype != torch.float32:
            grad_output = grad_output.float()
        empty = _empty_work(value, locs)
        # under torch.use_deterministic_algorithms (warn_only too) grad_value is summed in fixed point, which writes
        # all of it; the default backward adds into zeros with float atomics
        deterministic = torch.are_deterministic_algorithms_enabled() and not empty
        grad_value = torch.empty_like(value) if deterministic else torch.zeros_like(value)
        if empty:
            return grad_value, None, None, torch.zeros_like(locs), torch.zeros_like(weights), None
        grad_locs = torch.empty_like(locs)
        grad_weights = torch.empty_like(weights)
        args = (value.data_ptr(), shapes.data_ptr(), starts.data_ptr(), locs.data_ptr(), weights.data_ptr(),
                grad_output.data_ptr(), N, S, M, D, Lq, L, P, grad_value.data_ptr(), grad_locs.data_ptr(),
                grad_weights.data_ptr())
        with torch.cuda.device(value.device):
            if deterministic:
                n_scratch, n_workspace = deterministic_scratch_sizes(N, S, M, D)
                scratch = torch.empty(n_scratch, dtype=torch.int64, device=value.device)
                workspace = torch.empty(n_workspace, dtype=torch.float32, device=value.device)
                lib.call("fvit_msda_bwd_deterministic", *args, scratch.data_ptr(), workspace.data_ptr())
            else:
                lib.call("fvit_msda_bwd", *args)
        return grad_value, None, None, grad_locs, grad_weights, None


class MSDeformAttn(nn.Module):
    """Multi-scale deformable attention module of Deformable DETR, in the DINO (softmax weights) and MOTRv2
    (sigmoid_attn=True) variants. Parameter names, shapes and initial values are those of the detectors' module, so
    state_dicts load both ways.

    forward(query [N, Lq, C], reference_points [N, Lq, L, 2 or 4], input_flatten [N, S, C],
            input_spatial_shapes [L, 2], input_level_start_index [L], input_padding_mask [N, S] or None) -> [N, Lq, C]

    A float16 or bfloat16 value (autocast) is sampled in float32 and the result cast back. The padding mask zeroes
    value rows out of place.
    """

    def __init__(self, d_model: int = 256, n_levels: int = 4, n_heads: int = 8, n_points: int = 4,
                 sigmoid_attn: bool = False):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError(f"d_model must be divisible by n_heads, but got {d_model} and {n_heads}")
        self.im2col_step = 64  # kept for compatibility; the kernel does not use it
        self.d_model = d_model
        self.n_levels = n_levels
        self.n_heads = n_heads
        self.n_points = n_points
        self.sigmoid_attn = sigmoid_attn
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, d_model)
        self.output_proj = nn.Linear(d_model, d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        # offsets start at zero weight and a bias that places head h's points on the ray at angle 2*pi*h/n_heads,
        # at 1, 2, ..., n_points steps of the level's pixel (largest component of the direction scaled to 1)
        nn.init.constant_(self.sampling_offsets.weight, 0.0)
        angle = torch.arange(self.n_heads, dtype=torch.float32) * (2.0 * math.pi / self.n_heads)
        direction = torch.stack([angle.cos(), angle.sin()], -1)
        direction = direction / direction.abs().max(-1, keepdim=True)[0]
        steps = torch.arange(1, self.n_points + 1, dtype=torch.float32).view(1, 1, self.n_points, 1)
        bias = direction.view(self.n_heads, 1, 1, 2).repeat(1, self.n_levels, self.n_points, 1) * steps
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(bias.reshape(-1))
        nn.init.constant_(self.attention_weights.weight, 0.0)
        nn.init.constant_(self.attention_weights.bias, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight)
        nn.init.constant_(self.value_proj.bias, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight)
        nn.init.constant_(self.output_proj.bias, 0.0)

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None):
        N, Lq, _ = query.shape
        _, S, _ = input_flatten.shape
        M, L, P = self.n_heads, self.n_levels, self.n_points
        value = self.value_proj(input_flatten)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], 0.0)
        value = value.view(N, S, M, self.d_model // M)
        offsets = self.sampling_offsets(query).view(N, Lq, M, L, P, 2)
        logits = self.attention_weights(query).view(N, Lq, M, L * P)
        weights = logits.sigmoid() if self.sigmoid_attn else F.softmax(logits, -1)
        weights = weights.view(N, Lq, M, L, P)
        if reference_points.shape[-1] == 2:
            # offsets are in pixels of each level: divide by (W, H)
            normalizer = torch.stack([input_spatial_shapes[..., 1], input_spatial_shapes[..., 0]], -1)
            locations = reference_points[:, :, None, :, None, :] + offsets / normalizer[None, None, None, :, None, :]
        elif reference_points.shape[-1] == 4:
            # offsets are in units of half the reference box, split over the points
            locations = (reference_points[:, :, None, :, None, :2]
                         + offsets / P * reference_points[:, :, None, :, None, 2:] * 0.5)
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} "
                             "instead.")
        if value.dtype in (torch.float16, torch.bfloat16):
            out = MSDeformAttnFunction.apply(value.float(), input_spatial_shapes, input_level_start_index,
                                             locations.float(), weights.float(), self.im2col_step).to(value.dtype)
        else:
            out = MSDeformAttnFunction.apply(value, input_spatial_shapes, input_level_start_index, locations,
                                             weights, self.im2col_step)
        return self.output_proj(out)


__all__ = ["MSDeformAttn", "MSDeformAttnFunction"]
