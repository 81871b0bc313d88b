"""Restatement of the multi-scale deformable attention core (MSDeformAttn's sampling, include/fvit.h "Multi-scale
deformable attention") as an explicit bilinear gather in plain torch: runs on CPU or CUDA, in the inputs' dtype (fp64
for the tests, fp32 for bench_deform.py), and autograd gives its gradients.

Per level l with H x W pixels, a sampling location (x, y) reads pixel-centre coordinates h = y*H - 0.5, w = x*W - 0.5;
it contributes only if -1 < h < H and -1 < w < W, and each of its four corners (floor(h) + {0, 1}, floor(w) + {0, 1})
that falls outside the map reads zero: grid_sample(mode='bilinear', padding_mode='zeros', align_corners=False).
"""
from __future__ import annotations

import torch


def ms_deform_attn_core(value: torch.Tensor, spatial_shapes, sampling_locations: torch.Tensor,
                        attention_weights: torch.Tensor, level_start_index=None) -> torch.Tensor:
    """value [N, S, M, D], spatial_shapes [L, 2] (H, W), sampling_locations [N, Lq, M, L, P, 2] (x, y),
    attention_weights [N, Lq, M, L, P] -> [N, Lq, M*D]. Levels are consecutive rows of value from
    level_start_index (default: the running sum of H*W)."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    shapes = [(int(h), int(w)) for h, w in torch.as_tensor(spatial_shapes).tolist()]
    if level_start_index is None:
        starts, acc = [], 0
        for h, w in shapes:
            starts.append(acc)
            acc += h * w
    else:
        starts = [int(s) for s in torch.as_tensor(level_start_index).tolist()]
    v = value.permute(0, 2, 1, 3)                                   # N, M, S, D
    out = value.new_zeros(N, M, Lq, D)
    for lvl, ((H, W), start) in enumerate(zip(shapes, starts)):
        if H * W == 0:
            continue
        vl = v[:, :, start:start + H * W]                           # N, M, H*W, D
        xy = sampling_locations[:, :, :, lvl].permute(0, 2, 1, 3, 4)  # N, M, Lq, P, 2
        a = attention_weights[:, :, :, lvl].permute(0, 2, 1, 3)     # N, M, Lq, P
        h = xy[..., 1] * H - 0.5
        w = xy[..., 0] * W - 0.5
        inside = (h > -1) & (w > -1) & (h < H) & (w < W)
        h0, w0 = torch.floor(h).detach(), torch.floor(w).detach()
        fh, fw = h - h0, w - w0
        for dy in (0, 1):
            for dx in (0, 1):
                hi, wi = h0 + dy, w0 + dx
                ok = inside & (hi >= 0) & (hi < H) & (wi >= 0) & (wi < W)
                wt = (fh if dy else 1 - fh) * (fw if dx else 1 - fw) * ok.to(value.dtype)
                idx = (hi.clamp(0, H - 1) * W + wi.clamp(0, W - 1)).long().reshape(N, M, Lq * P, 1)
                corner = torch.gather(vl, 2, idx.expand(-1, -1, -1, D)).view(N, M, Lq, P, D)
                out = out + ((wt * a).unsqueeze(-1) * corner).sum(3)
    return out.permute(0, 2, 1, 3).reshape(N, Lq, M * D)


def ms_deform_attn_grads(value, spatial_shapes, sampling_locations, attention_weights, grad_out,
                         level_start_index=None):
    """(out, grad_value, grad_sampling_locations, grad_attention_weights) of the core by autograd, in the inputs'
    dtype."""
    v = value.detach().clone().requires_grad_(True)
    s = sampling_locations.detach().clone().requires_grad_(True)
    a = attention_weights.detach().clone().requires_grad_(True)
    out = ms_deform_attn_core(v, spatial_shapes, s, a, level_start_index)
    gv, gs, ga = torch.autograd.grad(out, (v, s, a), grad_out)
    return out.detach(), gv, gs, ga
