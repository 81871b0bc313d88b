"""The DINO detector's FasterViT backbone (downstream/object_detection/dino/models/dino/fastervit.py, `build_fastervit`)
at any input size. A drop-in for DINO's backbone.py: replace its `from .fastervit import build_fastervit` with
`from fastervit_b200.detection import build_fastervit`.

This is a different function from the classification model that `FasterViTBackbone` wraps, and checkpoints fine-tuned
with DINO were trained with it:
  * the window-token positional MLP sees its ws x ws grid shifted and scaled by (ws*ws) // 2, not ws // 2;
  * the carrier grid follows the input: each padded level map of nwh x nww windows gets cs*nwh x cs*nww carrier tokens,
    pooled with kernel / stride computed from the map at run time; their positional MLP sees that grid scaled by
    (hg*wg) // 2;
  * the tokenizer returns the pooled NCHW map reinterpreted as [hg*wg, C] tokens without a permute;
  * the carrier attention bias is the build-time table (res x res, res = 4 for the 224 configs) padded at the top-left
    by S_ct - res^2 zeros, or cropped there when the grid has fewer carriers than the table;
  * every level, the convolutional ones included, runs on its map zero-padded to a multiple of the window and crops.
The engine derives this geometry per input shape (engine.token_geometry); one plan is cached per shape, at most
`plan_cache_size` of them (default 2), least recently used first out.

Deviations from the reference, on purpose:
  * buffers keep their construction shapes: the reference reassigns the carrier `relative_bias` buffers to the last
    input's shape, after which its own state_dict no longer loads into a fresh model; here the per-shape positional
    tables live in the plans and checkpoints always round-trip;
  * `frozen_stages >= 2` freezes the levels (the reference raises there: it names a `self.network` that does not exist);
  * `train()` / `eval()` return the module (the reference's `train()` returns None);
  * `forward_raw` returns NCHW maps (the reference permutes them).
Train mode runs the levels-mode training plans (batch-statistics norm{i}, running-statistics updates, DropPath, the
frozen prefix, parameter gradients). Eval mode is inference: a grad-enabled eval forward, deploy mode and dropout raise
FvitError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lib as L
from .configs import _21K, _FAMILY
from .model import FasterViT

DEFAULT_PLAN_CACHE_SIZE = 2


def _det_configs() -> dict:
    cfgs = {}
    for sfx in "01234":
        depths, heads, dim, in_dim, _, ls, _, _ = _FAMILY[sfx]
        c = dict(depths=depths, num_heads=heads, window_size=[7, 7, 7, 7], dim=dim, ct_size=2, in_dim=in_dim,
                 mlp_ratio=4, drop_path_rate=0.1, hat=[False, False, True, False])
        if ls is not None:
            c["layer_scale"] = ls
        cfgs[f"faster_vit_{sfx}_224"] = c
    depths, heads, dim, in_dim, _, ls, _, _ = _FAMILY["4"]
    for res_name in ("224", "384", "512"):
        cfgs[f"faster_vit_4_21k_{res_name}"] = dict(
            depths=depths, num_heads=heads, window_size=list(_21K[res_name][1]), dim=dim, ct_size=2, in_dim=in_dim,
            mlp_ratio=4, drop_path_rate=0.1, layer_scale=ls, hat=[False, False, False, False])
    return cfgs


DET_CONFIGS = _det_configs()


class FasterViTDet(FasterViT):
    """Module tree, state_dict and interface of the detection copy's `FasterViT`: the classification model's
    patch_embed / levels (no norm, avgpool, head) plus one BatchNorm2d `norm{i}` per out index."""
    carriers_from_input = True   # engine.token_geometry: carrier grid, pooling and positional tables from the input

    def __init__(self, dim, in_dim, depths, ct_size, mlp_ratio, num_heads, window_size=(7, 7, 7, 7), resolution=224,
                 drop_path_rate=0.2, in_chans=3, num_classes=1000, qkv_bias=True, qk_scale=None, drop_rate=0.,
                 attn_drop_rate=0., layer_scale=None, layer_scale_conv=None, hat=(False, False, True, False),
                 do_propagation=False, norm_layer=nn.BatchNorm2d, out_indices=(0, 1, 2, 3), frozen_stages=-1,
                 **kwargs):
        if drop_rate or attn_drop_rate:
            raise L.FvitError("dropout (drop_rate / attn_drop_rate) is not implemented: it is 0 in every config")
        if norm_layer is not nn.BatchNorm2d:
            raise L.FvitError("the level norms are the reference default, BatchNorm2d")
        kwargs.pop("use_checkpoint", None)
        super().__init__(dim=dim, in_dim=in_dim, depths=depths, window_size=window_size, ct_size=ct_size,
                         mlp_ratio=mlp_ratio, num_heads=num_heads, resolution=resolution, drop_path_rate=drop_path_rate,
                         in_chans=in_chans, num_classes=0, qkv_bias=qkv_bias, qk_scale=qk_scale,
                         layer_scale=layer_scale, layer_scale_conv=layer_scale_conv, hat=hat,
                         do_propagation=do_propagation, any_res=False, **kwargs)
        del self.norm, self.avgpool, self.head
        self.num_classes = num_classes
        self.num_levels = len(depths)
        self.num_features = [int(dim * 2 ** i) for i in range(self.num_levels)]
        self.out_indices = tuple(out_indices)
        for i in self.out_indices:
            self.add_module(f"norm{i}", nn.BatchNorm2d(self.num_features[i]))
        self.plan_cache_size = DEFAULT_PLAN_CACHE_SIZE
        self.frozen_stages = frozen_stages
        self._freeze_stages()

    def set_plan_cache_size(self, n: int | None):
        """At most n input shapes keep a plan (launch list, activation buffers, packed weights) on the device; the least
        recently used one is dropped first. None: unbounded."""
        if n is not None and int(n) < 1:
            raise L.FvitError("plan_cache_size must be >= 1 (or None for unbounded)")
        self.plan_cache_size = None if n is None else int(n)
        if self._engine is not None:
            self._engine.trim_plans()
        return self

    def _freeze_stages(self):   # dino/models/dino/fastervit.py:801-812, levels in place of the missing `network`
        if self.frozen_stages >= 0:
            self.patch_embed.eval()
            for p in self.patch_embed.parameters():
                p.requires_grad = False
        if self.frozen_stages >= 2:
            for i in range(0, self.frozen_stages - 1):
                m = self.levels[i]
                m.eval()
                for p in m.parameters():
                    p.requires_grad = False

    def train(self, mode: bool = True):
        super().train(mode)
        self._freeze_stages()
        return self

    def switch_to_deploy(self):
        raise L.FvitError("deploy mode caches positional tables of one input shape; the detection backbone derives "
                          "them per input")

    def forward_raw(self, x: torch.Tensor) -> tuple:
        """Tuple of the normed level maps [B, C_i, H_i, W_i] for i in out_indices, each level's output before its
        Downsample through norm{i}. Under .train() (DINO fine-tuning): batch-statistics norms and BatchNorms (running
        statistics updated), stochastic depth, the frozen prefix on running statistics, differentiable outputs; under
        .eval(): running statistics, inference (torch.no_grad())."""
        if not self.training and torch.is_grad_enabled() and (
                x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise L.FvitError("the detection backbone has no eval-mode gradients: train it under .train(), or run eval "
                              "under torch.no_grad() (or with every parameter frozen)")
        if any(getattr(m, "deploy", False) for m in self.modules()):
            raise L.FvitError("deploy mode is not supported by the detection backbone")
        norms = [self._level_norm(i) for i in self.out_indices]
        return self._get_engine().forward_levels(x, self.out_indices, norms=norms, frozen_stages=self.frozen_stages)

    def _level_norm(self, i: int) -> nn.Module:
        return getattr(self, f"norm{i}")

    def forward(self, tensor_list):
        """{k: type(tensor_list)(map_k, mask resized to map_k)} for the k-th out index
        (dino/models/dino/fastervit.py:827-846); `tensor_list` is anything with .tensors and .mask."""
        outs = self.forward_raw(tensor_list.tensors)
        m = tensor_list.mask
        if m is None:
            raise L.FvitError("the input's mask is None: DINO passes the padding mask of the batch")
        res = {}
        for k, o in enumerate(outs):
            mask = torch.nn.functional.interpolate(m[None].float(), size=o.shape[-2:]).to(torch.bool)[0]
            res[k] = type(tensor_list)(o, mask)
        return res


def build_fastervit(modelname: str, **kw) -> FasterViTDet:
    """dino/models/dino/fastervit.py:853-960: one of the eight detection configs, keyword overrides on top (extra
    keywords such as use_checkpoint are accepted and ignored)."""
    if modelname not in DET_CONFIGS:
        raise L.FvitError(f"unknown detection backbone {modelname!r}; one of {sorted(DET_CONFIGS)}")
    cfg = dict(DET_CONFIGS[modelname])
    cfg.update(kw)
    return FasterViTDet(**cfg)
