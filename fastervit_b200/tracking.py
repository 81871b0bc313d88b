"""The MOTRv2 tracker's FasterViT backbone (downstream/object_tracking/motrv2/models/fastervit.py, `build_fastervit`) at
any input size. A drop-in for MOTRv2's models/backbone.py: replace its `from .fastervit import build_fastervit` with
`from fastervit_b200.tracking import build_fastervit`.

It is the detection backbone (fastervit_b200.detection: the same carrier geometry, derived per input shape) built with
the caller's norm classes:
  * `stem_norm_layer(n, eps=1e-4)` for PatchEmbed's two norms: nn.BatchNorm2d, or a frozen BatchNorm (the published
    recipe: a fixed affine from running statistics whose weight and bias are buffers; the stem convolutions still
    train);
  * `output_norm_layer(C_i)` for the level outputs: nn.BatchNorm2d, a frozen BatchNorm, or a channel LayerNorm (timm's
    LayerNorm2d, the published recipe), registered as norm0, norm1, norm2 and `norm` for level 3.
Norms are classified by what they are, not by their class (engine.norm_kind), so MOTRv2's own FrozenBatchNorm2d,
torchvision's and this module's FrozenBatchNorm2d all work; anything else raises FvitError at construction.

Deviations from the reference, on purpose, besides those fastervit_b200.detection lists:
  * `forward_raw` returns all requested levels (the reference's looks up `norm3`, which does not exist, and fails for
    index 3);
  * `train()` / `eval()` return the module (the reference's `train()` returns None).
Train mode runs the levels-mode training plans: batch-statistics BatchNorms update their running statistics, frozen
BatchNorms never change, LayerNorm weights and biases get gradients. Eval mode is inference: a grad-enabled eval forward
and deploy mode raise FvitError, as for the detection backbone.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lib as L
from .detection import DET_CONFIGS, FasterViTDet
from .engine import norm_kind
from .registry import load_state_dict_tolerant, read_checkpoint_state


def _track_configs() -> dict:
    cfgs = {k: dict(v) for k, v in DET_CONFIGS.items()}
    cfgs["faster_vit_0_224_hat_False"] = dict(cfgs["faster_vit_0_224"], hat=[False, False, False, False])
    return cfgs


TRACK_CONFIGS = _track_configs()


class FrozenBatchNorm2d(nn.Module):
    """BatchNorm2d with fixed statistics and affine, all four held as buffers (eps added before the rsqrt). A checkpoint's
    `num_batches_tracked` is dropped on load."""

    def __init__(self, n: int, eps: float = 1e-5):
        super().__init__()
        self.register_buffer("weight", torch.ones(n))
        self.register_buffer("bias", torch.zeros(n))
        self.register_buffer("running_mean", torch.zeros(n))
        self.register_buffer("running_var", torch.ones(n))
        self.eps = float(eps)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        state_dict.pop(prefix + "num_batches_tracked", None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)

    def forward(self, x):
        scale = self.weight * (self.running_var + self.eps).rsqrt()
        shift = self.bias - self.running_mean * scale
        return x * scale.reshape(1, -1, 1, 1) + shift.reshape(1, -1, 1, 1)


class FasterViTTrack(FasterViTDet):
    """Module tree, state_dict and interface of the tracking copy's `FasterViT`: the detection backbone with the
    caller's stem and output norm classes, the level-3 output norm registered as `norm`."""

    def __init__(self, stem_norm_layer=nn.BatchNorm2d, output_norm_layer=nn.BatchNorm2d, **kw):
        super().__init__(**kw)
        conv_down = self.patch_embed.conv_down
        for j in (1, 4):
            bn = stem_norm_layer(conv_down[j].num_features, eps=1e-4)
            if norm_kind(bn) not in ("bn", "frozen"):
                raise L.FvitError(f"stem norm {type(bn).__name__}: the stem takes nn.BatchNorm2d or a frozen BatchNorm "
                                  "(MOTRv2's --stem_norm_type choices)")
            conv_down[j] = bn
        for i in self.out_indices:   # (re-registered in order: the state_dict keys follow the reference's)
            delattr(self, f"norm{i}")
        for i in self.out_indices:
            norm = output_norm_layer(self.num_features[i])
            norm_kind(norm)
            self.add_module(self._norm_name(i), norm)
        self._freeze_stages()

    @staticmethod
    def _norm_name(i: int) -> str:
        return "norm" if i == 3 else f"norm{i}"

    def _level_norm(self, i: int) -> nn.Module:
        return getattr(self, self._norm_name(i))

    def _load_state_dict(self, pretrained: str, strict: bool = False):
        """motrv2/models/fastervit.py `_load_state_dict`: a checkpoint file (`state_dict` / `model` / bare dict, the
        `module.` and `encoder.` prefixes stripped), loaded tolerantly: mismatches are printed, not raised, unless
        strict. Returns (missing keys, unexpected keys)."""
        return load_state_dict_tolerant(self, read_checkpoint_state(pretrained), strict=strict)


def build_fastervit(modelname: str, stem_norm_layer, output_norm_layer, **kw) -> FasterViTTrack:
    """motrv2/models/fastervit.py:1027-1171: one of the nine tracking configs with the given norm classes, keyword
    overrides on top (extra keywords such as use_checkpoint are accepted and ignored)."""
    if modelname not in TRACK_CONFIGS:
        raise L.FvitError(f"unknown tracking backbone {modelname!r}; one of {sorted(TRACK_CONFIGS)}")
    cfg = dict(TRACK_CONFIGS[modelname])
    cfg.update(kw)
    return FasterViTTrack(stem_norm_layer=stem_norm_layer, output_norm_layer=output_norm_layer, **cfg)
