"""Dense-prediction backbone interface of FasterViT (SURVEY §8 f.3) — the surface the reference's downstream copies
expose (downstream/object_detection/dino/models/dino/fastervit.py:686-846): per-level feature maps taken *before* each
level's Downsample (`xo`, fastervit.py:705-709), one BatchNorm2d `norm{i}` per requested level (fastervit.py:795-799),
`forward_raw(x) -> tuple of [B, C_i, H_i, W_i]`, `forward(tensors, mask) -> {idx: (features, mask)}` with the padding
mask resized to every level (fastervit.py:829-846), frozen stages (fastervit.py:803-815).

The hot path is the same sm_90a launch list as classification: in eval the wrapped model's eval plan is run up to the
points where the level outputs are live and `fvit_feature_map_fwd` applies the level's folded BatchNorm while
converting the token-major activation to NCHW. In train mode a levels-mode train plan (engine_train.py) applies each
norm{i} with batch statistics and differentiates through it (`fvit_feature_map_bwd`); a grad-enabled eval forward is
differentiable through the running-statistics norms (`fvit_feature_map_eval_bwd`, engine_train._EvalDenseGradFunction). Variable input sizes go through the any-res entrypoints (one cached plan per shape; the
level geometry is padded to window multiples exactly as faster_vit_any_res.py:851-867 does).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .registry import create_model


class FasterViTBackbone(nn.Module):
    def __init__(self, model_name: str = "faster_vit_0_any_res", out_indices=(0, 1, 2, 3), frozen_stages: int = -1,
                 norm_layer=nn.BatchNorm2d, **kwargs):
        super().__init__()
        kwargs.setdefault("num_classes", 0)
        self.body = create_model(model_name, **kwargs)
        dim = self.body.cfg["dim"]
        self.num_levels = len(self.body.levels)
        self.num_features = [int(dim * 2 ** i) for i in range(self.num_levels)]
        self.out_indices = tuple(out_indices)
        if norm_layer is not nn.BatchNorm2d:
            raise NotImplementedError("the per-level norm is the reference default (BatchNorm2d), folded into the "
                                      "layout-conversion kernel")
        for i in self.out_indices:
            self.add_module(f"norm{i}", nn.BatchNorm2d(self.num_features[i]))
        self.frozen_stages = frozen_stages
        self._freeze_stages()

    def _freeze_stages(self):   # fastervit.py:803-815
        if self.frozen_stages >= 0:
            self.body.patch_embed.eval()
            for p in self.body.patch_embed.parameters():
                p.requires_grad = False
        if self.frozen_stages >= 2:
            for i in range(0, self.frozen_stages - 1):
                m = self.body.levels[i]
                m.eval()
                for p in m.parameters():
                    p.requires_grad = False

    def train(self, mode: bool = True):
        super().train(mode)
        self._freeze_stages()
        return self

    def enable_input_grad(self, enabled: bool = True):
        """train-mode image gradients through the backbone (FasterViT.enable_input_grad), the frozen prefix included"""
        self.body.enable_input_grad(enabled)
        return self

    def set_train_forwards_in_flight(self, n: int = 1):
        """train-mode forwards that may await their backward at once (FasterViT.set_train_forwards_in_flight)"""
        self.body.set_train_forwards_in_flight(n)
        return self

    def forward_raw(self, x: torch.Tensor) -> tuple:
        """fastervit.py:816-827: tuple of the normalised level outputs, NCHW. Under .train() (detector fine-tuning,
        dino/backbone.py:158-160) the body runs its training launch list up to the highest requested level, every
        norm{i} normalises with batch statistics (running statistics updated) and the outputs are differentiable;
        the frozen prefix runs on running statistics and gets no parameter gradient; when x requires grad (after
        enable_input_grad()) the image gradient crosses it with a data-only backward (no weight gradients). Under .eval() every norm{i} uses its running
        statistics; with grad enabled the outputs are differentiable too (norm-eval fine-tuning, perceptual losses:
        parameter gradients, and the image gradient when x requires grad), and a forward without backward costs what
        the inference forward costs."""
        norms = [getattr(self, f"norm{i}") for i in self.out_indices]
        return self.body._get_engine().forward_levels(x, self.out_indices, norms=norms, frozen_stages=self.frozen_stages)

    def forward(self, tensors: torch.Tensor, mask: torch.Tensor | None = None) -> dict:
        """fastervit.py:829-846 without the NestedTensor wrapper type: {idx: (features, mask resized to the level)}."""
        outs = self.forward_raw(tensors)
        res = {}
        for i, o in enumerate(outs):
            m = None
            if mask is not None:
                m = torch.nn.functional.interpolate(mask[None].float(), size=o.shape[-2:]).to(torch.bool)[0]
            res[i] = (o, m)
        return res
