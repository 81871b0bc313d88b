"""FasterViT nn.Module whose forward/backward run on the sm_90a (H100) kernels of libfvit_sm100.so.

The module tree below exists to own the parameters and buffers under exactly the names, shapes and
dtypes of the reference `state_dict` (fastervit/models/faster_vit.py, SURVEY.md App. C), so reference
checkpoints load with strict=True and the timm harness (EMA deepcopy, DDP hooks, distribute_bn,
state_dict round trips) sees ordinary nn.Parameters. None of the leaf modules' own `forward` is ever
called: `FasterViT.forward` hands the whole parameter set to fastervit_b200.engine, which executes the
hot path as hand-written CUDA kernels. There is no PyTorch/CPU fallback — CPU tensors raise.
"""
from __future__ import annotations

import math
import numbers
from typing import Sequence

import torch
import torch.nn as nn

from .configs import MODEL_SPECS, default_cfgs


def _pair(v) -> list[int]:
    return [int(v[0]), int(v[1])] if isinstance(v, (list, tuple)) else [int(v), int(v)]


class _Holder(nn.Module):
    """A module that only owns parameters/sub-modules; computing happens in the engine."""

    def forward(self, *a, **k):  # pragma: no cover - guard rail
        raise RuntimeError(f"{type(self).__name__} is executed by fastervit_b200.engine, not called directly")


def _cpb_mlp(out_dim: int) -> nn.Sequential:
    # Linear(2,512)+ReLU+Linear(512,out,no bias)  (fv.py:223-225, 322-324)
    return nn.Sequential(nn.Linear(2, 512, bias=True), nn.ReLU(), nn.Linear(512, out_dim, bias=False))


class TokenPosEmbed(_Holder):
    """PosEmbMLPSwinv1D, rank 2 (fv.py:313-367): additive embedding from a 2->512->dim MLP."""

    def __init__(self, dim: int, seq_length: int):
        super().__init__()
        self.cpb_mlp = _cpb_mlp(dim)
        self.register_buffer("relative_bias", torch.zeros(1, seq_length, dim))
        self.seq_length = seq_length
        self.deploy = False

    def switch_to_deploy(self):
        """fv.py:336-342: stop re-deriving the embedding from the MLP; `relative_bias` (as loaded from a checkpoint
        or left by the last forward) is used as is."""
        self.deploy = True


class RelPosBias(_Holder):
    """PosEmbMLPSwinv2D (fv.py:213-310): log-spaced relative coordinate table -> per-head bias."""

    def __init__(self, window: int, num_heads: int, seq_length: int):
        super().__init__()
        self.window, self.num_heads, self.seq_length = window, num_heads, seq_length
        self.cpb_mlp = _cpb_mlp(num_heads)
        r = torch.arange(-(window - 1), window, dtype=torch.float32)
        table = torch.stack(torch.meshgrid(r, r, indexing="ij"), dim=-1).unsqueeze(0)  # 1,2w-1,2w-1,2
        table = table / (window - 1) * 8
        table = torch.sign(table) * torch.log2(table.abs() + 1.0) / math.log2(8)
        self.register_buffer("relative_coords_table", table.contiguous())
        c = torch.arange(window)
        pos = torch.stack(torch.meshgrid(c, c, indexing="ij")).flatten(1)  # 2, w*w
        rel = pos[:, :, None] - pos[:, None, :] + (window - 1)
        self.register_buffer("relative_position_index", (rel[0] * (2 * window - 1) + rel[1]).contiguous())
        self.register_buffer("relative_bias", torch.zeros(1, num_heads, seq_length, seq_length))
        self.deploy = False

    def switch_to_deploy(self):
        """fv.py:263-269: the cached `relative_bias` buffer replaces the table MLP + gather + 16*sigmoid."""
        self.deploy = True


class WindowAttention(_Holder):
    """fv.py:515-568: qkv / proj linears + relative position bias."""

    def __init__(self, dim: int, num_heads: int, qkv_bias: bool, resolution: int, seq_length: int, qk_scale=None):
        super().__init__()
        self.num_heads, self.head_dim = num_heads, dim // num_heads
        self.scale = qk_scale or self.head_dim ** -0.5     # fv.py:544
        self.resolution = resolution
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.pos_emb_funct = RelPosBias(resolution, num_heads, seq_length)


class Mlp(_Holder):
    def __init__(self, dim: int, hidden: int):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class HAT(_Holder):
    """Hierarchical attention block (fv.py:571-701; fvar.py:572-707)."""

    def __init__(self, dim, num_heads, mlp_ratio, qkv_bias, sr_ratio: Sequence[int], window_size, last,
                 layer_scale, ct_size, do_propagation, any_res: bool, qk_scale=None):
        super().__init__()
        self.window_size, self.ct_size, self.last = window_size, ct_size, last
        self.sr_ratio = list(sr_ratio)
        self.do_propagation = do_propagation
        self.has_carriers = sr_ratio[0] > 1 or sr_ratio[1] > 1
        n_ct_win = ct_size ** 2 if self.has_carriers else 0
        n_ct = n_ct_win * sr_ratio[0] * sr_ratio[1]
        hidden = int(dim * mlp_ratio)
        use_ls = layer_scale is not None and type(layer_scale) in (int, float)

        def ls():
            return nn.Parameter(layer_scale * torch.ones(dim)) if use_ls else 1

        self.pos_embed = TokenPosEmbed(dim, window_size ** 2)
        self.norm1 = nn.LayerNorm(dim)
        self.attn = WindowAttention(dim, num_heads, qkv_bias, window_size, window_size ** 2 + n_ct_win, qk_scale)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, hidden)
        self.gamma3, self.gamma4 = ls(), ls()
        if self.has_carriers:
            self.hat_norm1 = nn.LayerNorm(dim)
            self.hat_norm2 = nn.LayerNorm(dim)
            self.hat_attn = WindowAttention(dim, num_heads, qkv_bias, int(n_ct ** 0.5), n_ct, qk_scale)
            self.hat_mlp = Mlp(dim, hidden)
            # the any-res variant only has a carrier positional embedding on square grids (fvar.py:658)
            if (not any_res) or sr_ratio[0] == sr_ratio[1]:
                self.hat_pos_embed = TokenPosEmbed(dim, n_ct)
            self.gamma1, self.gamma2 = ls(), ls()


class ConvBlock(_Holder):
    """fv.py:472-512."""

    def __init__(self, dim: int, layer_scale):
        super().__init__()
        self.conv1 = nn.Conv2d(dim, dim, 3, 1, 1)
        self.norm1 = nn.BatchNorm2d(dim, eps=1e-5)
        self.conv2 = nn.Conv2d(dim, dim, 3, 1, 1)
        self.norm2 = nn.BatchNorm2d(dim, eps=1e-5)
        if layer_scale is not None and type(layer_scale) in (int, float):
            self.gamma = nn.Parameter(layer_scale * torch.ones(dim))


class Downsample(_Holder):
    """fv.py:410-440: channel LayerNorm (timm LayerNorm2d, eps 1e-6) + 3x3 stride-2 conv, no bias."""

    def __init__(self, dim: int):
        super().__init__()
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.reduction = nn.Sequential(nn.Conv2d(dim, 2 * dim, 3, 2, 1, bias=False))


class PatchEmbed(_Holder):
    """fv.py:443-469."""

    def __init__(self, in_chans: int, in_dim: int, dim: int):
        super().__init__()
        self.conv_down = nn.Sequential(
            nn.Conv2d(in_chans, in_dim, 3, 2, 1, bias=False), nn.BatchNorm2d(in_dim, eps=1e-4), nn.ReLU(),
            nn.Conv2d(in_dim, dim, 3, 2, 1, bias=False), nn.BatchNorm2d(dim, eps=1e-4), nn.ReLU())


class TokenInitializer(_Holder):
    """fv.py:704-738 / fvar.py:710-750. The depthwise conv is registered under two names, as in the
    reference (state_dict keys `pos_embed.*` and `to_global_feature.pos.*` share storage)."""

    def __init__(self, dim: int, input_resolution: Sequence[int], window_size: int, ct_size: int):
        super().__init__()
        self.pool = []
        for r in input_resolution:
            out = int(ct_size * r / window_size)
            stride = int(r / out)
            self.pool.append((r - (out - 1) * stride, stride, out))  # (kernel, stride, outputs)
        self.pos_embed = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.to_global_feature = nn.Sequential()
        self.to_global_feature.add_module("pos", self.pos_embed)
        self.ct_size = ct_size


class FasterViTLayer(_Holder):
    """One resolution level (fv.py:741-843; fvar.py:753-870)."""

    def __init__(self, dim, depth, input_resolution: Sequence[int], num_heads, window_size, ct_size, conv,
                 downsample, mlp_ratio, qkv_bias, layer_scale, layer_scale_conv, only_local,
                 do_propagation, any_res: bool, qk_scale=None):
        super().__init__()
        self.conv, self.window_size, self.dim = conv, window_size, dim
        res = list(input_resolution)
        if any_res:  # fvar.py:805-808: level geometry is padded up to a multiple of the window
            res = [r + (window_size - r % window_size) % window_size for r in res]
        self.input_resolution = res
        if conv:
            self.blocks = nn.ModuleList([ConvBlock(dim, layer_scale_conv) for _ in range(depth)])
            self.sr_ratio = [1, 1]
        else:
            self.sr_ratio = [1, 1] if only_local else [res[0] // window_size, res[1] // window_size]
            self.blocks = nn.ModuleList([
                HAT(dim, num_heads, mlp_ratio, qkv_bias, self.sr_ratio, window_size, i == depth - 1,
                    layer_scale, ct_size, do_propagation, any_res, qk_scale) for i in range(depth)])
        self.downsample = Downsample(dim) if downsample else None
        want_gt = (len(self.blocks) > 0 and not only_local and not conv and
                   (any_res or res[0] // window_size > 1))
        self.do_gt = bool(want_gt)
        if self.do_gt:
            self.global_tokenizer = TokenInitializer(dim, res, window_size, ct_size)


class FasterViT(nn.Module):
    """Drop-in for the reference `FasterViT` (fv.py:846-972 / fvar.py:873-1002): same constructor
    signature, attributes (`num_classes`, `patch_embed`, `levels`, `norm`, `avgpool`, `head`), methods
    and state_dict; forward/backward execute on the library's H100 kernels."""

    def __init__(self, dim, in_dim, depths, window_size, ct_size, mlp_ratio, num_heads, resolution=224,
                 drop_path_rate=0.2, in_chans=3, num_classes=1000, qkv_bias=True, qk_scale=None,
                 drop_rate=0., attn_drop_rate=0., layer_scale=None, layer_scale_conv=None,
                 layer_norm_last=False, hat=(False, False, True, False), do_propagation=False,
                 any_res=False, **kwargs):
        super().__init__()
        if layer_norm_last:
            raise NotImplementedError("layer_norm_last=True is not used by any shipped FasterViT config")
        if drop_rate or attn_drop_rate:
            raise NotImplementedError("dropout is unused (0) in every FasterViT config")
        hat = [True] * len(depths) if hat is None else list(hat)
        self.any_res = bool(any_res)
        self.resolution = _pair(resolution)
        self.num_classes = num_classes
        self.num_features = int(dim * 2 ** (len(depths) - 1))
        self.drop_path_rate = float(drop_path_rate)
        self.cfg = dict(dim=dim, in_dim=in_dim, depths=list(depths), window_size=list(window_size),
                        ct_size=ct_size, mlp_ratio=mlp_ratio, num_heads=list(num_heads),
                        resolution=self.resolution if self.any_res else self.resolution[0],
                        hat=hat, do_propagation=bool(do_propagation), any_res=self.any_res,
                        in_chans=in_chans)
        if qk_scale is not None:
            self.cfg["qk_scale"] = float(qk_scale)
        # stochastic-depth schedule over all blocks (fv.py:901)
        self.drop_path_rates = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        self.patch_embed = PatchEmbed(in_chans, in_dim, dim)
        self.levels = nn.ModuleList()
        for i in range(len(depths)):
            self.levels.append(FasterViTLayer(
                dim=int(dim * 2 ** i), depth=depths[i],
                input_resolution=[int(2 ** (-2 - i) * r) for r in self.resolution],
                num_heads=num_heads[i], window_size=window_size[i], ct_size=ct_size, conv=(i < 2),
                downsample=(i < 3), mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, layer_scale=layer_scale,
                layer_scale_conv=layer_scale_conv, only_local=not hat[i], do_propagation=do_propagation,
                any_res=self.any_res, qk_scale=qk_scale))
        self.norm = nn.BatchNorm2d(self.num_features)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(self._init_weights)
        self._engine = None
        self._grad_allreduce = None
        self._train_input_grad = False
        self._train_forwards_in_flight = 1

    # fv.py:930-943: Linear trunc_normal(.02)/zero bias, norms to identity, convs keep torch default
    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, (nn.LayerNorm, nn.BatchNorm2d)):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'rpb'}

    # -- execution ------------------------------------------------------------------------------
    def _get_engine(self):
        if self._engine is None:
            from .engine import Engine
            self._engine = Engine(self)
        return self._engine

    def __deepcopy__(self, memo):
        # ModelEmaV2 deep-copies the model (train.py:522): the engine (workspaces, packed weights)
        # is per-instance state and is rebuilt lazily by the copy.
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k == "_engine" else copy.deepcopy(v, memo)
        return new

    def enable_grad_allreduce(self, group=None) -> None:
        """Data-parallel training without wrapping in DistributedDataParallel: after every backward the flat
        gradient buffer is averaged over `group` (default: the world) with a single NCCL all-reduce — the one
        collective of the path (train.py:551). Parameters must start identical on all ranks."""
        self._grad_allreduce = True if group is None else group

    def enable_input_grad(self, enabled: bool = True):
        """Train-mode image gradients: after this, an input with requires_grad under .train() gets its gradient
        (x.grad, fp32, local to the rank) from model(x), forward_features, forward_levels and the pooled features of a
        num_classes = 0 model -- a trainable front end, pixel-space prompts, adversarial training. Without it such an
        input raises, as it always did: the plan for it is a second one per input shape, and a caller that merely forgot
        to detach should hear about it. Eval mode needs no switch."""
        self._train_input_grad = bool(enabled)
        return self

    def set_train_forwards_in_flight(self, n: int = 1):
        """Let up to n train-mode forwards of the same input shape (and outputs) await their backward at once: losses
        over several views or crops through one model, the frames of a clip summed into one backward. Each such forward
        keeps its own set of saved activations, one train plan's device memory, until its backward has run or its
        outputs are freed; the sets are built as they are first needed and reused from step to step. A forward beyond n
        overwrites the oldest one, whose backward then raises. Forwards under torch.no_grad() (checkpointed segments)
        hold no set. Default 1: a second forward before the first one's backward raises there, so a forgotten
        backward() is reported rather than paid for in memory. Under enable_grad_allreduce() each forward's backward
        all-reduces its own gradients (the mean of a sum is the sum of the means): one all-reduce per forward, and the
        first backward of every new set times the all-reduce once, a collective that all ranks reach in the same
        order."""
        from .lib import FvitError
        if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < 1:
            raise FvitError(f"set_train_forwards_in_flight takes an integer n >= 1, got {n!r}")
        self._train_forwards_in_flight = int(n)
        if self._engine is not None:
            self._engine.trim_plans()
        return self

    def switch_to_deploy(self):
        """Put every positional-embedding module into deploy mode (the reference exposes `switch_to_deploy` per module,
        fv.py:263-269, 336-342; this is the loop a user writes over `model.modules()`). Inference then reads the
        cached `relative_bias` buffers and skips the positional MLP kernels for good."""
        for m in self.modules():
            if m is not self and hasattr(m, "switch_to_deploy"):
                m.switch_to_deploy()
        return self

    def release_eval_grad_plans(self) -> None:
        """Free the device memory of eval-mode gradients: the first backward of a grad-enabled eval forward builds a
        plan per input shape that holds a training step's saved activations and keeps it; this drops them (the next
        such backward builds its plan again)."""
        if self._engine is not None:
            self._engine.release_eval_grad_plans()

    def forward_levels(self, x, out_indices=(0, 1, 2, 3)):
        """Per-level feature maps [B, C_i, H_i, W_i] (each level's output before its Downsample), the `xo` a dense-
        prediction backbone taps (downstream/object_detection/dino/models/dino/fastervit.py:686-709, 816-827).
        Differentiable under .train(), and under .eval() with grad enabled (running-statistics BatchNorms; x.grad too
        when x requires grad). Parameters above the highest requested level, `norm` and `head` get no gradient."""
        return self._get_engine().forward_levels(x, tuple(out_indices))

    def forward_features(self, x):
        """The `norm`-ed last-level map [B, C, H, W] (fv.py:949-953); under .train() with batch statistics (running
        statistics updated), under .eval() with running statistics; differentiable in both (in eval when grad is
        enabled and x or a parameter requires grad)."""
        return self._get_engine().forward(x, features_only=True)

    def forward_head(self, x):
        """avg-pool + head (fv.py:955-958) of a forward_features map (or pooled features); eval mode only, and then
        differentiable w.r.t. the features and the head's parameters."""
        return self._get_engine().forward_head(x)

    def forward(self, x):
        return self._get_engine().forward(x)

    def _load_state_dict(self, pretrained, strict: bool = False):
        """The reference model's own loader (fv.py:967-972 -> _load_checkpoint / _load_state_dict, fv.py:112-209):
        tolerant by default — tensors whose shape differs from the model's (a head built for another
        `num_classes`, positional buffers of another resolution / window) are reported and skipped, missing
        `num_batches_tracked` counters are ignored, and only `strict=True` raises."""
        from .registry import load_state_dict_tolerant, read_checkpoint_state
        load_state_dict_tolerant(self, read_checkpoint_state(pretrained), strict=strict)


def build_model(name: str, pretrained: bool = False, **kwargs) -> FasterViT:
    """Entrypoint body shared by the 22 registered names (fv.py:977-1009 et al.): pop the overridable
    hyper-parameters, fill num_classes / in_chans from the pretrained cfg, attach pretrained_cfg."""
    spec = MODEL_SPECS[name]
    hp = {k: kwargs.pop(k, v) for k, v in spec["defaults"].items()}
    model_path = hp.pop("model_path")
    pcfg = dict(default_cfgs[name])
    kwargs.setdefault("num_classes", pcfg["num_classes"])
    kwargs.setdefault("in_chans", pcfg["input_size"][0])
    for k in ("pretrained_cfg", "pretrained_cfg_overlay"):  # passed by timm.create_model
        kwargs.pop(k, None)
    fixed = {k: v for k, v in spec["fixed"].items() if k not in kwargs}
    model = FasterViT(**hp, **fixed, any_res=spec["any_res"], **kwargs)
    model.pretrained_cfg = pcfg
    model.default_cfg = model.pretrained_cfg
    if pretrained:
        from pathlib import Path
        if not Path(model_path).is_file():
            torch.hub.download_url_to_file(url=pcfg["url"], dst=model_path)
        model._load_state_dict(model_path)
    return model
