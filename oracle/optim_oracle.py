"""CPU oracle for the optimizer step of the training loop — TEST INFRASTRUCTURE, not product code.

Restates, on plain torch CPU tensors (fp64 by default), the arithmetic the reference's training loop runs either
side of `loss.backward()` (the reference's fastervit/train.py:879-899):

  * `clip_coef`  — `utils.dispatch_clip_grad(..., mode='norm')` = torch.nn.utils.clip_grad_norm_ (train.py:889-892)
  * `adamw_step` — `optimizer.step()` for `--opt adamw` (TRAINING.md:28): torch.optim.AdamW, single-tensor form
  * `lamb_step`  — `optimizer.step()` for `--opt lamb` (TRAINING.md:105): timm.optim.Lamb
  * `ema_update` — `model_ema.update(model)` (train.py:898-899): timm.utils.ModelEmaV2

Parity pins: `adamw_step` and `clip_coef` are pinned against torch itself (tests/test_optim_cpu.py runs
torch.optim.AdamW / clip_grad_norm_ on the same data). **timm (pinned 0.9.6 in the reference's requirements.txt:1)
is not installable in this container, so `lamb_step` and `ema_update` restate timm's published algorithm
(timm/optim/lamb.py, timm/utils/model_ema.py) and are UNPINNED against timm's code**; the anchor is the call site
(train.py:896-899) plus the LAMB paper's update rule. Only tests/ and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import math
from typing import Sequence

import torch


def global_norm(grads: Sequence[torch.Tensor]) -> float:
    return math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))


def clip_coef(grads: Sequence[torch.Tensor], max_norm: float, eps: float = 1e-6) -> tuple[float, float]:
    """(total_norm, coefficient) of torch.nn.utils.clip_grad_norm_: coef = min(1, max_norm / (norm + 1e-6)).
    eps = 0 gives timm Lamb's internal `max_grad_norm` clipping (grad / max(norm / max_norm, 1))."""
    norm = global_norm(grads)
    if max_norm is None or max_norm <= 0:
        return norm, 1.0
    denom = norm + eps
    return norm, (1.0 if denom == 0 else min(1.0, max_norm / denom))


def adamw_step(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *, step: int, lr: float,
               beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8, weight_decay: float = 1e-2) -> None:
    """torch.optim.AdamW (`_single_tensor_adamw`), in place on p, m, v. `step` is the 1-based step number."""
    p.mul_(1 - lr * weight_decay)
    m.lerp_(g, 1 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / bc1)


def lamb_step(ps: Sequence[torch.Tensor], gs: Sequence[torch.Tensor], ms: Sequence[torch.Tensor],
              vs: Sequence[torch.Tensor], *, step: int, lr: float | Sequence[float], weight_decay: Sequence[float],
              beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-6, max_grad_norm: float | None = 1.0,
              trust_clip: bool = False, always_adapt: bool = False, grad_averaging: bool = True) -> None:
    """timm.optim.Lamb.step over a list of tensors (one param group per tensor: weight_decay[i], lr[i]).
    Global gradient-norm clipping first (max_grad_norm), then per-tensor trust ratio ||p|| / ||update||."""
    _, coef = clip_coef(gs, max_grad_norm if max_grad_norm else 0.0, eps=0.0)
    beta3 = 1 - beta1 if grad_averaging else 1.0
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    for i, (p, g, m, v) in enumerate(zip(ps, gs, ms, vs)):
        wd = weight_decay[i]
        lri = lr[i] if isinstance(lr, (list, tuple)) else lr
        g = g * coef
        m.mul_(beta1).add_(g, alpha=beta3)
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
        update = (m / bc1).div_(denom)
        if wd != 0:
            update.add_(p, alpha=wd)
        if wd != 0 or always_adapt:
            w_norm, u_norm = float(p.norm(2.0)), float(update.norm(2.0))
            trust = w_norm / u_norm if (w_norm > 0 and u_norm > 0) else 1.0
            if trust_clip:
                trust = min(trust, 1.0)
            update.mul_(trust)
        p.add_(update, alpha=-lri)


def ema_update(ema: torch.Tensor, src: torch.Tensor, decay: float) -> None:
    """ModelEmaV2._update: ema = decay * ema + (1 - decay) * model (floating entries of the state_dict)."""
    ema.copy_(decay * ema + (1.0 - decay) * src)
