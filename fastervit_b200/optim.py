"""Optimizer step, gradient clipping and weight EMA on the flat gradient buffer (SURVEY.md §8 f.1).

What the reference's training loop does either side of `loss.backward()` (train.py:879-899) —
`GradScaler.unscale_` + non-finite check, `dispatch_clip_grad(mode='norm')`, `optimizer.step()` (`--opt adamw` for
FasterViT-0..3, `--opt lamb` for 4..6; TRAINING.md:28,105) and `ModelEmaV2.update` — is hundreds of foreach /
per-tensor ATen launches. Here it is 3-4 launches of libfvit_sm100.so (csrc/optim_sm100.cu) over one chunk table:

  fvit_optim_sqnorm  -> fvit_optim_prepare  -> fvit_optim_adamw            (+ fused EMA)
                                             -> fvit_optim_lamb_stage1/2    (+ fused EMA)

`FusedAdamW` / `FusedLamb` are `torch.optim.Optimizer` subclasses (param_groups, lr schedulers, state_dict,
`GradScaler.step` all work unchanged) whose gradients and moments live in flat fp32 buffers. The backward pass of
fastervit_b200 hands autograd views of ONE flat buffer, so in the normal training loop the step reads the
gradients in place (zero copies); gradients that arrive as separate tensors are gathered with one launch.
Nothing in `step()` synchronises with the host: step count, bias corrections, clip coefficient and the
skip-on-overflow decision are device scalars.

`FlatEma` mirrors timm's `ModelEmaV2` (`.module`, `.update(model)`, `.set(model)`), one launch per update, or fused
into the optimizer's update kernel with `optimizer.attach_ema(ema, model)`.

There is no CPU path: `step()` / `update()` raise on CPU tensors (host-side layout logic is CPU-testable).
"""
from __future__ import annotations

import copy
from typing import Iterable, Sequence

import torch
import torch.nn as nn

from . import lib as L

CHUNK = 16384  # elements of one segment handled by one CTA (64 KiB per fp32 stream)


def _ru(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise L.FvitError(f"{what} runs on CUDA only (fastervit_b200 has no CPU fallback): move the model to a "
                          "CUDA device first")


def _device_guard(dev):
    return torch.cuda.device(dev)


# ------------------------------------------------------------------------------------ host-side tables
def build_chunks(numels: Sequence[int], chunk: int = CHUNK, active: Sequence[bool] | None = None) -> torch.Tensor:
    """int32 [nchunks, 4] table {segment, first element, count, 0}: every active segment is cut into runs of at
    most `chunk` elements (chunk % 4 == 0 keeps the runs 16-byte aligned relative to the segment start)."""
    assert chunk % 4 == 0 and chunk > 0
    rows = []
    for s, n in enumerate(numels):
        if active is not None and not active[s]:
            continue
        for st in range(0, n, chunk):
            rows.append((s, st, min(chunk, n - st), 0))
    if not rows:
        return torch.zeros((0, 4), dtype=torch.int32)
    return torch.tensor(rows, dtype=torch.int32)


def sequential_offsets(numels: Sequence[int], align: int = 64) -> tuple[list[int], int]:
    """Element offsets of consecutive segments, each aligned to `align` elements (256 B): the layout of the
    backward pass's flat gradient buffer (engine_train.TrainPlan._setup_train)."""
    offs, n = [], 0
    for k in numels:
        offs.append(n)
        n += _ru(k, align)
    return offs, n


def shared_storage_offsets(tensors: Sequence[torch.Tensor | None]) -> list[int] | None:
    """If every tensor is a dense fp32 view of ONE storage and the views do not overlap, return their element
    offsets in that storage, else None."""
    if not tensors or any(t is None for t in tensors):
        return None
    base = tensors[0].untyped_storage().data_ptr()
    offs = []
    for t in tensors:
        if t.dtype != torch.float32 or not t.is_contiguous() or t.untyped_storage().data_ptr() != base:
            return None
        offs.append(t.storage_offset())
    order = sorted(range(len(offs)), key=lambda i: offs[i])
    for a, b in zip(order, order[1:]):
        if offs[a] + tensors[a].numel() > offs[b]:
            return None
    return offs


def param_groups_weight_decay(model: nn.Module, weight_decay: float = 1e-5,
                              no_weight_decay_list: Iterable[str] = ()) -> list[dict]:
    """timm.optim.optim_factory.param_groups_weight_decay (what `create_optimizer_v2(model, ...)` of train.py builds
    with filter_bias_and_bn=True): 1-D parameters, biases and listed names get weight_decay 0."""
    skip = set(no_weight_decay_list)
    decay, no_decay = [], []
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        (no_decay if (p.ndim <= 1 or name.endswith(".bias") or name in skip) else decay).append(p)
    return [{"params": no_decay, "weight_decay": 0.0}, {"params": decay, "weight_decay": weight_decay}]


class _DeviceTables:
    """Chunk table + int64 pointer / offset tables on the device for a list of segments."""

    def __init__(self, numels: Sequence[int], device, chunk: int = CHUNK):
        self.numels = list(numels)
        self.device = device
        self.chunk = chunk
        self.chunks = build_chunks(self.numels, chunk).to(device)
        self.nchunks = self.chunks.shape[0]
        self._subsets: dict[tuple, torch.Tensor] = {}

    def subset(self, active: Sequence[bool]) -> torch.Tensor:
        key = tuple(bool(a) for a in active)
        if all(key):
            return self.chunks
        t = self._subsets.get(key)
        if t is None:
            t = build_chunks(self.numels, self.chunk, key).to(self.device)
            self._subsets[key] = t
        return t

    def i64(self, values: Sequence[int]) -> torch.Tensor:
        return torch.tensor(list(values), dtype=torch.int64).to(self.device)


# ------------------------------------------------------------------------------------ optimizers
class _FlatOptimizer(torch.optim.Optimizer):
    """Shared machinery: flat moment buffers, zero-copy / gathered flat gradients, device scalars."""

    _step_supports_amp_scaling = True   # torch.amp.GradScaler hands us grad_scale / found_inf (no host sync)
    _clip_eps = 1e-6                    # torch.nn.utils.clip_grad_norm_

    def __init__(self, params, defaults: dict, max_grad_norm: float | None):
        super().__init__(params, defaults)
        self.max_grad_norm = max_grad_norm
        self._lay = None        # layout, built at the first step (it adopts the gradient buffer's layout)
        self._ema = None        # (FlatEma, [ema parameter per optimizer segment])
        self._hp_cache = None

    # ---- layout -----------------------------------------------------------------------------------
    def _all_params(self) -> list[torch.Tensor]:
        return [p for g in self.param_groups for p in g["params"]]

    def _build_layout(self, grads: list[torch.Tensor | None]) -> None:
        ps = self._all_params()
        if not ps:
            raise L.FvitError("optimizer has no parameters")
        dev = ps[0].device
        for p in ps:
            _require_cuda(p, "the fused optimizer step")
            if p.dtype != torch.float32 or not p.is_contiguous() or p.device != dev:
                raise L.FvitError("parameters must be contiguous float32 tensors on one device")
        numels = [p.numel() for p in ps]
        offs = shared_storage_offsets(grads)
        if offs is not None:   # adopt the layout of the flat gradient buffer -> gradients are read in place
            flat_n = _ru(max(o + n for o, n in zip(offs, numels)), 64)
        else:
            offs, flat_n = sequential_offsets(numels)
        if flat_n >= 2 ** 31:
            raise L.FvitError("flat optimizer buffers are limited to 2^31 elements")
        tb = _DeviceTables(numels, dev)
        lay = dict(params=ps, ids=[id(p) for p in ps], numels=numels, offs=offs, flat_n=flat_n, tb=tb, dev=dev,
                   seg_off=tb.i64(offs), seg_p=tb.i64([p.data_ptr() for p in ps]),
                   p_key=tuple(p.data_ptr() for p in ps),
                   m=torch.zeros(flat_n, dtype=torch.float32, device=dev),
                   v=torch.zeros(flat_n, dtype=torch.float32, device=dev),
                   scal=torch.zeros(8, dtype=torch.float32, device=dev),
                   partials=torch.zeros(2 * max(tb.nchunks, 1), dtype=torch.float32, device=dev),
                   seg_hp=torch.zeros(len(ps), 2, dtype=torch.float32, device=dev),
                   gstage=None, seg_ema=None, ema_key=None)
        self._lay = lay
        self._hp_cache = None
        self._adopt_state()

    def _adopt_state(self) -> None:
        """Make self.state[p] views of the flat buffers, keeping any values already there (load_state_dict)."""
        lay = self._lay
        step = None
        for p, off, n in zip(lay["params"], lay["offs"], lay["numels"]):
            st = self.state[p]
            mv = lay["m"][off:off + n].view_as(p)
            vv = lay["v"][off:off + n].view_as(p)
            if "exp_avg" in st and st["exp_avg"].data_ptr() != mv.data_ptr():
                mv.copy_(st["exp_avg"])
                vv.copy_(st["exp_avg_sq"])
                if "step" in st:
                    step = float(st["step"])
            st["exp_avg"], st["exp_avg_sq"] = mv, vv
            st["step"] = lay["scal"][3]
        if step is not None:
            lay["scal"][3] = step

    def load_state_dict(self, state_dict) -> None:
        super().load_state_dict(state_dict)
        if self._lay is not None:
            self._adopt_state()

    # ---- per-step host work ---------------------------------------------------------------------------
    def _sync_hparams(self) -> None:
        lay = self._lay
        hp = []
        for g in self.param_groups:
            hp += [(float(g["lr"]), float(g["weight_decay"]))] * len(g["params"])
        if hp != self._hp_cache:
            lay["seg_hp"].copy_(torch.tensor(hp, dtype=torch.float32).view(-1, 2))
            self._hp_cache = hp

    def _flat_grad(self, grads: list[torch.Tensor | None], active: list[bool], chunks: torch.Tensor) -> int:
        """Device address of a flat fp32 buffer holding the gradients in the optimizer's layout."""
        lay = self._lay
        base = None
        for g, off, act in zip(grads, lay["offs"], active):
            if not act:
                continue
            if g.dtype != torch.float32 or not g.is_contiguous():
                base = None
                break
            b = g.data_ptr() - 4 * off
            if base is None:
                base = b
            elif b != base:
                base = None
                break
        if base is not None and base % 16 == 0:
            return base   # the backward pass's flat buffer, read in place
        if lay["gstage"] is None:
            lay["gstage"] = torch.zeros(lay["flat_n"], dtype=torch.float32, device=lay["dev"])
        src = [g.data_ptr() if act else 0 for g, act in zip(grads, active)]
        for g, act in zip(grads, active):
            if act and (g.dtype != torch.float32 or not g.is_contiguous()):
                raise L.FvitError("gradients must be contiguous float32 tensors")
        seg_src = lay["tb"].i64(src)
        L.call("fvit_optim_gather_f32", chunks.data_ptr(), chunks.shape[0], seg_src.data_ptr(),
               lay["seg_off"].data_ptr(), lay["gstage"].data_ptr())
        return lay["gstage"].data_ptr()

    def _ema_args(self) -> tuple[int | None, float]:
        if self._ema is None:
            return None, 0.0
        ema, eps_ = self._ema
        lay = self._lay
        key = tuple(e.data_ptr() for e in eps_)
        if lay["ema_key"] != key:
            lay["seg_ema"] = lay["tb"].i64(key)
            lay["ema_key"] = key
        ema._fused_steps += 1
        return lay["seg_ema"].data_ptr(), float(ema.decay)

    def attach_ema(self, ema: "FlatEma", model: nn.Module) -> None:
        """Fuse `ema.update(model)`'s parameter part into this optimizer's update kernel (the EMA then costs 8
        extra bytes per element instead of a separate 12-byte pass); `ema.update(model)` keeps handling the
        buffers (BatchNorm running statistics)."""
        by_id = {id(p): n for n, p in model.named_parameters()}
        ema_named = dict(ema.module.named_parameters())
        eps_ = []
        for p in self._all_params():
            name = by_id.get(id(p))
            if name is None or name not in ema_named:
                raise L.FvitError("attach_ema: optimizer parameter not found in the model / EMA module")
            eps_.append(ema_named[name])
        self._ema = (ema, eps_)
        ema._fused_into = self
        if self._lay is not None:
            self._lay["ema_key"] = None

    @property
    def grad_norm(self) -> torch.Tensor:
        """Device scalar: the (unscaled, pre-clip) global gradient norm of the last step."""
        return self._lay["scal"][0]

    @property
    def found_inf_flag(self) -> torch.Tensor:
        """Device scalar: 1 if the last step was skipped because of non-finite gradients."""
        return self._lay["scal"][1]

    # ---- the step -----------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ps = self._all_params()
        grads = [p.grad for p in ps]
        if self._lay is None or self._lay["ids"] != [id(p) for p in ps]:
            self._build_layout(grads)
        lay = self._lay
        active = [g is not None for g in grads]
        if not any(active):
            return loss
        L.bump_weights_epoch()   # parameters are about to change through raw pointers (no autograd version bump)
        with _device_guard(lay["dev"]):
            p_key = tuple(p.data_ptr() for p in ps)
            if p_key != lay["p_key"]:   # parameters were re-allocated (.to(), load with assign=True, ...)
                lay["seg_p"] = lay["tb"].i64(p_key)
                lay["p_key"] = p_key
            chunks = lay["tb"].subset(active)
            self._sync_hparams()
            gptr = self._flat_grad(grads, active, chunks)
            grad_scale = getattr(self, "grad_scale", None)   # set by torch.amp.GradScaler.step
            found_inf = getattr(self, "found_inf", None)
            for t in (grad_scale, found_inf):
                if t is not None and (t.dtype != torch.float32 or t.device != lay["dev"]):
                    raise L.FvitError("grad_scale / found_inf must be float32 device scalars")
            need_norm = (self.max_grad_norm is not None and self.max_grad_norm > 0) or grad_scale is not None \
                or self._always_check_finite
            nparts = 0
            if need_norm:
                L.call("fvit_optim_sqnorm", chunks.data_ptr(), chunks.shape[0], lay["seg_off"].data_ptr(), gptr,
                       lay["partials"].data_ptr())
                nparts = chunks.shape[0]
            b1, b2 = self.defaults["betas"]
            L.call("fvit_optim_prepare", lay["partials"].data_ptr(), nparts, L.ptr(grad_scale), L.ptr(found_inf),
                   float(self.max_grad_norm or 0.0), float(self._clip_eps), float(b1), float(b2),
                   lay["scal"].data_ptr())
            self._update(chunks, gptr)
        return loss

    _always_check_finite = False

    def _update(self, chunks: torch.Tensor, gptr: int) -> None:  # pragma: no cover - abstract
        raise NotImplementedError


class FusedAdamW(_FlatOptimizer):
    """torch.optim.AdamW semantics (`--opt adamw`, TRAINING.md:28) in one update launch. `max_grad_norm` fuses
    `--clip-grad <v> --clip-mode norm` (train.py:889-892) into the step (leave None when the training loop clips
    itself). Betas / eps are optimizer-wide; lr and weight_decay are per param group."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm: float | None = None):
        if isinstance(params, nn.Module):
            params = param_groups_weight_decay(params, weight_decay)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), max_grad_norm)

    def _update(self, chunks, gptr):
        lay = self._lay
        b1, b2 = self.defaults["betas"]
        seg_ema, decay = self._ema_args()
        L.call("fvit_optim_adamw", chunks.data_ptr(), chunks.shape[0], lay["seg_p"].data_ptr(),
               lay["seg_off"].data_ptr(), lay["seg_hp"].data_ptr(), gptr, lay["m"].data_ptr(), lay["v"].data_ptr(),
               float(b1), float(b2), float(self.defaults["eps"]), lay["scal"].data_ptr(), seg_ema, decay)


class FusedLamb(_FlatOptimizer):
    """timm.optim.Lamb semantics (`--opt lamb`, TRAINING.md:105-156; defaults of timm 0.9.6: betas (0.9, 0.999),
    eps 1e-6, bias correction, gradient averaging, global max_grad_norm 1.0, trust ratio only where weight decay
    applies) in two update launches."""

    _clip_eps = 0.0   # timm Lamb divides by max(norm / max_grad_norm, 1)

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.01,
                 max_grad_norm: float | None = 1.0, trust_clip: bool = False, always_adapt: bool = False):
        if isinstance(params, nn.Module):
            params = param_groups_weight_decay(params, weight_decay)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), max_grad_norm)
        self.trust_clip, self.always_adapt = bool(trust_clip), bool(always_adapt)

    def _update(self, chunks, gptr):
        lay = self._lay
        if "u" not in lay:
            lay["u"] = torch.zeros(lay["flat_n"], dtype=torch.float32, device=lay["dev"])
            lay["seg_norms"] = torch.zeros(len(lay["params"]), 2, dtype=torch.float32, device=lay["dev"])
        lay["seg_norms"].zero_()
        b1, b2 = self.defaults["betas"]
        seg_ema, decay = self._ema_args()
        common = (chunks.data_ptr(), chunks.shape[0], lay["seg_p"].data_ptr(), lay["seg_off"].data_ptr(),
                  lay["seg_hp"].data_ptr())
        L.call("fvit_optim_lamb_stage1", *common, gptr, lay["u"].data_ptr(), lay["m"].data_ptr(), lay["v"].data_ptr(),
               float(b1), float(b2), float(self.defaults["eps"]), lay["scal"].data_ptr(), lay["seg_norms"].data_ptr())
        L.call("fvit_optim_lamb_stage2", *common, lay["u"].data_ptr(), lay["seg_norms"].data_ptr(),
               int(self.trust_clip), int(self.always_adapt), lay["scal"].data_ptr(), seg_ema, decay)


# ------------------------------------------------------------------------------------ weight EMA
class FlatEma(nn.Module):
    """timm.utils.ModelEmaV2 (train.py:519-523, 898-899) with the update as one launch: `.module` is a deep copy of
    the model in eval mode; `update(model)` applies ema = decay * ema + (1 - decay) * model to every floating entry of
    the state_dict (integer buffers follow ModelEmaV2's float arithmetic and cast back, as `copy_` does there).

    Host cost per update is a pointer sweep over the state (~1 k data_ptr() calls): the (owner module, attribute)
    slots are resolved once per model, and the device tables are reused while no tensor was re-allocated."""

    def __init__(self, model: nn.Module, decay: float = 0.9999, device=None):
        super().__init__()
        self.module = copy.deepcopy(model)
        self.module.eval()
        self.decay = decay
        self.device = device
        if device is not None:
            self.module.to(device=device)
        self._slot_cache = None
        self._fused_into = None
        self._fused_steps = 0

    # ---- state_dict entries as (owner module, attribute name) slots, resolved once per model ------------------
    def _slots(self, model: nn.Module) -> dict:
        c = self._slot_cache
        if c is not None and c["model"] is model:
            return c
        ekeys, mkeys = list(self.module.state_dict().keys()), list(model.state_dict().keys())
        if ekeys != mkeys:
            raise L.FvitError("FlatEma: the model's state_dict keys differ from the EMA copy's")

        def owner(root: nn.Module, key: str):
            path, _, name = key.rpartition(".")
            return (root.get_submodule(path) if path else root), name
        c = dict(model=model, keys=ekeys, e=[owner(self.module, k) for k in ekeys], m=[owner(model, k) for k in ekeys],
                 pnames={n for n, _ in model.named_parameters()}, plans={})
        self._slot_cache = c
        return c

    @staticmethod
    def _read(slots) -> list[torch.Tensor]:
        out = []
        for mod, name in slots:
            t = mod._parameters.get(name)
            out.append(t if t is not None else mod._buffers[name])
        return out

    def _plan(self, c: dict, ev, mv, skip_params: bool) -> dict:
        # ModelEmaV2 walks state_dict().values(): a tensor registered under two names (the tokenizer's depthwise
        # conv, fv.py:727-731) is blended once per name. The first occurrences go into one launch; the repeats
        # follow in a second launch (same stream, so the order of the reference's loop is kept, without two CTAs
        # racing on one tensor). Parameters fused into the optimizer's kernel were already blended once there.
        seen: set[int] = set()
        first, repeats, ints = [], [], []
        for e, m, k in zip(ev, mv, c["keys"]):
            if not e.is_floating_point():
                ints.append((e, m))
                continue
            _require_cuda(e, "FlatEma")
            _require_cuda(m, "FlatEma")
            if e.dtype != torch.float32 or m.dtype != torch.float32 or not e.is_contiguous() or not m.is_contiguous() \
                    or e.shape != m.shape:
                raise L.FvitError("FlatEma needs contiguous float32 state of identical shapes")
            if e.data_ptr() in seen:
                repeats.append((e, m))
                continue
            seen.add(e.data_ptr())
            if not (skip_params and k in c["pnames"]):
                first.append((e, m))
        launches = []
        for fl in (first, repeats):
            if fl:
                tb = _DeviceTables([e.numel() for e, _ in fl], fl[0][0].device)
                launches.append(dict(tb=tb, dev=fl[0][0].device, seg_e=tb.i64([e.data_ptr() for e, _ in fl]),
                                     seg_m=tb.i64([m.data_ptr() for _, m in fl])))
        return dict(launches=launches, ie=[e for e, _ in ints], im=[m for _, m in ints])

    @torch.no_grad()
    def _blend(self, model: nn.Module, decay: float, skip_params: bool) -> None:
        c = self._slots(model)
        ev, mv = self._read(c["e"]), self._read(c["m"])
        key = (tuple(t.data_ptr() for t in ev), tuple(t.data_ptr() for t in mv), skip_params)
        plan = c["plans"].get(key)
        if plan is None:
            if len(c["plans"]) >= 4:
                c["plans"].clear()
            plan = c["plans"][key] = self._plan(c, ev, mv, skip_params)
        L.bump_weights_epoch()   # the EMA copy is written through raw pointers
        for t in plan["launches"]:
            with _device_guard(t["dev"]):
                L.call("fvit_optim_ema", t["tb"].chunks.data_ptr(), t["tb"].nchunks, t["seg_e"].data_ptr(),
                       t["seg_m"].data_ptr(), float(decay))
        if plan["ie"]:   # num_batches_tracked & co.: ModelEmaV2's float arithmetic, cast back to integers by copy_
            acc = torch._foreach_mul(plan["ie"], decay)
            torch._foreach_add_(acc, torch._foreach_mul(plan["im"], 1.0 - decay))
            torch._foreach_copy_(plan["ie"], acc)

    def update(self, model: nn.Module) -> None:
        fused = self._fused_into is not None and self._fused_steps > 0
        self._fused_steps = 0
        self._blend(model, self.decay, skip_params=fused)

    def set(self, model: nn.Module) -> None:
        self._blend(model, 0.0, skip_params=False)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)
