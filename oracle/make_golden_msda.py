"""Generate tests/golden/msda_*.pt from the UNMODIFIED reference's multi-scale deformable attention
(downstream/object_detection/dino/models/dino/ops and downstream/object_tracking/motrv2/models/ops of a checkout of
NVlabs/FasterViT).

    FASTERVIT_REFERENCE=<path to the reference checkout> python oracle/make_golden_msda.py

The reference's `ops.modules.MSDeformAttn` and `ops.functions.ms_deform_attn_core_pytorch` are imported by path; the
compiled MultiScaleDeformableAttention extension is replaced by an empty stand-in module (nothing here calls it). The
module's MSDeformAttnFunction is pointed at ms_deform_attn_core_pytorch (grid_sample), and everything runs on the CPU
in fp64. Written:
  * msda_core.pt: core cases (value, shapes, start index, locations, weights, grad_out) with the output and the three
    input gradients; locations outside [0, 1], levels with H = 1 or W = 1, odd D;
  * msda_module.pt: DINO cases with 2-d and 4-d reference points and a padding mask, and a MOTRv2 sigmoid_attn case:
    the (perturbed) state_dict, inputs, output, and the gradients of every parameter and of query, reference_points
    and input_flatten for loss = sum(out * grad_out);
  * msda_schema.pt: the state_dict schema (name, shape, dtype) of the default DINO and MOTRv2 modules, the default
    sampling_offsets.bias, and the complete state_dict of a small module built after torch.manual_seed(0).
The tests never need the reference.
"""
from __future__ import annotations

import importlib
import os
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
_REF = os.environ.get("FASTERVIT_REFERENCE")
DINO_DIR = Path(_REF or "", "downstream", "object_detection", "dino", "models", "dino")
MOTR_DIR = Path(_REF or "", "downstream", "object_tracking", "motrv2", "models")
if not _REF or not (DINO_DIR / "ops" / "modules" / "ms_deform_attn.py").is_file():
    raise SystemExit("make_golden_msda.py: set FASTERVIT_REFERENCE to a checkout of NVlabs/FasterViT")

# levels (H, W) of the core cases: H = 1 and W = 1 levels, odd sizes
CORE_CASES = {
    "odd_d": dict(N=2, Lq=7, M=2, D=5, P=3, levels=[(6, 4), (3, 2), (1, 5), (2, 1)], lo=-0.3, hi=1.3),
    "d8": dict(N=1, Lq=5, M=3, D=8, P=2, levels=[(4, 4), (2, 3)], lo=-0.6, hi=1.6),
    "d1_one_level": dict(N=2, Lq=4, M=1, D=1, P=4, levels=[(3, 5)], lo=-0.2, hi=1.2),
}
# module cases: (d_model, n_levels, n_heads, n_points), reference-point width, sigmoid_attn
MODULE_CASES = {
    "dino_ref2": dict(cfg=(32, 3, 4, 2), ref=2, sigmoid=False),
    "dino_ref4": dict(cfg=(32, 3, 4, 2), ref=4, sigmoid=False),
    "motr_sigmoid": dict(cfg=(24, 2, 3, 3), ref=2, sigmoid=True),
}
MODULE_LEVELS = [(5, 6), (3, 3), (2, 1)]


def _import_ops(models_dir: Path, tag: str):
    """(ops.modules.ms_deform_attn, ops.functions.ms_deform_attn_func) of one reference copy."""
    sys.modules.setdefault("MultiScaleDeformableAttention", types.ModuleType("MultiScaleDeformableAttention"))
    for k in [k for k in sys.modules if k == "ops" or k.startswith("ops.")]:
        del sys.modules[k]
    sys.path.insert(0, str(models_dir))
    try:
        mod = importlib.import_module("ops.modules.ms_deform_attn")
        fn = importlib.import_module("ops.functions.ms_deform_attn_func")
    finally:
        sys.path.remove(str(models_dir))
    for k in [k for k in sys.modules if k == "ops" or k.startswith("ops.")]:
        sys.modules[f"_ref_{tag}_{k}"] = sys.modules.pop(k)

    class CoreFunction:  # the module's MSDeformAttnFunction, computed by the reference's grid_sample restatement
        @staticmethod
        def apply(value, shapes, start_index, locations, weights, im2col_step):
            return fn.ms_deform_attn_core_pytorch(value, shapes, locations, weights)

    mod.MSDeformAttnFunction = CoreFunction
    return mod, fn


def _starts(levels):
    out, acc = [], 0
    for h, w in levels:
        out.append(acc)
        acc += h * w
    return out


def core_case(fn, c, gen):
    N, Lq, M, D, P, levels = c["N"], c["Lq"], c["M"], c["D"], c["P"], c["levels"]
    L, S = len(levels), sum(h * w for h, w in levels)
    f64 = dict(dtype=torch.float64)
    value = torch.randn(N, S, M, D, generator=gen, **f64)
    loc = c["lo"] + (c["hi"] - c["lo"]) * torch.rand(N, Lq, M, L, P, 2, generator=gen, **f64)
    w = torch.rand(N, Lq, M, L, P, generator=gen, **f64)
    go = torch.randn(N, Lq, M * D, generator=gen, **f64)
    shapes = torch.tensor(levels, dtype=torch.int64)
    v, s, a = (t.clone().requires_grad_(True) for t in (value, loc, w))
    out = fn.ms_deform_attn_core_pytorch(v, shapes, s, a)
    gv, gs, ga = torch.autograd.grad(out, (v, s, a), go)
    return dict(value=value, spatial_shapes=shapes, level_start_index=torch.tensor(_starts(levels)),
                sampling_locations=loc, attention_weights=w, grad_out=go, out=out.detach(), grad_value=gv,
                grad_sampling_locations=gs, grad_attention_weights=ga)


def module_case(mod, c, gen):
    d_model, L, M, P = c["cfg"]
    levels = MODULE_LEVELS[:L]
    S = sum(h * w for h, w in levels)
    kw = dict(sigmoid_attn=True) if c["sigmoid"] else {}
    m = mod.MSDeformAttn(d_model, L, M, P, **kw).double()
    with torch.no_grad():  # move off the init (zero offset weights, uniform attention) so every path carries gradient
        for p in m.parameters():
            p.add_(0.3 * torch.randn(p.shape, generator=gen, dtype=torch.float64))
    N, Lq = 2, 6
    f64 = dict(dtype=torch.float64)
    query = torch.randn(N, Lq, d_model, generator=gen, **f64)
    flat = torch.randn(N, S, d_model, generator=gen, **f64)
    if c["ref"] == 2:
        ref = torch.rand(N, Lq, L, 2, generator=gen, **f64)
    else:
        ref = torch.cat([torch.rand(N, Lq, L, 2, generator=gen, **f64),
                         0.1 + 0.5 * torch.rand(N, Lq, L, 2, generator=gen, **f64)], -1)
    mask = torch.rand(N, S, generator=gen) < 0.25
    go = torch.randn(N, Lq, d_model, generator=gen, **f64)
    shapes = torch.tensor(levels, dtype=torch.int64)
    starts = torch.tensor(_starts(levels))
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    q, r, x = (t.clone().requires_grad_(True) for t in (query, ref, flat))
    out = m(q, r, x, shapes, starts, mask)
    (out * go).sum().backward()
    return dict(cfg=c["cfg"], sigmoid_attn=c["sigmoid"], state_dict=sd, query=query, reference_points=ref,
                input_flatten=flat, input_spatial_shapes=shapes, input_level_start_index=starts,
                input_padding_mask=mask, grad_out=go, out=out.detach(),
                param_grads={k: p.grad.detach().clone() for k, p in m.named_parameters()},
                grad_query=q.grad, grad_reference_points=r.grad, grad_input_flatten=x.grad)


def schema(sd):
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def main():
    dino_mod, dino_fn = _import_ops(DINO_DIR, "dino")
    motr_mod, _ = _import_ops(MOTR_DIR, "motr")
    gen = torch.Generator().manual_seed(20261018)
    core = {name: core_case(dino_fn, c, gen) for name, c in CORE_CASES.items()}
    torch.save(core, GOLDEN / "msda_core.pt")
    modules = {name: module_case(motr_mod if c["sigmoid"] else dino_mod, c, gen) for name, c in MODULE_CASES.items()}
    torch.save(modules, GOLDEN / "msda_module.pt")
    torch.manual_seed(0)
    small = dino_mod.MSDeformAttn(32, 3, 4, 2)
    sch = dict(dino=schema(dino_mod.MSDeformAttn().state_dict()),
               motr=schema(motr_mod.MSDeformAttn(sigmoid_attn=True).state_dict()),
               default_offsets_bias=dino_mod.MSDeformAttn().sampling_offsets.bias.detach().clone(),
               im2col_step=dino_mod.MSDeformAttn().im2col_step,
               seed0_cfg=(32, 3, 4, 2), seed0_state_dict={k: v.clone() for k, v in small.state_dict().items()})
    torch.save(sch, GOLDEN / "msda_schema.pt")
    for f in ("msda_core.pt", "msda_module.pt", "msda_schema.pt"):
        print(f"wrote tests/golden/{f} ({(GOLDEN / f).stat().st_size / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
