"""Multi-scale deformable attention without a GPU: the fp64 oracle against the reference goldens
(oracle/make_golden_msda.py), the module's parameter schema and initialisation, the module's own arithmetic with the
oracle in place of the kernel, and the argument errors of MSDeformAttnFunction."""
from __future__ import annotations

from pathlib import Path

import pytest
import torch

from fastervit_b200 import deform
from fastervit_b200.deform import MSDeformAttn, MSDeformAttnFunction
from fastervit_b200.lib import FvitError
from oracle import msda_oracle

GOLDEN = Path(__file__).resolve().parent / "golden"
CORE = torch.load(GOLDEN / "msda_core.pt")
MODULES = torch.load(GOLDEN / "msda_module.pt")
SCHEMA = torch.load(GOLDEN / "msda_schema.pt")


def _close(got, want, tol):
    err = (got - want).abs().max().item()
    assert err <= tol * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize("case", sorted(CORE))
def test_oracle_matches_reference_core(case):
    c = CORE[case]
    out, gv, gs, ga = msda_oracle.ms_deform_attn_grads(c["value"], c["spatial_shapes"], c["sampling_locations"],
                                                       c["attention_weights"], c["grad_out"], c["level_start_index"])
    _close(out, c["out"], 1e-12)
    _close(gv, c["grad_value"], 1e-12)
    _close(gs, c["grad_sampling_locations"], 1e-12)
    _close(ga, c["grad_attention_weights"], 1e-12)


def test_golden_cases_cover_the_edges():
    locs = torch.cat([c["sampling_locations"].flatten() for c in CORE.values()])
    assert locs.min() < 0 and locs.max() > 1
    levels = torch.cat([c["spatial_shapes"] for c in CORE.values()])
    assert (levels[:, 0] == 1).any() and (levels[:, 1] == 1).any()
    assert any(c["value"].shape[-1] % 2 == 1 for c in CORE.values())


def _schema(sd):
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def test_module_schema_and_init():
    assert _schema(MSDeformAttn().state_dict()) == SCHEMA["dino"]
    assert _schema(MSDeformAttn(sigmoid_attn=True).state_dict()) == SCHEMA["motr"]
    m = MSDeformAttn()
    assert m.im2col_step == SCHEMA["im2col_step"]
    assert torch.equal(m.sampling_offsets.bias.detach(), SCHEMA["default_offsets_bias"])
    torch.manual_seed(0)
    small = MSDeformAttn(*SCHEMA["seed0_cfg"])
    sd = small.state_dict()
    assert list(sd) == list(SCHEMA["seed0_state_dict"])
    for k, v in SCHEMA["seed0_state_dict"].items():
        assert torch.equal(sd[k], v), k


@pytest.mark.parametrize("case", sorted(MODULES))
def test_reference_state_dict_loads_strict(case):
    c = MODULES[case]
    m = MSDeformAttn(*c["cfg"], sigmoid_attn=c["sigmoid_attn"]).double()
    m.load_state_dict(c["state_dict"], strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, c["state_dict"][k]), k


class _OracleFunction:
    """MSDeformAttnFunction with the fp64 oracle in place of the kernel (runs on the CPU)."""

    @staticmethod
    def apply(value, shapes, starts, locations, weights, im2col_step):
        return msda_oracle.ms_deform_attn_core(value, shapes, locations, weights, starts)


def run_module(c, device="cpu", dtype=torch.float64):
    """(out, param grads, grad query, grad reference_points, grad input_flatten) of golden module case c."""
    m = MSDeformAttn(*c["cfg"], sigmoid_attn=c["sigmoid_attn"]).to(device=device, dtype=dtype)
    m.load_state_dict(c["state_dict"])
    q, r, x = (c[k].to(device=device, dtype=dtype).requires_grad_(True)
               for k in ("query", "reference_points", "input_flatten"))
    out = m(q, r, x, c["input_spatial_shapes"].to(device), c["input_level_start_index"].to(device),
            c["input_padding_mask"].to(device))
    (out * c["grad_out"].to(device=device, dtype=dtype)).sum().backward()
    return out.detach(), {k: p.grad for k, p in m.named_parameters()}, q.grad, r.grad, x.grad


@pytest.mark.parametrize("case", sorted(MODULES))
def test_module_with_oracle_core_matches_reference(case, monkeypatch):
    monkeypatch.setattr(deform, "MSDeformAttnFunction", _OracleFunction)
    c = MODULES[case]
    out, pg, gq, gr, gx = run_module(c)
    _close(out, c["out"], 1e-12)
    for k, g in c["param_grads"].items():
        _close(pg[k], g, 1e-12)
    _close(gq, c["grad_query"], 1e-12)
    _close(gr, c["grad_reference_points"], 1e-12)
    _close(gx, c["grad_input_flatten"], 1e-12)


def test_module_rejects_reference_points_of_other_widths(monkeypatch):
    monkeypatch.setattr(deform, "MSDeformAttnFunction", _OracleFunction)
    c = MODULES["dino_ref2"]
    m = MSDeformAttn(*c["cfg"]).double()
    ref = torch.rand(*c["reference_points"].shape[:-1], 3, dtype=torch.float64)
    with pytest.raises(ValueError, match="2 or 4"):
        m(c["query"], ref, c["input_flatten"], c["input_spatial_shapes"], c["input_level_start_index"])


def test_module_rejects_indivisible_width():
    with pytest.raises(ValueError, match="divisible"):
        MSDeformAttn(d_model=30, n_heads=8)


def _core_args(N=2, Lq=3, M=2, D=4, L=2, P=2, levels=((4, 3), (2, 2))):
    S = sum(h * w for h, w in levels)
    return [torch.randn(N, S, M, D), torch.tensor(levels, dtype=torch.int64),
            torch.tensor([0, levels[0][0] * levels[0][1]], dtype=torch.int64)[:L],
            torch.rand(N, Lq, M, L, P, 2), torch.rand(N, Lq, M, L, P)]


def _raises(args, match):
    with pytest.raises(FvitError, match=match):
        MSDeformAttnFunction.apply(*args, 64)


def test_function_rejects_cpu_tensors():
    _raises(_core_args(), "CUDA")


@pytest.mark.parametrize("i", [0, 3, 4])
def test_function_rejects_other_float_dtypes(i):
    for dt in (torch.float64, torch.float16):
        args = _core_args()
        args[i] = args[i].to(dt)
        _raises(args, "float32")


@pytest.mark.parametrize("i", [1, 2])
def test_function_rejects_int32_geometry(i):
    args = _core_args()
    args[i] = args[i].int()
    _raises(args, "int64")


@pytest.mark.parametrize("i", [0, 3, 4])
def test_function_rejects_non_contiguous(i):
    args = _core_args()
    args[i] = args[i].transpose(0, 1).contiguous().transpose(0, 1)
    assert not args[i].is_contiguous()
    _raises(args, "contiguous")


def test_function_rejects_disagreeing_shapes():
    args = _core_args()
    args[0] = args[0][:, :, :1].contiguous()          # M of value != M of the locations
    _raises(args, "sampling_locations")
    args = _core_args()
    args[4] = args[4][:, :, :, :, :1].contiguous()    # P of the weights != P of the locations
    _raises(args, "attention_weights")
    args = _core_args()
    args[2] = args[2][:1].contiguous()                # one start index for two levels
    _raises(args, "level_start_index")
    args = _core_args()
    args[3] = args[3][..., :1].contiguous()           # locations without their y
    _raises(args, "sampling_locations")
    args = _core_args()
    args[0] = args[0][0]                              # value without its batch dimension
    _raises(args, "value")


def test_function_rejects_more_than_16_levels():
    L = 17
    levels = tuple((1, 1) for _ in range(L))
    args = [torch.randn(1, L, 1, 4), torch.tensor(levels, dtype=torch.int64), torch.arange(L),
            torch.rand(1, 2, 1, L, 1, 2), torch.rand(1, 2, 1, L, 1)]
    _raises(args, "at most 16")
