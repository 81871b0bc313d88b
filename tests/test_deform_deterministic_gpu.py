"""The deterministic backward of multi-scale deformable attention (fvit_msda_bwd_deterministic), which
MSDeformAttnFunction runs under torch.use_deterministic_algorithms: grad_value bitwise reproducible and independent of
the order of the samples and of the inputs' alignment, as accurate as the default backward against the fp64 oracle,
NaN for non-finite inputs; and with the flag off the backward launches exactly what it launched before.

The flag is only turned on through the `flag` fixture, which restores the previous setting. The fp64 oracle runs with
the flag off (its gather backward is not this library's to make deterministic)."""
from __future__ import annotations

from pathlib import Path

import pytest
import torch

from fastervit_b200 import lib
from fastervit_b200.deform import MSDeformAttnFunction
from test_deform_gpu import ENC4, ENC5, MODULES, SMALL, kernel, make_case, oracle, rel, run_module

pytestmark = pytest.mark.gpu


@pytest.fixture
def flag():
    """set(on, warn_only=False) switches torch.use_deterministic_algorithms; the previous setting is restored."""
    prev = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()

    def set_(on: bool, warn_only: bool = False):
        torch.use_deterministic_algorithms(on, warn_only=warn_only)

    yield set_
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


@pytest.fixture
def calls(monkeypatch):
    """Names of the library entry points MSDeformAttnFunction calls, in order."""
    names = []
    real = lib.call

    def record(name, *args):
        names.append(name)
        return real(name, *args)

    monkeypatch.setattr(lib, "call", record)
    return names


def sigmoid_weights(case, seed=5):
    """the MOTRv2 variant: independent sigmoid weights, most of them above 1 / (L * P)"""
    value, shapes, starts, loc, w, go = case
    g = torch.Generator(device="cuda").manual_seed(seed)
    return value, shapes, starts, loc, torch.sigmoid(2 * torch.randn(w.shape, device="cuda", generator=g)), go


def edge_locations(case, seed=6):
    """locations exactly at 0 and 1, and outside on either side"""
    value, shapes, starts, loc, w, go = case
    g = torch.Generator(device="cuda").manual_seed(seed)
    edge = torch.tensor([0.0, 1.0, -0.25, 1.25, 0.0, 1.0, -1.5, 2.0, 0.5], device="cuda")
    idx = torch.randint(0, len(edge), loc.shape, device="cuda", generator=g)
    return value, shapes, starts, edge[idx], w, go


def _enc4():
    S = sum(h * w for h, w in ENC4)
    return make_case(N=2, Lq=S, M=8, D=32, P=4, levels=ENC4)


def _dec():
    return make_case(N=2, Lq=1100, M=8, D=32, P=4, levels=ENC4, seed=1)


def _width(D):
    return lambda: make_case(N=2, Lq=37, M=3, D=D, P=3, levels=[(9, 7), (5, 4), (3, 2)], seed=D, lo=-0.3, hi=1.3)


CASES = {
    "dino_enc_4scale": _enc4,
    "dino_decoder_lq1100": _dec,
    **{f"D{D}": _width(D) for D in (1, 3, 32, 33, 3096)},
    "sigmoid_weights": lambda: sigmoid_weights(_dec()),
    "edge_locations": lambda: edge_locations(make_case(N=2, Lq=64, M=4, D=8, P=4, levels=[(5, 3), (1, 1), (2, 6)])),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_bitwise_reproducible_and_order_independent(name, flag):
    value, shapes, starts, loc, w, go = CASES[name]()
    flag(True)
    first = kernel(value, shapes, starts, loc, w, go)
    second = kernel(value, shapes, starts, loc, w, go)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    # the same samples with the queries in another order: grad_value sums the same contributions in another order
    perm = torch.randperm(loc.shape[1], device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    permuted = kernel(value, shapes, starts, loc[:, perm].contiguous(), w[:, perm].contiguous(),
                      go[:, perm].contiguous())
    assert torch.equal(permuted[1], first[1])
    assert torch.equal(permuted[2], first[2][:, perm]) and torch.equal(permuted[3], first[3][:, perm])
    assert torch.count_nonzero(first[1]) > 0


def _kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_alignment_does_not_change_the_gradients(flag):
    # the deterministic backward runs one channel per lane for any alignment; the default backward takes that layout
    # (msda_bwd_kernel<1>) only for a value that is not 16-byte aligned, and its location and weight gradients come
    # from the same source (compiled into differently ordered fp32 code)
    value, shapes, starts, loc, w, go = _dec()
    buf = torch.empty(value.numel() + 1, device="cuda")
    shifted = buf[1:].view(value.shape)
    shifted.copy_(value)
    assert shifted.data_ptr() % 16 == 4 and shifted.is_contiguous()
    default_scalar = kernel(shifted, shapes, starts, loc, w, go)
    flag(True)
    aligned = kernel(value, shapes, starts, loc, w, go)
    unaligned = kernel(shifted, shapes, starts, loc, w, go)
    for a, b in zip(aligned, unaligned):
        assert torch.equal(a, b)
    assert rel(aligned[2], default_scalar[2].double()) <= 1e-6
    assert rel(aligned[3], default_scalar[3].double()) <= 1e-6


ACCURACY = {
    "enc_4scale": lambda: make_case(N=2, Lq=sum(h * w for h, w in ENC4), M=8, D=32, P=4, levels=ENC4),
    "enc_5scale": lambda: make_case(N=2, Lq=sum(h * w for h, w in ENC5), M=8, D=32, P=4, levels=ENC5),
    "decoder": _dec,
    **{f"ref_D{D}": (lambda D=D: make_case(N=1, Lq=2, M=2, D=D, P=2, levels=SMALL, seed=D))
       for D in (30, 32, 64, 71, 1025, 2048, 3096)},
    **{f"narrow_D{D}": (lambda D=D: make_case(N=3, Lq=9, M=3, D=D, P=3, levels=[(5, 7), (1, 4), (3, 1)], seed=D,
                                              lo=-0.6, hi=1.6)) for D in (1, 2, 3, 5, 36)},
    "edges": lambda: edge_locations(make_case(N=1, Lq=1, M=2, D=8, P=4, levels=[(5, 3), (1, 1), (2, 6)])),
}


@pytest.mark.parametrize("name", sorted(ACCURACY))
def test_accuracy_against_fp64_and_default_path(name, flag):
    case = ACCURACY[name]()
    want = oracle(*case)
    default = kernel(*case)
    flag(True)
    got = kernel(*case)
    assert torch.equal(got[0], default[0])
    assert rel(got[2], default[2].double()) <= 1e-5 and rel(got[3], default[3].double()) <= 1e-5
    for gname, a, b in zip(("grad_value", "grad_sampling_locations", "grad_attention_weights"), got[1:], want[1:]):
        assert rel(a, b) <= 1e-4, (gname, rel(a, b))
    assert rel(got[1], default[1].double()) <= 1e-4


def test_contention_accuracy(flag):
    # every sample of every query lands on the centre of one pixel of each level: thousands of sums per element
    N, Lq, M, D, P, levels = 2, 4096, 8, 32, 4, [(8, 8), (4, 4)]
    value, shapes, starts, loc, w, go = make_case(N, Lq, M, D, P, levels)
    loc.copy_(torch.tensor([(2 + 0.5) / 8, (5 + 0.5) / 8], device="cuda"))
    loc[:, :, :, 1] = torch.tensor([(1 + 0.5) / 4, (2 + 0.5) / 4], device="cuda")
    go.uniform_(0.0, 1.0)
    want = oracle(value, shapes, starts, loc, w, go)
    flag(True)
    got = kernel(value, shapes, starts, loc, w, go)
    assert rel(got[1], want[1]) <= 1e-5
    assert torch.equal(got[1], kernel(value, shapes, starts, loc, w, go)[1])


@pytest.mark.parametrize("case", sorted(MODULES))
def test_module_matches_reference_goldens(case, flag, calls):
    # warn_only counts as enabled; with it the module's Linears run too (cuBLAS determinism is PyTorch's matter)
    c = MODULES[case]
    flag(True, warn_only=True)
    out, pg, gq, gr, gx = run_module(c)
    assert calls == ["fvit_msda_fwd", "fvit_msda_bwd_deterministic"]
    assert rel(out, c["out"]) <= 1e-5
    for k, g in c["param_grads"].items():
        assert rel(pg[k], g) <= 1e-4, k
    for name, got in (("grad_query", gq), ("grad_reference_points", gr), ("grad_input_flatten", gx)):
        assert rel(got, c[name]) <= 1e-4, name


CORE = torch.load(Path(__file__).resolve().parent / "golden" / "msda_core.pt")


@pytest.mark.parametrize("case", sorted(CORE))
def test_core_matches_reference_goldens(case, flag):
    c = CORE[case]
    args = [c[k].cuda() for k in ("value", "spatial_shapes", "level_start_index", "sampling_locations",
                                  "attention_weights", "grad_out")]
    args = [t.float() if t.is_floating_point() else t for t in args]
    flag(True)
    got = kernel(*args)
    for k, a in zip(("out", "grad_value", "grad_sampling_locations", "grad_attention_weights"), got):
        assert rel(a, c[k]) <= (1e-5 if k == "out" else 1e-4), k


@pytest.mark.parametrize("where", ["grad_out_inf", "grad_out_nan", "weight_inf"])
def test_non_finite_inputs_give_non_finite_grad_value(where, flag):
    value, shapes, starts, loc, w, go = _width(32)()
    if where == "grad_out_inf":
        go[0, 3, 5] = float("inf")
    elif where == "grad_out_nan":
        go[1, 0, 0] = float("nan")
    else:
        w[0, 1, 2, 0, 1] = float("inf")
    flag(True)
    gv = kernel(value, shapes, starts, loc, w, go)[1]
    assert torch.isnan(gv).all()


def test_default_path_launches_as_before(flag, calls):
    value, shapes, starts, loc, w, go = _dec()
    v = value.clone().requires_grad_(True)
    out = MSDeformAttnFunction.apply(v, shapes, starts, loc, w, 64)
    lib.reset_launch_count()
    calls.clear()
    out.backward(go)
    torch.cuda.synchronize()
    assert calls == ["fvit_msda_bwd"] and lib.launch_count() == 1
    names = _kernel_names(lambda: MSDeformAttnFunction.apply(v, shapes, starts, loc, w, 64).backward(go))
    assert any("msda_bwd_kernel<4>" in n for n in names), names
    assert not any("fixed" in n or "msda_bound" in n for n in names), names

    # the flag on: the bound pass, the fixed-point accumulation and the conversion
    flag(True)
    out = MSDeformAttnFunction.apply(v, shapes, starts, loc, w, 64)
    lib.reset_launch_count()
    calls.clear()
    out.backward(go)
    torch.cuda.synchronize()
    assert calls == ["fvit_msda_bwd_deterministic"] and lib.launch_count() == 3


def test_cuda_graph_replay_equals_eager(flag):
    value, shapes, starts, loc, w, go = make_case(N=2, Lq=300, M=8, D=32, P=4, levels=ENC4)
    v, s, a = (t.clone().requires_grad_(True) for t in (value, loc, w))
    flag(True)

    def step():
        out = MSDeformAttnFunction.apply(v, shapes, starts, s, a, 64)
        return (out, *torch.autograd.grad(out, (v, s, a), go))

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    eager = [t.clone() for t in step()]
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(static, eager):
        assert torch.equal(x, y)

