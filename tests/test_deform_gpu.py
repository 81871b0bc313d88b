"""Multi-scale deformable attention kernels (fvit_msda_fwd / fvit_msda_bwd) on the GPU against the fp64 oracle built
from the fp32 inputs the kernel sees, and MSDeformAttn against the reference goldens.

Tolerances: the forward is within 1e-5 of max |ref| (each output is one fp32 sum of L*P*4 products); each gradient
is within 1e-4 of max |ref| of its tensor (sums over D channels, grad_value accumulated by float atomics). Test
locations are multiples of 2^-10, so that h = y*H - 0.5 and w = x*W - 0.5 are exact in fp32 too and both sides take
the same corners (the location gradient jumps where h or w crosses an integer)."""
from __future__ import annotations

from pathlib import Path

import pytest
import torch

from fastervit_b200.deform import MSDeformAttn, MSDeformAttnFunction
from oracle import msda_oracle

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"


def _levels(h, w, n):
    """n DETR levels (strides 8, 16, ...) of an h x w image, the backbone's ceil-halving."""
    out, hh, ww = [], -(-h // 8), -(-w // 8)
    for _ in range(n):
        out.append((hh, ww))
        hh, ww = -(-hh // 2), -(-ww // 2)
    return out


ENC4 = _levels(200, 333, 4)              # DINO 4-scale at 800 x 1333, scaled down by 4
ENC5 = [(50, 84)] + ENC4                 # 5-scale adds the stride-4 level
SMALL = [(6, 4), (3, 2)]                 # the reference test's levels


def make_case(N, Lq, M, D, P, levels, seed=0, lo=-0.2, hi=1.2):
    g = torch.Generator(device="cuda").manual_seed(seed)
    L, S = len(levels), sum(h * w for h, w in levels)
    dev = dict(device="cuda", generator=g)
    value = torch.randn(N, S, M, D, **dev)
    loc = lo + (hi - lo) * torch.rand(N, Lq, M, L, P, 2, **dev)
    loc = torch.round(loc * 1024) / 1024
    w = torch.rand(N, Lq, M, L, P, **dev)
    w = w / w.sum((-1, -2), keepdim=True)
    go = torch.randn(N, Lq, M * D, **dev)
    shapes = torch.tensor(levels, dtype=torch.int64, device="cuda")
    starts = torch.cat([shapes.new_zeros(1), (shapes[:, 0] * shapes[:, 1]).cumsum(0)[:-1]])
    return value, shapes, starts, loc, w, go


def kernel(value, shapes, starts, loc, w, go):
    v, s, a = (t.clone().requires_grad_(True) for t in (value, loc, w))
    out = MSDeformAttnFunction.apply(v, shapes, starts, s, a, 64)
    gv, gs, ga = torch.autograd.grad(out, (v, s, a), go)
    return out.detach(), gv, gs, ga


def oracle(value, shapes, starts, loc, w, go):
    return msda_oracle.ms_deform_attn_grads(value.double(), shapes, loc.double(), w.double(), go.double(), starts)


def rel(got, want):
    want = want.to(got.device)
    return ((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def check(case):
    got, want = kernel(*case), oracle(*case)
    assert got[0].shape == want[0].shape and got[0].dtype == torch.float32
    assert rel(got[0], want[0]) <= 1e-5, ("out", rel(got[0], want[0]))
    for name, a, b in zip(("grad_value", "grad_sampling_locations", "grad_attention_weights"), got[1:], want[1:]):
        assert rel(a, b) <= 1e-4, (name, rel(a, b))


@pytest.mark.parametrize("levels", [ENC4, ENC5], ids=["4scale", "5scale"])
def test_dino_encoder_shapes(levels):
    S = sum(h * w for h, w in levels)
    check(make_case(N=2, Lq=S, M=8, D=32, P=4, levels=levels))


def test_decoder_shape():
    # 900 queries + 2 x 100 denoising queries
    check(make_case(N=2, Lq=1100, M=8, D=32, P=4, levels=ENC4, seed=1))


@pytest.mark.parametrize("D", [30, 32, 64, 71, 1025, 2048, 3096])
def test_reference_channel_counts(D):
    check(make_case(N=1, Lq=2, M=2, D=D, P=2, levels=SMALL, seed=D))


@pytest.mark.parametrize("D", [1, 2, 3, 5, 36])
def test_narrow_and_odd_heads(D):
    check(make_case(N=3, Lq=9, M=3, D=D, P=3, levels=[(5, 7), (1, 4), (3, 1)], seed=D, lo=-0.6, hi=1.6))


def test_single_query_and_edges():
    value, shapes, starts, loc, w, go = make_case(N=1, Lq=1, M=2, D=8, P=4, levels=[(5, 3), (1, 1), (2, 6)])
    # locations exactly at 0 and 1, and outside on either side
    edge = torch.tensor([0.0, 1.0, -0.25, 1.25, 0.0, 1.0, -1.5, 2.0], device="cuda")
    loc.copy_(edge[torch.randint(0, len(edge), loc.shape, device="cuda")])
    check((value, shapes, starts, loc, w, go))
    w0 = torch.zeros_like(w)
    out, gv, gs, ga = kernel(value, shapes, starts, loc, w0, go)
    assert torch.count_nonzero(out) == 0 and torch.count_nonzero(gv) == 0 and torch.count_nonzero(gs) == 0
    want = oracle(value, shapes, starts, loc, w0, go)[3]
    assert rel(ga, want) <= 1e-4


def test_batch_not_divisible_by_im2col_step():
    value, shapes, starts, loc, w, go = make_case(N=3, Lq=5, M=2, D=16, P=2, levels=SMALL)
    out = MSDeformAttnFunction.apply(value, shapes, starts, loc, w, 2)
    ref = oracle(value, shapes, starts, loc, w, go)[0]
    assert rel(out, ref) <= 1e-5


def test_grad_value_contention():
    # every sample of every query lands on the centre of one pixel of each level: thousands of atomics per address
    N, Lq, M, D, P, levels = 2, 4096, 8, 32, 4, [(8, 8), (4, 4)]
    value, shapes, starts, loc, w, go = make_case(N, Lq, M, D, P, levels)
    loc.copy_(torch.tensor([(2 + 0.5) / 8, (5 + 0.5) / 8], device="cuda"))
    loc[:, :, :, 1] = torch.tensor([(1 + 0.5) / 4, (2 + 0.5) / 4], device="cuda")
    go.uniform_(0.0, 1.0)
    got, want = kernel(value, shapes, starts, loc, w, go), oracle(value, shapes, starts, loc, w, go)
    assert torch.count_nonzero(want[1].abs() > 0) == N * M * D * 2
    assert rel(got[1], want[1]) <= 1e-4
    assert rel(got[0], want[0]) <= 1e-5


def test_cuda_graph_replay_equals_eager():
    value, shapes, starts, loc, w, go = make_case(N=2, Lq=300, M=8, D=32, P=4, levels=ENC4)
    v, s, a = (t.clone().requires_grad_(True) for t in (value, loc, w))

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
    assert torch.equal(static[0], eager[0])
    assert torch.equal(static[2], eager[2]) and torch.equal(static[3], eager[3])   # no atomics: bitwise
    assert rel(static[1], eager[1].double()) <= 1e-6                               # atomics: order may differ


MODULES = torch.load(GOLDEN / "msda_module.pt")


def run_module(c, **autocast):
    m = MSDeformAttn(*c["cfg"], sigmoid_attn=c["sigmoid_attn"]).cuda()
    m.load_state_dict({k: v.float() for k, v in c["state_dict"].items()}, strict=True)
    q, r, x = (c[k].float().cuda().requires_grad_(True) for k in ("query", "reference_points", "input_flatten"))
    with torch.autocast("cuda", **autocast) if autocast else torch.enable_grad():
        out = m(q, r, x, c["input_spatial_shapes"].cuda(), c["input_level_start_index"].cuda(),
                c["input_padding_mask"].cuda())
    (out.float() * c["grad_out"].float().cuda()).sum().backward()
    return out, {k: p.grad for k, p in m.named_parameters()}, q.grad, r.grad, x.grad


@pytest.mark.parametrize("case", sorted(MODULES))
def test_module_matches_reference(case):
    c = MODULES[case]
    out, pg, gq, gr, gx = run_module(c)
    assert rel(out, c["out"]) <= 1e-5
    for k, g in c["param_grads"].items():
        assert rel(pg[k], g) <= 1e-4, k
    for name, got in (("grad_query", gq), ("grad_reference_points", gr), ("grad_input_flatten", gx)):
        assert rel(got, c[name]) <= 1e-4, name


@pytest.mark.parametrize("case", ["dino_ref2", "motr_sigmoid"])
def test_module_fp16_value(case):
    # under fp16 autocast value_proj yields fp16: it is sampled in fp32 and the output comes back in fp16
    c = MODULES[case]
    out, pg, gq, gr, gx = run_module(c, dtype=torch.float16)
    assert out.dtype == torch.float16
    assert rel(out, c["out"]) <= 1e-2
    assert rel(gx, c["grad_input_flatten"]) <= 2e-2
    assert rel(pg["value_proj.weight"], c["param_grads"]["value_proj.weight"]) <= 2e-2
