"""Every compiled fvit_gemm kernel variant against the fp64 reference of _gemm_variants.py, at the edges the plans
reach: a single row, partial last M / N tiles, 8- and 16-wide last N tiles, odd n, K = 8 / 196 (tail 4) / 784, the
library's own tile width, 48 and 256 (two 128-wide tiles), more than three work units per CTA, both B layouts. Each
call must land on its variant, keep every element it may not write bitwise at its sentinel, meet the per-element
bound, and match the generic kernel bit for bit on the same call with an exact no-op feature added."""
import pytest
import torch

from fastervit_b200 import lib as L

import _gemm_variants as V

pytestmark = pytest.mark.gpu

_WORST = {}   # largest error / bound per variant (reported by the last test)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _grid(r: V.Recipe):
    """(m, n, kc, tile_n, b_mn) of the edge grid for recipe r; b_mn None = the recipe's own layout."""
    btaps = "b_taps" in r.sig
    n16 = 48 if (r.direct or btaps) else 40          # last N tile of a 32-wide tiling: 16 / 8 columns
    # 3 N tiles (128, 128, 16) per tap x (SMs + 1) M tiles (5 M tiles x 27 N tiles x split-K for the weight gradient)
    m_multi = 5 * 128 - 37 if btaps else (_sms() + 1) * 128 - 37
    out = [(1, 64, 8, 0, None),
           (77, n16, 196, 32, None),
           (m_multi, 272, 196, 256, None)]
    if not r.direct and not btaps:
        out.append((77, 27, 784, 0, None))
    if not btaps and "taps" not in r.sig:
        out.append((300, 208, 784, 48, not r.b_mn))      # the other B layout; N tiles 48 x 4 + 16
    else:
        out.append((300, 208, 784, 48, None))
    return out


def _generic_twin(r: V.Recipe, m, n, kc, **kw) -> V.Case:
    """The same call with an exact no-op feature added that sends it to the generic kernel: col_scale2 = ones, else
    row_scale = ones, else BatchNorm statistics (an extra output)."""
    for extra in (dict(ones_cs2=True), dict(ones_rs=True), dict(add_stats=True)):
        if (extra.get("ones_cs2") and r.has(V.CS2)) or (extra.get("ones_rs") and r.has(V.RS)):
            continue
        if extra.get("add_stats") and r.has(V.ATOMIC):
            continue
        twin = r(m, n, kc, **kw, **extra)
        if twin.variant() == L.GEMM_F_GENERIC:
            return twin
    raise AssertionError(f"no generic twin for {V.name(r.variant)}")


_ATOMIC_OUTS = ("col_sum", "col_sumsq", "out_colsum")


def _run_and_check(r, m, n, kc, **kw):
    case = r(m, n, kc, **kw)
    assert case.variant() == r.variant, (V.name(case.variant()), V.name(r.variant))
    case.run()
    torch.cuda.synchronize()
    worst = V.check_case(case)
    _WORST[r.variant] = max(_WORST.get(r.variant, 0.0), worst)
    return case


@pytest.mark.parametrize("variant", sorted(V.RECIPES), ids=[V.name(v) for v in sorted(V.RECIPES)])
def test_variant_edge_grid(variant):
    r = V.RECIPES[variant]
    for i, (m, n, kc, tile_n, b_mn) in enumerate(_grid(r)):
        kw = dict(tile_n=tile_n, b_mn=b_mn, seed=i)
        case = _run_and_check(r, m, n, kc, **kw)
        twin = _generic_twin(r, m, n, kc, **kw)
        twin.run()
        torch.cuda.synchronize()
        V.check_case(twin)
        for k, o in case.outs.items():
            if k in _ATOMIC_OUTS or r.has(V.ATOMIC):
                continue   # float atomics in a different order: both checked against the bound
            if k == "out_f32" and r.has(V.RESID) and (r.has(V.CS2) or r.has(V.RS)):
                # the specialisations contract v * col_scale2 * row_scale + resid into one fma, the generic kernel
                # (run-time switches between them) rounds the product first: a few ulps apart, both within the bound
                continue
            assert torch.equal(V.bits(o.buf), V.bits(twin.outs[k].buf)), (V.name(variant), k, (m, n, kc, tile_n))
    for sig in r.extra_sigs:   # the other signatures the plans launch the variant with
        n = 48 if (r.direct or "b_taps" in sig) else 40
        _run_and_check(r, 300, n, 196, tile_n=32, sig=sig)


@pytest.mark.parametrize("variant", sorted(v for v in V.RECIPES if not V.RECIPES[v].direct),
                         ids=[V.name(v) for v in sorted(V.RECIPES) if not V.RECIPES[v].direct])
def test_staged_variants_scalar_store_path(variant):
    """Leading dimensions that are not multiples of 4 (fp32) / 8 (fp16): the element-wise loads and stores of every
    staged variant (vec_ok = 0), for each signature the plans launch it with."""
    r = V.RECIPES[variant]
    n = 48 if "b_taps" in r.sig else 40
    for sig in (r.sig, *r.extra_sigs):
        case = _run_and_check(r, 77, n, 196, tile_n=32, vec=False, sig=sig)
        assert not V.vec_ok(L._gemm_args(**case.kw))


def test_stem_weight_gradient_shape():
    """The stem's first convolution weight gradient of every training step: m = 16, n = 27, ld 27 (scalar atomics),
    K = 25088 output pixels (batch 2 at 224^2), split-K 49, MN-major A and B, device-scalar alpha."""
    r = V.RECIPES[V.SPLITK_WGRAD]
    case = _run_and_check(r, 16, 27, 25088, sig=V.STEM_WGRAD_SIG, split_k=49, ld32=27)
    assert case.kw["out_f32"].stride(0) == 27 and not V.vec_ok(L._gemm_args(**case.kw))


def _gelu_sweep(m, n):
    v = torch.linspace(-12.0, 12.0, m * n - 6, device="cuda", dtype=torch.float64)
    v = torch.cat([v, torch.tensor([60000.0, -60000.0, 0.0, -0.0, 0.0, 1e-4], device="cuda", dtype=torch.float64)])
    return v.view(m, n)


@pytest.mark.parametrize("variant,sig", [
    (V.A(2) | V.O16, ()),
    (V.DIRECT | V.A(2) | V.O16, ()),
    (V.A(2) | V.O16 | V.PRE | V.PREGRAD, ()),
    (V.DIRECT | V.A(2) | V.O16 | V.PRE | V.PREGRAD, ()),
    (V.A(3) | V.O16 | V.APTR, ()),
    (V.A(3) | V.O16, ("aux_scale", "row_map", "taps")),
    (V.A(5) | V.O16 | V.APTR, ()),
], ids=lambda x: V.name(x) if isinstance(x, int) else ",".join(x) or "-")
def test_gelu_edges(variant, sig):
    """Pre-activations over [-12, 12], +-60000 and exact zeros through GELU, the saved gelu' (pre_is_grad), the
    GELU_BWD multiply (with and without the BatchNorm affine on aux) and MUL_AUX, against fp64 erf-GELU."""
    r = V.RECIPES[variant]
    m, n = 128, 64
    pre = _gelu_sweep(m, n)
    kw = dict(sig=sig, gelu_pre=pre)
    case = r(m, n, 64 if r.act == L.ACT_GELU else 72, **kw)
    if r.act != L.ACT_GELU:   # the sweep is aux; the accumulator stays random
        assert torch.equal(case.kw["aux"].double(), pre.half().double())
    assert case.variant() == variant
    case.run()
    torch.cuda.synchronize()
    V.check_case(case)


def test_generic_only_features():
    """What no specialisation has: the ReLU-derivative epilogue, and bf16 operands through the whole epilogue."""
    relu_bwd = V.Recipe(V.A(L.ACT_RELU_BWD) | V.O16, ("aux_scale", "row_map"))
    case = relu_bwd(300, 200, 136, tile_n=64)
    assert case.variant() == L.GEMM_F_GENERIC
    case.run()
    torch.cuda.synchronize()
    V.check_case(case)
    full = V.Recipe(V.A(L.ACT_GELU) | V.RESID | V.O32 | V.O16 | V.PRE | V.CS2 | V.RS | V.STATS,
                    ("col_scale", "col_shift", "row_map"))
    case = full(300, 200, 136, bf16=True)
    assert case.kw["a"].dtype == torch.bfloat16 and case.variant() == L.GEMM_F_GENERIC
    case.run()
    torch.cuda.synchronize()
    V.check_case(case)


def test_zz_report_worst_ratio():
    """(last) every variant ran; the largest error / bound ratio seen, per variant"""
    if set(_WORST) != set(V.RECIPES):
        pytest.skip("only with the whole file")
    print("\nworst |err| / bound:", ", ".join(f"{V.name(v)} {x:.3f}" for v, x in sorted(_WORST.items())))
