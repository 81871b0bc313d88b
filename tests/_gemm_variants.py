"""Recipes, an fp64 reference and a per-element comparator for the compiled kernel variants of fvit_gemm.

Every launch of fvit_gemm runs one compile-time instantiation of its kernel (a FVIT_GEMM_F_* feature mask, each with
its own folded epilogue code) or the generic kernel. RECIPES has one recipe per instantiated variant: called with a
shape it builds the operands, epilogue inputs and sentinel-filled output buffers of one lib.gemm call that lands on
that variant, using the optional inputs the model plans pass with it (its signature, recorded as plain data so the
CPU test can hold the plans' launches against it). `reference` evaluates the epilogue contract of include/fvit.h in
fp64 on the same 16-bit operands, together with a per-element error bound; `assert_within` compares against it.

Imports without a GPU (the CPU tests use the table and the comparator); the GPU file runs the recipes.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from fastervit_b200 import lib as L

U32 = 2.0 ** -24   # unit roundoff of fp32
U16 = 2.0 ** -11   # unit roundoff of fp16
HALF_SUB = 2.0 ** -25   # half the fp16 subnormal spacing: absolute rounding error near zero
# fp32 accumulation: |acc - exact| <= C_ACC * U32 * K * (|A| |B|^T)_ij. The tensor cores add the 16 products of an
# MMA step and the running sum with about one rounding per step, so the realistic error is a few U32 * (|A||B|^T),
# far below the worst case K U32 (|A||B|^T). Over the whole grid of test_gemm_variants_gpu.py the fp32 outputs stayed
# within 0.26 of their bound at C_ACC = 1/4 (H100 SXM, 700 W); 1/8 keeps a factor 2 of margin.
C_ACC = 0.125
# erf-GELU of the epilogue (common.h fvit_erf_core): Abramowitz-Stegun 7.1.26, |erf error| < 1.5e-7 in exact
# arithmetic. Evaluated in fp32: z = |x|/sqrt2 (1 rounding), t = rcp.approx(1 + p z) (rel. error <= 2^-23 + 1 fma
# rounding), the degree-5 Horner polynomial in t (5 fmas, all terms positive after the first two: <= 6 U32 relative),
# e = ex2.approx(-log2(e) z^2) (2^-22 relative, plus the 2 roundings of the argument, 2 U32 |arg| relative in e; with
# e |arg| <= log2(e) / e < 0.54), and 1 - poly e (1 fma). poly * e <= 1, so the fp32 evaluation adds at most
# (1 + 2 + 6 + 4 + 2 * 0.54 + 1) U32 < 16 U32 absolute, and 0.5 x (1 + erf) two more roundings: GELU_ERF bounds the
# erf the epilogue uses, and |gelu error| <= 0.5 |x| GELU_ERF + 2 U32 |gelu|.
GELU_ERF = 1.5e-7 + 16 * U32
GELU_LIP = 1.13     # max |gelu'(x)|  (at x ~ 2.4: 1.1289)
GELU_CURV = 0.80    # max |gelu''(x)| = phi(0) * 2

SIG_FIELDS = ("col_scale", "col_shift", "aux_scale", "row_map", "taps", "b_taps")


def signature_of(**present) -> tuple:
    """Optional-input signature of a call: which of SIG_FIELDS it passes (taps: ntaps > 1, b_taps: b_ntaps > 1)."""
    return tuple(f for f in SIG_FIELDS if present.get(f))


def act_bits(code: int) -> int:
    return code << L.GEMM_F_ACT_SHIFT


_FLAG_NAMES = [(L.GEMM_F_RESID, "RESID"), (L.GEMM_F_O32, "O32"), (L.GEMM_F_O16, "O16"), (L.GEMM_F_STATS, "STATS"),
               (L.GEMM_F_PRE, "PRE"), (L.GEMM_F_ATOMIC, "ATOMIC"), (L.GEMM_F_ALPHAPTR, "ALPHAPTR"),
               (L.GEMM_F_CS2, "CS2"), (L.GEMM_F_RS, "RS"), (L.GEMM_F_OSUM, "OSUM"), (L.GEMM_F_PREGRAD, "PREGRAD"),
               (L.GEMM_F_DIRECT, "DIRECT")]


def name(v: int) -> str:
    if v == L.GEMM_F_GENERIC:
        return "GENERIC"
    return "|".join([f"ACT{(v >> L.GEMM_F_ACT_SHIFT) & 7}"] + [s for bit, s in _FLAG_NAMES if v & bit])


@dataclass(frozen=True)
class Recipe:
    """One instantiated variant: its mask and the optional inputs the plans pass with it (`sig`; `extra_sigs` are
    further signatures the plans launch it with, each run once by the GPU file)."""
    variant: int
    sig: tuple
    extra_sigs: tuple = ()
    b_mn: bool = False          # the B layout of the plans' launches (the GPU grid also runs the other where allowed)
    a_mn: bool = False

    @property
    def act(self) -> int:
        return (self.variant >> L.GEMM_F_ACT_SHIFT) & 7

    def has(self, bit: int) -> bool:
        return bool(self.variant & bit)

    @property
    def direct(self) -> bool:
        return self.has(L.GEMM_F_DIRECT)

    def __call__(self, m, n, kc, **kw) -> "Case":
        return make_case(self, m, n, kc, **kw)


def _r(v, sig, extra=(), **kw):
    return Recipe(v, tuple(sig), tuple(tuple(s) for s in extra), **kw)


A = act_bits
O16, O32, RESID, STATS, PRE, ATOMIC, APTR, CS2, RS, OSUM, PREGRAD, DIRECT = (
    L.GEMM_F_O16, L.GEMM_F_O32, L.GEMM_F_RESID, L.GEMM_F_STATS, L.GEMM_F_PRE, L.GEMM_F_ATOMIC, L.GEMM_F_ALPHAPTR,
    L.GEMM_F_CS2, L.GEMM_F_RS, L.GEMM_F_OSUM, L.GEMM_F_PREGRAD, L.GEMM_F_DIRECT)
SPLITK_WGRAD = A(0) | O32 | ATOMIC | APTR

_RECIPE_LIST = [
    # inference / shared forward
    _r(A(0) | O16, ["col_shift"]),                                          # qkv + bias
    _r(A(2) | O16, ["col_shift"]),                                          # fc1 + bias
    _r(A(1) | O16, ["col_scale", "col_shift", "row_map"]),                  # eval stem conv1 (BatchNorm folded)
    _r(A(1) | O32 | O16, ["col_scale", "col_shift", "row_map", "taps"]),    # eval stem conv2
    _r(A(0) | RESID | O32, ["col_shift"],                                   # proj / fc2 + residual
       [["col_scale", "col_shift"], ["row_map", "taps"]]),                  # downsample into the stream, conv dgrad
    _r(A(0) | RESID | O32 | O16, ["col_scale", "col_shift", "row_map", "taps"]),   # eval conv2 + residual
    _r(A(0) | O32, ["col_shift"], [[], ["row_map", "taps"]]),               # head, downsample
    _r(A(0) | O32 | O16, ["row_map", "taps"]),                              # downsample -> next level
    # training forward
    _r(A(0) | O16 | STATS, ["col_shift", "row_map", "taps"], [["col_shift", "row_map"]]),   # conv + BN statistics
    _r(A(2) | O16 | PRE, ["col_shift"]),
    _r(A(2) | O16 | PRE | PREGRAD, ["col_shift"]),
    _r(A(0) | RESID | O32 | RS, ["col_shift"]),                             # branch + stochastic depth
    _r(A(0) | RESID | O32 | CS2 | PRE, ["col_shift"]),                      # branch with layer scale
    _r(A(0) | RESID | O32 | CS2 | PRE | RS, ["col_shift"]),
    # backward
    _r(SPLITK_WGRAD, ["b_taps"], a_mn=True, b_mn=True),                     # conv weight gradient, split-K
    _r(A(0) | O32 | APTR, [], [["b_taps"], ["row_map"]], a_mn=True, b_mn=True),   # weight gradient, one pass
    _r(A(0) | O16 | APTR, [], b_mn=True),                                   # data gradient
    _r(A(3) | O16 | APTR, [], b_mn=True),                                   # data gradient * gelu'
    _r(A(3) | O16, ["aux_scale", "row_map", "taps"]),                       # conv data gradient * gelu'(BatchNorm(aux))
    _r(A(3) | O16 | APTR | OSUM, [], b_mn=True),
    _r(A(5) | O16 | APTR, [], b_mn=True),                                   # fc2 data gradient * saved gelu'
    _r(A(5) | O16 | APTR | OSUM, [], b_mn=True),
    # row-per-thread (direct) forms
    _r(DIRECT | A(0) | O16, ["col_shift"], [[], ["row_map"], ["taps"], ["row_map", "taps"],
                                           ["col_shift", "row_map", "taps"]]),
    _r(DIRECT | A(1) | O16, ["col_scale", "col_shift", "row_map"]),
    _r(DIRECT | A(2) | O16, ["col_shift"], [["col_scale", "col_shift", "row_map", "taps"]]),
    _r(DIRECT | A(2) | O16 | PRE | PREGRAD, ["col_shift"]),
    _r(DIRECT | A(0) | O16 | APTR, [], b_mn=True),
    _r(DIRECT | A(3) | O16, ["aux_scale", "row_map", "taps"]),
    _r(DIRECT | A(5) | O16 | APTR, [], b_mn=True),
    _r(DIRECT | A(5) | O16 | APTR | OSUM, [], b_mn=True),
]
RECIPES = {r.variant: r for r in _RECIPE_LIST}

# the stem's first weight gradient: m = 16, n = 27 (3 x 3 x 3), ld 27, split-K over the output pixels
STEM_WGRAD_SIG = ()


def covered_triples() -> set:
    """(variant, signature, vec_ok) of every call the GPU file makes through the recipes."""
    out = set()
    for v, r in RECIPES.items():
        for sig in (r.sig, *r.extra_sigs):
            out.add((v, sig, True))
            if not r.direct:
                out.add((v, sig, False))   # test_staged_variants_scalar_store_path
    out.add((SPLITK_WGRAD, STEM_WGRAD_SIG, False))   # test_stem_weight_gradient_shape
    return out


def _ru(x, q):
    return -(-x // q) * q


# ---------------------------------------------------------------------------------------------------- cases
F32_SENTINEL = -7777.25
F16_SENTINEL_BITS = 0x7E5A   # a NaN payload: nothing the epilogue computes


def _f32_buf(rows, ld, dev):
    return torch.full((rows, ld), F32_SENTINEL, device=dev, dtype=torch.float32)


def _f16_buf(rows, ld, dev, h=torch.float16):
    return torch.full((rows, ld), F16_SENTINEL_BITS, device=dev, dtype=torch.int16).view(h)


@dataclass
class Out:
    buf: torch.Tensor          # the whole allocation (sentinel-filled)
    view: torch.Tensor         # what the call is given
    cols: int                  # logical columns written
    by_orow: bool              # rows are row_map[m] (else m)
    before: torch.Tensor       # a copy of buf before the call


class Case:
    """One lib.gemm call built by a recipe: `kw` are its arguments, `outs` its output buffers."""

    def __init__(self, recipe, m, n, kc, kw, outs, ops, vecs):
        self.recipe, self.m, self.n, self.kc = recipe, m, n, kc
        self.kw, self.outs, self.ops, self.vecs = kw, outs, ops, vecs

    def snapshot(self):
        for o in self.outs.values():
            o.before = o.buf.clone()

    def run(self):
        self.snapshot()
        L.gemm(**self.kw)

    def variant(self) -> int:
        return L.gemm_variant(**self.kw)


def _shift_rows(x: torch.Tensor, s: int) -> torch.Tensor:
    """y[i] = x[i + s], zero outside (what TMA's out-of-range fill gives a shifted box)"""
    y = torch.zeros_like(x)
    r = x.shape[0]
    if s >= 0:
        if s < r:
            y[: r - s] = x[s:]
    elif -s < r:
        y[-s:] = x[: r + s]
    return y


def make_case(r: Recipe, m: int, n: int, kc: int, *, tile_n: int = 0, b_mn: bool | None = None, vec: bool = True,
              sig: tuple | None = None, seed: int = 0, device="cuda", split_k: int = 7, alpha_val: float = 0.75,
              osum_alpha_val: float = 3 * 2.0 ** -9, gelu_pre=None, ones_cs2: bool = False, ones_rs: bool = False,
              add_stats: bool = False, bf16: bool = False, ld32: int | None = None) -> Case:
    """Operands and epilogue inputs of one call of variant r at [m, n] x kc.

    vec=False: leading dimensions that defeat the 16-byte store path (fp32 ld = 1 mod 4, fp16 ld = 1 mod 8).
    gelu_pre: optional [m, n] fp64 values the pre-activation should take (GELU edge sweeps: the operands then make
    the accumulator exactly these values rounded to fp16). ones_cs2 / ones_rs / add_stats add an exact no-op feature
    (the generic-kernel twin of the call). bf16: bf16 operands, aux and 16-bit outputs (generic kernel only)."""
    sig = r.sig if sig is None else sig
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(1000 * seed + 7 * m + 3 * n + kc)
    b_mn = r.b_mn if b_mn is None else b_mn
    taps = "taps" in sig
    btaps = "b_taps" in sig
    atomic = r.has(ATOMIC)
    ncols = 9 * n if btaps else n   # logical output columns
    kw: dict = dict(tile_n=tile_n, act=r.act)
    h = torch.bfloat16 if bf16 else torch.float16
    vecs: dict = {}
    # ---- operands
    if btaps:   # conv weight gradient: out[co][t n + ci] = sum_q A[q][co] B[q + s_t][ci]
        assert n % 4 == 0
        a = torch.randn(kc, _ru(m, 8), device=dev, generator=g).to(h)[:, :m]
        b = (torch.randn(kc, _ru(n, 8), device=dev, generator=g) / math.sqrt(kc)).to(h)[:, :n]
        P = 6
        shifts = [(dy - 1) * P + (dx - 1) for dy in range(3) for dx in range(3)]
        kw.update(a=a, b=b, a_mn=True, b_mn=True, b_taps=shifts, m=m, n=n, kc=kc)
        ae = a.double().t()
        be = [_shift_rows(b.double(), s).t() for s in shifts]
        acc = torch.cat([ae @ x.t() for x in be], 1)
        mag = torch.cat([ae.abs() @ x.abs().t() for x in be], 1)
        ktot = kc
    elif taps:  # 3x3 convolution: A rows shifted by (dy - 1) P + (dx - 1), out-of-range rows zero
        P = 10
        shifts = [(dy - 1) * P + (dx - 1) for dy in range(3) for dx in range(3)]
        kp = _ru(kc, 64)
        a = torch.randn(m, _ru(kc, 8) + 8, device=dev, generator=g).to(h)[:, :kc]
        w = (torch.randn(n, 9, kc, device=dev, generator=g) / math.sqrt(9 * kc)).to(h)
        b = torch.zeros(n, 9, kp, device=dev, dtype=h)
        b[:, :, :kc] = w
        b = b.view(n, 9 * kp)
        kw.update(a=a, b=b, taps=[(s, 0) for s in shifts], m=m, n=n, kc=kc)
        ae = torch.cat([_shift_rows(a.double(), s) for s in shifts], 1)
        be = w.double().reshape(n, 9 * kc)
        acc, mag = ae @ be.t(), ae.abs() @ be.abs().t()
        ktot = 9 * kc
    else:
        if r.a_mn:
            a = torch.randn(kc, _ru(m, 8), device=dev, generator=g).to(h)[:, :m]
            ae = a.double().t()
        else:
            a = torch.randn(m, _ru(kc, 8) + 8, device=dev, generator=g).to(h)[:, :kc]
            ae = a.double()
        if b_mn:
            b = (torch.randn(kc, _ru(n, 8), device=dev, generator=g) / math.sqrt(kc)).to(h)[:, :n]
            be = b.double().t()
        else:
            b = (torch.randn(n, _ru(kc, 8) + 8, device=dev, generator=g) / math.sqrt(kc)).to(h)[:, :kc]
            be = b.double()
        if gelu_pre is not None and r.act == L.ACT_GELU:   # A = [pre, 0...], B = identity: acc = pre exactly
            assert not r.a_mn and not b_mn and kc >= n
            a = torch.zeros(m, _ru(kc, 8) + 8, device=dev, dtype=h)
            a[:, :n] = gelu_pre.to(h)
            a = a[:, :kc]
            b = torch.zeros(n, _ru(kc, 8) + 8, device=dev, dtype=h)
            b[:, :n] = torch.eye(n, device=dev, dtype=h)
            b = b[:, :kc]
            ae, be = a.double(), b.double()
        kw.update(a=a, b=b, a_mn=r.a_mn, b_mn=b_mn, m=m, n=n, kc=kc)
        acc, mag = ae @ be.t(), ae.abs() @ be.abs().t()
        ktot = kc
    # ---- row map (scatter into a taller output; every 5th row dropped)
    rows_out = m + 3
    row_map = None
    if "row_map" in sig:
        rows_out = m + 37
        row_map = torch.randperm(rows_out, device=dev, generator=g)[:m].int()
        row_map[::5] = -1
        kw["row_map"] = row_map
        vecs["row_map"] = row_map
    # ---- per-column / per-row vectors
    if "col_scale" in sig:
        vecs["col_scale"] = kw["col_scale"] = torch.rand(ncols, device=dev, generator=g) + 0.5
    if "col_shift" in sig:
        vecs["col_shift"] = kw["col_shift"] = torch.randn(ncols, device=dev, generator=g) * 0.5
    if r.has(CS2) or ones_cs2:
        cs2 = torch.ones(ncols, device=dev) if ones_cs2 else torch.rand(ncols, device=dev, generator=g) * 0.5 + 0.75
        vecs["col_scale2"] = kw["col_scale2"] = cs2
    if r.has(RS) or ones_rs:
        if ones_rs:
            rs = torch.ones(m, device=dev)
        else:
            rs = torch.where(torch.rand(m, device=dev, generator=g) < 0.25, 0.0, 1.0 / 0.75)
        vecs["row_scale"] = kw["row_scale"] = rs
    if r.has(APTR):
        vecs["alpha_ptr"] = kw["alpha_ptr"] = torch.full((1,), alpha_val, device=dev)
    if atomic:
        kw["split_k"] = split_k
    if r.act in (L.ACT_GELU_BWD, L.ACT_RELU_BWD, L.ACT_MUL_AUX):
        ld = _ru(ncols, 16) + 16 if r.direct else _ru(ncols + 1, 8) + (0 if vec else 1)
        if r.act == L.ACT_MUL_AUX:
            aux = torch.rand(m, ld, device=dev, generator=g) * 1.2 - 0.1
        else:
            aux = torch.randn(m, ld, device=dev, generator=g) * 2.0
        if gelu_pre is not None:
            aux[:, :ncols] = gelu_pre
        aux = aux.to(h)
        vecs["aux"] = kw["aux"] = aux[:, :ncols]
        if "aux_scale" in sig:
            vecs["aux_scale"] = kw["aux_scale"] = torch.rand(ncols, device=dev, generator=g) + 0.5
            vecs["aux_shift"] = kw["aux_shift"] = torch.randn(ncols, device=dev, generator=g) * 0.5
    # ---- outputs (sentinel-filled, with padding columns and rows beyond the written ones)
    outs: dict = {}
    ld32 = ld32 or _ru(ncols + 1, 4) + (0 if vec else 1)
    if r.direct:
        ld16 = _ru(ncols, 16) + 16
    elif vec:
        ld16 = _ru(ncols + 1, 8)
        if ld16 % 16 == 0:
            ld16 += 8   # keeps the staged variants off their direct twins
    else:
        ld16 = _ru(ncols + 1, 8) + 1
    if r.has(RESID):
        res = torch.randn(rows_out, ld32, device=dev, generator=g)
        vecs["resid"] = kw["resid"] = res[:, :ncols]
    if r.has(O32):
        buf = _f32_buf(rows_out, ld32, dev)
        if atomic:
            buf[:m, :ncols] = 0.0   # split-K adds into a zeroed output
        outs["out_f32"] = Out(buf, buf[:, :ncols], ncols, True, buf)
    if r.has(O16):
        buf = _f16_buf(rows_out, ld16, dev, h)
        outs["out_f16"] = Out(buf, buf[:, :ncols], ncols, True, buf)
    if r.has(PRE):
        buf = _f16_buf(m + 3, ld16, dev, h)
        outs["out_pre16"] = Out(buf, buf[:, :ncols], ncols, False, buf)
        if r.has(PREGRAD):
            kw["pre_is_grad"] = True
    if r.has(STATS) or add_stats:
        for f in ("col_sum", "col_sumsq"):
            buf = torch.full((1, ncols + 4), F32_SENTINEL, device=dev)
            buf[0, :ncols] = torch.randn(ncols, device=dev, generator=g)
            outs[f] = Out(buf, buf[0, :ncols], ncols, False, buf)
    if r.has(OSUM):
        buf = torch.full((1, ncols + 4), F32_SENTINEL, device=dev)
        buf[0, :ncols] = torch.randn(ncols, device=dev, generator=g)
        outs["out_colsum"] = Out(buf, buf[0, :ncols], ncols, False, buf)
        vecs["out_colsum_alpha"] = kw["out_colsum_alpha"] = torch.full((1,), osum_alpha_val, device=dev)
    for k, o in outs.items():
        kw[k] = o.view
    case = Case(r, m, ncols, kc, kw, outs, dict(acc=acc, mag=mag, ktot=ktot, u16=2.0 ** -8 if bf16 else U16), vecs)
    case.snapshot()
    return case


# ---------------------------------------------------------------------------------------------------- reference
def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _phi(x):
    return torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def _gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * _phi(x)


def _gelu_err(x):
    return 0.5 * x.abs() * GELU_ERF + 2 * U32 * _gelu(x).abs()


def _gelu_grad_err(x):
    # cdf: 0.5 GELU_ERF; x phi(x) e-term: e relative error 2^-22 + 2 U32 |arg| (arg = x^2 / 2 log2 e), 3 roundings
    return 0.5 * GELU_ERF + x.abs() * _phi(x) * (8 + x * x) * U32 + 2 * U32 * _gelu_grad(x).abs()


def acc_bound(mag: torch.Tensor, k: int) -> torch.Tensor:
    return C_ACC * U32 * k * mag


def reference(case: Case, got16: torch.Tensor | None = None) -> dict:
    """fp64 value and per-element error bound of every output, m-indexed ([m, cols]; [cols] for column vectors).
    got16: the kernel's out_f16 (out_colsum sums the rounded 16-bit outputs the kernel wrote)."""
    r, vecs, kw = case.recipe, case.vecs, case.kw
    acc, mag, K, u16 = case.ops["acc"], case.ops["mag"], case.ops["ktot"], case.ops["u16"]
    d = lambda t: t.double()
    alpha = kw.get("alpha", 1.0) * (float(vecs["alpha_ptr"][0]) if "alpha_ptr" in vecs else 1.0)
    res: dict = {}
    if r.has(ATOMIC):   # only alpha; partial products added atomically
        v = alpha * acc
        e = (C_ACC * K + kw["split_k"]) * U32 * abs(alpha) * mag + U32 * v.abs()
        res["out_f32"] = (v, e)
        return res
    s = alpha * (d(vecs["col_scale"]) if "col_scale" in vecs else torch.ones_like(acc[0]))
    sh = d(vecs["col_shift"]) if "col_shift" in vecs else torch.zeros_like(acc[0])
    v1 = acc * s + sh
    e1 = acc_bound(mag, K) * s.abs() + U32 * ((acc * s).abs() + v1.abs())
    pre, epre = v1, e1
    act = r.act
    if act == L.ACT_RELU:
        v2, e2 = v1.clamp_min(0.0), e1
    elif act == L.ACT_GELU:
        v2, e2 = _gelu(v1), GELU_LIP * e1 + _gelu_err(v1)
        if r.has(PREGRAD):
            pre, epre = _gelu_grad(v1), GELU_CURV * e1 + _gelu_grad_err(v1)
    elif act in (L.ACT_GELU_BWD, L.ACT_RELU_BWD):
        a = d(vecs["aux"])
        ea = torch.zeros_like(a)
        if "aux_scale" in vecs:
            a = a * d(vecs["aux_scale"]) + d(vecs["aux_shift"])
            ea = U32 * a.abs()
        if act == L.ACT_GELU_BWD:
            gg = _gelu_grad(a)
            eg = GELU_CURV * ea + _gelu_grad_err(a)
            v2 = v1 * gg
            e2 = e1 * gg.abs() + v1.abs() * eg + U32 * v2.abs()
        else:
            v2 = torch.where(a > 0, v1, torch.zeros_like(v1))
            e2 = torch.where(a.abs() <= ea, v1.abs() + e1, e1)   # a sign the fp32 affine may round either way
    elif act == L.ACT_MUL_AUX:
        a = d(vecs["aux"])
        v2 = v1 * a
        e2 = e1 * a.abs() + U32 * v2.abs()
    else:
        v2, e2 = v1, e1
    f = torch.ones_like(v2)
    if "col_scale2" in vecs:
        f = f * d(vecs["col_scale2"])
    if "row_scale" in vecs:
        f = f * d(vecs["row_scale"])[:, None]
    v3 = v2 * f
    e3 = e2 * f.abs() + 2 * U32 * v3.abs()
    if "resid" in vecs:
        rm = vecs.get("row_map")
        rows = rm.long().clamp_min(0) if rm is not None else torch.arange(case.m, device=acc.device)
        v4 = v3 + d(vecs["resid"])[rows]
        e4 = e3 + U32 * v4.abs()
    else:
        v4, e4 = v3, e3
    if r.has(O32):
        res["out_f32"] = (v4, e4 + U32 * v4.abs())
    if r.has(O16):
        res["out_f16"] = (v4, e4 * (1 + u16) + u16 * v4.abs() + HALF_SUB)
    if r.has(PRE):
        res["out_pre16"] = (pre, epre * (1 + u16) + u16 * pre.abs() + HALF_SUB)
    valid = torch.ones(case.m, dtype=torch.bool, device=acc.device)
    if "row_map" in vecs:
        valid = vecs["row_map"] >= 0
    depth = 16 + 5 * -(-case.m // 128)   # longest chain of fp32 additions in the column reductions
    if "col_sum" in case.outs:
        base_s, base_q = d(case.outs["col_sum"].before[0, :case.n]), d(case.outs["col_sumsq"].before[0, :case.n])
        x, ex = v1[valid], e1[valid]
        s1 = base_s + x.sum(0)
        s2 = base_q + (x * x).sum(0)
        res["col_sum"] = (s1, ex.sum(0) + depth * U32 * (x.abs().sum(0) + base_s.abs()))
        res["col_sumsq"] = (s2, (2 * x.abs() * ex + ex * ex).sum(0) + (depth + 1) * U32 * (x * x).sum(0)
                            + depth * U32 * base_q.abs())
    if "out_colsum" in case.outs and got16 is not None:
        oa = float(vecs["out_colsum_alpha"][0])
        base = d(case.outs["out_colsum"].before[0, :case.n])
        rm = vecs.get("row_map")
        rows = rm[valid].long() if rm is not None else torch.arange(case.m, device=acc.device)
        x = d(got16[rows])
        res["out_colsum"] = (base + oa * x.sum(0),
                             depth * U32 * abs(oa) * x.abs().sum(0) + U32 * (base.abs() + abs(oa) * x.abs().sum(0)))
    return res


def assert_within(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """Every element within its own bound; returns the largest |got - ref| / bound."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        idx = bad.nonzero()[0].tolist()
        i = tuple(idx)
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound, e.g. {i}: got {got[i].item()!r} "
                             f"want {ref[i].item()!r} (|err| {err[i].item():.3g} > bound {bound[i].item():.3g})")
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def vec_ok(g) -> bool:
    """The launcher's 16-byte store rule (gemm_sm100.cu, p.vec_ok) on a filled GemmArgs."""
    ok = True
    for p, ld, q, al in ((g.out_f32, g.ld_out_f32, 4, 16), (g.out_f16, g.ld_out_f16, 8, 16),
                         (g.resid, g.ld_resid, 4, 16), (g.out_pre16, g.ld_out_pre16, 4, 8), (g.aux, g.ld_aux, 4, 8)):
        if p:
            ok = ok and ld % q == 0 and p % al == 0
    return ok


def check_case(case: Case) -> float:
    """Written elements against the fp64 reference, everything else bitwise equal to its sentinel. Returns the worst
    error / bound ratio."""
    worst = 0.0
    rm = case.vecs.get("row_map")
    m = case.m
    valid = torch.ones(m, dtype=torch.bool, device=case.ops["acc"].device) if rm is None else rm >= 0
    orow = torch.arange(m, device=valid.device) if rm is None else rm.long()
    got16 = None
    if "out_f16" in case.outs:
        got16 = case.outs["out_f16"].buf[:, :case.n].double()
    refs = reference(case, got16)
    for k, o in case.outs.items():
        written = torch.zeros(o.buf.shape, dtype=torch.bool, device=o.buf.device)
        if o.buf.shape[0] == 1:    # column vector
            written[0, :o.cols] = True
            got = o.buf[0, :o.cols]
            ref, bound = refs[k]
        else:
            rows = orow[valid] if o.by_orow else torch.arange(m, device=valid.device)[valid]
            written[rows, :o.cols] = True
            got = o.buf[rows, :o.cols]
            ref, bound = refs[k][0][valid], refs[k][1][valid]
        worst = max(worst, assert_within(got, ref, bound, f"{name(case.recipe.variant)} {k}"))
        nb, bb = bits(o.buf), bits(o.before)
        changed = (nb != bb) & ~written
        assert not changed.any(), f"{name(case.recipe.variant)} {k}: {int(changed.sum())} elements outside the " \
                                  f"written range changed, e.g. {tuple(changed.nonzero()[0].tolist())}"
    return worst
