"""Every attention entry point against fp64 at the geometry classes of tests/_attn_geometry.py, at softmax's edges, under
a narrowed persistent grid and at the SIMT kernels' own shapes, element by element.

Each result must sit within C_ATTN * U16 * M + U16 * |ref| (+ half an fp16 subnormal) of the fp64 reference on the same
fp16 operands, M being the reference formula on absolute values (_attn_geometry.reference), and within the whole-tensor
bars of tests/test_attn_gpu.py (2e-3 forward, 4e-3 backward). Every call also checks the memory contract:
  - outputs are windows of NaN-filled matrices: 16 columns either side and 3 rows past the end stay bitwise NaN, and
    head-pad columns come out exactly zero;
  - operands have a leading dimension past their width, NaN in the extra columns and in 3 rows past groups * S (the TMA
    maps cover exactly the declared extents, so a read outside an operand turns a result into NaN);
  - dbias is prefilled and must come back as prefill + gradient, with a NaN tail past heads * S * S;
  - the key-loop backward's fp32 dq scratch starts NaN-filled.
Lines starting "ratio" report the smallest C_ATTN each result would pass with (run with -s)."""
import zlib

import pytest
import torch

import _attn_geometry as G
from _attn_geometry import Case

pytestmark = pytest.mark.gpu

EDGE, TAIL, XCOL = 16, 3, 8   # sentinel columns either side of an output, rows past its end, extra operand columns


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


class Window:
    """a [rows, cols] output inside a NaN-filled [rows + TAIL, EDGE + cols + EDGE] matrix"""

    def __init__(self, rows, cols, dtype=torch.half):
        self.big = torch.full((rows + TAIL, EDGE + cols + EDGE), float("nan"), device="cuda", dtype=dtype)
        self.rows, self.cols = rows, cols
        self.t = self.big[:rows, EDGE:EDGE + cols]

    def ptr(self):
        return self.t.data_ptr()

    def ld(self):
        return self.big.stride(0)

    def untouched(self):
        b = self.big.view(torch.int16 if self.big.element_size() == 2 else torch.int32)
        nan = b[-1, 0].item()   # (never written: TAIL rows)
        return bool((b[:, :EDGE] == nan).all() and (b[:, EDGE + self.cols:] == nan).all() and (b[self.rows:] == nan).all())

    def check_sentinels(self, what):
        assert self.untouched(), f"{what}: a write outside the output window"


def _operand(x: torch.Tensor) -> torch.Tensor:
    """x [rows, cols] copied into a NaN-filled [rows + TAIL, cols + XCOL] matrix; returns the [rows, cols] view"""
    big = torch.full((x.shape[0] + TAIL, x.shape[1] + XCOL), float("nan"), device="cuda", dtype=x.dtype)
    big[:x.shape[0], :x.shape[1]] = x
    return big[:x.shape[0], :x.shape[1]]


def _with_tail(x: torch.Tensor, n=64) -> torch.Tensor:
    """flat fp32 copy of x followed by n NaNs; returns the big buffer"""
    big = torch.full((x.numel() + n,), float("nan"), device="cuda", dtype=torch.float32)
    big[:x.numel()] = x.reshape(-1)
    return big


def _padded(x: torch.Tensor, hdp: int) -> torch.Tensor:
    """[rows, n, heads, hd] -> [rows, n * heads * hdp] zero-padded"""
    rows, n, heads, hd = x.shape
    out = torch.zeros(rows, n, heads, hdp, device=x.device, dtype=x.dtype)
    out[..., :hd] = x
    return out.reshape(rows, n * heads * hdp)


# ---------------------------------------------------------------------------------------------- inputs
MODES = ["plain", "shift", "dominant first", "dominant last", "dominant tile", "uniform", "wide", "negative"]


def _dominant_key(c: Case, mode: str) -> int:
    if mode == "dominant first":
        return 0
    if mode == "dominant last":
        return c.S - 1
    # the last key of a 128-key tile when the window spans several, else a key in the middle of the window
    return 127 if c.S > 128 else c.S // 2


def inputs(c: Case, mode: str = "plain", seed: int = 0):
    """fp16 operands, bias and dO of a case under a softmax-edge mode. Returns a dict with the kernel's bias (`bias`,
    shifted in "shift" mode) and the reference's (`ref_bias`), and `shift` (per query row) for the lse check."""
    g = torch.Generator(device="cuda").manual_seed(1009 * seed + zlib.crc32(c.id.encode()) % 100003 + MODES.index(mode))
    rows, S, heads, hd = c.groups * c.S, c.S, c.heads, c.hd
    dev = "cuda"
    qk_mul = {"wide": 3.0, "negative": 0.5, "uniform": 0.0}.get(mode, 1.0)
    d = {}
    if c.entry == "fvit_hat_attn_fwd":
        x = torch.randn(rows, c.C, device=dev, generator=g).half()
        w = torch.zeros(3, heads, 64, c.C, device=dev)
        w[:, :, :hd] = torch.randn(3, heads, hd, c.C, device=dev, generator=g) * c.C ** -0.5
        w[:2] *= qk_mul
        qb = torch.zeros(3, heads, 64, device=dev)
        qb[:, :, :hd] = torch.randn(3, heads, hd, device=dev, generator=g) * 0.2
        qb[:2] *= qk_mul
        d.update(x=x, w16=w.reshape(3 * heads * 64, c.C).half(), qb=qb.reshape(-1).contiguous())
    else:
        qkv = torch.randn(rows, 3, heads, hd, device=dev, generator=g)
        qkv[:, :2] *= qk_mul
        d["qkv16"] = _padded(qkv, c.width).half()
    d["do16"] = _padded(torch.randn(rows, 1, heads, hd, device=dev, generator=g), c.width).half()
    bias = torch.randn(heads, S, S, device=dev, generator=g) * 2
    shift = torch.zeros(S, device=dev)
    if mode == "shift":
        shift = torch.where(torch.arange(S, device=dev) % 2 == 0, 80.0, -80.0)
    elif mode.startswith("dominant"):
        bias[:, :, _dominant_key(c, mode)] += 40
    elif mode == "uniform":
        bias = (torch.randn(heads, S, 1, device=dev, generator=g) * 2).expand(heads, S, S).contiguous()
    elif mode == "wide":
        bias = torch.randn(heads, S, S, device=dev, generator=g) * 20
    elif mode == "negative":
        bias = -130 + torch.randn(heads, S, S, device=dev, generator=g)
    d["ref_bias"] = bias.double()
    d["bias"] = (bias + shift[None, :, None]).contiguous()
    d["shift"] = shift
    return d


# ---------------------------------------------------------------------------------------------- one call
def run(c: Case, d: dict, sm_limit: int | None = None, dbias_prefill: torch.Tensor | None = None) -> dict:
    """Launch the case's entry point on `d` (inputs()) with every output inside NaN sentinels; returns the windows."""
    lib = _lib()
    rows, S, heads, hd, w = c.groups * c.S, c.S, c.heads, c.hd, c.width
    scale = hd ** -0.5
    use_bias = c.bias != "no_bias"
    bias_big = _with_tail(d["bias"]) if use_bias else None
    bptr = bias_big.data_ptr() if use_bias else None
    o = {}
    limit = c.sm_limit if sm_limit is None else sm_limit
    lib.load().fvit_set_sm_limit(limit)
    try:
        if c.entry == "fvit_hat_attn_fwd":
            x, w16 = _operand(d["x"]), _operand(d["w16"])
            o["out"] = Window(rows, heads * w)
            o["qkv_out"] = Window(rows, 3 * heads * w) if c.save_qkv else None
            lib.call("fvit_hat_attn_fwd", x.data_ptr(), x.stride(0), c.C, w16.data_ptr(), w16.stride(0),
                     d["qb"].data_ptr(), c.groups, S, heads, w, bptr, scale, o["out"].ptr(), o["out"].ld(),
                     o["qkv_out"].ptr() if c.save_qkv else None, o["qkv_out"].ld() if c.save_qkv else 0)
            torch.cuda.synchronize()
            return o
        qkv = _operand(d["qkv16"])
        if c.entry in ("fvit_attn_tc_fwd", "fvit_attn_core_fwd"):
            o["out"] = Window(rows, heads * w)
            extra = (None,) if c.entry == "fvit_attn_core_fwd" else ()
            lib.call(c.entry, qkv.data_ptr(), qkv.stride(0), c.groups, S, heads, w if c.entry != "fvit_attn_core_fwd"
                     else hd, bptr, scale, o["out"].ptr(), o["out"].ld(), *extra)
            torch.cuda.synchronize()
            return o
        if c.entry in ("fvit_attn_loop_fwd", "fvit_attn_loop_bwd_long"):
            o["out"] = Window(rows, heads * w)
            lse = c.lse or c.entry == "fvit_attn_loop_bwd_long"
            o["lse"] = torch.full((rows + TAIL, heads), float("nan"), device="cuda") if lse else None
            lib.call("fvit_attn_loop_fwd", qkv.data_ptr(), qkv.stride(0), c.groups, S, heads, w, bptr, scale,
                     o["out"].ptr(), o["out"].ld(), o["lse"].data_ptr() if lse else None)
            if c.entry == "fvit_attn_loop_fwd":
                torch.cuda.synchronize()
                return o
        do = _operand(d["do16"])
        o["dqkv"] = Window(rows, 3 * heads * w)
        o["dbias"] = None
        if c.bias == "bias":
            pre = dbias_prefill if dbias_prefill is not None else torch.zeros(heads, S, S, device="cuda")
            o["dbias"] = _with_tail(pre)
            o["dbias_prefill"] = pre
        dbptr = o["dbias"].data_ptr() if o["dbias"] is not None else None
        if c.entry == "fvit_attn_loop_bwd_long":
            scr = torch.full((rows, heads * w + 4), float("nan"), device="cuda")
            lib.call("fvit_attn_loop_bwd_long", qkv.data_ptr(), qkv.stride(0), do.data_ptr(), do.stride(0), o["out"].ptr(),
                     o["out"].ld(), o["lse"].data_ptr(), c.groups, S, heads, w, bptr, scale, o["dqkv"].ptr(),
                     o["dqkv"].ld(), dbptr, scr.data_ptr(), scr.stride(0))
        else:
            lib.call(c.entry, qkv.data_ptr(), qkv.stride(0), do.data_ptr(), do.stride(0), c.groups, S, heads, hd, w,
                     bptr, scale, o["dqkv"].ptr(), o["dqkv"].ld(), dbptr)
        torch.cuda.synchronize()
        return o
    finally:
        lib.load().fvit_set_sm_limit(0)


# ---------------------------------------------------------------------------------------------- reference + checks
def ref_of(c: Case, d: dict) -> dict:
    groups, S, heads, hd, w = c.groups, c.S, c.heads, c.hd, c.width
    scale = hd ** -0.5
    bias = d["ref_bias"] if c.bias != "no_bias" else None
    qk_err = None
    if c.entry == "fvit_hat_attn_fwd":
        x64, w64 = d["x"].double(), d["w16"].double()
        qkv64 = x64 @ w64.t() + d["qb"].double()
        r_qkv = (qkv64, x64.abs() @ w64.abs().t() + d["qb"].double().abs())
        q, k, v = G.heads_view(qkv64, groups, S, 3, heads, w, hd)
        # the kernel's q and k are fp16 roundings of the projection: each logit is off by up to 2 U16 scale |q||k|
        qk_err = 2.01 * scale * (q.abs() @ k.abs().transpose(-2, -1))
    else:
        q, k, v = G.heads_view(d["qkv16"], groups, S, 3, heads, w, hd)
        r_qkv = None
    bwd = c.entry in G.BWD
    do = G.heads_view(d["do16"], groups, S, 1, heads, w, hd)[0] if bwd else None
    r = G.reference(q, k, v, bias, scale, do, qk_err=qk_err)
    r["qkv"] = r_qkv
    return r


def _report(c, mode, name, val, sink):
    sink[name] = max(sink.get(name, 0.0), val)
    print(f"ratio {c.entry} {c.id} {mode} {name} {val:.3f}")


def _check16(c, mode, name, got, ref, mag, bar, sink):
    assert torch.isfinite(got).all(), f"{name}: non-finite values"
    _report(c, mode, name, G.needed_c(got, ref, mag), sink)
    G.assert_within(got, ref, G.bound16(ref, mag), f"{c.id} {mode} {name}")
    G.assert_whole(got, ref, bar, f"{c.id} {mode} {name}", mag)


def check(c: Case, d: dict, o: dict, r: dict, mode: str = "plain") -> dict:
    """every output of a run() against the reference; returns {output: needed C_ATTN}"""
    groups, S, heads, hd, w = c.groups, c.S, c.heads, c.hd, c.width
    sink = {}
    if "out" in o:
        win = o["out"]
        win.check_sentinels("out")
        got = G.heads_view(win.t, groups, S, 1, heads, w, hd)[0]
        _check16(c, mode, "out", got, r["out"], r["M_out"], G.FWD_BAR, sink)
        if w > hd:
            assert (win.t.view(-1, heads, w)[..., hd:] == 0).all(), "pad columns of out"
    if o.get("lse") is not None:
        lse = o["lse"]
        assert torch.isnan(lse[groups * S:]).all(), "lse rows past the end"
        got = lse[:groups * S].double().view(groups, S, heads).permute(0, 2, 1)
        want = r["lse"] + d["shift"].double()[None, None, :] * G.LOG2E
        err = (got - want).abs()
        over = (err - 8 * G.U32 * want.abs()).clamp_min(0) / G.U16
        _report(c, mode, "lse", float(over.max()), sink)
        G.assert_within(got, want, G.C_ATTN * G.U16 + 8 * G.U32 * want.abs(), f"{c.id} {mode} lse")
    if o.get("qkv_out") is not None:
        win = o["qkv_out"]
        win.check_sentinels("qkv_out")
        ref, mag = r["qkv"]
        G.assert_within(win.t, ref, G.U16 * ref.abs() + G.HALF_SUB + 4 * c.C * G.U32 * mag, f"{c.id} qkv_out")
        assert (win.t.view(-1, 3, heads, w)[..., hd:] == 0).all(), "pad columns of qkv_out"
    if "dqkv" in o:
        win = o["dqkv"]
        win.check_sentinels("dqkv")
        got = G.heads_view(win.t, groups, S, 3, heads, w, hd)
        for i, name in enumerate(("dq", "dk", "dv")):
            _check16(c, mode, name, got[i], r[name], r["M_" + name], G.BWD_BAR, sink)
        if w > hd:
            assert (win.t.view(-1, 3, heads, w)[..., hd:] == 0).all(), "pad columns of dqkv"
        if o["dbias"] is not None:
            n = heads * S * S
            big = o["dbias"]
            assert torch.isnan(big[n:]).all(), "dbias past heads * S * S"
            pre = o["dbias_prefill"].double()
            gotb = big[:n].double().view(heads, S, S)
            want = pre + r["dbias"]
            # fp32 atomic sums of `groups` windows onto the prefill
            acc = (groups + 2) * G.U32 * (r["M_dbias"] + pre.abs())
            over = ((gotb - want).abs() - acc).clamp_min(0) / (G.U16 * r["M_dbias"]).clamp_min(1e-300)
            _report(c, mode, "dbias", float(over.max()), sink)
            G.assert_within(gotb, want, G.C_ATTN * G.U16 * r["M_dbias"] + acc, f"{c.id} {mode} dbias")
            G.assert_whole(gotb - pre, r["dbias"], G.BWD_BAR, f"{c.id} {mode} dbias", r["M_dbias"])
    return sink


def run_and_check(c: Case, mode: str = "plain", seed: int = 0) -> dict:
    d = inputs(c, mode, seed)
    pre = None
    if c.bias == "bias" and c.entry in G.BWD:
        g = torch.Generator(device="cuda").manual_seed(seed + 7)
        pre = torch.randn(c.heads, c.S, c.S, device="cuda", generator=g) * 0.5
    o = run(c, d, dbias_prefill=pre)
    return check(c, d, o, ref_of(c, d), mode)


# ---------------------------------------------------------------------------------------------- a. every case
@pytest.mark.parametrize("case", G.CASES, ids=[c.id for c in G.CASES])
def test_case_matches_fp64(case):
    run_and_check(case)


# ---------------------------------------------------------------------------------------------- b. softmax edges
_F, _B, _LF, _LB, _H, _SF, _SB = G.ENTRIES
EDGE_CASES = [
    Case(_F, 53, 4, 32, 13), Case(_F, 53, 4, 49, 6), Case(_F, 49, 4, 80, 12), Case(_F, 100, 2, 80, 3),
    Case(_B, 53, 4, 32, 11), Case(_B, 8, 4, 49, 10), Case(_B, 53, 4, 80, 5),
    Case(_LF, 148, 8, 32, 6), Case(_LF, 196, 4, 49, 3), Case(_LF, 148, 4, 80, 4), Case(_LF, 100, 3, 64, 4),
    Case(_LB, 148, 8, 32, 5), Case(_LB, 196, 4, 49, 3), Case(_LB, 148, 4, 80, 4),
    Case(_H, 53, 4, 49, 9, C=192),
    Case(_SF, 53, 4, 24, 7), Case(_SF, 53, 2, 96, 5), Case(_SF, 229, 2, 16, 2),
    Case(_SB, 85, 4, 16, 3, hdp=32), Case(_SB, 85, 2, 96, 2),
]


@pytest.mark.parametrize("mode", MODES[1:])
@pytest.mark.parametrize("case", EDGE_CASES, ids=[c.id for c in EDGE_CASES])
def test_softmax_edges(case, mode):
    """A per-row shift by +-80 (lse moves by shift * log2 e, nothing else moves), one dominant key (+40) at key 0, the
    window's last key and a tile's last key, uniform rows (q = k = 0, bias constant along the row: out is the mean of
    v over the window), a bias of std 20 with q and k scaled up 3x, and every logit below -100."""
    if mode == "uniform":
        d = inputs(case, mode)
        r = ref_of(case, d)
        if case.entry != "fvit_hat_attn_fwd":
            v = G.heads_view(d["qkv16"], case.groups, case.S, 3, case.heads, case.width, case.hd)[2]
            torch.testing.assert_close(r["out"], v.mean(-2, keepdim=True).expand_as(r["out"]))
        o = run(case, d)
        check(case, d, o, r, mode)
    else:
        run_and_check(case, mode)


def test_edge_cases_cover_every_entry_and_width():
    got = {(c.entry, c.width if c.entry not in G.SIMT else "simt") for c in EDGE_CASES}
    want = {(e, w) for e in G.TC[:4] for w in (32, 64, 80)} | {(_H, 64), (_SF, "simt"), (_SB, "simt")}
    assert want <= got, want - got
    # the dominant key on the last key of a partial 128-key tile with S % 32 != 0 (padded keys in the same 32-column
    # chunk as real ones)
    assert any(c.entry == _LF and c.S > 128 and c.S % 128 and c.S % 32 for c in EDGE_CASES)


# ---------------------------------------------------------------------------------------------- c. memory contract
@pytest.mark.parametrize("case", [Case(_F, 53, 4, 32, 6, bias="no_bias"), Case(_LF, 148, 2, 64, 3, bias="no_bias"),
                                  Case(_B, 49, 2, 32, 5, bias="no_dbias"), Case(_B, 25, 2, 64, 5, bias="no_bias"),
                                  Case(_LB, 148, 2, 32, 3, bias="no_dbias"), Case(_LB, 148, 2, 64, 3, bias="no_bias"),
                                  Case(_SF, 53, 2, 96, 3, bias="no_bias"), Case(_SB, 85, 2, 16, 3, hdp=32, bias="no_bias"),
                                  Case(_SB, 53, 2, 96, 3, bias="no_dbias")], ids=lambda c: c.id)
def test_null_bias_and_dbias(case):
    run_and_check(case, seed=3)


def test_dbias_accumulates_into_its_prefill():
    """the three backward kernels add to dbias: two calls give twice the gradient on top of the prefill"""
    for c in (Case(_B, 49, 2, 32, 5), Case(_LB, 148, 2, 32, 3), Case(_SB, 53, 2, 24, 3, hdp=24)):
        d = inputs(c, seed=5)
        pre = torch.full((c.heads, c.S, c.S), 3.0, device="cuda")
        o1 = run(c, d, dbias_prefill=pre)
        o2 = run(c, d, dbias_prefill=o1["dbias"][:c.heads * c.S * c.S].view(c.heads, c.S, c.S).clone())
        r = ref_of(c, d)
        n = c.heads * c.S * c.S
        got = o2["dbias"][:n].double().view(c.heads, c.S, c.S)
        bound = 2 * G.C_ATTN * G.U16 * r["M_dbias"] + 4 * (c.groups + 2) * G.U32 * (r["M_dbias"] + 3.0)
        G.assert_within(got, 3.0 + 2 * r["dbias"], bound, f"{c.id} twice")
        assert torch.isnan(o2["dbias"][n:]).all()


# ---------------------------------------------------------------------------------------------- d. reduced grid
SM_CASES = [Case(_F, 49, 8, 32, 6), Case(_B, 49, 8, 32, 6), Case(_LF, 148, 6, 32, 4), Case(_LB, 148, 6, 32, 4),
            Case(_H, 53, 6, 49, 5, save_qkv=True)]


@pytest.mark.parametrize("case", SM_CASES, ids=lambda c: c.id)
def test_reduced_grid_gives_the_full_grid_result(case):
    """fvit_set_sm_limit(n) for n in {1, 3, heads - 1, 116}: out, lse, qkv_out, dq, dk and dv bitwise equal to the
    full-grid call (every item is computed whole by one CTA, in the same order); dbias within the fp32 atomic-sum bound
    (the CTAs' flush order changes). tc_bwd's head-major item walk is taken below one CTA per head."""
    d = inputs(case, seed=11)
    full = run(case, d, sm_limit=0)
    r = ref_of(case, d)
    check(case, d, full, r)
    for n in (1, 3, case.heads - 1, 116):
        if case.entry == _B:
            assert (G.geometry_class(case.entry, case.S, case.width, case.groups, case.heads, sms=n)[3] == "head-major") \
                == (n < case.heads)
        got = run(case, d, sm_limit=n)
        for key in ("out", "qkv_out", "dqkv"):
            if full.get(key) is not None and got.get(key) is not None:
                assert torch.equal(got[key].big.view(torch.int16), full[key].big.view(torch.int16)), (n, key)
        if full.get("lse") is not None:
            assert torch.equal(got["lse"].view(torch.int32), full["lse"].view(torch.int32)), (n, "lse")
        if full.get("dbias") is not None:
            nn_ = case.heads * case.S * case.S
            bound = 2 * (case.groups + 2) * G.U32 * r["M_dbias"].reshape(-1).float()
            assert ((got["dbias"][:nn_] - full["dbias"][:nn_]).abs() <= bound).all(), (n, "dbias")
            assert torch.isnan(got["dbias"][nn_:]).all()


# ---------------------------------------------------------------------------------------------- e. SIMT shapes
_BIG_S = G.largest_simt_bwd_S(16)
SIMT_SHAPES = [Case(_SF, 53, 2, 81, 4), Case(_SF, 85, 2, 96, 3), Case(_SF, 53, 2, 128, 3), Case(_SF, 85, 2, 128, 2),
               Case(_SB, 53, 2, 81, 3), Case(_SB, 53, 2, 96, 4), Case(_SB, 85, 2, 96, 3), Case(_SB, 53, 2, 128, 2),
               Case(_SB, 85, 2, 16, 4, hdp=32), Case(_SB, 125, 2, 24, 3, hdp=32), Case(_SB, 173, 2, 16, 2, hdp=16),
               Case(_SB, _BIG_S, 1, 16, 2, hdp=16)]


@pytest.mark.parametrize("case", SIMT_SHAPES, ids=lambda c: c.id)
def test_simt_at_its_own_shapes(case):
    run_and_check(case, seed=2)


def test_simt_backward_refuses_the_first_window_it_cannot_hold():
    lib = _lib()
    c = Case(_SB, _BIG_S + 1, 1, 16, 2, hdp=16)
    assert G.simt_bwd_smem(c.S, 16) > G.SMEM_MAX >= G.simt_bwd_smem(c.S - 1, 16)
    d = inputs(c)
    with pytest.raises(lib.FvitError, match="shared memory"):
        run(c, d)
    # nothing written: run() raised before returning its windows, so repeat the call by hand
    qkv, do = _operand(d["qkv16"]), _operand(d["do16"])
    out = Window(c.groups * c.S, 3 * c.heads * 16)
    dbias = _with_tail(torch.zeros(c.heads, c.S, c.S, device="cuda")).fill_(float("nan"))
    with pytest.raises(lib.FvitError, match=f"S={c.S}"):
        lib.call(_SB, qkv.data_ptr(), qkv.stride(0), do.data_ptr(), do.stride(0), c.groups, c.S, 1, 16, 16,
                 d["bias"].data_ptr(), 0.25, out.ptr(), out.ld(), dbias.data_ptr())
    torch.cuda.synchronize()
    assert torch.isnan(out.big.float()).all() and torch.isnan(dbias).all()


# ---------------------------------------------------------------------------------------------- model level
_CFG96 = dict(dim=24, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 1, 1, 2], window_size=[7, 7, 7, 7], ct_size=2,
              mlp_ratio=4, resolution=224, hat=[False, False, True, False], do_propagation=False)


def _setup96(seed):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from test_attn_geometry_cpu import HD96
    model = F.create_model("faster_vit_0_224", drop_path_rate=0.0, **HD96)
    O.synth_fill_(model.state_dict(), seed)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    x = O.synth_input(2, 224, seed + 100, torch.float32)
    return model.cuda(), sd64, x, torch.tensor([3, 7])


def _simt96(model):
    for plan in model._get_engine().plans.values():
        launches = list(G.attention_launches(plan))
        assert any(a.entry.startswith("fvit_attn_core_") and a.hd == 96 for a in launches), launches


def test_hd96_model_eval_logits_match_fp64():
    from test_hd80_model_gpu import _oracle
    model, sd64, x, target = _setup96(5)
    ref_logits = _oracle(sd64, _CFG96, x, target, training=False)[0]
    with torch.no_grad():
        out = model.eval()(x.cuda())
    torch.cuda.synchronize()
    assert ((out.double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 1e-3
    _simt96(model)


def test_hd96_model_train_step_matches_fp64():
    from test_hd80_model_gpu import _compare_grads, _oracle
    model, sd64, x, target = _setup96(6)
    ref_logits, ref_loss, ref_grads, _, _ = _oracle(sd64, _CFG96, x, target, training=True)
    model.train()
    logits = model(x.cuda())
    loss = torch.nn.functional.cross_entropy(logits, target.cuda())
    loss.backward()
    torch.cuda.synchronize()
    assert ((logits.detach().double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 3e-3
    assert abs(loss.item() - ref_loss) < 1e-4 * abs(ref_loss) + 1e-4
    med = _compare_grads(model, ref_grads)
    print(f"hd96 train: median rel-L2 {med:.2e}")
    _simt96(model)
