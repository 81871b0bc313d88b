"""Train-mode BatchNorm statistics against fp64 torch, sweeping a per-channel offset of r standard deviations.

Every producer sums in fp32 in one pass. Moments about K lose about 2^-24 * ((mean - K) / std)^2 of the variance per
summed term, so the statistics can be taken about a pivot K near the batch mean (include/fvit.h "Pivoted
statistics"):
- fvit_colstats_pivot_f32 (fp32 residual stream: the head `norm`, the backbone's `norm{i}`) pivots on each channel's
  first listed value, so it is exact whatever the running statistics; the training plans use it;
- the GEMM epilogue sums whatever col_shift centres: with col_shift = bias - K (fvit_bn_col_shift) and
  fvit_bn_finalize_pivot(shifted = 1) the statistics are exact for K within a few std of the batch mean. The training
  plans take K = the running mean when the plan is built: a pretrained or fine-tuned model gets the exact
  statistics, a fresh one (K = 0) the one-pass sum of before.

Bounds: rstd within 1e-4 relative; the batch mean within 1e-5 std beyond one fp32 ulp of the mean itself (an fp32
mean of 1000 std cannot be closer than ~6e-5 std).

Measured rstd relative error on an H100 80GB HBM3 (400 W), r = 0 / 1 / 10 / 100 / 1000:
- 9-tap conv GEMM (fv0 level 0, batch 16), about 0:     8.2e-7 / 1.3e-6 / 4.8e-5 / 6.1e-3 / 1.5
  about K within 3 std of the mean:                     3.3e-6 / 2.1e-6 / 2.8e-6 / 2.9e-6 / 2.6e-6
- linear GEMM, about 0:                                  5.0e-7 / 8.7e-7 / 6.2e-5 / 3.8e-3 / 0.84
  about K within 3 std:                                  2.5e-6 / 4.2e-6 / 2.8e-6 / 3.2e-6 / 3.3e-6
- head norm (3136 rows x 1568), fvit_colstats_f32:       5.2e-7 / 1.1e-6 / 7.3e-5 / 9.3e-3 / 6.3e2
  fvit_colstats_pivot_f32:                               2.8e-6 / 4.2e-6 / 5.7e-6 / 4.8e-6 / 4.0e-6
- dense level (50176 rows x 64), fvit_colstats_f32:      9.0e-7 / 3.6e-6 / 2.5e-4 / 2.3e-2 / 6.2e2
  fvit_colstats_pivot_f32:                               6.0e-6 / 8.7e-6 / 1.1e-5 / 5.1e-6 / 8.8e-6
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

R_SWEEP = [0, 1, 10, 100, 1000]
EPS, MOM = 1e-5, 0.1


def _lib():
    from fastervit_b200 import lib
    lib.load()
    return lib


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _finalize(L, s, pivot, shifted, n, w, b, rm, rv):
    """fvit_bn_finalize (pivot None: the one-pass statistics about 0) or fvit_bn_finalize_pivot"""
    C = w.numel()
    out = {k: torch.full((C,), float("nan"), device="cuda") for k in ("scale", "shift", "mean", "rstd")}
    tail = (w.data_ptr(), b.data_ptr(), EPS, MOM, rm.data_ptr(), rv.data_ptr(), None, out["scale"].data_ptr(),
            out["shift"].data_ptr(), out["mean"].data_ptr(), out["rstd"].data_ptr(), C)
    if pivot is None:
        L.call("fvit_bn_finalize", s[0].data_ptr(), s[1].data_ptr(), float(n), *tail)
    else:
        L.call("fvit_bn_finalize_pivot", s[0].data_ptr(), s[1].data_ptr(), pivot.data_ptr(), int(shifted), float(n), *tail)
    torch.cuda.synchronize()
    return out


def _errors(out, v, w, b, rm0, rv0, rm, rv, centre):
    """max errors of one finalize against fp64 statistics of v [n, C] (the exact values the kernel summed, before
    `centre` was subtracted); the normalised data is v - centre. Returns (rstd rel, mean / std, others...)"""
    n = v.shape[0]
    mean, var = v.mean(0), v.var(0, unbiased=False)
    std = var.sqrt()
    rstd = (var + EPS).rsqrt()
    md = mean - centre
    scale = w.double() * rstd
    shift = b.double() - md * scale
    ulp = 2.0 ** -23

    def excess(got, want, slack):   # error beyond `slack` (fp32 representation of the value), in std
        return ((got.double() - want).abs() - slack).clamp_min(0).div(std).max().item()

    rm_want = (1 - MOM) * rm0.double() + MOM * mean
    e = dict(
        rstd=((out["rstd"].double() - rstd).abs() / rstd).max().item(),
        mean=excess(out["mean"], md, ulp * md.abs()),
        scale=((out["scale"].double() - scale).abs() / scale.abs()).max().item(),
        # relative to the range of the normalised output, b + (|mean| + std) * scale
        shift=((out["shift"].double() - shift).abs() / (b.double().abs() + (md.abs() + std) * scale.abs())).max().item(),
        rmean=excess(rm, rm_want, ulp * (rm0.double().abs() + rm_want.abs())),
        rvar=((rv.double() - ((1 - MOM) * rv0.double() + MOM * var * n / (n - 1))).abs()
              / ((1 - MOM) * rv0.double() + MOM * var)).max().item())
    return e


def _assert_bounds(e, what):
    assert e["rstd"] <= 1e-4, (what, e)
    assert e["mean"] <= 1e-5, (what, e)          # beyond one fp32 ulp of the mean
    assert e["scale"] <= 1e-4, (what, e)
    assert e["shift"] <= 1e-4, (what, e)
    assert e["rmean"] <= 1e-5, (what, e)
    assert e["rvar"] <= 1e-4, (what, e)


def _bn_params(C, g):
    w = (torch.rand(C, device="cuda", generator=g) + 0.5)
    b = torch.randn(C, device="cuda", generator=g) * 0.1
    rv0 = torch.rand(C, device="cuda", generator=g) + 0.5
    return w, b, rv0


def _conv_problem(g):
    """fv0 level 0 at batch 16: 64 -> 64 channels, 56 x 56, zero-bordered NHWC rows (every CTA takes >= 3 units)"""
    B, C, H, W = 16, 64, 56, 56
    Hp, Wp = H + 2, W + 2
    rows = B * Hp * Wp
    assert rows // 128 >= 3 * _sms()
    xp = torch.zeros(B, Hp, Wp, C, device="cuda", dtype=torch.half)
    xp[:, 1:-1, 1:-1] = torch.randn(B, H, W, C, device="cuda", generator=g).half()
    a = xp.view(rows, C)
    wt = (torch.randn(C, 9, C, device="cuda", generator=g) / 24).half()
    taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    inside = torch.zeros(B, Hp, Wp, dtype=torch.bool, device="cuda")
    inside[:, 1:-1, 1:-1] = True
    row_map = torch.where(inside.view(-1), torch.arange(rows, device="cuda"), -1).int()
    acc = torch.zeros(rows, C, dtype=torch.float64, device="cuda")
    ad, wd = a.double(), wt.double()
    for t, (sh, _) in enumerate(taps):
        lo, hi = max(0, -sh), rows - max(0, sh)
        acc[lo:hi] += ad[lo + sh:hi + sh] @ wd[:, t].T
    return dict(a=a, b=wt.view(C, 9 * C), kc=C, taps=taps, row_map=row_map, acc=acc[inside.view(-1)])


def _linear_problem(g):
    """plain linear layer, m >= 3 units per CTA, a row map with holes"""
    n, k = 96, 256
    m = 128 * 3 * _sms() + 77
    a = torch.randn(m, k, device="cuda", generator=g).half()
    b = (torch.randn(n, k, device="cuda", generator=g) / 16).half()
    row_map = torch.arange(m, device="cuda").int()
    row_map[5::9] = -1
    return dict(a=a, b=b, kc=k, taps=None, row_map=row_map, acc=(a.double() @ b.double().T)[row_map >= 0])


def _gemm_stats(L, P, col_shift):
    C = P["b"].shape[0]
    m = P["a"].shape[0]
    s = torch.zeros(2, C, device="cuda")
    raw = torch.full((m, C), float("nan"), device="cuda").half()
    L.gemm(P["a"], P["b"], kc=P["kc"], taps=P["taps"], col_shift=col_shift, row_map=P["row_map"], out_f16=raw,
           col_sum=s[0], col_sumsq=s[1])
    return s, raw[P["row_map"] >= 0]


@pytest.mark.parametrize("shape", ["conv9", "linear"])
@pytest.mark.parametrize("r", R_SWEEP)
def test_gemm_epilogue_stats_about_running_mean(shape, r):
    """GEMM col_sum / col_sumsq -> finalize, for channel offsets of r std: (1) about 0, the one-pass path
    (fvit_bn_finalize, which fresh running statistics reproduce: K = 0); (2) about a running mean within 3 std of the
    batch mean (a few steps in, or a pretrained checkpoint): col_shift = bias - K, fvit_bn_finalize_pivot."""
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(1000 + r)
    P = _conv_problem(g) if shape == "conv9" else _linear_problem(g)
    C = P["b"].shape[0]
    std = P["acc"].std(0)
    sign = torch.where(torch.rand(C, device="cuda", generator=g) < 0.5, -1.0, 1.0).double()
    bias = (r * std * sign).float()
    v = P["acc"] + bias.double()
    w, b, rv0 = _bn_params(C, g)
    res = {}
    # (1) about 0: the one-pass statistics of the previous version
    rm0 = torch.zeros(C, device="cuda")
    rm, rv = rm0.clone(), rv0.clone()
    s, _ = _gemm_stats(L, P, bias)
    res["legacy"] = _errors(_finalize(L, s, None, 0, v.shape[0], w, b, rm, rv), v, w, b, rm0, rv0, rm, rv, 0.0)
    rm, rv = rm0.clone(), rv0.clone()
    pv = rm0.clone()
    cs = torch.full((C,), float("nan"), device="cuda")
    L.call("fvit_bn_col_shift", bias.data_ptr(), pv.data_ptr(), C, cs.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(cs, bias - pv)
    s, _ = _gemm_stats(L, P, cs)
    res["K=0"] = _errors(_finalize(L, s, pv, 1, v.shape[0], w, b, rm, rv), v, w, b, rm0, rv0, rm, rv, 0.0)
    # (2) running mean within 3 std of the batch mean
    rm0 = (v.mean(0) + (torch.rand(C, device="cuda", generator=g).double() * 6 - 3) * std).float()
    rm, rv = rm0.clone(), rv0.clone()
    pv = rm0.clone()
    L.call("fvit_bn_col_shift", bias.data_ptr(), pv.data_ptr(), C, cs.data_ptr())
    s, raw = _gemm_stats(L, P, cs)
    res["K~mean"] = _errors(_finalize(L, s, pv, 1, v.shape[0], w, b, rm, rv), v, w, b, rm0, rv0, rm, rv,
                            rm0.double())
    # the raw output the BatchNorm later normalises is centred on the pivot as well
    cen = v - rm0.double()
    assert (raw.double() - cen).abs().max().item() <= 1e-3 * cen.abs().max().item()
    print(f"\n[bn-stats] gemm {shape} r={r}: " + "; ".join(
        f"{k}: rstd {e['rstd']:.2e} mean/std {e['mean']:.2e} rvar {e['rvar']:.2e}" for k, e in res.items()))
    _assert_bounds(res["K~mean"], ("K~mean", shape, r))
    # K = 0 is the one-pass arithmetic: no worse than it (atomics reorder the sums between runs; at r = 1000 both are
    # rounding noise of order 1)
    if r <= 100:
        assert res["K=0"]["rstd"] <= max(4 * res["legacy"]["rstd"], 1e-5), res
    if r <= 1:
        _assert_bounds(res["legacy"], ("legacy", shape, r))


@pytest.mark.parametrize("shape", ["head", "level"])
@pytest.mark.parametrize("r", R_SWEEP)
def test_colstats_f32_first_row_pivot(shape, r):
    """fp32 residual-stream statistics over a row list: the head-norm shape (B*49 rows x 1568, fv4 at batch 64) and a
    dense-level shape (fv0 level 0 at batch 16, 50176 rows x 64, rows of stride 72 > C); channel offsets r std."""
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(2000 + r)
    if shape == "head":
        nrows, C, ld, total = 64 * 49, 1568, 1568, 64 * 64
    else:
        nrows, C, ld, total = 16 * 56 * 56, 64, 72, 16 * 58 * 58
    rows = torch.randperm(total, device="cuda", generator=g)[:nrows].int()
    std = torch.rand(C, device="cuda", generator=g).double() * 1.5 + 0.5
    sign = torch.where(torch.rand(C, device="cuda", generator=g) < 0.5, -1.0, 1.0).double()
    x = torch.full((total, ld), float("nan"), device="cuda")
    x[:, :C] = (torch.randn(total, C, device="cuda", generator=g, dtype=torch.float64) * std + r * std * sign).float()
    v = x[rows.long(), :C].double()
    w, b, rv0 = _bn_params(C, g)
    rm0 = torch.randn(C, device="cuda", generator=g) * 0.2
    res = {}
    s = torch.zeros(2, C, device="cuda")
    L.call("fvit_colstats_f32", x.data_ptr(), ld, rows.data_ptr(), nrows, C, s[0].data_ptr(), s[1].data_ptr())
    rm, rv = rm0.clone(), rv0.clone()
    res["legacy"] = _errors(_finalize(L, s, None, 0, nrows, w, b, rm, rv), v, w, b, rm0, rv0, rm, rv, 0.0)
    s.zero_()
    pv = torch.full((C,), float("nan"), device="cuda")
    L.call("fvit_colstats_pivot_f32", x.data_ptr(), ld, rows.data_ptr(), nrows, C, pv.data_ptr(), s[0].data_ptr(),
           s[1].data_ptr())
    rm, rv = rm0.clone(), rv0.clone()
    out = _finalize(L, s, pv, 0, nrows, w, b, rm, rv)
    assert torch.equal(pv, x[rows[0].long(), :C])
    res["pivot"] = _errors(out, v, w, b, rm0, rv0, rm, rv, 0.0)
    print(f"\n[bn-stats] colstats {shape} r={r}: " + "; ".join(
        f"{k}: rstd {e['rstd']:.2e} mean/std {e['mean']:.2e} rvar {e['rvar']:.2e}" for k, e in res.items()))
    _assert_bounds(res["pivot"], ("pivot", shape, r))
    if r <= 1:
        _assert_bounds(res["legacy"], ("legacy", shape, r))


# ------------------------------------------------------------------------------------------------------- end to end
def _bn_prefixes(sd):
    return sorted(k[:-len(".running_mean")] for k in sd if k.endswith(".running_mean"))


@pytest.mark.parametrize("case", ["tiny_a", "tiny_ar"])
def test_train_step_on_pixel_range_input(case):
    """One train step on an un-normalised image batch (pixel range, 120 +- 60): the stem BatchNorms see offsets of
    several std. Logits, loss and gradients against the fp64 oracle; every running statistic after one update
    (the plan is fresh, so no earlier step moved them)."""
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES, cfg_of
    entry, kw, _ = CASES[case]
    cfg = cfg_of(case)
    model = F.create_model(entry, drop_path_rate=0.0, **kw)
    O.synth_fill_(model.state_dict(), 4321)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    model = model.cuda().train()
    x = O.synth_input(2, cfg["resolution"], 77, torch.float32) * 60 + 120
    target = torch.tensor([1, 3])
    logits = model(x.cuda())
    loss = torch.nn.functional.cross_entropy(logits, target.cuda())
    loss.backward()
    torch.cuda.synchronize()
    ref_loss, ref_logits, ref_grads = O.loss_and_grads(sd64, cfg, x.double(), target, training=True)
    stats = {}
    with torch.no_grad():
        O.forward(sd64, cfg, x.double(), training=True, bn_stats=stats)
    assert ((logits.double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 3e-3
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item()) + 1e-4
    sd = model.state_dict()
    prefixes = _bn_prefixes(sd)
    assert set(stats) == set(prefixes)
    for p in prefixes:
        mean, var = stats[p]
        for leaf, batch in (("running_mean", mean), ("running_var", var)):
            want = (1 - MOM) * sd64[f"{p}.{leaf}"] + MOM * batch
            d = (sd[f"{p}.{leaf}"].double().cpu() - want).abs().max().item()
            assert d <= 1e-3 * max(want.abs().max().item(), 1e-6) + 1e-6, (p, leaf, d)
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    l2s = []
    for k, p in model.named_parameters():
        want = ref_grads[k]
        err = (p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5)
        l2s.append(err)
        assert err < (6e-2 if k.startswith("patch_embed.") else 4e-2), (k, err)
    assert sorted(l2s)[len(l2s) // 2] <= 4e-3, sorted(l2s)[len(l2s) // 2]


def test_forward_features_with_large_residual_offset():
    """forward_features on tiny_a whose last-level residual stream carries per-channel offsets >= 100 std (the last
    block's fc2 bias, after its layer scale): the head `norm` statistics come from fvit_colstats_pivot_f32."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent))
    import _dense_oracle as DO
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES, cfg_of
    entry, kw, _ = CASES["tiny_a"]
    cfg = cfg_of("tiny_a")
    model = F.create_model(entry, drop_path_rate=0.0, **kw)
    sdm = model.state_dict()
    O.synth_fill_(sdm, 1234)
    last = len(model.levels) - 1
    blk = f"levels.{last}.blocks.{len(model.levels[last].blocks) - 1}"
    C = sdm[f"{blk}.mlp.fc2.bias"].numel()
    g = torch.Generator().manual_seed(5)
    sign = torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    # the stream's per-channel std is a few units here: an fc2 bias of 1000 (over the layer scale gamma2, where the
    # block has one) puts every channel >= 100 std away from 0
    gamma = sdm.get(f"{blk}.gamma2", torch.ones(C))
    sdm[f"{blk}.mlp.fc2.bias"].copy_(1000.0 * sign / gamma)
    sd = {k: v.detach().clone() for k, v in sdm.items()}
    model = model.cuda().train()
    x = O.synth_input(2, cfg["resolution"], 56, torch.float32)
    rm0, rv0 = model.norm.running_mean.clone(), model.norm.running_var.clone()
    f = model.forward_features(x.cuda())
    wgt = torch.randn(tuple(f.shape), generator=g, dtype=torch.float64)
    (f * wgt.float().cuda()).sum().backward()
    ref_out, ref_g, stats = DO.levels_loss_and_grads(sd, cfg, x, {"norm": wgt}, final="norm")
    mean, var = stats["norm"]
    assert (mean.abs() / var.sqrt()).min().item() >= 100       # the offset the test is about
    assert ((f.double().cpu() - ref_out["norm"]).abs().max() / ref_out["norm"].abs().max()).item() < 3e-3
    m = model.norm.momentum
    for got, want in ((model.norm.running_mean, (1 - m) * rm0.double().cpu() + m * mean),
                      (model.norm.running_var, (1 - m) * rv0.double().cpu() + m * var)):
        assert (got.double().cpu() - want).abs().max().item() <= 1e-3 * want.abs().max().item()
    for k in ("norm.weight", "norm.bias"):
        want = ref_g[k]
        got = dict(model.named_parameters())[k].grad.double().cpu()
        assert (got - want).norm().item() <= 4e-2 * want.norm().item(), k
