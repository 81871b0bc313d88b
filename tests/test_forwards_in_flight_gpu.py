"""GPU tests of several train-mode forwards awaiting one backward (FasterViT.set_train_forwards_in_flight): a loss over
two views against two separate steps and against fp64 autograd of the oracle, the pool's choice of instance, dense
outputs with the image gradient, a MOTRv2 clip in flight against the same clip through reentrant checkpointing, the
detection backbone under its plan-cache bound, and the fused optimizer fed from summed gradients.

Noise bar between a summed and a separate-steps backward: train-mode batch statistics and split-K weight gradients are
sums of float atomics, so two runs of the same step differ in the last bits and fp16 roundings downstream follow (the
parent build differs from itself by 2.4e-5 ... 3.1e-5 in fv4's sampled gradients; the stem, at the end of the backward
chain, by up to a few percent of its own largest gradient). Each test therefore runs its reference arm twice and
measures that noise: per tensor, max |difference| over the larger of its own max |g| and 1e-2 of the model's largest
gradient. The arm under test must stay within 4x the noise's worst tensor and 4x its median."""
import copy

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


def _tiny(case="tiny_a", **kw):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES, cfg_of
    entry, ckw, _ = CASES[case]
    model = F.create_model(entry, drop_path_rate=0.0, **ckw, **kw)
    O.synth_fill_(model.state_dict(), 1234)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    return model, sd64, cfg_of(case)


def _grads(model) -> dict:
    return {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def _assert_noise(got: dict, want: dict, again: dict) -> tuple:
    """`got` agrees with `want` within the run-to-run noise of `want`'s computation (`again` is a second run of it)"""
    assert got.keys() == want.keys() == again.keys() and got
    gmax = max(v.abs().max().item() for v in want.values())

    def errs(x):
        return {k: (x[k] - w).abs().max().item() / max(w.abs().max().item(), 1e-2 * gmax) for k, w in want.items()}
    e, n = errs(got), errs(again)
    worst_e, worst_n = max(e.values()), max(n.values())
    med_e, med_n = (sorted(v.values())[len(v) // 2] for v in (e, n))
    assert worst_e <= 4 * worst_n + 1e-4, (worst_e, worst_n, sorted(e.items(), key=lambda kv: -kv[1])[:5])
    assert med_e <= 4 * med_n + 1e-5, (med_e, med_n)
    return worst_e, worst_n, med_e, med_n


def _assert_stats_equal(a, b) -> None:
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        if k.endswith("num_batches_tracked"):
            assert torch.equal(sa[k], sb[k]), k
        elif k.endswith(("running_mean", "running_var")):
            # (batch statistics are atomics sums too: measured 3.7e-5 of max |running mean| between two runs)
            assert (sa[k] - sb[k]).abs().max().item() <= 2e-4 * max(sb[k].abs().max().item(), 1e-3), k


def _views(B, res, seeds):
    from oracle import fastervit_oracle as O
    return [O.synth_input(B, res, s, torch.float32).cuda() for s in seeds]


# --------------------------------------------------------------------------------------------- 1: views = steps
@pytest.mark.parametrize("graphs", ["1", "0"])
def test_sum_of_views_equals_sum_of_steps(graphs, monkeypatch):
    monkeypatch.setenv("FVIT_CUDA_GRAPH", graphs)
    from oracle import fastervit_oracle as O
    m0, sd64, cfg = _tiny()
    ma = copy.deepcopy(m0).cuda().train().set_train_forwards_in_flight(2)
    mb = copy.deepcopy(m0).cuda().train()
    mc = copy.deepcopy(m0).cuda().train()   # separate steps, once per step: the running statistics of arm (b)
    xs = _views(2, 224, (11, 12))
    tg = [torch.tensor([3, 700]).cuda(), torch.tensor([998, 5]).cuda()]
    ce = nn.functional.cross_entropy
    for step in range(3):
        for x, t in zip(xs, tg):
            ce(mc(x), t).backward()
    for step in range(3):   # (a plan's launch lists become CUDA graphs from its second run on)
        for m in (ma, mb):
            m.zero_grad(set_to_none=True)
        (ce(ma(xs[0]), tg[0]) + ce(ma(xs[1]), tg[1])).backward()
        gb = []
        for _ in range(2):
            mb.zero_grad(set_to_none=True)
            for x, t in zip(xs, tg):
                ce(mb(x), t).backward()
            gb.append(_grads(mb))
        torch.cuda.synchronize()
        r = _assert_noise(_grads(ma), *gb)
        print(f"graphs={graphs} step {step}: worst / median difference {r[0]:.2e} / {r[2]:.2e}, noise {r[1]:.2e} / {r[3]:.2e}")
    _assert_stats_equal(ma, mc)
    eng = ma._get_engine()
    assert [len(p) for p in eng.pools.values()] == [2]
    assert all(not p.in_flight() for p in next(iter(eng.pools.values())))
    assert [len(p) for p in mb._get_engine().pools.values()] == [1]
    if graphs == "0":
        assert all(not p.use_graphs and not p._graphs for p in next(iter(eng.pools.values())))
    # against fp64 autograd of the oracle: the sum of the two forwards' gradients, at test_train_gpu.py's bars
    ref = {}
    for x, t in zip(xs, tg):
        _, _, g = O.loss_and_grads(sd64, cfg, x.double().cpu(), t.cpu(), training=True)
        for k, v in g.items():
            ref[k] = ref.get(k, 0) + v
    gmax = max(v.abs().max().item() for v in ref.values())
    bad, l2s = [], []
    for k, p in ma.named_parameters():
        want = ref[k]
        err = (p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5)
        l2s.append(err)
        if err > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, err))
    assert not bad, bad[:10]
    assert sorted(l2s)[len(l2s) // 2] <= 4e-3


# --------------------------------------------------------------------------------------------- 2: pool semantics
def test_pool_semantics():
    from fastervit_b200.lib import FvitError
    m0, _, _ = _tiny()
    m = m0.cuda().train().set_train_forwards_in_flight(2)
    eng = m._get_engine()
    xs = _views(2, 224, (1, 2, 3))
    o = [m(x).sum() for x in xs]           # the third forward overwrites the first's instance
    with pytest.raises(FvitError, match="stale forward.*set_train_forwards_in_flight"):
        o[0].backward()
    o[1].backward()
    o[2].backward()
    (pool,) = eng.pools.values()
    assert len(pool) == 2 and not any(p.in_flight() for p in pool)
    del o
    # outputs dropped without a backward free their instance: three forwards, the first dropped, build no third
    m2 = copy.deepcopy(m0).cuda().train().set_train_forwards_in_flight(3)
    eng2 = m2._get_engine()
    m2(xs[0])
    keep = [m2(xs[1]), m2(xs[2])]
    (pool2,) = eng2.pools.values()
    assert len(pool2) == 2
    sum(k.sum() for k in keep).backward()
    # steady state: no instance is built after the first step of a loop
    first = None
    for _ in range(4):
        m2.zero_grad(set_to_none=True)
        (m2(xs[0]).sum() + m2(xs[1]).sum()).backward()
        ids = [id(p) for p in pool2]
        first = first or ids
        assert ids == first and eng2.pools[next(iter(eng2.pools))] is pool2
    # n = 1 raises as before
    m.set_train_forwards_in_flight(1)
    assert len(pool) == 1
    l1 = m(xs[0]).sum()
    l2 = m(xs[1]).sum()
    with pytest.raises(FvitError, match="stale forward"):
        l1.backward()
    l2.backward()


# --------------------------------------------------------------------------------------------- 3: dense outputs
def _dense_weights(outs, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(o.shape, device="cuda", generator=g) for o in outs]


@pytest.mark.parametrize("kind", ["forward_levels", "backbone_frozen1"])
def test_dense_views_with_image_gradient(kind):
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES
    if kind == "forward_levels":
        m0, _, _ = _tiny()
        run = lambda m, x: m.forward_levels(x, (1, 2, 3))   # noqa: E731
    else:
        entry, ckw, _ = CASES["tiny_a"]
        m0 = FasterViTBackbone(entry, out_indices=(1, 2, 3), frozen_stages=1, drop_path_rate=0.0, **ckw)
        O.synth_fill_(m0.state_dict(), 99)
        run = lambda m, x: m.forward_raw(x)   # noqa: E731
    ma = copy.deepcopy(m0).cuda().train().enable_input_grad().set_train_forwards_in_flight(2)
    mb = copy.deepcopy(m0).cuda().train().enable_input_grad()
    xs = _views(2, 224, (21, 22))
    for step in range(3):
        for m in (ma, mb):
            m.zero_grad(set_to_none=True)
        xa = [x.clone().requires_grad_(True) for x in xs]
        outs = [run(ma, x) for x in xa]
        ws = [_dense_weights(o, 5 + i) for i, o in enumerate(outs)]
        sum((o * w).sum() for oo, ww in zip(outs, ws) for o, w in zip(oo, ww)).backward()
        gb, dxb = [], []
        for _ in range(2):
            mb.zero_grad(set_to_none=True)
            xb = [x.clone().requires_grad_(True) for x in xs]
            for x, w in zip(xb, ws):
                sum((o * wk).sum() for o, wk in zip(run(mb, x), w)).backward()
            gb.append(_grads(mb))
            dxb.append({str(i): x.grad for i, x in enumerate(xb)})
        torch.cuda.synchronize()
        r = _assert_noise(_grads(ma), *gb)
        rx = _assert_noise({str(i): x.grad for i, x in enumerate(xa)}, *dxb)
        print(f"{kind} step {step}: parameters {r}, images {rx}")
    if kind == "backbone_frozen1":
        assert all(p.grad is None for p in ma.body.patch_embed.parameters())


# --------------------------------------------------------------------------------------------- 4: MOTRv2 clip
def _layernorm2d():
    class LayerNorm2d(nn.LayerNorm):   # timm's LayerNorm2d: the module classifies it by what it is
        def __init__(self, n, eps=1e-6):
            super().__init__(n, eps=eps)
    return LayerNorm2d


def test_motrv2_clip_in_flight_equals_checkpointed_clip():
    from torch.utils.checkpoint import checkpoint
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    from oracle import fastervit_oracle as O
    torch.manual_seed(0)
    m0 = build_fastervit("faster_vit_0_224", FrozenBatchNorm2d, _layernorm2d(), dim=32, in_dim=16, depths=[1, 1, 2, 1],
                         num_heads=[1, 2, 4, 8], drop_path_rate=0.3)
    O.synth_fill_(m0.state_dict(), 4321)
    ma = copy.deepcopy(m0).cuda().train().set_train_forwards_in_flight(5)
    mb = copy.deepcopy(m0).cuda().train()
    frames = _views(1, [96, 160], range(30, 35))
    dummy = torch.zeros(1, device="cuda", requires_grad=True)   # (makes the checkpointed outputs require grad)

    def clip_a(ws):
        maps = [ma.forward_raw(f) for f in frames]
        sum((o * w).sum() for oo, ww in zip(maps, ws) for o, w in zip(oo, ww)).backward()

    def clip_b(ws):
        maps = [checkpoint(lambda f, _d: mb.forward_raw(f), f, dummy, use_reentrant=True) for f in frames[:4]]
        maps.append(mb.forward_raw(frames[4]))
        sum((o * w).sum() for oo, ww in zip(maps, ws) for o, w in zip(oo, ww)).backward()

    with torch.no_grad():
        shapes = [o.shape for o in ma.forward_raw(frames[0])]
    ws = [[torch.randn(s, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7 * i + j))
           for j, s in enumerate(shapes)] for i in range(5)]
    nbt = [{k: v.clone() for k, v in m.state_dict().items() if k.endswith("num_batches_tracked")} for m in (ma, mb)]
    assert nbt[0]
    for step in range(3):   # steps 1 and 2 replay captured graphs inside the recompute
        for m in (ma, mb):
            m.zero_grad(set_to_none=True)
        ga = []
        for _ in range(2):
            ma.zero_grad(set_to_none=True)
            torch.manual_seed(100 + step)
            clip_a(ws)
            ga.append(_grads(ma))
        torch.manual_seed(100 + step)
        clip_b(ws)
        torch.cuda.synchronize()
        r = _assert_noise(_grads(mb), *ga)
        print(f"clip step {step}: worst / median difference {r[0]:.2e} / {r[2]:.2e}, noise {r[1]:.2e} / {r[3]:.2e}")
    # the masks really are drawn: a different seed moves the gradients well past the noise
    ga = _grads(ma)
    ma.zero_grad(set_to_none=True)
    torch.manual_seed(999)
    clip_a(ws)
    gmax = max(g.abs().max().item() for g in ga.values())
    assert max((ma.get_parameter(k).grad - g).abs().max().item() for k, g in ga.items()) > 0.05 * gmax
    # running statistics: five updates per clip in flight, nine with the recompute (as the reference's checkpoint path)
    sa, sb = ma.state_dict(), mb.state_dict()
    for k in nbt[0]:
        assert int(sa[k] - nbt[0][k]) == 5 * 7 and int(sb[k] - nbt[1][k]) == 9 * 3, k
    (pool,) = ma._get_engine().pools.values()
    assert len(pool) == 5 and [len(p) for p in mb._get_engine().pools.values()] == [1]
    for k in sa:   # frozen stem buffers never move
        if k.startswith("patch_embed."):
            assert torch.equal(sa[k], sb[k]), k


# --------------------------------------------------------------------------------------------- 5: detection bound
def test_detection_views_survive_the_plan_cache_bound():
    from fastervit_b200.detection import build_fastervit
    from oracle import fastervit_oracle as O
    m0 = build_fastervit("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8],
                         drop_path_rate=0.0, out_indices=(1, 2, 3))
    O.synth_fill_(m0.state_dict(), 5)
    ma = copy.deepcopy(m0).cuda().train().set_train_forwards_in_flight(2)
    mb = copy.deepcopy(m0).cuda().train()
    assert ma.plan_cache_size == 2
    a1, a2 = _views(1, [96, 160], (1, 2))
    b, c, d = (_views(1, hw, (s,))[0] for hw, s in (([224, 224], 3), ([250, 333], 4), ([320, 480], 5)))
    order = (a1, b, a2, c, d)   # d trims the first shape's key while both of its views are in flight
    for step in range(2):
        for m in (ma, mb):
            m.zero_grad(set_to_none=True)
        outs = [ma.forward_raw(x) for x in order]
        eng = ma._get_engine()
        assert len(eng.plans) == 2 and all(k[0] != tuple(a1.shape) for k in eng.plans)
        ws = [_dense_weights(o, 40 + i) for i, o in enumerate(outs)]
        sum((o * w).sum() for oo, ww in zip(outs, ws) for o, w in zip(oo, ww)).backward()
        gb = []
        for _ in range(2):
            mb.zero_grad(set_to_none=True)
            for x, w in zip(order, ws):
                sum((o * wk).sum() for o, wk in zip(mb.forward_raw(x), w)).backward()
            gb.append(_grads(mb))
        torch.cuda.synchronize()
        r = _assert_noise(_grads(ma), *gb)
        print(f"detection step {step}: {r}")


# --------------------------------------------------------------------------------------------- 6: optimizer
def test_fused_adamw_after_a_two_view_backward():
    from fastervit_b200.optim import FusedAdamW
    m0, _, _ = _tiny()
    ma = copy.deepcopy(m0).cuda().train().set_train_forwards_in_flight(2)
    mb = copy.deepcopy(m0).cuda().train()
    xs = _views(2, 224, (7, 8))
    ce = nn.functional.cross_entropy
    t = torch.tensor([1, 2]).cuda()
    (ce(ma(xs[0]), t) + ce(ma(xs[1]), t)).backward()
    for pa, pb in zip(ma.parameters(), mb.parameters()):
        pb.grad = pa.grad.clone()
    oa, ob = FusedAdamW(ma, lr=1e-2, weight_decay=0.05), FusedAdamW(mb, lr=1e-2, weight_decay=0.05)
    oa.step()
    ob.step()
    torch.cuda.synchronize()
    for (k, pa), pb in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(pa, pb), k
    assert any(not torch.equal(pa, p0.cuda()) for pa, p0 in zip(ma.parameters(), m0.parameters()))
