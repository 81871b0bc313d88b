"""Host-side checks of the attention geometry table (tests/_attn_geometry.py): every attention launch of the plans the
package builds falls in a geometry class that a case of tests/test_attn_geometry_gpu.py runs, the class function agrees
with the table, and the per-element comparator passes one fp16 ulp of error but fails a scaled or swapped head. Also
the plan-build refusal of windows the SIMT attention backward cannot hold in shared memory. Plans are built on the CPU
with the depths reduced and every model's dims and heads kept; nothing is launched."""
import pytest
import torch

import fastervit_b200 as F
from fastervit_b200 import lib as L

import _attn_geometry as G

_DEPTHS = [1, 1, 1, 1]
# a model with 96-wide heads at levels 2 and 3 (fvit_attn_core_fwd / _bwd in every mode), and the 13 x 13 any-res
# windows (S = 169 + 4 = 173: SIMT forward, S % 4 != 0)
HD96 = dict(dim=24, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 1, 1, 2])
AR173 = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8], resolution=[416, 416],
             window_size=[7, 7, 13, 13])


def _modes(desc, model, H, W):
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    yield f"{desc} eval", Plan(model.eval(), 2, H, W, False, cpu)
    yield f"{desc} train", TrainPlan(model.train(), 2, H, W, cpu)
    yield f"{desc} eval-gradient", TrainPlan(model.eval(), 2, H, W, cpu, spec=dict(kind=None, eval=True))


def _res(m):
    r = m.cfg["resolution"]
    return (r, r) if isinstance(r, int) else tuple(r)


def plans():
    """(description, plan) of every plan kind the package builds, at the geometries its users run: every registered
    entrypoint at its default resolution (the 21k models at 224, 384, 512 and 768) in eval, train and eval-gradient
    mode, the any-res model at 576 x 960, the detection backbone at DETR sizes, the tracking backbone at 800 x 1536, and
    the reduced models whose windows the kernels special-case"""
    from fastervit_b200.engine import Plan
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    for name in F.list_models():
        m = F.create_model(name, drop_path_rate=0.1, depths=_DEPTHS)
        yield from _modes(f"{name} {_res(m)}", m, *_res(m))
    m = F.create_model("faster_vit_0_any_res", drop_path_rate=0.1, depths=_DEPTHS, resolution=[576, 960],
                       window_size=[7, 7, 12, 6])
    yield from _modes("faster_vit_0_any_res 576x960 w[7, 7, 12, 6]", m, 576, 960)
    from fastervit_b200.detection import build_fastervit as det_build
    det = det_build("faster_vit_0_224", out_indices=(0, 1, 2, 3), drop_path_rate=0.1, depths=_DEPTHS)
    spec = dict(kind="levels", outs=tuple((i, getattr(det, f"norm{i}")) for i in range(4)), frozen=-1)
    for H, W in ((480, 640), (512, 1333), (608, 1088), (704, 1173), (800, 1067), (800, 1333)):
        yield f"detection {H}x{W} eval", Plan(det.eval(), 2, H, W, False, cpu)
        yield f"detection {H}x{W} levels train", TrainPlan(det.train(), 2, H, W, cpu, spec)
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit as trk_build
    from test_tracking_cpu import _layernorm2d
    trk = trk_build("faster_vit_0_224", FrozenBatchNorm2d, _layernorm2d(), out_indices=(0, 1, 2, 3), drop_path_rate=0.1,
                    frozen_stages=0, depths=_DEPTHS).train()
    outs = tuple((i, trk._level_norm(i)) for i in range(4))
    yield "tracking 800x1536 levels train", TrainPlan(trk, 2, 800, 1536, cpu, spec=dict(kind="levels", outs=outs, frozen=0))
    from oracle.configs import CASES as OC
    entry, kw, _ = OC["tiny_ar85"]
    m = F.create_model(entry, drop_path_rate=0.1, **kw)
    yield from _modes("tiny_ar85", m, *_res(m))
    yield from _modes("fv0-like, 96-wide heads", F.create_model("faster_vit_0_224", drop_path_rate=0.1, **HD96), 224, 224)
    yield from _modes("any-res, 13 x 13 windows", F.create_model("faster_vit_0_any_res", drop_path_rate=0.1, **AR173),
                      416, 416)


@pytest.fixture(scope="module")
def plan_launches():
    return [(desc, sorted(set(G.attention_launches(plan)))) for desc, plan in plans()]


def uncovered(plan_launches, cases):
    covered = {c.cls for c in cases}
    return [(desc, a, G.launch_class(a)) for desc, launches in plan_launches for a in launches
            if G.launch_class(a) not in covered]


def test_every_plan_attention_launch_is_covered(plan_launches):
    missing = uncovered(plan_launches, G.CASES)
    assert not missing, "attention launches in no tested geometry class:\n" + "\n".join(
        f"  {desc}: {a.entry} S={a.S} hdp={a.hdp} hd={a.hd} groups={a.groups} heads={a.heads} -> {cls}"
        for desc, a, cls in missing[:20])
    names = {a.entry for _, launches in plan_launches for a in launches}
    assert names == set(G.ENTRIES), set(G.ENTRIES) - names      # the plans reach every entry point
    assert sum(len(v) for _, v in plan_launches) > 300


def test_dropping_a_launched_class_is_noticed(plan_launches):
    """The coverage check names the launch when the only case of a class some plan launches is removed."""
    launched = {G.launch_class(a) for _, launches in plan_launches for a in launches}
    by_cls = {}
    for c in G.CASES:
        by_cls.setdefault(c.cls, []).append(c)
    only = [cls for cls, cs in by_cls.items() if len(cs) == 1 and cls in launched]
    assert only
    for cls in only[:: max(1, len(only) // 6)]:
        miss = uncovered(plan_launches, [c for c in G.CASES if c.cls != cls])
        assert miss and all(m[2] == cls for m in miss), cls
        assert any(m[1].entry == cls[0] for m in miss)


def test_cases_cover_every_geometry_class():
    got = {c.cls for c in G.CASES}
    assert G.required_classes() <= got, sorted(G.required_classes() - got, key=str)
    assert got <= G.required_classes(), sorted(got - G.required_classes(), key=str)
    assert len({c.id for c in G.CASES}) == len(G.CASES)
    # bias = NULL and dbias = NULL at 32, 64 and in the SIMT kernels
    for entry, width in ((e, w) for e in ("fvit_attn_tc_fwd", "fvit_attn_loop_fwd") for w in (32, 64)):
        assert any(c.entry == entry and c.width == width and c.bias == "no_bias" for c in G.CASES), (entry, width)
    for entry in ("fvit_attn_tc_bwd", "fvit_attn_loop_bwd_long"):
        for mode in ("no_bias", "no_dbias"):
            assert any(c.entry == entry and c.width in (32, 64) and c.bias == mode for c in G.CASES), (entry, mode)
    assert any(c.entry == "fvit_attn_core_fwd" and c.bias == "no_bias" for c in G.CASES)
    for mode in ("no_bias", "no_dbias"):
        assert any(c.entry == "fvit_attn_core_bwd" and c.bias == mode for c in G.CASES), mode
    # the key-loop kernels stage bias rows by TMA: S % 4 == 0 with a bias, and always in the backward
    for c in G.CASES:
        if c.entry == "fvit_attn_loop_bwd_long" or (c.entry == "fvit_attn_loop_fwd" and c.bias != "no_bias"):
            assert c.S % 4 == 0, c.id
        if c.entry == "fvit_attn_core_bwd":
            assert G.simt_bwd_smem(c.S, c.hd) <= G.SMEM_MAX, c.id


def test_geometry_class_restates_the_dispatch():
    cls = G.geometry_class
    assert cls("fvit_attn_tc_fwd", 53, 64, 37, 4) == ("fvit_attn_tc_fwd", 64, "slot 64", "partial tile")
    assert cls("fvit_attn_tc_fwd", 16, 32, 16, 4)[2:] == ("slot 16", "full tiles")
    assert cls("fvit_attn_tc_fwd", 17, 32, 16, 4)[2:] == ("slot 32", "full tiles")
    assert cls("fvit_attn_tc_fwd", 128, 80, 3, 2)[2:] == ("slot 128", "full tiles")
    assert cls("fvit_attn_tc_bwd", 49, 32, 6, 8)[3] == "one head per CTA"
    assert cls("fvit_attn_tc_bwd", 49, 32, 6, 8, sms=7)[3] == "head-major"
    assert cls("fvit_attn_tc_bwd", 49, 32, 6, 8, sms=8)[3] == "one head per CTA"
    assert cls("fvit_attn_loop_fwd", 148, 32, 2, 2, lse=True)[2:] == ("2 tiles", "partial key tile", "lse")
    assert cls("fvit_attn_loop_bwd_long", 384, 80, 2, 2)[2:] == ("3+ tiles", "S % 128 == 0")
    # SIMT forward: S = 53 at 24 wide is 31 KB (one-shot, 128 threads); S = 64 at 16 wide is 29 KB with 256 threads;
    # 96-wide heads at S = 53 take 73 KB; S = 229 at 16 wide needs 259 KB -> streaming
    assert cls("fvit_attn_core_fwd", 53, 24, 2, 2)[1:] == ("one-shot <= 48 KB", "block 128", "hd <= 80")
    assert cls("fvit_attn_core_fwd", 64, 16, 2, 2)[1:] == ("one-shot <= 48 KB", "block 256", "hd <= 80")
    assert cls("fvit_attn_core_fwd", 53, 96, 2, 2)[1:] == ("one-shot > 48 KB", "block 128", "hd > 80, % 8 == 0")
    assert cls("fvit_attn_core_fwd", 229, 16, 2, 2)[1:] == ("streaming", "block 256", "hd <= 80")
    assert cls("fvit_attn_core_fwd", 36, 81, 2, 2)[3] == "hd > 80, % 8 != 0"
    assert cls("fvit_attn_core_bwd", 85, 32, 2, 2, hd=16)[1:] == ("> 48 KB", "hdp > hd (pad columns)")
    assert cls("fvit_attn_core_bwd", 229, 16, 2, 2)[1] == "refused (> 227 KB)"
    # the largest window the SIMT backward holds at 16-wide heads, and the first it refuses (train_sm100.cu:1771)
    s = G.largest_simt_bwd_S(16)
    assert G.simt_bwd_smem(s, 16) <= 227 * 1024 < G.simt_bwd_smem(s + 1, 16)
    from fastervit_b200.engine_train_levels import _simt_bwd_smem
    assert all(_simt_bwd_smem(S, hd) == G.simt_bwd_smem(S, hd) for S in (16, 85, 173, 229) for hd in (16, 96))


def test_comparator_passes_one_ulp_and_fails_a_scaled_or_swapped_head():
    g = torch.Generator().manual_seed(0)
    groups, heads, S, hd = 3, 4, 20, 16
    q, k, v, do = (torch.randn(groups, heads, S, hd, generator=g).half().double() for _ in range(4))
    v[:, 2] *= 0.05                  # a head whose outputs are 20x smaller than the others
    bias = torch.randn(heads, S, S, generator=g, dtype=torch.float64)
    r = G.reference(q, k, v, bias, hd ** -0.5, do)
    for name in ("out", "dv", "dq"):
        ref, mag = r[name], r["M_" + name]
        b = G.bound16(ref, mag)
        got = ref.half()
        G.assert_within(got, ref, b, name)
        ulp = ref.half().double()
        step = torch.nextafter(ulp.half(), torch.full_like(ulp.half(), float("inf"))).double() - ulp
        G.assert_within(ulp + step, ref, b, name + " + 1 ulp")      # one fp16 ulp past the rounded value
        scaled = got.clone()
        scaled[:, 2] *= 1.01
        with pytest.raises(AssertionError, match="scaled"):
            G.assert_within(scaled, ref, b, name + " scaled")
        swapped = got.clone()
        swapped[:, [0, 1]] = swapped[:, [1, 0]]
        with pytest.raises(AssertionError, match="swapped"):
            G.assert_within(swapped, ref, b, name + " swapped")
    # the whole-tensor bar alone lets the small head be 1 % wrong
    scaled = r["out"].clone()
    scaled[:, 2] *= 1.01
    G.assert_whole(scaled, r["out"], G.FWD_BAR, "whole")


def test_reference_matches_autograd():
    g = torch.Generator().manual_seed(1)
    q, k, v, do = (torch.randn(2, 3, 11, 8, generator=g, dtype=torch.float64) for _ in range(4))
    bias = torch.randn(3, 11, 11, generator=g, dtype=torch.float64, requires_grad=True)
    r = G.reference(q, k, v, bias.detach(), 0.3, do)
    x = [t.clone().requires_grad_(True) for t in (q, k, v)]
    att = x[0] @ x[1].transpose(-2, -1) * 0.3 + bias
    o = att.softmax(-1) @ x[2]
    o.backward(do)
    torch.testing.assert_close(r["out"], o.detach())
    torch.testing.assert_close(r["lse"], torch.logsumexp(att.detach(), -1) * G.LOG2E)
    for name, t in zip(("dq", "dk", "dv"), x):
        torch.testing.assert_close(r[name], t.grad)
    torch.testing.assert_close(r["dbias"], bias.grad)
    for name in ("out", "dq", "dk", "dv", "dbias"):
        assert (r["M_" + name] >= r[name].abs() * (1 - 1e-12)).all(), name


# ---------------------------------------------------------------------------------------------- plan-build refusal
def _train_plans(name, kw, res):
    from fastervit_b200.engine_train import TrainPlan
    cpu = torch.device("cpu")
    m = F.create_model(name, drop_path_rate=0.0, **kw)
    return (lambda: TrainPlan(m.train(), 2, *res, cpu),
            lambda: TrainPlan(m.eval(), 2, *res, cpu, spec=dict(kind=None, eval=True)), m)


@pytest.mark.parametrize("name,kw,res,sizes,hd", [
    # 15 x 15 windows at 16-wide heads: 229 tokens with the carriers at level 2 need 267 KiB, 225 at level 3 259 KiB
    ("faster_vit_0_any_res", dict(resolution=[480, 480], window_size=[7, 7, 15, 15], dim=16, in_dim=16,
                                  depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]), (480, 480), (229, 225), 16),
    # 11 x 11 windows with 96-wide heads: S = 125 at level 2 needs 251 KiB, 121 at level 3 242 KiB
    ("faster_vit_0_any_res", dict(resolution=[352, 352], window_size=[7, 7, 11, 11], dim=24, in_dim=16,
                                  depths=[1, 1, 2, 1], num_heads=[1, 1, 1, 2]), (352, 352), (125, 121), 96),
])
def test_windows_the_simt_backward_cannot_hold_are_refused_at_plan_build(name, kw, res, sizes, hd):
    """the train and eval-gradient plans raise while they are built, naming the level (the backward is emitted from
    the last level on: level 3 is met first), S and the head width; the eval plan builds"""
    from fastervit_b200.engine import Plan
    train, eval_grad, m = _train_plans(name, kw, res)
    assert all(G.simt_bwd_smem(S, hd) > G.SMEM_MAX for S in sizes)
    for build in (train, eval_grad):
        with pytest.raises(L.FvitError, match=rf"^level 3 .*{sizes[1]}-token windows with {hd}-wide heads.* "
                                              rf"{G.simt_bwd_smem(sizes[1], hd) / 1024:.0f} KiB"):
            build()
    # inference streams what does not fit: the eval plan builds, with the SIMT forward at both window sizes
    plan = Plan(m.eval(), 2, *res, False, torch.device("cpu"))
    got = {a.S for a in G.attention_launches(plan) if a.entry == "fvit_attn_core_fwd"}
    assert set(sizes) <= got, got


def test_96_wide_heads_at_7x7_windows_still_train():
    """S = 16 / 49 / 53 with 96-wide heads: at most 92 KiB of the SIMT backward's shared memory"""
    kw = dict(HD96, resolution=[224, 224], window_size=[7, 7, 7, 7])
    train, eval_grad, _ = _train_plans("faster_vit_0_any_res", kw, (224, 224))
    for build in (train, eval_grad):
        launches = {(a.entry, a.S, a.hd) for a in G.attention_launches(build())}
        bwd = {(S, hd) for e, S, hd in launches if e == "fvit_attn_core_bwd"}
        assert {(16, 96), (49, 96), (53, 96)} <= bwd, bwd
        assert max(G.simt_bwd_smem(S, hd) for S, hd in bwd) <= 92 * 1024
