"""Host-side checks of the DINO detection backbone (fastervit_b200.detection): state_dict schema and checkpoint loading
against the reference module, the per-input carrier geometry against what the reference used at every golden shape, the
kernels the plans pick at DETR training sizes (the plans are built on the CPU, nothing is launched), and the plan cache
bound."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_token_init.py
from _token_init import detr_shapes, level_sizes  # noqa: E402

GOLDEN = Path(__file__).parent / "golden"
CASES = ["det_tiny_fv0", "det_tiny_fv4", "det_tiny_21k"]


def _golden(case):
    return torch.load(GOLDEN / f"{case}.pt", weights_only=False)


def _schema(sd):
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def test_state_dict_schema_of_the_eight_names():
    from fastervit_b200.detection import build_fastervit
    want = torch.load(GOLDEN / "det_schema.pt", weights_only=False)
    assert len(want) == 8
    for name, keys in want.items():
        torch.manual_seed(0)
        with torch.no_grad():
            got = _schema(build_fastervit(name, out_indices=(1, 2, 3), use_checkpoint=False).state_dict())
        assert got == keys, name


@pytest.mark.parametrize("case", CASES)
def test_tiny_schema_and_classification_checkpoint_keys(case):
    import fastervit_b200 as F
    from fastervit_b200.detection import build_fastervit
    g = _golden(case)
    det = build_fastervit(g["name"], out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **g["kwargs"])
    assert [k[:2] for k in _schema(det.state_dict())] == [k[:2] for k in g["state_keys"]]   # (the golden ran in fp64)
    cls = F.create_model(g["name"], **{k: v for k, v in g["kwargs"].items() if k != "do_propagation"})
    res = det.load_state_dict(cls.state_dict(), strict=False)
    assert sorted(res.missing_keys) == g["load_cls"]["missing"]
    assert sorted(res.unexpected_keys) == g["load_cls"]["unexpected"]


@pytest.mark.parametrize("case", ["det_tiny_fv0", "det_tiny_fv4"])
def test_carrier_geometry_matches_the_reference(case):
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import Plan, grid_coords, token_geometry
    g = _golden(case)
    det = build_fastervit(g["name"], drop_path_rate=0.0, **g["kwargs"]).eval()
    shapes0 = {k: tuple(v.shape) for k, v in det.state_dict().items()}
    for (H, W), ref in g["shapes"].items():
        geo_ref = ref["geometry"]
        Hc, Wc = level_sizes(H, W)[2]
        geo = token_geometry(det, 2, Hc, Wc)
        (kh, sh, oh), (kw, sw, ow) = geo["pool"]
        assert ((kh, kw), (sh, sw)) == geo_ref["pool"], (H, W)
        assert (geo["Hp"], geo["Wp"]) == geo_ref["level_in"][2:]
        assert (oh, ow) == (geo_ref["hg"], geo_ref["wg"]) and oh * ow == geo_ref["s_ct"] == geo_ref["tokens"][1]
        s = oh * ow // 2
        assert torch.equal(geo["hat_pe_coords"][ow + 1], torch.tensor([(1 - s) / s, (1 - s) / s]))
        assert torch.equal(geo["pe_coords"][0], torch.tensor([-1.0, -1.0]))   # (0 - 49 // 2) / (49 // 2)
        assert torch.allclose(geo["pe_coords"][-1], torch.tensor([(6 - 24) / 24, (6 - 24) / 24]))
        plan = Plan(det, 2, H, W, False, torch.device("cpu"))
        tl = next(w["tl"] for _, name, w in plan.marks if name == "levels.2.out")
        n_ct, S, ncw, nwin = tl["n_ct"], tl["S"], tl["ncw"], tl["nwin"]
        assert n_ct == geo_ref["s_ct"] and S == 49 + 4
        tok = [op for op in plan.ops if op[2] in ("fvit_token_init_fwd", "fvit_token_init_nchw_fwd")]
        assert [op[2] for op in tok] == ["fvit_token_init_nchw_fwd"] and tok[0][1][9:15] == (kh, kw, sh, sw, oh, ow)
        # the carrier bias: the 4 x 4 table padded (or cropped) to S_ct, in a plan buffer
        bias = [op[1] for op in plan.prep_ops if op[2] == "unless_deploy" and op[1][1].__name__ == "fvit_attn_bias_fwd"]
        bias += [op[1] for op in plan.prep_ops if op[2] == "fvit_attn_bias_fwd"]
        assert sorted({(a[3], a[4]) for a in bias}) == sorted({(n_ct, 16), (53, 49), (49, 49)})   # level 3: no carriers
        assert torch.equal(grid_coords(2, 4, 4)[-1], torch.tensor([(1 - 4) / 4, (3 - 4) / 4]))
    # the modules' buffers keep their construction shapes (the plans own the per-shape tables)
    assert {k: tuple(v.shape) for k, v in det.state_dict().items()} == shapes0


def _launches(plan):
    """every launch of a plan's lists as (name, args), deploy-guarded ones unwrapped"""
    for ops in (v for v in vars(plan).values() if isinstance(v, list)):
        for op in ops:
            if isinstance(op, tuple) and len(op) == 3 and isinstance(op[2], str):
                yield op[2], (op[1][2] if op[0] == "unless_deploy" else op[1])


# where each entry point keeps (Hp, Wp) and (kh, kw, sh, sw, oh, ow) in its argument list (include/fvit.h)
_TOKEN_INIT_ARGS = {"fvit_token_init_nchw_fwd": (4, 9), "fvit_token_init_nchw_bwd": (7, 11),
                    "fvit_token_init_nchw_dgrad": (5, 9)}
# where each attention entry point keeps S
_ATTN_S = {"fvit_attn_tc_fwd": 3, "fvit_hat_attn_fwd": 7, "fvit_attn_loop_fwd": 3, "fvit_attn_core_fwd": 3,
           "fvit_attn_tc_bwd": 5, "fvit_attn_core_bwd": 5, "fvit_attn_loop_bwd_long": 8}


@pytest.mark.parametrize("hw", [(64, 64), (96, 96)] + detr_shapes(40))
def test_detr_size_plans_launch_what_the_kernel_tests_cover(hw):
    """The eval plan and the levels-mode train plan (batch 2, the spec forward_levels passes) of the fv0-like detection
    backbone at DETR training sizes: the tokenizer launches carry token_geometry's pool, whose windows tile the padded
    map exactly; carrier attention takes the tile kernels only where they fit (forward S <= 128, tensor-core backward S
    <= 64) and the key-loop kernels only for S % 4 == 0 (TMA-staged bias rows); every bias-table backward matches its
    forward's (S, L); every scatter_add_rows map is injective (a plain read-modify-write, include/fvit.h)."""
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import Plan, token_geometry
    from fastervit_b200.engine_train import TrainPlan
    H, W = hw
    det = build_fastervit("faster_vit_0_224", out_indices=(0, 1, 2, 3), drop_path_rate=0.0, dim=16, in_dim=16,
                          depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    geos = {}
    for i, (Hc, Wc) in enumerate(level_sizes(H, W)):
        if det.levels[i].conv:
            continue
        geo = token_geometry(det, i, Hc, Wc)
        if geo["has_ct"]:
            (kh, sh, oh), (kw, sw, ow) = geo["pool"]
            assert (oh - 1) * sh + kh == geo["Hp"] and (ow - 1) * sw + kw == geo["Wp"], (hw, i, geo["pool"])
            geos[i] = ((geo["Hp"], geo["Wp"]), (kh, kw, sh, sw, oh, ow))
    assert geos, "level 2 has carriers at every size"
    n_ct = {g[1][4] * g[1][5] for g in geos.values()}
    spec = dict(kind="levels", outs=tuple((i, getattr(det, f"norm{i}")) for i in range(4)), frozen=-1)
    cpu = torch.device("cpu")
    plans = [Plan(det.eval(), 2, H, W, False, cpu), TrainPlan(det.train(), 2, H, W, cpu, spec)]
    for plan in plans:
        launches = list(_launches(plan))
        names = [n for n, _ in launches]
        tok = [(n, a) for n, a in launches if n in _TOKEN_INIT_ARGS]
        assert names.count("fvit_token_init_nchw_fwd") == len(geos), hw
        assert "fvit_token_init_fwd" not in names and "fvit_token_init_bwd" not in names
        for n, a in tok:
            hp, kp = _TOKEN_INIT_ARGS[n]
            assert (tuple(a[hp:hp + 2]), tuple(a[kp:kp + 6])) in geos.values(), (hw, n, a[hp:hp + 2], a[kp:kp + 6])
        carrier_s = set()
        for n, a in launches:
            if n not in _ATTN_S:
                continue
            S = a[_ATTN_S[n]]
            if S in n_ct:
                carrier_s.add(S)
            if n in ("fvit_attn_tc_fwd", "fvit_hat_attn_fwd"):
                assert S <= 128, (hw, n, S)
            if n == "fvit_attn_tc_bwd":
                assert S <= 64, (hw, n, S)
            if n in ("fvit_attn_loop_fwd", "fvit_attn_loop_bwd_long"):
                assert S % 4 == 0, (hw, n, S)
        assert carrier_s == n_ct, (hw, carrier_s, n_ct)
        bias_fwd = {a[5]: (a[3], a[4]) for n, a in launches if n == "fvit_attn_bias_fwd"}
        assert {(S, L) for S, L in bias_fwd.values() if S in n_ct} == {(s, 16) for s in n_ct}   # the 4 x 4 table
        for n, a in launches:
            if n == "fvit_attn_bias_bwd":
                assert bias_fwd.get(a[1]) == (a[4], a[5]), (hw, bias_fwd.get(a[1]), a[4:6])
    train = plans[1]
    assert any(n == "fvit_token_init_nchw_bwd" for n, _ in _launches(train))
    by_ptr = {t.data_ptr(): t for t in train.bufs.named.values()}
    scatters = [a for n, a in _launches(train) if n == "fvit_scatter_add_rows"]
    assert scatters, "the carriers' backward scatters them back"
    for a in scatters:
        mp = by_ptr[a[4]].flatten()[:a[5]]
        valid = mp[mp >= 0]
        assert valid.numel() == torch.unique(valid).numel(), (hw, "map repeats a destination row")


def test_classification_geometry_is_unchanged():
    """token_geometry on a classification model restates the construction-time grid, pool and side // 2 scaling"""
    import fastervit_b200 as F
    from fastervit_b200.engine import token_geometry
    m = F.create_model("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    geo = token_geometry(m, 2, 14, 14)
    assert geo["sr"] == [2, 2] and geo["pool"] == m.levels[2].global_tokenizer.pool and geo["tokens"] == "map"
    r = torch.arange(7, dtype=torch.float32)
    grid = torch.stack(torch.meshgrid(r, r, indexing="ij"))
    assert torch.equal(geo["pe_coords"], ((grid - 3) / 3).flatten(1).t())
    assert not geo["own_tables"] and geo["hat_pe_coords"].shape == (16, 2)
    from fastervit_b200 import lib as L
    with pytest.raises(L.FvitError, match="built for"):
        token_geometry(m, 2, 21, 21)


def test_conv_levels_run_on_the_window_padded_map():
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import Plan
    det = build_fastervit("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]).eval()
    plan = Plan(det, 1, 96, 160, False, torch.device("cpu"))      # level 0: 24 x 40 -> 28 x 42
    lv = next(w["lv"] for _, name, w in plan.marks if name == "levels.0.out")
    assert (lv["H"], lv["W"], lv["Hb"], lv["Wb"]) == (24, 40, 28, 42)
    assert int((lv["interior"] >= 0).sum()) == 28 * 42 and lv["pix"].numel() == 24 * 40
    assert sum(1 for op in plan.ops if op[0] == "zero") >= 2
    assert plan.logits is None and plan.pooled is None


class _FakePlan:
    pass


def test_plan_cache_drops_the_least_recently_used_and_its_prepped_entry():
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import Engine
    det = build_fastervit("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    assert det.plan_cache_size == 2
    eng = det._get_engine()
    plans = {k: _FakePlan() for k in "abc"}
    for k, p in plans.items():
        eng.plans[k] = p
        eng._prepped[id(p)] = ("packed", k)
        eng.trim_plans()
    assert list(eng.plans) == ["b", "c"] and id(plans["a"]) not in eng._prepped
    det.set_plan_cache_size(1)
    assert list(eng.plans) == ["c"] and set(eng._prepped) == {id(plans["c"])}
    det.set_plan_cache_size(None)
    for k in "xyz":
        eng.plans[k] = _FakePlan()
        eng.trim_plans()
    assert len(eng.plans) == 4
    # classification models keep every plan
    import fastervit_b200 as F
    e2 = Engine(F.create_model("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]))
    for k in range(5):
        e2.plans[k] = _FakePlan()
        e2.trim_plans()
    assert len(e2.plans) == 5


def test_interface_and_rejections():
    from fastervit_b200 import lib as L
    from fastervit_b200.detection import FasterViTDet, build_fastervit
    det = build_fastervit("faster_vit_0_224", out_indices=(1, 2, 3), frozen_stages=2, dim=16, in_dim=16,
                          depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    assert isinstance(det, FasterViTDet) and det.num_features == [16, 32, 64, 128] and det.out_indices == (1, 2, 3)
    assert det.train() is det and det.eval() is det and det.enable_input_grad() is det
    assert not any(p.requires_grad for p in det.patch_embed.parameters())
    assert not any(p.requires_grad for p in det.levels[0].parameters())
    assert all(p.requires_grad for p in det.levels[1].parameters())
    det.train()
    assert not det.levels[0].training and det.levels[1].training
    assert not hasattr(det, "norm") and not hasattr(det, "head") and hasattr(det, "norm3") and not hasattr(det, "norm0")
    with pytest.raises(L.FvitError):
        build_fastervit("faster_vit_0_224", drop_rate=0.1)
    with pytest.raises(L.FvitError):
        build_fastervit("faster_vit_5_224")
    with pytest.raises(L.FvitError):
        det.switch_to_deploy()
    with pytest.raises(L.FvitError, match="no eval-mode gradients"):
        det.eval().forward_raw(torch.zeros(1, 3, 64, 64))
