"""Host-side checks of the MOTRv2 tracking backbone (fastervit_b200.tracking): state_dict schema against the reference
module for the nine names, the norm classes the builder accepts and refuses, checkpoint loading through
`_load_state_dict`, and the train plans the norm kinds produce (built on the CPU, nothing is launched)."""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = Path(__file__).parent / "golden"
CASES = ["track_tiny_fv0", "track_tiny_fv4", "track_tiny_21k", "track_tiny_hatf"]


def _layernorm2d():
    """timm's LayerNorm2d as the reference imports it (the oracle's stand-in of timm.models.layers)"""
    sys.path.insert(0, str(ROOT / "oracle" / "ref_shim"))
    try:
        from timm.models.layers import LayerNorm2d
    finally:
        sys.path.remove(str(ROOT / "oracle" / "ref_shim"))
    return LayerNorm2d


def _schema(sd):
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def _classes(pair):
    from fastervit_b200.tracking import FrozenBatchNorm2d
    stem, out = pair.split("_")
    cls = {"bn": nn.BatchNorm2d, "frozen": FrozenBatchNorm2d, "ln": _layernorm2d()}
    return cls[stem], cls[out]


def _tiny(case, pair, **kw):
    from fastervit_b200.tracking import build_fastervit
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    stem, out = _classes(pair)
    return g, build_fastervit(g["name"], stem, out, out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **g["kwargs"], **kw)


def test_state_dict_schema_of_the_nine_names():
    from fastervit_b200.tracking import build_fastervit
    want = torch.load(GOLDEN / "track_schema.pt", weights_only=False)
    assert len(want) == 18
    for (name, pair), keys in want.items():
        stem, out = _classes(pair)
        torch.manual_seed(0)
        with torch.no_grad():
            got = _schema(build_fastervit(name, stem, out, use_checkpoint=False).state_dict())
        assert got == keys, (name, pair)


@pytest.mark.parametrize("case", CASES)
def test_tiny_schemas_match_the_reference(case):
    for pair in ("frozen_ln", "bn_ln", "frozen_frozen", "bn_bn"):
        g, m = _tiny(case, pair)
        assert [k[:2] for k in _schema(m.state_dict())] == [k[:2] for k in g["pairs"][pair]["state_keys"]], pair


def test_reference_shaped_norm_classes_are_accepted():
    """torchvision's FrozenBatchNorm2d, the reference's LayerNorm2d and this package's FrozenBatchNorm2d: classified by
    what they are"""
    from fastervit_b200.engine import norm_kind
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    kinds = {FrozenBatchNorm2d: "frozen", _layernorm2d(): "ln", nn.BatchNorm2d: "bn"}
    try:
        from torchvision.ops import FrozenBatchNorm2d as TvFrozen
        kinds[TvFrozen] = "frozen"
    except ImportError:   # (torchvision is optional: the structural check is the same for it)
        pass
    for cls, kind in kinds.items():
        assert norm_kind(cls(8)) == kind, cls
    for stem in [c for c, k in kinds.items() if k != "ln"]:
        m = build_fastervit("faster_vit_0_224", stem, _layernorm2d(), dim=16, in_dim=16, depths=[1, 1, 2, 1],
                            num_heads=[1, 2, 4, 8])
        assert isinstance(m.patch_embed.conv_down[1], stem) and m.patch_embed.conv_down[1].eps == 1e-4
        assert isinstance(m.norm, _layernorm2d()) and not hasattr(m, "norm3")


def test_unsupported_norms_raise():
    from fastervit_b200 import lib as L
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    kw = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])

    class LNNoBias(nn.LayerNorm):
        def __init__(self, n):
            super().__init__(n, bias=False)
    for stem, out in ((nn.BatchNorm2d, lambda n: nn.GroupNorm(4, n)), (_layernorm2d(), FrozenBatchNorm2d),
                      (nn.BatchNorm2d, LNNoBias), (nn.BatchNorm2d, nn.LayerNorm)):
        with pytest.raises(L.FvitError, match="accepted|stem"):
            build_fastervit("faster_vit_0_224", stem, out, **kw)
    with pytest.raises(L.FvitError, match="unknown tracking backbone"):
        build_fastervit("faster_vit_0_any_res", nn.BatchNorm2d, nn.BatchNorm2d)


@pytest.mark.parametrize("case", CASES)
def test_classification_checkpoint_keys_match_the_reference(case, tmp_path, capsys):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g, m = _tiny(case, "frozen_ln")
    want = g["pairs"]["frozen_ln"]["load_cls"]
    name = g["name"] if g["name"] != "faster_vit_0_224_hat_False" else "faster_vit_0_224"
    cls = F.create_model(name, **{k: v for k, v in g["kwargs"].items() if k != "do_propagation"})
    O.synth_fill_(cls.state_dict(), g["seeds"]["w"] + 1)
    path = tmp_path / "cls.pth"
    torch.save({"model": {"module." + k: v for k, v in cls.state_dict().items()}}, path)
    missing, unexpected = m._load_state_dict(str(path))
    assert sorted(missing) == want["missing"] and sorted(unexpected) == want["unexpected"]
    assert "do not match exactly" in capsys.readouterr().out
    assert torch.equal(m.norm.weight.detach(), want["norm_weight"])   # the BatchNorm's weight, in the level-3 LayerNorm


def test_frozen_state_dict_round_trip():
    from fastervit_b200.tracking import FrozenBatchNorm2d
    _, a = _tiny("track_tiny_fv0", "frozen_frozen")
    sd = a.state_dict()
    frozen = [n for n, m in a.named_modules() if isinstance(m, FrozenBatchNorm2d)]
    assert len(frozen) == 6   # the two stem norms and the four level norms
    assert not any(k.startswith(tuple(f + "." for f in frozen)) and k.endswith("num_batches_tracked") for k in sd)
    assert all(not list(m.parameters()) for m in a.modules() if isinstance(m, FrozenBatchNorm2d))
    _, b = _tiny("track_tiny_fv0", "frozen_frozen")
    # a BatchNorm checkpoint carries num_batches_tracked: a frozen BatchNorm drops it
    sd_bn = dict(sd, **{"patch_embed.conv_down.1.num_batches_tracked": torch.tensor(3)})
    res = b.load_state_dict(sd_bn, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    for k, v in b.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("pair", ["frozen_ln", "frozen_frozen", "bn_ln"])
@pytest.mark.parametrize("frozen_stages", [-1, 0, 2])
def test_train_plan_for_each_norm_kind(pair, frozen_stages):
    """the levels-mode train plan of each norm pair (built on the CPU): which kernels the level outputs and the stem
    take, and which parameters get a gradient slice"""
    from fastervit_b200.engine_train import TrainPlan
    _, m = _tiny("track_tiny_fv0", pair, frozen_stages=frozen_stages)
    m.train()
    outs = tuple((i, m._level_norm(i)) for i in range(4))
    plan = TrainPlan(m, 2, 96, 160, torch.device("cpu"), spec=dict(kind="levels", outs=outs, frozen=frozen_stages))
    fwd = [op[2] for op in plan.ops]
    bwd = [op[2] for op in plan.bwd_ops]
    stem, out = pair.split("_")
    if out == "ln":
        assert fwd.count("fvit_feature_map_ln_fwd") == 4 and "fvit_feature_map_fwd" not in fwd
        assert bwd.count("fvit_feature_map_ln_bwd") == 4
        for i in range(4):
            assert id(m._level_norm(i).weight) in plan._goff and id(m._level_norm(i).bias) in plan._goff
    else:
        assert fwd.count("fvit_feature_map_fwd") == 4 and "fvit_feature_map_ln_fwd" not in fwd
        assert "fvit_feature_map_bwd" not in bwd and "fvit_feature_map_ln_bwd" not in bwd
    if stem == "frozen":
        assert "fvit_bn_finalize_pivot" not in fwd[:fwd.index("fvit_affine_rows")]   # (the stem: a fixed affine)
    stem_w = m.patch_embed.conv_down[0].weight
    # stem convolutions take a weight gradient unless the stem is frozen (frozen_stages >= 0)
    assert (id(stem_w) in plan._on_path) == (frozen_stages < 0)
    # running statistics are written only for batch-statistics BatchNorms
    frozen_bufs = {b.data_ptr() for mod in m.modules() if not isinstance(mod, nn.BatchNorm2d)
                   for n, b in mod.named_buffers(recurse=False) if n.startswith("running")}
    for fn, args, name in plan.ops:
        if name == "fvit_bn_finalize_pivot":
            assert not frozen_bufs & set(a for a in args if isinstance(a, int))
