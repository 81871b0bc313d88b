"""GPU tests of the MOTRv2 tracking backbone (fastervit_b200.tracking) against the goldens of the unmodified reference
module, for every norm pair (stem, output) in {(Frozen, LN) -- the published recipe, (BN, LN), (Frozen, Frozen),
(BN, BN)}: eval level maps and masks at every golden shape, train steps with frozen_stages -1, 0 and 2 (maps, running
statistics after the step, parameter gradients), and the recipe's full 800 x 1536 step with the image gradient."""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLDEN = Path(__file__).parent / "golden"
TOL = 5e-3   # max |error| / max |reference| of a level map (as test_detection_gpu.py)
CASES = ["track_tiny_fv0", "track_tiny_fv4", "track_tiny_21k", "track_tiny_hatf"]
PAIRS = ["frozen_ln", "bn_ln", "frozen_frozen", "bn_bn"]


class _Nested:   # util.misc.NestedTensor: .tensors and .mask
    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask


def _layernorm2d():
    sys.path.insert(0, str(ROOT / "oracle" / "ref_shim"))
    try:
        from timm.models.layers import LayerNorm2d
    finally:
        sys.path.remove(str(ROOT / "oracle" / "ref_shim"))
    return LayerNorm2d


def _model(g, pair, **kw):
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    from oracle import fastervit_oracle as O
    stem, out = pair.split("_")
    cls = {"bn": nn.BatchNorm2d, "frozen": FrozenBatchNorm2d, "ln": _layernorm2d()}
    m = build_fastervit(g["name"], cls[stem], cls[out], out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **g["kwargs"],
                        **kw)
    O.synth_fill_(m.state_dict(), g["seeds"]["w"])
    return m.cuda()


def _sample(t, step=1):
    f = t.detach().flatten()
    return f[::max(1, (f.numel() + 511) // 512)][::step].double().cpu()


def _rel_l2(a, b, floor):
    return ((a.double() - b.double()).norm() / max(b.double().norm().item(), floor * b.numel() ** 0.5)).item()


@pytest.mark.parametrize("pair", PAIRS)
@pytest.mark.parametrize("case", CASES)
def test_level_maps_match_the_reference_at_every_shape(case, pair):
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    m = _model(g, pair).eval()
    for (H, W), ref in g["pairs"][pair]["shapes"].items():
        x = O.synth_input(2, [H, W], ref["x_seed"], torch.float32).cuda()
        mask = torch.zeros(2, H, W, dtype=torch.bool, device="cuda")
        mask[1, :, W - W // 4:] = True
        with torch.no_grad():
            outs = m(_Nested(x, mask))
        assert sorted(outs) == [0, 1, 2, 3]
        for k, o in outs.items():
            want = ref["levels"][k]
            assert tuple(o.tensors.shape) == tuple(want["shape"]), (H, W, k)
            err = (_sample(o.tensors) - want["sample"].double()).abs().max().item() / want["amax"]
            assert err < TOL, (case, pair, H, W, k, err)
            assert torch.equal(o.mask.cpu(), g["masks"][(H, W)][k]), (H, W, k)


def _train_step(g, pair, H, W, fs, ref, want_dx=False):
    from oracle import fastervit_oracle as O
    m = _model(g, pair, frozen_stages=fs).train()
    if want_dx:
        m.enable_input_grad()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    x = O.synth_input(ref["batch"], [H, W], ref["x_seed"], torch.float32).cuda().requires_grad_(want_dx)
    outs = m(_Nested(x, torch.zeros(ref["batch"], H, W, dtype=torch.bool, device="cuda")))
    maps = [outs[k].tensors for k in range(4)]
    gen = torch.Generator().manual_seed(ref["g_seed"])
    gs = [torch.randn(tuple(t.shape), generator=gen, dtype=torch.float64).float().cuda() for t in maps]
    sum((t * gk).sum() for t, gk in zip(maps, gs)).backward()
    tag = (g["case"], pair, H, W, fs)
    for k, t in enumerate(maps):
        want = ref["levels"][k]
        err = (_sample(t) - want["sample"].double()).abs().max().item() / want["amax"]
        assert err < TOL, (*tag, "map", k, err)
    sd = m.state_dict()
    for key, want in ref["stats_after"].items():
        err = (_sample(sd[key]) - want["sample"].double()).abs().max().item() / max(want["amax"], 1e-6)
        assert err < TOL, (*tag, key, err)
    # frozen BatchNorms: every buffer bitwise unchanged by the step
    from fastervit_b200.tracking import FrozenBatchNorm2d
    for name, mod in m.named_modules():
        if isinstance(mod, FrozenBatchNorm2d):
            for bn_, buf in mod.named_buffers(recurse=False):
                assert torch.equal(buf, before[f"{name}.{bn_}"]), (*tag, name, bn_)
    named = dict(m.named_parameters())
    gr = ref["grads"]
    assert {n for n, p in named.items() if p.grad is not None} == set(gr["names"]), tag
    # tolerances of test_detection_gpu.py::test_train_mode_matches_the_reference
    floor = 1e-3 * max(gr["amax"])
    want = dict(zip(gr["names"], gr["samples"].split(gr["len"])))
    rel = {n: _rel_l2(_sample(named[n].grad, st), want[n], floor) for n, st in zip(gr["names"], gr["step"])}
    bad = sorted(((e, n) for n, e in rel.items() if e > (6e-2 if n.startswith("patch_embed.") else 4e-2)),
                 reverse=True)
    med = sorted(rel.values())[len(rel) // 2]
    assert not bad and med <= 4e-3, (*tag, med, bad[:8])
    return m, x


@pytest.mark.parametrize("pair", PAIRS)
@pytest.mark.parametrize("case", CASES)
def test_train_mode_matches_the_reference(case, pair):
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    train = {}   # (the train steps live in one file per train shape: <case>_train_<H>x<W>.pt)
    for f in sorted(GOLDEN.glob(f"{case}_train_*.pt")):
        train |= torch.load(f, weights_only=False)["pairs"][pair]
    assert len(train) == 6
    for (H, W, fs), ref in train.items():
        m, _ = _train_step(g, pair, H, W, fs, ref)
        if fs < 0 and pair.startswith("frozen"):   # a frozen-BatchNorm stem with trainable convolutions
            assert m.patch_embed.conv_down[0].weight.grad is not None
            assert m.patch_embed.conv_down[3].weight.grad is not None


def test_full_size_recipe_step_with_the_image_gradient():
    """(Frozen, LN) at 800 x 1536, batch 1: several hundred level-2 carriers (the key-loop attention kernels)"""
    g = torch.load(GOLDEN / "track_tiny_fv0_full.pt", weights_only=False)
    ((H, W, fs), ref), = g["train"].items()
    _, x = _train_step(g, "frozen_ln", H, W, fs, ref, want_dx=True)
    want = ref["x_grad"]
    assert _rel_l2(_sample(x.grad), want["sample"], 1e-3 * want["amax"]) <= 4e-2


def test_load_into_the_frozen_stem_reaches_the_next_forward():
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / "track_tiny_fv0.pt", weights_only=False)
    m = _model(g, "frozen_ln").eval()
    x = O.synth_input(1, [96, 160], 3, torch.float32).cuda()
    with torch.no_grad():
        a = [t.clone() for t in m.forward_raw(x)]
    sd = m.state_dict()
    sd["patch_embed.conv_down.1.weight"] = sd["patch_embed.conv_down.1.weight"] * 1.5
    sd["patch_embed.conv_down.4.running_mean"] = sd["patch_embed.conv_down.4.running_mean"] + 0.25
    m.load_state_dict(sd)
    with torch.no_grad():
        b = m.forward_raw(x)
    fresh = _model(g, "frozen_ln").eval()
    fresh.load_state_dict(sd)
    with torch.no_grad():
        c = fresh.forward_raw(x)
    for ta, tb, tc in zip(a, b, c):
        assert not torch.equal(ta, tb)
        assert torch.equal(tb, tc)
    # the same through a train step: the buffers feed the train plan's stem too, and stay as loaded
    m.train()
    sum(t.sum() for t in m.forward_raw(x)).backward()
    assert torch.equal(m.state_dict()["patch_embed.conv_down.1.weight"], sd["patch_embed.conv_down.1.weight"])


def test_eval_gradients_raise():
    from fastervit_b200 import lib as L
    g = torch.load(GOLDEN / "track_tiny_fv0.pt", weights_only=False)
    m = _model(g, "frozen_ln").eval()
    with pytest.raises(L.FvitError, match="no eval-mode gradients"):
        m.forward_raw(torch.randn(1, 3, 96, 128, device="cuda"))
