"""GPU tests of the DINO detection backbone (fastervit_b200.detection) at any input size: normed level maps against the
goldens of the unmodified reference module at every golden shape (224^2, a carrier grid smaller than the bias table,
non-square and odd sizes, 160 carriers on the key-loop attention), and a shape sweep under the plan-cache bound."""
import gc
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_token_init.py
from _token_init import detr_shapes  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"
TOL = 5e-3   # max |error| / max |reference| of a level map (the level-map tolerance of test_backbone_gpu.py)


class _Nested:   # DINO's util.misc.NestedTensor: .tensors and .mask
    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask


def _sample(t):
    f = t.detach().flatten()
    return f[::max(1, (f.numel() + 511) // 512)].double().cpu()


def _model(g):
    from fastervit_b200.detection import build_fastervit
    from oracle import fastervit_oracle as O
    det = build_fastervit(g["name"], out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **g["kwargs"])
    O.synth_fill_(det.state_dict(), g["seeds"]["w"])
    return det.cuda().eval()


@pytest.mark.parametrize("case", ["det_tiny_fv0", "det_tiny_fv4", "det_tiny_21k", "det_tiny_hd64"])
def test_level_maps_match_the_reference_at_every_shape(case):
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    det = _model(g)
    for (H, W), ref in g["shapes"].items():
        x = O.synth_input(2, [H, W], ref["x_seed"], torch.float32).cuda()
        mask = torch.zeros(2, H, W, dtype=torch.bool, device="cuda")
        mask[1, :, W - W // 4:] = True
        with torch.no_grad():
            outs = det(_Nested(x, mask))
        assert sorted(outs) == [0, 1, 2, 3]
        for k, o in outs.items():
            want = ref["levels"][k]
            assert isinstance(o, _Nested) and tuple(o.tensors.shape) == tuple(want["shape"]), (H, W, k)
            err = (_sample(o.tensors) - want["sample"].double()).abs().max().item() / want["amax"]
            assert err < TOL, (case, H, W, k, err)
            assert torch.equal(o.mask.cpu(), ref["masks"][k]), (H, W, k)


def test_shape_sweep_under_the_plan_cache_bound():
    from fastervit_b200.detection import build_fastervit
    from oracle import fastervit_oracle as O
    det = build_fastervit("faster_vit_0_224", out_indices=(1, 2, 3), dim=32, in_dim=16, depths=[1, 1, 2, 1],
                          num_heads=[1, 2, 4, 8])
    O.synth_fill_(det.state_dict(), 3)
    det = det.cuda().eval()
    shapes = detr_shapes(10)
    xs = {hw: O.synth_input(1, list(hw), 7, torch.float32).cuda() for hw in shapes}
    gc.collect()     # (earlier tests' models: a model and its engine reference each other)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    # footprint of each shape's plan on its own (bound 1: every other plan is gone)
    det.set_plan_cache_size(1)
    foot = {}
    for hw in shapes:
        with torch.no_grad():
            outs = det.forward_raw(xs[hw])
        del outs
        torch.cuda.synchronize()
        foot[hw] = torch.cuda.memory_allocated() - base
    det.set_plan_cache_size(2)
    first = None
    with torch.no_grad():
        for hw in shapes:
            outs = det.forward_raw(xs[hw])
            if first is None:
                first = [o.clone() for o in outs]
            del outs
    eng = det._get_engine()
    assert len(eng.plans) == 2 and len(eng._prepped) <= 2
    torch.cuda.synchronize()     # (no gc.collect(): an evicted plan's memory is freed when it is dropped)
    two = sum(sorted(foot.values())[-2:]) + sum(o.numel() * o.element_size() for o in first)
    assert torch.cuda.memory_allocated() - base <= two + (4 << 20), (torch.cuda.memory_allocated() - base, two)
    # the first shape's plan was evicted: its rebuild gives bitwise the same maps
    with torch.no_grad():
        again = det.forward_raw(xs[shapes[0]])
    for a, b in zip(first, again):
        assert torch.equal(a, b)


def _map_grads(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(sh, generator=g, dtype=torch.float64).float().cuda() for sh in shapes]


def _rel_l2(a, b, floor):
    return ((a.double() - b.double()).norm() / max(b.double().norm().item(), floor * b.numel() ** 0.5)).item()


@pytest.mark.parametrize("case", ["det_tiny_fv0", "det_tiny_fv4", "det_tiny_21k"])
def test_train_mode_matches_the_reference(case):
    """train mode at 96 x 160 (window-padded conv levels, 8 carriers: the cropped bias table) and 320 x 480 (non-square
    carrier grid), frozen_stages -1 and 2, and at the DETR training sizes of <case>_detr.pt, 480 x 544 and 544 x 800 (100
    and 160 carriers: the key-loop attention, one and two key tiles; pools of kernel 8 x 8 and 8 x 11 on the fallback
    tokenizer backward): the normed maps, every BatchNorm's running statistics after the step, and the parameter
    gradients of loss = sum_k <map_k, G_k> against the reference's fp64 train step"""
    from fastervit_b200.detection import build_fastervit
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    train = g["train"] | torch.load(GOLDEN / f"{case}_detr.pt", weights_only=False)["train"]
    assert len(train) == 5
    for (H, W, fs), ref in train.items():
        det = build_fastervit(g["name"], out_indices=(0, 1, 2, 3), drop_path_rate=0.0, frozen_stages=fs, **g["kwargs"])
        O.synth_fill_(det.state_dict(), g["seeds"]["w"])
        det = det.cuda().train()
        x = O.synth_input(2, [H, W], ref["x_seed"], torch.float32).cuda()
        outs = det(_Nested(x, torch.zeros(2, H, W, dtype=torch.bool, device="cuda")))
        maps = [outs[k].tensors for k in range(4)]
        gs = _map_grads([tuple(m.shape) for m in maps], ref["g_seed"])
        sum((m * gk).sum() for m, gk in zip(maps, gs)).backward()
        for k, m in enumerate(maps):
            want = ref["levels"][k]
            err = (_sample(m) - want["sample"].double()).abs().max().item() / want["amax"]
            assert err < TOL, (case, H, W, fs, "map", k, err)
        sd = det.state_dict()
        for key, want in ref["bn_after"].items():
            err = (_sample(sd[key]) - want["sample"].double()).abs().max().item() / max(want["amax"], 1e-6)
            assert err < TOL, (case, H, W, fs, key, err)
        named = dict(det.named_parameters())
        assert {n for n, p in named.items() if p.grad is not None} == set(ref["grads"]), (case, fs)
        # tolerances of tests/test_dense_train_gpu.py: rel-L2 <= 4e-2 (6e-2 for patch_embed.*) against a floor of 1e-3 of
        # the largest gradient element, median <= 4e-3 (DESIGN.md section 4)
        floor = 1e-3 * max(d["amax"] for d in ref["grads"].values())
        rel = {n: _rel_l2(_sample(named[n].grad), d["sample"], floor) for n, d in ref["grads"].items()}
        bad = sorted(((e, n) for n, e in rel.items() if e > (6e-2 if n.startswith("patch_embed.") else 4e-2)),
                     reverse=True)
        med = sorted(rel.values())[len(rel) // 2]
        assert not bad and med <= 4e-3, (case, H, W, fs, med, bad[:8])


def test_backward_after_its_plan_was_evicted():
    """a train forward keeps its plan alive until its backward: two other shapes evict it from the cache (bound 2) in
    between, and the gradients equal those of an uninterrupted step"""
    from fastervit_b200.detection import build_fastervit
    from oracle import fastervit_oracle as O

    def model():
        det = build_fastervit("faster_vit_0_224", out_indices=(1, 2, 3), drop_path_rate=0.0, dim=16, in_dim=16,
                              depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
        O.synth_fill_(det.state_dict(), 5)
        return det.cuda().train()
    x = O.synth_input(2, [96, 160], 3, torch.float32).cuda()

    def loss(det, inp):
        return sum((o * (k + 1.0)).square().mean() for k, o in enumerate(det.forward_raw(inp)))
    a = model()
    loss(a, x).backward()
    b = model()
    lb = loss(b, x)
    for hw in ((128, 192), (160, 224)):
        loss(b, O.synth_input(2, list(hw), 4, torch.float32).cuda())
    eng = b._get_engine()
    assert len(eng.plans) == 2 and all(k[0] != tuple(x.shape) for k in eng.plans)
    lb.backward()
    # (the same step up to the order of the split-K weight-gradient reductions)
    gmax = max(p.grad.abs().max().item() for p in a.parameters() if p.grad is not None)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        if pa.grad is not None:
            assert _rel_l2(pb.grad, pa.grad, 1e-3 * gmax) <= 2e-2, n


def test_eval_gradients_raise():
    from fastervit_b200 import lib as L
    from fastervit_b200.detection import build_fastervit
    det = build_fastervit("faster_vit_0_224", dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8]).cuda()
    x = torch.randn(1, 3, 96, 128, device="cuda")
    with pytest.raises(L.FvitError, match="no eval-mode gradients"):
        det.eval().forward_raw(x)             # grad enabled, parameters require grad
    with pytest.raises(L.FvitError, match="no eval-mode gradients"):
        det.eval()._get_engine().forward_levels(x.requires_grad_(), (1, 2), norms=(det.norm1, det.norm2)) \
            [0].sum().backward()
