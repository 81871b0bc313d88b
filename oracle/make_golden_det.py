"""Generate tests/golden/det_*.pt from the UNMODIFIED reference's detection backbone
(downstream/object_detection/dino/models/dino/fastervit.py of a checkout of NVlabs/FasterViT).

    FASTERVIT_REFERENCE=<path to the reference checkout> python oracle/make_golden_det.py [case ...]

The module is imported by path (the DINO package's __init__ pulls in its compiled deformable-attention op), behind the
timm stand-in and a util.misc.NestedTensor stand-in (oracle/ref_shim). Each case fills the reference module's own
state_dict with the oracle's deterministic synthetic weights (synth_fill_), runs its eval forward in fp64 at every shape
of SHAPES (batch 2) and stores samples of the normed level maps together with the carrier geometry the reference used
(pool kernel / stride, tokenizer output grid, carrier sequence length), and the train steps of TRAIN (maps, running
statistics after the step, parameter-gradient samples); those of TRAIN_DETR go to <case>_detr.pt. It also stores the
missing / unexpected keys of load_state_dict(classification state_dict, strict=False), and `det_schema.pt` holds the
state_dict schema (keys, shapes, dtypes) of the eight full-size build_fastervit names. The tests never need the
reference.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import time
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "ref_shim"))
_REF = os.environ.get("FASTERVIT_REFERENCE")
DET_PY = Path(_REF or "", "downstream", "object_detection", "dino", "models", "dino", "fastervit.py")
if not _REF or not DET_PY.is_file():
    raise SystemExit("make_golden_det.py: set FASTERVIT_REFERENCE to a checkout of NVlabs/FasterViT")
sys.path.insert(0, _REF)
warnings.filterwarnings("ignore")

from oracle import fastervit_oracle as O  # noqa: E402
from oracle.make_golden import summarize  # noqa: E402

SEED_W, SEED_X = 1234, 5
GOLDEN = ROOT / "tests" / "golden"
NAMES = ["faster_vit_0_224", "faster_vit_1_224", "faster_vit_2_224", "faster_vit_3_224", "faster_vit_4_224",
         "faster_vit_4_21k_224", "faster_vit_4_21k_384", "faster_vit_4_21k_512"]
# 224^2; 96 x 160 (carrier grid 2 x 4 < the 4 x 4 the bias table was built for: its top-left is cropped);
# 320 x 480 (non-square grid); 250 x 333 (odd sizes, padding in every level); 480 x 800 (160 carriers: key-loop kernel)
SHAPES = [(224, 224), (96, 160), (320, 480), (250, 333), (480, 800)]
CASES = {
    # fv0-like: no layer scale, no propagation
    "det_tiny_fv0": ("faster_vit_0_224", dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])),
    # fv4-like: layer scale (the entry's 1e-5, randomised by synth_fill_), propagation, head dim 24
    "det_tiny_fv4": ("faster_vit_4_224", dict(dim=24, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8],
                                              do_propagation=True)),
    # 21k-like: no carrier tokens anywhere, window 14 at level 2
    "det_tiny_21k": ("faster_vit_4_21k_224", dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])),
    # 64-wide heads at levels 2 and 3 (the fused QKV + attention kernel of the inference plan, as fv1 ... fv3 take)
    "det_tiny_hd64": ("faster_vit_2_224", dict(dim=32, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 2, 4])),
}
# train mode (batch 2, drop_path_rate 0): loss = sum_k <map_k, G_k> with G_k seeded normal; frozen_stages -1 and 2.
# The reference's _freeze_stages raises for frozen_stages >= 2 (it names a missing `self.network`): the generator
# freezes what it means to -- patch_embed and levels[:frozen_stages - 1] in eval mode without gradients -- itself.
TRAIN = [((96, 160), -1), ((320, 480), -1), ((96, 160), 2)]
# DETR training sizes with more than 64 carriers: 480 x 544 and 544 x 800 (100 and 160 carriers: the key-loop attention
# with one and two key tiles; tokenizer pools of kernel 8 x 8 and 8 x 11, stride 3). Their input seeds continue TRAIN's;
# they are stored in a file of their own, <case>_detr.pt, so that each golden file stays small.
TRAIN_DETR = [((480, 544), -1), ((544, 800), -1)]
SEED_G = 11


def map_grads(shapes, seed: int) -> list:
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]


def load_det():
    spec = importlib.util.spec_from_file_location("fastervit_det_reference", DET_PY)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def schema(sd: dict) -> list:
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def run_case(det, case: str) -> None:
    import fastervit  # the reference classification package
    from util.misc import NestedTensor
    name, kw = CASES[case]
    t0 = time.time()
    net = det.build_fastervit(name, out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **kw).double()
    sd = net.state_dict()
    O.synth_fill_(sd, SEED_W)
    out: dict = {"case": case, "name": name, "kwargs": kw, "seeds": {"w": SEED_W, "x": SEED_X},
                 "state_keys": schema(sd), "shapes": {}}
    # classification checkpoint -> detection module (dino/models/dino/backbone.py: load_state_dict(strict=False))
    cls = fastervit.create_model(name, **{k: v for k, v in kw.items() if k != "do_propagation"})  # (fixed by the entry)
    res = det.build_fastervit(name, out_indices=(0, 1, 2, 3), **kw).load_state_dict(cls.state_dict(), strict=False)
    out["load_cls"] = {"missing": sorted(res.missing_keys), "unexpected": sorted(res.unexpected_keys)}
    net.eval()
    tok = net.levels[2].global_tokenizer if net.levels[2].do_gt else None
    blk = net.levels[2].blocks[0]
    avg_pool = torch.nn.functional.avg_pool2d
    for si, (H, W) in enumerate(SHAPES):
        geo: dict = {}
        hooks = []
        if tok is not None:
            hooks.append(tok.register_forward_hook(
                lambda m, i, o: geo.update(level_in=tuple(i[0].shape), tokens=tuple(o[0].shape), hg=o[1], wg=o[2])))
            hooks.append(blk.hat_attn.register_forward_hook(lambda m, i, o: geo.update(s_ct=i[0].shape[1])))

        def pool(x, kernel_size, stride, **k):
            geo["pool"] = (tuple(kernel_size), tuple(stride))
            return avg_pool(x, kernel_size, stride, **k)
        torch.nn.functional.avg_pool2d = pool
        try:
            x = O.synth_input(2, [H, W], SEED_X + si, torch.float64)
            mask = torch.zeros(2, H, W, dtype=torch.bool)
            mask[1, :, W - W // 4:] = True
            with torch.no_grad():
                outs = net(NestedTensor(x, mask))
        finally:
            torch.nn.functional.avg_pool2d = avg_pool
            for h in hooks:
                h.remove()
        out["shapes"][(H, W)] = {"x_seed": SEED_X + si, "geometry": geo,
                                 "levels": {i: summarize(o.tensors) for i, o in outs.items()},
                                 "masks": {i: o.mask.clone() for i, o in outs.items()}}
        print(f"  {case} {H}x{W}: {geo}", flush=True)
    out["train"] = {}
    detr = {k: out[k] for k in ("case", "name", "kwargs", "seeds")} | {"train": {}}
    if case != "det_tiny_hd64":
        for ti, ((H, W), fs) in enumerate(TRAIN + TRAIN_DETR):
            dst = out if ti < len(TRAIN) else detr
            dst["train"][(H, W, fs)] = run_train(det, name, kw, H, W, fs, SEED_X + 50 + ti)
    GOLDEN.mkdir(parents=True, exist_ok=True)
    for res, path in ((out, GOLDEN / f"{case}.pt"), (detr, GOLDEN / f"{case}_detr.pt")):
        if res["train"] or res is out:
            torch.save(res, path, _use_new_zipfile_serialization=False)
            print(f"{case}: {path.name} {path.stat().st_size / 1024:.0f} KiB, {time.time() - t0:.1f}s", flush=True)


def run_train(det, name: str, kw: dict, H: int, W: int, fs: int, x_seed: int) -> dict:
    from util.misc import NestedTensor
    net = det.build_fastervit(name, out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **kw).double()
    O.synth_fill_(net.state_dict(), SEED_W)
    net.train()
    frozen = [net.patch_embed] + [net.levels[i] for i in range(fs - 1)] if fs >= 0 else []
    for m in frozen:
        m.eval()
        for p in m.parameters():
            p.requires_grad = False
    x = O.synth_input(2, [H, W], x_seed, torch.float64)
    outs = net(NestedTensor(x, torch.zeros(2, H, W, dtype=torch.bool)))
    maps = [outs[k].tensors for k in range(4)]
    gs = map_grads([tuple(m.shape) for m in maps], SEED_G)
    loss = sum((m * gk).sum() for m, gk in zip(maps, gs))
    loss.backward()
    sd = net.state_dict()
    res = {"x_seed": x_seed, "g_seed": SEED_G, "loss": loss.item(),
           "levels": {k: summarize(m) for k, m in enumerate(maps)},
           "bn_after": {k: summarize(v) for k, v in sd.items() if k.endswith(("running_mean", "running_var"))},
           "grads": {k: summarize(p.grad) for k, p in net.named_parameters() if p.grad is not None}}
    print(f"  train {H}x{W} frozen_stages {fs}: loss {loss.item():.6f}, {len(res['grads'])} gradients", flush=True)
    return res


def run_schema(det) -> None:
    out = {}
    for name in NAMES:
        out[name] = schema(det.build_fastervit(name, out_indices=(1, 2, 3)).state_dict())
    path = GOLDEN / "det_schema.pt"
    torch.save(out, path, _use_new_zipfile_serialization=False)
    print(f"schema: {path.name} {path.stat().st_size / 1024:.0f} KiB", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(8)
    det = load_det()
    cases = sys.argv[1:] or list(CASES) + ["schema"]
    for c in cases:
        run_schema(det) if c == "schema" else run_case(det, c)
