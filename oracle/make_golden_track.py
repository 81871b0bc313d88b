"""Generate tests/golden/track_*.pt from the UNMODIFIED reference's tracking backbone
(downstream/object_tracking/motrv2/models/fastervit.py of a checkout of NVlabs/FasterViT).

    FASTERVIT_REFERENCE=<path to the reference checkout> python oracle/make_golden_track.py [case ...]

The module is imported by path behind the timm / util.misc stand-ins (oracle/ref_shim), and built with its own
FrozenBatchNorm2d and the stand-in's LayerNorm2d. Each case is a reduced config (the det goldens' widths) run with the
norm pairs (stem, output) of NORMS, (Frozen, LN) being MOTRv2's published recipe. Per pair it stores:
  * eval: the normed level maps (samples) and masks at every shape of SHAPES (batch 2, fp64);
  * train: steps of loss = sum_k <map_k, G_k> (G_k seeded normal, drop_path_rate 0) at TRAIN, with the maps, every
    running statistic after the step (the frozen BatchNorms' must come back unchanged) and parameter-gradient samples.
    The reference's _freeze_stages raises for frozen_stages >= 2 (it names a missing `self.network`): the generator
    freezes patch_embed and levels[:frozen_stages - 1] itself, as make_golden_det.py does;
  * load_cls: the missing / unexpected keys of the reference's `_load_state_dict` given a classification checkpoint
    with a `module.` prefix, and the value the level-3 LayerNorm weight received.
The eval results, load_cls and the state_dict keys go to <case>.pt; the train steps go to one file per train shape,
<case>_train_<H>x<W>.pt, so that each golden file stays small. For (Frozen, LN) on the fv0-like case, one train step at the recipe's full 800 x 1536, batch 1 (several hundred level-2
carriers: the key-loop attention kernels), with the image gradient, goes to track_tiny_fv0_full.pt. track_schema.pt holds
the state_dict schema of the nine full-size names under (Frozen, LN) and (BN, BN). The tests never need the reference.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile
import time
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "ref_shim"))
_REF = os.environ.get("FASTERVIT_REFERENCE")
TRACK_PY = Path(_REF or "", "downstream", "object_tracking", "motrv2", "models", "fastervit.py")
if not _REF or not TRACK_PY.is_file():
    raise SystemExit("make_golden_track.py: set FASTERVIT_REFERENCE to a checkout of NVlabs/FasterViT")
sys.path.insert(0, _REF)
warnings.filterwarnings("ignore")

from oracle import fastervit_oracle as O  # noqa: E402
from oracle.make_golden import summarize  # noqa: E402

SEED_W, SEED_X, SEED_G = 1234, 5, 11
GOLDEN = ROOT / "tests" / "golden"
NAMES = ["faster_vit_0_224", "faster_vit_0_224_hat_False", "faster_vit_1_224", "faster_vit_2_224", "faster_vit_3_224",
         "faster_vit_4_224", "faster_vit_4_21k_224", "faster_vit_4_21k_384", "faster_vit_4_21k_512"]
# 224^2; 96 x 160 (cropped carrier bias table); 250 x 333 (odd sizes); 200 x 384 (the recipe's 800 x 1536 at a quarter)
SHAPES = [(224, 224), (96, 160), (250, 333), (200, 384)]
TRAIN = [((96, 160), -1), ((96, 160), 0), ((96, 160), 2), ((320, 480), -1), ((320, 480), 0), ((320, 480), 2)]
FULL = (800, 1536)
NORMS = ["frozen_ln", "bn_ln", "frozen_frozen", "bn_bn"]
TINY = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
CASES = {
    "track_tiny_fv0": ("faster_vit_0_224", TINY),                                          # carriers at level 2
    "track_tiny_fv4": ("faster_vit_4_224", dict(TINY, dim=24, do_propagation=True)),       # layer scale, propagation
    "track_tiny_21k": ("faster_vit_4_21k_224", TINY),                                      # no carriers, window 14
    "track_tiny_hatf": ("faster_vit_0_224_hat_False", TINY),
}
GRAD_SAMPLE = 32   # values per gradient sample: the files hold 97 train steps, so each is packed small


def load_track():
    spec = importlib.util.spec_from_file_location("fastervit_track_reference", TRACK_PY)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def norm_classes(ref, pair: str):
    from timm.models.layers import LayerNorm2d
    stem, out = pair.split("_")
    cls = {"bn": torch.nn.BatchNorm2d, "frozen": ref.FrozenBatchNorm2d, "ln": LayerNorm2d}
    return cls[stem], cls[out]


def schema(sd: dict) -> list:
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def pack_grads(named: dict) -> dict:
    """gradient samples of one step packed into one tensor: summarize's strided sample, thinned to <= GRAD_SAMPLE values
    (`step`: the extra stride), concatenated in `names` order"""
    names, amax, steps, lens, parts = [], [], [], [], []
    for k, t in named.items():
        s = summarize(t)
        step = max(1, (s["sample"].numel() + GRAD_SAMPLE - 1) // GRAD_SAMPLE)
        part = s["sample"][::step]
        names.append(k)
        amax.append(s["amax"])
        steps.append(step)
        lens.append(part.numel())
        parts.append(part)
    return {"names": names, "amax": amax, "step": steps, "len": lens, "samples": torch.cat(parts)}


def build(ref, name, kw, pair, **extra):
    stem, out = norm_classes(ref, pair)
    net = ref.build_fastervit(name, stem, out, out_indices=(0, 1, 2, 3), drop_path_rate=0.0, **kw, **extra).double()
    O.synth_fill_(net.state_dict(), SEED_W)
    return net


def levels_of(outs) -> list:
    return [outs[k].tensors for k in range(len(outs))]


def run_case(ref, case: str) -> None:
    from util.misc import NestedTensor
    name, kw = CASES[case]
    t0 = time.time()
    out: dict = {"case": case, "name": name, "kwargs": kw, "seeds": {"w": SEED_W, "x": SEED_X}, "pairs": {},
                 "masks": {}}
    train: dict = {}   # (H, W) -> pair -> (H, W, frozen_stages) -> step
    for pair in NORMS:
        net = build(ref, name, kw, pair)
        res: dict = {"state_keys": schema(net.state_dict()), "shapes": {}}
        net.eval()
        for si, (H, W) in enumerate(SHAPES):
            x = O.synth_input(2, [H, W], SEED_X + si, torch.float64)
            mask = torch.zeros(2, H, W, dtype=torch.bool)
            mask[1, :, W - W // 4:] = True
            with torch.no_grad():
                outs = net(NestedTensor(x, mask))
            res["shapes"][(H, W)] = {"x_seed": SEED_X + si, "levels": {i: summarize(o.tensors) for i, o in outs.items()}}
            out["masks"][(H, W)] = {i: o.mask.clone() for i, o in outs.items()}   # (the same for every pair)
        for ti, ((H, W), fs) in enumerate(TRAIN):
            train.setdefault((H, W), {}).setdefault(pair, {})[(H, W, fs)] = run_train(
                ref, name, kw, pair, H, W, fs, SEED_X + 50 + ti, batch=2)
        if pair == "frozen_ln":
            res["load_cls"] = load_cls(ref, name, kw, pair)
        out["pairs"][pair] = res
        print(f"  {case} {pair}: {time.time() - t0:.1f}s", flush=True)
    save(out, GOLDEN / f"{case}.pt")
    for (H, W), pairs in train.items():
        save({k: out[k] for k in ("case", "name", "kwargs", "seeds")} | {"pairs": pairs},
             GOLDEN / f"{case}_train_{H}x{W}.pt")
    if case == "track_tiny_fv0":
        full = {k: out[k] for k in ("case", "name", "kwargs", "seeds")}
        full["train"] = {(*FULL, -1): run_train(ref, name, kw, "frozen_ln", *FULL, -1, SEED_X + 90, batch=1,
                                                  want_dx=True)}
        save(full, GOLDEN / f"{case}_full.pt")


def save(obj, path: Path) -> None:
    GOLDEN.mkdir(parents=True, exist_ok=True)
    torch.save(obj, path, _use_new_zipfile_serialization=False)
    print(f"{path.name}: {path.stat().st_size / 1024:.0f} KiB", flush=True)


def run_train(ref, name, kw, pair, H, W, fs, x_seed, batch, want_dx=False) -> dict:
    from util.misc import NestedTensor
    net = build(ref, name, kw, pair)
    net.train()
    frozen = [net.patch_embed] + [net.levels[i] for i in range(fs - 1)] if fs >= 0 else []
    for m in frozen:
        m.eval()
        for p in m.parameters():
            p.requires_grad = False
    x = O.synth_input(batch, [H, W], x_seed, torch.float64).requires_grad_(want_dx)
    outs = net(NestedTensor(x, torch.zeros(batch, H, W, dtype=torch.bool)))
    maps = levels_of(outs)
    g = torch.Generator().manual_seed(SEED_G)
    gs = [torch.randn(tuple(m.shape), generator=g, dtype=torch.float64) for m in maps]
    loss = sum((m * gk).sum() for m, gk in zip(maps, gs))
    loss.backward()
    sd = net.state_dict()
    res = {"x_seed": x_seed, "g_seed": SEED_G, "batch": batch, "loss": loss.item(),
           "levels": {k: summarize(m) for k, m in enumerate(maps)},
           "stats_after": {k: summarize(v) for k, v in sd.items() if k.endswith(("running_mean", "running_var"))},
           "grads": pack_grads({k: p.grad for k, p in net.named_parameters() if p.grad is not None})}
    if want_dx:
        res["x_grad"] = summarize(x.grad)
    print(f"  train {pair} {H}x{W} frozen_stages {fs}: loss {loss.item():.6f}, {len(res['grads']['names'])} gradients",
          flush=True)
    return res


def load_cls(ref, name, kw, pair) -> dict:
    """the reference's _load_state_dict (through _load_checkpoint) of a classification checkpoint saved by DDP
    (`module.` prefix): the missing / unexpected keys it prints and the level-3 LayerNorm weight it received"""
    import contextlib
    import io
    import fastervit  # the reference classification package
    cls = fastervit.create_model(name if name != "faster_vit_0_224_hat_False" else "faster_vit_0_224",
                                 **{k: v for k, v in kw.items() if k != "do_propagation"})
    O.synth_fill_(cls.state_dict(), SEED_W + 1)
    net = build(ref, name, kw, pair)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp, "cls.pth")
        torch.save({"model": {"module." + k: v for k, v in cls.state_dict().items()}}, path)
        msg = io.StringIO()
        with contextlib.redirect_stdout(msg):
            net._load_state_dict(str(path))
    keys = {"missing": [], "unexpected": []}
    for line in msg.getvalue().splitlines():   # (fastervit.py:95-100: one line per list)
        for tag, prefix in (("unexpected", "unexpected key in source state_dict: "),
                            ("missing", "missing keys in source state_dict: ")):
            if line.startswith(prefix):
                keys[tag] = sorted(line[len(prefix):].split(", "))
    return {**keys, "norm_weight": net.norm.weight.detach().float().clone()}


def run_schema(ref) -> None:
    out = {}
    for pair in ("frozen_ln", "bn_bn"):
        stem, o = norm_classes(ref, pair)
        for name in NAMES:
            torch.manual_seed(0)
            out[(name, pair)] = schema(ref.build_fastervit(name, stem, o).state_dict())
    save(out, GOLDEN / "track_schema.pt")


if __name__ == "__main__":
    torch.set_num_threads(8)
    ref = load_track()
    cases = sys.argv[1:] or list(CASES) + ["schema"]
    for c in cases:
        run_schema(ref) if c == "schema" else run_case(ref, c)
