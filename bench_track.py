"""Tracking-backbone benchmark: MOTRv2's published recipe, faster_vit_4_21k_224 with a frozen-BatchNorm stem and
LayerNorm2d level norms (fastervit_b200.tracking), batch 1 at 800 x 1536.

    python bench_track.py [--rounds 3] [--reps 10]

It reports, alternating the arms within each round and taking the median over --rounds rounds:
  * train step (train mode: forward + backward of sum_k <map_k, G_k> with fixed pre-made G_k; no optimizer) of the
    recipe (Frozen, LN) against the same model with (BatchNorm2d, BatchNorm2d), CUDA events, median of --reps steps;
  * the no_grad eval forward of the recipe;
  * fvit_feature_map_ln_fwd / _bwd at each level of that shape (the level rows and row maps of the train plan), CUDA
    events over --launches launches, with the algorithmic bytes (forward: x read once, map written once; backward: dy
    and x read once, g read and written, the per-pixel mean / rstd) and the rate they give;
and the card name and power limit, read in the same process. Prints one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess

import torch
import torch.nn as nn

H, W = 800, 1536


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if q.returncode == 0 else ("?", "?")
    return dict(gpu=name, power_limit=power)


class _Nested:
    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask


def _layernorm2d():
    class LayerNorm2d(nn.LayerNorm):   # timm's LayerNorm2d: the module classifies it by what it is
        def __init__(self, n, eps=1e-6):
            super().__init__(n, eps=eps)
    return LayerNorm2d


def model(pair: str):
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    torch.manual_seed(0)
    stem, out = {"frozen_ln": (FrozenBatchNorm2d, _layernorm2d()), "bn_bn": (nn.BatchNorm2d, nn.BatchNorm2d)}[pair]
    return build_fastervit("faster_vit_4_21k_224", stem, out).cuda()


def timed(fn, reps: int) -> float:
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * reps)]
    for i in range(reps):
        ev[2 * i].record()
        fn()
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    return statistics.median(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(reps))


def kernels(m, x, launches: int) -> list:
    """the LN output kernels on the train plan's level rows"""
    from fastervit_b200 import lib as L
    eng = m._get_engine()
    plan = next(p for k, p in eng.plans.items() if k[1])   # (the train plan of this shape)
    res = []
    for d in plan.dense:
        B, T, C = plan.B, d["T"], d["C"]
        ln = d["norm"]
        out = torch.empty(B, C, T, device="cuda")
        gs = torch.tensor([1.0, 1.0], device="cuda")
        g = d["lv"]["g"]
        dw, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        fwd = lambda: L.call("fvit_feature_map_ln_fwd", d["x"].data_ptr(), C, d["rows"].data_ptr(), B, T, C,  # noqa: E731
                             ln.weight.data_ptr(), ln.bias.data_ptr(), float(ln.eps), out.data_ptr(),
                             d["pmean"].data_ptr(), d["prstd"].data_ptr())
        bwd = lambda: L.call("fvit_feature_map_ln_bwd", d["dy"].data_ptr(), d["x"].data_ptr(), C,  # noqa: E731
                             d["rows"].data_ptr(), B, T, C, d["pmean"].data_ptr(), d["prstd"].data_ptr(),
                             ln.weight.data_ptr(), gs.data_ptr(), None, g.data_ptr(), C, dw.data_ptr(), db.data_ptr())
        row = dict(level=d["level"], C=C, pixels=B * T)
        for name, fn, nbytes in (("fwd", fwd, 4 * (2 * B * T * C + 2 * B * T)),
                                 ("bwd", bwd, 4 * (4 * B * T * C + 2 * B * T + 2 * C))):
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / launches
            row[name] = dict(us=round(us, 2), bytes=nbytes, tb_s=round(nbytes / us / 1e6, 3))
        res.append(row)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = False
    models = {p: model(p) for p in ("frozen_ln", "bn_bn")}
    x = torch.randn(1, 3, H, W, device="cuda")
    nt = _Nested(x, torch.zeros(1, H, W, dtype=torch.bool, device="cuda"))
    grads = None

    def step(m):
        nonlocal grads
        outs = m(nt)
        maps = [outs[k].tensors for k in sorted(outs)]
        if grads is None:
            gen = torch.Generator(device="cuda").manual_seed(0)
            grads = [torch.randn(t.shape, device="cuda", generator=gen) for t in maps]
        torch.autograd.backward(maps, grads)

    def fwd_eval(m):
        with torch.no_grad():
            m(nt)

    for m in models.values():   # warm-up: plans built, weights packed, graphs captured
        m.train()
        for _ in range(3):
            step(m)
        m.zero_grad(set_to_none=True)
    models["frozen_ln"].eval()
    for _ in range(3):
        fwd_eval(models["frozen_ln"])
    rounds = {"train_frozen_ln": [], "train_bn_bn": [], "eval_frozen_ln": []}
    for _ in range(a.rounds):
        for pair, m in models.items():
            m.train()
            rounds[f"train_{pair}"].append(timed(lambda: step(m), a.reps))
        models["frozen_ln"].eval()
        rounds["eval_frozen_ln"].append(timed(lambda: fwd_eval(models["frozen_ln"]), a.reps))
    models["frozen_ln"].train()
    step(models["frozen_ln"])
    res = dict(card(), shape=[1, 3, H, W], model="faster_vit_4_21k_224",
               ms={k: round(statistics.median(v), 3) for k, v in rounds.items()},
               rounds_ms={k: [round(t, 3) for t in v] for k, v in rounds.items()},
               peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
               ln_kernels=kernels(models["frozen_ln"], x, a.launches))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
