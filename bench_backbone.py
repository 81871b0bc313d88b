"""Dense-prediction training measurement: the backbone train step (differentiable forward_levels / FasterViTBackbone)
against the classification train step, and the fvit_feature_map_bwd kernels on their own.

    python bench_backbone.py [--steps 10] [--warmup 3] [--rounds 3] [--kernel-iters 50] [--out DIR]

Prints the card name and power limit, then one line per measurement and a final JSON line. Every step is timed with
CUDA events around `steps` train steps (forward + torch.autograd.backward from fixed, pre-made output gradients, so no
loss code is timed), after `warmup` steps of every arm; the arms of one comparison alternate `rounds` times and the
median of the rounds is reported. Nothing is written unless --out is given.

Workloads:
  * faster_vit_4_224, batch 128: forward_levels(x, (0, 1, 2, 3)) train step vs the classification train step;
  * faster_vit_0_any_res at 576 x 960 (window_size [7, 7, 12, 6], ct_size 2, dim 64), batch 8: FasterViTBackbone with
    out_indices (1, 2, 3) (the DINO 4-scale taps), frozen_stages -1 vs 1;
  * kernel time and achieved bytes/s of fvit_feature_map_bwd_stats / fvit_feature_map_bwd (BatchNorm mode) at the four
    fv4 batch-128 level shapes; the bytes are the algorithm's HBM traffic computed from the shapes below.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def card() -> dict:
    info = dict(name=torch.cuda.get_device_name(0), power_limit_w=None, sm_max_mhz=None)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception:   # noqa: BLE001 - the query is informational
        pass
    return info


def timed(fn, steps: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def compare(arms: dict, steps: int, warmup: int, rounds: int) -> dict:
    """ms per step of every arm: all arms warmed up, then `rounds` alternating timed windows, median of the rounds"""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    res = {k: [] for k in arms}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for k in order:
            res[k].append(timed(arms[k], steps))
    return {k: dict(ms=statistics.median(v), rounds=v) for k, v in res.items()}


def fv4_workload(args) -> dict:
    import fastervit_b200 as F
    B = 128
    torch.manual_seed(0)
    model = F.create_model("faster_vit_4_224").cuda().train()
    x = torch.randn(B, 3, 224, 224, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    dlogits = torch.randn(B, model.num_classes, device="cuda", generator=g) / B
    with torch.no_grad():
        shapes = [tuple(f.shape) for f in model.eval().forward_levels(x[:1], (0, 1, 2, 3))]
    model.train()
    dmaps = [torch.randn((B,) + s[1:], device="cuda", generator=g) * 1e-4 for s in shapes]

    def cls_step():
        torch.autograd.backward(model(x), dlogits)
        model.zero_grad(set_to_none=True)

    def levels_step():
        torch.autograd.backward(model.forward_levels(x, (0, 1, 2, 3)), dmaps)
        model.zero_grad(set_to_none=True)

    res = compare({"classification": cls_step, "backbone_levels_0123": levels_step}, args.steps, args.warmup, args.rounds)
    res["ratio_backbone_over_classification"] = res["backbone_levels_0123"]["ms"] / res["classification"]["ms"]
    res["batch"] = B
    res["level_maps_mb"] = sum(B * s[1] * s[2] * s[3] * 4 for s in shapes) / 1e6
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 1e9
    del model
    torch.cuda.empty_cache()
    return res


def any_res_workload(args) -> dict:
    from fastervit_b200.backbone import FasterViTBackbone
    B, H, W = 8, 576, 960
    kw = dict(resolution=[H, W], window_size=[7, 7, 12, 6], ct_size=2, dim=64)
    torch.manual_seed(0)
    bbs = {fs: FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=fs, **kw).cuda().train()
           for fs in (-1, 1)}
    x = torch.randn(B, 3, H, W, device="cuda")
    with torch.no_grad():
        shapes = [tuple(o.shape) for o in bbs[-1].eval().forward_raw(x[:1])]
    bbs[-1].train()
    g = torch.Generator(device="cuda").manual_seed(2)
    douts = [torch.randn((B,) + s[1:], device="cuda", generator=g) * 1e-3 for s in shapes]

    def step(bb):
        def fn():
            torch.autograd.backward(bb.forward_raw(x), douts)
            bb.zero_grad(set_to_none=True)
        return fn

    res = compare({f"frozen_stages_{fs}": step(bb) for fs, bb in bbs.items()}, args.steps, args.warmup, args.rounds)
    res["batch"], res["hw"] = B, [H, W]
    del bbs
    torch.cuda.empty_cache()
    return res


def kernel_workload(args) -> dict:
    """fvit_feature_map_bwd_stats / fvit_feature_map_bwd (BatchNorm mode) at the fv4 batch-128 level shapes. Bytes:
    stats reads dy and the level rows (+ the row map); apply reads dy, the rows, the row map and reads + writes g."""
    from fastervit_b200 import lib as L
    B = 128
    out = {}
    for i, (C, H) in enumerate(((196, 56), (392, 28), (784, 14), (1568, 7))):
        T = H * H     # (square 224 x 224 input: level maps 56^2 .. 7^2)
        n = B * T
        xs = torch.randn(n, C, device="cuda")
        g = torch.zeros(n, C, device="cuda")
        rows = torch.arange(n, dtype=torch.int32, device="cuda")
        dy = torch.randn(B, C, T, device="cuda")
        mean, rstd = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        w = torch.ones(C, device="cuda")
        acc = torch.zeros(1 + 2 * C, device="cuda")
        gs = torch.tensor([1.0, 1.0], device="cuda")

        def stats():
            L.call("fvit_feature_map_bwd_stats", dy.data_ptr(), xs.data_ptr(), C, rows.data_ptr(), B, T, C, mean.data_ptr(),
                   rstd.data_ptr(), acc.data_ptr() + 4, acc.data_ptr() + 4 * (1 + C), acc.data_ptr())

        def apply():
            L.call("fvit_feature_map_bwd", dy.data_ptr(), xs.data_ptr(), C, rows.data_ptr(), B, T, C, mean.data_ptr(),
                   rstd.data_ptr(), w.data_ptr(), acc.data_ptr() + 4, acc.data_ptr() + 4 * (1 + C), gs.data_ptr(), None,
                   g.data_ptr(), C, None, None)

        for fn in (stats, apply):
            fn()
        ms_s = timed(stats, args.kernel_iters)
        ms_a = timed(apply, args.kernel_iters)
        by_s = 4.0 * (2 * n * C + n)
        by_a = 4.0 * (4 * n * C + n)
        out[f"level{i}"] = dict(C=C, T=T, stats_ms=ms_s, stats_gbps=by_s / ms_s / 1e6, apply_ms=ms_a,
                                apply_gbps=by_a / ms_a / 1e6, map_mb=4.0 * n * C / 1e6)
        del xs, g, rows, dy
        torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the JSON result (nothing is written without it)")
    ap.add_argument("--only", default="fv4,anyres,kernels")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_backbone.py needs a CUDA device (an H100); nothing to measure on the CPU")
    torch.cuda.set_device(0)
    res = dict(card=card())
    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit_w']} W, max SM clock "
          f"{res['card']['sm_max_mhz']} MHz")
    parts = args.only.split(",")
    if "kernels" in parts:
        res["feature_map_bwd"] = kernel_workload(args)
        for k, v in res["feature_map_bwd"].items():
            print(f"fvit_feature_map_bwd {k} C={v['C']} T={v['T']} ({v['map_mb']:.0f} MB map): stats {v['stats_ms']:.3f} ms "
                  f"({v['stats_gbps']:.0f} GB/s), apply {v['apply_ms']:.3f} ms ({v['apply_gbps']:.0f} GB/s)")
    if "fv4" in parts:
        r = res["fv4_b128"] = fv4_workload(args)
        print(f"fv4 b128 train step: classification {r['classification']['ms']:.1f} ms, backbone levels (0,1,2,3) "
              f"{r['backbone_levels_0123']['ms']:.1f} ms, ratio {r['ratio_backbone_over_classification']:.3f} "
              f"(peak memory {r['peak_mem_gb']:.1f} GB)")
    if "anyres" in parts:
        r = res["fv0_any_res_576x960_b8"] = any_res_workload(args)
        print(f"fv0 any-res 576x960 b8 backbone (1,2,3) train step: frozen_stages -1 {r['frozen_stages_-1']['ms']:.2f} ms, "
              f"frozen_stages 1 {r['frozen_stages_1']['ms']:.2f} ms")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        Path(args.out, "bench_backbone.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
