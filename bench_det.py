"""Detection-backbone benchmark: the DINO FasterViT backbone (fastervit_b200.detection) on the input sizes of DETR's
multi-scale training augmentation, batch 2, out_indices (1, 2, 3), for faster_vit_0_224 and faster_vit_4_224.

    python bench_det.py [--shapes 20] [--reps 10] [--names faster_vit_0_224,faster_vit_4_224]

The shapes are drawn with a fixed seed: short side from 480..800 in steps of 32, long side at an aspect ratio of
1..1.8 capped at 1333 (the range DETR's RandomResize produces; a padded batch takes its largest image's size). Per
name it reports, under the default bound of 2 cached plans:
  * cold call: host time of building the shape's plan (launch list, row maps, buffers: Plan.__init__) and the rest of
    that first call's wall time, ending in a device synchronise (weight packing, the eager first run and its host
    launch overhead), each shape once; for the eval forward and for the train step;
  * warm eval forward (no_grad) and warm train step (train mode: forward_raw + backward of sum_k <map_k, G_k> with
    fixed G_k; no optimizer), CUDA events, median over --reps calls per shape, then the median over the shapes;
  * peak allocated device memory over the sweep;
and the card name and power limit, read in the same process. Prints one JSON line per name; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import time

import torch


def detr_shapes(n: int, seed: int = 0) -> list[tuple[int, int]]:
    g = torch.Generator().manual_seed(seed)
    out = []
    while len(out) < n:
        s = 480 + 32 * int(torch.randint(0, 11, (1,), generator=g))
        long = min(int(s * (1.0 + 0.8 * float(torch.rand(1, generator=g)))), 1333)
        hw = (s, long) if float(torch.rand(1, generator=g)) < 0.5 else (long, s)
        if hw not in out:
            out.append(hw)
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if q.returncode == 0 else ("?", "?")
    return dict(gpu=name, power_limit=power)


def bench(name: str, shapes: list, reps: int) -> dict:
    from fastervit_b200.detection import build_fastervit
    from fastervit_b200.engine import Plan
    torch.manual_seed(0)
    det = build_fastervit(name, out_indices=(1, 2, 3)).cuda().eval()
    det.requires_grad_(False)   # (the eval sweep: inference)
    # host plan-build time: Plan.__init__ is all host work (row maps, buffers, the launch list)
    build_ms = []
    orig = Plan.__init__

    def timed_init(self, *a, **k):
        t0 = time.perf_counter()
        orig(self, *a, **k)
        build_ms.append((time.perf_counter() - t0) * 1e3)
    Plan.__init__ = timed_init
    torch.cuda.reset_peak_memory_stats()

    def sweep(step) -> tuple[list, list, list]:
        build_ms.clear()
        cold, warm = [], []
        for hw in shapes:
            x = torch.randn(2, 3, *hw, device="cuda")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(x)
            torch.cuda.synchronize()
            cold.append((time.perf_counter() - t0) * 1e3)
            ts = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step(x)
                b.record()
                b.synchronize()
                ts.append(a.elapsed_time(b))
            warm.append(statistics.median(ts))
        return cold, warm, list(build_ms)

    def eval_step(x):
        with torch.no_grad():
            det.forward_raw(x)

    def train_step(x):
        outs = det.forward_raw(x)
        sum((o * (0.01 * (k + 1))).sum() for k, o in enumerate(outs)).backward()

    try:
        det.eval()
        cold_e, warm_e, build_e = sweep(eval_step)
        det.train().requires_grad_(True)
        cold_t, warm_t, build_t = sweep(train_step)
    finally:
        Plan.__init__ = orig

    def med(v):
        return round(statistics.median(v), 2)
    return dict(name=name, batch=2, shapes=len(shapes), plan_cache_size=det.plan_cache_size,
                warm_eval_ms_median=med(warm_e), warm_train_step_ms_median=med(warm_t),
                warm_eval_ms_per_shape={f"{h}x{w}": round(t, 2) for (h, w), t in zip(shapes, warm_e)},
                cold_eval_plan_build_host_ms_median=med(build_e),
                cold_eval_first_call_minus_plan_build_ms_median=med([c - b for c, b in zip(cold_e, build_e)]),
                cold_train_plan_build_host_ms_median=med(build_t),
                cold_train_first_call_minus_plan_build_ms_median=med([c - b for c, b in zip(cold_t, build_t)]),
                peak_allocated_mib=round(torch.cuda.max_memory_allocated() / 2 ** 20, 1), **card())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--names", default="faster_vit_0_224,faster_vit_4_224")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det.py needs a CUDA device")
    shapes = detr_shapes(a.shapes)
    for name in a.names.split(","):
        print(json.dumps(bench(name, shapes, a.reps)), flush=True)


if __name__ == "__main__":
    main()
