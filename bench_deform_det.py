"""Multi-scale deformable attention backward: the default (float atomics) against the deterministic one (int64 fixed
point, what MSDeformAttnFunction runs under torch.use_deterministic_algorithms).

    python bench_deform_det.py [--rounds 7] [--iters 20] [--out DIR]

At bench_deform.py's workloads it times, with CUDA events (warm-up first, `iters` calls per timing, the two arms
alternating within each round, median of `rounds`):
  * atomic: zeroing grad_value and fvit_msda_bwd, as the Function runs it with the flag off;
  * deterministic: fvit_msda_bwd_deterministic (zeroing its scratch and bound workspace, the bound pass, the fixed-point
    accumulation, the conversion to fp32).
It reports the slowdown (deterministic / atomic), the scratch bytes and the per-kernel device time of the
deterministic arm (torch.profiler, in a separate pass after the timing). Before timing it checks that two deterministic
calls agree bitwise and reports how far the two arms' gradients are apart. The card name and power limit are read in
the same run. One JSON line per workload, and a summary table, go to stdout (and DIR if given).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from bench_deform import D, M, P, WORKLOADS, card  # noqa: E402
from fastervit_b200 import deform, lib  # noqa: E402


def time_alternating(arms: dict, iters: int, rounds: int) -> dict:
    """Median over rounds of the mean time (ms) of `iters` back-to-back calls of each arm; arms alternate per round."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for k in order:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                arms[k]()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) / iters)
    return {k: statistics.median(v) for k, v in res.items()}


def kernel_us(fn, iters: int) -> dict:
    """Mean device time per call (µs) of each kernel / memset that fn launches, from torch.profiler."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.replace("void ", "").replace("fvit::(anonymous namespace)::", "").split("(")[0]
            tot[name] += e.device_time_total
    return {k: round(v / iters, 1) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def bench(name: str, N: int, levels, Lq, iters: int, rounds: int) -> dict:
    L, S = len(levels), sum(h * w for h, w in levels)
    Lq = S if Lq is None else Lq
    g = torch.Generator(device="cuda").manual_seed(0)
    value = torch.randn(N, S, M, D, device="cuda", generator=g)
    loc = torch.rand(N, Lq, M, L, P, 2, device="cuda", generator=g) * 1.2 - 0.1
    w = torch.softmax(torch.randn(N, Lq, M, L * P, device="cuda", generator=g), -1).view(N, Lq, M, L, P)
    go = torch.randn(N, Lq, M * D, device="cuda", generator=g)
    shapes = torch.tensor(levels, dtype=torch.int64, device="cuda")
    starts = torch.cat([shapes.new_zeros(1), (shapes[:, 0] * shapes[:, 1]).cumsum(0)[:-1]])
    gv, gl, ga = torch.empty_like(value), torch.empty_like(loc), torch.empty_like(w)
    dv, dl, da = torch.empty_like(value), torch.empty_like(loc), torch.empty_like(w)
    n_scratch, n_ws = deform.deterministic_scratch_sizes(N, S, M, D)
    scratch = torch.empty(n_scratch, dtype=torch.int64, device="cuda")
    ws = torch.empty(n_ws, dtype=torch.float32, device="cuda")
    head = (value.data_ptr(), shapes.data_ptr(), starts.data_ptr(), loc.data_ptr(), w.data_ptr(), go.data_ptr(),
            N, S, M, D, Lq, L, P)

    def atomic():
        gv.zero_()
        lib.call("fvit_msda_bwd", *head, gv.data_ptr(), gl.data_ptr(), ga.data_ptr())

    def deterministic():
        lib.call("fvit_msda_bwd_deterministic", *head, dv.data_ptr(), dl.data_ptr(), da.data_ptr(),
                 scratch.data_ptr(), ws.data_ptr())

    # guards on what is being timed: the deterministic arm reproduces itself bitwise; its distance to the atomic one
    atomic()
    deterministic()
    first = dv.clone()
    deterministic()
    reproducible = bool(torch.equal(first, dv))
    del first
    rel = {k: float(f"{((a - b).abs().max() / b.abs().max()).item():.2e}")
           for k, a, b in (("grad_value", dv, gv), ("grad_loc", dl, gl), ("grad_attn", da, ga))}
    t = time_alternating({"atomic": atomic, "deterministic": deterministic}, iters, rounds)
    kern = kernel_us(deterministic, iters)
    torch.cuda.empty_cache()
    return dict(workload=name, N=N, S=S, Lq=Lq, M=M, D=D, L=L, P=P, levels=levels,
                atomic_bwd_ms=round(t["atomic"], 4), deterministic_bwd_ms=round(t["deterministic"], 4),
                slowdown=round(t["deterministic"] / t["atomic"], 2), scratch_bytes=n_scratch * 8,
                grad_value_bytes=value.numel() * 4, deterministic_kernels_us=kern,
                deterministic_reproducible=reproducible, max_rel_diff_to_atomic=rel)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workload", action="append", choices=sorted(WORKLOADS))
    ap.add_argument("--out", default="", help="also write the JSON lines here (a directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deform_det.py needs a CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for name in args.workload or list(WORKLOADS):
        r = dict(bench(name, **WORKLOADS[name], iters=args.iters, rounds=args.rounds), **info)
        rows.append(r)
        print(json.dumps(r), flush=True)
    print(f"\n{'workload':18s} {'atomic ms':>10s} {'determ. ms':>10s} {'slowdown':>9s} {'scratch MB':>11s}")
    for r in rows:
        print(f"{r['workload']:18s} {r['atomic_bwd_ms']:10.3f} {r['deterministic_bwd_ms']:10.3f} "
              f"{r['slowdown']:9.2f} {r['scratch_bytes'] / 1e6:11.1f}")
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_deform_det.jsonl").write_text("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
