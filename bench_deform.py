"""Multi-scale deformable attention core: fvit_msda_fwd / fvit_msda_bwd against the grid_sample-style fallback.

    python bench_deform.py [--rounds 5] [--iters 20] [--out DIR]

For each workload it times, with CUDA events (warm-up first, `iters` launches per timing, median of `rounds`):
  * kernel fwd: MSDeformAttnFunction's forward launch (fvit_msda_fwd);
  * kernel bwd: the backward as MSDeformAttnFunction runs it, zeroing grad_value and then fvit_msda_bwd;
  * oracle fwd / fwd+bwd: oracle/msda_oracle.py's explicit bilinear gather in fp32 on the same card, the torch path
    a DINO user falls back to without the extension (fwd under no_grad; fwd+bwd by autograd).
Achieved bytes/s are algorithmic bytes over time: value read once, locations, weights and output (forward); plus
grad_out read, grad_value read and written, and the location and weight gradients written (backward). The card name and
power limit are read in the same run. One JSON line per workload, and a summary table, go to stdout (and DIR if given).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from fastervit_b200 import lib  # noqa: E402
from oracle import msda_oracle  # noqa: E402

M, D, P = 8, 32, 4     # DINO / MOTRv2: d_model 256, 8 heads, 4 points
DINO4 = [(100, 167), (50, 84), (25, 42), (13, 21)]          # 800 x 1333, strides 8..64
WORKLOADS = {
    "dino_enc_4scale": dict(N=2, levels=DINO4, Lq=None),
    "dino_enc_5scale": dict(N=2, levels=[(200, 334)] + DINO4, Lq=None),
    "dino_dec_cross": dict(N=2, levels=DINO4, Lq=1100),      # 900 queries + 2 x 100 denoising queries
    "motrv2_enc": dict(N=1, levels=[(100, 192), (50, 96), (25, 48), (13, 24)], Lq=None),   # 800 x 1536
}


def card() -> dict:
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def time_ms(fn, iters: int, rounds: int) -> float:
    """Median over rounds of the mean time of `iters` back-to-back calls, CUDA events."""
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        res.append(a.elapsed_time(b) / iters)
    return statistics.median(res)


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
    out = torch.empty(N, Lq, M * D, device="cuda")
    gv, gl, ga = torch.empty_like(value), torch.empty_like(loc), torch.empty_like(w)
    sizes = (N, S, M, D, Lq, L, P)

    def fwd():
        lib.call("fvit_msda_fwd", value.data_ptr(), shapes.data_ptr(), starts.data_ptr(), loc.data_ptr(),
                 w.data_ptr(), *sizes, out.data_ptr())

    def bwd():
        gv.zero_()
        lib.call("fvit_msda_bwd", value.data_ptr(), shapes.data_ptr(), starts.data_ptr(), loc.data_ptr(),
                 w.data_ptr(), go.data_ptr(), *sizes, gv.data_ptr(), gl.data_ptr(), ga.data_ptr())

    def oracle_fwd():
        with torch.no_grad():
            msda_oracle.ms_deform_attn_core(value, levels, loc, w, starts)

    def oracle_fwd_bwd():
        msda_oracle.ms_deform_attn_grads(value, levels, loc, w, go, starts)

    # the kernels against the fp32 oracle, as a guard on what is being timed
    fwd()
    bwd()
    ref = msda_oracle.ms_deform_attn_grads(value, levels, loc, w, go, starts)
    errs = {k: ((a - b).abs().max() / b.abs().max()).item()
            for k, a, b in zip(("out", "grad_value", "grad_loc", "grad_attn"), (out, gv, gl, ga), ref)}
    del ref
    t_fwd, t_bwd = time_ms(fwd, iters, rounds), time_ms(bwd, iters, rounds)
    t_ofwd = time_ms(oracle_fwd, iters, rounds)
    t_obwd = time_ms(oracle_fwd_bwd, iters, rounds)
    f4 = 4
    bytes_fwd = f4 * (value.numel() + loc.numel() + w.numel() + out.numel())
    bytes_bwd = f4 * (value.numel() + loc.numel() + w.numel() + go.numel() + 2 * gv.numel() + gl.numel() + ga.numel())
    torch.cuda.empty_cache()
    return dict(workload=name, N=N, S=S, Lq=Lq, M=M, D=D, L=L, P=P, levels=levels,
                kernel_fwd_ms=round(t_fwd, 4), kernel_bwd_ms=round(t_bwd, 4),
                oracle_fp32_fwd_ms=round(t_ofwd, 3), oracle_fp32_fwd_bwd_ms=round(t_obwd, 3),
                speedup_fwd=round(t_ofwd / t_fwd, 1), speedup_fwd_bwd=round(t_obwd / (t_fwd + t_bwd), 1),
                kernel_fwd_GBps=round(bytes_fwd / t_fwd / 1e6, 1), kernel_bwd_GBps=round(bytes_bwd / t_bwd / 1e6, 1),
                max_rel_err_vs_fp32_oracle={k: float(f"{v:.2e}") for k, v in errs.items()})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workload", action="append", choices=sorted(WORKLOADS))
    ap.add_argument("--out", default="", help="also write the JSON lines here (a directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deform.py needs a CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for name in args.workload or list(WORKLOADS):
        r = dict(bench(name, **WORKLOADS[name], iters=args.iters, rounds=args.rounds), **info)
        rows.append(r)
        print(json.dumps(r), flush=True)
    print(f"\n{'workload':18s} {'fwd ms':>8s} {'bwd ms':>8s} {'fwd GB/s':>9s} {'bwd GB/s':>9s} "
          f"{'oracle fwd':>10s} {'oracle f+b':>10s} {'x fwd':>6s} {'x f+b':>6s}")
    for r in rows:
        print(f"{r['workload']:18s} {r['kernel_fwd_ms']:8.3f} {r['kernel_bwd_ms']:8.3f} {r['kernel_fwd_GBps']:9.1f} "
              f"{r['kernel_bwd_GBps']:9.1f} {r['oracle_fp32_fwd_ms']:10.2f} {r['oracle_fp32_fwd_bwd_ms']:10.2f} "
              f"{r['speedup_fwd']:6.1f} {r['speedup_fwd_bwd']:6.1f}")
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_deform.jsonl").write_text("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
