"""The stride-1 3x3 convolution GEMMs of the conv levels, timed on their own.

    python bench_conv_taps.py [--model fv4|fv0] [--batch 128] [--tile-n 0,32,64,96,128] [--iters 20] [--out DIR]

Each conv level runs its ConvBlock GEMMs as one 9-tap `fvit_gemm` over the zero-bordered NHWC activation matrix (rows
B x (H+2) x (W+2), row map to the interior pixels), in the three epilogue variants of a training step:
  fwd    raw conv + BatchNorm column statistics (fp16 out)             -- conv1 / conv2 forward
  dgelu  data gradient * GELU'(BN(aux)) (fp16 out)                      -- conv2 data gradient
  dres   data gradient + residual (fp32 out)                            -- conv1 data gradient
A training step of faster_vit_4_224 runs 2 x 2 x depth of them per level (forward and data gradient of both convs).

Prints the card name and power limit, one JSON line per (level, variant, tile_n) and a final JSON line. tile_n 0 is the
library's own choice. Times are CUDA events around `iters` launches after 3 warm-up launches, median of `rounds`
windows. Bytes are the traffic the algorithm needs from HBM (activation and weights read once, outputs written
once); `unit_us` is the time of one 128-row x tile_n work unit on one SM (time x SMs / units).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench_eval_grad import card, timed  # noqa: E402

LEVELS = {"fv4": [(196, 56), (392, 28)], "fv0": [(64, 56), (128, 28)]}


def _ru(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def level_bench(C: int, H: int, B: int, tiles: list[int], iters: int, rounds: int) -> list[dict]:
    from fastervit_b200 import lib as L
    W, P = H, H + 2
    rows, ld, npix = B * P * P, _ru(C, 8), B * H * H
    kp = _ru(C, 64)
    g = torch.Generator(device="cuda").manual_seed(0)
    inside = torch.zeros(B, P, P, dtype=torch.bool, device="cuda")
    inside[:, 1:-1, 1:-1] = True
    inside = inside.reshape(-1)
    x = torch.randn(rows, ld, device="cuda", generator=g).half()
    x[~inside] = 0
    x[:, C:] = 0
    w = torch.zeros(C, 9 * kp, device="cuda", dtype=torch.float16)
    for t in range(9):
        w[:, t * kp:t * kp + C] = (torch.randn(C, C, device="cuda", generator=g) / (3 * C ** 0.5)).half()
    row_map = torch.where(inside, torch.arange(rows, device="cuda", dtype=torch.int32),
                          torch.full((rows,), -1, device="cuda", dtype=torch.int32))
    taps = [((dy - 1) * P + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    o16 = torch.empty(rows, ld, device="cuda", dtype=torch.float16)
    aux = torch.randn(rows, ld, device="cuda", generator=g).half()
    sc, sh = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
    csum, csq = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    r32 = torch.randn(rows, C, device="cuda", generator=g)
    common = dict(m=rows, n=C, kc=C, taps=taps, row_map=row_map)
    variants = {
        "fwd": (lambda tn: L.gemm(x, w, tile_n=tn, col_shift=sh, out_f16=o16, col_sum=csum, col_sumsq=csq, **common),
                npix * C * 2),
        "dgelu": (lambda tn: L.gemm(x, w, tile_n=tn, act=L.ACT_GELU_BWD, aux=aux, aux_scale=sc, aux_shift=sh,
                                    out_f16=o16, **common), 2 * npix * C * 2),
        "dres": (lambda tn: L.gemm(x, w, tile_n=tn, resid=r32, out_f32=r32, **common), 2 * npix * C * 4),
    }
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    flops = 2.0 * npix * C * C * 9
    out = []
    for vname, (fn, out_bytes) in variants.items():
        nbytes = rows * C * 2 + 9 * C * C * 2 + out_bytes
        for tn in tiles:
            for _ in range(3):
                fn(tn)
            ms = statistics.median(timed(lambda: fn(tn), iters) for _ in range(rounds))
            r = dict(C=C, H=H, batch=B, m=rows, n=C, kc=C, variant=vname, tile_n=tn, ms=round(ms, 4),
                     tflops=round(flops / (ms * 1e-3) / 1e12, 1), GB=round(nbytes / 1e9, 3),
                     TB_s=round(nbytes / (ms * 1e-3) / 1e12, 3))
            if tn:
                units = -(-rows // 128) * -(-C // tn)
                r.update(units=units, unit_us=round(ms * 1e3 * min(sms, units) / units, 3))
            out.append(r)
            print(json.dumps(r), flush=True)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="fv4", choices=sorted(LEVELS))
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--tile-n", default="0,32,64,96,128")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_taps.py measures on a CUDA device; none is visible")
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    tiles = [int(t) for t in args.tile_n.split(",")]
    res = dict(card=info, model=args.model, runs=[])
    for C, H in LEVELS[args.model]:
        res["runs"] += level_bench(C, H, args.batch, tiles, args.iters, args.rounds)
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / f"bench_conv_taps_{args.model}.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
