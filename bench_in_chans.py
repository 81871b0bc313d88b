"""What the input channel count costs: FasterViT with in_chans = 1, 3, 4 and 13, and the stem kernels that depend on it.

    python bench_in_chans.py [--steps 10] [--warmup 3] [--rounds 3] [--kernel-iters 50] [--chans 1,3,4,13] [--out DIR]

Prints the card name and power limit, one line per measurement and a final JSON line. Nothing is written unless --out
is given. Steps are timed with CUDA events around `steps` calls after `warmup` calls, `rounds` times, and the median of
the rounds is reported.

Measurements:
  * faster_vit_0_224 at batch 256 and faster_vit_4_224 at batch 128: the eval forward (torch.no_grad) and the train step
    (train-mode forward + cross-entropy + backward) at every channel count, in images per second;
  * kernel time and algorithmic bytes/s of fvit_stem_im2col (fp32 image in, fp16 rows of stem_ld = round_up(9 cin, 32)
    out) and of fvit_stem_col2im (fp32 tap rows in, fp32 image gradient out) at the fv0 batch-256 shape. The bytes are
    the traffic the algorithm needs: every input element read once and every output element written once.
"""
from __future__ import annotations

import argparse
import gc
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench_eval_grad import card, compare, timed  # noqa: E402


def models(chans: list[int], steps: int, warmup: int, rounds: int) -> list[dict]:
    """one model at a time: four fv4 training plans at batch 128 do not fit in 80 GB together, so the channel counts
    run one after the other (each warmed up, then `rounds` timed windows) instead of alternating"""
    import fastervit_b200 as F
    out = []
    for name, B in (("faster_vit_0_224", 256), ("faster_vit_4_224", 128)):
        tgt = torch.randint(0, 1000, (B,), device="cuda")
        for mode in ("eval_fwd", "train_step"):
            ms = {}
            for c in chans:
                net = F.create_model(name, in_chans=c).cuda().train(mode == "train_step")
                x = torch.randn(B, c, 224, 224, device="cuda")

                def step():
                    if mode == "eval_fwd":
                        with torch.no_grad():
                            net(x)
                    else:
                        net.zero_grad(set_to_none=True)
                        torch.nn.functional.cross_entropy(net(x), tgt).backward()
                ms[c] = compare({c: step}, steps, warmup, rounds)[c]
                del net, x, step
                gc.collect()   # (a model's plans and their CUDA graphs sit in reference cycles)
                torch.cuda.empty_cache()
            for c in chans:
                out.append(dict(model=name, batch=B, mode=mode, in_chans=c, ms=round(ms[c], 3),
                                img_s=round(B / (ms[c] * 1e-3), 1), vs_rgb=round(ms[c] / ms[3], 4) if 3 in ms else None))
                print(json.dumps(out[-1]), flush=True)
    return out


def kernels(chans: list[int], iters: int) -> list[dict]:
    from fastervit_b200 import lib as L
    L.load()
    B, H, W = 256, 224, 224
    H1, W1 = (H + 1) // 2, (W + 1) // 2
    npix = B * H1 * W1
    out = []
    for c in chans:
        sld = 32 if c == 3 else (9 * c + 31) // 32 * 32
        x = torch.randn(B, c, H, W, device="cuda")
        col = torch.empty(npix, sld, device="cuda", dtype=torch.float16)
        runs = [("fvit_stem_im2col", lambda: L.call("fvit_stem_im2col", x.data_ptr(), *x.stride(), B, c, H, W,
                                                     col.data_ptr(), sld), x.numel() * 4 + col.numel() * 2)]
        if c != 3:   # (RGB takes fvit_stem_conv_dgrad: bench_eval_grad.py)
            ldc = (9 * c + 3) // 4 * 4
            dcol = torch.randn(npix, ldc, device="cuda")
            dx = torch.empty(B, c, H, W, device="cuda")
            runs.append(("fvit_stem_col2im", lambda: L.call("fvit_stem_col2im", dcol.data_ptr(), ldc, B, c, H, W,
                                                             dx.data_ptr()), npix * 9 * c * 4 + dx.numel() * 4))
        for name, fn, nbytes in runs:
            for _ in range(3):
                fn()
            ms = timed(fn, iters)
            out.append(dict(kernel=name, in_chans=c, shape=f"{B} x {c} x {H} x {W}", ms=round(ms, 4),
                            GB=round(nbytes / 1e9, 3), TB_s=round(nbytes / (ms * 1e-3) / 1e12, 3)))
            print(json.dumps(out[-1]), flush=True)
        torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--chans", default="1,3,4,13")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_in_chans.py measures on a CUDA device; none is visible")
    chans = [int(c) for c in args.chans.split(",")]
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    res = dict(card=info, kernels=kernels(chans, args.kernel_iters),
               models=models(chans, args.steps, args.warmup, args.rounds))
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_in_chans.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
