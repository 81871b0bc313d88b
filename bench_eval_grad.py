"""Eval-mode gradient measurement: what a differentiable eval forward costs, and the eval backward kernels on their own.

    python bench_eval_grad.py [--steps 10] [--warmup 3] [--rounds 3] [--kernel-iters 50] [--parent DIR] [--out DIR]

Prints the card name and power limit, one line per measurement and a final JSON line. Steps are timed with CUDA events
around `steps` calls after `warmup` calls of every arm; the arms of one comparison alternate `rounds` times and the
median of the rounds is reported. Nothing is written unless --out is given.

Measurements:
  * with --parent DIR (a checkout of the parent commit with its library built): the default `bench.py` line and its
    fv0_fwd / fv4_fwd / fv0_fwd_b8 entries, parent and this tree alternating;
  * faster_vit_0_224 eval forward at batch 256 and at batch 8 (latency): under torch.no_grad() against grad enabled
    with parameters that require grad and no backward (the output is dropped);
  * faster_vit_4_224 at batch 128: the eval input-gradient step (eval forward + backward to x and the parameters) next
    to the train step and the no_grad inference forward;
  * kernel time and achieved bytes/s of fvit_bn_eval_bwd, fvit_pool_bn_eval_bwd and fvit_stem_conv_dgrad at the fv4
    batch-128 shapes; the bytes are the algorithm's HBM traffic computed from the shapes below.
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
    """ms per call of every arm: all arms warmed up, then `rounds` alternating timed windows, median of the rounds"""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, steps))
    return {k: statistics.median(v) for k, v in res.items()}


def bench_line(tree: Path, steps: int, warmup: int) -> dict:
    """the default bench.py line of the tree at `tree` (its own code and library)"""
    env = dict(os.environ, PYTHONPATH=str(tree))
    r = subprocess.run([sys.executable, str(tree / "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
                        str(warmup)], cwd=tree, env=env, capture_output=True, text=True, timeout=3600)
    line = json.loads([s for s in r.stdout.splitlines() if s.startswith("{")][-1])
    also = line.get("also_measured") or {}
    pick = {k: also[k].get("value") for k in ("fv0_fwd", "fv4_fwd", "fv0_fwd_b8") if isinstance(also.get(k), dict)}
    return dict(value=line["value"], **pick)


def model_of(entry: str):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    m = F.create_model(entry, drop_path_rate=0.0)
    O.synth_fill_(m.state_dict(), 1)
    return m.cuda()


def forward_overhead(steps, warmup, rounds) -> list:
    out = []
    m = model_of("faster_vit_0_224").eval()
    for batch in (256, 8):
        x = torch.randn(batch, 3, 224, 224, device="cuda")

        def no_grad():
            with torch.no_grad():
                m(x)

        def grad_enabled():
            m(x)
        # (batch 8 is host-bound and the host is shared: more, longer rounds there)
        r = compare({"no_grad": no_grad, "grad_enabled": grad_enabled}, steps * (4 if batch == 8 else 1), warmup,
                    rounds * (3 if batch == 8 else 1))
        out.append(dict(workload=f"faster_vit_0_224 eval forward, batch {batch}", no_grad_ms=round(r["no_grad"], 4),
                        grad_enabled_ms=round(r["grad_enabled"], 4),
                        ratio=round(r["grad_enabled"] / r["no_grad"], 4)))
        print(json.dumps(out[-1]), flush=True)
    assert not m._get_engine().eval_grad_plans(), "a forward without backward built an eval-grad plan"
    return out


def input_grad_step(steps, warmup, rounds) -> dict:
    m = model_of("faster_vit_4_224")
    B = 128
    x = torch.randn(B, 3, 224, 224, device="cuda")
    gl = torch.randn(B, 1000, device="cuda") / B

    def infer():
        m.eval()
        with torch.no_grad():
            m(x)

    def eval_grad():
        m.eval()
        xg = x.detach().requires_grad_(True)
        torch.autograd.backward(m(xg), gl)

    def train():
        m.train()
        torch.autograd.backward(m(x), gl)
    # the eval-grad plan and the train plan each hold a training step's activations: one at a time on an 80 GB card
    r = compare({"inference": infer, "eval_input_grad": eval_grad}, steps, warmup, rounds)
    m.release_eval_grad_plans()
    torch.cuda.empty_cache()
    r.update(compare({"train": train}, steps, warmup, rounds))
    m.eval()
    res = dict(workload="faster_vit_4_224, batch 128", **{f"{k}_ms": round(v, 3) for k, v in r.items()},
               **{f"{k}_img_s": round(B / (v / 1e3), 1) for k, v in r.items()},
               eval_over_train_plus_inference=round(r["eval_input_grad"] / (r["train"] + r["inference"]), 4))
    print(json.dumps(res), flush=True)
    return res


def kernels(iters: int) -> list:
    from fastervit_b200 import lib as L
    L.load()
    dev = "cuda"
    out = []

    def run(name, fn, nbytes):
        for _ in range(3):
            fn()
        ms = timed(fn, iters)
        out.append(dict(kernel=name, ms=round(ms, 4), GB=round(nbytes / 1e9, 3), TB_s=round(nbytes / (ms * 1e-3) / 1e12, 3)))
        print(json.dumps(out[-1]), flush=True)
    vec = lambda n: torch.rand(n, device=dev) + 0.5
    # BatchNorm on running statistics: the stem's first BN (fp16 gradient in, 1.6 M pixel rows x 64) and a level-0
    # ConvBlock norm2 (fp32 residual-stream gradient in, 401 k rows x 196, rows padded to 200)
    for tag, rows, C, ld, g16 in (("stem bn1, 1605632 x 64, fp16 dy", 128 * 112 * 112, 64, 64, 1),
                                  ("level-0 norm2, 401408 x 196, fp32 dy", 128 * 56 * 56, 196, 200, 0)):
        gin = torch.randn(rows, ld if g16 else C, device=dev, dtype=torch.float16 if g16 else torch.float32)
        raw = torch.randn(rows, ld, device=dev, dtype=torch.float16)
        o = torch.empty(rows, ld, device=dev, dtype=torch.float16)
        mu, var, w, b, dw, db = (vec(C) for _ in range(6))
        sc = torch.ones(1, device=dev)
        nbytes = rows * C * ((2 if g16 else 4) + 2 + 2)
        run(f"fvit_bn_eval_bwd {tag}", lambda: L.call(
            "fvit_bn_eval_bwd", gin.data_ptr(), g16, gin.stride(0), None, raw.data_ptr(), ld, None, rows, C, mu.data_ptr(),
            var.data_ptr(), 1e-5, w.data_ptr(), b.data_ptr(), 1, None, sc.data_ptr(), o.data_ptr(), ld, None, dw.data_ptr(),
            db.data_ptr()), nbytes)
    B, T, C = 128, 49, 1568
    xs = torch.randn(B * T, C, device=dev)
    g = torch.empty(B * T, C, device=dev)
    dpool = torch.randn(B, C, device=dev)
    mu, var, w, dw, db = (vec(C) for _ in range(5))
    sc = torch.ones(1, device=dev)
    run("fvit_pool_bn_eval_bwd 128 x 49 x 1568", lambda: L.call(
        "fvit_pool_bn_eval_bwd", xs.data_ptr(), C, None, B, T, C, mu.data_ptr(), var.data_ptr(), 1e-5, w.data_ptr(),
        dpool.data_ptr(), C, sc.data_ptr(), g.data_ptr(), C, dw.data_ptr(), db.data_ptr()), B * T * C * 8 + B * C * 4)
    H = W = 224
    cout = 64
    dz = torch.randn(B * 112 * 112, cout, device=dev, dtype=torch.float16)
    wgt = torch.randn(cout, 3, 3, 3, device=dev)
    dx = torch.empty(B, 3, H, W, device=dev)
    run("fvit_stem_conv_dgrad 128 x 112 x 112 x 64 -> 128 x 3 x 224 x 224", lambda: L.call(
        "fvit_stem_conv_dgrad", dz.data_ptr(), cout, B, H, W, wgt.data_ptr(), cout, sc.data_ptr(), dx.data_ptr()),
        dz.numel() * 2 + dx.numel() * 4)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--parent", default="", help="checkout of the parent commit, library built: A/B the default line")
    ap.add_argument("--bench-rounds", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    res = dict(card=info)
    if args.parent:
        lines = []
        for _ in range(args.bench_rounds):
            for tag, tree in (("parent", Path(args.parent).resolve()), ("new", ROOT)):
                lines.append(dict(tree=tag, **bench_line(tree, 20, 5)))
                print(json.dumps(lines[-1]), flush=True)
        res["bench_default"] = lines
    res["forward_overhead"] = forward_overhead(args.steps * 2, args.warmup, args.rounds)
    res["input_grad_step"] = input_grad_step(args.steps, args.warmup, args.rounds)
    res["kernels"] = kernels(args.kernel_iters)
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_eval_grad.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
