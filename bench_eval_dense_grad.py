"""Eval-mode gradients of the dense-prediction outputs: what a differentiable eval forward_levels / backbone step costs,
and fvit_feature_map_eval_bwd on its own.

    python bench_eval_dense_grad.py [--steps 10] [--warmup 3] [--rounds 3] [--kernel-iters 50] [--parent DIR] [--out DIR]

Prints the card name, power limit and maximum SM clock, one line per measurement and a final JSON line. Steps are timed
with CUDA events around `steps` calls after `warmup` calls of every arm; the arms of one comparison alternate `rounds`
times and the median of the rounds is reported. Nothing is written unless --out is given.

Measurements:
  * faster_vit_4_224 at batch 128, forward_levels(x, (0, 1, 2, 3)) with a fixed gradient on every map: the eval step
    with the image gradient (eval forward + backward to x and the parameters) next to the train-mode levels step and the
    no_grad inference forward_levels;
  * faster_vit_0_any_res at 576 x 960, batch 8, FasterViTBackbone(out_indices=(1, 2, 3)) under .eval(): the step with
    the image gradient next to the no_grad forward;
  * fvit_feature_map_eval_bwd time and achieved bytes/s at the fv4 batch-128 level shapes; the bytes are the apply's HBM
    traffic (dy read, gradient rows read and written, row map);
  * with --parent DIR (a checkout of the parent commit with its library built): the default `bench.py` line, parent and
    this tree alternating, and whether the fv0_fwd logits of `bench.py --dump-outputs` are bitwise equal.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench_eval_grad import bench_line, card, compare, model_of, timed  # noqa: E402


def levels_step(steps, warmup, rounds) -> dict:
    m = model_of("faster_vit_4_224")
    B, idx = 128, (0, 1, 2, 3)
    x = torch.randn(B, 3, 224, 224, device="cuda")
    with torch.no_grad():
        shapes = [tuple(f.shape) for f in m.eval().forward_levels(x[:1], idx)]
    dmaps = [torch.randn((B,) + s[1:], device="cuda") / B for s in shapes]

    def infer():
        m.eval()
        with torch.no_grad():
            m.forward_levels(x, idx)

    def eval_grad():
        m.eval()
        xg = x.detach().requires_grad_(True)
        torch.autograd.backward(m.forward_levels(xg, idx), dmaps)

    def train():
        m.train()
        torch.autograd.backward(m.forward_levels(x, idx), dmaps)
    # the eval levels plan and the train levels plan each hold a training step's activations: one at a time
    r = compare({"inference": infer, "eval_input_grad": eval_grad}, steps, warmup, rounds)
    m.release_eval_grad_plans()
    torch.cuda.empty_cache()
    r.update(compare({"train": train}, steps, warmup, rounds))
    m.eval()
    res = dict(workload="faster_vit_4_224, batch 128, forward_levels (0, 1, 2, 3)",
               **{f"{k}_ms": round(v, 3) for k, v in r.items()},
               eval_over_train_plus_inference=round(r["eval_input_grad"] / (r["train"] + r["inference"]), 4))
    print(json.dumps(res), flush=True)
    del m
    torch.cuda.empty_cache()
    return res


def backbone_step(steps, warmup, rounds) -> dict:
    from fastervit_b200.backbone import FasterViTBackbone
    from oracle import fastervit_oracle as O
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), drop_path_rate=0.0, resolution=[576, 960])
    O.synth_fill_(bb.state_dict(), 1)
    bb = bb.cuda().eval()
    x = torch.randn(8, 3, 576, 960, device="cuda")
    with torch.no_grad():
        dmaps = [torch.randn_like(o) / 8 for o in bb.forward_raw(x)]

    def infer():
        with torch.no_grad():
            bb.forward_raw(x)

    def eval_grad():
        xg = x.detach().requires_grad_(True)
        torch.autograd.backward(bb.forward_raw(xg), dmaps)
    r = compare({"inference": infer, "eval_input_grad": eval_grad}, steps, warmup, rounds)
    res = dict(workload="faster_vit_0_any_res 576 x 960, batch 8, FasterViTBackbone (1, 2, 3)",
               **{f"{k}_ms": round(v, 3) for k, v in r.items()})
    print(json.dumps(res), flush=True)
    del bb
    torch.cuda.empty_cache()
    return res


def kernels(iters: int) -> list:
    from fastervit_b200 import lib as L
    L.load()
    out = []
    B = 128
    for lvl, (C, HW) in enumerate(((196, 56), (392, 28), (784, 14), (1568, 7))):
        T = HW * HW
        dy = torch.randn(B, C, T, device="cuda")
        # the row map of a zero-bordered level buffer (as the conv levels store their maps)
        bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(HW), torch.arange(HW), indexing="ij")
        rows = (bi * (HW + 2) ** 2 + (yi + 1) * (HW + 2) + xi + 1).reshape(-1).to(torch.int32).cuda()
        g = torch.zeros(B * (HW + 2) ** 2, C, device="cuda")
        rstd, w = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
        gs = torch.tensor([1.0, 1.0], device="cuda")
        fn = lambda: L.call("fvit_feature_map_eval_bwd", dy.data_ptr(), rows.data_ptr(), B, T, C, rstd.data_ptr(),
                            w.data_ptr(), None, None, gs.data_ptr(), None, g.data_ptr(), C, None, None)
        for _ in range(3):
            fn()
        ms = timed(fn, iters)
        nbytes = B * T * C * 12 + B * T * 4
        out.append(dict(kernel=f"fvit_feature_map_eval_bwd fv4 level {lvl}: {B} x {C} x {HW}^2", ms=round(ms, 4),
                        GB=round(nbytes / 1e9, 3), TB_s=round(nbytes / (ms * 1e-3) / 1e12, 3)))
        print(json.dumps(out[-1]), flush=True)
        del dy, g
    return out


def fv0_logits_bitwise(parent: Path) -> bool:
    """bench.py --workload fv0_fwd --dump-outputs of both trees: are the logits bitwise equal?"""
    import numpy as np
    with tempfile.TemporaryDirectory() as td:
        for tag, tree in (("parent", parent), ("new", ROOT)):
            env = dict(os.environ, PYTHONPATH=str(tree))
            subprocess.run([sys.executable, str(tree / "bench.py"), "--gpus", "1", "--steps", "3", "--warmup", "1",
                            "--workload", "fv0_fwd", "--no-also", "--dump-outputs", str(Path(td) / tag)], cwd=tree,
                           env=env, capture_output=True, text=True, timeout=1800, check=True)
        a, b = (np.load(Path(td) / t / "logits.npy") for t in ("parent", "new"))
        return bool(a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all())


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
        parent = Path(args.parent).resolve()
        lines = []
        for _ in range(args.bench_rounds):
            for tag, tree in (("parent", parent), ("new", ROOT)):
                lines.append(dict(tree=tag, **bench_line(tree, 20, 5)))
                print(json.dumps(lines[-1]), flush=True)
        res["bench_default"] = lines
        res["fv0_fwd_logits_bitwise_equal"] = fv0_logits_bitwise(parent)
        print(json.dumps(dict(fv0_fwd_logits_bitwise_equal=res["fv0_fwd_logits_bitwise_equal"])), flush=True)
    res["kernels"] = kernels(args.kernel_iters)
    res["levels_step"] = levels_step(args.steps, args.warmup, args.rounds)
    res["backbone_step"] = backbone_step(args.steps, args.warmup, args.rounds)
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_eval_dense_grad.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
