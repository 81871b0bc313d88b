"""80-wide attention heads (FasterViT-5 / -6): the tensor-core attention kernels at padded head dim 80 against the SIMT
attention cores that served these heads before, and the fv5 / fv6 models of this tree against a parent checkout.

    python bench_hd80.py [--parent DIR] [--rounds 3] [--steps 10] [--warmup 3] [--kernel-iters 20] [--out DIR]
                         [--parts kernels,models,bench]

Prints the card name and power limit, then one JSON line per measurement and a final JSON line:
  kernels   fvit_attn_core_fwd / _bwd (SIMT, unpadded 80-wide heads) against fvit_attn_tc_fwd / _bwd (S <= 63) or
            fvit_attn_loop_fwd / fvit_attn_loop_bwd_long (S = 148) at fv5's batch-128 shapes -- level 2 (512 windows of
            53 tokens, 16 heads), level 3 (128 x 49, 32 heads), carriers (128 x 16, 16 heads) -- and the any-res level-2
            shape at 576 x 960, batch 16 (240 x 148, 16 heads). Achieved algorithmic TFLOP/s: 4 * groups * heads * S^2 *
            80 for the forward, 2.5 x that for the backward. CUDA events around `kernel-iters` launches, all arms warmed
            up, median of `rounds` alternating windows.
  models    (with --parent) the FasterViT-5 / -6 depths at half width (dim 160, heads [2, 4, 8, 16]: 80-wide heads at
            levels 2 and 3, level 3 at 1280 channels). The full-width entrypoints do not run in either tree: their
            2560-channel level 3 exceeds fvit_ln_fwd's 2048-channel limit. Eval forward of the fv5 model at batch 128,
            training steps of both at the largest batch of 256, 192, 128, 96, 64 that fits the card; parent and this
            tree alternate in fresh processes, median of `rounds`; the fv5 logits of the two trees on one seeded batch
            are compared.
  bench     (with --parent) the default bench.py line of both trees, and whether `bench.py --workload fv0_fwd
            --dump-outputs` gives bitwise-equal logits.
"""
from __future__ import annotations

import argparse
import gc
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

from bench_eval_grad import card, compare, timed  # noqa: E402

HDP = 80
# (tag, groups, S, heads)
SHAPES = [("fv5 level 2, batch 128", 512, 53, 16), ("fv5 level 3, batch 128", 128, 49, 32),
          ("fv5 carriers, batch 128", 128, 16, 16), ("fv5 any-res level 2, 576 x 960, batch 16", 240, 148, 16)]
BATCHES = (256, 192, 128, 96, 64)
HALF = dict(dim=160, num_heads=[2, 4, 8, 16])
MODELS = {"fv5_half": "faster_vit_5_224", "fv6_half": "faster_vit_6_224"}


def kernels(iters: int, rounds: int) -> list:
    from fastervit_b200 import lib as L
    L.load()
    out = []
    for tag, groups, S, h in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(S)
        rows = groups * S
        qkv = torch.randn(rows, 3 * h * HDP, device="cuda", generator=g).half()
        do = torch.randn(rows, h * HDP, device="cuda", generator=g).half()
        bias = torch.randn(h, S, S, device="cuda", generator=g)
        o16 = torch.empty(rows, h * HDP, device="cuda", dtype=torch.half)
        lse = torch.empty(rows, h, device="cuda")
        dqkv = torch.empty(rows, 3 * h * HDP, device="cuda", dtype=torch.half)
        dbias = torch.zeros(h, S, S, device="cuda")
        scratch = torch.empty(rows, h * HDP, device="cuda")
        sc = HDP ** -0.5
        ld3, ld1 = 3 * h * HDP, h * HDP

        def simt_fwd():
            L.call("fvit_attn_core_fwd", qkv.data_ptr(), ld3, groups, S, h, HDP, bias.data_ptr(), sc, o16.data_ptr(), ld1,
                   None)

        def simt_bwd():
            L.call("fvit_attn_core_bwd", qkv.data_ptr(), ld3, do.data_ptr(), ld1, groups, S, h, HDP, HDP, bias.data_ptr(),
                   sc, dqkv.data_ptr(), ld3, dbias.data_ptr())

        if S <= 63:
            def tc_fwd():
                L.call("fvit_attn_tc_fwd", qkv.data_ptr(), ld3, groups, S, h, HDP, bias.data_ptr(), sc, o16.data_ptr(), ld1)

            def tc_bwd():
                L.call("fvit_attn_tc_bwd", qkv.data_ptr(), ld3, do.data_ptr(), ld1, groups, S, h, HDP, HDP, bias.data_ptr(),
                       sc, dqkv.data_ptr(), ld3, dbias.data_ptr())
            names = ("fvit_attn_tc_fwd", "fvit_attn_tc_bwd")
        else:
            def tc_fwd():
                L.call("fvit_attn_loop_fwd", qkv.data_ptr(), ld3, groups, S, h, HDP, bias.data_ptr(), sc, o16.data_ptr(),
                       ld1, lse.data_ptr())

            def tc_bwd():
                L.call("fvit_attn_loop_bwd_long", qkv.data_ptr(), ld3, do.data_ptr(), ld1, o16.data_ptr(), ld1,
                       lse.data_ptr(), groups, S, h, HDP, bias.data_ptr(), sc, dqkv.data_ptr(), ld3, dbias.data_ptr(),
                       scratch.data_ptr(), ld1)
            names = ("fvit_attn_loop_fwd", "fvit_attn_loop_bwd_long")
        arms = {"simt_fwd": simt_fwd, "tc_fwd": tc_fwd, "tc_bwd": tc_bwd}
        res = dict(shape=tag, groups=groups, S=S, heads=h, tc_fwd_kernel=names[0], tc_bwd_kernel=names[1])
        try:
            simt_bwd()
            arms["simt_bwd"] = simt_bwd
        except L.FvitError as e:   # the SIMT backward keeps the whole window in shared memory
            res["simt_bwd"] = f"unsupported: {e}"
        tc_fwd()   # the loop backward reads the forward's output and log-sum-exp rows
        ms = compare(arms, iters, 3, rounds)
        flops = 4.0 * groups * h * S * S * HDP
        for k, v in ms.items():
            f = flops * (2.5 if k.endswith("bwd") else 1.0)
            res[k] = dict(ms=round(v, 4), tflops=round(f / (v * 1e-3) / 1e12, 1))
        for d in ("fwd", "bwd"):
            if isinstance(res.get(f"simt_{d}"), dict):
                res[f"speedup_{d}"] = round(res[f"simt_{d}"]["ms"] / res[f"tc_{d}"]["ms"], 2)
        out.append(res)
        print(json.dumps(res), flush=True)
        del qkv, do, bias, o16, lse, dqkv, dbias, scratch
        torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------ model workloads (run in a child process per tree)
def _model(tag: str):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    m = F.create_model(MODELS[tag], drop_path_rate=0.0, **HALF)
    O.synth_fill_(m.state_dict(), 1)
    return m.cuda()


def _train_fn(m, B: int):
    x = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    gl = torch.randn(B, 1000, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)) / B

    def step():
        torch.autograd.backward(m(x), gl)
    return step


def child_search() -> dict:
    """largest batch of BATCHES whose training step runs, per entry point"""
    out = {}
    for entry in MODELS:
        for B in BATCHES:
            m = _model(entry).train()
            try:
                _train_fn(m, B)()
                torch.cuda.synchronize()
                out[entry] = B
            except torch.OutOfMemoryError:
                pass
            del m
            gc.collect()
            torch.cuda.empty_cache()
            if entry in out:
                break
    return out


def child_models(steps: int, warmup: int, batches: dict, logits_path: str) -> dict:
    res = {}
    m = _model("fv5_half").eval()
    x = torch.randn(128, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    with torch.no_grad():
        torch.save(m(x).float().cpu(), logits_path)

    def infer():
        with torch.no_grad():
            m(x)
    for _ in range(warmup):
        infer()
    ms = timed(infer, steps)
    res["fv5_half_eval_b128"] = dict(ms=round(ms, 3), img_s=round(128 / (ms * 1e-3), 1))
    del m
    gc.collect()
    torch.cuda.empty_cache()
    for entry in MODELS:
        B = batches[entry]
        m = _model(entry).train()
        step = _train_fn(m, B)
        for _ in range(warmup):
            step()
        ms = timed(step, steps)
        res[f"{entry}_train"] = dict(batch=B, ms=round(ms, 3), img_s=round(B / (ms * 1e-3), 1))
        del m, step
        gc.collect()
        torch.cuda.empty_cache()
    return res


def _run_child(tree: Path, *args) -> dict:
    env = dict(os.environ, PYTHONPATH=str(tree))
    r = subprocess.run([sys.executable, str(ROOT / "bench_hd80.py"), "--tree", str(tree), *args], cwd=tree, env=env,
                       capture_output=True, text=True, timeout=3600)
    lines = [s for s in r.stdout.splitlines() if s.startswith("{")]
    if r.returncode or not lines:
        raise RuntimeError(f"child in {tree} failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def models(parent: Path, steps: int, warmup: int, rounds: int, tmp: Path) -> dict:
    batches = _run_child(ROOT, "--child", "search")
    print(json.dumps(dict(train_batches=batches)), flush=True)
    runs = {"parent": [], "new": []}
    for r in range(rounds):
        for tag, tree in (("parent", parent), ("new", ROOT)):
            got = _run_child(tree, "--child", "models", "--steps", str(steps), "--warmup", str(warmup), "--batches",
                             json.dumps(batches), "--logits", str(tmp / f"logits_{tag}_{r}.pt"))
            runs[tag].append(got)
            print(json.dumps(dict(tree=tag, round=r, **got)), flush=True)
    res = {"train_batches": batches}
    for key in runs["new"][0]:
        med = {tag: statistics.median(x[key]["ms"] for x in runs[tag]) for tag in runs}
        res[key] = dict(batch=runs["new"][0][key].get("batch", 128), parent_ms=med["parent"], new_ms=med["new"],
                        speedup=round(med["parent"] / med["new"], 3))
    a, b = torch.load(tmp / "logits_parent_0.pt"), torch.load(tmp / "logits_new_0.pt")
    res["fv5_half_logits_max_rel"] = ((a - b).abs().max() / a.abs().max()).item()
    res["fv5_half_logits_within_1e-3"] = res["fv5_half_logits_max_rel"] < 1e-3
    print(json.dumps(dict(models=res)), flush=True)
    return res


def bench_lines(parent: Path, tmp: Path) -> dict:
    import numpy as np
    res = {}
    for tag, tree in (("parent", parent), ("new", ROOT)):
        env = dict(os.environ, PYTHONPATH=str(tree))
        r = subprocess.run([sys.executable, str(tree / "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "5"],
                           cwd=tree, env=env, capture_output=True, text=True, timeout=3600)
        res[f"{tag}_default"] = json.loads([s for s in r.stdout.splitlines() if s.startswith("{")][-1])
        d = tmp / f"dump_{tag}"
        r = subprocess.run([sys.executable, str(tree / "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "2",
                            "--workload", "fv0_fwd", "--no-also", "--dump-outputs", str(d)], cwd=tree, env=env,
                           capture_output=True, text=True, timeout=3600)
        assert r.returncode == 0, r.stderr[-3000:]
        print(json.dumps({tag: res[f"{tag}_default"].get("value")}), flush=True)
    files = sorted(p.name for p in (tmp / "dump_new").glob("*.npy"))
    assert files
    res["fv0_fwd_dump_bitwise_equal"] = all(
        np.array_equal(np.load(tmp / "dump_parent" / f), np.load(tmp / "dump_new" / f)) for f in files)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="", help="checkout of the parent commit, library built")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=20)
    ap.add_argument("--out", default="")
    ap.add_argument("--parts", default="kernels,models,bench", help="comma-separated subset of kernels, models, bench")
    # child-process mode: models of the tree at --tree
    ap.add_argument("--child", choices=["search", "models"], default="")
    ap.add_argument("--tree", default="")
    ap.add_argument("--batches", default="")
    ap.add_argument("--logits", default="")
    args = ap.parse_args()
    if args.child:
        sys.path.insert(0, str(Path(args.tree).resolve()))
        if args.child == "search":
            print(json.dumps(child_search()))
        else:
            print(json.dumps(child_models(args.steps, args.warmup, json.loads(args.batches), args.logits)))
        return
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    res = dict(card=info)
    parts = args.parts.split(",")
    if "kernels" in parts:
        res["kernels"] = kernels(args.kernel_iters, args.rounds)
    if args.parent:
        with tempfile.TemporaryDirectory() as tmp:
            parent = Path(args.parent).resolve()
            if "models" in parts:
                res["models"] = models(parent, args.steps, args.warmup, args.rounds, Path(tmp))
            if "bench" in parts:
                res["bench"] = bench_lines(parent, Path(tmp))
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_hd80.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
