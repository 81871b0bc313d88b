"""Full-width FasterViT-5 / -6 (dim 320, level 3 at 2560 channels): the models end to end and the LayerNorm kernels at
their level-3 shape.

    python bench_fv56.py [--parent DIR] [--rounds 3] [--steps 10] [--warmup 3] [--kernel-iters 50] [--out DIR]
                         [--parts kernels,models] [--models fv5,fv6]

Prints the card name and power limit, then one JSON line per measurement and a final JSON line:
  kernels   fvit_ln_fwd, fvit_ln_bwd and fvit_ln_dgrad at the level-3 shape of fv5 / fv6 at batch 128 (128 x 49 rows of
            2560 channels): CUDA events around `kernel-iters` launches, median of `rounds` alternating windows, and
            TB/s from the bytes each kernel has to move, computed from the shapes (R rows, C channels):
              fvit_ln_fwd    x fp32 in, y and xhat fp16 out, mean and rstd fp32 out    8RC + 8R
              fvit_ln_bwd    dy and xhat fp16 in, g fp32 in and out                     12RC (+ rstd, dgamma, dbeta)
              fvit_ln_dgrad  the same as fvit_ln_bwd without dgamma / dbeta             12RC
            With --parent, the parent build's fvit_ln_bwd / fvit_ln_dgrad at the same shape (its generic kernels: that
            build's vectorised backward stops at 1792 channels), loaded from DIR's library into the same process and
            alternated with this build's, and the g / dgamma / dbeta of the two builds compared.
  models    each in a fresh process: eval forward at batch 128, and the training step the reference recipe runs
            (train-mode forward, cross-entropy backward, fused LAMB with clip 5.0 and model EMA) at batch 128, or the
            largest of 96 and 64 that fits the card. img/s from CUDA events over `steps` calls after `warmup`, median of
            `rounds`; torch.cuda.max_memory_allocated of the training process. The reference README's 449 / 352 img/s
            for fv5 / fv6 are TensorRT inference throughputs on other hardware: context only, not a like-for-like
            comparison.
"""
from __future__ import annotations

import argparse
import ctypes as C
import gc
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench_eval_grad import card, compare, timed  # noqa: E402

ROWS, CH = 128 * 49, 2560
ENTRIES = {"fv5": "faster_vit_5_224", "fv6": "faster_vit_6_224"}
TRAIN_BATCHES = (128, 96, 64)


# ------------------------------------------------------------------------------------------------------- kernels
def _ln_tensors():
    g = torch.Generator(device="cuda").manual_seed(5)
    t = dict(x=torch.randn(ROWS, CH, device="cuda", generator=g) * 1.7 + 0.3,
             gamma=torch.rand(CH, device="cuda", generator=g) + 0.5,
             beta=torch.randn(CH, device="cuda", generator=g) * 0.1,
             y=torch.empty(ROWS, CH, device="cuda", dtype=torch.half),
             xhat=torch.empty(ROWS, CH, device="cuda", dtype=torch.half),
             mean=torch.empty(ROWS, device="cuda"), rstd=torch.empty(ROWS, device="cuda"),
             dy=(torch.randn(ROWS, CH, device="cuda", generator=g) * 0.5).half(),
             g0=torch.randn(ROWS, CH, device="cuda", generator=g), one=torch.ones(1, device="cuda"))
    return t


def _bwd_arms(lib, t, tag):
    """fvit_ln_bwd / fvit_ln_dgrad of one library on its own g / dgamma / dbeta buffers (use_g = 1 as in the plans)"""
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    g, gd = t["g0"].clone(), t["g0"].clone()
    dgam, dbet = torch.zeros(CH, device="cuda"), torch.zeros(CH, device="cuda")
    args = (t["dy"].data_ptr(), CH, None, t["xhat"].data_ptr(), CH, t["rstd"].data_ptr(), t["gamma"].data_ptr(), ROWS, CH)

    def check(rc, name):
        if rc != 0:
            raise RuntimeError(f"{tag} {name}: {lib.fvit_last_error().decode()}")

    def bwd():
        check(lib.fvit_ln_bwd(*args, g.data_ptr(), CH, None, 1, 0, t["one"].data_ptr(), dgam.data_ptr(), dbet.data_ptr(),
                              stream()), "fvit_ln_bwd")

    def dgrad():
        check(lib.fvit_ln_dgrad(*args, gd.data_ptr(), CH, None, 1, 0, stream()), "fvit_ln_dgrad")
    return {f"{tag}_ln_bwd": bwd, f"{tag}_ln_dgrad": dgrad}, (g, gd, dgam, dbet)


def kernels(parent: Path | None, iters: int, rounds: int) -> dict:
    from fastervit_b200 import lib as L
    lib = L.load()
    t = _ln_tensors()

    def fwd():
        L.call("fvit_ln_fwd", t["x"].data_ptr(), CH, None, ROWS, CH, None, 1, 0, None, 0, t["gamma"].data_ptr(),
               t["beta"].data_ptr(), 1e-5, t["y"].data_ptr(), CH, None, t["mean"].data_ptr(), t["rstd"].data_ptr(),
               t["xhat"].data_ptr(), CH)
    fwd()
    arms = {"new_ln_fwd": fwd}
    new_arms, new_out = _bwd_arms(lib, t, "new")
    arms.update(new_arms)
    res = dict(rows=ROWS, C=CH)
    par_out = None
    if parent is not None:
        plib = C.CDLL(str(parent / "fastervit_b200" / "libfvit_sm100.so"))
        plib.fvit_last_error.restype = C.c_char_p
        L._bind_ops(plib)
        if C.cast(plib.fvit_ln_bwd, C.c_void_p).value == C.cast(lib.fvit_ln_bwd, C.c_void_p).value:
            raise RuntimeError("the parent library resolved to this build's")
        par_arms, par_out = _bwd_arms(plib, t, "parent")
        arms.update(par_arms)
    # one call of each on fresh buffers for the comparison, then the timed windows
    for k in [k for k in arms if k != "new_ln_fwd"]:
        arms[k]()
    torch.cuda.synchronize()
    if par_out is not None:
        names = ("g", "g_dgrad", "dgamma", "dbeta")
        res["new_vs_parent_max_rel"] = {
            n: ((a - b).abs().max() / b.abs().max()).item() for n, a, b in zip(names, new_out, par_out)}
    ms = compare(arms, iters, 3, rounds)
    nbytes = {"ln_fwd": 8.0 * ROWS * CH + 8.0 * ROWS, "ln_bwd": 12.0 * ROWS * CH, "ln_dgrad": 12.0 * ROWS * CH}
    for k, v in ms.items():
        res[k] = dict(us=round(v * 1e3, 2), tb_s=round(nbytes[k.split("_", 1)[1]] / (v * 1e-3) / 1e12, 3))
    if parent is not None:
        for k in ("ln_bwd", "ln_dgrad"):
            res[f"speedup_{k}"] = round(ms[f"parent_{k}"] / ms[f"new_{k}"], 2)
    print(json.dumps(dict(kernels=res)), flush=True)
    return res


# ------------------------------------------------------------------------------------- models (one child process each)
def _model(entry: str):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    m = F.create_model(ENTRIES[entry], drop_path_rate=0.0)
    O.synth_fill_(m.state_dict(), 1)
    return m.cuda()


def child_eval(entry: str, steps: int, warmup: int, rounds: int) -> dict:
    m = _model(entry).eval()
    x = torch.randn(128, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

    def infer():
        with torch.no_grad():
            m(x)
    for _ in range(warmup):
        infer()
    ms = statistics.median(timed(infer, steps) for _ in range(rounds))
    return dict(batch=128, ms=round(ms, 2), img_s=round(128 / (ms * 1e-3), 1),
                max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))


def child_train(entry: str, B: int, steps: int, warmup: int, rounds: int) -> dict:
    from fastervit_b200 import optim as FO
    m = _model(entry).train()
    opt = FO.FusedLamb(m, lr=5e-3, weight_decay=0.15, eps=1e-8, max_grad_norm=5.0)   # faster_vit_6_224_1k.yaml
    ema = FO.FlatEma(m, decay=0.9998)
    opt.attach_ema(ema, m)
    x = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    y = torch.randint(0, 1000, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))

    def step():
        m.zero_grad(set_to_none=True)
        torch.nn.functional.cross_entropy(m(x), y).backward()
        opt.step()
        ema.update(m)
    try:
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
    except torch.OutOfMemoryError:
        return dict(batch=B, oom=True, max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    ms = statistics.median(timed(step, steps) for _ in range(rounds))
    ok = all(torch.isfinite(p).all().item() for p in m.parameters())
    return dict(batch=B, ms=round(ms, 2), img_s=round(B / (ms * 1e-3), 1), params_finite=ok,
                max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                total_memory_gib=round(torch.cuda.get_device_properties(0).total_memory / 2 ** 30, 2))


def _run_child(*args) -> dict:
    r = subprocess.run([sys.executable, str(ROOT / "bench_fv56.py"), "--child", *args], cwd=ROOT,
                       capture_output=True, text=True, timeout=3600)
    lines = [s for s in r.stdout.splitlines() if s.startswith("{")]
    if r.returncode or not lines:
        raise RuntimeError(f"child {args} failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def models(entries: list, steps: int, warmup: int, rounds: int) -> dict:
    res = {}
    for entry in entries:
        got = _run_child("eval", entry, str(steps), str(warmup), str(rounds))
        res[f"{entry}_eval"] = got
        print(json.dumps({f"{entry}_eval": got}), flush=True)
        for B in TRAIN_BATCHES:
            got = _run_child("train", entry, str(steps), str(warmup), str(rounds), str(B))
            print(json.dumps({f"{entry}_train": got}), flush=True)
            if not got.get("oom"):
                res[f"{entry}_train"] = got
                break
            res.setdefault(f"{entry}_train_oom", []).append(got)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="", help="checkout of the parent commit, library built")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default="")
    ap.add_argument("--parts", default="kernels,models", help="comma-separated subset of kernels, models")
    ap.add_argument("--models", default="fv5,fv6", help="comma-separated subset of fv5, fv6")
    ap.add_argument("--child", nargs="+", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        kind, entry, steps, warmup, rounds = args.child[:5]
        if kind == "eval":
            print(json.dumps(child_eval(entry, int(steps), int(warmup), int(rounds))))
        else:
            print(json.dumps(child_train(entry, int(args.child[5]), int(steps), int(warmup), int(rounds))))
        return
    assert torch.cuda.is_available(), "bench_fv56.py measures on a CUDA device"
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    res = dict(card=info)
    parts = args.parts.split(",")
    if "kernels" in parts:
        res["kernels"] = kernels(Path(args.parent).resolve() if args.parent else None, args.kernel_iters, args.rounds)
        gc.collect()
        torch.cuda.empty_cache()
    if "models" in parts:
        res["models"] = models(args.models.split(","), args.steps, args.warmup, args.rounds)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_fv56.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
