"""Step times of the data-only backward and of the train-mode image gradient (H100; run on the GPU, no fallback).

Arms alternate inside every round and the median over rounds is reported, with the card's name and power limit read in
the same run. Prints one JSON line.
  eval input-gradient step (x.requires_grad, cross-entropy backward), full backward (every parameter requires grad, the
    behaviour before data-only stages) against data-only (requires_grad_(False) on every parameter);
  FasterViTBackbone frozen_stages=2: .train() step with and without x.requires_grad, .eval() with x.requires_grad;
  fv4 train step with and without the image gradient;
  fvit_bn_eval_dgrad / fvit_ln_dgrad alone, against fvit_bn_eval_bwd / fvit_ln_bwd and fvit_cast_scale_f16, with the
    bytes each has to move computed from the shapes."""
import argparse
import json
import statistics
import subprocess
import time

import torch


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def _alternate(arms: dict, rounds, steps, warmup):
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(_time(fn, steps))
    return {k: round(statistics.median(v), 3) for k, v in ms.items()}


def _eval_input_grad(name, batch, a):
    """One model; the two plans do not fit side by side at fv4's batch 128, so the arms alternate round by round with
    the eval-grad plans released in between (each arm's plan build and warm-up are outside its timed window)."""
    import fastervit_b200 as F
    m = F.create_model(name).cuda().eval()
    x = torch.randn(batch, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (batch,), device="cuda")

    def fn():
        xg = x.detach().requires_grad_(True)
        torch.nn.functional.cross_entropy(m(xg), y).backward()
        for p in m.parameters():
            p.grad = None
    ms = {"full": [], "data_only": []}
    for _ in range(a.rounds):
        for arm in ms:
            for p in m.parameters():
                p.requires_grad_(arm == "full")
            for _ in range(a.warmup):
                fn()
            ms[arm].append(_time(fn, a.steps))
            m.release_eval_grad_plans()
            torch.cuda.empty_cache()
    res = {k: round(statistics.median(v), 3) for k, v in ms.items()}
    res["ratio"] = round(res["data_only"] / res["full"], 3)
    res["img_per_s"] = {k: round(batch / res[k] * 1e3, 1) for k in ("full", "data_only")}
    return res


def _backbone(a):
    from fastervit_b200.backbone import FasterViTBackbone
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2, 3), frozen_stages=2, resolution=[576, 960]).cuda()
    bb.enable_input_grad()
    x = torch.randn(8, 3, 576, 960, device="cuda")

    def step(train, dx):
        def fn():
            bb.train(train)
            xg = x.detach().requires_grad_(dx)
            sum(o.square().mean() for o in bb.forward_raw(xg)).backward()
            for p in bb.parameters():
                p.grad = None
        return fn
    return _alternate({"train": step(True, False), "train_dx": step(True, True), "eval_dx": step(False, True)},
                      a.rounds, a.steps, a.warmup)


def _fv4_train(a):
    import fastervit_b200 as F
    m = F.create_model("faster_vit_4_224").cuda().train().enable_input_grad()
    x = torch.randn(128, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (128,), device="cuda")

    def step(dx):
        def fn():
            xg = x.detach().requires_grad_(dx)
            torch.nn.functional.cross_entropy(m(xg), y).backward()
            for p in m.parameters():
                p.grad = None
        return fn
    return _alternate({"train": step(False), "train_dx": step(True)}, a.rounds, a.steps, a.warmup)


def _kernels(a):
    from fastervit_b200 import lib as L
    L.load()
    out = {}
    for tag, rows, C in (("stem_bn1_1.6Mx64", 128 * 112 * 112, 64), ("level0_401kx196", 128 * 56 * 56, 196)):
        ld = (C + 7) // 8 * 8
        g32 = torch.randn(rows, C, device="cuda")
        g16 = torch.randn(rows, ld, device="cuda").half()
        raw = torch.randn(rows, ld, device="cuda").half()
        o16 = torch.empty(rows, ld, device="cuda", dtype=torch.float16)
        v = [torch.rand(C, device="cuda") + 0.5 for _ in range(4)]
        dw, db, one = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda"), torch.ones(1, device="cuda")
        arms = {
            "bn_eval_dgrad_f16_relu": lambda: L.call("fvit_bn_eval_dgrad", g16.data_ptr(), 1, ld, None, raw.data_ptr(), ld, None,
                                                     rows, C, v[0].data_ptr(), v[1].data_ptr(), 1, None, None, o16.data_ptr(), ld, None),
            "bn_eval_dgrad_f32_none": lambda: L.call("fvit_bn_eval_dgrad", g32.data_ptr(), 0, C, None, None, 0, None, rows, C,
                                                     v[0].data_ptr(), None, 0, None, None, o16.data_ptr(), ld, None),
            "bn_eval_bwd_f16_relu": lambda: L.call("fvit_bn_eval_bwd", g16.data_ptr(), 1, ld, None, raw.data_ptr(), ld, None, rows, C,
                                                   v[2].data_ptr(), v[3].data_ptr(), 1e-5, v[0].data_ptr(), v[1].data_ptr(), 1, None,
                                                   one.data_ptr(), o16.data_ptr(), ld, None, dw.data_ptr(), db.data_ptr()),
            "bn_eval_bwd_f32_none": lambda: L.call("fvit_bn_eval_bwd", g32.data_ptr(), 0, C, None, raw.data_ptr(), ld, None, rows, C,
                                                   v[2].data_ptr(), v[3].data_ptr(), 1e-5, v[0].data_ptr(), v[1].data_ptr(), 0, None,
                                                   one.data_ptr(), o16.data_ptr(), ld, None, dw.data_ptr(), db.data_ptr()),
            "cast_scale_f16": lambda: L.call("fvit_cast_scale_f16", g32.data_ptr(), C, None, rows, C, v[0].data_ptr(), None,
                                             o16.data_ptr(), ld, None),
        }
        nbytes = {"bn_eval_dgrad_f16_relu": rows * ld * 6, "bn_eval_dgrad_f32_none": rows * (C * 4 + ld * 2),
                  "bn_eval_bwd_f16_relu": rows * ld * 6, "bn_eval_bwd_f32_none": rows * (C * 4 + ld * 4),
                  "cast_scale_f16": rows * (C * 4 + ld * 2)}
        if True:
            xh = torch.randn(rows, ld, device="cuda").half()
            rs = torch.rand(rows, device="cuda") + 0.5
            g = torch.zeros(rows, C, device="cuda")
            arms["ln_dgrad"] = lambda: L.call("fvit_ln_dgrad", g16.data_ptr(), ld, None, xh.data_ptr(), ld, rs.data_ptr(),
                                              v[0].data_ptr(), rows, C, g.data_ptr(), C, None, 1, 0)
            arms["ln_bwd"] = lambda: L.call("fvit_ln_bwd", g16.data_ptr(), ld, None, xh.data_ptr(), ld, rs.data_ptr(),
                                            v[0].data_ptr(), rows, C, g.data_ptr(), C, None, 1, 0, one.data_ptr(), dw.data_ptr(),
                                            db.data_ptr())
            nbytes["ln_dgrad"] = rows * (2 * C * 2 + 2 * C * 4 + 4)
            nbytes["ln_bwd"] = rows * (4 * C * 2 + 2 * C * 4 + 4)     # (the vectorised path reads dy / xhat twice)
        ms = _alternate(arms, a.rounds, 50, 5)
        out[tag] = {k: dict(us=round(ms[k] * 1e3, 1), TB_per_s=round(nbytes[k] / (ms[k] * 1e-3) / 1e12, 2)) for k in arms}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_data_grad.py measures on a CUDA device; none found")
    parts = {"fv4_eval_input_grad_b128": lambda: _eval_input_grad("faster_vit_4_224", 128, a),
             "fv0_eval_input_grad_b256": lambda: _eval_input_grad("faster_vit_0_224", 256, a),
             "backbone_fv0_576x960_b8_fs2": lambda: _backbone(a), "fv4_train_b128": lambda: _fv4_train(a),
             "kernels": lambda: _kernels(a)}
    res = {"card": _card(), "unit": "ms per step, median of rounds"}
    for k, fn in parts.items():
        if not a.only or k in a.only.split(","):
            res[k] = fn()
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
