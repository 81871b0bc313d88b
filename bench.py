#!/usr/bin/env python3
"""bench.py — images/sec of the FasterViT hot path on an H100 (sm_90a).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload fv0_fwd] [--impl reference] [--dump-outputs DIR]

One "step" = one pass of the hot path over one synthetic batch. Default workload = BASELINE.json
configs[1]: faster_vit_0_224 forward-only, batch 256 per GPU (random-init weights, synthetic N(0,1)
images). `value` is whole-job img/s with inputs resident in HBM; `e2e` is the same metric through the
public API (create_model(...)(x)) with pinned-host inputs uploaded and logits downloaded every step.
`--impl reference` times the reference's CPU implementation of the path (the oracle port of
fastervit/models/faster_vit.py — the Python reference cannot travel to the GPU box) on the host cores.
Under torchrun (N > 1) every rank runs an independent replica on its own batch (the forward path has
no exchange step; weak scaling) and the time is the max over ranks.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

WORKLOADS = {
    # name: (entrypoint, create kwargs, per-GPU batch, resolution (H, W), mode)
    "fv0_fwd": ("faster_vit_0_224", {}, 256, (224, 224), "fwd"),
    "fv4_fwd": ("faster_vit_4_224", {}, 128, (224, 224), "fwd"),
    "ar0_fwd": ("faster_vit_0_any_res", dict(resolution=[576, 960], window_size=[7, 7, 12, 6], ct_size=2, dim=64),
                32, (576, 960), "fwd"),
    # training steps: forward (batch-statistics BN) + cross-entropy + backward; drop_path_rate = 0 (stochastic
    # depth is a per-window mask multiply: same FLOPs) ; no optimizer (the metric is fwd+bwd img/s)
    "fv0_train": ("faster_vit_0_224", dict(drop_path_rate=0.0), 256, (224, 224), "train"),
    "fv4_train": ("faster_vit_4_224", dict(drop_path_rate=0.0), 128, (224, 224), "train"),
    # side measurements of the `also_measured` block (not BASELINE configs): small-batch latency of the forward launch
    # graph, and a training step of a 21k fine-tuning model whose 24 x 24 windows (S = 576) take the long-window
    # attention backward (fvit_attn_loop_bwd_long)
    # the default workload with the entrypoint's own stochastic-depth rate (fv.py:1138: 0.3): per-step mask generation
    # inside the captured step + the row-scale epilogues, same FLOPs
    "fv4_train_droppath": ("faster_vit_4_224", {}, 128, (224, 224), "train"),
    "fv0_fwd_b8": ("faster_vit_0_224", {}, 8, (224, 224), "fwd"),
    "fv4_21k_384_train": ("faster_vit_4_21k_384", dict(drop_path_rate=0.0), 16, (384, 384), "train"),  # fits 80 GB
}
ORACLE_CASE = {"fv0_fwd": "fv0", "fv4_fwd": "fv4", "ar0_fwd": "ar0", "fv0_train": "fv0", "fv4_train": "fv4"}
# algorithmic forward GFLOP per image (BASELINE.md §2, measured on the reference with FlopCounterMode)
ALG_GFLOP_FWD = {"fv0_fwd": 6.7237, "fv4_fwd": 85.3574, "ar0_fwd": 73.0828,
                 "fv0_train": 20.3580, "fv4_train": 258.1946, "fv4_train_droppath": 258.1946}  # train entries: fwd+bwd (BASELINE.md §2)


# published numbers for the same metric (BASELINE.md §1: the reference README's inference-throughput column, hardware
# "not stated in repo", paper: A100 / TensorRT); nothing is published for forward+backward or for any-res
PUBLISHED_IMG_S = {"fv0_fwd": 5802.0, "fv4_fwd": 849.0}


def peaks() -> dict:
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return dict(tensor=float(d["bf16_tflops_sustained"]), hbm=float(d["hbm_gbs"]), src="measured")
    # NVIDIA H100 SXM data sheet (700 W): 989 TFLOP/s dense FP16 / BF16, 3.35 TB/s HBM3 -- not reached figures
    return dict(tensor=989.0, hbm=3350.0, src="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi sampler of the SM clock during the timed steps. It is started before the warm-up steps (nvidia-smi needs
    ~1 s before its first sample) and every line is time-stamped on arrival; `stop()` reports the samples that fall
    inside the timed region [mark_begin, mark_end]. If the timed region is too short to hold two samples, the
    samples of the warm-up + timed period (the GPU is under the same load) are used and `window` says so."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.proc, self.lines = index, None, []
        self.t0 = self.t1 = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._pump, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append((time.time(), line.strip()))

    def mark_begin(self):
        self.t0 = time.time()

    def mark_end(self):
        self.t1 = time.time()

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        t0 = self.t0 if self.t0 is not None else 0.0
        t1 = self.t1 if self.t1 is not None else time.time()
        inside = [ln for ts, ln in self.lines if t0 <= ts <= t1 + 0.15]
        window = "timed region"
        if len(inside) < 2:   # short run: fall back to everything sampled while the same steps were running
            inside = [ln for ts, ln in self.lines if ts <= t1 + 0.15]
            window = "warm-up + timed region (timed region shorter than two sampling periods)"
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in inside:
            f = [t.strip() for t in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])), mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "window": window, "reasons": sorted(reasons)}


def cpu_reference_rate(workload: str, steps: int, warmup: int, budget_s: float = 20.0) -> dict:
    """Time the CPU port of the reference path (oracle) with all host threads on a bounded sample."""
    from oracle import fastervit_oracle as O
    from oracle.configs import cfg_of
    import fastervit_b200 as F
    entry, kwargs, _, hw, mode = WORKLOADS[workload]
    cfg = cfg_of(ORACLE_CASE[workload])
    torch.manual_seed(0)
    model = F.create_model(entry, **{**kwargs, 'drop_path_rate': 0.0}).eval()  # parameter container only
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    bs = {"fv0_fwd": 16, "fv4_fwd": 4, "ar0_fwd": 2, "fv0_train": 8, "fv4_train": 2}[workload]
    x = O.synth_input(bs, hw, 1)
    tgt = torch.randint(0, 1000, (bs,), generator=torch.Generator().manual_seed(2))

    def run(xb, tb):
        if mode == "train":
            O.loss_and_grads(sd, cfg, xb, tb, training=True)
        else:
            with torch.no_grad():
                O.forward(sd, cfg, xb)
    # "all the host threads it can use": intra-op parallelism of torch CPU ops stops scaling (and
    # oversubscribes cgroup-limited containers) well before 100+ threads, so pick the fastest of a
    # few candidate thread counts on one small forward and report the count used
    cands = sorted({c for c in (avail, 64, 32, 16, 8) if 1 <= c <= avail})
    best, cores = None, cands[0]
    for c in cands:  # ascending; stop as soon as more threads stop helping (keeps the probe short)
        torch.set_num_threads(c)
        run(x[:1], tgt[:1])
        t0 = time.perf_counter()
        run(x[:1], tgt[:1])
        dt = time.perf_counter() - t0
        if best is None or dt < best:
            best, cores = dt, c
        elif dt > 1.3 * best:
            break
    torch.set_num_threads(cores)
    for _ in range(max(1, warmup)):
        run(x, tgt)
    t0 = time.perf_counter()
    n = 0
    while n < steps and (n == 0 or time.perf_counter() - t0 < budget_s):
        run(x, tgt)
        n += 1
    dt = time.perf_counter() - t0
    what = "train-mode forward + cross-entropy + autograd backward" if mode == "train" else "eval forward"
    return dict(value=bs * n / dt, unit="img/s", cores=cores, kind="port",
                sample=f"{entry} {what} (oracle port of the reference nn.Modules, fp32 torch CPU ops), "
                       f"batch {bs} x {n} iterations in {dt:.1f}s, {cores} threads",
                ms_per_step=1e3 * dt / n, steps_done=n, batch=bs)


def quick_measure(workload: str, dev, pk: dict, steps: int = 8, warmup: int = 3) -> dict:
    """One more BASELINE config measured in the same process (device-resident rotating inputs, CUDA events over
    `steps` steps after `warmup`), with the GEMM kernel's share and roofline fraction from the per-launch table.
    Used for the `also_measured` block so that the driver-run record covers every single-GPU config."""
    import gc
    import fastervit_b200 as F
    entry, kwargs, batch, hw, mode = WORKLOADS[workload]
    gc.collect()   # the previous workload's plans (CUDA graphs and their memory pools) sit in reference cycles
    torch.cuda.empty_cache()
    torch.manual_seed(0)
    model = F.create_model(entry, **kwargs).to(dev)
    model = model.train() if mode == "train" else model.eval()
    g = torch.Generator(device=dev).manual_seed(11)
    xs = [torch.randn(batch, 3, hw[0], hw[1], device=dev, generator=g) for _ in range(2)]
    targets = torch.randint(0, 1000, (batch,), device=dev, generator=g)

    def step(xb):
        if mode == "train":
            torch.nn.functional.cross_entropy(model(xb), targets).backward()
            model.zero_grad(set_to_none=True)
        else:
            model(xb)
    with torch.set_grad_enabled(mode == "train"):
        for i in range(warmup):
            step(xs[i % 2])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            step(xs[i % 2])
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    value = batch / (ms / 1e3)
    plan = next(iter(model._engine.plans.values()))
    with torch.no_grad():
        plan.profile(xs[0])
        prof = plan.profile(xs[1])
    gm_ms = sum(r["ms"] for r in prof if r["name"] == "fvit_gemm")
    gm_fl = sum(r["flops"] for r in prof if r["name"] == "fvit_gemm")
    tot = sum(r["ms"] for r in prof)
    simt = sum(r["ms"] for r in prof if r["name"] in ("fvit_attn_core_fwd", "fvit_attn_core_bwd"))
    alg = ALG_GFLOP_FWD.get(workload, 0.0) * 1e9   # (0: no algorithmic FLOP count in BASELINE.md for this config)
    out = {"workload": f"{entry} {'fwd+bwd' if mode == 'train' else 'forward'}, batch {batch}, 3x{hw[0]}x{hw[1]}",
           "value": round(value, 1), "unit": "img/s", "ms_per_step": round(ms, 4), "steps": steps, "warmup": warmup,
           "model_frac_of_tensor_peak": round(value * alg / 1e12 / pk["tensor"], 4) if alg else None,
           "gemm": {"share_of_step": round(gm_ms / tot, 4), "achieved_tflops": round(gm_fl / (gm_ms / 1e3) / 1e12, 1),
                    "frac": round(gm_fl / (gm_ms / 1e3) / 1e12 / pk["tensor"], 4)},
           "simt_attention_ms": round(simt, 4),
           "vs_baseline": round(value / PUBLISHED_IMG_S[workload], 3) if workload in PUBLISHED_IMG_S else None}
    if mode == "train":
        out["drop_path_rate"] = float(getattr(model, "drop_path_rate", 0.0))
    long_bwd = [r["ms"] for r in prof if r["name"] == "fvit_attn_loop_bwd_long"]
    if long_bwd:
        out["attn_loop_bwd_long"] = {"launches": len(long_bwd), "ms": round(sum(long_bwd), 4)}
    if batch <= 16 and mode == "fwd":
        # latency of ONE synchronous call through model(x) (host enqueue of the graph launch + device time + the wait)
        with torch.no_grad():
            lat = []
            for i in range(30):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model(xs[i % 2])
                torch.cuda.synchronize()
                lat.append((time.perf_counter() - t0) * 1e3)
        lat.sort()
        out["latency_ms"] = {"median": round(lat[len(lat) // 2], 4), "p10": round(lat[3], 4), "p90": round(lat[26], 4),
                             "what": "wall clock of one synchronous model(x) call, 30 calls"}
    del plan, model, xs
    gc.collect()
    torch.cuda.empty_cache()
    return out


def optimizer_leg(model, x, targets, pk) -> dict:
    """Time the fused optimizer step that follows backward in the reference loop (train.py:879-899): clip-grad-norm
    + LAMB (fv4-6) or AdamW (fv0-3) + ModelEmaV2, on the gradients of one real backward pass, CUDA events over
    10 steps after 3 warm-ups. Algorithmic bytes per parameter: sqnorm 4 + AdamW 28 (+8 fused EMA) or LAMB 40
    (+8); compared with the measured HBM peak."""
    from fastervit_b200 import optim as FO
    from fastervit_b200 import lib as L
    n_params = sum(p.numel() for p in model.parameters())
    use_lamb = n_params > 100e6   # TRAINING.md: `--opt lamb` for FasterViT-4/5/6, `--opt adamw` below
    out = {}
    for fused_ema in (True, False):
        opt = (FO.FusedLamb(model, lr=5e-3, weight_decay=0.12, max_grad_norm=1.0) if use_lamb
               else FO.FusedAdamW(model, lr=5e-4, weight_decay=0.05, max_grad_norm=5.0))
        ema = FO.FlatEma(model, decay=0.9998)
        if fused_ema:
            opt.attach_ema(ema, model)
        loss = torch.nn.functional.cross_entropy(model(x), targets)
        loss.backward()

        def one():
            opt.step()
            ema.update(model)
        for _ in range(3):
            one()
        torch.cuda.synchronize()
        L.reset_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        torch.cuda._sleep(int(3e8))   # ~150 ms spin: the 10 steps are enqueued behind it, so e0..e1 is device time
        e0.record()
        for _ in range(10):
            one()
        e1.record()
        host_ms = (time.perf_counter() - t0) * 1e3 / 10   # host enqueue cost per step (step() + ema.update())
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        bytes_per = 4 + (40 if use_lamb else 28) + (8 if fused_ema else 12)
        gbs = n_params * bytes_per / (ms / 1e3) / 1e9
        out["fused_ema" if fused_ema else "separate_ema"] = {
            "ms": round(ms, 4), "host_enqueue_ms": round(host_ms, 4), "launches": L.launch_count() / 10,
            "alg_bytes_per_param": bytes_per,
            "achieved_gbs": round(gbs, 1), "frac_of_hbm_peak": round(gbs / pk["hbm"], 4),
            "zero_copy_grads": opt._lay["gstage"] is None}
        model.zero_grad(set_to_none=True)
        del opt, ema
    return {"what": ("clip-grad-norm + " + ("LAMB" if use_lamb else "AdamW") + " + ModelEmaV2 update on the flat "
                     "gradient buffer (train.py:879-899), after the timed fwd+bwd steps; not part of `value`"),
            "params": n_params, "bound": "hbm", "peak_gbs": pk["hbm"], **out}


def dump_outputs(out_dir: Path, model, last: dict, mode: str, n_grad: int = 1 << 21) -> None:
    """What the last timed step handed its caller: the logits, and for a training step the loss and the parameter
    gradients. The gradients are sampled: n_grad positions of the concatenated gradients (model.parameters() order)
    drawn with a fixed seed, stored with their positions, so two builds can be compared element for element."""
    import numpy as np
    out_dir.mkdir(parents=True, exist_ok=True)
    np.save(out_dir / "logits.npy", last["logits"].float().cpu().numpy())
    if mode == "train":
        np.save(out_dir / "loss.npy", last["loss"].double().cpu().numpy().reshape(1))
        grads = [p.grad.detach().reshape(-1).float() if p.grad is not None else torch.zeros(p.numel(), device=p.device)
                 for p in model.parameters()]
        flat = torch.cat(grads)
        n = min(n_grad, flat.numel())
        idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(1234))[:n].sort().values
        np.save(out_dir / "grad_sample.npy", flat[idx.to(flat.device)].cpu().numpy())
        np.save(out_dir / "grad_sample_index.npy", idx.double().numpy())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", default="fv4_train", choices=sorted(ORACLE_CASE),
                    help="default: BASELINE.json configs[2]/[4] (the metric is fwd+bwd images/sec); fv0_fwd = configs[1]")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--batch", type=int, default=0, help="override the per-GPU batch")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-also", action="store_true", help="skip the also_measured block (other BASELINE configs)")
    ap.add_argument("--profile-out", default="", help="write the per-launch timing table (JSON) here")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps, write what the last timed step computed as DIR/<name>.npy (float32 / "
                         "float64): logits, and for training the loss and a fixed, seeded sample of the parameter "
                         "gradients")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    entry, kwargs, batch, hw, mode = WORKLOADS[args.workload]
    if args.batch:
        batch = args.batch
    what = ("fwd+bwd training step (train-mode BN, cross-entropy, no optimizer, drop_path_rate=0)" if mode == "train"
            else "forward-only (eval)")
    config = {"workload": f"{entry} {what}, batch {batch}/GPU, 3x{hw[0]}x{hw[1]} synthetic N(0,1), "
                          "random-init weights", "global_batch": batch * world,
              "parallelism": (f"dp{world}: batch sharded, NCCL all-reduce of the flat gradient buffer" if mode == "train"
                              else f"dp{world} replicas"),
              "l2": "inputs larger than L2 (rotating device batches; no explicit flush)"}

    # ------------------------------------------------------------------ reference arm (CPU)
    if args.impl == "reference":
        if rank != 0:
            return
        r = cpu_reference_rate(args.workload, args.steps, args.warmup, budget_s=120.0)
        # the config this arm really ran: the same model / mode / input shape / metric (img/s is batch-normalised), but
        # each step is a bounded sample of the workload -- a small batch on the host cores -- and it says so
        config = {"workload": f"{entry} {what}, 3x{hw[0]}x{hw[1]} synthetic N(0,1), random-init weights; CPU sample: "
                              f"batch {r['batch']} per step on {r['cores']} host threads (the GPU arm runs batch "
                              f"{batch}/GPU; a full batch is ~1 min per step on these cores)",
                  "global_batch": r["batch"], "parallelism": f"{r['cores']} CPU threads, 1 process",
                  "sample_of": f"batch {batch}/GPU workload of the GPU arm", "l2": "n/a (CPU)"}
        line = {"impl": "reference", "metric": "images/sec", "value": r["value"], "unit": "img/s",
                "n_gpus": args.gpus, "steps": r["steps_done"], "warmup": args.warmup,
                "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "fp32", "data": "synthetic", "config": config,
                "cpu_baseline": {k: r[k] for k in ("value", "unit", "cores", "kind", "sample")},
                "e2e": {"value": r["value"], "unit": "img/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        print(json.dumps(line))
        return

    # ------------------------------------------------------------------ GPU arm
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the CUDA path has no CPU fallback; use --impl reference)")
    import fastervit_b200 as F
    from fastervit_b200 import lib as L
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
            os.environ["NCCL_DEBUG"] = "WARN"   # keep NCCL's version banner off stdout (one JSON line contract)
        # NCCL's CTAs cannot share an SM with a GEMM CTA: keep their number small and known, the backward launches in
        # the shadow of an all-reduce are capped to (SM count) - FVIT_NCCL_CTAS SMs (engine_train._allreduce_shadow)
        os.environ.setdefault("NCCL_MAX_CTAS", os.environ.get("FVIT_NCCL_CTAS", "16"))
        dist.init_process_group("nccl", device_id=dev)

    torch.manual_seed(0)
    model = F.create_model(entry, **kwargs).to(dev)
    model = model.train() if mode == "train" else model.eval()
    if mode == "train" and dist is not None:
        model.enable_grad_allreduce()
    nbuf = 2
    g = torch.Generator(device=dev).manual_seed(1 + rank)
    xs = [torch.randn(batch, 3, hw[0], hw[1], device=dev, generator=g) for _ in range(nbuf)]

    def sync_all():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()

    targets = torch.randint(0, 1000, (batch,), device=dev, generator=g)

    last = {}

    def step(xb, keep=False):
        if mode == "train":
            logits = model(xb)
            loss = torch.nn.functional.cross_entropy(logits, targets)
            loss.backward()
            if keep:   # the last timed step: its gradients stay in place for --dump-outputs
                last.update(logits=logits.detach(), loss=loss.detach())
            else:
                model.zero_grad(set_to_none=True)
            return loss
        out = model(xb)
        if keep:
            last["logits"] = out
        return out

    sampler = ClockSampler(local_rank)
    sampler.start()   # before the warm-up: nvidia-smi takes about a second to deliver its first sample
    with torch.set_grad_enabled(mode == "train"):
        for i in range(args.warmup):
            step(xs[i % nbuf])
        sync_all()
        sampler.mark_begin()
        L.reset_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            out = step(xs[i % nbuf], keep=bool(args.dump_outputs) and i == args.steps - 1)
        e1.record()
        sync_all()
        sampler.mark_end()
        launches = L.launch_count()
        ms = e0.elapsed_time(e1)
        clocks = sampler.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(Path(args.dump_outputs), model, last, mode)
    if mode == "train":
        model.zero_grad(set_to_none=True)
    t = torch.tensor([ms], device=dev)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total = t.item()
    grad_sync = None
    if mode == "train" and dist is not None:
        # after the all-reduce every rank must hold the same averaged gradient although the inputs differ
        loss = torch.nn.functional.cross_entropy(model(xs[0]), targets)
        loss.backward()
        digest = torch.stack([torch.cat([p.grad.flatten()[:64] for p in model.parameters()]).double().sum(),
                              sum(p.grad.double().abs().sum() for p in model.parameters())])
        both = [torch.empty_like(digest) for _ in range(world)]
        dist.all_gather(both, digest)
        grad_sync = bool(all(torch.allclose(b, both[0], rtol=1e-6, atol=0) for b in both))
        model.zero_grad(set_to_none=True)
    value = batch * world * args.steps / (ms_total / 1e3)

    # ------------------------------------------------------------------ end to end (host buffers)
    e2e = None
    if not args.no_e2e:
        host_in = [torch.randn(batch, 3, hw[0], hw[1]).pin_memory() for _ in range(2)]
        host_out = torch.empty(batch, model.num_classes).pin_memory()
        dev_in = [torch.empty(batch, 3, hw[0], hw[1], device=dev) for _ in range(2)]
        copy_stream = torch.cuda.Stream(device=dev)
        steps_e = max(3, min(args.steps, 10))

        def e2e_loop(n):
            # prefetch on a side stream (what timm's PrefetchLoader does for train.py / validate.py),
            # forward on the current stream, logits back to pinned host memory every step
            ready = [torch.cuda.Event(), torch.cuda.Event()]
            done = [torch.cuda.Event(), torch.cuda.Event()]
            with torch.cuda.stream(copy_stream):
                dev_in[0].copy_(host_in[0], non_blocking=True)
                ready[0].record(copy_stream)
            for i in range(n):
                cur, nxt = i % 2, (i + 1) % 2
                if i + 1 < n:
                    with torch.cuda.stream(copy_stream):
                        if i >= 1:
                            copy_stream.wait_event(done[nxt])
                        dev_in[nxt].copy_(host_in[nxt], non_blocking=True)
                        ready[nxt].record(copy_stream)
                torch.cuda.current_stream().wait_event(ready[cur])
                res = step(dev_in[cur])
                done[cur].record()
                if mode == "train":
                    host_loss.copy_(res.detach().reshape(1), non_blocking=True)
                else:
                    host_out.copy_(res, non_blocking=True)
            torch.cuda.synchronize()

        host_loss = torch.empty(1).pin_memory()
        with torch.set_grad_enabled(mode == "train"):
            e2e_loop(2)
            sync_all()
            t0 = time.perf_counter()
            e2e_loop(steps_e)
            dt = time.perf_counter() - t0
        t = torch.tensor([dt], device=dev)
        if dist is not None:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e = {"value": batch * world * steps_e / t.item(), "unit": "img/s",
               "h2d_bytes_per_step": batch * 3 * hw[0] * hw[1] * 4,
               "d2h_bytes_per_step": 4 if mode == "train" else batch * model.num_classes * 4,
               "steps": steps_e, "note": "pinned host input uploaded on a prefetch stream, "
                                         + ("loss" if mode == "train" else "logits") + " copied back, wall clock"}

    # ------------------------------------------------------------------ roofline of the dominant kernel
    pk = peaks()
    roofline = None
    prof_table = None
    if rank == 0:
        plan = next(iter(model._engine.plans.values()))
        with torch.no_grad():
            plan.profile(xs[0])
            prof = plan.profile(xs[1])
        by = {}
        for r in prof:
            d = by.setdefault(r["name"], dict(ms=0.0, n=0, flops=0.0))
            d["ms"] += r["ms"]
            d["n"] += 1
            d["flops"] += r["flops"]
        tot = sum(d["ms"] for d in by.values())
        gm = by.get("fvit_gemm")
        prof_table = {k: dict(ms=round(v["ms"], 4), launches=v["n"], share=round(v["ms"] / tot, 4),
                              gflop=round(v["flops"] / 1e9, 3)) for k, v in sorted(by.items(), key=lambda kv: -kv[1]["ms"])}
        if gm:
            ach = gm["flops"] / (gm["ms"] / 1e3) / 1e12
            roofline = {"kernel": "gemm_wgmma_kernel (fvit_gemm: conv taps + linear layers; fwd, dgrad and wgrad launches)",
                        "bound": "tensor",
                        "achieved": round(ach, 2), "peak": pk["tensor"], "unit": "TFLOP/s",
                        "frac": round(ach / pk["tensor"], 4),
                        "traffic": None, "traffic_unit": "DRAM bytes per launch: not measured",
                        "peak_source": f"{pk['src']} (bf16 dense)",
                        "launches_per_step": gm["n"], "avg_launch_ms": round(gm["ms"] / gm["n"], 5),
                        "alg_gflop_per_launch": round(gm["flops"] / gm["n"] / 1e9, 3),
                        "share_of_step": round(gm["ms"] / tot, 4)}
        if args.profile_out:
            Path(args.profile_out).write_text(json.dumps({"per_kernel": prof_table, "launches": prof}, indent=1))

    # ------------------------------------------------------------------ optimizer step (SURVEY §8 f.1), reported
    # beside the metric (the BASELINE metric is fwd+bwd; the optimizer is NOT inside `value` / `e2e`)
    opt_info = None
    if rank == 0 and mode == "train" and world == 1:   # (with N > 1 a lone backward would wait on the all-reduce)
        try:
            opt_info = optimizer_leg(model, xs[0], targets, pk)
        except Exception as exc:  # the headline line must survive a failure of this side measurement
            opt_info = {"error": f"{type(exc).__name__}: {exc}"}

    # ------------------------------------------------------------------ CPU baseline (rank 0, N == 1)
    cpu = None
    if rank == 0 and world == 1:
        # bounded sample of the reference path on the host cores (FVIT_BENCH_CPU_BUDGET_S: seconds, default 15)
        cpu = cpu_reference_rate(args.workload, steps=1000, warmup=1,
                                 budget_s=float(os.environ.get("FVIT_BENCH_CPU_BUDGET_S", "15")))
        cpu = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}

    # ------------------------------------------------------------------ the other single-GPU BASELINE configs
    also = None
    if rank == 0 and world == 1 and not args.no_also and args.workload == "fv4_train":
        del model, xs
        torch.cuda.empty_cache()
        also = {}
        for wl in ("fv0_fwd", "fv0_train", "ar0_fwd", "fv4_fwd", "fv4_train_droppath", "fv0_fwd_b8", "fv4_21k_384_train"):
            try:
                also[wl] = quick_measure(wl, dev, pk)
            except Exception as exc:  # a side measurement must not take the headline line down
                also[wl] = {"error": f"{type(exc).__name__}: {exc}"}

    if rank == 0:
        alg = ALG_GFLOP_FWD[args.workload] * 1e9
        line = {"metric": "images/sec", "value": round(value, 2), "unit": "img/s", "n_gpus": world,
                "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_total / args.steps, 4),
                "higher_is_better": True, "scaling": "weak",
                "vs_baseline": (round(value / world / PUBLISHED_IMG_S[args.workload], 3)
                                if args.workload in PUBLISHED_IMG_S else None),
                "dtype": "fp16 operands, fp32 accumulate / residual / statistics", "data": "synthetic",
                "config": config, "e2e": e2e, "gpu_launches": int(launches),
                "launches_per_step": launches / args.steps, "clocks": clocks, "roofline": roofline,
                "cpu_baseline": cpu, "optimizer_step": opt_info, "also_measured": also, "per_kernel": prof_table,
                "grad_sync_check": grad_sync,
                "data_parallel": ({"grad_buckets": len(getattr(plan, "grad_buckets", [])),
                                   "allreduce_busbw_gbs": round(getattr(plan, "ar_busbw", 0.0) / 1e9, 1),
                                   "nccl_max_ctas": os.environ.get("NCCL_MAX_CTAS"),
                                   "sm_capped_launches": len(getattr(plan, "_ar_shadow", None) or {})}
                                  if world > 1 and mode == "train" else None),
                "model_tflops": round(value * alg / 1e12, 2),
                "model_frac_of_tensor_peak": round(value / world * alg / 1e12 / pk["tensor"], 4)}
        print(json.dumps(line))
    if dist is not None:
        # orderly teardown with a watchdog: release the captured launch lists first, and never let a stuck
        # communicator teardown keep the ranks alive after the result line is out
        sys.stdout.flush()
        import gc
        try:
            for plan in list(model._engine.plans.values()):
                plan._graphs.clear()
        except Exception:  # noqa: BLE001
            pass
        gc.collect()
        torch.cuda.synchronize()
        killer = threading.Timer(30.0, lambda: os._exit(0))
        killer.daemon = True
        killer.start()
        dist.destroy_process_group()
        killer.cancel()


if __name__ == "__main__":
    main()
