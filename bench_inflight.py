"""Clips in flight against checkpointed clips: MOTRv2's tracking-backbone recipe (faster_vit_4_21k_224, frozen-BatchNorm
stem, LayerNorm2d level norms, batch 1 at 800 x 1536; fastervit_b200.tracking) trained on clips of 2 ... 5 frames.

    python bench_inflight.py [--rounds 3] [--reps 3] [--probe-max 12]

Arms, per clip length L (fixed pre-made map gradients, one backward of sum_f sum_k <map_fk, G_fk>, no optimizer):
  * checkpointed: frames 0 ... L-2 through torch.utils.checkpoint (reentrant) -- forwards under no_grad, recomputed
    inside the backward -- and the last frame plain, on the default single train plan instance; the backbone part of
    MOTRv2's --use_checkpoint recipe;
  * in flight: L grad-enabled forwards, then the backward, with set_train_forwards_in_flight(5) (L instances in use).
The arms alternate within each round; each timing is the median of --reps clips (CUDA events), the result the median over
--rounds rounds. Peak allocated memory is read over one clip of each arm, with both models resident. Then, with the
checkpointed model freed, the in-flight model takes clips of 6, 7, ... frames (n = L, eager launches for the new
instances) until an allocation fails or --probe-max: where the activation sets stop fitting on the card. The card name
and power limit are read in the same process. Prints one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics

import torch
from torch.utils.checkpoint import checkpoint

from bench_track import H, W, _layernorm2d, card

GIB = 2 ** 30


def model(n: int):
    from fastervit_b200.tracking import FrozenBatchNorm2d, build_fastervit
    torch.manual_seed(0)
    m = build_fastervit("faster_vit_4_21k_224", FrozenBatchNorm2d, _layernorm2d()).cuda().train()
    return m.set_train_forwards_in_flight(n)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--probe-max", type=int, default=12)
    a = ap.parse_args()
    lengths = (2, 3, 4, 5)
    gen = torch.Generator(device="cuda").manual_seed(0)
    frames = [torch.randn(1, 3, H, W, device="cuda", generator=gen) for _ in range(max(a.probe_max, 5))]
    ck, fl = model(1), model(5)
    fl.load_state_dict(ck.state_dict())
    with torch.no_grad():
        shapes = [o.shape for o in ck.forward_raw(frames[0])]
    grads = [torch.randn(s, device="cuda", generator=gen) for s in shapes]
    dummy = torch.zeros(1, device="cuda", requires_grad=True)   # (makes the checkpointed outputs require grad)

    def loss(maps) -> torch.Tensor:
        return sum((o * g).sum() for mm in maps for o, g in zip(mm, grads))

    def clip_ck(L: int) -> None:
        maps = [checkpoint(lambda f, _d: ck.forward_raw(f), f, dummy, use_reentrant=True) for f in frames[:L - 1]]
        maps.append(ck.forward_raw(frames[L - 1]))
        loss(maps).backward()

    def clip_fl(L: int) -> None:
        loss([fl.forward_raw(f) for f in frames[:L]]).backward()

    arms = {"checkpointed": clip_ck, "in_flight": clip_fl}

    def timed(fn, L: int) -> float:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * a.reps)]
        for i in range(a.reps):
            ev[2 * i].record()
            fn(L)
            ev[2 * i + 1].record()
        torch.cuda.synchronize()
        return statistics.median(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(a.reps))

    resident = {}
    for L in lengths:   # warm-up: instances built, weights packed, graphs captured
        for name, fn in arms.items():
            for _ in range(3):
                fn(L)
        torch.cuda.synchronize()
        resident[L] = round(torch.cuda.memory_allocated() / GIB, 2)
    times = {f"{name}_{L}": [] for L in lengths for name in arms}
    for _ in range(a.rounds):
        for L in lengths:
            for name, fn in arms.items():
                times[f"{name}_{L}"].append(timed(fn, L))
    peak = {}
    for L in lengths:
        for name, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            fn(L)
            torch.cuda.synchronize()
            peak[f"{name}_{L}"] = round(torch.cuda.max_memory_allocated() / GIB, 2)
    pools = {name: [len(p) for p in m._get_engine().pools.values()] for name, m in (("checkpointed", ck), ("in_flight", fl))}

    # where the activation sets stop fitting: the checkpointed model freed, clips of growing length in flight
    del ck, arms, clip_ck
    gc.collect()
    torch.cuda.empty_cache()
    os.environ["FVIT_CUDA_GRAPH"] = "0"    # (new instances launch eagerly: no capture pools in the probe)
    probe, fits = {}, 5
    for L in range(5, a.probe_max + 1):
        fl.set_train_forwards_in_flight(L)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        try:
            clip_fl(L)
            torch.cuda.synchronize()
        except torch.cuda.OutOfMemoryError:
            probe[L] = "out of memory"
            break
        probe[L] = round(torch.cuda.max_memory_allocated() / GIB, 2)
        fits = L
    fl.zero_grad(set_to_none=True)
    res = dict(card(), shape=[1, 3, H, W], model="faster_vit_4_21k_224 (Frozen, LN)",
               ms={k: round(statistics.median(v), 2) for k, v in times.items()},
               rounds_ms={k: [round(t, 2) for t in v] for k, v in times.items()},
               peak_gib_both_models_resident=peak, resident_gib_after_warmup=resident, pools=pools,
               in_flight_probe_peak_gib=probe, longest_clip_in_flight_that_fits=fits,
               total_gib=round(torch.cuda.get_device_properties(0).total_memory / GIB, 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
