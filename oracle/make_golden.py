"""Generate tests/golden/*.pt from the UNMODIFIED reference (a checkout of NVlabs/FasterViT).

    FASTERVIT_REFERENCE=<path to the reference checkout> python oracle/make_golden.py [case ...]

Imports <reference>/fastervit behind the 5-symbol timm stand-in (oracle/ref_shim), fills the
reference model's own state_dict with deterministic synthetic weights (oracle synth_fill_), runs the
reference module in fp64 (eval forward; train-mode forward + CrossEntropy backward, drop_path_rate=0)
and stores logits, loss, per-level activation samples and per-parameter gradient samples. It also runs
the oracle restatement on the same weights and asserts agreement, which is what pins the oracle.
The tests never need the reference: they read only the committed fixtures.
"""
from __future__ import annotations

import os
import sys
import time
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "ref_shim"))
_REF = os.environ.get("FASTERVIT_REFERENCE")
if not _REF or not Path(_REF, "fastervit").is_dir():
    raise SystemExit("make_golden.py: set FASTERVIT_REFERENCE to a checkout of NVlabs/FasterViT")
sys.path.insert(0, _REF)
warnings.filterwarnings("ignore")

from oracle import fastervit_oracle as O  # noqa: E402
from oracle.configs import CASES  # noqa: E402

SEED_W, SEED_X, SEED_T = 1234, 1, 2
GOLDEN = ROOT / "tests" / "golden"
MAX_SAMPLE = 512
GRAD_SAMPLE_STEP = {"fv4": 2}  # 649 gradient tensors: half of each strided sample


def sample(t: torch.Tensor) -> torch.Tensor:
    """Deterministic strided subsample (<= MAX_SAMPLE values) of a tensor, stored as fp32."""
    f = t.detach().flatten()
    stride = max(1, (f.numel() + MAX_SAMPLE - 1) // MAX_SAMPLE)
    return f[::stride].float().clone()


def summarize(t: torch.Tensor) -> dict:
    return {"shape": tuple(t.shape), "l2": t.detach().double().norm().item(),
            "amax": t.detach().double().abs().max().item(), "sample": sample(t)}


def batch_for(case: str) -> tuple[int, int]:
    """(eval batch, train batch)"""
    return {"fv0": (2, 2), "fv4": (1, 2), "ar0": (1, 0), "tiny_a": (2, 3), "tiny_qk": (2, 3), "tiny_b": (2, 3),
            "tiny_ar": (2, 2), "tiny_ar85": (2, 2), "tiny_ar68": (2, 2), "tiny_ar148": (1, 2), "tiny_21k": (2, 2), "tiny_21k224": (2, 3)}[case]


def run_case(case: str) -> None:
    import fastervit  # the reference package
    entry, kwargs, cfg = CASES[case]
    t0 = time.time()
    model = fastervit.create_model(entry, drop_path_rate=0.0, **kwargs).double()
    sd = model.state_dict()
    O.synth_fill_(sd, SEED_W)  # in place: state_dict tensors alias the module's storage
    res = cfg["resolution"]
    b_eval, b_train = batch_for(case)
    out: dict = {"case": case, "entry": entry, "kwargs": kwargs, "cfg": cfg,
                 "seeds": {"w": SEED_W, "x": SEED_X, "t": SEED_T},
                 "n_params": sum(p.numel() for p in model.parameters()),
                 "state_keys": [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]}

    # ---- eval forward (the validate.py:291-298 path)
    x = O.synth_input(b_eval, res, SEED_X, torch.float64)
    model.eval()
    acts: dict = {}
    hooks = []
    for name, mod in model.named_modules():
        if name == "patch_embed" or (name.startswith("levels.") and name.count(".") == 1) or name == "norm" \
                or (name.count(".") == 3 and ".blocks." in name):
            hooks.append(mod.register_forward_hook(
                lambda m, i, o, name=name: acts.__setitem__(name, o[0] if isinstance(o, tuple) else o)))
    with torch.no_grad():
        logits = model(x)
    for h in hooks:
        h.remove()
    out["eval"] = {"batch": b_eval, "logits": logits.clone(),
                   "acts": {k: summarize(v) for k, v in acts.items()}}
    # fp32 reference vs fp64 reference: the reference's own noise floor
    m32 = fastervit.create_model(entry, drop_path_rate=0.0, **kwargs)
    m32.load_state_dict({k: (v.float() if v.is_floating_point() else v) for k, v in sd.items()})
    m32.eval()
    with torch.no_grad():
        l32 = m32(x.float())
    out["eval"]["ref_fp32_vs_fp64"] = ((l32.double() - logits).abs().max() / logits.abs().max()).item()
    del m32

    # ---- oracle vs reference (eval)
    sd_o = {k: v.clone() for k, v in sd.items()}
    with torch.no_grad():
        lo = O.forward(sd_o, cfg, x, training=False)
    err = ((lo - logits).abs().max() / logits.abs().max()).item()
    out["eval"]["oracle_vs_ref"] = err
    assert err < 1e-9, f"{case}: oracle eval logits differ from the reference by {err:.3e}"

    # ---- train-mode forward + backward
    if b_train > 0:
        xt = O.synth_input(b_train, res, SEED_X + 100, torch.float64)
        gt = torch.Generator().manual_seed(SEED_T)
        target = torch.randint(0, 1000, (b_train,), generator=gt)
        model.train()
        model.zero_grad()
        lt = model(xt)
        loss = torch.nn.functional.cross_entropy(lt, target)
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
        new_sd = model.state_dict()
        bn_after = {k: new_sd[k].clone() for k in new_sd if k.endswith(("running_mean", "running_var"))}
        out["train"] = {"batch": b_train, "target": target, "logits": lt.detach().clone(),
                        "loss": loss.item(), "grads": {k: summarize(g) for k, g in grads.items()},
                        "bn_after": {k: summarize(v) for k, v in bn_after.items()}}
        # every GRAD_SAMPLE_STEP-th point of each gradient sample (the fixture stays under 1 MB)
        step = GRAD_SAMPLE_STEP.get(case, 1)
        if step > 1:
            for d in out["train"]["grads"].values():
                d["sample"] = d["sample"][::step].clone()
            out["train"]["grad_sample_step"] = step
        lo_loss, lo_logits, lo_grads = O.loss_and_grads(sd_o, cfg, xt, target, training=True)
        e1 = ((lo_logits - lt.detach()).abs().max() / lt.detach().abs().max()).item()
        # analytically-zero gradients (biases feeding a train-mode BatchNorm, the key bias of a
        # softmax) are pure rounding noise in any implementation: compare against a global floor
        floor = 1e-6 * max(g.norm().item() for g in grads.values())
        out["train"]["grad_floor"] = floor
        worst = 0.0
        for k, g in grads.items():
            assert k in lo_grads, f"oracle produced no grad for {k}"
            e = ((lo_grads[k] - g).norm() / g.norm().clamp_min(floor)).item()
            worst = max(worst, e)
        out["train"]["oracle_vs_ref"] = {"logits": e1, "grads_worst_rel_l2": worst}
        assert e1 < 1e-9 and worst < 1e-7, f"{case}: oracle train parity {e1:.3e} / {worst:.3e}"

    GOLDEN.mkdir(parents=True, exist_ok=True)
    path = GOLDEN / f"{case}.pt"
    torch.save(out, path, _use_new_zipfile_serialization=False)  # (the legacy format has no per-tensor padding)
    print(f"{case}: {path.name} {path.stat().st_size / 1024:.0f} KiB, params {out['n_params']:,}, "
          f"oracle-vs-ref eval {err:.2e}"
          + (f", train logits {out['train']['oracle_vs_ref']['logits']:.2e}, grads "
             f"{out['train']['oracle_vs_ref']['grads_worst_rel_l2']:.2e}" if b_train else "")
          + f", ref fp32-vs-fp64 {out['eval']['ref_fp32_vs_fp64']:.2e}, {time.time() - t0:.1f}s", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(8)
    cases = sys.argv[1:] or list(CASES)
    for c in cases:
        run_case(c)
