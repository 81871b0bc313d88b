"""GPU parity of the training path (train-mode forward with batch-statistics BatchNorm + full backward)
against the reference's fp64 outputs/gradients stored in tests/golden/*.pt (drop_path_rate = 0).

Tolerances: logits 2e-3 max-rel (train-mode BN at batch 2-3 amplifies the fp16-operand noise slightly),
loss 1e-4 relative, BN running statistics 1e-3; parameter gradients: relative L2-norm error of the sampled
values <= 4e-2 and max element error <= 8e-2 of max(|g|_max, 1e-3 * global max) — fp16 operands with fp32
accumulation through ~50 layers; analytically-zero gradients (biases feeding a BatchNorm) are compared
against the global floor."""
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"


def _run(case):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    tr = g["train"]
    model = F.create_model(g["entry"], drop_path_rate=0.0, **g["kwargs"])
    O.synth_fill_(model.state_dict(), g["seeds"]["w"])
    model = model.cuda().train()
    x = O.synth_input(tr["batch"], g["cfg"]["resolution"], g["seeds"]["x"] + 100, torch.float32).cuda()
    logits = model(x)
    loss = torch.nn.functional.cross_entropy(logits, tr["target"].cuda())
    loss.backward()
    torch.cuda.synchronize()
    return g, tr, model, logits, loss


def _sample(t, n=512):
    f = t.detach().flatten()
    stride = max(1, (f.numel() + n - 1) // n)
    return f[::stride].float().cpu()


@pytest.mark.parametrize("case", ["tiny_a", "tiny_qk", "tiny_b", "tiny_ar", "tiny_ar85", "tiny_ar68", "tiny_ar148", "tiny_21k224", "tiny_21k", "fv0",
                                  "fv4"])
def test_train_step_matches_reference(case):
    g, tr, model, logits, loss = _run(case)
    ref = tr["logits"].to(logits.device)
    # train-mode logits pass through batch-statistics BatchNorms (fp16 operand noise is renormalised at every
    # block), measured 0.6e-3 .. 2.0e-3 across the cases; the eval-mode 1e-3 bar is tests/test_model_gpu.py
    assert ((logits.double() - ref).abs().max() / ref.abs().max()).item() < 3e-3
    assert abs(loss.item() - tr["loss"]) < 1e-4 * abs(tr["loss"]) + 1e-4
    sd = model.state_dict()
    for k, want in tr["bn_after"].items():
        d = (_sample(sd[k]) - want["sample"]).abs().max().item()
        assert d <= 1e-3 * max(want["amax"], 1e-6) + 1e-6, (k, d)
    gmax = max(w["amax"] for w in tr["grads"].values())
    bad, l2s = [], []
    for k, p in model.named_parameters():
        want = tr["grads"][k]
        assert p.grad is not None and tuple(p.grad.shape) == tuple(want["shape"]), k
        smp = _sample(p.grad)[::tr.get("grad_sample_step", 1)]
        floor = max(want["amax"], 1e-3 * gmax)
        emax = (smp - want["sample"]).abs().max().item() / floor
        el2 = (smp - want["sample"]).norm().item() / max(want["sample"].norm().item(), 1e-3 * gmax * smp.numel() ** 0.5)
        l2s.append(el2)
        # the stem sits at the end of the backward chain and its BatchNorm biases are sums over >= 1e5 positions of
        # sign-cancelling terms: the fp16-operand arithmetic model alone (oracle quant="fp16", fp32 backward) gives
        # 3.4e-2 / 3.7e-2 relative L2 on patch_embed.conv_down.1.bias for tiny_ar85 / tiny_ar148, so the stem gets
        # 6e-2 where every other tensor has 4e-2
        l2_cap = 6e-2 if k.startswith("patch_embed.") else 4e-2
        if emax > 8e-2 or el2 > l2_cap:
            bad.append((k, emax, el2))
    assert not bad, bad[:10]
    # the ceilings above are set by a handful of ill-conditioned tensors (tiny-batch BatchNorm biases); the bulk of
    # the gradients must sit at the fp16-operand noise floor. Measured medians: 0.6e-3 .. 1.4e-3 on the reduced
    # models, 2.2e-3 on fv0, 3.0e-3 on fv4 (649 tensors, 35 layers of fp16 activation gradients): bound 4e-3
    med = sorted(l2s)[len(l2s) // 2]
    print(f"{case}: {len(l2s)} gradients, median rel-L2 {med:.2e}, worst {max(l2s):.2e}")
    assert med <= 4e-3, med


def test_backward_of_a_stale_forward_raises():
    """Two train-mode forwards of the same shape share the plan's saved-activation buffers: differentiating the
    first after the second ran must raise instead of returning gradients of mixed state; so must an input that
    requires grad (no image gradient is produced)."""
    from fastervit_b200.lib import FvitError
    g, tr, model, logits, loss = _run("tiny_a")
    from oracle import fastervit_oracle as O
    x = O.synth_input(tr["batch"], g["cfg"]["resolution"], 9, torch.float32).cuda()
    l1 = model(x).sum()
    l2 = model(x * 0.5).sum()
    with pytest.raises(FvitError):
        l1.backward()
    l2.backward()      # the latest forward is still differentiable
    with pytest.raises(FvitError):
        model(x.clone().requires_grad_(True))


def test_second_step_and_grad_accumulation_semantics():
    """Two consecutive steps give independent, correct gradients (buffers are re-zeroed) and gradients of
    repeated backward calls accumulate into .grad like any autograd function."""
    g, tr, model, logits, loss = _run("tiny_a")
    g1 = {k: p.grad.clone() for k, p in model.named_parameters()}
    from oracle import fastervit_oracle as O
    x = O.synth_input(tr["batch"], g["cfg"]["resolution"], g["seeds"]["x"] + 100, torch.float32).cuda()
    # running stats changed after step 1, but train-mode outputs only depend on batch statistics
    logits2 = model(x)
    loss2 = torch.nn.functional.cross_entropy(logits2, tr["target"].cuda())
    loss2.backward()   # accumulates: .grad should now be ~2x
    gmax = max(v.abs().max().item() for v in g1.values())
    gmax_ref = max(w["amax"] for w in tr["grads"].values())
    for k, p in model.named_parameters():
        ref = 2 * g1[k]
        if tr["grads"][k]["amax"] < 1e-4 * gmax_ref:
            continue  # analytically zero (conv bias ahead of a train-mode BatchNorm): pure rounding noise
        # split-K / reduction atomics make the summation order (not the math) run-dependent
        tol = 2e-2 * max(ref.abs().max().item(), 1e-2 * gmax)
        assert (p.grad - ref).abs().max().item() <= tol, k
    model.zero_grad(set_to_none=True)
    # batch statistics are summed with atomics: their last-bit differences flip fp16 roundings downstream, so two
    # runs agree to the fp16 noise floor (same size as the parity tolerance), not bitwise
    d = (logits2 - logits).abs().max().item()
    assert d <= 2e-3 * logits.abs().max().item(), d


def test_train_then_eval_uses_running_stats():
    g, tr, model, logits, loss = _run("tiny_a")
    model.eval()
    from oracle import fastervit_oracle as O
    x = O.synth_input(2, g["cfg"]["resolution"], 5, torch.float32).cuda()
    with torch.no_grad():
        out = model(x)
        ref = O.forward({k: v.detach().cpu().clone() for k, v in model.state_dict().items()}, g["cfg"], x.cpu())
    assert ((out.cpu() - ref).abs().max() / ref.abs().max()).item() < 1e-3


def test_stochastic_depth_matches_oracle_with_explicit_masks():
    """DropPath (timm semantics: one Bernoulli draw per window / per image, scaled by 1/keep). The RNG is
    not reproducible across implementations, so the same explicit masks are forced into the kernels and fed
    to the fp64 oracle; logits and gradients must agree."""
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import cfg_of
    kw = dict(dim=24, in_dim=16, depths=[1, 2, 2, 2], num_heads=[1, 2, 8, 16])
    cfg = dict(cfg_of("tiny_b"))
    model = F.create_model("faster_vit_4_224", drop_path_rate=0.3, **kw)
    O.synth_fill_(model.state_dict(), 4321)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    model = model.cuda().train()
    B = 3
    x = O.synth_input(B, 224, 77, torch.float32)
    target = torch.tensor([5, 900, 17])
    plan = model._get_engine()._plan(x.cuda())
    g = torch.Generator().manual_seed(5)
    masks = {}
    for d in plan.drop_specs:
        m = torch.bernoulli(torch.full((d["groups"],), d["keep"]), generator=g) / d["keep"]
        masks[d["name"]] = m
    assert any((m == 0).any() for m in masks.values()) and len(masks) >= 10
    plan.forced_drop_masks = masks
    logits = model(x.cuda())
    loss = torch.nn.functional.cross_entropy(logits, target.cuda())
    loss.backward()
    ref_loss, ref_logits, ref_grads = O.loss_and_grads(sd64, cfg, x.double(), target, training=True,
                                                       drop_masks={k: v.double() for k, v in masks.items()})
    assert ((logits.double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 2e-3
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    for k, p in model.named_parameters():
        want = ref_grads[k]
        err = (p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5)
        assert err < 4e-2, (k, err)


def test_gradient_buckets_partition_the_flat_buffer():
    """The data-parallel buckets (issued as the backward pass finishes them) tile the flat gradient buffer, fall
    on parameter boundaries and are listed last-level-first."""
    g, tr, model, logits, loss = _run("tiny_a")
    plan = next(p for p in model._get_engine().plans.values() if p.training)
    total = plan.gflat.numel()     # parameter slices are padded to 256-byte boundaries
    assert sorted(plan.grad_buckets) == sorted(set(plan.grad_buckets))
    covered = sorted(plan.grad_buckets)
    assert covered[0][0] == 0 and covered[-1][1] == total
    for (a0, a1), (b0, b1) in zip(covered, covered[1:]):
        assert a1 == b0
    offs = set(plan._goff.values()) | {total}
    assert all(lo in offs and hi in offs for lo, hi in plan.grad_buckets)
    assert plan.grad_buckets[0][1] == total and plan.grad_buckets[-1][0] == 0
    # every parameter's slice lies inside exactly one bucket
    for p in model.parameters():
        o = plan._goff[id(p)]
        assert sum(1 for lo, hi in plan.grad_buckets if lo <= o and o + p.numel() <= hi) == 1


def test_train_step_with_num_classes_not_a_multiple_of_four():
    """The loss gradient is kept in 16-byte padded rows, so any `num_classes` trains (a 10-class fine-tuning head):
    loss, logits and every gradient against the fp64 oracle."""
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import cfg_of
    kw = dict(dim=32, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8], num_classes=10)
    model = F.create_model("faster_vit_0_224", drop_path_rate=0.0, **kw)
    O.synth_fill_(model.state_dict(), 99)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    model = model.cuda().train()
    x = O.synth_input(3, 224, 12, torch.float32)
    target = torch.tensor([3, 9, 0])
    logits = model(x.cuda())
    assert logits.shape == (3, 10)
    loss = torch.nn.functional.cross_entropy(logits, target.cuda())
    loss.backward()
    ref_loss, ref_logits, ref_grads = O.loss_and_grads(sd64, cfg_of("tiny_a"), x.double(), target, training=True)
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item()) + 1e-4
    assert ((logits.double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 3e-3
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    for k, p in model.named_parameters():
        want = ref_grads[k]
        err = (p.grad.double().cpu() - want).norm().item() / max(want.norm().item(), 1e-3 * gmax * want.numel() ** 0.5)
        assert err < (6e-2 if k.startswith("patch_embed.") else 4e-2), (k, err)


def test_stochastic_depth_draws_fresh_masks_inside_the_captured_step():
    """With drop_path_rate > 0 the per-step Bernoulli masks are drawn inside the launch list; once that list is a CUDA
    graph (third call onwards) every replay must still draw NEW masks from torch's CUDA generator."""
    import fastervit_b200 as F
    kw = dict(dim=32, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
    torch.manual_seed(0)
    model = F.create_model("faster_vit_0_224", drop_path_rate=0.5, **kw).cuda().train()
    x = torch.randn(4, 3, 224, 224, device="cuda")
    outs = []
    for _ in range(5):
        logits = model(x)
        logits.sum().backward()
        model.zero_grad(set_to_none=True)
        outs.append(logits.detach().clone())
    assert all(torch.isfinite(o).all() for o in outs)
    # same input, same weights (no optimizer): only the masks differ from step to step
    diffs = [(outs[i] - outs[i + 1]).abs().max().item() for i in range(4)]
    # (atomics make identical-mask steps differ by ~2e-3 of max|logits|; different masks move them by O(0.1 .. 1))
    assert min(diffs[2:]) > 3e-2 * outs[0].abs().max().item(), diffs
