"""GPU parity: FasterViT forward on the sm_90a kernels vs the golden logits produced by the unmodified
reference in fp64 (tests/golden/*.pt, see oracle/make_golden.py). Tolerance: the north-star's
"outputs within 1e-3 rel" measured as max|d|/max|ref| and as relative L2."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pathlib import Path

GOLDEN = Path(__file__).parent / "golden"


def _setup(case):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    g = torch.load(GOLDEN / f"{case}.pt", weights_only=False)
    model = F.create_model(g["entry"], drop_path_rate=0.0, **g["kwargs"]).eval()
    O.synth_fill_(model.state_dict(), g["seeds"]["w"])
    x = O.synth_input(g["eval"]["batch"], g["cfg"]["resolution"], g["seeds"]["x"], torch.float32)
    return g, model.cuda(), x.cuda()


@pytest.mark.parametrize("case", ["tiny_a", "tiny_qk", "tiny_b", "tiny_ar", "tiny_ar85", "tiny_ar68", "tiny_ar148", "tiny_21k", "tiny_21k224", "fv0", "fv4", "ar0"])
def test_eval_logits_match_reference(case):
    g, model, x = _setup(case)
    with torch.no_grad():
        out = model(x)
    ref = g["eval"]["logits"].to(out.device)
    assert out.shape == ref.shape and out.dtype == torch.float32
    d = out.double() - ref
    max_rel = (d.abs().max() / ref.abs().max()).item()
    l2_rel = (d.norm() / ref.norm()).item()
    print(f"{case}: max-rel {max_rel:.3e}  l2-rel {l2_rel:.3e}")
    assert max_rel < 1e-3 and l2_rel < 1e-3
    # the forward must be repeatable (persistent buffers are fully rewritten each call)
    with torch.no_grad():
        out2 = model(x)
    assert torch.equal(out, out2)


def _sample(t, n=512):
    f = t.detach().flatten()
    stride = max(1, (f.numel() + n - 1) // n)
    return f[::stride].float().cpu()


@pytest.mark.parametrize("case", ["tiny_a", "tiny_qk", "tiny_b", "tiny_ar", "tiny_ar85", "tiny_ar68", "tiny_ar148", "tiny_21k", "tiny_21k224", "fv0", "fv4", "ar0"])
def test_per_module_activations_match_reference_hooks(case):
    """SURVEY 8c: the reference's per-module outputs (forward hooks on patch_embed, every ConvBlock / HAT block,
    every level, the final BatchNorm; fp64, strided samples in tests/golden) against the same points of the
    launch list. Tolerance per activation: max |d| <= 1e-2 * max|ref| and relative L2 of the sample <= 5e-3
    (fp16 tensor-core operands, fp32 accumulation / residual stream)."""
    g, model, x = _setup(case)
    plan = model._get_engine()._plan(x)
    with torch.no_grad(), torch.cuda.device(x.device):
        acts = plan.debug_activations(x)
        acts["norm"] = model.forward_features(x)
    want = g["eval"]["acts"]
    assert set(want) <= set(acts), sorted(set(want) - set(acts))
    worst = (0.0, 0.0, "")
    for name, w in want.items():
        got = acts[name]
        assert tuple(got.shape) == tuple(w["shape"]), (name, tuple(got.shape), w["shape"])
        d = _sample(got) - w["sample"]
        emax = d.abs().max().item() / w["amax"]
        el2 = d.norm().item() / max(w["sample"].norm().item(), 1e-30)
        worst = max(worst, (emax, el2, name))
        assert emax <= 1e-2 and el2 <= 5e-3, (name, emax, el2)
    print(f"{case}: worst activation {worst[2]}: max-rel {worst[0]:.2e}, l2-rel {worst[1]:.2e}")


def test_cpu_input_raises():
    import fastervit_b200 as F
    model = F.create_model("faster_vit_0_224").eval()
    with pytest.raises(Exception):
        model(torch.zeros(1, 3, 224, 224))


def test_batch_independence():
    """Samples do not interact in eval mode: a batch of 3 equals three batches of 1."""
    g, model, x = _setup("tiny_a")
    x3 = torch.cat([x, x[:1] * 0.5], 0)
    with torch.no_grad():
        full = model(x3)
        singles = torch.cat([model(x3[i:i + 1]) for i in range(3)], 0)
    assert (full - singles).abs().max().item() <= 1e-5 * full.abs().max().item()


def test_forward_features_and_head_split():
    """forward == forward_head(forward_features(x)); forward_features returns the BatchNorm-ed [B, C, H, W] map of
    fv.py:949-953 (checked against the reference's `norm` hook), forward_head pools it (fv.py:955-958)."""
    g, model, x = _setup("tiny_a")
    with torch.no_grad():
        full = model(x)
        feats = model.forward_features(x)
        assert feats.shape == (x.shape[0], model.num_features, 7, 7) and feats.dtype == torch.float32
        again = model.forward_head(feats)
        pooled = model.forward_head(feats.mean((2, 3)))          # an already pooled [B, C] tensor is accepted too
    assert (again - full).abs().max().item() <= 1e-3 * full.abs().max().item()
    assert (pooled - full).abs().max().item() <= 1e-3 * full.abs().max().item()
    w = g["eval"]["acts"]["norm"]
    d = _sample(feats) - w["sample"]
    assert d.abs().max().item() <= 1e-2 * w["amax"] and d.norm().item() <= 5e-3 * w["sample"].norm().item()


def test_weight_layout_guards():
    """`.to(memory_format=channels_last)` re-strides the 4-D conv weights and coordinate tables: the engine re-lays
    them out (same logits, channels_last input consumed through its strides); half-precision parameters raise."""
    from fastervit_b200.lib import FvitError
    g, model, x = _setup("tiny_a")
    with torch.no_grad():
        ref = model(x)
        model = model.to(memory_format=torch.channels_last)
        assert not model.patch_embed.conv_down[3].weight.is_contiguous()
        out = model(x.to(memory_format=torch.channels_last))
    assert (out - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    with pytest.raises(FvitError):
        model.half()(x)


def test_stale_eval_plan_is_repacked_after_raw_pointer_updates():
    """The fused optimizer writes parameters through raw pointers (no autograd version bump): the next eval forward
    must run on re-packed fp16 operands, not on the ones cached before the step."""
    from fastervit_b200 import optim as FO
    g, model, x = _setup("tiny_a")
    with torch.no_grad():
        before = model(x)
    model.train()
    opt = FO.FusedAdamW(model, lr=1e-2, weight_decay=0.0)
    torch.nn.functional.cross_entropy(model(x), torch.tensor([1, 2], device=x.device)).backward()
    opt.step()
    model.eval()
    with torch.no_grad():
        after = model(x)
    assert (after - before).abs().max().item() > 1e-3 * before.abs().max().item()


def test_21k_large_window_model_runs_and_trains():
    """faster_vit_4_21k_224 (window 14: S = 196, head_dim 49, fv.py:1253-1290) runs through the key-loop attention
    kernel at full size; its parity is pinned on the reduced tiny_21k goldens. Windows of more than two tiles
    (tiny_21k: 24 x 24 = 576 tokens) train through fvit_attn_loop_bwd_long -- gradient parity against the reference
    is tests/test_train_gpu.py[tiny_21k]; here: the plan takes that kernel and not the SIMT fallback."""
    import fastervit_b200 as F
    torch.manual_seed(0)
    model = F.create_model("faster_vit_4_21k_224").cuda().eval()
    x = torch.randn(2, 3, 224, 224, device="cuda")
    with torch.no_grad():
        out = model(x)
        one = model(x[:1])
    assert out.shape == (2, 1000) and torch.isfinite(out).all()
    assert (out[:1] - one).abs().max().item() <= 1e-4 * out.abs().max().item() + 1e-6
    del model
    g, tiny, xt = _setup("tiny_21k")
    tiny.train()
    loss = tiny(xt).sum()
    loss.backward()
    torch.cuda.synchronize()
    grads = [p.grad for p in tiny.parameters()]
    assert all(gr is not None and torch.isfinite(gr).all() for gr in grads)
    plan = next(p for p in tiny._engine.plans.values() if p.training)
    names = [o[2] for o in plan.bwd_ops]
    assert "fvit_attn_loop_bwd_long" in names and "fvit_attn_core_bwd" not in names
