"""Reduced FasterViT-5 models (80-wide heads at levels 2 and 3, layer scale 1e-5, carrier tokens and propagation)
against the fp64 oracle, with every attention on the tensor-core kernels at padded head dim 80: the 224 model and an
any-res model with window_size [7, 7, 12, 6], whose 148-token level-2 windows train through the key-loop kernels.

Bars (DESIGN.md section 4): eval logits 1e-3, train logits 3e-3, loss 1e-4, BatchNorm running statistics 1e-3,
per-parameter gradients 8e-2 max element / 4e-2 relative L2 (6e-2 for the stem) with a median relative L2 <= 4e-3,
and the eval-mode image gradient 3e-2 relative L2 (tests/test_eval_grad_gpu.py)."""
import pytest
import torch

from test_hd80_plan_cpu import AR80, HD80, attention_launches

pytestmark = pytest.mark.gpu

_CFG224 = dict(dim=80, in_dim=16, depths=[1, 1, 2, 2], num_heads=[1, 2, 4, 8], window_size=[7, 7, 7, 7], ct_size=2,
               mlp_ratio=4, resolution=224, hat=[False, False, True, False], do_propagation=True)
CASES = {
    "fv5_224": ("faster_vit_5_224", HD80, _CFG224),
    "fv5_ar148": ("faster_vit_5_any_res", AR80,
                  dict(_CFG224, window_size=AR80["window_size"], resolution=AR80["resolution"], any_res=True)),
}
_BUF = ("running_mean", "running_var", "num_batches_tracked", "relative_coords_table", "relative_position_index",
        "relative_bias")


def _setup(case, seed):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    entry, kw, cfg = CASES[case]
    model = F.create_model(entry, drop_path_rate=0.0, **kw)
    O.synth_fill_(model.state_dict(), seed)
    sd64 = {k: (v.double().clone() if v.is_floating_point() else v.clone()) for k, v in model.state_dict().items()}
    x = O.synth_input(2, cfg["resolution"], seed + 100, torch.float32)
    target = torch.tensor([7, 901])
    return model.cuda(), sd64, cfg, x, target


def _oracle(sd64, cfg, x, target, training):
    """fp64 CPU autograd of the oracle: (logits, loss, {parameter: grad}, dx, {bn prefix: (batch mean, var)})"""
    from oracle import fastervit_oracle as O
    leaf = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and not k.endswith(_BUF) else v.clone())
            for k, v in sd64.items()}
    for k in list(leaf):
        if ".global_tokenizer.to_global_feature.pos." in k:
            leaf[k] = leaf[k.replace(".to_global_feature.pos.", ".pos_embed.")]
    xl = x.double().clone().requires_grad_(True)
    stats = {}
    logits = O.forward(leaf, cfg, xl, training=training, bn_stats=stats)
    loss = torch.nn.functional.cross_entropy(logits, target)
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names] + [xl], allow_unused=True)
    return (logits.detach(), loss.item(), {k: g for k, g in zip(names, grads[:-1]) if g is not None}, grads[-1],
            stats)


def _rel_l2(got, want, floor):
    return (got - want).norm().item() / max(want.norm().item(), floor * want.numel() ** 0.5)


def _compare_grads(model, ref_grads):
    gmax = max(v.abs().max().item() for v in ref_grads.values())
    bad, l2s = [], []
    for k, p in model.named_parameters():
        want = ref_grads[k]
        assert p.grad is not None and p.grad.shape == want.shape, k
        got = p.grad.double().cpu()
        emax = (got - want).abs().max().item() / max(want.abs().max().item(), 1e-3 * gmax)
        el2 = _rel_l2(got, want, 1e-3 * gmax)
        l2s.append(el2)
        if emax > 8e-2 or el2 > (6e-2 if k.startswith("patch_embed.") else 4e-2):
            bad.append((k, emax, el2))
    assert not bad, bad[:10]
    med = sorted(l2s)[len(l2s) // 2]
    assert med <= 4e-3, med
    return med


def _assert_tensor_core_attention(model):
    plans = list(model._get_engine().plans.values())
    assert plans
    for plan in plans:
        launches = set(attention_launches(plan))
        assert launches and all(d == 80 for _, _, d in launches), launches
        assert not any(n.startswith("fvit_attn_core_") for n, _, _ in launches), launches


@pytest.mark.parametrize("case", list(CASES))
def test_train_step_matches_fp64(case):
    model, sd64, cfg, x, target = _setup(case, 811)
    ref_logits, ref_loss, ref_grads, _, stats = _oracle(sd64, cfg, x, target, training=True)
    model.train()
    logits = model(x.cuda())
    loss = torch.nn.functional.cross_entropy(logits, target.cuda())
    loss.backward()
    torch.cuda.synchronize()
    assert ((logits.detach().double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 3e-3
    assert abs(loss.item() - ref_loss) < 1e-4 * abs(ref_loss) + 1e-4
    sd = model.state_dict()
    assert stats
    for prefix, (mean, var) in stats.items():
        for key, batch in ((".running_mean", mean), (".running_var", var)):
            want = 0.9 * sd64[prefix + key] + 0.1 * batch
            d = (sd[prefix + key].double().cpu() - want).abs().max().item()
            assert d <= 1e-3 * max(want.abs().max().item(), 1e-6) + 1e-6, (prefix + key, d)
    med = _compare_grads(model, ref_grads)
    print(f"{case}: train median rel-L2 {med:.2e}")
    _assert_tensor_core_attention(model)


@pytest.mark.parametrize("case", list(CASES))
def test_eval_logits_and_image_gradient_match_fp64(case):
    """model.eval(); model(x) with x requiring grad: logits, parameter gradients and the image gradient"""
    model, sd64, cfg, x, target = _setup(case, 977)
    ref_logits, _, ref_grads, ref_dx, _ = _oracle(sd64, cfg, x, target, training=False)
    model.eval()
    with torch.no_grad():
        plain = model(x.cuda())
    xg = x.cuda().requires_grad_(True)
    logits = model(xg)
    torch.nn.functional.cross_entropy(logits, target.cuda()).backward()
    torch.cuda.synchronize()
    for out in (plain, logits.detach()):
        assert ((out.double().cpu() - ref_logits).abs().max() / ref_logits.abs().max()).item() < 1e-3
    med = _compare_grads(model, ref_grads)
    dx = _rel_l2(xg.grad.double().cpu(), ref_dx, 0.0)
    print(f"{case}: eval-gradient median rel-L2 {med:.2e}, dx rel-L2 {dx:.2e}")
    assert dx <= 3e-2, dx
    _assert_tensor_core_attention(model)
