"""fp64 reference of the dense-prediction outputs in training (test infrastructure): the oracle's FasterViT.forward
(oracle/fastervit_oracle.py, pinned against the reference's golden outputs) restated with the graph kept at the level
outputs, a forward that stops after a given level, the final `norm` / pooled features as outputs (num_classes = 0,
fv.py:955-958), per-level BatchNorm2d with batch statistics (the backbone's norm{i}, dino/fastervit.py:816-827) and a
frozen prefix whose BatchNorms run in eval mode (fastervit.py:801-812). It is assembled from the oracle's own blocks,
so both follow the same reference lines."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import fastervit_oracle as O

_BUF = ("running_mean", "running_var", "num_batches_tracked", "relative_coords_table", "relative_position_index",
        "relative_bias")


def dense_forward(sd: dict, cfg: dict, x: torch.Tensor, *, stop_level: int | None = None, eval_bn_prefixes=(),
                  bn_stats: dict | None = None, final: str | None = None, training: bool = True,
                  drop_masks: dict | None = None) -> dict:
    """{"levels": {i: level output before its Downsample}, "norm": BatchNorm-ed last map, "pooled": [B, C]} with the
    autograd graph kept. BatchNorms under one of `eval_bn_prefixes` use running statistics; all others batch
    statistics (their running-statistic targets go to bn_stats as in oracle._bn); training=False: all of them use
    running statistics. drop_masks: explicit stochastic-depth factors, as in oracle.forward. Kept equal to
    oracle.forward by tests/test_dense_oracle_cpu.py."""
    depths, heads, wss = cfg["depths"], cfg["num_heads"], cfg["window_size"]
    ct_size, hat = cfg["ct_size"], cfg.get("hat", [False, False, True, False])
    any_res = bool(cfg.get("any_res", False))
    res = cfg["resolution"]
    res = [res, res] if not isinstance(res, (list, tuple)) else list(res)
    nlev = len(depths)
    stop = nlev - 1 if stop_level is None else stop_level

    def bn(t, prefix, eps):
        frozen = any(prefix.startswith(p) for p in eval_bn_prefixes)
        return O._bn(t, sd, prefix, eps, training and not frozen, bn_stats)

    out = {"levels": {}}
    x = O._conv(x, sd["patch_embed.conv_down.0.weight"], None, 2, None)
    x = F.relu(bn(x, "patch_embed.conv_down.1", 1e-4))
    x = O._conv(x, sd["patch_embed.conv_down.3.weight"], None, 2, None)
    x = F.relu(bn(x, "patch_embed.conv_down.4", 1e-4))
    for i in range(stop + 1):
        lp = f"levels.{i}"
        if i < 2:
            for j in range(depths[i]):
                bp = f"{lp}.blocks.{j}"
                h = O._conv(x, sd[bp + ".conv1.weight"], sd[bp + ".conv1.bias"], 1, None)
                h = F.gelu(bn(h, bp + ".norm1", 1e-5))
                h = O._conv(h, sd[bp + ".conv2.weight"], sd[bp + ".conv2.bias"], 1, None)
                h = bn(h, bp + ".norm2", 1e-5)
                if bp + ".gamma" in sd:
                    h = h * sd[bp + ".gamma"].view(1, -1, 1, 1)
                x = x + O._dp(h, drop_masks, bp)
        else:
            ws = wss[i]
            B, C, H, W = x.shape
            lvl_res = [int(2 ** (-2 - i) * res[0]), int(2 ** (-2 - i) * res[1])]
            if any_res:
                Hp, Wp = H + (ws - H % ws) % ws, W + (ws - W % ws) % ws
                if Hp != H or Wp != W:
                    x = F.pad(x, (0, Wp - W, 0, Hp - H))
                tok_res = [lvl_res[0] + (ws - lvl_res[0] % ws) % ws, lvl_res[1] + (ws - lvl_res[1] % ws) % ws]
                sr = (tok_res[0] // ws, tok_res[1] // ws) if hat[i] else (1, 1)
                do_gt = bool(hat[i]) and depths[i] > 0
            else:
                Hp, Wp = H, W
                tok_res = lvl_res
                s = lvl_res[0] // ws if hat[i] else 1
                sr = (s, s)
                do_gt = bool(hat[i]) and depths[i] > 0 and lvl_res[0] // ws > 1
            ct = O.token_initializer(sd, lp + ".global_tokenizer", x, tok_res, ws, ct_size, None) if do_gt else None
            xw = O.window_partition(x, ws)
            for j in range(depths[i]):
                xw, ct = O.hat_block(sd, f"{lp}.blocks.{j}", xw, ct, num_heads=heads[i], ws=ws, sr=sr, ct_size=ct_size,
                                     last=(j == depths[i] - 1), do_propagation=cfg.get("do_propagation", False),
                                     square=(sr[0] == sr[1]), quant=None, masks=drop_masks,
                                     qk_scale=cfg.get("qk_scale"))
            x = O.window_reverse(xw, ws, Hp, Wp, B)
            if Hp != H or Wp != W:
                x = x[:, :, :H, :W].contiguous()
        out["levels"][i] = x
        if i < 3 and i < stop:
            xn = O._ln(x.permute(0, 2, 3, 1), sd, lp + ".downsample.norm", 1e-6).permute(0, 3, 1, 2)
            x = O._conv(xn, sd[lp + ".downsample.reduction.0.weight"], None, 2, None)
    if final is not None:
        assert stop == nlev - 1
        out["norm"] = bn(x, "norm", 1e-5)
        out["pooled"] = out["norm"].mean(dim=(2, 3))
    return out


def leaves(sd: dict, frozen_prefixes=()) -> dict:
    """fp64 copies of the state dict; parameters (not buffers, not the frozen prefix) require grad"""
    leaf = {}
    for k, v in sd.items():
        v = v.detach().cpu()
        if torch.is_floating_point(v):
            v = v.double().clone()
            if not k.endswith(_BUF) and not any(k.startswith(p) for p in frozen_prefixes):
                v.requires_grad_(True)
        leaf[k] = v
    for k in list(leaf):   # the tokenizer conv is registered twice (fv.py:726-728)
        if ".global_tokenizer.to_global_feature.pos." in k:
            leaf[k] = leaf[k.replace(".to_global_feature.pos.", ".pos_embed.")]
    return leaf


def levels_loss_and_grads(sd: dict, cfg: dict, x: torch.Tensor, weights: dict, *, level_norms: dict | None = None,
                          frozen_prefixes=(), final: str | None = None) -> tuple[dict, dict, dict]:
    """loss = sum_i <weights[i], out_i> over level outputs (out_i = BatchNorm2d `level_norms[i]` of the level map with
    batch statistics, when given), or over out["norm"] / out["pooled"] with `final` and weights {final: w}.
    Returns (outputs, d loss / d parameter for every parameter that receives a gradient, BatchNorm running-stat
    targets). `frozen_prefixes` both freeze the parameters and run their BatchNorms in eval mode."""
    leaf = leaves(sd, frozen_prefixes)
    stats: dict = {}
    stop = max(k for k in weights if isinstance(k, int)) if final is None else len(cfg["depths"]) - 1
    fw = dense_forward(leaf, cfg, x.double(), stop_level=stop, eval_bn_prefixes=frozen_prefixes, bn_stats=stats,
                       final=final)
    outs, loss = {}, 0.0
    for k, w in weights.items():
        if final is not None:
            o = fw[final]
        else:
            o = fw["levels"][k]
            if level_norms and level_norms.get(k):
                o = O._bn(o, leaf, level_norms[k], 1e-5, True, stats)
        outs[k] = o
        loss = loss + (o * w.double()).sum()
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names], allow_unused=True)
    return ({k: v.detach() for k, v in outs.items()}, {k: g for k, g in zip(names, grads) if g is not None}, stats)
