"""CPU oracle for FasterViT.forward — TEST INFRASTRUCTURE, not product code.

A functional restatement (plain torch CPU ops, fp32 or fp64) of the reference algorithm in
the reference's fastervit/models/faster_vit.py ("fv.py") and faster_vit_any_res.py ("fvar.py"),
driven by a reference-schema state_dict. Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module; the product (fastervit_b200/) never does.

Parity pin: the reference ships no tests/golden vectors for this path (SURVEY.md §4), so the oracle is
pinned against outputs of the reference itself, generated in the build container by
oracle/make_golden.py (which imports the unmodified reference behind oracle/ref_shim/timm) and
committed under tests/golden/. tests/test_oracle_golden.py re-checks the oracle against them.

Gradients come from torch autograd over this functional graph (the reference has no backward code
either: fv.py relies on autograd, train.py:879-896).

`quant="fp16"` additionally rounds every tensor-core operand (GEMM / conv inputs and weights, Q, K, P, V)
to fp16 — a model of the CUDA path's arithmetic used to budget tolerances; it is NOT the reference.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch
import torch.nn.functional as F


# ---------------------------------------------------------------------------------- helpers
def _q(t: torch.Tensor, quant: Optional[str]) -> torch.Tensor:
    if quant is None:
        return t
    qd = {"fp16": torch.float16, "bf16": torch.bfloat16}[quant]
    return t.to(qd).to(t.dtype)


def _linear(x, w, b, quant):
    return F.linear(_q(x, quant), _q(w, quant), b)


def _conv(x, w, b, stride, quant, groups=1):
    return F.conv2d(_q(x, quant), _q(w, quant), b, stride=stride, padding=1, groups=groups)


def _bn(x, sd, prefix, eps, training, stats_out=None):
    """nn.BatchNorm2d: running stats in eval, batch stats (biased var) in training (fv.py:459-493,925)."""
    w, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
    if training:
        mean = x.mean(dim=(0, 2, 3))
        var = x.var(dim=(0, 2, 3), unbiased=False)
        if stats_out is not None:
            n = x.numel() / x.shape[1]
            stats_out[prefix] = (mean.detach(), (var * n / max(n - 1, 1)).detach())
    else:
        mean, var = sd[prefix + ".running_mean"], sd[prefix + ".running_var"]
    return (x - mean[None, :, None, None]) * torch.rsqrt(var[None, :, None, None] + eps) \
        * w[None, :, None, None] + b[None, :, None, None]


def _ln(x, sd, prefix, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)


def window_partition(x, ws):  # fv.py:83-87
    B, C, H, W = x.shape
    x = x.view(B, C, H // ws, ws, W // ws, ws)
    return x.permute(0, 2, 4, 3, 5, 1).reshape(-1, ws * ws, C)


def window_reverse(win, ws, H, W, B):  # fv.py:90-93
    x = win.view(B, H // ws, W // ws, ws, ws, -1)
    return x.permute(0, 5, 1, 3, 2, 4).reshape(B, win.shape[2], H, W)


def ct_dewindow(ct, W, H, ws):  # fv.py:96-101 (argument naming kept literally)
    bs, N = ct.shape[0], ct.shape[2]
    ct2 = ct.view(-1, W // ws, H // ws, ws, ws, N).permute(0, 5, 1, 3, 2, 4)
    return ct2.reshape(bs, N, W * H).transpose(1, 2)


def ct_window(ct, W, H, ws):  # fv.py:104-109
    bs, N = ct.shape[0], ct.shape[2]
    ct = ct.view(bs, H // ws, ws, W // ws, ws, N)
    return ct.permute(0, 1, 3, 2, 4, 5)


def rel_coords_table(ws: int, dtype) -> torch.Tensor:
    """PosEmbMLPSwinv2D buffer `relative_coords_table` (fv.py:226-243): log-spaced offsets."""
    rc = torch.arange(-(ws - 1), ws, dtype=torch.float32)
    tab = torch.stack(torch.meshgrid([rc, rc], indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    tab = tab / (ws - 1)  # pretrained_window_size == window_size (fv.py:550-553)
    tab = tab * 8
    tab = torch.sign(tab) * torch.log2(torch.abs(tab) + 1.0) / math.log2(8)
    return tab.to(dtype)


def rel_position_index(ws: int) -> torch.Tensor:
    """PosEmbMLPSwinv2D buffer `relative_position_index` (fv.py:244-254)."""
    c = torch.arange(ws)
    coords = torch.stack(torch.meshgrid([c, c], indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - 1
    rel[:, :, 1] += ws - 1
    rel[:, :, 0] *= 2 * ws - 1
    return rel.sum(-1)


def attn_bias(sd, prefix, ws, num_heads, seq_len, dtype, quant=None):
    """PosEmbMLPSwinv2D.forward (fv.py:266-310): 16*sigmoid(cpb_mlp(table))[index], zero rows/cols for
    the (seq_len - ws*ws) carrier tokens on the top/left."""
    tab = sd.get(prefix + ".relative_coords_table")
    tab = rel_coords_table(ws, dtype) if tab is None else tab.to(dtype)
    idx = sd.get(prefix + ".relative_position_index")
    idx = rel_position_index(ws) if idx is None else idx
    h = F.relu(F.linear(tab, sd[prefix + ".cpb_mlp.0.weight"], sd[prefix + ".cpb_mlp.0.bias"]))
    table = F.linear(h, sd[prefix + ".cpb_mlp.2.weight"]).view(-1, num_heads)
    bias = table[idx.view(-1)].view(ws * ws, ws * ws, -1).permute(2, 0, 1).contiguous()
    bias = 16 * torch.sigmoid(bias)
    n_glob = seq_len - ws * ws
    return F.pad(bias, (n_glob, 0, n_glob, 0))


def pos_embed_1d(sd, prefix, seq_len, dtype):
    """PosEmbMLPSwinv1D.forward, rank=2 (fv.py:339-367): cpb_mlp on a centred, normalised n x n grid."""
    n = int(seq_len ** 0.5)
    r = torch.arange(0, n, dtype=dtype)
    tab = torch.stack(torch.meshgrid([r, r], indexing="ij")).contiguous().unsqueeze(0)
    tab = tab - n // 2
    tab = tab / (n // 2)
    tab = tab.flatten(2).transpose(1, 2)
    h = F.relu(F.linear(tab, sd[prefix + ".cpb_mlp.0.weight"], sd[prefix + ".cpb_mlp.0.bias"]))
    return F.linear(h, sd[prefix + ".cpb_mlp.2.weight"])


def window_attention(sd, prefix, x, num_heads, resolution, quant, qk_scale=None):
    """WindowAttention.forward (fv.py:557-568); scale = qk_scale or head_dim ** -0.5 (fv.py:544)."""
    B, N, C = x.shape
    hd = C // num_heads
    qkv = _linear(x, sd[prefix + ".qkv.weight"], sd.get(prefix + ".qkv.bias"), quant)
    qkv = qkv.reshape(B, -1, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    attn = (_q(q, quant) @ _q(k, quant).transpose(-2, -1)) * (qk_scale or hd ** -0.5)
    attn = attn + attn_bias(sd, prefix + ".pos_emb_funct", resolution, num_heads, N, x.dtype).unsqueeze(0)
    attn = attn.softmax(dim=-1)
    out = (_q(attn, quant) @ _q(v, quant)).transpose(1, 2).reshape(B, -1, C)
    return _linear(out, sd[prefix + ".proj.weight"], sd[prefix + ".proj.bias"], quant)


def mlp(sd, prefix, x, quant):
    """Mlp.forward (fv.py:398-407): fc2(GELU_erf(fc1(x)))."""
    h = F.gelu(_linear(x, sd[prefix + ".fc1.weight"], sd[prefix + ".fc1.bias"], quant))
    return _linear(h, sd[prefix + ".fc2.weight"], sd[prefix + ".fc2.bias"], quant)


def _gamma(sd, key):
    g = sd.get(key)
    return 1 if g is None else g


def _dp(t, masks, key):
    """timm DropPath with an explicit mask: t * (bernoulli/keep)[:, None, ...] (identity without a mask)."""
    if masks is None or key not in masks:
        return t
    m = masks[key].to(t.dtype)
    return t * m.view(-1, *([1] * (t.dim() - 1)))


def hat_block(sd, prefix, x, ct, *, num_heads, ws, sr, ct_size, last, do_propagation, square, quant, masks=None,
              qk_scale=None):
    """HAT.forward (fv.py:662-701; fvar.py:668-707). sr = (sr_h, sr_w). `masks` (optional) holds explicit
    stochastic-depth factors per drop_path call site: prefix + .attn/.mlp (per window), .hat_attn/.hat_mlp
    (per image) — the reference draws them with torch RNG (fv.py:679-680, 690-691)."""
    B, T, N = x.shape
    x = x + pos_embed_1d(sd, prefix + ".pos_embed", T, x.dtype)
    do_sr = sr[0] > 1 or sr[1] > 1
    if do_sr:
        Bg, Ng, Hg = ct.shape
        ct = ct_dewindow(ct, ct_size * sr[0], ct_size * sr[1], ct_size)
        if square:
            ct = ct + pos_embed_1d(sd, prefix + ".hat_pos_embed", ct.shape[1], x.dtype)
        n_ct = ct.shape[1]
        ct = ct + _dp(_gamma(sd, prefix + ".gamma1") * window_attention(
            sd, prefix + ".hat_attn", _ln(ct, sd, prefix + ".hat_norm1", 1e-5), num_heads,
            int(n_ct ** 0.5), quant, qk_scale), masks, prefix + ".hat_attn")
        ct = ct + _dp(_gamma(sd, prefix + ".gamma2") * mlp(
            sd, prefix + ".hat_mlp", _ln(ct, sd, prefix + ".hat_norm2", 1e-5), quant), masks, prefix + ".hat_mlp")
        ct = ct_window(ct, ct_size * sr[0], ct_size * sr[1], ct_size)
        ct = ct.reshape(x.shape[0], -1, N)
        x = torch.cat((ct, x), dim=1)
    x = x + _dp(_gamma(sd, prefix + ".gamma3") * window_attention(
        sd, prefix + ".attn", _ln(x, sd, prefix + ".norm1", 1e-5), num_heads, ws, quant, qk_scale), masks, prefix + ".attn")
    x = x + _dp(_gamma(sd, prefix + ".gamma4") * mlp(sd, prefix + ".mlp", _ln(x, sd, prefix + ".norm2", 1e-5), quant),
                masks, prefix + ".mlp")
    if do_sr:
        ctr, x = x.split([x.shape[1] - ws * ws, ws * ws], dim=1)
        ct = ctr.reshape(Bg, Ng, Hg)
        if last and do_propagation:
            img = ctr.transpose(1, 2).reshape(B, N, ct_size, ct_size)
            # the reference round-trips the carrier image through fp32 here (fv.py:700)
            up = F.interpolate(img.to(torch.float32), size=ws, mode="nearest").to(x.dtype)
            x = x + _gamma(sd, prefix + ".gamma1") * up.flatten(2).transpose(1, 2)
    return x, ct


def token_initializer(sd, prefix, x, res_hw, ws, ct_size, quant):
    """TokenInitializer (fv.py:704-738; fvar.py:710-750): depthwise 3x3 + AvgPool + window-major order."""
    ks, ss = [], []
    for r in res_hw:
        out = int(ct_size * r / ws)
        s = int(r / out)
        ks.append(r - (out - 1) * s)
        ss.append(s)
    x = F.conv2d(x, sd[prefix + ".pos_embed.weight"], sd[prefix + ".pos_embed.bias"], padding=1,
                 groups=x.shape[1])
    x = F.avg_pool2d(x, kernel_size=tuple(ks), stride=tuple(ss))
    B, C, H, W = x.shape
    ct = x.view(B, C, H // ct_size, ct_size, W // ct_size, ct_size)
    return ct.permute(0, 2, 4, 3, 5, 1).reshape(-1, H * W, C)


def forward(sd: dict, cfg: dict, x: torch.Tensor, *, training: bool = False,
            quant: Optional[str] = None, capture: Optional[dict] = None,
            bn_stats: Optional[dict] = None, drop_masks: Optional[dict] = None) -> torch.Tensor:
    """FasterViT.forward (fv.py:949-965 / fvar.py:979-995) for a reference-schema state_dict.

    cfg keys: dim, in_dim, depths, num_heads, window_size, ct_size, mlp_ratio, resolution (int or
    [H, W]), hat, do_propagation, any_res (bool). DropPath is the identity (drop_path_rate = 0 in
    every parity run; its RNG is not reproducible across implementations).
    """
    depths, heads, wss = cfg["depths"], cfg["num_heads"], cfg["window_size"]
    ct_size, hat = cfg["ct_size"], cfg.get("hat", [False, False, True, False])
    any_res = bool(cfg.get("any_res", False))
    res = cfg["resolution"]
    res = [res, res] if not isinstance(res, (list, tuple)) else list(res)
    cap = (lambda k, v: capture.__setitem__(k, v.detach())) if capture is not None else (lambda k, v: None)

    # PatchEmbed (fv.py:457-469): conv s2 -> BN(1e-4) -> ReLU -> conv s2 -> BN(1e-4) -> ReLU
    x = _conv(x, sd["patch_embed.conv_down.0.weight"], None, 2, quant)
    x = F.relu(_bn(x, sd, "patch_embed.conv_down.1", 1e-4, training, bn_stats))
    x = _conv(x, sd["patch_embed.conv_down.3.weight"], None, 2, quant)
    x = F.relu(_bn(x, sd, "patch_embed.conv_down.4", 1e-4, training, bn_stats))
    cap("patch_embed", x)

    for i in range(len(depths)):
        lp = f"levels.{i}"
        if i < 2:
            # ConvBlock (fv.py:502-512)
            for j in range(depths[i]):
                bp = f"{lp}.blocks.{j}"
                h = _conv(x, sd[bp + ".conv1.weight"], sd[bp + ".conv1.bias"], 1, quant)
                h = F.gelu(_bn(h, sd, bp + ".norm1", 1e-5, training, bn_stats))
                h = _conv(h, sd[bp + ".conv2.weight"], sd[bp + ".conv2.bias"], 1, quant)
                h = _bn(h, sd, bp + ".norm2", 1e-5, training, bn_stats)
                if bp + ".gamma" in sd:
                    h = h * sd[bp + ".gamma"].view(1, -1, 1, 1)
                x = x + _dp(h, drop_masks, bp)  # DropPath per image (fv.py:511)
        else:
            ws = wss[i]
            B, C, H, W = x.shape
            lvl_res = [int(2 ** (-2 - i) * res[0]), int(2 ** (-2 - i) * res[1])]
            if any_res:
                # fvar.py:805-808, 851-859: pad the map up to a multiple of the window
                Hp = H + (ws - H % ws) % ws
                Wp = W + (ws - W % ws) % ws
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
            ct = token_initializer(sd, lp + ".global_tokenizer", x, tok_res, ws, ct_size, quant) if do_gt else None
            if ct is not None:
                cap(f"{lp}.ct0", ct)
            xw = window_partition(x, ws)
            for j in range(depths[i]):
                xw, ct = hat_block(sd, f"{lp}.blocks.{j}", xw, ct, num_heads=heads[i], ws=ws, sr=sr,
                                   ct_size=ct_size, last=(j == depths[i] - 1),
                                   do_propagation=cfg.get("do_propagation", False),
                                   square=(sr[0] == sr[1]), quant=quant, masks=drop_masks,
                                   qk_scale=cfg.get("qk_scale"))
                cap(f"{lp}.blocks.{j}", xw)
            x = window_reverse(xw, ws, Hp, Wp, B)
            if Hp != H or Wp != W:
                x = x[:, :, :H, :W].contiguous()
        cap(f"{lp}.out", x)
        if i < 3:
            # Downsample (fv.py:437-440): LayerNorm2d(eps 1e-6) -> conv 3x3 s2 (no bias)
            xn = _ln(x.permute(0, 2, 3, 1), sd, lp + ".downsample.norm", 1e-6).permute(0, 3, 1, 2)
            x = _conv(xn, sd[lp + ".downsample.reduction.0.weight"], None, 2, quant)
            cap(f"{lp}.down", x)

    x = _bn(x, sd, "norm", 1e-5, training, bn_stats)  # fv.py:953 (layer_norm_last=False everywhere)
    cap("norm", x)
    x = x.mean(dim=(2, 3))  # AdaptiveAvgPool2d(1) + flatten (fv.py:957-958)
    cap("pooled", x)
    return _linear(x, sd["head.weight"], sd["head.bias"], quant)


# ---------------------------------------------------------------------------------- weights
def synth_fill_(sd: dict, seed: int) -> dict:
    """Deterministic, order-independent synthetic weights for a reference-schema state_dict (in place).

    Fresh-init FasterViT has O(1e-5) layer-scales and unit norms, which would hide whole branches from a
    parity check (SURVEY.md §8c), so norm affines, BN running stats and layer-scales are randomised to
    O(0.1..1). Each tensor's values depend only on (seed, key, shape). Index/coordinate buffers and
    `relative_bias` caches are left untouched.
    """
    import zlib
    for key in sorted(sd.keys()):
        t = sd[key]
        if not torch.is_floating_point(t):
            continue
        if key.endswith(("relative_coords_table", "relative_bias")):
            continue
        # the tokenizer conv is registered under two names sharing one storage (fv.py:726-728)
        canon = key.replace(".to_global_feature.pos.", ".pos_embed.")
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(canon.encode())) % (2 ** 31))
        shape = tuple(t.shape)
        leaf = key.rsplit(".", 1)[-1]
        if leaf == "running_var":
            v = torch.rand(shape, generator=g, dtype=torch.float64) + 0.5
        elif leaf == "running_mean":
            v = torch.randn(shape, generator=g, dtype=torch.float64) * 0.2
        elif leaf.startswith("gamma"):
            v = torch.rand(shape, generator=g, dtype=torch.float64) * 0.25 + 0.05
        elif t.dim() == 1 and leaf == "weight":  # norm scales
            v = 1.0 + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif t.dim() == 1:  # biases (linear, conv, norm)
            v = 0.05 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif t.dim() == 4:  # conv weights ~ 1/sqrt(fan_in)
            fan_in = shape[1] * shape[2] * shape[3]
            v = torch.randn(shape, generator=g, dtype=torch.float64) / math.sqrt(fan_in)
        elif t.dim() == 2:
            if ".cpb_mlp.0." in key:
                v = torch.randn(shape, generator=g, dtype=torch.float64) * 0.5
            elif ".cpb_mlp.2." in key:
                v = torch.randn(shape, generator=g, dtype=torch.float64) * 0.05
            else:
                v = torch.randn(shape, generator=g, dtype=torch.float64) * 0.04
        else:
            v = torch.randn(shape, generator=g, dtype=torch.float64) * 0.05
        t.copy_(v.to(t.dtype))
    return sd


def synth_input(batch: int, hw, seed: int, dtype=torch.float32) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    hw = (hw, hw) if isinstance(hw, int) else tuple(hw)
    return torch.randn((batch, 3) + hw, generator=g, dtype=torch.float64).to(dtype)


def loss_and_grads(sd: dict, cfg: dict, x: torch.Tensor, target: torch.Tensor, *, training=True,
                   quant=None, drop_masks=None) -> tuple[torch.Tensor, torch.Tensor, dict]:
    """CrossEntropy(logits, target) and d loss / d parameter for every float tensor with requires-grad
    semantics in the reference (all nn.Parameters; buffers excluded by name)."""
    buf = ("running_mean", "running_var", "num_batches_tracked", "relative_coords_table",
           "relative_position_index", "relative_bias")
    leaf = {}
    for k, v in sd.items():
        if torch.is_floating_point(v) and not k.endswith(buf):
            leaf[k] = v.detach().clone().requires_grad_(True)
        else:
            leaf[k] = v
    # the tokenizer's conv is registered twice in the reference (fv.py:726-728): tie the alias
    for k in list(leaf.keys()):
        if ".global_tokenizer.to_global_feature.pos." in k:
            leaf[k] = leaf[k.replace(".to_global_feature.pos.", ".pos_embed.")]
    logits = forward(leaf, cfg, x, training=training, quant=quant, drop_masks=drop_masks)
    loss = F.cross_entropy(logits, target)
    names = [k for k, v in leaf.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and ".to_global_feature.pos." not in k]
    grads = torch.autograd.grad(loss, [leaf[k] for k in names], allow_unused=True)
    return loss.detach(), logits.detach(), {k: g for k, g in zip(names, grads) if g is not None}
