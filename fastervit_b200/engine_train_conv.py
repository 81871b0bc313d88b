"""Train-mode forward and backward emitters for the convolutional part of FasterViT (PatchEmbed,
ConvBlock levels, Downsample) — methods of TrainPlan.

BatchNorm2d runs with batch statistics: the convolution GEMM stores the raw output (fp16) centred on a per-channel
pivot (the running mean when the plan was built) and its sum / sum-of-squares, `fvit_bn_finalize_pivot` turns them
into scale/shift (and updates the running statistics),
`fvit_affine_rows` normalises + activates (+ residual). The backward is the mirror image: `fvit_bn_bwd`,
the data-gradient convolution as a 9-tap GEMM over the flipped-transposed packed weights, and the
weight gradient as nine MN-major GEMMs (one per tap: dW_t = dZ^T X shifted by the tap) with split-K.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lib as L
from .engine import P, _ru


def _bn_train(self, name: str, bn: nn.BatchNorm2d, count: int, ls=None) -> dict:
    """statistics accumulators + finalize launch; returns the saved vectors. A BatchNorm on running statistics (the
    frozen prefix, an eval-mode plan, a frozen BatchNorm of the stem) has no accumulators: its GEMM gets col_sum =
    col_sumsq = None."""
    C = bn.running_mean.numel()   # (a frozen BatchNorm need not have num_features)
    nb = self.bufs
    st = nb.new(name + ".stats", (2, C), torch.float32)
    frozen = id(bn) in self._frozen_bn
    if not frozen:
        self.fwd_zero.append(st)
    # moments about `pivot` (include/fvit.h "Pivoted statistics"): fvit_colstats_pivot_f32 fills it, or _bn_col_shift
    # (convolution GEMMs) sets it once; shifted: the normalised rows are the GEMM output centred on it
    d = dict(bn=bn, st=st, sc=nb.new(name + ".scale", (C,), torch.float32), sh=nb.new(name + ".shift", (C,), torch.float32),
             mu=nb.new(name + ".mean", (C,), torch.float32), rs=nb.new(name + ".rstd", (C,), torch.float32),
             s12=nb.new(name + ".s12", (2, C), torch.float32), pivot=nb.new(name + ".pivot", (C,), torch.float32),
             shifted=False, count=count, name=name,
             col_sum=None if frozen else st[0].data_ptr(), col_sumsq=None if frozen else st[1].data_ptr())
    return d


def _bn_col_shift(self, d: dict, bias) -> int | None:
    """col_shift of the convolution GEMM feeding BatchNorm d. The GEMM writes and sums conv + bias - K with K the
    running mean when the plan is built (a pretrained or fine-tuned model: within a few std of the batch mean; 0 for
    a fresh one, which is the plain one-pass sum). K stays fixed for the plan's life, so steps on the same input
    round the same way. The frozen prefix normalises with running statistics and keeps the plain bias."""
    bn = d["bn"]
    if id(bn) in self._frozen_bn:
        return P(bias)
    with torch.no_grad():
        d["pivot"].copy_(bn.running_mean.to(d["pivot"].device))
    cs = self.bufs.new(d["name"] + ".col_shift", (bn.num_features,), torch.float32)
    self._op(self.prep_ops, "fvit_bn_col_shift", P(bias), d["pivot"].data_ptr(), bn.num_features, cs.data_ptr())
    d["shifted"] = True
    return cs.data_ptr()


def _bn_finalize(self, d: dict, ls=None) -> None:
    bn = d["bn"]
    if id(bn) in self._frozen_bn:
        # frozen prefix (an eval()-ed module of the backbone, fastervit.py:801-812): running statistics, not updated
        self._op(self.ops, "fvit_affine_fold", d["sc"].data_ptr(), d["sh"].data_ptr(), bn.running_mean.numel(),
                 bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                 float(bn.eps), None, P(ls))
        return
    self._bn_batch_stats.append(bn)
    self._op(self.ops, "fvit_bn_finalize_pivot", d["st"][0].data_ptr(), d["st"][1].data_ptr(), d["pivot"].data_ptr(),
             int(d["shifted"]), float(d["count"]), bn.weight.data_ptr(), bn.bias.data_ptr(), float(bn.eps),
             float(bn.momentum), bn.running_mean.data_ptr(), bn.running_var.data_ptr(), P(ls), d["sc"].data_ptr(),
             d["sh"].data_ptr(), d["mu"].data_ptr(), d["rs"].data_ptr(), bn.num_features)


def _emit_conv_part_train(self) -> dict:
    m, B, nb = self.model, self.B, self.bufs
    cfg = m.cfg
    dim, in_dim = cfg["dim"], cfg["in_dim"]
    H1, W1 = (self.H + 1) // 2, (self.W + 1) // 2
    H0, W0 = (H1 + 1) // 2, (W1 + 1) // 2
    ld_in = _ru(in_dim, 8)
    pl_rows = B * (H0 + 1) * (W0 + 1)
    npix1 = B * H1 * W1
    stem_map = self._parity_plane_map("stem.map", H1, W1)
    pe = m.patch_embed.conv_down
    st = dict(H1=H1, W1=W1, H0=H0, W0=W0, pl_rows=pl_rows, ld_in=ld_in, npix1=npix1, stem_map=stem_map)
    # conv1: im2col + GEMM -> raw1 (plane layout) + statistics
    k1, sld = self.stem_cols()
    st.update(k1=k1, sld=sld)
    col16 = nb.new("stem.col16", (npix1, sld), torch.float16)
    self._x_args.append(dict(B=B, cin=cfg["in_chans"], H=self.H, W=self.W, out=col16.data_ptr(), ldo=sld))
    self.ops.append(("im2col", len(self._x_args) - 1, "fvit_stem_im2col"))
    w1 = nb.new("stem.conv1.w16", (in_dim, sld), torch.float16)
    self._op(self.prep_ops, "fvit_cast_pad_f16", pe[0].weight.data_ptr(), k1, w1.data_ptr(), sld, in_dim, k1, sld)
    raw1 = nb.new("stem.raw1", (4 * pl_rows, ld_in), torch.float16)
    planes = nb.new("stem.planes", (4 * pl_rows, ld_in), torch.float16)
    bn1 = _bn_train(self, "stem.bn1", pe[1], npix1)
    self._gemm(a=col16.data_ptr(), a_rows=npix1, lda=sld, b=w1.data_ptr(), ldb=sld, m=npix1, n=in_dim,
               kc=sld, col_shift=_bn_col_shift(self, bn1, None), row_map=stem_map.data_ptr(), out_f16=raw1.data_ptr(),
               ld_o16=ld_in, col_sum=bn1["col_sum"], col_sumsq=bn1["col_sumsq"], flops=2.0 * npix1 * in_dim * k1)
    _bn_finalize(self, bn1)
    self._op(self.ops, "fvit_affine_rows", raw1.data_ptr(), ld_in, stem_map.data_ptr(), npix1, in_dim, bn1["sc"].data_ptr(),
             bn1["sh"].data_ptr(), L.ACT_RELU, None, 0, None, 0, planes.data_ptr(), ld_in, None)
    # conv2 (stride 2) -> raw2 in the level-0 layout
    lvl = self._conv_level_train_buffers(0, dim, H0, W0, len(m.levels[0].blocks))
    self._zero_window_padding(lvl)
    w2, ldw2 = self._pack_conv("stem.conv2", pe[3])
    raw2 = nb.new("stem.raw2", (lvl["rows"], lvl["ld"]), torch.float16)
    bn2 = _bn_train(self, "stem.bn2", pe[4], B * H0 * W0)
    to_l0 = self._plane_to_padded_map("stem.to_l0", B, H0, W0, lvl["Hb"], lvl["Wb"])
    self._gemm(a=planes.data_ptr(), a_rows=pl_rows, lda=ld_in, a_planes=4, a_plane_stride=pl_rows * ld_in, b=w2.data_ptr(),
               ldb=ldw2, m=pl_rows, n=dim, kc=in_dim, taps=self._s2_taps(W0), m_alg=B * H0 * W0,
               col_shift=_bn_col_shift(self, bn2, None), row_map=to_l0.data_ptr(),
               out_f16=raw2.data_ptr(), ld_o16=lvl["ld"], col_sum=bn2["col_sum"], col_sumsq=bn2["col_sumsq"])
    _bn_finalize(self, bn2)
    self._op(self.ops, "fvit_affine_rows", raw2.data_ptr(), lvl["ld"], lvl["pix"].data_ptr(), B * H0 * W0, dim,
             bn2["sc"].data_ptr(), bn2["sh"].data_ptr(), L.ACT_RELU, None, 0, lvl["x32"].data_ptr(), dim,
             lvl["x16s"][0].data_ptr(), lvl["ld"], None)
    st.update(col16=col16, w1=w1, raw1=raw1, planes=planes, bn1=bn1, w2=w2, ldw2=ldw2, raw2=raw2, bn2=bn2, to_l0=to_l0)
    self.stem_sv = st
    # conv levels
    self.conv_lv = []
    Hc, Wc, Cc = H0, W0, dim
    prev = None
    for i, level in enumerate(m.levels):
        if not level.conv or i > self.stop_level:
            break
        if i > 0:
            Hc, Wc, Cc = (Hc + 1) // 2, (Wc + 1) // 2, Cc * 2
            lvl = self._conv_level_train_buffers(i, Cc, Hc, Wc, len(level.blocks))
            self._zero_window_padding(lvl)
            self._emit_downsample_train(i - 1, prev, lvl)
        self._emit_conv_blocks_train(i, level, lvl)
        lvl["kind"] = "conv"
        lvl["level_index"] = i
        self._level_of[i] = lvl
        self.conv_lv.append(lvl)
        prev = lvl
    self.conv_out = prev
    return prev


def _conv_level_train_buffers(self, i: int, Cc: int, Hc: int, Wc: int, depth: int) -> dict:
    """Plan._conv_level_buffers with the backward's fp16 gradient operands (dzA, dzB, dyA), one fp16 operand copy of
    the map per block boundary (x16s: every block's saved input, then the level output) and the fp32 gradient g with
    one guaranteed-zero row at the end"""
    nb = self.bufs
    d = self._conv_level_buffers(i, Cc, Hc, Wc, f16=("dzA", "dzB", "dyA"))
    rows = d["rows"]
    d.update(kind="conv", zero_row=rows, g=nb.new(f"l{i}.g", (rows + 1, Cc), torch.float32),
             x16s=[nb.new(f"l{i}.x16.{j}", (rows, d["ld"]), torch.float16) for j in range(depth + 1)])
    d["x16"] = d["x16s"][-1]  # level output operand (input of the downsample LayerNorm is x32)
    return d


def _emit_conv_blocks_train(self, i: int, level, lv: dict) -> None:
    B, nb = self.B, self.bufs
    # the blocks compute the whole (window-padded, conv_level_pad) map: statistics and affine passes over cpix
    Cc, Wp, rows, ld, npix, pix = lv["C"], lv["Wb"] + 2, lv["rows"], lv["ld"], lv["cnpix"], lv["cpix"]
    taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
    lv["taps"] = taps
    lv["blocks_sv"] = []
    for j, blk in enumerate(level.blocks):
        if hasattr(blk, "gamma"):
            raise L.FvitError("layer_scale_conv is not supported by the training kernels (unused by every shipped config)")
        nm = f"l{i}.b{j}"
        rate = self._drop_rate(i)
        self._block_counter += 1
        rs = self._drop_buf(f"levels.{i}.blocks.{j}", rate, B, (lv["Hb"] + 2) * (lv["Wb"] + 2))
        w1, ld1 = self._pack_conv(nm + ".conv1", blk.conv1)
        w2, ld2 = self._pack_conv(nm + ".conv2", blk.conv2)
        rawA = nb.new(nm + ".rawA", (rows, ld), torch.float16)
        rawB = nb.new(nm + ".rawB", (rows, ld), torch.float16)
        h16 = nb.new(nm + ".h16", (rows, ld), torch.float16)   # kept for the conv2 weight gradient (zero borders)
        bnA = _bn_train(self, nm + ".bn1", blk.norm1, npix)
        bnB = _bn_train(self, nm + ".bn2", blk.norm2, npix)
        xin, xout = lv["x16s"][j], lv["x16s"][j + 1]
        self._gemm(a=xin.data_ptr(), a_rows=rows, lda=ld, b=w1.data_ptr(), ldb=ld1, m=rows, n=Cc, kc=Cc, taps=taps,
                   m_alg=npix, col_shift=_bn_col_shift(self, bnA, blk.conv1.bias), row_map=lv["interior"].data_ptr(),
                   out_f16=rawA.data_ptr(), ld_o16=ld, col_sum=bnA["col_sum"], col_sumsq=bnA["col_sumsq"])
        _bn_finalize(self, bnA)
        self._op(self.ops, "fvit_affine_rows", rawA.data_ptr(), ld, pix.data_ptr(), npix, Cc, bnA["sc"].data_ptr(),
                 bnA["sh"].data_ptr(), L.ACT_GELU, None, 0, None, 0, h16.data_ptr(), ld, None)
        self._gemm(a=h16.data_ptr(), a_rows=rows, lda=ld, b=w2.data_ptr(), ldb=ld2, m=rows, n=Cc, kc=Cc, taps=taps,
                   m_alg=npix, col_shift=_bn_col_shift(self, bnB, blk.conv2.bias), row_map=lv["interior"].data_ptr(),
                   out_f16=rawB.data_ptr(), ld_o16=ld, col_sum=bnB["col_sum"], col_sumsq=bnB["col_sumsq"])
        _bn_finalize(self, bnB)
        self._op(self.ops, "fvit_affine_rows", rawB.data_ptr(), ld, pix.data_ptr(), npix, Cc, bnB["sc"].data_ptr(),
                 bnB["sh"].data_ptr(), L.ACT_NONE, lv["x32"].data_ptr(), Cc, lv["x32"].data_ptr(), Cc, xout.data_ptr(), ld, rs)
        # data-gradient operands: flipped / transposed packed weights
        wT1 = nb.new(nm + ".conv1.wT16", (Cc, 9 * _ru(Cc, 64)), torch.float16)
        wT2 = nb.new(nm + ".conv2.wT16", (Cc, 9 * _ru(Cc, 64)), torch.float16)
        self._op(self.prep_ops, "fvit_pack_conv3x3_f16", blk.conv1.weight.data_ptr(), wT1.data_ptr(), Cc, Cc, _ru(Cc, 64), 1)
        self._op(self.prep_ops, "fvit_pack_conv3x3_f16", blk.conv2.weight.data_ptr(), wT2.data_ptr(), Cc, Cc, _ru(Cc, 64), 1)
        lv["blocks_sv"].append(dict(blk=blk, rawA=rawA, rawB=rawB, h16=h16, bnA=bnA, bnB=bnB, xin=xin, wT1=wT1, wT2=wT2,
                                    rs=rs))


def _emit_downsample_train(self, i: int, src: dict, dst: dict) -> None:
    """Downsample i in training: LayerNorm saves xhat / rstd; the conv also emits a fp16 copy of the next
    level's input (the conv-level operand, or the token level's x0 for the tokenizer weight gradient)."""
    B, nb = self.B, self.bufs
    ds_mod = self.model.levels[i].downsample
    Cs, Hs, Ws = src["C"], src["H"], src["W"]
    Ho, Wo = (Hs + 1) // 2, (Ws + 1) // 2
    ld = _ru(Cs, 8)
    pl_rows = B * (Ho + 1) * (Wo + 1)
    npix = B * Hs * Ws
    planes = nb.new(f"ds{i}.planes", (4 * pl_rows, ld), torch.float16)
    omap = self._parity_plane_map(f"ds{i}.omap", Hs, Ws)
    src_rows = src["pix"] if src["kind"] == "conv" else src["crop_map"]
    src_x = src["x32"] if src["kind"] == "conv" else src["xs"]
    xh = nb.new(f"ds{i}.xhat", (npix, Cs), torch.float16)
    rs = nb.new(f"ds{i}.rstd", (npix,), torch.float32)
    mu = nb.new(f"ds{i}.mean", (npix,), torch.float32)
    self._op(self.ops, "fvit_ln_fwd", src_x.data_ptr(), Cs, src_rows.data_ptr(), npix, Cs, None, 1, 0, None, 0,
             ds_mod.norm.weight.data_ptr(), ds_mod.norm.bias.data_ptr(), float(ds_mod.norm.eps), planes.data_ptr(), ld,
             omap.data_ptr(), mu.data_ptr(), rs.data_ptr(), xh.data_ptr(), Cs)
    w16, ldw = self._pack_conv(f"ds{i}.conv", ds_mod.reduction[0])
    if "x16s" in dst:   # a conv level: its residual stream and first block's input operand
        out32, out16, ld16 = dst["x32"], dst["x16s"][0], dst["ld"]
    else:               # a token level: its residual stream and x0, the tokenizer's weight-gradient operand
        out32, ld16 = dst["xs"], 2 * Cs
        out16 = dst["x0_16"] = nb.new(f"ds{i}.x0_16", (dst["xs"].shape[0], 2 * Cs), torch.float16)
    rmap = self._downsample_row_map(i, dst, Ho, Wo)
    self._gemm(a=planes.data_ptr(), a_rows=pl_rows, lda=ld, a_planes=4, a_plane_stride=pl_rows * ld, b=w16.data_ptr(),
               ldb=ldw, m=pl_rows, n=2 * Cs, kc=Cs, taps=self._s2_taps(Wo), m_alg=B * Ho * Wo, row_map=rmap.data_ptr(),
               out_f32=out32.data_ptr(), ld_o32=dst["C"], out_f16=out16.data_ptr(), ld_o16=ld16)
    # backward-side maps / packed operands: the border rows of the plane-space output read the gradient's zero row
    rmap_g = nb.i32(f"ds{i}.rmap_g", torch.where(rmap >= 0, rmap, torch.full_like(rmap, dst["zero_row"])))
    wT = _s2_dgrad_operands(self, f"ds{i}", ds_mod.reduction[0], Wo)
    dst["ds"] = dict(i=i, mod=ds_mod, Cs=Cs, Ho=Ho, Wo=Wo, ld=ld, pl_rows=pl_rows, npix=npix, planes=planes, omap=omap,
                     src_rows=src_rows, xh=xh, rs=rs, rmap_g=rmap_g, wT=wT,
                     dY=nb.new(f"ds{i}.dY16", (pl_rows, 2 * Cs), torch.float16),
                     dplanes=nb.new(f"ds{i}.dplanes16", (4 * pl_rows, ld), torch.float16))


def _s2_dgrad_operands(self, name: str, conv: nn.Conv2d, Wo: int) -> list:
    """data-gradient operands of a 3x3 stride-2 convolution over parity planes (Plan._s2_taps): for each input plane,
    the flipped / transposed weights of the taps that read it, [(packed fp16 buffer, tap indices)] * 4"""
    cout, cin = conv.weight.shape[:2]
    taps = self._s2_taps(Wo)
    co_pad = _ru(cout, 64)
    wT = []
    for p in range(4):
        tl_ = [t for t in range(9) if taps[t][1] == p]
        buf = self.bufs.new(f"{name}.wT.{p}", (cin, len(tl_) * co_pad), torch.float16)
        self._op(self.prep_ops, "fvit_pack_conv3x3_taps_f16", conv.weight.data_ptr(), buf.data_ptr(), cout, cin, co_pad, 1,
                 len(tl_), *(tl_ + [0] * (9 - len(tl_))))
        wT.append((buf, tl_))
    return wT


# ====================================================================================== backward
def _bn_bwd(self, d: dict, gin, g_is_f16: int, ldg: int, g_rows, raw, ldr: int, r_rows, nrows: int, act: int, out,
            ldo: int, o_rows, row_scale=None, data_only=False) -> None:
    """BatchNorm2d backward of d (_bn_train) into fp16 rows `out`: batch statistics (fvit_bn_bwd), or the running
    statistics of an eval-mode plan (fvit_bn_eval_bwd: no mean(dy) terms, one pass). data_only (running statistics,
    no stochastic depth: a frozen or eval stage), or a frozen BatchNorm of the stem (no parameters; the convolutions
    around it keep their weight gradients): the streaming fvit_bn_eval_dgrad, dy times the forward's folded scale"""
    bn = d["bn"]
    if data_only or id(bn) in self._fixed_bn:
        self._op(self.bwd_ops, "fvit_bn_eval_dgrad", gin, g_is_f16, ldg, g_rows, raw, ldr, r_rows, nrows,
                 bn.running_mean.numel(),
                 d["sc"].data_ptr(), d["sh"].data_ptr(), act, None, None, out, ldo, o_rows)
        return
    if self.eval_grad:
        self._op(self.bwd_ops, "fvit_bn_eval_bwd", gin, g_is_f16, ldg, g_rows, raw, ldr, r_rows, nrows, bn.num_features,
                 bn.running_mean.data_ptr(), bn.running_var.data_ptr(), float(bn.eps), bn.weight.data_ptr(),
                 bn.bias.data_ptr(), act, None, ("scal", 1), out, ldo, o_rows, self.G(bn.weight), self.G(bn.bias))
        return
    self._op(self.bwd_ops, "fvit_bn_bwd", gin, g_is_f16, ldg, g_rows, raw, ldr, r_rows, nrows, bn.num_features,
             d["mu"].data_ptr(), d["rs"].data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(), act, None,
             d["s12"][0].data_ptr(), d["s12"][1].data_ptr(), ("scal", 1), out, ldo, o_rows, self.G(bn.weight),
             self.G(bn.bias), row_scale)


def _conv_wgrad(self, *, dz, lddz, x, ldx, x_rows, rows, cout, cin, shifts, conv_weight, name: str, bias=None,
                bias_rows=None, bias_nrows=0) -> None:
    """dW[co][ci][t] = sum_q dz[q][co] * x[q + shift_t][ci]: ONE MN-major split-K GEMM whose N dimension
    enumerates (tap, ci) -- every dz tile is fetched once for the nine shifted views of x -- plus a repack.
    bias: db[co] += sum over the rows `bias_rows` of dz (scaled by 1/S), a column sum beside the GEMM."""
    nt = len(shifts)
    scr = ("scr", self._scratch(name + ".dWtaps", nt * cout * cin))
    sk = self._split_k(cout, cin, rows, nt)
    n0 = len(self.bwd_ops)
    self._gemm(a=dz, a_rows=rows, lda=lddz, a_mn=True, b=x, b_rows=x_rows, ldb=ldx, b_mn=True, b_taps=list(shifts), m=cout,
               n=cin, kc=rows, split_k=sk, alpha_ptr=("scal", 1), out_f32=scr, ld_o32=nt * cin, target=self.bwd_ops,
               flops=2.0 * rows * cout * cin * nt)
    self._op(self.bwd_ops, "fvit_unpack_conv_grad", scr, nt * cin, self.G(conv_weight), cout, cin)
    if bias is not None:
        self._op(self.bwd_ops, "fvit_colsum", dz, 1, lddz, bias_rows, None, 0, bias_nrows, cout, None, ("scal", 1),
                 self.G(bias), None)
    self._side_from(n0, dz)   # (its own zeroed scratch slice in, a parameter gradient out: a leaf pair)


def _s2_conv_bwd(self, *, conv: nn.Conv2d, wT: list, dY, lddy: int, planes, dplanes, ld: int, pl_rows: int, Wo: int,
                 npix: int, name: str, data_only: bool) -> None:
    """Backward of a 3x3 stride-2 convolution over the parity planes `planes` (ld wide) from the gradient dY of its
    pl_rows plane-space output rows (npix of them real pixels): the weight gradient unless data_only, then the gradient
    of the planes into dplanes, one GEMM per plane over the taps that read it (wT: _s2_dgrad_operands)"""
    cout, cin = conv.weight.shape[:2]
    taps = self._s2_taps(Wo)
    if not data_only:
        _conv_wgrad(self, dz=dY, lddz=lddy, x=planes, ldx=ld, x_rows=4 * pl_rows, rows=pl_rows, cout=cout, cin=cin,
                    shifts=[p * pl_rows + s for (s, p) in taps], conv_weight=conv.weight, name=name)
    for p, (buf, tl_) in enumerate(wT):
        self._gemm(a=dY, a_rows=pl_rows, lda=lddy, b=buf.data_ptr(), b_rows=cin, ldb=buf.shape[1], m=pl_rows, n=cin,
                   kc=cout, taps=[(-taps[t][0], 0) for t in tl_], out_f16=dplanes + 2 * p * pl_rows * ld, ld_o16=ld,
                   target=self.bwd_ops, flops=2.0 * npix * cin * cout * len(tl_))


def _emit_downsample_bwd(self, ds: dict, src: dict, dst: dict) -> None:
    """Downsample backward into the source level's output gradient; data-only (with the level in front of it, stage
    1 + i): no weight gradient, LayerNorm dx only"""
    data_only = self.data_only[1 + ds["i"]]
    Cs, ld, pl_rows = ds["Cs"], ds["ld"], ds["pl_rows"]
    # gradient of the conv output in plane space (border rows read the buffer's zero row)
    self._op(self.bwd_ops, "fvit_cast_scale_f16", dst["g"].data_ptr(), 2 * Cs, ds["rmap_g"].data_ptr(), pl_rows, 2 * Cs,
             None, None, ds["dY"].data_ptr(), 2 * Cs, None)
    _s2_conv_bwd(self, conv=ds["mod"].reduction[0], wT=ds["wT"], dY=ds["dY"].data_ptr(), lddy=2 * Cs,
                 planes=ds["planes"].data_ptr(), dplanes=ds["dplanes"].data_ptr(), ld=ld, pl_rows=pl_rows, Wo=ds["Wo"],
                 npix=self.B * ds["Ho"] * ds["Wo"], name=f"ds{ds['i']}", data_only=data_only)
    self._ln_bwd(ds["mod"].norm, ds["dplanes"].data_ptr(), ld, ds["omap"].data_ptr(), ds["xh"].data_ptr(),
                 ds["rs"].data_ptr(), ds["npix"], Cs, src["g"].data_ptr(), ds["src_rows"].data_ptr(), 0, 0, data_only)


def _emit_conv_blocks_bwd(self, lv: dict, input_grad: bool = True) -> None:
    """input_grad=False: nothing below reads the gradient of the level's input (the frozen prefix ends here), so the
    first block's conv1 data-gradient GEMM is not emitted. A data-only level: the two BatchNorm passes without their
    reductions and the two data-gradient GEMMs per block."""
    Cc, rows, ld, npix = lv["C"], lv["rows"], lv["ld"], lv["cnpix"]
    data_only = self.data_only[1 + lv["level_index"]]
    g = lv["g"].data_ptr()
    pix, interior = lv["cpix"].data_ptr(), lv["interior"].data_ptr()   # (the whole computed map, _emit_conv_blocks_train)
    shifts = [s for (s, _) in lv["taps"]]
    for sv in reversed(lv["blocks_sv"]):
        blk, bnA, bnB = sv["blk"], sv["bnA"], sv["bnB"]
        # x_out = x_in + BN2(conv2(h)); h = GELU(BN1(conv1(x_in)))
        self._before_write(lv["dzB"].data_ptr())
        _bn_bwd(self, bnB, g, 0, Cc, pix, sv["rawB"].data_ptr(), ld, pix, npix, L.ACT_NONE, lv["dzB"].data_ptr(), ld, pix,
                sv["rs"], data_only)
        # h = GELU(BN1(rawA)) was kept by the forward; the pre-activation BN1(rawA) is re-derived inside the dgrad
        # epilogue from rawA and the BatchNorm affine (aux_scale / aux_shift).
        # conv biases sit in front of a batch-statistics BatchNorm: their gradient sum_rows(dz) is identically zero
        # (BN backward removes the per-channel mean), so it is left at the zero the buffer was cleared to. Running
        # statistics (eval-mode plan) remove nothing: there it is a column sum of dz.
        bias_b = blk.conv2.bias if self.eval_grad else None
        bias_a = blk.conv1.bias if self.eval_grad else None
        if not data_only:
            _conv_wgrad(self, dz=lv["dzB"].data_ptr(), lddz=ld, x=sv["h16"].data_ptr(), ldx=ld, x_rows=rows, rows=rows,
                        cout=Cc, cin=Cc, shifts=shifts, conv_weight=blk.conv2.weight, name="convB", bias=bias_b,
                        bias_rows=pix, bias_nrows=npix)
        self._gemm(a=lv["dzB"].data_ptr(), a_rows=rows, lda=ld, b=sv["wT2"].data_ptr(), b_rows=Cc, ldb=9 * _ru(Cc, 64),
                   m=rows, n=Cc, kc=Cc, taps=lv["taps"], act=L.ACT_GELU_BWD, aux=sv["rawA"].data_ptr(), ld_aux=ld,
                   aux_scale=bnA["sc"].data_ptr(), aux_shift=bnA["sh"].data_ptr(), row_map=interior,
                   out_f16=lv["dyA"].data_ptr(), ld_o16=ld, target=self.bwd_ops, m_alg=npix)
        self._before_write(lv["dzA"].data_ptr())
        _bn_bwd(self, bnA, lv["dyA"].data_ptr(), 1, ld, pix, sv["rawA"].data_ptr(), ld, pix, npix, L.ACT_NONE,
                lv["dzA"].data_ptr(), ld, pix, None, data_only)
        if not data_only:
            _conv_wgrad(self, dz=lv["dzA"].data_ptr(), lddz=ld, x=sv["xin"].data_ptr(), ldx=ld, x_rows=rows, rows=rows,
                        cout=Cc, cin=Cc, shifts=shifts, conv_weight=blk.conv1.weight, name="convA", bias=bias_a,
                        bias_rows=pix, bias_nrows=npix)
        if sv is lv["blocks_sv"][0] and not input_grad:
            continue
        # g += conv1 data gradient
        self._gemm(a=lv["dzA"].data_ptr(), a_rows=rows, lda=ld, b=sv["wT1"].data_ptr(), b_rows=Cc, ldb=9 * _ru(Cc, 64),
                   m=rows, n=Cc, kc=Cc, taps=lv["taps"], row_map=interior, resid=g, ld_resid=Cc, out_f32=g, ld_o32=Cc,
                   target=self.bwd_ops, m_alg=npix)


def _emit_conv_part_bwd(self) -> None:
    ops = self.bwd_ops
    m, B = self.model, self.B
    for idx in range(len(self.conv_lv) - 1, -1, -1):
        lv = self.conv_lv[idx]
        if not self._needed(1 + idx):  # nothing below reads a gradient: no dgrad / wgrad / BatchNorm backward from here
            return
        if lv is self.feat:           # levels mode with a conv top level: its output gradient enters here
            self._inject(idx)
        _emit_conv_blocks_bwd(self, lv, input_grad=self._needed(idx))
        if idx > 0:
            if not self._needed(idx):
                return
            _emit_downsample_bwd(self, lv["ds"], self.conv_lv[idx - 1], lv)
            self._inject(idx - 1)
    if not self._needed(0):
        return
    data_only = self.data_only[0]
    # PatchEmbed
    st, lv0 = self.stem_sv, self.conv_lv[0]
    pe = m.patch_embed.conv_down
    nb = self.bufs
    dim, in_dim = lv0["C"], m.cfg["in_dim"]
    H0, W0, pl_rows, ld_in, npix1 = st["H0"], st["W0"], st["pl_rows"], st["ld_in"], st["npix1"]
    inv = ("scal", 1)
    bb, aa, cc = torch.meshgrid(torch.arange(B), torch.arange(H0), torch.arange(W0), indexing="ij")
    q_of_pix = nb.i32("stem.q_of_pix", (bb * (H0 + 1) * (W0 + 1) + (aa + 1) * (W0 + 1) + cc + 1).reshape(-1))
    dY2 = nb.new("stem.dY2", (pl_rows, lv0["ld"]), torch.float16)
    bn2, bn1 = st["bn2"], st["bn1"]
    _bn_bwd(self, bn2, lv0["g"].data_ptr(), 0, dim, lv0["pix"].data_ptr(), st["raw2"].data_ptr(), lv0["ld"],
            lv0["pix"].data_ptr(), B * H0 * W0, L.ACT_RELU, dY2.data_ptr(), lv0["ld"], q_of_pix.data_ptr(), None, data_only)
    dplanes = nb.new("stem.dplanes16", (4 * pl_rows, ld_in), torch.float16)
    _s2_conv_bwd(self, conv=pe[3], wT=_s2_dgrad_operands(self, "stem", pe[3], W0), dY=dY2.data_ptr(), lddy=lv0["ld"],
                 planes=st["planes"].data_ptr(), dplanes=dplanes.data_ptr(), ld=ld_in, pl_rows=pl_rows, Wo=W0,
                 npix=B * H0 * W0, name="stem2", data_only=data_only)
    dz1 = nb.new("stem.dz1", (npix1, ld_in), torch.float16)
    _bn_bwd(self, bn1, dplanes.data_ptr(), 1, ld_in, st["stem_map"].data_ptr(), st["raw1"].data_ptr(), ld_in,
            st["stem_map"].data_ptr(), npix1, L.ACT_RELU, dz1.data_ptr(), ld_in, None, None, data_only)
    k1, sld = st["k1"], st["sld"]
    if not data_only:
        self._gemm(a=dz1.data_ptr(), a_rows=npix1, lda=ld_in, a_mn=True, b=st["col16"].data_ptr(), b_rows=npix1, ldb=sld,
                   b_mn=True, m=in_dim, n=k1, kc=npix1, split_k=self._split_k(in_dim, k1, npix1), alpha_ptr=inv,
                   out_f32=self.G(pe[0].weight), ld_o32=k1, target=self.bwd_ops)
    if self.want_dx:
        # the image gradient (fp32 NCHW, like x): the backward of conv1, 3x3 / stride 2 / pad 1, as a gather
        cin = m.cfg["in_chans"]
        self.dx = nb.new("stem.dx", (B, cin, self.H, self.W), torch.float32)
        if cin == 3:
            self._op(ops, "fvit_stem_conv_dgrad", dz1.data_ptr(), ld_in, B, self.H, self.W, pe[0].weight.data_ptr(),
                     in_dim, inv, self.dx.data_ptr())
        else:
            # any other channel count: the tap products dcol = dz1 . W1 / S on tensor cores, then a gather of them
            ldc = _ru(k1, 4)
            dcol = nb.new("stem.dcol", (npix1, ldc), torch.float32)
            self._gemm(a=dz1.data_ptr(), a_rows=npix1, lda=ld_in, b=st["w1"].data_ptr(), b_rows=in_dim, ldb=sld, b_mn=True,
                       m=npix1, n=k1, kc=in_dim, alpha_ptr=inv, out_f32=dcol.data_ptr(), ld_o32=ldc, target=self.bwd_ops)
            self._op(ops, "fvit_stem_col2im", dcol.data_ptr(), ldc, B, cin, self.H, self.W, self.dx.data_ptr())


class ConvPartEmitters:
    """TrainPlan mixin: launch-list emitters of PatchEmbed, the conv levels and the Downsamples (the functions above take the
    plan as `self`)."""
    _bn_train = _bn_train
    _bn_finalize = _bn_finalize
    _emit_conv_part_train = _emit_conv_part_train
    _conv_level_train_buffers = _conv_level_train_buffers
    _emit_conv_blocks_train = _emit_conv_blocks_train
    _emit_downsample_train = _emit_downsample_train
    _bn_bwd = _bn_bwd
    _conv_wgrad = _conv_wgrad
    _emit_downsample_bwd = _emit_downsample_bwd
    _emit_conv_blocks_bwd = _emit_conv_blocks_bwd
    _emit_conv_part_bwd = _emit_conv_part_bwd
