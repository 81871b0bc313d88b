"""Forward(train)/backward emitters of TrainPlan (methods; imported into the class body).

Every function appends launches to plan.ops (train forward) or plan.bwd_ops. Shapes / row maps are the
ones built by Plan (engine.py); `sv` dicts hold the activations saved for the backward pass.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lib as L
from .engine import P, _ru, norm_kind


def _drop_buf(self, name: str, rate: float, groups: int, group_size: int):
    """row-scale vector (mask / keep per row) of one stochastic-depth site (timm DropPath: one Bernoulli draw
    per leading index — per window for x, per image for carrier tokens and ConvBlocks; fv.py:500,630,652).
    Returns the device pointer or None when the rate is 0."""
    if rate <= 0.0:
        return None
    buf = self.bufs.new(name + ".droppath", (groups * group_size,), torch.float32)
    self.drop_specs.append(dict(name=name, buf=buf, groups=groups, gs=group_size, keep=1.0 - rate))
    return buf.data_ptr()


def _gen_drop_masks(self) -> None:
    forced = getattr(self, "forced_drop_masks", None) or {}
    for d in self.drop_specs:
        if d["name"] in forced:
            m = forced[d["name"]].to(device=d["buf"].device, dtype=torch.float32)
        else:
            m = torch.bernoulli(torch.full((d["groups"],), d["keep"], device=d["buf"].device)) / d["keep"]
        d["buf"].view(d["groups"], d["gs"]).copy_(m.view(-1, 1).expand(d["groups"], d["gs"]))


# ====================================================================================== forward (train)
def _build_forward(self) -> None:
    m, B = self.model, self.B
    cfg = m.cfg
    self.drop_specs: list[dict] = []
    self._block_counter = 0
    self._bn_modules = [mod for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    self._bn_batch_stats: list = []   # BatchNorms this forward normalises with batch statistics (_bn_finalize)
    self.lv: list[dict] = []          # per-level geometry/buffers (+ "sv": saved activations)
    self.ds: list[dict] = []          # per-downsample saved state
    self._level_of: dict[int, dict] = {}
    prev = self._emit_conv_part_train()
    Hc, Wc, Cc = prev["H"], prev["W"], prev["C"]
    for i, level in enumerate(m.levels):
        if level.conv:
            continue
        if i > self.stop_level:   # levels mode: the forward ends at the highest requested level
            break
        Hc, Wc, Cc = (Hc + 1) // 2, (Wc + 1) // 2, Cc * 2
        tl = self._token_level_buffers(i, level, Cc, Hc, Wc)
        # gradient buffer mirroring xs, plus one guaranteed-zero row at the end
        tl["level_index"] = i
        tl["g"] = self.bufs.new(f"l{i}.g", (tl["xs"].shape[0] + 1, Cc), torch.float32)
        tl["zero_row"] = tl["xs"].shape[0]
        if tl["padded"]:
            self.ops.append(("zero", tl["xs"], "memset"))
        self._emit_downsample_train(i - 1, prev, tl)
        self._emit_token_level_train(i, level, tl)
        tl["kind"] = "tok"
        self._level_of[i] = tl
        self.lv.append(tl)
        prev = tl
    self.feat = prev
    if self.kind == "levels":
        self._emit_dense_outputs()
        # num_batches_tracked counts the BatchNorms that ran on batch statistics (not the frozen prefix's, not the
        # levels above the last requested one)
        self._bn_modules = self._bn_batch_stats
    else:
        self._emit_head_train(prev)
        if self.eval_grad:
            self._bn_modules = []     # (running statistics: num_batches_tracked stays)


def _level_rows(lv: dict) -> tuple:
    """(fp32 activation, row map of the B*H*W pixels) of a level's output: the zero-bordered conv map or the
    window-major token buffer through its crop map (any-res window padding and carrier rows excluded)"""
    if lv["kind"] == "conv":
        return lv["x32"], lv["pix"]
    return lv["xs"], lv["crop_map"]


def _const_vec(self, value: float, n: int) -> torch.Tensor:
    cache = self.__dict__.setdefault("_const_vecs", {})
    if (value, n) not in cache:
        cache[(value, n)] = self.bufs.new(f"const.{value}.{n}", (n,), torch.float32).fill_(value)
    return cache[(value, n)]


def _emit_dense_outputs(self) -> None:
    """Levels mode forward tail: every requested level output (x before its Downsample, live in the level's buffer
    until the plan's next forward: the backward never writes it) as an NCHW fp32 map in a static buffer, through its
    BatchNorm2d with batch statistics (fvit_colstats_pivot_f32 -> fvit_bn_finalize_pivot, which also updates the running
    statistics -> fvit_feature_map_fwd), through a frozen BatchNorm (fvit_affine_fold of its running statistics ->
    fvit_feature_map_fwd), through a channel LayerNorm (fvit_feature_map_ln_fwd, which saves the per-pixel mean / rstd),
    or raw.
    Eval plan (engine_train._EvalDenseGradFunction): the outputs come from the inference launch list, so this forward
    writes no BatchNorm output map; it only keeps each norm's running mean / rstd for the backward's xhat (one
    fvit_affine_fold with unit weight and zero bias: rstd = rsqrt(running_var + eps), nothing updated). Frozen
    BatchNorms and LayerNorms run as in train mode (their math does not depend on it)."""
    B, nb = self.B, self.bufs
    self.dense, self.outputs = [], []
    tot = 1
    for k, (i, bn) in enumerate(self.spec["outs"]):
        lv = self._level_of[i]
        x, rows = _level_rows(lv)
        C, H, W = lv["C"], lv["H"], lv["W"]
        T = H * W
        out = None if self.eval_grad else nb.new(f"dense.out{k}", (B, C, H, W), torch.float32)
        kind = None if bn is None else norm_kind(bn)
        d = dict(level=i, lv=lv, x=x, rows=rows, C=C, T=T, bn=bn if kind == "bn" else None, norm=bn, kind=kind, out=out,
                 dy=nb.new(f"dense.dy{k}", (B, C, H, W), torch.float32), acc=tot)
        tot += 2 * _ru(C, 4)
        if bn is not None and bn.weight.numel() != C:
            raise L.FvitError(f"the norm of level {i} has {bn.weight.numel()} features, the level has {C} channels")
        if kind in ("frozen", "ln"):
            if out is None:
                out = nb.new(f"dense.out{k}", (B, C, H, W), torch.float32)
            if kind == "frozen":   # running statistics, never written
                sc = nb.new(f"dense.norm{k}.scale", (C,), torch.float32)
                sh = nb.new(f"dense.norm{k}.shift", (C,), torch.float32)
                self._op(self.ops, "fvit_affine_fold", sc.data_ptr(), sh.data_ptr(), C, bn.weight.data_ptr(),
                         bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(), float(bn.eps), None,
                         None)
                self._op(self.ops, "fvit_feature_map_fwd", x.data_ptr(), C, rows.data_ptr(), B, T, C, sc.data_ptr(),
                         sh.data_ptr(), out.data_ptr())
                d.update(sc=sc, mu=None, rs=None)
            else:
                mu = nb.new(f"dense.norm{k}.pmean", (B * T,), torch.float32)
                rs = nb.new(f"dense.norm{k}.prstd", (B * T,), torch.float32)
                self._op(self.ops, "fvit_feature_map_ln_fwd", x.data_ptr(), C, rows.data_ptr(), B, T, C,
                         bn.weight.data_ptr(), bn.bias.data_ptr(), float(bn.eps), out.data_ptr(), mu.data_ptr(),
                         rs.data_ptr())
                d.update(mu=None, rs=None, pmean=mu, prstd=rs)
            d["out"] = out
            self.dense.append(d)
            if not self.eval_grad:
                self.outputs.append(out)
            continue
        if self.eval_grad:
            if bn is not None:
                rs = nb.new(f"dense.norm{k}.rstd", (C,), torch.float32)
                self._op(self.ops, "fvit_affine_fold", rs.data_ptr(), nb.new(f"dense.norm{k}.nshift", (C,), torch.float32).data_ptr(),
                         C, _const_vec(self, 1.0, C).data_ptr(), _const_vec(self, 0.0, C).data_ptr(),
                         bn.running_mean.data_ptr(), bn.running_var.data_ptr(), float(bn.eps), None, None)
                d.update(mu=bn.running_mean, rs=rs)
            else:
                d.update(mu=None, rs=None)
            self.dense.append(d)
            continue
        if bn is not None:
            st = self._bn_train(f"dense.norm{k}", bn, B * T)
            self._op(self.ops, "fvit_colstats_pivot_f32", x.data_ptr(), C, rows.data_ptr(), B * T, C, st["pivot"].data_ptr(),
                     st["st"][0].data_ptr(), st["st"][1].data_ptr())
            self._bn_finalize(st)
            d.update(sc=st["sc"], sh=st["sh"], mu=st["mu"], rs=st["rs"])
        else:
            d.update(sc=_const_vec(self, 1.0, C), sh=_const_vec(self, 0.0, C), mu=None, rs=None)
        self._op(self.ops, "fvit_feature_map_fwd", x.data_ptr(), C, rows.data_ptr(), B, T, C, d["sc"].data_ptr(),
                 d["sh"].data_ptr(), out.data_ptr())
        self.dense.append(d)
        self.outputs.append(out)
    # backward-side accumulators, cleared by every backward's prologue: [0] = max |dy| over all outputs, then per
    # output the per-channel sums s1 = sum dy, s2 = sum dy * xhat of the statistics pass
    self._dense_acc = nb.new("dense.acc", (tot,), torch.float32)
    acc = self._dense_acc.data_ptr()
    for d in self.dense:
        d["s1"], d["s2"] = acc + 4 * d["acc"], acc + 4 * (d["acc"] + _ru(d["C"], 4))
        bn = d["bn"]
        self._op(self._scale_ops, "fvit_feature_map_bwd_stats", d["dy"].data_ptr(), d["x"].data_ptr(), d["C"],
                 d["rows"].data_ptr(), B, d["T"], d["C"], P(d["mu"]), P(d["rs"]), d["s1"] if bn is not None else None,
                 d["s2"] if bn is not None else None, acc)
    self._op(self._scale_ops, "fvit_grad_scale_finalize", acc, 64.0, ("scal", 0))


def _inject(self, level: int, g=True) -> None:
    """Backward: add the gradients of the requested outputs of `level` to the level's residual-stream gradient g
    (scaled by S). Called right after g is complete from above (the Downsample backward wrote it; for the top level:
    the cleared buffer), before the level's own blocks read it. g=False: only the norm's weight / bias gradients
    (an output inside the frozen prefix)."""
    if self.kind != "levels":
        return
    for d in self.dense:
        if d["level"] != level:
            continue
        bn, lv = d["bn"], d["lv"]
        if d["kind"] == "ln":   # per-pixel statistics: the same backward in train and eval mode
            ln = d["norm"]
            self._op(self.bwd_ops, "fvit_feature_map_ln_bwd", d["dy"].data_ptr(), d["x"].data_ptr(), d["C"],
                     d["rows"].data_ptr(), self.B, d["T"], d["C"], d["pmean"].data_ptr(), d["prstd"].data_ptr(),
                     ln.weight.data_ptr(), ("scal", 0), None, lv["g"].data_ptr() if g else None, d["C"],
                     self.G(ln.weight), self.G(ln.bias))
            continue
        if d["kind"] == "frozen":   # a fixed per-channel scale of dy, no parameters
            if g:
                self._op(self.bwd_ops, "fvit_feature_map_eval_bwd", d["dy"].data_ptr(), d["rows"].data_ptr(), self.B,
                         d["T"], d["C"], d["sc"].data_ptr(), _const_vec(self, 1.0, d["C"]).data_ptr(), None, None,
                         ("scal", 0), None, lv["g"].data_ptr(), d["C"], None, None)
            continue
        if bn is None and not g:
            continue
        if self.eval_grad:   # running statistics: a per-channel scale of dy, and dw / dbeta straight from the stats pass
            self._op(self.bwd_ops, "fvit_feature_map_eval_bwd", d["dy"].data_ptr(), d["rows"].data_ptr(), self.B, d["T"],
                     d["C"], P(d["rs"]), bn.weight.data_ptr() if bn is not None else None,
                     d["s1"] if bn is not None else None, d["s2"] if bn is not None else None, ("scal", 0), None,
                     lv["g"].data_ptr() if g else None, d["C"], self.G(bn.weight) if bn is not None else None,
                     self.G(bn.bias) if bn is not None else None)
            continue
        self._op(self.bwd_ops, "fvit_feature_map_bwd", d["dy"].data_ptr(), d["x"].data_ptr(), d["C"],
                 d["rows"].data_ptr(), self.B, d["T"], d["C"], P(d["mu"]), P(d["rs"]),
                 bn.weight.data_ptr() if bn is not None else None, d["s1"] if bn is not None else None,
                 d["s2"] if bn is not None else None, ("scal", 0), None, lv["g"].data_ptr() if g else None, d["C"],
                 self.G(bn.weight) if bn is not None else None, self.G(bn.bias) if bn is not None else None)


def _posemb_train(self, nm: str, tpe, coords: torch.Tensor, Cc: int, own: bool = False) -> dict:
    """Plan._emit_pos_embed saving the MLP's hidden activations, plus the scratch slice of its output gradient"""
    hidden = self.bufs.new(nm + ".hidden", (coords.shape[0], 512), torch.float32)
    pe = self._emit_pos_embed(nm, tpe, coords, Cc, hidden=hidden, own=own)
    pe["dout"] = ("scr", self._scratch(nm + ".dpe", pe["npts"] * Cc))
    return pe


def _bias_train(self, nm: str, rpb, S: int, own: bool = False) -> dict:
    """Plan._emit_bias saving the table MLP's hidden activations, plus the scratch slices of the bias and table
    gradients"""
    npts = rpb.relative_coords_table.shape[1] * rpb.relative_coords_table.shape[2]
    hidden = self.bufs.new(nm + ".hidden", (npts, 512), torch.float32)
    bs = self._emit_bias(nm, rpb, S, hidden=hidden, own=own)
    bs["dbias"] = ("scr", self._scratch(nm + ".dbias", rpb.num_heads * S * S))
    bs["dtable"] = ("scr", self._scratch(nm + ".dtable", npts * rpb.num_heads))
    return bs


def _attn_fwd_train(self, nm: str, attn, gamma, rows: int, groups: int, S: int, y16, qkv, ao, bias, stream_buf,
                    u16, rs=None) -> dict:
    """Train-mode Plan._emit_attention: the three-launch attention with the layer scale un-folded, so that the branch
    output u = proj(...) + b can be saved (u16) for the layer-scale gradient."""
    Cc, h, hd = attn.qkv.in_features, attn.num_heads, attn.head_dim
    hdp = self._head_pad(hd)
    kind = self._attn_kind(S, hdp)
    if kind == "tile" and S % 4 == 0 and _attn_bwd_entry(S, hdp, True) != "fvit_attn_tc_bwd":
        # one window per 128-row tile either way; the key-loop forward also writes the log-sum-exp rows its tensor-core
        # backward needs (fvit_attn_tc_bwd stops at 64-row window slots, and at 63 tokens for 80-wide heads: without
        # this, 65..128-token windows -- any-res models with 8 x 8 ... 11 x 11 windows -- would train through the SIMT
        # backward)
        kind = "loop"
    use_tc = kind != "simt"
    if not use_tc:
        hdp = hd
    Cp = h * hdp
    wq, ldq, qb_ptr, wp, ldp = self._pack_attention(nm, attn, hdp)
    self._gemm(a=y16.data_ptr(), a_rows=rows, lda=Cc, b=wq.data_ptr(), ldb=ldq, m=rows, n=3 * Cp, kc=Cc,
               col_shift=qb_ptr, out_f16=qkv.data_ptr(), ld_o16=3 * Cp, flops=2.0 * rows * 3 * Cc * Cc)
    scale = float(getattr(attn, "scale", hd ** -0.5))   # qk_scale or head_dim ** -0.5 (fv.py:544)
    lse = None
    if kind == "loop":
        lse = self.bufs.new(nm + ".lse", (rows, h), torch.float32)   # log-sum-exp rows, read by the backward kernel
        self._op(self.ops, "fvit_attn_loop_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hdp, bias["out"].data_ptr(),
                 scale, ao.data_ptr(), Cp, lse.data_ptr())
    elif use_tc:
        self._op(self.ops, "fvit_attn_tc_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hdp, bias["out"].data_ptr(),
                 scale, ao.data_ptr(), Cp)
    else:
        self._op(self.ops, "fvit_attn_core_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hd, bias["out"].data_ptr(),
                 scale, ao.data_ptr(), Cp, None)
    self.op_flops[len(self.ops) - 1] = 4.0 * groups * h * S * S * hd
    # x += droppath_row * gamma * u, u = proj(...) + b saved (u16) when gamma is a layer-scale parameter
    ls = gamma if isinstance(gamma, torch.Tensor) else None
    u16 = u16 if ls is not None else None
    n = attn.proj.weight.shape[0]
    self._gemm(a=ao.data_ptr(), a_rows=rows, lda=Cp, b=wp.data_ptr(), ldb=ldp, m=rows, n=n, kc=Cp,
               col_shift=P(attn.proj.bias), col_scale2=P(ls), row_scale=rs, out_pre16=P(u16),
               ld_pre16=n if ls is not None else 0, resid=stream_buf, ld_resid=n, out_f32=stream_buf, ld_o32=n,
               flops=2.0 * rows * n * Cc)
    return dict(nm=nm, rs=rs, attn=attn, wq=wq, ldq=ldq, wp=wp, ldp=ldp, hd=hd, hdp=hdp, Cp=Cp, use_tc=use_tc, kind=kind, lse=lse,
                scale=scale, S=S, groups=groups, rows=rows, qkv=qkv, ao=ao, y16=y16, bias=bias, u16=u16)


def _emit_token_level_train(self, i: int, level, tl: dict) -> None:
    B, Cc, S, ncw, ws = self.B, tl["C"], tl["S"], tl["ncw"], tl["ws"]
    nW, n_ct = tl["nW"], tl["n_ct"]
    nb = self.bufs
    xs_ptr = tl["xs"].data_ptr()
    has_ct = ncw > 0
    hid = int(Cc * self.model.cfg["mlp_ratio"])
    heads = level.blocks[0].attn.num_heads
    Cp = heads * self._head_pad(Cc // heads)
    rows = nW * S
    tl["blocks_sv"] = []
    if level.do_gt and has_ct:
        tk = level.global_tokenizer
        (kh, sh_, oh), (kw, sw_, ow) = tl["pool"]
        entry = "fvit_token_init_nchw_fwd" if tl["tokens"] == "nchw" else "fvit_token_init_fwd"
        self._op(self.ops, entry, xs_ptr, Cc, tl["pix_map"].data_ptr(), B, tl["Hp"], tl["Wp"], Cc,
                 tk.pos_embed.weight.data_ptr(), tk.pos_embed.bias.data_ptr(), kh, kw, sh_, sw_, oh, ow,
                 tl["ct_rows"].data_ptr(), xs_ptr, Cc)

    def new16(name, r, c):
        return nb.new(name, (r, c), torch.float16)

    def new32(name, r):
        return nb.new(name, (r,), torch.float32)

    for j, blk in enumerate(level.blocks):
        nm = f"l{i}.b{j}"
        key = f"levels.{i}.blocks.{j}"
        rate = self._drop_rate(i)
        self._block_counter += 1
        sv: dict = dict(blk=blk)
        sv["rs_attn"] = self._drop_buf(key + ".attn", rate, nW, S)
        sv["rs_mlp"] = self._drop_buf(key + ".mlp", rate, nW, S)
        if has_ct:
            sv["rs_hat_attn"] = self._drop_buf(key + ".hat_attn", rate, B, n_ct)
            sv["rs_hat_mlp"] = self._drop_buf(key + ".hat_mlp", rate, B, n_ct)
        sv["pe"] = self._posemb_train(nm + ".pe", blk.pos_embed, tl["pe_coords"], Cc, own=tl["own_tables"])
        if has_ct:
            ctr_ptr = xs_ptr + tl["ctr0"] * Cc * 4
            rows_c = B * n_ct
            sv["hat_pe"] = None
            if tl["hat_pe_coords"] is not None:
                sv["hat_pe"] = self._posemb_train(nm + ".hat_pe", blk.hat_pos_embed, tl["hat_pe_coords"], Cc,
                                                  own=tl["own_tables"])
            c = dict(y1=new16(nm + ".c.y1", rows_c, Cc), xh1=new16(nm + ".c.xh1", rows_c, Cc), rs1=new32(nm + ".c.rs1", rows_c),
                     mu1=new32(nm + ".c.mu1", rows_c), y2=new16(nm + ".c.y2", rows_c, Cc), xh2=new16(nm + ".c.xh2", rows_c, Cc),
                     rs2=new32(nm + ".c.rs2", rows_c), mu2=new32(nm + ".c.mu2", rows_c),
                     qkv=new16(nm + ".c.qkv", rows_c, 3 * Cp), ao=new16(nm + ".c.ao", rows_c, Cp),
                     p=new16(nm + ".c.p", rows_c, hid), h=new16(nm + ".c.h", rows_c, hid),
                     u1=new16(nm + ".c.u1", rows_c, Cc), u2=new16(nm + ".c.u2", rows_c, Cc))
            sv["c"] = c
            self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, tl["ct_gather"].data_ptr(), rows_c, Cc,
                     sv["hat_pe"]["out"].data_ptr() if sv["hat_pe"] else None, n_ct, 0, ctr_ptr, Cc,
                     blk.hat_norm1.weight.data_ptr(), blk.hat_norm1.bias.data_ptr(), float(blk.hat_norm1.eps),
                     c["y1"].data_ptr(), Cc, None, c["mu1"].data_ptr(), c["rs1"].data_ptr(), c["xh1"].data_ptr(), Cc)
            sv["c_bias"] = self._bias_train(nm + ".hat_bias", blk.hat_attn.pos_emb_funct, n_ct, own=tl["own_tables"])
            sv["c_attn"] = self._attn_fwd_train(nm + ".hat_attn", blk.hat_attn, blk.gamma1, rows_c, B, n_ct, c["y1"],
                                                c["qkv"], c["ao"], sv["c_bias"], ctr_ptr, c["u1"], sv["rs_hat_attn"])
            self._op(self.ops, "fvit_ln_fwd", ctr_ptr, Cc, None, rows_c, Cc, None, 1, 0, None, 0,
                     blk.hat_norm2.weight.data_ptr(), blk.hat_norm2.bias.data_ptr(), float(blk.hat_norm2.eps),
                     c["y2"].data_ptr(), Cc, None, c["mu2"].data_ptr(), c["rs2"].data_ptr(), c["xh2"].data_ptr(), Cc)
            sv["c_mlp"] = self._mlp_fwd_train(nm + ".hat_mlp", blk.hat_mlp, blk.gamma2, rows_c, c["y2"], c["p"], c["h"],
                                              ctr_ptr, c["u2"], sv["rs_hat_mlp"])
        w = dict(y1=new16(nm + ".w.y1", rows, Cc), xh1=new16(nm + ".w.xh1", rows, Cc), rs1=new32(nm + ".w.rs1", rows),
                 mu1=new32(nm + ".w.mu1", rows), y2=new16(nm + ".w.y2", rows, Cc), xh2=new16(nm + ".w.xh2", rows, Cc),
                 rs2=new32(nm + ".w.rs2", rows), mu2=new32(nm + ".w.mu2", rows), qkv=new16(nm + ".w.qkv", rows, 3 * Cp),
                 ao=new16(nm + ".w.ao", rows, Cp), p=new16(nm + ".w.p", rows, hid), h=new16(nm + ".w.h", rows, hid),
                 u1=new16(nm + ".w.u1", rows, Cc), u2=new16(nm + ".w.u2", rows, Cc))
        sv["w"] = w
        self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, tl["norm1_gather"].data_ptr() if has_ct else None, rows, Cc,
                 sv["pe"]["out"].data_ptr(), S, ncw, xs_ptr, Cc, blk.norm1.weight.data_ptr(), blk.norm1.bias.data_ptr(),
                 float(blk.norm1.eps), w["y1"].data_ptr(), Cc, None, w["mu1"].data_ptr(), w["rs1"].data_ptr(),
                 w["xh1"].data_ptr(), Cc)
        sv["w_bias"] = self._bias_train(nm + ".bias", blk.attn.pos_emb_funct, S, own=tl["own_tables"])
        sv["w_attn"] = self._attn_fwd_train(nm + ".attn", blk.attn, blk.gamma3, rows, nW, S, w["y1"], w["qkv"], w["ao"],
                                            sv["w_bias"], xs_ptr, w["u1"], sv["rs_attn"])
        self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, None, rows, Cc, None, 1, 0, None, 0, blk.norm2.weight.data_ptr(),
                 blk.norm2.bias.data_ptr(), float(blk.norm2.eps), w["y2"].data_ptr(), Cc, None, w["mu2"].data_ptr(),
                 w["rs2"].data_ptr(), w["xh2"].data_ptr(), Cc)
        sv["w_mlp"] = self._mlp_fwd_train(nm + ".mlp", blk.mlp, blk.gamma4, rows, w["y2"], w["p"], w["h"], xs_ptr, w["u2"],
                                          sv["rs_mlp"])
        if has_ct and blk.last and blk.do_propagation:
            g1 = blk.gamma1.data_ptr() if isinstance(blk.gamma1, torch.Tensor) else None
            self._op(self.ops, "fvit_propagate_fwd", xs_ptr, Cc, tl["prop_src"].data_ptr(), rows, Cc, g1)
            sv["prop"] = True
        tl["blocks_sv"].append(sv)
    # level-wide backward scratch
    tl["dz"] = nb.new(f"l{i}.dz", (max(rows, 1), Cc), torch.float16)
    tl["dy"] = nb.new(f"l{i}.dy", (max(rows, 1), Cc), torch.float16)
    tl["dp"] = nb.new(f"l{i}.dp", (max(rows, 1), hid), torch.float16)
    tl["dao"] = nb.new(f"l{i}.dao", (max(rows, 1), Cp), torch.float16)
    tl["dqkv"] = nb.new(f"l{i}.dqkv", (max(rows, 1), 3 * Cp), torch.float16)


def _mlp_fwd_train(self, nm: str, mlp, gamma, rows: int, y16, p16, h16, stream_buf, u16, rs=None) -> dict:
    n1, k1 = mlp.fc1.weight.shape
    w1, ld1 = self._pack_linear(nm + ".fc1", mlp.fc1)
    # fc1: gelu'(pre-activation) saved through out_pre16 (one erf evaluation yields GELU and its derivative, so the
    # fc2 data-gradient epilogue is a plain multiply: FVIT_ACT_MUL_AUX), GELU output is the fc2 operand
    self._gemm(a=y16.data_ptr(), a_rows=rows, lda=k1, b=w1.data_ptr(), ldb=ld1, m=rows, n=n1, kc=k1,
               col_shift=mlp.fc1.bias.data_ptr(), act=L.ACT_GELU, out_f16=h16.data_ptr(), ld_o16=n1,
               out_pre16=p16.data_ptr(), ld_pre16=n1, pre_is_grad=True)
    # fc2: x += droppath_row * gamma * u, u = fc2(h) saved (u16) when gamma is a layer-scale parameter
    n2, k2 = mlp.fc2.weight.shape
    w2, ld2 = self._pack_linear(nm + ".fc2", mlp.fc2)
    ls = gamma if isinstance(gamma, torch.Tensor) else None
    u16 = u16 if ls is not None else None
    self._gemm(a=h16.data_ptr(), a_rows=rows, lda=k2, b=w2.data_ptr(), ldb=ld2, m=rows, n=n2, kc=k2,
               col_shift=P(mlp.fc2.bias), col_scale2=P(ls), row_scale=rs, out_pre16=P(u16),
               ld_pre16=n2 if ls is not None else 0, resid=stream_buf, ld_resid=n2, out_f32=stream_buf, ld_o32=n2)
    return dict(rs=rs, mlp=mlp, w1=w1, ld1=ld1, w2=w2, ld2=ld2, rows=rows, y16=y16, p16=p16, h16=h16, u16=u16)


def _emit_head_train(self, prev: dict) -> None:
    """BatchNorm2d with batch statistics folded into the pool (fv.py:953-958 under .train()); the eval-grad plan folds
    the running statistics instead (fvit_pool_bn_eval_bwd reads them directly)."""
    m, B, nb = self.model, self.B, self.bufs
    nf = m.num_features
    T = prev["H"] * prev["W"]
    sN = nb.new("norm.scale", (nf,), torch.float32)
    tN = nb.new("norm.shift", (nf,), torch.float32)
    mu = rs = None
    if self.eval_grad:
        self._op(self.ops, "fvit_affine_fold", sN.data_ptr(), tN.data_ptr(), nf, m.norm.weight.data_ptr(),
                 m.norm.bias.data_ptr(), m.norm.running_mean.data_ptr(), m.norm.running_var.data_ptr(), float(m.norm.eps),
                 None, None)
    else:
        st = nb.new("norm.stats", (2, nf), torch.float32)
        self.fwd_zero.append(st)
        mu = nb.new("norm.mean", (nf,), torch.float32)
        rs = nb.new("norm.rstd", (nf,), torch.float32)
        pv = nb.new("norm.pivot", (nf,), torch.float32)
        # the fp32 residual stream carries per-channel offsets: moments about each channel's first value
        self._op(self.ops, "fvit_colstats_pivot_f32", prev["xs"].data_ptr(), nf, prev["crop_map"].data_ptr(), B * T, nf,
                 pv.data_ptr(), st[0].data_ptr(), st[1].data_ptr())
        self._op(self.ops, "fvit_bn_finalize_pivot", st[0].data_ptr(), st[1].data_ptr(), pv.data_ptr(), 0, float(B * T),
                 m.norm.weight.data_ptr(), m.norm.bias.data_ptr(), float(m.norm.eps), float(m.norm.momentum),
                 m.norm.running_mean.data_ptr(),
                 m.norm.running_var.data_ptr(), None, sN.data_ptr(), tN.data_ptr(), mu.data_ptr(), rs.data_ptr(), nf)
    pooled = nb.new("head.pooled", (B, _ru(nf, 8)), torch.float16)
    self._op(self.ops, "fvit_pool_affine_fwd", prev["xs"].data_ptr(), nf, prev["crop_map"].data_ptr(), B, T, nf,
             sN.data_ptr(), tN.data_ptr(), pooled.data_ptr(), pooled.stride(0))
    if self.kind == "pooled":
        # num_classes = 0: the head is nn.Identity and the pooled features are the output (fv.py:955-958); the fp16
        # classifier operand is widened to a fp32 output buffer (the eval plan returns the same fp16 values)
        pooled32 = nb.new("head.pooled32", (B, nf), torch.float32)
        self._op(self.ops, "fvit_affine_rows", pooled.data_ptr(), pooled.stride(0), None, B, nf,
                 _const_vec(self, 1.0, nf).data_ptr(), _const_vec(self, 0.0, nf).data_ptr(), L.ACT_NONE, None, 0,
                 pooled32.data_ptr(), nf, None, 0, None)
        self.outputs = [pooled32]
        self.head_sv = dict(pooled=pooled, mu=mu, rs=rs, T=T, nf=nf)
        return
    hw16, ldh = self._pack_linear("head", m.head)
    self.logits = nb.new("logits", (B, m.num_classes), torch.float32)
    self._gemm(a=pooled.data_ptr(), a_rows=B, lda=pooled.stride(0), b=hw16.data_ptr(), ldb=ldh, m=B, n=m.num_classes,
               kc=nf, col_shift=m.head.bias.data_ptr(), out_f32=self.logits.data_ptr(), ld_o32=m.num_classes)
    self.head_sv = dict(pooled=pooled, hw16=hw16, ldh=ldh, mu=mu, rs=rs, T=T, nf=nf)


# ====================================================================================== backward
def _build_backward(self) -> None:
    m = self.model
    # gradient buckets of the data-parallel all-reduce, in completion order. The flat buffer follows
    # .parameters() order (patch_embed, levels.0 .. levels.n, norm, head); the backward pass finishes
    # [levels.n, norm, head] first, then one transformer level at a time, then the conv part.
    # Transformer levels are cut further: a bucket point after every group of blocks whose gradients add up to
    # FVIT_BUCKET_MB (default 100 MB; fv4: every 2 level-2 blocks / every level-3 block), so that the reduction of a
    # level overlaps that level's own backward and no single burst lands on the few large conv weight-gradient launches
    # at the end. The rest of a level (downsample, tokenizer) goes with the level-end point.
    import os
    first = {}
    for name, p in m.named_parameters():
        if name.startswith("levels.") and id(p) in self._goff:
            first.setdefault(int(name.split(".")[1]), self._goff[id(p)])
    # (level norms outside the model have slices after [0, total): they are final once every injection ran, a bucket
    # point of their own at the end)
    total = self._n_model_flat
    group_floats = int(float(os.environ.get("FVIT_BUCKET_MB", "100")) * 1e6 / 4)
    self.grad_buckets = []

    def point(lo: int, hi: int) -> None:
        if hi > lo:
            self.grad_buckets.append((lo, hi))
            self.bwd_ops.append(("bucket", (lo, hi), "grad_bucket"))

    for lv in self.conv_lv:
        if lv["cpix"] is not lv["pix"]:
            # a window-padded conv level (conv_level_pad): its blocks' backward writes the padding rows of g, which
            # nothing above it does; they start every backward at zero
            self.bwd_ops.append(("zero", lv["g"], "memset"))
    if self.kind is None:
        self._emit_head_bwd(self.feat)
    elif self.kind == "pooled":
        self._emit_pooled_bwd(self.feat)
    else:
        for d in self.dense:      # outputs of levels the backward does not reach: their norm's weight / bias gradients only
            if not self._needed(1 + d["level"]):
                self._inject(d["level"], g=False)
        if self.feat["kind"] == "tok" and self._needed(1 + self.feat["level_index"]):
            self._inject(self.feat["level_index"])   # (a conv top level: _emit_conv_part_bwd)
    toks = [lv for lv in self.lv]
    hi = total
    for idx in range(len(toks) - 1, -1, -1):
        tl = toks[idx]
        if not self._needed(1 + tl["level_index"]):
            break
        src = toks[idx - 1] if idx > 0 else self.conv_out
        if self.data_only[1 + tl["level_index"]]:   # no parameter gradient, so no bucket point: the data gradient alone
            self._emit_token_level_bwd(tl, None)
            if not self._needed(tl["level_index"]):
                break
            self._emit_downsample_bwd(tl["ds"], src, tl)
            self._inject(tl["level_index"] - 1)
            continue
        lo = first.get(tl["level_index"], hi)
        # offsets of the level's blocks in the flat buffer (module order = offset order, contiguous)
        spans = []
        for blk in m.levels[tl["level_index"]].blocks:
            offs = [(self._goff[id(q)], q.numel()) for q in blk.parameters()]
            spans.append((min(o for o, _ in offs), max(o + _ru(n, 64) for o, n in offs)))
        contiguous = all(a[1] == b[0] for a, b in zip(spans, spans[1:])) and spans and lo <= spans[0][0] and spans[-1][1] <= hi
        state = dict(top=spans[-1][1] if spans else hi)   # blocks above `top` have been handed to a bucket already

        def after_block(k: int, spans=spans, state=state) -> None:
            if group_floats > 0 and contiguous and k > 0 and state["top"] - spans[k][0] >= group_floats:
                point(spans[k][0], state["top"])
                state["top"] = spans[k][0]
        self._emit_token_level_bwd(tl, after_block)
        if contiguous and state["top"] < spans[-1][1]:   # some block groups are out already: the rest in two pieces
            point(spans[-1][1], hi)
            point(lo, state["top"])
        else:
            point(lo, hi)
        hi = lo
        if not self._needed(tl["level_index"]):
            break     # the Downsample in front of this level belongs to a stage nobody needs a gradient from: the end
        self._emit_downsample_bwd(tl["ds"], src, tl)
        self._inject(tl["level_index"] - 1)
    else:
        self._emit_conv_part_bwd()
    point(0, hi)
    point(total, self.gflat.numel())


def _emit_pooled_bwd(self, feat: dict) -> None:
    """Backward of the pooled features of a num_classes = 0 model: BatchNorm (batch statistics) + average pool, from
    the autograd gradient scaled by S on the device (fvit_vec_mul), as _emit_head_bwd does from the head GEMM."""
    B, nb, nf = self.B, self.bufs, self.head_sv["nf"]
    self._dpool_in = nb.new("grad.dpool_in", (B, nf), torch.float32)
    self.dense = [dict(dy=self._dpool_in)]
    dpool = nb.new("grad.dpool", (B, nf), torch.float32)
    self._op(self.bwd_ops, "fvit_vec_mul", self._dpool_in.data_ptr(), 1, ("scal", 0), 0, dpool.data_ptr(), B * nf)
    _pool_bn_bwd(self, feat, dpool)


def _pool_bn_bwd(self, feat: dict, dpool) -> None:
    """head norm + average pool backward from dpool (scaled by S) into the last level's gradient rows"""
    B, nb, hs, m = self.B, self.bufs, self.head_sv, self.model
    nf, T = hs["nf"], hs["T"]
    if self.eval_grad:
        self._op(self.bwd_ops, "fvit_pool_bn_eval_bwd", feat["xs"].data_ptr(), nf, feat["crop_map"].data_ptr(), B, T, nf,
                 m.norm.running_mean.data_ptr(), m.norm.running_var.data_ptr(), float(m.norm.eps),
                 m.norm.weight.data_ptr(), dpool.data_ptr(), nf, ("scal", 1), feat["g"].data_ptr(), nf,
                 self.G(m.norm.weight), self.G(m.norm.bias))
        return
    s12 = nb.new("grad.head_s12", (2, nf), torch.float32)
    self._op(self.bwd_ops, "fvit_pool_bn_bwd", feat["xs"].data_ptr(), nf, feat["crop_map"].data_ptr(), B, T, nf,
             hs["mu"].data_ptr(), hs["rs"].data_ptr(), m.norm.weight.data_ptr(), dpool.data_ptr(), nf,
             s12[0].data_ptr(), s12[1].data_ptr(), ("scal", 1), feat["g"].data_ptr(), nf, self.G(m.norm.weight),
             self.G(m.norm.bias))


def _emit_head_bwd(self, feat: dict) -> None:
    m, B, nb = self.model, self.B, self.bufs
    hs = self.head_sv
    nf, ncls = hs["nf"], m.num_classes
    ldl = _ru(ncls, 8)
    ncp = _ru(ncls, 4)   # the loss gradient is kept in rows padded to 16 bytes (any num_classes; padding stays zero)
    self._dlogits = nb.new("grad.dlogits", (B, ncp), torch.float32)
    self._ncls = ncls
    dl16 = nb.new("grad.dl16", (B, ldl), torch.float16)
    dpool = nb.new("grad.dpool", (B, nf), torch.float32)
    inv = ("scal", 1)
    ops = self.bwd_ops
    self._op(ops, "fvit_cast_scale_f16", self._dlogits.data_ptr(), ncp, None, B, ncp, None, ("scal", 0),
             dl16.data_ptr(), ldl, None)
    self._op(ops, "fvit_colsum", self._dlogits.data_ptr(), 0, ncp, None, None, 0, B, ncls, None, None,
             self.G(m.head.bias), None)
    # dW_head = dl^T pooled ; dpooled = dl W_head
    self._gemm(a=dl16.data_ptr(), a_rows=B, lda=ldl, a_mn=True, b=hs["pooled"].data_ptr(), b_rows=B,
               ldb=hs["pooled"].stride(0), b_mn=True, m=ncls, n=nf, kc=B, alpha_ptr=inv, out_f32=self.G(m.head.weight),
               ld_o32=nf, target=ops)
    self._gemm(a=dl16.data_ptr(), a_rows=B, lda=ldl, b=hs["hw16"].data_ptr(), b_rows=ncls, ldb=hs["ldh"], b_mn=True,
               m=B, n=nf, kc=ncls, out_f32=dpool.data_ptr(), ld_o32=nf, target=ops)
    _pool_bn_bwd(self, feat, dpool)


def _emit_attn_core_bwd(self, at: dict, dao, dqkv, groups: int, S: int, want_dbias: bool = True) -> None:
    """backward of the attention core: the wgmma tile kernel (S <= 64), the wgmma key-loop kernel (S > 64: needs the
    forward's output and log-sum-exp; per-pair partial dQ reduced into an fp32 scratch matrix -- any-res S = 148, the
    14 x 14 ... 48 x 48 windows of the 21k models) or the generic SIMT kernel."""
    attn = at["attn"]
    h, hd, hdp, Cp = attn.num_heads, at["hd"], at["hdp"], at["Cp"]
    ops = self.bwd_ops
    dbias = at["bias"]["dbias"] if want_dbias else None   # (NULL: every kernel skips the accumulation, fvit.h)
    self._before_write(dqkv.data_ptr())
    if at.get("kind") == "loop":
        # one scratch matrix per plan, sized for the largest attention of the model (the blocks' backward passes run
        # one after the other on the main stream; the kernel leaves nothing in it)
        need = groups * S * Cp
        scr = getattr(self, "_dq_scratch", None)
        if scr is None or scr.numel() < need:
            scr = self.bufs.new(f"grad.attn_dq32.{need}", (need,), torch.float32)   # (a smaller one stays alive: its
            self._dq_scratch = scr                                                  # launches keep their pointer)
        self._op(ops, "fvit_attn_loop_bwd_long", at["qkv"].data_ptr(), 3 * Cp, dao.data_ptr(), Cp, at["ao"].data_ptr(), Cp,
                 at["lse"].data_ptr(), groups, S, h, hdp, at["bias"]["out"].data_ptr(), at["scale"], dqkv.data_ptr(), 3 * Cp,
                 dbias, scr.data_ptr(), Cp)
    else:
        entry = _attn_bwd_entry(S, hdp, at["use_tc"])
        if entry == "fvit_attn_core_bwd" and _simt_bwd_smem(S, hd) > 227 * 1024:
            # refused here, while the plan is built, rather than by the kernel in the middle of the first backward
            level = at["nm"].split(".")[0][1:]
            raise L.FvitError(f"level {level} ({at['nm']}): the attention backward of {S}-token windows with {hd}-wide "
                              f"heads runs on fvit_attn_core_bwd, which holds a whole window in shared memory and needs "
                              f"{_simt_bwd_smem(S, hd) / 1024:.0f} KiB of the 227 KiB an SM has; this model trains only "
                              f"with smaller windows (or head widths the tensor-core kernels take)")
        self._op(ops, entry, at["qkv"].data_ptr(), 3 * Cp, dao.data_ptr(), Cp, groups, S, h, hd,
                 hdp, at["bias"]["out"].data_ptr(), at["scale"], dqkv.data_ptr(), 3 * Cp, dbias)
    self.bwd_flops[len(ops) - 1] = 10.0 * groups * h * S * S * hd


def _attn_bwd_entry(S: int, hdp: int, use_tc: bool) -> str:
    """tensor-core attention backward when the tile fits (S <= 64, head slices of 32/64/80, shared memory budget:
    S <= 63 at 80)"""
    if use_tc and S <= 64 and hdp in (32, 64, 80):
        ss = (S * S * 4 + 15) // 16 * 16
        if 1024 + (2 if hdp == 32 else 1) * 4 * 128 * hdp * 2 + 2 * 128 * 128 * 2 + 128 * 132 * 4 + ss + 128 <= 227 * 1024:
            return "fvit_attn_tc_bwd"
    return "fvit_attn_core_bwd"


def _simt_bwd_smem(S: int, hd: int) -> int:
    """shared memory of fvit_attn_core_bwd (train_sm100.cu): q, k, v, dO rows of hd + 1 floats, the [S, S + 1] P / dS
    matrix and one row vector, all for one whole window"""
    return (4 * S * (hd + 1) + S * (S + 1) + S) * 4


def _posemb_bwd(self, pe: dict) -> None:
    mod = pe["mod"]
    n0 = len(self.bwd_ops)
    self._op(self.bwd_ops, "fvit_cpb_mlp_bwd", pe["coords"].data_ptr(), pe["npts"], mod.cpb_mlp[2].weight.data_ptr(),
             pe["hidden"].data_ptr(), pe["dout"], pe["D"], None, self.G(mod.cpb_mlp[0].weight),
             self.G(mod.cpb_mlp[0].bias), self.G(mod.cpb_mlp[2].weight))
    self._bwd_side.update(range(n0, len(self.bwd_ops)))


def _bias_bwd(self, bs: dict) -> None:
    """Gradient of the relative-position bias MLP. Its inputs (this block's dbias / dtable scratch slices) are written
    once per backward pass and its outputs are parameter gradients nobody downstream reads: a leaf chain, run as a
    side branch of the launch graph (TrainPlan._bwd_side) so that these small latency-bound launches overlap the GEMMs."""
    rpb = bs["mod"]
    n0 = len(self.bwd_ops)
    self._op(self.bwd_ops, "fvit_attn_bias_bwd", bs["dbias"], bs["out"].data_ptr(), rpb.relative_position_index.data_ptr(),
             rpb.num_heads, bs["S"], rpb.window ** 2, ("scal", 1), bs["dtable"])
    self._op(self.bwd_ops, "fvit_cpb_mlp_bwd", rpb.relative_coords_table.data_ptr(), bs["npts"],
             rpb.cpb_mlp[2].weight.data_ptr(), bs["hidden"].data_ptr(), bs["dtable"], rpb.num_heads, None,
             self.G(rpb.cpb_mlp[0].weight), self.G(rpb.cpb_mlp[0].bias), self.G(rpb.cpb_mlp[2].weight))
    self._bwd_side.update(range(n0, len(self.bwd_ops)))


# TrainPlan._branch of a branch without layer scale
_ONE = dict(gamma=None, s=None, inv_s=("scal", 2), w_alpha=("scal", 1))


def _branch_entry(self, tl: dict, br: dict, g_ptr: int, rows: int, Cc: int, rs, u16, bias, data_only: bool) -> bool:
    """Entry of the backward of a residual branch x += gamma * (... + bias) on gradient rows g_ptr[0:rows]: tl["dz"] =
    fp16 operand copy of g (layer scale, its normaliser and the drop-path row scale folded in), and unless data_only the
    layer-scale gradient from the saved branch output u16 -- in one pass with the bias gradient (fvit_branch_grad)
    where that kernel applies. Returns whether the bias gradient was taken."""
    ops, dz = self.bwd_ops, tl["dz"].data_ptr()
    self._before_write(dz)
    if not data_only and Cc % 8 == 0 and bias is not None:
        has_g = br["gamma"] is not None
        self._op(ops, "fvit_branch_grad", g_ptr, Cc, rows, Cc, P(br["gamma"]), br["s"], rs, dz, Cc, br["w_alpha"],
                 self.G(bias), P(u16), Cc, ("scal", 1), self.G(br["gamma"]) if has_g else None)
        return True
    self._op(ops, "fvit_cast_scale_f16", g_ptr, Cc, None, rows, Cc, P(br["gamma"]), br["s"], dz, Cc, rs)
    if br["gamma"] is not None and not data_only:
        self._op(ops, "fvit_colsum", g_ptr, 0, Cc, None, u16.data_ptr(), Cc, rows, Cc, None, ("scal", 1),
                 self.G(br["gamma"]), rs)
    return False


def _mlp_bwd(self, tl: dict, ms: dict, gamma, g_ptr: int, rows: int, ln: nn.LayerNorm, xh, rs, data_only: bool) -> None:
    """Backward of x += gamma * fc2(gelu(fc1(LN(x)))) on gradient rows g_ptr[0:rows]; data_only: the data gradient
    alone (no weight-gradient GEMM, no bias / layer-scale / LayerNorm parameter gradient)."""
    mlp = ms["mlp"]
    Cc, hid = mlp.fc1.weight.shape[1], mlp.fc1.weight.shape[0]
    br = self._branch(gamma)
    dz, dp, dy = tl["dz"].data_ptr(), tl["dp"].data_ptr(), tl["dy"].data_ptr()
    bias_done = _branch_entry(self, tl, br, g_ptr, rows, Cc, ms["rs"], ms["u16"], mlp.fc2.bias, data_only)
    # fc2: dW2, db2, dp = (dz W2) o gelu'(p)   (p16 holds gelu'(p), saved by the forward epilogue); fc1's bias gradient =
    # column sums of dp, taken in the epilogue of the GEMM that produces dp
    fc1_db = (self.G(mlp.fc1.bias), ("scal", 1)) if mlp.fc1.bias is not None and not data_only else None
    self._linear_bwd(lin=mlp.fc2, w16=ms["w2"].data_ptr(), ldw=ms["ld2"], x16=ms["h16"].data_ptr(), ldx=hid, dz16=dz,
                     lddz=Cc, rows=rows, n_out=Cc, k_in=hid, br=br, dx16=dp, lddx=hid, dx_act=L.ACT_MUL_AUX,
                     dx_aux=ms["p16"].data_ptr(), ld_aux=hid, bias_done=bias_done, dx_colsum=fc1_db, data_only=data_only)
    self._linear_bwd(lin=mlp.fc1, w16=ms["w1"].data_ptr(), ldw=ms["ld1"], x16=ms["y16"].data_ptr(), ldx=Cc, dz16=dp,
                     lddz=hid, rows=rows, n_out=hid, k_in=Cc, br=_ONE, dx16=dy, lddx=Cc,
                     bias_done=mlp.fc1.bias is not None, data_only=data_only)
    self._ln_bwd(ln, dy, Cc, None, xh.data_ptr(), rs.data_ptr(), rows, Cc, g_ptr, None, 1, 0, data_only)


def _attn_bwd(self, tl: dict, at: dict, gamma, g_ptr: int, ln: nn.LayerNorm, xh, rs, pe, data_only: bool,
              in_map=None, carrier: bool = False) -> None:
    """Backward of x += gamma * proj(attn(qkv(LN(x + pe)))) on gradient rows g_ptr[0:rows], then of the positional
    embedding pe (_posemb_train, or None) added at the LayerNorm's input.
    Window tokens: the LayerNorm backward routes the gradient of the rows it gathered back through in_map
    (norm1_gather: the carrier slots to the raster carrier rows). Carrier tokens (carrier=True): g_ptr addresses the
    raster carrier rows of the level's gradient; hat_norm1's input gradient is accumulated there in place, then moved
    to the xs carrier rows hat_norm1 gathered from (ct_gather).
    data_only: the data gradient alone (no weight-gradient GEMM, no bias / layer-scale / attention-bias / positional-MLP
    / LayerNorm parameter gradient)."""
    ops = self.bwd_ops
    attn = at["attn"]
    Cc, h, hd, hdp, Cp = attn.qkv.in_features, attn.num_heads, at["hd"], at["hdp"], at["Cp"]
    rows, S, groups = at["rows"], at["S"], at["groups"]
    unpad = hdp != hd and not data_only   # parameter gradients of head-padded operands are un-padded
    br = self._branch(gamma)
    dz, dy, dao, dqkv = tl["dz"].data_ptr(), tl["dy"].data_ptr(), tl["dao"], tl["dqkv"]
    bias_done = _branch_entry(self, tl, br, g_ptr, rows, Cc, at["rs"], at["u16"], attn.proj.bias, data_only)
    # proj
    gWp = ("scr", self._scratch("dWproj_pad", Cc * Cp)) if unpad else None
    self._linear_bwd(lin=attn.proj, w16=at["wp"].data_ptr(), ldw=at["ldp"], x16=at["ao"].data_ptr(), ldx=Cp, dz16=dz,
                     lddz=Cc, rows=rows, n_out=Cc, k_in=Cp, br=br, gW=gWp, dx16=dao.data_ptr(), lddx=Cp, flops_k=Cc,
                     bias_done=bias_done, data_only=data_only)
    if unpad:
        self._op(ops, "fvit_unpad_heads_f32", gWp, Cp, self.G(attn.proj.weight), Cc, Cc, Cp, hd, hdp, 0, 1, None)
        self._bwd_side.add(len(ops) - 1)   # fresh scratch in, parameter gradient out: leaf launch
    # attention core
    _emit_attn_core_bwd(self, at, dao, dqkv, groups, S, want_dbias=not data_only)
    if not data_only:
        _bias_bwd(self, at["bias"])
    # qkv: with padded heads the weight-gradient GEMM scatters its rows through a row map, only the bias is un-padded
    gbq = ("scr", self._scratch("dbqkv_pad", 3 * Cp)) if unpad else None
    self._linear_bwd(lin=attn.qkv, w16=at["wq"].data_ptr(), ldw=at["ldq"], x16=at["y16"].data_ptr(), ldx=Cc,
                     dz16=dqkv.data_ptr(), lddz=3 * Cp, rows=rows, n_out=3 * Cp, k_in=Cc, br=_ONE,
                     gW_row_map=_unpad_row_map(self, 3 * h, hd, hdp) if unpad else None, bias_to=gbq, dx16=dy,
                     lddx=Cc, flops_k=Cc * (3 * Cc) / (3 * Cp), data_only=data_only)
    if unpad and attn.qkv.bias is not None:
        self._op(ops, "fvit_unpad_heads_f32", gbq, 1, self.G(attn.qkv.bias), 1, 3 * Cp, 1, hd, hdp, 1, 0, None)
        self._bwd_side.add(len(ops) - 1)   # fresh scratch in, parameter gradient out: leaf launch
    # LayerNorm (with the gather routing of the forward), then the positional embedding: its gradient summed over the
    # windows (over the images for the carriers)
    self._ln_bwd(ln, dy, Cc, None, xh.data_ptr(), rs.data_ptr(), rows, Cc, g_ptr, in_map, 1, int(not carrier),
                 data_only)
    if pe is not None and not data_only:
        self._op(ops, "fvit_group_sum", g_ptr, Cc, groups, S, 0 if carrier else tl["ncw"], Cc, ("scal", 1), pe["dout"])
        _posemb_bwd(self, pe)
    if carrier:
        self._op(ops, "fvit_scatter_add_rows", g_ptr, Cc, tl["g"].data_ptr(), Cc, tl["ct_gather"].data_ptr(), rows, Cc)


def _unpad_row_map(self, heads3: int, hd: int, hdp: int) -> int:
    """device int32 map: row r of a head-padded [heads3 * hdp, .] matrix -> row of the un-padded [heads3 * hd, .]
    parameter layout, -1 for padding rows (lets the qkv weight-gradient GEMM scatter straight into the flat gradient
    buffer instead of writing a padded scratch matrix that a second pass un-pads)."""
    cache = self.__dict__.setdefault("_unpad_maps", {})
    key = (heads3, hd, hdp)
    if key not in cache:
        r = torch.arange(heads3 * hdp)
        m = torch.where(r % hdp < hd, (r // hdp) * hd + r % hdp, torch.full_like(r, -1))
        cache[key] = self.bufs.i32(f"unpad_rows.{heads3}.{hd}.{hdp}", m)
    return cache[key].data_ptr()


def _emit_token_level_bwd(self, tl: dict, after_block=None) -> None:
    """Backward of a transformer level from its gradient rows tl["g"], the blocks in reverse order -- per block the
    carrier propagation, the window tokens' MLP and attention branches, then the carrier tokens' -- and then the global
    tokenizer. after_block(k) runs once block k's parameter gradients are final. A data-only level
    (TrainPlan.data_only): the data-gradient GEMMs, the attention core without dbias, LayerNorm dx and the carrier-token
    routing -- no weight-gradient GEMM, no bias / layer-scale / positional-MLP gradient."""
    B, Cc, S, ncw = self.B, tl["C"], tl["S"], tl["ncw"]
    nW, n_ct = tl["nW"], tl["n_ct"]
    ops = self.bwd_ops
    g_ptr = tl["g"].data_ptr()
    has_ct = ncw > 0
    rows = nW * S
    do = self.data_only[1 + tl["level_index"]]
    for sv in reversed(tl["blocks_sv"]):
        blk = sv["blk"]
        w = sv["w"]
        if sv.get("prop"):
            g1 = blk.gamma1 if isinstance(blk.gamma1, torch.Tensor) else None
            self._op(ops, "fvit_propagate_bwd", g_ptr, Cc, tl["xs"].data_ptr(), Cc, tl["prop_src"].data_ptr(), rows, Cc,
                     P(g1), ("scal", 1), self.G(g1) if g1 is not None and not do else None)
        # window branch (reverse order): MLP, attention + norm1 (routes carrier-slot gradients to the raster buffer)
        _mlp_bwd(self, tl, sv["w_mlp"], blk.gamma4, g_ptr, rows, blk.norm2, w["xh2"], w["rs2"], do)
        _attn_bwd(self, tl, sv["w_attn"], blk.gamma3, g_ptr, blk.norm1, w["xh1"], w["rs1"], sv["pe"], do,
                  in_map=tl["norm1_gather"].data_ptr() if has_ct else None)
        if has_ct:
            c = sv["c"]
            gc_ptr = g_ptr + tl["ctr0"] * Cc * 4   # the raster carrier rows
            _mlp_bwd(self, tl, sv["c_mlp"], blk.gamma2, gc_ptr, B * n_ct, blk.hat_norm2, c["xh2"], c["rs2"], do)
            _attn_bwd(self, tl, sv["c_attn"], blk.gamma1, gc_ptr, blk.hat_norm1, c["xh1"], c["rs1"], sv["hat_pe"], do,
                      carrier=True)
        if after_block is not None:
            after_block(tl["blocks_sv"].index(sv))   # this block's parameter gradients are final
    level = self.model.levels[tl["level_index"]]
    if level.do_gt and has_ct:
        tk = level.global_tokenizer
        (kh, sh_, oh), (kw, sw_, ow) = tl["pool"]
        nchw = "_nchw" if tl["tokens"] == "nchw" else ""
        if do:
            self._op(ops, f"fvit_token_init{nchw}_dgrad", g_ptr, Cc, tl["pix_map"].data_ptr(), tl["ct_rows"].data_ptr(), B, tl["Hp"],
                     tl["Wp"], Cc, tk.pos_embed.weight.data_ptr(), kh, kw, sh_, sw_, oh, ow, g_ptr, Cc)
            return
        self._op(ops, f"fvit_token_init{nchw}_bwd", g_ptr, Cc, tl["x0_16"].data_ptr(), Cc, tl["pix_map"].data_ptr(),
                 tl["ct_rows"].data_ptr(), B, tl["Hp"], tl["Wp"], Cc, tk.pos_embed.weight.data_ptr(), kh, kw, sh_, sw_, oh, ow,
                 ("scal", 1), g_ptr, Cc, self.G(tk.pos_embed.weight), self.G(tk.pos_embed.bias))


class TokenLevelEmitters:
    """TrainPlan mixin: launch-list emitters of the transformer levels, the head and the build drivers (the functions
    above take the plan as `self`; `_attn_bwd_entry` is a plain helper)."""
    _drop_buf = _drop_buf
    _gen_drop_masks = _gen_drop_masks
    _build_forward = _build_forward
    _posemb_train = _posemb_train
    _bias_train = _bias_train
    _attn_fwd_train = _attn_fwd_train
    _emit_token_level_train = _emit_token_level_train
    _mlp_fwd_train = _mlp_fwd_train
    _emit_head_train = _emit_head_train
    _emit_dense_outputs = _emit_dense_outputs
    _inject = _inject
    _emit_pooled_bwd = _emit_pooled_bwd
    _build_backward = _build_backward
    _emit_head_bwd = _emit_head_bwd
    _emit_attn_core_bwd = _emit_attn_core_bwd
    _posemb_bwd = _posemb_bwd
    _bias_bwd = _bias_bwd
    _mlp_bwd = _mlp_bwd
    _attn_bwd = _attn_bwd
    _unpad_row_map = _unpad_row_map
    _emit_token_level_bwd = _emit_token_level_bwd
