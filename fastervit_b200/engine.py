"""Execution engine: turns a FasterViT module + input shape into a static plan of libfvit_sm100.so
kernel launches over persistent device buffers, and runs it.

Data layout in HBM (all activations are token-major / NHWC row matrices):
  * conv levels (fv.py:502-512): zero-bordered maps, row = b*(H+2)*(W+2) + (y+1)*(W+2) + (x+1); a fp32
    copy carries the residual stream, a fp16 copy is the tensor-core operand. A 3x3/s1 convolution is a
    9-tap GEMM whose tap (dy,dx) shifts the A-operand rows by (dy-1)*(W+2)+(dx-1) (no im2col);
  * stride-2 convolutions (fv.py:434, 461) read four parity planes plane[(y&1)*2+(x&1)][b][(y>>1)+1][(x>>1)+1]
    with a zero top row / left column, which makes every tap a unit-stride shifted box as well;
  * transformer levels (fv.py:662-701): one fp32 buffer xs[nW*S + B*n_ct, C]; window w owns rows
    [w*S, (w+1)*S): its ct_size^2 carrier tokens first, then its ws*ws tokens (the `torch.cat` of
    fv.py:687 materialised once); the tail B*n_ct rows hold the raster-ordered carrier tokens while
    the carrier branch runs. window_partition / window_reverse / ct_dewindow / ct_window / cat / split
    (fv.py:83-109, 687, 695) never move data: they are int32 row maps consumed by the LayerNorm
    kernel (gather) and the GEMM epilogue (scatter).
Tensor-core operands are fp16, accumulation fp32, residual stream / LayerNorm / softmax / BN fp32.
"""
from __future__ import annotations

import ctypes as C
import gc

import torch
import torch.nn as nn

from . import lib as L

STEM_MAX_CIN = 64   # in_chans limit of the stem kernels (FVIT_STEM_MAX_CIN, include/fvit.h)
LN_MAX_C = 2560     # widest LayerNorm row of fvit_ln_fwd / fvit_ln_bwd / fvit_ln_dgrad (FVIT_LN_MAX_C, include/fvit.h)


def _ru(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def P(t):
    """device pointer of an optional tensor"""
    return None if t is None else t.data_ptr()


def norm_kind(m) -> str:
    """What a 2-D norm module computes, judged by what it is (callers bring their own classes):
    "bn"     nn.BatchNorm2d: batch statistics in train mode, running statistics in eval mode;
    "frozen" a fixed affine from running statistics: buffers weight / bias / running_mean / running_var, an eps and no
             parameters (torchvision.ops.FrozenBatchNorm2d, DETR-family copies of it);
    "ln"     a per-pixel LayerNorm over the channels (timm LayerNorm2d): an nn.LayerNorm subclass over one dimension
             with an elementwise affine and a bias.
    Anything else raises FvitError."""
    if isinstance(m, nn.BatchNorm2d):
        return "bn"
    bufs = dict(m.named_buffers(recurse=False))
    if (not any(True for _ in m.parameters()) and isinstance(getattr(m, "eps", None), float)
            and all(isinstance(bufs.get(n), torch.Tensor) and bufs[n].dim() == 1
                    for n in ("weight", "bias", "running_mean", "running_var"))):
        return "frozen"
    if (isinstance(m, nn.LayerNorm) and type(m) is not nn.LayerNorm and len(m.normalized_shape) == 1
            and m.elementwise_affine and m.weight is not None and m.bias is not None):
        return "ln"
    raise L.FvitError(f"unsupported norm {type(m).__name__}: accepted are nn.BatchNorm2d, a frozen BatchNorm (buffers "
                      "weight / bias / running_mean / running_var, an eps, no parameters) and a channel LayerNorm "
                      "(an nn.LayerNorm subclass such as timm's LayerNorm2d, one normalized dimension, affine, with a "
                      "bias)")


def norm_params(m) -> tuple:
    """the trainable tensors of a level norm (None: a raw output): weight and bias of a BatchNorm2d or a channel
    LayerNorm, none for a frozen BatchNorm"""
    return () if m is None or norm_kind(m) == "frozen" else (m.weight, m.bias)


# ---------------------------------------------------------------------------------- index maps
def _ct_dewindow_perm(cs: int, sr: list[int]) -> torch.Tensor:
    """raster position r -> window-major carrier index it is read from; the literal index algebra of
    ct_dewindow(ct, cs*sr[0], cs*sr[1], cs) (fv.py:96-101, call fv.py:673 / fvar.py:679)."""
    Wd, Hd = cs * sr[0], cs * sr[1]
    idx = torch.arange(Wd * Hd).view(1, Wd // cs, Hd // cs, cs, cs, 1)
    return idx.permute(0, 5, 1, 3, 2, 4).reshape(Wd * Hd)


def _ct_window_perm(cs: int, sr: list[int]) -> torch.Tensor:
    """window-major slot q (= window*cs*cs + slot) -> raster position it receives; the index algebra of
    ct_window(ct, cs*sr[0], cs*sr[1], cs).reshape(nW, cs*cs, C) (fv.py:104-109, 683-685)."""
    Wd, Hd = cs * sr[0], cs * sr[1]
    idx = torch.arange(Wd * Hd).view(1, Hd // cs, cs, Wd // cs, cs, 1)
    return idx.permute(0, 1, 3, 2, 4, 5).reshape(Wd * Hd)


def grid_coords(h: int, w: int, norm: int) -> torch.Tensor:
    """[h*w, 2] inputs of a rank-2 positional MLP (PosEmbMLPSwinv1D, fv.py:355-365): the 'ij' grid arange(h) x arange(w),
    shifted and divided by `norm`"""
    r, c = torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32)
    grid = torch.stack(torch.meshgrid(r, c, indexing="ij"))
    return ((grid - norm) / norm).flatten(1).t().contiguous()


def conv_level_pad(model, i: int, Hc: int, Wc: int) -> tuple[int, int]:
    """(Hb, Wb): the map a convolutional level runs on. The detection backbone pads every level, the convolutional ones
    included, to a multiple of its window and crops after (dino/models/dino/fastervit.py:686-707); classification
    models run conv levels on the map as it is."""
    if not getattr(model, "carriers_from_input", False):
        return Hc, Wc
    ws = model.levels[i].window_size
    return _ru(Hc, ws), _ru(Wc, ws)


def token_geometry(model, i: int, Hc: int, Wc: int) -> dict:
    """Window and carrier geometry of transformer level i for an Hc x Wc input map: the one function that decides it for
    the inference and the training plans.
      Hp, Wp, nwh, nww   the map padded to the window, and its window grid
      has_ct, sr         carrier tokens present; the carrier window grid the ct_dewindow / ct_window maps follow
      pool               ((kh, sh, oh), (kw, sw, ow)) of the tokenizer's average pool
      tokens             "map": tokenizer output (b, y, x) is carrier (y, x) of the grid (fv.py:733-738);
                         "nchw": the pooled NCHW map is read back as [oh*ow, C] tokens (fvit_token_init_nchw_fwd)
      pe_coords, hat_pe_coords   inputs of the window-token / carrier positional MLPs (None: no such MLP)
      own_tables         positional tables / biases are plan buffers, not the modules' `relative_bias`
    Classification models: the carrier grid is the sr_ratio fixed at construction (another window grid raises), the pool
    is TokenInitializer.pool and the positional grids are scaled by side // 2 (fv.py:355-360). The detection backbone
    (model.carriers_from_input, fastervit_b200.detection): everything follows the input -- carrier grid cs*nwh x cs*nww,
    pool from the padded map (dino/models/dino/fastervit.py:569-592), grids scaled by (h*w) // 2 (fastervit.py:192-196)."""
    level = model.levels[i]
    ws, cs = level.window_size, model.cfg["ct_size"]
    det = bool(getattr(model, "carriers_from_input", False))
    Hp, Wp = _ru(Hc, ws), _ru(Wc, ws)
    if not (model.any_res or det) and (Hp != Hc or Wp != Wc):
        raise L.FvitError(f"level {i}: {Hc}x{Wc} map is not a multiple of window {ws} "
                          "(use a *_any_res model for such resolutions)")
    nwh, nww = Hp // ws, Wp // ws
    has_ct = len(level.blocks) > 0 and level.blocks[0].has_carriers
    g = dict(Hp=Hp, Wp=Wp, nwh=nwh, nww=nww, has_ct=has_ct, sr=None, pool=None, tokens="map", hat_pe_coords=None,
             pe_coords=grid_coords(ws, ws, (ws * ws) // 2 if det else ws // 2), own_tables=det)
    if not has_ct:
        return g
    if det:
        pool = []
        for r in (Hp, Wp):
            out = int(cs * r / ws)
            stride = int(r / out)
            pool.append((r - (out - 1) * stride, stride, out))
        hg, wg = pool[0][2], pool[1][2]
        if (hg, wg) != (cs * nwh, cs * nww):
            raise L.FvitError(f"level {i}: carrier grid {hg}x{wg} does not tile the {nwh}x{nww} windows")
        g.update(sr=[nwh, nww], pool=pool, tokens="nchw", hat_pe_coords=grid_coords(hg, wg, (hg * wg) // 2))
        return g
    sr = list(level.sr_ratio)
    if sr != [nwh, nww]:
        raise L.FvitError(f"level {i}: input gives {nwh}x{nww} windows but the model was built for {sr}")
    n = int((cs * cs * sr[0] * sr[1]) ** 0.5)
    g.update(sr=sr, pool=level.global_tokenizer.pool if level.do_gt else None,
             hat_pe_coords=grid_coords(n, n, n // 2) if hasattr(level.blocks[0], "hat_pos_embed") else None)
    return g


class _Bufs:
    """Device buffer factory: zero-initialised persistent tensors, named for debugging."""

    def __init__(self, device):
        self.device = device
        self.named: dict[str, torch.Tensor] = {}
        self.nbytes = 0

    def new(self, name: str, shape, dtype) -> torch.Tensor:
        t = torch.zeros(shape, dtype=dtype, device=self.device)
        self.named[name] = t
        self.nbytes += t.numel() * t.element_size()
        return t

    def i32(self, name: str, host: torch.Tensor) -> torch.Tensor:
        t = host.to(torch.int32).contiguous().to(self.device)
        self.named[name] = t
        return t


def dependency_chains(ops: list) -> list[list[int]]:
    """Partition a list of plain launches (fn, args, name) into chains that may run concurrently: two launches that
    share a device-pointer argument (one writes what the other reads, e.g. the bias-table MLP and the gather that
    follows it) stay in list order inside one chain. Anything that is not a plain launch (host-side pseudo ops) makes
    the whole list one serial chain-less result ([]): the caller then runs it in order."""
    parent = list(range(len(ops)))

    def find(i: int) -> int:
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i
    owner: dict[int, int] = {}
    for i, (fn, args, _) in enumerate(ops):
        if isinstance(fn, str) or not isinstance(args, tuple):
            return []
        for a in args:
            if isinstance(a, int) and not isinstance(a, bool) and a >= (1 << 40):   # CUDA device pointers (0x7f.. range); sizes / strides are far below
                j = owner.setdefault(a, i)
                if j != i:
                    parent[find(i)] = find(j)
    groups: dict[int, list[int]] = {}
    for i in range(len(ops)):
        groups.setdefault(find(i), []).append(i)
    return list(groups.values())


class Plan:
    """Static launch list for one (batch, height, width, training) signature."""
    STEM_LD = 32  # fp16 row width of the stem im2col matrix (27 taps zero padded to 32; TMA zero-fills the rest of the K block)

    def __init__(self, model, B: int, H: int, W: int, training: bool, device):
        self.model, self.B, self.H, self.W, self.training, self.device = model, B, H, W, training, device
        self.lib = L.load()
        self.bufs = _Bufs(device)
        self.prep_ops: list[tuple] = []   # weight preparation (fp32 params -> packed fp16 / folded vectors)
        self.ops: list[tuple] = []        # the forward pass
        self._gemm_keep: list = []        # keeps ctypes structs alive
        self._x_args: list = []           # stem-conv calls that take the input pointer at run time
        self.op_flops: dict[int, float] = {}  # op index -> algorithmic FLOPs (GEMM launches)
        import os
        # with graphs on, a training plan's independent launches (weight re-packing, leaf gradient chains) run as
        # parallel branches of the graph (engine_train.py)
        self.use_graphs = os.environ.get("FVIT_CUDA_GRAPH", "1") != "0" and device.type == "cuda"
        self._graphs: dict = {}
        self._x_static = None
        self._deploy_mods: list = []
        self.marks: list[tuple[int, str, dict]] = []   # (ops issued so far, reference module name, where its output lives)
        self.check_ln_widths()
        self._build()

    # ---- per-module activation taps (parity tests against the reference's forward hooks) ---------
    def _mark(self, name: str, **where) -> None:
        self.marks.append((len(self.ops), name, where))

    def _extract(self, where: dict) -> torch.Tensor:
        """The activation a mark points at, in the reference's layout (NCHW maps / [nW, ws*ws, C] windows)."""
        B = self.B
        if where["kind"] == "conv":      # zero-bordered NHWC fp32 map
            lv = where["lv"]
            t = lv["x32"].view(B, lv["Hb"] + 2, lv["Wb"] + 2, lv["C"])[:, 1:lv["H"] + 1, 1:lv["W"] + 1]
            return t.permute(0, 3, 1, 2).clone()
        tl = where["tl"]
        if where["kind"] == "tok_map":   # window-major token buffer read through the (cropped) pixel map
            t = tl["xs"][tl["crop_map"].long()].view(B, tl["H"], tl["W"], tl["C"])
            return t.permute(0, 3, 1, 2).clone()
        nW, S, ncw = tl["nW"], tl["S"], tl["ncw"]   # "windows": HAT block output x (fv.py:701)
        return tl["xs"][:nW * S].view(nW, S, tl["C"])[:, ncw:].clone()   # (a copy: xs is rewritten by the next block)

    def debug_activations(self, x: torch.Tensor, prep: bool = True) -> dict[str, torch.Tensor]:
        """Run the forward launch list piecewise and return {reference module name: activation} at every mark —
        the per-module outputs the golden fixtures sample with forward hooks (oracle/make_golden.py)."""
        if prep:
            self.run_ops(self.prep_ops, None)
        out, done = {}, 0
        for upto, name, where in self.marks:
            self.run_ops(self.ops[done:upto], x)
            done = upto
            out[name] = self._extract(where)
        self.run_ops(self.ops[done:], x)
        return out

    def _deploy_guard(self, lst: list, start: int, mod) -> None:
        """ops lst[start:] derive mod.relative_bias from its MLP: skipped once mod.switch_to_deploy() was called
        (fv.py:263-269, 336-342 — the buffer then holds what a checkpoint or the last forward left there)"""
        for i in range(start, len(lst)):
            fn, args, name = lst[i]
            lst[i] = ("unless_deploy", (mod, fn, args), name)
        self._deploy_mods.append(mod)

    # ---- op emitters --------------------------------------------------------------------------
    def _op(self, target: list, name: str, *args) -> None:
        target.append((getattr(self.lib, name), args, name))

    def _gemm(self, *, a, a_rows, lda, b, ldb, m, n, kc, b_rows=0, taps=None, a_planes=1, a_plane_stride=0,
              a_mn=False, b_mn=False, b_taps=None, split_k=1, alpha_ptr=None, act=L.ACT_NONE, col_scale=None, col_shift=None, col_scale2=None, row_scale=None, aux=None, ld_aux=0,
              aux_scale=None, aux_shift=None, resid=None, ld_resid=0, row_map=None, out_f32=None, ld_o32=0,
              out_f16=None, ld_o16=0, out_pre16=None, ld_pre16=0, pre_is_grad=False, col_sum=None, col_sumsq=None,
              out_colsum=None, out_colsum_alpha=None, target=None, m_alg=None, flops=None) -> None:
        """Emit one fvit_gemm launch (fields: GemmArgs, include/fvit.h) into `target` (default: the forward list) and
        record its algorithmic FLOPs in op_flops / bwd_flops: `flops`, else 2*m_alg*n*kc*ntaps with m_alg = the number
        of output rows that are real work (pixels / tokens, without layout padding). A pointer may be symbolic,
        ("scal" | "scr", i): TrainPlan._finish_train resolves it once its device scalars and scratch exist."""
        g = L.GemmArgs()
        g.a_rows, g.lda, g.a_plane_stride, g.a_planes, g.a_mn_major = a_rows, lda, a_plane_stride, a_planes, int(a_mn)
        g.b_rows, g.ldb, g.b_mn_major = b_rows or n, ldb, int(b_mn)
        g.m, g.n, g.kc = m, n, kc
        taps = taps or [(0, 0)]
        g.ntaps = len(taps)
        for i, (s, p) in enumerate(taps):
            g.tap_shift[i], g.tap_plane[i] = s, p
        if b_taps is not None:   # conv weight gradient: taps folded into N (include/fvit.h: b_ntaps)
            assert len(taps) == 1 and a_mn and b_mn
            g.b_ntaps = len(b_taps)
            for i, sft in enumerate(b_taps):
                g.tap_shift[i] = sft
        g.split_k, g.alpha, g.act, g.pre_is_grad = split_k, 1.0, act, int(pre_is_grad)
        g.ld_aux, g.ld_resid, g.ld_out_f32, g.ld_out_f16, g.ld_out_pre16 = ld_aux, ld_resid, ld_o32, ld_o16, ld_pre16
        g._sym = {}
        for f, v in (("a", a), ("b", b), ("alpha_ptr", alpha_ptr), ("col_scale", col_scale), ("col_shift", col_shift),
                     ("col_scale2", col_scale2), ("row_scale", row_scale), ("aux", aux), ("aux_scale", aux_scale),
                     ("aux_shift", aux_shift), ("resid", resid), ("row_map", row_map), ("out_f32", out_f32),
                     ("out_f16", out_f16), ("out_pre16", out_pre16), ("col_sum", col_sum), ("col_sumsq", col_sumsq),
                     ("out_colsum", out_colsum), ("out_colsum_alpha", out_colsum_alpha)):
            if isinstance(v, tuple):
                g._sym[f] = v
            else:
                setattr(g, f, v)
        self._gemm_keep.append(g)
        lst = self.ops if target is None else target
        lst.append((self.lib.fvit_gemm, (C.byref(g),), "fvit_gemm"))
        if flops is None:
            flops = 2.0 * (m_alg if m_alg is not None else m) * n * kc * len(taps)
        if lst is self.ops:
            self.op_flops[len(lst) - 1] = flops
        elif lst is getattr(self, "bwd_ops", None):
            self.bwd_flops[len(lst) - 1] = flops

    # ---- weight preparation emitters ------------------------------------------------------------
    def _pack_linear(self, name: str, lin: nn.Linear) -> tuple[torch.Tensor, int]:
        n, k = lin.weight.shape
        ld = _ru(k, 8)
        w16 = self.bufs.new(name + ".w16", (n, ld), torch.float16)
        self._op(self.prep_ops, "fvit_cast_pad_f16", lin.weight.data_ptr(), k, w16.data_ptr(), ld, n, k, ld)
        return w16, ld

    def _pack_conv(self, name: str, conv: nn.Conv2d) -> tuple[torch.Tensor, int]:
        cout, cin = conv.weight.shape[:2]
        kc_pad = _ru(cin, 64)
        w16 = self.bufs.new(name + ".w16", (cout, 9 * kc_pad), torch.float16)
        self._op(self.prep_ops, "fvit_pack_conv3x3_f16", conv.weight.data_ptr(), w16.data_ptr(), cout, cin,
                 kc_pad, 0)
        return w16, 9 * kc_pad

    def _fold(self, name: str, n: int, bn: nn.BatchNorm2d | None = None, bias=None, ls=None):
        """(scale, shift) device vectors for the GEMM epilogue; see fvit_affine_fold."""
        sc = self.bufs.new(name + ".scale", (n,), torch.float32)
        sh = self.bufs.new(name + ".shift", (n,), torch.float32)
        self._op(self.prep_ops, "fvit_affine_fold", sc.data_ptr(), sh.data_ptr(), n,
                 P(bn.weight) if bn is not None else None, P(bn.bias) if bn is not None else None,
                 P(bn.running_mean) if bn is not None else None,
                 P(bn.running_var) if bn is not None else None,
                 float(bn.eps) if bn is not None else 0.0, P(bias), P(ls))
        return sc, sh

    # ---- plan construction ----------------------------------------------------------------------
    def _build(self) -> None:
        m, B = self.model, self.B
        cfg = m.cfg
        if self.training:
            raise L.FvitError("training-mode forward/backward kernels are not built yet in this round; "
                              "call model.eval() (there is no PyTorch fallback)")
        dim, in_dim, depths = cfg["dim"], cfg["in_dim"], cfg["depths"]
        nb = self.bufs
        # ---------------- stem: conv1 (SIMT, fp32) -> parity planes -> conv2 (tensor cores) -> L0
        H1, W1 = (self.H + 1) // 2, (self.W + 1) // 2     # after conv1
        H0, W0 = (H1 + 1) // 2, (W1 + 1) // 2             # after conv2 = level-0 map
        ld_in = _ru(in_dim, 8)
        pl_rows = B * (H0 + 1) * (W0 + 1)
        stem_planes = nb.new("stem.planes", (4 * pl_rows, ld_in), torch.float16)
        stem_map = self._parity_plane_map("stem.map", H1, W1)
        pe = m.patch_embed.conv_down
        s1, t1 = self._fold("stem.bn1", in_dim, pe[1])
        # conv1 (fv.py:458-460) on tensor cores: im2col rows [pixel, 9*in_chans -> stem_ld] (one HBM-bound
        # kernel), then a GEMM (one K block up to 7 channels) with the BN + ReLU epilogue scattering into the planes
        k1, sld = self.stem_cols()
        col16 = nb.new("stem.col16", (B * H1 * W1, sld), torch.float16)
        self._x_args.append(dict(B=B, cin=cfg["in_chans"], H=self.H, W=self.W, out=col16.data_ptr(), ldo=sld))
        self.ops.append(("im2col", len(self._x_args) - 1, "fvit_stem_im2col"))
        w1 = nb.new("stem.conv1.w16", (in_dim, sld), torch.float16)
        self._op(self.prep_ops, "fvit_cast_pad_f16", pe[0].weight.data_ptr(), k1, w1.data_ptr(), sld, in_dim, k1, sld)
        self._gemm(a=col16.data_ptr(), a_rows=B * H1 * W1, lda=sld, b=w1.data_ptr(), ldb=sld,
                   m=B * H1 * W1, n=in_dim, kc=sld, col_scale=s1.data_ptr(), col_shift=t1.data_ptr(),
                   act=L.ACT_RELU, row_map=stem_map.data_ptr(), out_f16=stem_planes.data_ptr(), ld_o16=ld_in,
                   flops=2.0 * B * H1 * W1 * in_dim * k1)

        lvl = self._conv_level_buffers(0, dim, H0, W0)
        self._zero_window_padding(lvl)
        w16, ldw = self._pack_conv("stem.conv2", pe[3])
        s2, t2 = self._fold("stem.bn2", dim, pe[4])
        self._gemm(a=stem_planes.data_ptr(), a_rows=pl_rows, lda=ld_in, a_planes=4,
                   a_plane_stride=pl_rows * ld_in, b=w16.data_ptr(), ldb=ldw, m=pl_rows, n=dim, kc=in_dim,
                   taps=self._s2_taps(W0), col_scale=s2.data_ptr(), col_shift=t2.data_ptr(), act=L.ACT_RELU,
                   m_alg=lvl["npix"], row_map=self._plane_to_padded_map("stem.to_l0", B, H0, W0, lvl["Hb"], lvl["Wb"]).data_ptr(),
                   out_f32=lvl["x32"].data_ptr(), ld_o32=lvl["C"], out_f16=lvl["x16"].data_ptr(),
                   ld_o16=lvl["ld"])

        self._mark("patch_embed", kind="conv", lv=lvl)
        # ---------------- levels
        Hc, Wc, Cc = H0, W0, dim
        for i, level in enumerate(m.levels):
            if level.conv:
                if i > 0:
                    lvl = self._conv_level_buffers(i, Cc, Hc, Wc)
                    self._zero_window_padding(lvl)
                    self._emit_downsample_conv(i - 1, prev, lvl, to_conv=True)
                    self._mark(f"levels.{i - 1}", kind="conv", lv=lvl)
                self._emit_conv_blocks(i, level, lvl)
                self._mark(f"levels.{i}.out", kind="conv", lv=lvl)
                prev = dict(kind="conv", **lvl)
            else:
                tl = self._token_level_buffers(i, level, Cc, Hc, Wc)
                if tl["padded"]:
                    # window-padding pixels enter the level as zero tokens (fvar.py:853-855) and are
                    # modified in place by the blocks, so they are re-zeroed every forward; all other
                    # rows are fully overwritten by the downsample GEMM / tokenizer
                    self.ops.append(("zero", tl["xs"], "memset"))
                self._emit_downsample_conv(i - 1, prev, tl, to_conv=False)
                self._mark(f"levels.{i - 1}", kind="tok_map", tl=tl)
                self._emit_token_level(i, level, tl)
                self._mark(f"levels.{i}.out", kind="tok_map", tl=tl)
                prev = dict(kind="tok", **tl)
                if level.downsample is None:
                    self._mark(f"levels.{i}", kind="tok_map", tl=tl)
            if level.downsample is not None:
                Hc, Wc, Cc = (Hc + 1) // 2, (Wc + 1) // 2, Cc * 2
        self.feat = prev
        if getattr(m, "head", None) is None:   # the downstream backbones: level maps only, no classifier tail
            self.pooled = self.logits = None
            return
        # ---------------- head: BN folded into the average pool, then the classifier GEMM
        nf = m.num_features
        sN, tN = self._fold("norm", nf, m.norm)
        T = prev["H"] * prev["W"]
        pooled = nb.new("head.pooled", (B, _ru(nf, 8)), torch.float16)
        self.pooled = pooled
        self.norm_fold = (sN, tN)
        self._op(self.ops, "fvit_pool_affine_fwd", prev["xs"].data_ptr(), nf, prev["crop_map"].data_ptr(), B, T,
                 nf, sN.data_ptr(), tN.data_ptr(), pooled.data_ptr(), pooled.stride(0))
        if isinstance(m.head, nn.Linear):
            hw16, ldh = self._pack_linear("head", m.head)
            self.logits = nb.new("logits", (B, m.num_classes), torch.float32)
            self._gemm(a=pooled.data_ptr(), a_rows=B, lda=pooled.stride(0), b=hw16.data_ptr(), ldb=ldh, m=B,
                       n=m.num_classes, kc=nf, col_shift=m.head.bias.data_ptr(),
                       out_f32=self.logits.data_ptr(), ld_o32=m.num_classes)
        else:
            self.logits = None

    # ---- geometry helpers -----------------------------------------------------------------------
    def stem_cols(self) -> tuple[int, int]:
        """(9 * in_chans, stem_ld): the taps of the first stem convolution and the fp16 row width of its im2col matrix,
        zero padded to a multiple of 32 (STEM_LD for RGB)"""
        cin = self.model.cfg["in_chans"]
        if not 1 <= cin <= STEM_MAX_CIN:
            raise L.FvitError(f"in_chans={cin}: the stem kernels support 1 <= in_chans <= {STEM_MAX_CIN}")
        return 9 * cin, (self.STEM_LD if cin == 3 else _ru(9 * cin, 32))

    def check_ln_widths(self) -> None:
        """Raise FvitError for a model whose LayerNorm rows (a Downsample's channel norm, the norms of the transformer
        blocks) are wider than the LayerNorm kernels take, before any buffer is allocated or kernel launched."""
        for i, level in enumerate(self.model.levels):
            normed = level.downsample is not None or (not level.conv and len(level.blocks) > 0)
            if normed and level.dim > LN_MAX_C:
                raise L.FvitError(f"level {i}: {level.dim}-channel LayerNorm rows, but the LayerNorm kernels take at "
                                  f"most {LN_MAX_C} channels")

    def _s2_taps(self, Wo: int) -> list[tuple[int, int]]:
        """9 taps of a 3x3 stride-2 pad-1 convolution over the parity-plane layout: input row 2*oh+r-1
        lives in plane parity (r+1)&1 at plane row oh + (r==0 ? -1 : 0) (+1 border offset cancels)."""
        taps = []
        for r in range(3):
            ph, da = (1, -1) if r == 0 else ((0, 0) if r == 1 else (1, 0))
            for s in range(3):
                pw, db = (1, -1) if s == 0 else ((0, 0) if s == 1 else (1, 0))
                taps.append((da * (Wo + 1) + db, ph * 2 + pw))
        return taps

    def _parity_plane_map(self, name: str, H: int, W: int) -> torch.Tensor:
        """pixel (b, y, x) of an H x W map -> its row in the four parity planes that feed a 3x3 stride-2 convolution:
        plane (y&1)*2 + (x&1), plane row (y>>1)+1 and column (x>>1)+1 behind the zero top row / left column."""
        B = self.B
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        pl_rows = B * (Ho + 1) * (Wo + 1)
        bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(H), torch.arange(W), indexing="ij")
        return self.bufs.i32(name, (((yi & 1) * 2 + (xi & 1)) * pl_rows + bi * (Ho + 1) * (Wo + 1)
                                    + ((yi >> 1) + 1) * (Wo + 1) + (xi >> 1) + 1).reshape(-1))

    def _plane_to_padded_map(self, name: str, B: int, Ho: int, Wo: int, Hb: int | None = None,
                             Wb: int | None = None) -> torch.Tensor:
        """plane-space output row (b, a+1, c+1) -> zero-bordered level row of an (Hb, Wb) map (default (Ho, Wo); larger
        when the level runs on a window-padded map, conv_level_pad); border rows -> -1."""
        Hb, Wb = Hb or Ho, Wb or Wo
        bi, ai, ci = torch.meshgrid(torch.arange(B), torch.arange(Ho + 1), torch.arange(Wo + 1), indexing="ij")
        dst = bi * (Hb + 2) * (Wb + 2) + ai * (Wb + 2) + ci  # (a-1)+1 = a
        dst = torch.where((ai >= 1) & (ci >= 1), dst, torch.full_like(dst, -1))
        return self.bufs.i32(name, dst.reshape(-1))

    def _downsample_row_map(self, i: int, dst: dict, Ho: int, Wo: int) -> torch.Tensor:
        """plane-space output row (b, a+1, c+1) of Downsample i -> the row of pixel (a, c) in the next level: its
        zero-bordered conv map, or its window-major token buffer (dst["pix_map_host"]); border rows -> -1."""
        if "pix_map_host" not in dst:
            return self._plane_to_padded_map(f"ds{i}.rmap", self.B, Ho, Wo, dst["Hb"], dst["Wb"])
        full = torch.full((self.B, Ho + 1, Wo + 1), -1, dtype=torch.int64)
        full[:, 1:, 1:] = dst["pix_map_host"][:, :Ho, :Wo]
        return self.bufs.i32(f"ds{i}.rmap", full.reshape(-1))

    def _conv_level_buffers(self, i: int, Cc: int, Hc: int, Wc: int, f16=("x16", "h16")) -> dict:
        """geometry, row maps and buffers of a conv level's zero-bordered map: the fp32 residual stream x32 and one
        [rows, ld] fp16 matrix per name in f16. The map is Hb x Wb (conv_level_pad): the blocks compute every pixel of
        it, the Hc x Wc top-left part (pix) is the level's input and output."""
        B, nb = self.B, self.bufs
        Hb, Wb = conv_level_pad(self.model, i, Hc, Wc)
        rows = B * (Hb + 2) * (Wb + 2)
        ld = _ru(Cc, 8)
        bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(Hb + 2), torch.arange(Wb + 2), indexing="ij")
        inside = (yi >= 1) & (yi <= Hb) & (xi >= 1) & (xi <= Wb)
        ident = torch.arange(rows).view(B, Hb + 2, Wb + 2)
        interior = nb.i32(f"l{i}.interior", torch.where(inside, ident, torch.full_like(ident, -1)).reshape(-1))
        pix = nb.i32(f"l{i}.pix", ident[:, 1:Hc + 1, 1:Wc + 1].reshape(-1))  # pixel (b,y,x) -> padded row
        # the pixels the blocks compute (their BatchNorms' statistics included): the whole Hb x Wb map
        cpix = pix if (Hb, Wb) == (Hc, Wc) else nb.i32(f"l{i}.cpix", ident[:, 1:-1, 1:-1].reshape(-1))
        d = dict(C=Cc, H=Hc, W=Wc, Hb=Hb, Wb=Wb, ld=ld, rows=rows, npix=B * Hc * Wc, interior=interior, pix=pix,
                 cpix=cpix, cnpix=B * Hb * Wb,
                 x32=nb.new(f"l{i}.x32", (rows, Cc), torch.float32))
        for k in f16:
            d[k] = nb.new(f"l{i}.{k}", (rows, ld), torch.float16)
        return d

    def _zero_window_padding(self, lv: dict) -> None:
        """A conv level on a window-padded map (conv_level_pad) enters with zeros there (F.pad, dino/models/dino/
        fastervit.py:690-691), which the blocks then overwrite: re-zeroed every forward before the map is written."""
        if (lv["Hb"], lv["Wb"]) != (lv["H"], lv["W"]):
            for t in (lv["x32"], lv["x16s"][0] if "x16s" in lv else lv["x16"]):   # (train plans: the first block's operand)
                self.ops.append(("zero", t, "memset"))

    # ---- conv levels ------------------------------------------------------------------------------
    def _emit_conv_blocks(self, i: int, level, lv: dict) -> None:
        Cc, Wp = lv["C"], lv["Wb"] + 2
        taps = [((dy - 1) * Wp + (dx - 1), 0) for dy in range(3) for dx in range(3)]
        for j, blk in enumerate(level.blocks):
            nm = f"l{i}.b{j}"
            w1, ld1 = self._pack_conv(nm + ".conv1", blk.conv1)
            w2, ld2 = self._pack_conv(nm + ".conv2", blk.conv2)
            s1, t1 = self._fold(nm + ".bn1", Cc, blk.norm1, bias=blk.conv1.bias)
            s2, t2 = self._fold(nm + ".bn2", Cc, blk.norm2, bias=blk.conv2.bias, ls=getattr(blk, "gamma", None))
            # h = GELU(BN(conv1(x)))                                        (fv.py:504-506)
            self._gemm(a=lv["x16"].data_ptr(), a_rows=lv["rows"], lda=lv["ld"], b=w1.data_ptr(), ldb=ld1,
                       m=lv["rows"], n=Cc, kc=Cc, taps=taps, col_scale=s1.data_ptr(), col_shift=t1.data_ptr(),
                       m_alg=lv["npix"],act=L.ACT_GELU, row_map=lv["interior"].data_ptr(), out_f16=lv["h16"].data_ptr(),
                       ld_o16=lv["ld"])
            # x = x + gamma * BN(conv2(h))                                   (fv.py:507-511)
            self._gemm(a=lv["h16"].data_ptr(), a_rows=lv["rows"], lda=lv["ld"], b=w2.data_ptr(), ldb=ld2,
                       m=lv["rows"], n=Cc, kc=Cc, taps=taps, col_scale=s2.data_ptr(), col_shift=t2.data_ptr(),
                       m_alg=lv["npix"],resid=lv["x32"].data_ptr(), ld_resid=Cc, row_map=lv["interior"].data_ptr(),
                       out_f32=lv["x32"].data_ptr(), ld_o32=Cc, out_f16=lv["x16"].data_ptr(), ld_o16=lv["ld"])
            self._mark(f"levels.{i}.blocks.{j}", kind="conv", lv=lv)

    def _emit_downsample_conv(self, i: int, src: dict, dst: dict, to_conv: bool) -> None:
        """Downsample of level i (fv.py:437-440): channel LayerNorm (eps 1e-6) scattered into parity
        planes, then the 3x3/s2 convolution as a 9-tap GEMM writing the next level's layout."""
        B, nb = self.B, self.bufs
        ds = self.model.levels[i].downsample
        Cs, Hs, Ws = src["C"], src["H"], src["W"]
        Ho, Wo = (Hs + 1) // 2, (Ws + 1) // 2
        ld = _ru(Cs, 8)
        pl_rows = B * (Ho + 1) * (Wo + 1)
        planes = nb.new(f"ds{i}.planes", (4 * pl_rows, ld), torch.float16)
        omap = self._parity_plane_map(f"ds{i}.omap", Hs, Ws)
        src_rows = src["pix"] if src["kind"] == "conv" else src["crop_map"]
        src_x = src["x32"] if src["kind"] == "conv" else src["xs"]
        self._op(self.ops, "fvit_ln_fwd", src_x.data_ptr(), Cs, src_rows.data_ptr(), B * Hs * Ws, Cs,
                 None, 1, 0, None, 0, ds.norm.weight.data_ptr(), ds.norm.bias.data_ptr(), float(ds.norm.eps),
                 planes.data_ptr(), ld, omap.data_ptr(), None, None, None, 0)
        w16, ldw = self._pack_conv(f"ds{i}.conv", ds.reduction[0])
        if to_conv:
            out = dict(out_f32=dst["x32"].data_ptr(), out_f16=dst["x16"].data_ptr(), ld_o16=dst["ld"])
        else:
            out = dict(out_f32=dst["xs"].data_ptr())
        rmap = self._downsample_row_map(i, dst, Ho, Wo)
        self._gemm(a=planes.data_ptr(), a_rows=pl_rows, lda=ld, a_planes=4, a_plane_stride=pl_rows * ld,
                   b=w16.data_ptr(), ldb=ldw, m=pl_rows, n=2 * Cs, kc=Cs, taps=self._s2_taps(Wo),
                   m_alg=B * Ho * Wo, row_map=rmap.data_ptr(), ld_o32=dst["C"], **out)

    # ---- transformer levels -----------------------------------------------------------------------
    def _token_level_buffers(self, i: int, level, Cc: int, Hc: int, Wc: int) -> dict:
        B, nb = self.B, self.bufs
        ws, cs = level.window_size, self.model.cfg["ct_size"]
        geo = token_geometry(self.model, i, Hc, Wc)
        Hp, Wp, nwh, nww, has_ct, sr = geo["Hp"], geo["Wp"], geo["nwh"], geo["nww"], geo["has_ct"], geo["sr"]
        ncw = cs * cs if has_ct else 0
        S = ncw + ws * ws
        nwin = nwh * nww
        nW = B * nwin
        n_ct = ncw * nwin
        xs = nb.new(f"l{i}.xs", (nW * S + B * n_ct, Cc), torch.float32)
        heads = level.blocks[0].attn.num_heads
        hdp = self._head_pad(Cc // heads)
        Cp = heads * hdp  # channel count with every head zero-padded to hdp (tensor-core attention)
        bi, yi, xi = torch.meshgrid(torch.arange(B), torch.arange(Hp), torch.arange(Wp), indexing="ij")
        win = (bi * nwh + yi // ws) * nww + xi // ws
        pix_map = win * S + ncw + (yi % ws) * ws + (xi % ws)          # [B, Hp, Wp] -> xs row
        d = dict(C=Cc, H=Hc, W=Wc, Hp=Hp, Wp=Wp, ws=ws, cs=cs, S=S, ncw=ncw, nwin=nwin, nW=nW, n_ct=n_ct,
                 xs=xs, pix_map_host=pix_map, padded=(Hp != Hc or Wp != Wc), pool=geo["pool"], tokens=geo["tokens"],
                 pe_coords=geo["pe_coords"], hat_pe_coords=geo["hat_pe_coords"], own_tables=geo["own_tables"],
                 pix_map=nb.i32(f"l{i}.pix_map", pix_map.reshape(-1)),
                 crop_map=nb.i32(f"l{i}.crop_map", pix_map[:, :Hc, :Wc].reshape(-1)),
                 xn16=nb.new(f"l{i}.xn16", (nW * S, Cc), torch.float16),
                 qkv16=nb.new(f"l{i}.qkv16", (nW * S, 3 * Cp), torch.float16),
                 ao16=nb.new(f"l{i}.ao16", (nW * S, Cp), torch.float16),
                 h16=nb.new(f"l{i}.h16", (nW * S, int(Cc * self.model.cfg["mlp_ratio"])), torch.float16))
        if has_ct:
            ctr0 = nW * S
            dew = _ct_dewindow_perm(cs, sr)     # raster r -> window-major index p
            winp = _ct_window_perm(cs, sr)      # window-major slot q -> raster r
            b_off = torch.arange(B).view(B, 1)
            p = dew.view(1, -1)
            d["ct_gather"] = nb.i32(f"l{i}.ct_gather", ((b_off * nwin + p // ncw) * S + p % ncw).reshape(-1))
            # norm1 gather: carrier slots come from the raster buffer, window tokens stay in place
            rows = torch.arange(nW * S).view(B, nwin, S).clone()
            q = torch.arange(nwin * ncw).view(nwin, ncw)
            rows[:, :, :ncw] = ctr0 + b_off.view(B, 1, 1) * n_ct + winp[q].view(1, nwin, ncw)
            d["norm1_gather"] = nb.i32(f"l{i}.norm1_gather", rows.reshape(-1))
            d["ctr0"] = ctr0
            d["ctn16"] = nb.new(f"l{i}.ctn16", (B * n_ct, Cc), torch.float16)
            d["ctqkv16"] = nb.new(f"l{i}.ctqkv16", (B * n_ct, 3 * Cp), torch.float16)
            d["ctao16"] = nb.new(f"l{i}.ctao16", (B * n_ct, Cp), torch.float16)
            d["cth16"] = nb.new(f"l{i}.cth16", (B * n_ct, int(Cc * self.model.cfg["mlp_ratio"])), torch.float16)
            if geo["tokens"] == "nchw":
                # tokenizer token t of image b is window-major carrier t (the first block's ct_dewindow input)
                bt, t = torch.meshgrid(torch.arange(B), torch.arange(n_ct), indexing="ij")
                d["ct_rows"] = nb.i32(f"l{i}.ct_rows", ((bt * nwin + t // ncw) * S + t % ncw).reshape(-1))
            else:
                # tokenizer output (b, y0, x0) over the (cs*nwh) x (cs*nww) carrier grid -> xs row
                oh, ow = cs * nwh, cs * nww
                bt, y0, x0 = torch.meshgrid(torch.arange(B), torch.arange(oh), torch.arange(ow), indexing="ij")
                wloc = (y0 // cs) * nww + x0 // cs
                d["ct_rows"] = nb.i32(f"l{i}.ct_rows", ((bt * nwin + wloc) * S + (y0 % cs) * cs + x0 % cs).reshape(-1))
            # propagation source (nearest-neighbour upsample cs -> ws, fv.py:656, 699-700)
            r = torch.arange(nW * S)
            t = r % S - ncw
            src = (r // S) * S + ((t // ws) * cs // ws) * cs + (t % ws) * cs // ws
            d["prop_src"] = nb.i32(f"l{i}.prop_src", torch.where(t >= 0, src, torch.full_like(src, -1)))
        return d

    @staticmethod
    def _attn_kind(S: int, hdp: int) -> str:
        """Which attention core serves a window sequence of S tokens with padded head dim hdp: "tile" (one 128-row
        wgmma tile, fvit_attn_tc_fwd), "loop" (key-loop wgmma kernel for longer windows: its TMA-staged bias rows
        need S % 4 == 0) or "simt" (generic fallback for geometries neither covers)."""
        if hdp > 80:
            return "simt"
        if S <= 128:
            return "tile"
        return "loop" if S % 4 == 0 else "simt"

    @staticmethod
    def _head_pad(hd: int) -> int:
        """Padded head dim of the tensor-core attention kernels (TMA boxes need 16-byte rows; the
        kernels are instantiated for 32, 64 and 80). Larger heads use the generic SIMT core unpadded."""
        return 32 if hd <= 32 else (64 if hd <= 64 else (80 if hd <= 80 else hd))

    def _emit_attention(self, nm: str, attn, gamma, rows: int, groups: int, S: int, xin, ld_in, qkv, ao,
                        bias_buf, stream_buf) -> None:
        """x += gamma * proj(softmax(q k^T * scale + bias) v) with q,k,v = qkv(xin)  (fv.py:557-568).
        Three launches: qkv GEMM (+bias), attention core, proj GEMM (+bias, layer-scale, residual)."""
        Cc, h, hd = attn.qkv.in_features, attn.num_heads, attn.head_dim
        hdp = self._head_pad(hd)
        use_tc = self._attn_kind(S, hdp) != "simt"
        if not use_tc:
            hdp = hd
        Cp = h * hdp
        wq, ldq, qb_ptr, wp, ldp = self._pack_attention(nm, attn, hdp)
        scale = float(getattr(attn, "scale", hd ** -0.5))   # qk_scale or head_dim ** -0.5 (fv.py:544)
        # the fused kernel takes 64-wide (padded) heads, where the projection is long enough to amortise its serial
        # projection / softmax phases
        fused = self._attn_kind(S, hdp) == "tile" and hdp == 64
        if fused:
            # ONE kernel: qkv projection + softmax(q k^T * scale + bias) + P v; the qkv matrix never reaches HBM
            self._op(self.ops, "fvit_hat_attn_fwd", xin.data_ptr(), ld_in, Cc, wq.data_ptr(), ldq, qb_ptr, groups, S, h,
                     hdp, bias_buf.data_ptr(), scale, ao.data_ptr(), Cp, None, 0)
            self.op_flops[len(self.ops) - 1] = 2.0 * rows * 3 * Cc * Cc + 4.0 * groups * h * S * S * hd
        else:
            self._gemm(a=xin.data_ptr(), a_rows=rows, lda=ld_in, b=wq.data_ptr(), ldb=ldq, m=rows, n=3 * Cp, kc=Cc,
                       col_shift=qb_ptr, out_f16=qkv.data_ptr(), ld_o16=3 * Cp)
            self.op_flops[len(self.ops) - 1] = 2.0 * rows * 3 * Cc * Cc  # algorithmic (un-padded heads)
        if fused:
            pass
        elif use_tc and S > 128:
            self._op(self.ops, "fvit_attn_loop_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hdp,
                     bias_buf.data_ptr(), scale, ao.data_ptr(), Cp, None)
        elif use_tc:
            self._op(self.ops, "fvit_attn_tc_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hdp,
                     bias_buf.data_ptr(), scale, ao.data_ptr(), Cp)
        else:
            self._op(self.ops, "fvit_attn_core_fwd", qkv.data_ptr(), 3 * Cp, groups, S, h, hd,
                     bias_buf.data_ptr(), scale, ao.data_ptr(), Cp, None)
        if not fused:
            self.op_flops[len(self.ops) - 1] = 4.0 * groups * h * S * S * hd
        # proj: K dimension is the (head-padded) attention output
        lin = attn.proj
        n = lin.weight.shape[0]
        if isinstance(gamma, torch.Tensor):
            sc, sh = self._fold(nm + ".proj.ls", n, bias=lin.bias, ls=gamma)
            cs_, sh_ = sc.data_ptr(), sh.data_ptr()
        else:
            cs_, sh_ = None, lin.bias.data_ptr()
        self._gemm(a=ao.data_ptr(), a_rows=rows, lda=Cp, b=wp.data_ptr(), ldb=ldp, m=rows, n=n, kc=Cp,
                   col_scale=cs_, col_shift=sh_, resid=stream_buf, ld_resid=n, out_f32=stream_buf, ld_o32=n,
                   flops=2.0 * rows * n * Cc)

    def _pack_attention(self, nm: str, attn, hdp: int) -> tuple:
        """fp16 operands of an attention's qkv and proj Linears with every head zero-padded from head_dim to hdp (the
        rows of qkv, the columns of proj), and qkv's bias padded alike: (wq, ldq, qkv bias pointer, wp, ldp)"""
        Cc, hd = attn.qkv.in_features, attn.head_dim
        if hdp == hd:
            wq, ldq = self._pack_linear(nm + ".qkv", attn.qkv)
            wp, ldp = self._pack_linear(nm + ".proj", attn.proj)
            return wq, ldq, P(attn.qkv.bias), wp, ldp
        Cp = attn.num_heads * hdp
        ldq = _ru(Cc, 8)
        wq = self.bufs.new(nm + ".qkv.w16", (3 * Cp, ldq), torch.float16)
        self._op(self.prep_ops, "fvit_cast_headpad_f16", attn.qkv.weight.data_ptr(), Cc, wq.data_ptr(), ldq, 3 * Cp, Cc,
                 hd, hdp, 1, 0)
        qb_ptr = None
        if attn.qkv.bias is not None:
            qbp = self.bufs.new(nm + ".qkv.bias_pad", (3 * Cp,), torch.float32)
            self._op(self.prep_ops, "fvit_vec_headpad_f32", attn.qkv.bias.data_ptr(), qbp.data_ptr(), 3 * Cp, hd, hdp)
            qb_ptr = qbp.data_ptr()
        n = attn.proj.weight.shape[0]
        wp = self.bufs.new(nm + ".proj.w16", (n, Cp), torch.float16)
        self._op(self.prep_ops, "fvit_cast_headpad_f16", attn.proj.weight.data_ptr(), Cc, wp.data_ptr(), Cp, n, Cp, hd,
                 hdp, 0, 1)
        return wq, ldq, qb_ptr, wp, Cp

    def _emit_bias(self, nm: str, rpb, S: int, hidden=None, own: bool = False) -> dict:
        """PosEmbMLPSwinv2D (fv.py:276-307): table MLP + gather + 16*sigmoid, written straight into the
        module's `relative_bias` buffer (which the reference also overwrites every forward). With a `hidden` buffer
        (training) the MLP also saves its hidden activations for the backward, and so runs in deploy mode too.
        own: into a plan buffer instead (token_geometry's own_tables: S changes with the input, and a module buffer
        reallocated for one shape would leave every other cached plan pointing at freed memory)."""
        npts = rpb.relative_coords_table.shape[1] * rpb.relative_coords_table.shape[2]
        table = self.bufs.new(nm + ".table", (npts, rpb.num_heads), torch.float32)
        if own:
            out = self.bufs.new(nm + ".out", (1, rpb.num_heads, S, S), torch.float32)
        else:
            if tuple(rpb.relative_bias.shape) != (1, rpb.num_heads, S, S):
                rpb.relative_bias = torch.zeros(1, rpb.num_heads, S, S, device=self.device)
            out = rpb.relative_bias
        tgt = self.prep_ops  # batch independent: recomputed only when the weights change
        n0 = len(tgt)
        self._op(tgt, "fvit_cpb_mlp_fwd", rpb.relative_coords_table.data_ptr(), npts, rpb.cpb_mlp[0].weight.data_ptr(),
                 rpb.cpb_mlp[0].bias.data_ptr(), rpb.cpb_mlp[2].weight.data_ptr(), rpb.num_heads,
                 table.data_ptr(), P(hidden))
        self._op(tgt, "fvit_attn_bias_fwd", table.data_ptr(), rpb.relative_position_index.data_ptr(),
                 rpb.num_heads, S, rpb.window ** 2, out.data_ptr())
        if hidden is None and not own:
            self._deploy_guard(tgt, n0, rpb)
        return dict(mod=rpb, out=out, hidden=hidden, npts=npts, S=S)

    def _emit_pos_embed(self, nm: str, tpe, coords_host: torch.Tensor, Cc: int, hidden=None, own: bool = False) -> dict:
        """PosEmbMLPSwinv1D rank 2 (fv.py:355-365): MLP over the grid coordinates `coords_host` ([npts, 2],
        token_geometry), written into the module's `relative_bias` buffer; the add itself is fused into the following
        LayerNorm. `hidden`, `own`: as _emit_bias."""
        npts = coords_host.shape[0]
        coords = self.bufs.new(nm + ".coords", (npts, 2), torch.float32)
        coords.copy_(coords_host)
        if own:
            out = self.bufs.new(nm + ".out", (1, npts, Cc), torch.float32)
        else:
            if tuple(tpe.relative_bias.shape) != (1, npts, Cc):
                tpe.relative_bias = torch.zeros(1, npts, Cc, device=self.device)
            out = tpe.relative_bias
        n0 = len(self.prep_ops)
        self._op(self.prep_ops, "fvit_cpb_mlp_fwd", coords.data_ptr(), npts, tpe.cpb_mlp[0].weight.data_ptr(),
                 tpe.cpb_mlp[0].bias.data_ptr(), tpe.cpb_mlp[2].weight.data_ptr(), Cc, out.data_ptr(), P(hidden))
        if hidden is None and not own:
            self._deploy_guard(self.prep_ops, n0, tpe)
        return dict(mod=tpe, out=out, hidden=hidden, coords=coords, npts=npts, D=Cc)

    def _emit_branch_out(self, nm: str, lin: nn.Linear, gamma, a, lda, rows, stream_buf, act=L.ACT_NONE,
                         out16=None, ld16=0) -> None:
        """x += gamma * (a @ W^T + b) in place on the fp32 residual stream (fv.py:679-680, 690-691)."""
        n, k = lin.weight.shape
        w16, ldw = self._pack_linear(nm, lin)
        if isinstance(gamma, torch.Tensor):
            sc, sh = self._fold(nm + ".ls", n, bias=lin.bias, ls=gamma)
            cs_, sh_ = sc.data_ptr(), sh.data_ptr()
        else:
            cs_, sh_ = None, lin.bias.data_ptr()
        self._gemm(a=a.data_ptr(), a_rows=rows, lda=lda, b=w16.data_ptr(), ldb=ldw, m=rows, n=n, kc=k,
                   col_scale=cs_, col_shift=sh_, resid=stream_buf, ld_resid=n, out_f32=stream_buf, ld_o32=n)

    def _emit_fc1(self, nm: str, lin: nn.Linear, a, lda, rows, out16) -> None:
        n, k = lin.weight.shape
        w16, ldw = self._pack_linear(nm, lin)
        self._gemm(a=a.data_ptr(), a_rows=rows, lda=lda, b=w16.data_ptr(), ldb=ldw, m=rows, n=n, kc=k,
                   col_shift=lin.bias.data_ptr(), act=L.ACT_GELU, out_f16=out16.data_ptr(), ld_o16=n)

    def _emit_token_level(self, i: int, level, tl: dict) -> None:
        B, Cc, S, ncw, ws = self.B, tl["C"], tl["S"], tl["ncw"], tl["ws"]
        nW, n_ct = tl["nW"], tl["n_ct"]
        xs = tl["xs"]
        xs_ptr = xs.data_ptr()
        has_ct = ncw > 0
        # (the downsample GEMM that fills the window tokens was emitted before this call)
        if level.do_gt and has_ct:
            tk = level.global_tokenizer
            (kh, sh_, oh), (kw, sw_, ow) = tl["pool"]
            entry = "fvit_token_init_nchw_fwd" if tl["tokens"] == "nchw" else "fvit_token_init_fwd"
            self._op(self.ops, entry, xs_ptr, Cc, tl["pix_map"].data_ptr(), B, tl["Hp"], tl["Wp"],
                     Cc, tk.pos_embed.weight.data_ptr(), tk.pos_embed.bias.data_ptr(), kh, kw, sh_, sw_, oh, ow,
                     tl["ct_rows"].data_ptr(), xs_ptr, Cc)
        own = tl["own_tables"]
        for j, blk in enumerate(level.blocks):
            nm = f"l{i}.b{j}"
            pe = self._emit_pos_embed(nm + ".pe", blk.pos_embed, tl["pe_coords"], Cc, own=own)["out"]
            if has_ct:
                ctr_ptr = xs_ptr + tl["ctr0"] * Cc * 4
                rows_c = B * n_ct
                hat_pe = None
                if tl["hat_pe_coords"] is not None:
                    hat_pe = self._emit_pos_embed(nm + ".hat_pe", blk.hat_pos_embed, tl["hat_pe_coords"], Cc,
                                                  own=own)["out"]
                # ct = dewindow(ct) + hat_pos_embed ; LN -> fp16                 (fv.py:673-679)
                self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, tl["ct_gather"].data_ptr(), rows_c, Cc,
                         hat_pe.data_ptr() if hat_pe is not None else None, n_ct, 0, ctr_ptr, Cc,
                         blk.hat_norm1.weight.data_ptr(), blk.hat_norm1.bias.data_ptr(), float(blk.hat_norm1.eps),
                         tl["ctn16"].data_ptr(), Cc, None, None, None, None, 0)
                hb = self._emit_bias(nm + ".hat_bias", blk.hat_attn.pos_emb_funct, n_ct, own=own)["out"]
                self._emit_attention(nm + ".hat_attn", blk.hat_attn, blk.gamma1, rows_c, B, n_ct, tl["ctn16"], Cc,
                                     tl["ctqkv16"], tl["ctao16"], hb, ctr_ptr)
                self._op(self.ops, "fvit_ln_fwd", ctr_ptr, Cc, None, rows_c, Cc, None, 1, 0, None, 0,
                         blk.hat_norm2.weight.data_ptr(), blk.hat_norm2.bias.data_ptr(), float(blk.hat_norm2.eps),
                         tl["ctn16"].data_ptr(), Cc, None, None, None, None, 0)
                self._emit_fc1(nm + ".hat_fc1", blk.hat_mlp.fc1, tl["ctn16"], Cc, rows_c, tl["cth16"])
                self._emit_branch_out(nm + ".hat_fc2", blk.hat_mlp.fc2, blk.gamma2, tl["cth16"],
                                      tl["cth16"].stride(0), rows_c, ctr_ptr)
            # x = cat(ct_window(ct), x + pos_embed) ; LN(norm1) -> fp16          (fv.py:665, 683-690)
            rows = nW * S
            self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, tl["norm1_gather"].data_ptr() if has_ct else None, rows,
                     Cc, pe.data_ptr(), S, ncw, xs_ptr, Cc, blk.norm1.weight.data_ptr(), blk.norm1.bias.data_ptr(),
                     float(blk.norm1.eps), tl["xn16"].data_ptr(), Cc, None, None, None, None, 0)
            ab = self._emit_bias(nm + ".bias", blk.attn.pos_emb_funct, S, own=own)["out"]
            self._emit_attention(nm + ".attn", blk.attn, blk.gamma3, rows, nW, S, tl["xn16"], Cc, tl["qkv16"],
                                 tl["ao16"], ab, xs_ptr)
            self._op(self.ops, "fvit_ln_fwd", xs_ptr, Cc, None, rows, Cc, None, 1, 0, None, 0,
                     blk.norm2.weight.data_ptr(), blk.norm2.bias.data_ptr(), float(blk.norm2.eps),
                     tl["xn16"].data_ptr(), Cc, None, None, None, None, 0)
            self._emit_fc1(nm + ".fc1", blk.mlp.fc1, tl["xn16"], Cc, rows, tl["h16"])
            self._emit_branch_out(nm + ".fc2", blk.mlp.fc2, blk.gamma4, tl["h16"], tl["h16"].stride(0), rows, xs_ptr)
            if has_ct and blk.last and blk.do_propagation:
                g1 = blk.gamma1.data_ptr() if isinstance(blk.gamma1, torch.Tensor) else None
                self._op(self.ops, "fvit_propagate_fwd", xs_ptr, Cc, tl["prop_src"].data_ptr(), rows, Cc, g1)
            self._mark(f"levels.{i}.blocks.{j}", kind="windows", tl=tl)

    # ---- CUDA graphs --------------------------------------------------------------------------------
    def run_captured(self, key: str, fn) -> None:
        """Run `fn` (a closure that only enqueues kernels / memsets on the current stream over this plan's persistent
        buffers) through a CUDA graph: first call eager (warm-up: lazy function attributes, descriptor cache), second
        call captured, later calls are ONE graph launch instead of hundreds of ctypes launches. FVIT_CUDA_GRAPH=0
        disables; a failed capture falls back to eager launches for good (reported once)."""
        st = self._graphs.get(key)
        if not self.use_graphs or st == "off":
            fn()
            return
        if st is None:
            fn()
            self._graphs[key] = "warm"
            return
        if st == "warm":
            try:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                n0 = L.launch_count()
                # Dead reference cycles (e.g. the plans of a dropped model, with their CUDA graphs and memory pools)
                # are collected now, not by an automatic collection in the middle of the capture: freeing device
                # memory there invalidates the capture and leaves torch's RNG in capture state.
                gc.collect()
                gc_on = gc.isenabled()
                gc.disable()
                try:
                    # thread_local: other threads (NCCL's watchdog polling its events) must not invalidate the capture
                    with torch.cuda.graph(g, capture_error_mode="thread_local"):
                        fn()
                finally:
                    if gc_on:
                        gc.enable()
                self._graphs[key] = (g, L.launch_count() - n0)
                st = self._graphs[key]
            except Exception as exc:  # noqa: BLE001 - capture problems must not take the model down
                import warnings
                warnings.warn(f"fastervit_b200: CUDA-graph capture of the {key} launch list failed ({exc}); "
                              "continuing with eager launches")
                self._graphs[key] = "off"
                torch.cuda.synchronize()
                fn()
                return
        g, n = st
        g.replay()
        self.lib.fvit_add_launch_count(n)

    def static_input(self, x: torch.Tensor) -> torch.Tensor:
        """Captured launch lists read the image through a fixed pointer: copy the caller's tensor (any strides) into
        the plan's input buffer (0.15 % of an fv4 step's HBM traffic)."""
        if self._x_static is None or self._x_static.shape != x.shape:
            self._x_static = torch.empty(x.shape, dtype=torch.float32, device=x.device)
        self._x_static.copy_(x, non_blocking=True)
        return self._x_static

    # ---- execution --------------------------------------------------------------------------------
    def weights_key(self) -> tuple:
        """What the packed fp16 operands of an eval plan were derived from: autograd versions (in-place torch
        writes) plus the library-wide raw-write epoch, which the fused optimizer / EMA kernels and the train-mode
        BatchNorm kernels bump because they update parameters through raw pointers without touching versions."""
        k = 0
        for p in self.model.parameters():
            k += p._version
        for b_ in self.model.buffers():
            k += b_._version
        return (k, L.weights_epoch(), sum(1 << (i % 60) for i, m in enumerate(self._deploy_mods) if m.deploy))

    def run_ops(self, ops: list, x: torch.Tensor | None, side: set | None = None) -> None:
        """Enqueue a launch list on the current stream. `side` (absolute op indices, engine_train.py) names leaf
        launches that go to the plan's side stream instead: forked after everything enqueued so far, joined at the
        next bucket point and at the end of the list -- under graph capture these become parallel branches."""
        st = L.stream_ptr()
        lib = self.lib
        shadow = getattr(self, "_ar_shadow", None) if getattr(self, "_ar_active", None) is not None else None
        base = getattr(self, "_op_base", 0)
        cur = side_stream = None
        forked = False
        side_reads = getattr(self, "_side_reads", None) or {}
        side_events: dict = {}   # buffer pointer -> event behind the last side launch that reads it (this call only)
        if side:
            cur = torch.cuda.current_stream()
            side_stream = self._side_streams(1)[0]
        for idx, (fn, args, name) in enumerate(ops):
            if shadow is not None:
                # launches in the shadow of a gradient all-reduce leave NCCL's SMs alone (engine_train.py)
                lib.fvit_set_sm_limit(shadow.get(base + idx, 0))
            if fn == "im2col":
                a = self._x_args[args]
                rc = lib.fvit_stem_im2col(x.data_ptr(), x.stride(0), x.stride(1), x.stride(2), x.stride(3),
                                          a["B"], a["cin"], a["H"], a["W"], a["out"], a["ldo"], st)
            elif fn == "zero":
                args.zero_()
                continue
            elif fn == "unless_deploy":
                mod, fn2, args2 = args
                if mod.deploy:
                    continue
                rc = fn2(*args2, st)
            elif fn == "wait_side":   # the next launch overwrites buffers a side-branch launch may still be reading
                for k in args:
                    ev = side_events.pop(k, None)
                    if ev is not None:
                        cur.wait_event(ev)
                continue
            elif fn == "bucket":   # gradient slice [lo, hi) of the flat buffer is final (engine_train.py)
                if forked:
                    cur.wait_stream(side_stream)
                    forked = False
                red = getattr(self, "_ar_active", None)
                if red is not None:
                    red.reduce(*args)
                continue
            elif side and (base + idx) in side:
                side_stream.wait_stream(cur)
                forked = True
                rc = fn(*args, side_stream.cuda_stream)
                keys = side_reads.get(base + idx)
                if keys:
                    ev = torch.cuda.Event()
                    ev.record(side_stream)
                    for k in keys:
                        side_events[k] = ev
            else:
                rc = fn(*args, st)
            if rc != 0:
                lib.fvit_set_sm_limit(0)
                raise L.FvitError(f"{name}: {lib.fvit_last_error().decode()}")
        if forked:
            cur.wait_stream(side_stream)
        if shadow is not None:
            lib.fvit_set_sm_limit(0)

    def _side_streams(self, n: int) -> list:
        ss = getattr(self, "_sides", None)
        if ss is None:
            ss = self._sides = []
        while len(ss) < n:
            ss.append(torch.cuda.Stream(device=self.device))
        return ss[:n]

    def run_ops_branches(self, ops: list, n_streams: int = 8) -> None:
        """Enqueue a list of plain launches whose only mutual dependencies are shared pointer arguments (weight
        re-packing: every launch writes its own operand buffer) as `n_streams` parallel branches: launches that
        share a device pointer stay in order on one stream, the rest are dealt round-robin. A few hundred small
        launches then cost the HBM time of the large ones instead of a serial chain of launch latencies."""
        cache = self.__dict__.setdefault("_branch_chains", {})
        chains = cache.get(id(ops))
        if chains is None:
            chains = cache[id(ops)] = dependency_chains(ops)
        if len(chains) < 2 * n_streams:
            self.run_ops(ops, None)
            return
        cur = torch.cuda.current_stream()
        streams = self._side_streams(n_streams)
        lib = self.lib
        for s in streams:
            s.wait_stream(cur)
        try:
            for k, chain in enumerate(chains):
                sp = streams[k % n_streams].cuda_stream
                for i in chain:
                    fn, args, name = ops[i]
                    if fn(*args, sp) != 0:
                        raise L.FvitError(f"{name}: {lib.fvit_last_error().decode()}")
        finally:
            for s in streams:
                cur.wait_stream(s)

    @staticmethod
    def _op_desc(op) -> dict:
        """Shape / epilogue summary of a fvit_gemm launch for the per-launch profile."""
        if op[2] != "fvit_gemm":
            return {}
        g = op[1][0]._obj
        ep = "".join(c for c, on in (("A", g.a_mn_major), ("B", g.b_mn_major), ("r", bool(g.resid)),
                                     ("m", bool(g.row_map)), ("3", bool(g.out_f32)), ("h", bool(g.out_f16)),
                                     ("s", bool(g.col_sum)), ("p", bool(g.out_pre16)), ("x", bool(g.aux))) if on)
        return dict(shape=f"m{g.m} n{g.n} k{g.kc}x{g.ntaps} sk{g.split_k} act{g.act} {ep}")

    def profile(self, x: torch.Tensor) -> list[dict]:
        """Time every launch of one forward with CUDA events on the current stream (the GPU is kept busy
        by a spin kernel while the launches are enqueued, so the intervals are back-to-back device
        time, not host enqueue latency). Returns [{name, ms, flops}] in launch order."""
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(self.ops) + 1)]
        torch.cuda.synchronize()
        torch.cuda._sleep(int(4e8))
        evs[0].record()
        for i, op in enumerate(self.ops):
            self.run_ops([op], x)
            evs[i + 1].record()
        torch.cuda.synchronize()
        return [dict(name=op[2], ms=evs[i].elapsed_time(evs[i + 1]), flops=self.op_flops.get(i, 0.0),
                     **self._op_desc(op)) for i, op in enumerate(self.ops)]


def forwards_in_flight(model) -> int:
    """how many train-mode forwards of one input key may await their backward at once (set_train_forwards_in_flight)"""
    return getattr(model, "_train_forwards_in_flight", 1)


class Engine:
    """Per-model cache of plans keyed by input signature; owns packed weights and workspaces."""

    def __init__(self, model):
        self.model = model
        self.plans: dict = {}     # in least-recently-used-first order; a train key maps to the first of its instances
        self.pools: dict = {}     # train key -> its TrainPlan instances, each holding the activations of one forward
        self._prepped: dict = {}
        self._ptr_sig: tuple | None = None
        self._fwd_seq = 0         # train forwards handed an instance so far (the age of an instance's last forward)

    def trim_plans(self) -> None:
        """Keep at most model.plan_cache_size plans (None or absent: no bound), dropping the least recently used; a
        train key's instances go together. Pools above the model's forwards-in-flight bound lose their last instances.
        A dropped plan's device memory goes once nothing holds it: an autograd node of a forward that has not run its
        backward yet keeps its plan until then. Its `_prepped` entry goes with it (keyed by id(), which a new plan may
        reuse: a stale entry would skip that plan's weight packing)."""
        cap = getattr(self.model, "plan_cache_size", None)
        while cap is not None and len(self.plans) > cap:
            key = next(iter(self.plans))
            plan = self.plans.pop(key)
            self._prepped.pop(id(plan), None)
            self.pools.pop(key, None)
        n = forwards_in_flight(self.model)
        for pool in self.pools.values():
            del pool[n:]

    def _train_instance(self, key, x: torch.Tensor, spec: dict | None) -> Plan:
        """The instance of a train key's pool the next forward runs on: one that no autograd node holds (TrainPlan.
        in_flight), else a new one while the pool is smaller than the model's forwards-in-flight bound, else the one
        with the oldest forward, whose node's backward then raises the stale-forward error."""
        pool = self.pools[key]
        plan = next((p for p in pool if not p.in_flight()), None)
        if plan is None and len(pool) < forwards_in_flight(self.model):
            from .engine_train import TrainPlan
            with torch.cuda.device(x.device):
                plan = TrainPlan(self.model, x.shape[0], x.shape[2], x.shape[3], x.device, spec=spec)
            plan._norm_sig = pool[0]._norm_sig
            plan.adopt_pivots(pool[0])
            pool.append(plan)
        if plan is None:
            plan = min(pool, key=lambda p: p.fwd_seq)
        self._fwd_seq += 1
        plan.fwd_seq = self._fwd_seq
        return plan

    def _check_weights(self) -> tuple:
        """The kernels read parameters / buffers through raw pointers as dense row-major fp32 (int64 for the
        position index): anything else (`model.half()`, `.to(memory_format=torch.channels_last)`, which re-strides
        every 4-D conv weight and the relative-coordinate tables) would be silently mis-read. Half / bf16
        parameters raise; non-contiguous tensors are re-laid out in place (values unchanged — memory format of the
        weights is irrelevant to these kernels; channels_last *inputs* are consumed through their strides).
        Returns the pointer signature the cached plans were built against."""
        ptrs = []
        named = list(self.model.named_parameters())
        self._params = [p for _, p in named]   # (for Engine.forward: one module walk per call is enough)
        for name, t in named + list(self.model.named_buffers()):
            if t.is_floating_point() and t.dtype != torch.float32:
                raise L.FvitError(f"{name} is {t.dtype}: fastervit_b200 keeps parameters and buffers in float32 (the "
                                  "kernels form their own fp16 tensor-core operands); drop .half() / .bfloat16()")
            if not t.is_contiguous():
                t.data = t.data.contiguous()
            ptrs.append(t.data_ptr())
        return tuple(ptrs)

    def _plan(self, x: torch.Tensor, spec: dict | None = None) -> Plan:
        if not x.is_cuda:
            raise L.FvitError("FasterViT (fastervit_b200) runs on CUDA only: move the model and input to a "
                              "CUDA device (`.cuda()`); there is no CPU / PyTorch fallback path")
        if x.dim() != 4 or x.dtype != torch.float32:
            raise L.FvitError(f"expected a float32 [B, C, H, W] tensor, got {tuple(x.shape)} {x.dtype}")
        if x.shape[1] != self.model.cfg["in_chans"]:
            raise L.FvitError(f"the model takes {self.model.cfg['in_chans']}-channel images, got {tuple(x.shape)}")
        p0 = next(self.model.parameters())
        if p0.device != x.device:
            raise L.FvitError(f"model is on {p0.device} but the input is on {x.device}")
        training = self.model.training
        sig = self._check_weights()
        if sig != self._ptr_sig:
            # parameters were re-allocated (.to(), .data = ..., load_state_dict(assign=True)): every cached plan
            # holds dangling pointers
            self.plans.clear()
            self.pools.clear()
            self._prepped.clear()
            self._ptr_sig = sig
        key = (tuple(x.shape), training, x.device.index)
        norm_sig = ()
        if spec is not None:
            # dense train plans: one per (requested outputs, norms present, frozen prefix) besides the input shape
            key += (spec["kind"], tuple((i, None if bn is None else id(bn)) for i, bn in spec.get("outs", ())),
                    spec.get("frozen", -1), bool(spec.get("eval")), spec.get("want_dx"), spec.get("data_only"))
            # the level norms are not the model's own tensors (the backbone's norm{i}): the plan reads them through raw
            # pointers too, so a reallocation of one of them (`bn.weight.data = ...`) rebuilds it
            norm_sig = self._norm_sig(spec)
        plan = self.plans.pop(key, None)
        if plan is not None and getattr(plan, "_norm_sig", ()) != norm_sig:
            self._prepped.pop(id(plan), None)
            self.pools.pop(key, None)
            plan = None
        if plan is not None:
            self.plans[key] = plan     # most recently used last
            return self._train_instance(key, x, spec) if key in self.pools else plan
        if getattr(self.model, "carriers_from_input", False) and spec is not None and spec.get("eval"):
            raise L.FvitError("the detection backbone has no eval-mode gradients: train it under .train(), or run eval "
                              "under torch.no_grad()")
        with torch.cuda.device(x.device):
            if training or (spec is not None and spec.get("eval")):
                from .engine_train import TrainPlan
                plan = TrainPlan(self.model, x.shape[0], x.shape[2], x.shape[3], x.device, spec=spec)
            else:
                plan = Plan(self.model, x.shape[0], x.shape[2], x.shape[3], training, x.device)
        plan._norm_sig = norm_sig
        self.plans[key] = plan
        if training and not (spec is not None and spec.get("eval")):
            # train plans: a pool of instances (the eval-grad plans recompute in their backward and stay one per key)
            self.pools[key] = [plan]
            self._fwd_seq += 1
            plan.fwd_seq = self._fwd_seq
        self.trim_plans()
        return plan

    @staticmethod
    def _norm_sig(spec: dict) -> tuple:
        """pointer signature of the level norms of a dense spec (fp32, dense, like the model's own tensors)"""
        ptrs = []
        for i, bn in spec.get("outs", ()):
            if bn is None:
                continue
            for name in ("weight", "bias", "running_mean", "running_var"):
                t = getattr(bn, name, None)   # (a channel LayerNorm has no running statistics)
                if t is None:
                    continue
                if t.dtype != torch.float32 or not t.is_contiguous():
                    raise L.FvitError(f"the norm of level {i}: {name} must be a dense float32 tensor")
                ptrs.append(t.data_ptr())
        return tuple(ptrs)

    def _train_wants_dx(self, x: torch.Tensor) -> bool:
        """does this train-mode forward need the plan with the image gradient; an input that requires grad on a model
        that did not ask for it (FasterViT.enable_input_grad) raises"""
        if not (torch.is_grad_enabled() and x.requires_grad):
            return False
        if not x.is_cuda:
            return False    # (_plan raises for a CPU input, as for any other)
        if not getattr(self.model, "_train_input_grad", False):
            raise L.FvitError("the input requires grad, but train-mode image gradients are off for this model: call "
                              "model.enable_input_grad() to get x.grad from the backward, or detach the input")
        return True

    def _dense_train(self, x: torch.Tensor, spec: dict) -> tuple:
        """Train-mode forward of a pooled / levels plan: an autograd node whose backward runs the plan's backward
        launch list from the output gradients (engine_train._DenseFunction)."""
        if self._train_wants_dx(x):
            spec = dict(spec, want_dx=True)    # (its own plan: one built for a plain input keeps its launch lists)
        plan = self._plan(x, spec)
        from .engine_train import _DenseFunction
        with torch.cuda.device(x.device):
            if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in plan.params)):
                return _DenseFunction.apply(plan, x, *plan.params)
            plan.run_forward(x)
            return tuple(o.clone() for o in plan.outputs)

    def forward(self, x: torch.Tensor, features_only: bool = False) -> torch.Tensor:
        if self.model.training:
            if features_only:
                # forward_features under .train(): the final norm with batch statistics (fv.py:949-953)
                return self._dense_train(x, dict(kind="levels", outs=((len(self.model.levels) - 1, self.model.norm),)))[0]
            if not isinstance(self.model.head, nn.Linear):
                # num_classes = 0: the pooled features (fv.py:955-958)
                return self._dense_train(x, dict(kind="pooled"))[0]
        want_dx = self.model.training and self._train_wants_dx(x)
        plan = self._plan(x, dict(kind=None, want_dx=True) if want_dx else None)
        if plan.training:
            from .engine_train import _FasterViTFunction
            with torch.cuda.device(x.device):
                if torch.is_grad_enabled() and (want_dx or any(p.requires_grad for p in plan.params)):
                    return _FasterViTFunction.apply(plan, x, *plan.params)
                return plan.run_forward(x).clone()
        params = self._params
        if features_only:
            # forward_features: the `norm`-ed last-level map, differentiable like forward_levels
            return self._eval_dense(x, ((len(self.model.levels) - 1, self.model.norm),), -1, features=True)[0]
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            # differentiable eval forward: the inference launch list as below, the backward recomputes it
            # (engine_train._EvalGradFunction)
            from .engine_train import _EvalGradFunction
            return _EvalGradFunction.apply_fast(self, plan, x, *params)
        return self._run_eval(plan, x, features_only)

    def eval_grad_plan(self, x: torch.Tensor, want_dx: bool = True, data_only: tuple | None = None) -> Plan:
        """The plan the backward of a differentiable eval forward runs (built at the first such backward): a TrainPlan
        whose BatchNorms use their running statistics and whose backward also writes the image gradient (want_dx).
        data_only: engine_train.stage_mask of the stages that get no parameter gradient; one plan per mask."""
        kind = None if isinstance(self.model.head, nn.Linear) else "pooled"
        spec = dict(kind=kind, eval=True)
        if not want_dx or (data_only is not None and any(data_only)):
            spec.update(want_dx=bool(want_dx), data_only=None if data_only is None else tuple(map(bool, data_only)))
        return self._plan(x, spec)

    def eval_grad_plans(self) -> list:
        """the eval-grad plans built so far (one per input shape)"""
        return [p for p in self.plans.values() if getattr(p, "eval_grad", False)]

    def release_eval_grad_plans(self) -> None:
        """Drop the eval-grad plans: each holds a training step's saved activations on the device for the model's
        lifetime otherwise. The next eval-mode backward builds its plan again."""
        for k in [k for k, p in self.plans.items() if getattr(p, "eval_grad", False)]:
            del self.plans[k]

    def _run_eval(self, plan: Plan, x: torch.Tensor, features_only: bool = False) -> torch.Tensor:
        """the inference launch list (re-packing the fp16 weights first when they changed); returns a new tensor"""
        with torch.cuda.device(x.device):
            wk = plan.weights_key()
            if self._prepped.get(id(plan)) != wk:
                plan.run_ops(plan.prep_ops, None)
                self._prepped[id(plan)] = wk
            if plan.use_graphs:
                xs_ = plan.static_input(x)
                plan.run_captured("forward", lambda: plan.run_ops(plan.ops, xs_))
            else:
                plan.run_ops(plan.ops, x)
            if features_only:
                # forward_features (fv.py:949-953): the BatchNorm-ed last-level map, NCHW fp32 like the reference
                f = plan.feat
                nf = self.model.num_features
                out = torch.empty(plan.B, nf, f["H"], f["W"], dtype=torch.float32, device=x.device)
                L.call("fvit_feature_map_fwd", f["xs"].data_ptr(), nf, f["crop_map"].data_ptr(), plan.B,
                       f["H"] * f["W"], nf, plan.norm_fold[0].data_ptr(), plan.norm_fold[1].data_ptr(), out.data_ptr())
                return out
        if plan.logits is None:
            # num_classes = 0: head is nn.Identity, forward returns the pooled features (fv.py:955-958)
            return plan.pooled[:, :self.model.num_features].float()
        return plan.logits.clone()

    def forward_levels(self, x: torch.Tensor, out_indices: tuple, norms=None, frozen_stages: int = -1) -> tuple:
        """Each requested level's output before its Downsample as an NCHW fp32 map; `norms` = one BatchNorm2d (or None)
        per index, `frozen_stages` = the backbone's frozen prefix (fastervit.py:801-812).
        Eval: the inference launch list is run piecewise up to the marks where those activations are live, and each
        norm is applied with its running statistics. With grad enabled and the image or a parameter on the outputs'
        path requiring grad, the outputs are differentiable (engine_train._EvalDenseGradFunction).
        Train: a levels-mode train plan, differentiable; the norms use batch statistics."""
        norms = tuple(norms) if norms is not None else (None,) * len(out_indices)
        if len(norms) != len(out_indices) or (self.model.training and not out_indices):
            raise L.FvitError("forward_levels: give one norm (or None) per requested level, and at least one level")
        outs = tuple(zip(out_indices, norms))
        if self.model.training:
            return self._dense_train(x, dict(kind="levels", outs=outs, frozen=int(frozen_stages)))
        if not outs:
            return self._eval_levels(self._plan(x), x, ())
        return self._eval_dense(x, outs, int(frozen_stages), features=False)

    def _eval_dense(self, x: torch.Tensor, outs: tuple, frozen: int, features: bool) -> tuple:
        """Eval-mode dense outputs (forward_levels, forward_features): the inference launch list, wrapped in an
        autograd node when a gradient can flow (nothing is built for it until its backward runs)."""
        plan = self._plan(x)
        params = self._dense_params(outs)
        if torch.is_grad_enabled() and (x.requires_grad or self._path_requires_grad(outs, params)):
            from .engine_train import _EvalDenseGradFunction
            return _EvalDenseGradFunction.apply(self, plan, (outs, frozen, features), x, *params)
        return self._eval_dense_fwd(plan, x, outs, features)

    def _dense_params(self, outs: tuple) -> list:
        """the parameters an eval levels plan of these outputs hands gradients to, in its flat-buffer order
        (TrainPlan._setup_train): the model's, then the level norms that are not the model's own (the backbone's)"""
        params = list(self._params)
        known = {id(p) for p in params}
        for _, bn in outs:
            for p in norm_params(bn):
                if id(p) not in known:
                    known.add(id(p))
                    params.append(p)
        return params

    def _path_requires_grad(self, outs: tuple, params: list) -> bool:
        from .engine_train import levels_path
        on = levels_path(self.model, outs)
        return any(p.requires_grad for p in params if id(p) in on)

    def _eval_dense_fwd(self, plan: Plan, x: torch.Tensor, outs: tuple, features: bool) -> tuple:
        if features:
            return (self._run_eval(plan, x, features_only=True),)
        feats = self._eval_levels(plan, x, tuple(i for i, _ in outs))
        if all(bn is None for _, bn in outs):
            return feats
        res = []
        for (idx, bn), f in zip(outs, feats):
            if bn is None:
                res.append(f)
                continue
            B, C, H, W = f.shape
            if norm_kind(bn) == "ln":   # a channel LayerNorm: the same kernel as in train mode, no statistics saved
                rows = f.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous()
                out = torch.empty(B, C, H, W, dtype=torch.float32, device=f.device)
                with torch.cuda.device(f.device):
                    L.call("fvit_feature_map_ln_fwd", rows.data_ptr(), C, None, B, H * W, C, bn.weight.data_ptr(),
                           bn.bias.data_ptr(), float(bn.eps), out.data_ptr(), None, None)
                res.append(out)
                continue
            # the level norm folded into the layout-conversion kernel, running statistics (fastervit.py:816-827)
            scale = (bn.weight * torch.rsqrt(bn.running_var + bn.eps)).float().contiguous()
            shift = (bn.bias - bn.running_mean * scale).float().contiguous()
            rows = f.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous()     # token-major view of the level output
            out = torch.empty(B, C, H, W, dtype=torch.float32, device=f.device)
            with torch.cuda.device(f.device):
                L.call("fvit_feature_map_fwd", rows.data_ptr(), C, None, B, H * W, C, scale.data_ptr(), shift.data_ptr(),
                       out.data_ptr())
            res.append(out)
        return tuple(res)

    def eval_dense_plan(self, x: torch.Tensor, outs: tuple, frozen: int, want_dx: bool | None = None,
                        data_only: tuple | None = None) -> Plan:
        """The plan the backward of a differentiable eval-mode dense output runs (built at the first such backward): a
        levels-mode TrainPlan whose BatchNorms (the level norms too) use their running statistics. want_dx (default:
        frozen = -1): its backward also writes the image gradient, crossing the frozen prefix and the `data_only`
        stages (engine_train.stage_mask) with the activation gradient alone."""
        spec = dict(kind="levels", outs=outs, frozen=frozen, eval=True)
        if want_dx is not None:
            spec.update(want_dx=bool(want_dx), data_only=None if data_only is None else tuple(map(bool, data_only)))
        return self._plan(x, spec)

    def _eval_levels(self, plan: Plan, x: torch.Tensor, out_indices: tuple) -> tuple:
        with torch.cuda.device(x.device):
            wk = plan.weights_key()
            if self._prepped.get(id(plan)) != wk:
                plan.run_ops(plan.prep_ops, None)
                self._prepped[id(plan)] = wk
            want = {f"levels.{i}.out": i for i in out_indices}
            outs, done = {}, 0
            for upto, name, where in plan.marks:
                if name in want:
                    plan.run_ops(plan.ops[done:upto], x)
                    done = upto
                    outs[want[name]] = plan._extract(where)
            plan.run_ops(plan.ops[done:], x)
        return tuple(outs[i] for i in out_indices)

    def forward_head(self, feats: torch.Tensor) -> torch.Tensor:
        """avgpool + flatten + head (fv.py:955-958) on the [B, C, H, W] map `forward_features` returns (an already
        pooled [B, C] tensor is accepted too), eval mode: pooling kernel + one fvit_gemm. With grad enabled and the
        features or the head's parameters requiring grad, the output is differentiable (engine_train._EvalHeadFunction:
        fvit_head_eval_bwd, fp32)."""
        m = self.model
        if m.training and torch.is_grad_enabled():
            raise L.FvitError("forward_head is an inference helper; the autograd training path is forward()")
        if (not feats.is_cuda or feats.dim() not in (2, 4) or feats.shape[1] != m.num_features
                or feats.dtype != torch.float32):
            raise L.FvitError(f"forward_head expects a CUDA float32 [B, {m.num_features}, H, W] (or pooled [B, "
                              f"{m.num_features}]) tensor, got {tuple(feats.shape)} {feats.dtype} on {feats.device}")
        self._check_weights()
        params = tuple(m.head.parameters()) if isinstance(m.head, nn.Linear) else ()
        if torch.is_grad_enabled() and (feats.requires_grad or any(p.requires_grad for p in params)):
            from .engine_train import _EvalHeadFunction
            return _EvalHeadFunction.apply(self, feats, *params)
        return self._head_fwd(feats)

    def _head_fwd(self, feats: torch.Tensor) -> torch.Tensor:
        m = self.model
        with torch.cuda.device(feats.device):
            nf, Bf = m.num_features, feats.shape[0]
            ld = _ru(nf, 8)
            f32 = feats.contiguous()
            a16 = torch.zeros(Bf, ld, dtype=torch.float16, device=feats.device)
            if feats.dim() == 4:
                L.call("fvit_nchw_pool_f16", f32.data_ptr(), Bf, nf, f32.shape[2] * f32.shape[3], a16.data_ptr(), ld)
            else:
                L.call("fvit_cast_pad_f16", f32.data_ptr(), nf, a16.data_ptr(), ld, Bf, nf, ld)
            if not isinstance(m.head, torch.nn.Linear):
                return a16[:, :nf].float()
            w16 = torch.zeros(m.num_classes, ld, dtype=torch.float16, device=feats.device)
            L.call("fvit_cast_pad_f16", m.head.weight.data_ptr(), nf, w16.data_ptr(), ld, m.num_classes, nf, ld)
            out = torch.empty(Bf, m.num_classes, dtype=torch.float32, device=feats.device)
            L.gemm(a16, w16, kc=nf, col_shift=m.head.bias, out_f32=out)
        return out
