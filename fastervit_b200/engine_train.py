"""Training plan: train-mode forward (batch-statistics BatchNorm, saved activations) and the backward pass
of FasterViT as static launch lists over libfvit_sm100.so.

The reference has no backward code — fv.py relies on autograd (train.py:879-896) — so this module *is*
the backward of SURVEY §8 row a16: per layer it emits the weight-gradient GEMM (both operands MN-major:
dW = dZ^T X, split-K with fp32 atomics into one flat gradient buffer), the data-gradient GEMM (B = the
forward's packed weight read as an MN-major operand, so no transposed copies exist), and the HBM-bound
reductions (bias / LayerNorm / BatchNorm / layer-scale / positional-MLP gradients).

Numerics: activation gradients are fp16 operands (fp32 along the residual stream) multiplied by a
power-of-two scale S chosen on the device from max|dlogits| (scal[0] = S, scal[1] = 1/S); a branch whose
layer scale gamma is tiny (1e-5 at init for fv3+) is additionally normalised by s_b = 2^-floor(log2 max|gamma|)
so no fp16 product underflows. Parameter gradients are fp32 and exact in scale.
"""
from __future__ import annotations

import weakref

import torch

from . import lib as L
from .engine import Plan, _ru, norm_kind, norm_params
from .engine_train_conv import ConvPartEmitters
from .engine_train_levels import _ONE, TokenLevelEmitters


def levels_path(model, outs) -> set[int]:
    """ids of the parameters the level outputs `outs` ((level, norm or None), ...) depend on: the stem, the levels up to
    the highest requested one without its Downsample, and the level norms' weights and biases (engine.norm_params)"""
    stop = max(i for i, _ in outs)
    on = set()
    for name, p in model.named_parameters():
        if name.startswith("levels."):
            li = int(name.split(".")[1])
            if li < stop or (li == stop and not name.startswith(f"levels.{li}.downsample.")):
                on.add(id(p))
        elif name.startswith("patch_embed."):
            on.add(id(p))
    for _, bn in outs:
        on.update(map(id, norm_params(bn)))
    return on


def stage_mask(model, needs_grad) -> tuple:
    """Per stage (0 = the stem, 1 + i = levels[i] with the Downsample that follows it) whether none of its parameters
    takes a gradient: `needs_grad(p)` says which parameters do. Such a stage's backward is data-only."""
    mods = [model.patch_embed, *model.levels]
    return tuple(not any(needs_grad(p) for p in mod.parameters()) for mod in mods)


def _sm_count() -> int:
    """SMs of the current device; plans built without one (host-side tests) assume an H100 SXM's 132."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return 132


class TrainPlan(Plan, ConvPartEmitters, TokenLevelEmitters):
    """Train-mode forward + backward launch lists. `spec` selects what the forward returns and the backward starts from:
    None = the logits (classification step, fv.py:949-965); {"kind": "pooled"} = the pooled features of a
    num_classes = 0 model (fv.py:955-958); {"kind": "levels", "outs": ((level, BatchNorm2d or None), ...),
    "frozen": frozen_stages} = NCHW level outputs taken before each level's Downsample, each optionally through a
    batch-statistics BatchNorm2d (forward_levels, forward_features, FasterViTBackbone; the backbone's frozen prefix,
    downstream/.../dino/fastervit.py:801-812, runs its BatchNorms on running statistics and gets no backward).
    {"kind": None | "pooled", "eval": True} = the eval-grad plan, the backward of an eval()-mode forward: every BatchNorm
    on its running statistics (not updated), no stochastic depth, and a backward that also yields the image gradient
    `dx` (engine.Engine.forward).
    "want_dx": the backward continues through conv1 into `self.dx`, the fp32 NCHW image gradient (default: an eval plan
    without a frozen prefix). "data_only" (eval plans): a stage_mask() of stages whose parameters get no gradient; the
    frozen prefix always is one. A data-only stage's backward carries the activation gradient alone (no weight-gradient
    GEMM, no bias / norm / layer-scale / positional-MLP reduction), and is not emitted at all when nothing below it
    reads that gradient (`_needed`)."""

    def __init__(self, model, B: int, H: int, W: int, device, spec: dict | None = None):
        self.bwd_ops: list[tuple] = []
        self.fwd_zero: list[torch.Tensor] = []   # accumulators zeroed before every forward (BN statistics)
        self.saved_levels: list[dict] = []
        self.spec = spec
        self.kind = None if spec is None else spec["kind"]
        self.eval_grad = bool(spec is not None and spec.get("eval"))
        nlev = len(model.levels)
        outs = tuple(spec.get("outs", ())) if spec is not None else ()
        for i, bn in outs:
            if not 0 <= i < nlev:
                raise L.FvitError(f"out index {i} is not a level of this model (0 .. {nlev - 1})")
            if bn is not None and norm_kind(bn) == "bn" and (bn.weight is None or bn.running_mean is None
                                                              or bn.momentum is None):
                raise L.FvitError("level norms must be affine BatchNorm2d modules with running statistics and a momentum")
        self.stop_level = max(i for i, _ in outs) if self.kind == "levels" else nlev - 1
        fs = int(spec.get("frozen", -1)) if spec is not None else -1
        self.stem_frozen = fs >= 0                       # fastervit.py:801-812
        self.n_frozen_lv = fs - 1 if fs >= 2 else 0      # levels[0 .. fs-2]
        frozen_mods = ([model.patch_embed] if self.stem_frozen else []) + [model.levels[i] for i in range(self.n_frozen_lv)]
        self._frozen_bn = {id(b) for fm in ([model] if self.eval_grad else frozen_mods) for b in fm.modules()
                           if isinstance(b, torch.nn.BatchNorm2d)}
        # frozen BatchNorms of the stem (the tracking backbone's FrozenBatchNorm2d): a fixed affine from running
        # statistics in every mode, crossed by the data gradient alone, while the convolutions around them still train
        stem_norms = (model.patch_embed.conv_down[1], model.patch_embed.conv_down[4])
        if any(norm_kind(b) not in ("bn", "frozen") for b in stem_norms):
            raise L.FvitError("the stem norms are BatchNorm2d or frozen BatchNorms")
        self._fixed_bn = {id(b) for b in stem_norms if norm_kind(b) == "frozen"}
        self._frozen_bn |= self._fixed_bn
        self._frozen_params = {id(p) for fm in frozen_mods for p in fm.parameters()}
        stages = [model.patch_embed, *model.levels]
        mask = spec.get("data_only") if spec is not None else None
        if mask is not None and (not self.eval_grad or len(mask) != len(stages)):
            raise L.FvitError("data_only is a per-stage mask (stem, then one entry per level) of an eval plan")
        self.data_only = tuple(s < len(frozen_mods) or bool(mask is not None and mask[s]) for s in range(len(stages)))
        self.want_dx = bool(spec.get("want_dx", self.eval_grad and fs < 0)) if spec is not None else False
        # the lowest stage the backward has to reach: -1 = the image, else the first stage with a parameter gradient
        self._bwd_low = -1 if self.want_dx else min((s for s, d in enumerate(self.data_only) if not d), default=len(stages))
        self._data_only_params = {id(p) for s, mod in enumerate(stages) if self.data_only[s] for p in mod.parameters()}
        super().__init__(model, B, H, W, True, device)

    def _needed(self, stage: int) -> bool:
        """does anything read the gradient this stage's backward produces (a trained stage below it, or the image)"""
        return stage >= self._bwd_low

    # ------------------------------------------------------------------------------ infrastructure
    def _setup_train(self) -> None:
        m, nb = self.model, self.bufs
        self.params = [p for p in m.parameters()]
        n_model = len(self.params)
        # level norms that are not part of the model (the backbone's norm{i}) get flat-buffer slices after the model's,
        # so that the data-parallel buckets reduce them too
        known = {id(p) for p in self.params}
        for _, bn in (self.spec or {}).get("outs", ()):
            for p in norm_params(bn):
                if id(p) not in known:
                    known.add(id(p))
                    self.params.append(p)
        offs, n = {}, 0
        for k, p in enumerate(self.params):
            if k == n_model:
                self._n_model_flat = n         # end of the model's own slices
            if self.eval_grad and id(p) in self._data_only_params:
                continue   # no slice: nothing accumulates a gradient for it (a train plan keeps one layout per model)
            offs[id(p)] = n
            n += _ru(p.numel(), 64)            # 256-byte aligned slices
        if n_model == len(self.params):
            self._n_model_flat = n
        self.gflat = nb.new("grad.flat", (n,), torch.float32)
        self._goff = offs
        self._on_path = self._params_on_path()
        self.scratch_n = 0
        self._scratch_req: list[tuple[str, int]] = []
        self._bwd_side: set[int] = set()     # backward launches that run as a side branch (engine_train_levels.py)
        self._bwd_side_wgrad: set[int] = set()    # weight-gradient launches: side branch on a single GPU only (below)
        self._side_reads: dict[int, tuple] = {}   # side launch -> shared gradient buffers it reads (WAR hazards)
        # device scalars: [0] S, [1] 1/S, [2] 1.0, then per-branch (s_b, 1/s_b, 1/(S s_b))
        self._nscal = 3
        self._branch_slots: list[tuple[int, object]] = []

    def G(self, p: torch.Tensor) -> int:
        """device pointer of the flat-buffer gradient slice of parameter p"""
        return self.gflat.data_ptr() + 4 * self._goff[id(p)]

    def _drop_rate(self, level: int) -> float:
        """stochastic-depth rate of the next block (the schedule of fv.py:901, in block order). Blocks in the frozen
        prefix run without it: the reference eval()s that prefix (fastervit.py:801-812), where DropPath is the
        identity."""
        rate = self.model.drop_path_rates[self._block_counter]
        return 0.0 if level < self.n_frozen_lv or self.eval_grad else rate

    def _params_on_path(self) -> set[int]:
        """ids of the parameters the requested outputs depend on (the rest get no gradient: .grad stays None, as under
        autograd). Levels mode: the stem and levels up to the highest requested one without its Downsample, the level
        norms; not the frozen prefix, nor `norm` / `head` unless forward_features asked for `norm`."""
        if self.kind != "levels":
            return {id(p) for p in self.params} - self._data_only_params
        return levels_path(self.model, self.spec["outs"]) - self._data_only_params

    def grad_views_on_path(self) -> list:
        """grad_views() with None for the parameters off the path of the requested outputs"""
        return [g if id(p) in self._on_path else None for p, g in zip(self.params, self.grad_views())]

    def _load_grads(self, grads) -> None:
        """copy autograd's per-step output gradients into the static buffers the captured backward reads"""
        if self.kind is None:
            self._dlogits[:, :self._ncls].copy_(grads)
        else:
            for d, gr in zip(self.dense, grads):
                if gr is None:      # autograd leaves the gradient of an unused output unset: zeros
                    d["dy"].zero_()
                else:
                    d["dy"].copy_(gr)

    def grad_views(self) -> list[torch.Tensor]:
        """Per-parameter views of a *copy* of the flat gradient buffer: autograd's AccumulateGrad may keep
        the tensors it is handed, and the flat buffer itself is reused (zeroed) by the next backward."""
        flat = self.gflat.clone()
        return [flat[self._goff[id(p)]: self._goff[id(p)] + p.numel()].view_as(p) if id(p) not in self._data_only_params
                else None for p in self.params]   # (a data-only stage's parameters: None, as autograd expects)

    def _scratch(self, name: str, n: int) -> int:
        """reserve n zero-initialised fp32 (re-zeroed at the start of every backward); returns offset"""
        off = self.scratch_n
        self.scratch_n += _ru(n, 64)
        self._scratch_req.append((name, off))
        return off

    def _branch(self, gamma) -> dict:
        """device-scalar pointers of a residual branch: dgrad alpha (1/s_b) and wgrad alpha (1/(S s_b))"""
        if not isinstance(gamma, torch.Tensor):
            return _ONE
        slot = self._nscal
        self._nscal += 3
        self._branch_slots.append((slot, gamma))
        return dict(gamma=gamma, s=("scal", slot), inv_s=("scal", slot + 1), w_alpha=("scal", slot + 2))

    def _finish_train(self) -> None:
        nb = self.bufs
        self.scal = nb.new("grad.scalars", (_ru(self._nscal, 16),), torch.float32)
        self.scal[2] = 1.0
        self.scr = nb.new("grad.scratch", (max(self.scratch_n, 64),), torch.float32)
        sp = self.scal.data_ptr()
        for slot, gamma in self._branch_slots:
            self._op(self.prep_ops, "fvit_pow2_norm", gamma.data_ptr(), gamma.numel(), sp + 4 * slot)
        # resolve symbolic pointers ("scal", i) / ("scr", off) in the op lists
        def res(v):
            if isinstance(v, tuple) and len(v) == 2 and v[0] == "scal":
                return sp + 4 * v[1]
            if isinstance(v, tuple) and len(v) == 2 and v[0] == "scr":
                return self.scr.data_ptr() + 4 * v[1]
            return v
        for lst in (self.ops, self.bwd_ops, self.prep_ops, self._scale_ops):
            for i, (fn, args, name) in enumerate(lst):
                if isinstance(args, tuple):
                    lst[i] = (fn, tuple(res(a) for a in args), name)
        for g in self._gemm_keep:
            for f, v in g._sym.items():
                setattr(g, f, res(v))
        # per-backward prologue: zero accumulators, pick the gradient scale, per-branch wgrad alphas
        pro: list[tuple] = [("zero", self.gflat, "memset"), ("zero", self.scr, "memset")]
        for lv in self.lv:
            pro.append(("zero", lv["g"], "memset"))
        if self.kind == "levels":
            if self.feat["kind"] == "conv":   # the top level's gradient is accumulated into a cleared buffer
                pro.append(("zero", self.feat["g"], "memset"))
            pro.append(("zero", self._dense_acc, "memset"))
        self._bwd_prologue = pro
        self._branch_alpha_ops = []
        for slot, _ in self._branch_slots:
            self._branch_alpha_ops.append((self.lib.fvit_vec_mul, (sp + 4, 0, sp + 4 * (slot + 1), 0, sp + 4 * (slot + 2), 1),
                                           "fvit_vec_mul"))

    # ------------------------------------------------------------------------------ weight gradients as a side branch
    # A weight-gradient GEMM reads an activation gradient (a per-level buffer every block reuses) and a saved
    # activation, and adds into parameter-gradient memory nobody reads before the next bucket point: a leaf. As a
    # side-branch launch it runs beside the data-gradient chain -- two persistent grids share the SMs, each filling
    # the other's tail waves. The one hazard is write-after-read on the reused gradient buffers: the launch that next
    # overwrites such a buffer first waits for the event behind its last side-branch reader (`wait_side`).
    def _side_from(self, first: int, *reads: int) -> None:
        """make backward launches [first, now) side-branch launches that read the reusable buffers `reads`"""
        for i in range(first, len(self.bwd_ops)):
            self._bwd_side_wgrad.add(i)
            self._side_reads[i] = tuple(reads)

    def _side_set(self):
        """Launches that go to the side branch (graphs only). Under a gradient all-reduce the weight-gradient GEMMs stay
        there too: a second persistent grid does compete with NCCL's CTAs for the SMs the capped launches leave free."""
        if not self.use_graphs:
            return None
        return self._bwd_side | self._bwd_side_wgrad

    def _before_write(self, *ptrs: int) -> None:
        """the next backward launch overwrites `ptrs`: order it behind their side-branch readers"""
        self.bwd_ops.append(("wait_side", tuple(ptrs), "wait_side"))

    def _split_k(self, m: int, n: int, k_rows: int, ntaps: int = 1) -> int:
        tiles = ((m + 127) // 128) * ((n + 127) // 128) * ntaps
        kb = (k_rows + 63) // 64
        sms = _sm_count()
        best, best_cost = 1, float("inf")
        for sk in range(1, max(1, min(64, kb // 8)) + 1):
            # time model (us): waves of CTAs x (K blocks of one unit x ~0.26 us per 128x128x64 block + epilogue);
            # the split-K epilogue is a pass of fp32 vector reductions into L2 (~10 us per tile)
            cost = -(-tiles * sk // sms) * (kb / sk * 0.26 + (10.0 if sk > 1 else 3.0))
            if cost < best_cost - 1e-9:
                best, best_cost = sk, cost
        return best

    # ------------------------------------------------------------------------------ linear layer backward
    def _linear_bwd(self, *, lin, w16, ldw, x16, ldx, dz16, lddz, rows, n_out, k_in, br, gW=None, gW_ld=None,
                    dx16=None, lddx=0, dx_act=L.ACT_NONE, dx_aux=None, ld_aux=0, dx_alpha=None, bias_to=None,
                    flops_k=None, want_dgrad=True, bias_done=False, dx_colsum=None, gW_row_map=None,
                    data_only=False) -> None:
        """dW[n_out, k_in] += alpha_w * dz16^T @ x16 ; db += alpha_w * colsum(dz16) ; dx16 = alpha_d * dz16 @ W.
        data_only: the last of the three alone."""
        fk = k_in if flops_k is None else flops_k
        if not data_only:
            gW = self.G(lin.weight) if gW is None else gW
            gW_ld = k_in if gW_ld is None else gW_ld
            n0 = len(self.bwd_ops)
            self._gemm(a=dz16, a_rows=rows, lda=lddz, a_mn=True, b=x16, b_rows=rows, ldb=ldx, b_mn=True, m=n_out, n=k_in,
                       kc=rows, split_k=self._split_k(n_out, k_in, rows), alpha_ptr=br["w_alpha"], out_f32=gW,
                       ld_o32=gW_ld, row_map=gW_row_map, target=self.bwd_ops, flops=2.0 * rows * n_out * fk)
            if (lin.bias is not None or bias_to is not None) and not bias_done:
                dst = bias_to if bias_to is not None else self.G(lin.bias)
                self._op(self.bwd_ops, "fvit_colsum", dz16, 1, lddz, None, None, 0, rows, n_out, None, br["w_alpha"], dst,
                         None)
            self._side_from(n0, dz16)   # (weight gradient + bias column sums: both only read dz16)
        if want_dgrad:
            self._before_write(dx16)
            self._gemm(a=dz16, a_rows=rows, lda=lddz, b=w16, b_rows=n_out, ldb=ldw, b_mn=True, m=rows, n=k_in, kc=n_out,
                       alpha_ptr=dx_alpha if dx_alpha is not None else br["inv_s"], act=dx_act, aux=dx_aux, ld_aux=ld_aux,
                       out_f16=dx16, ld_o16=lddx, out_colsum=dx_colsum[0] if dx_colsum else None,
                       out_colsum_alpha=dx_colsum[1] if dx_colsum else None, target=self.bwd_ops,
                       flops=2.0 * rows * n_out * fk)

    def _ln_bwd(self, ln, dy, lddy: int, dy_map, xh, rs, rows: int, C: int, g, g_map, use_g: int, clear_moved: int,
                data_only: bool) -> None:
        """LayerNorm backward into the gradient rows g (through g_map; fvit_ln_bwd in include/fvit.h): with the weight /
        bias gradients (fvit_ln_bwd), or the input gradient alone in a data-only stage (fvit_ln_dgrad)"""
        args = (dy, lddy, dy_map, xh, C, rs, ln.weight.data_ptr(), rows, C, g, C, g_map, use_g, clear_moved)
        if data_only:
            self._op(self.bwd_ops, "fvit_ln_dgrad", *args)
        else:
            self._op(self.bwd_ops, "fvit_ln_bwd", *args, ("scal", 1), self.G(ln.weight), self.G(ln.bias))

    # ------------------------------------------------------------------------------ plan construction
    def _build(self) -> None:
        m, B = self.model, self.B
        self.bwd_flops: dict[int, float] = {}
        self._scale_ops: list[tuple] = []   # levels mode: per-output statistics passes + the gradient-scale finalize
        self._setup_train()
        self._build_forward()
        self._build_backward()
        self._finish_train()

    # forward / backward emitters: the ConvPartEmitters / TokenLevelEmitters mixins (engine_train_conv.py, engine_train_levels.py)

    # ------------------------------------------------------------------------------ execution
    def claim(self) -> "_Claim":
        """Mark this instance in flight (engine.Engine._train_instance then hands the next forward another one): its
        saved activations belong to the autograd node that keeps the returned token, until release(token) after that
        node's backward, or until the node, and the token with it, is freed without one."""
        token = _Claim()
        self._claim = weakref.ref(token)
        return token

    def release(self, token: "_Claim") -> None:
        if self.in_flight() and self._claim() is token:
            self._claim = None

    def in_flight(self) -> bool:
        ref = getattr(self, "_claim", None)
        return ref is not None and ref() is not None

    def adopt_pivots(self, first: "TrainPlan") -> None:
        """Centre this instance's BatchNorm sums on the pivots of its pool's first instance (engine_train_conv.
        _bn_col_shift: the running means when that one was built), so that a forward of one input key rounds the same
        way whichever instance it runs on."""
        for name, t in first.bufs.named.items():
            if name.endswith(".pivot"):
                self.bufs.named[name].copy_(t)

    def run_forward(self, x: torch.Tensor) -> torch.Tensor:
        # saved activations / batch statistics / drop masks live in this plan's persistent buffers: a new forward
        # invalidates the state an earlier, not yet differentiated forward left behind (checked in backward)
        self.fwd_generation = getattr(self, "fwd_generation", 0) + 1
        if not self.eval_grad:   # (the eval-grad forward writes no parameter or buffer)
            L.bump_weights_epoch()   # BatchNorm running statistics are updated through raw pointers
        def body(xin):
            for t in self.fwd_zero:
                t.zero_()
            if self.drop_specs:
                self._gen_drop_masks()   # stochastic-depth masks of this step (torch RNG, like timm's DropPath)
            if self.use_graphs:
                self.run_ops_branches(self.prep_ops)
            else:
                self.run_ops(self.prep_ops, None)
            self.run_ops(self.ops, xin)
            for bn in self._bn_modules:
                bn.num_batches_tracked += 1
        if self.use_graphs and not getattr(self, "forced_drop_masks", None):
            xs_ = self.static_input(x)
            self.run_captured("train forward", lambda: body(xs_))
        else:
            body(x)
        return self.logits if self.kind is None else None   # (pooled / levels mode: self.outputs)

    def _bwd_start(self, dlogits: torch.Tensor | None) -> None:
        if dlogits is not None:
            self._dlogits[:, :self._ncls].copy_(dlogits)
        self.run_ops(self._bwd_prologue, None)
        if self.kind == "levels":
            # every requested output's statistics pass (with the max |dy| fused in), then S over all of them
            self.run_ops(self._scale_ops, None)
        else:
            src = self._dlogits if self.kind is None else self._dpool_in
            rc = self.lib.fvit_grad_scale_init(src.data_ptr(), src.numel(), 64.0, self.scal.data_ptr(), L.stream_ptr())
            if rc:
                raise L.FvitError(self.lib.fvit_last_error().decode())
        self.run_ops(self._branch_alpha_ops, None)

    def run_backward(self, dlogits) -> None:
        """backward launch list from the output gradient(s): the logits' (classification), the pooled features'
        (pooled mode) or a list with one NCHW map gradient (or None) per requested level output"""
        grp = getattr(self.model, "_grad_allreduce", None)
        if grp is None:
            self._load_grads(dlogits)

            def body():
                self._bwd_start(None)
                self.run_ops(self.bwd_ops, None, side=self._side_set())
            self.run_captured("backward", body)
            return
        # data parallel: each bucket's all-reduce is issued the moment the launches that finish its gradients are
        # enqueued, so NCCL (its own stream) overlaps the rest of the backward pass. The launch list is cut at the
        # bucket points: every segment is one CUDA graph (like the single-GPU backward), the all-reduces in between are
        # ordinary NCCL calls -- collectives captured INTO a graph work too, but live graphs holding NCCL work make
        # destroy_process_group() hang at exit, so they stay outside.
        self._load_grads(dlogits)
        red = GradBucketReducer(self.gflat, None if grp is True else grp)
        if getattr(self, "_ar_shadow", None) is None:
            self._ar_shadow = self._allreduce_shadow(red.world, red.measure_busbw())
        if getattr(self, "_bwd_segments", None) is None:
            segs, start = [], 0
            for i, op in enumerate(self.bwd_ops):
                if op[0] == "bucket":
                    segs.append((start, i, op[1]))
                    start = i + 1
            segs.append((start, len(self.bwd_ops), None))
            self._bwd_segments = segs
        self._ar_active = red
        try:
            for n, (lo, hi, bucket) in enumerate(self._bwd_segments):
                def body(lo=lo, hi=hi, first=(n == 0)):
                    if first:
                        self._bwd_start(None)
                    self._op_base = lo
                    try:
                        self.run_ops(self.bwd_ops[lo:hi], None, side=self._side_set())
                    finally:
                        self._op_base = 0
                if hi > lo or n == 0:   # (the list ends with a bucket point: nothing to capture after it)
                    self.run_captured(f"backward segment {n}", body)
                if bucket is not None:
                    red.reduce(*bucket)
        finally:
            self._ar_active = None
        red.finish(self.grad_buckets)

    def _allreduce_shadow(self, world: int, busbw: float | None = None) -> dict:
        """{backward op index: SM cap} for the launches that run while a bucket's all-reduce is in flight. NCCL's CTAs
        cannot co-reside with a GEMM CTA (227 KB of shared memory, one per SM): a full-width persistent grid launched
        into the reduction would run its last CTAs as a second wave, doubling that launch. The window is estimated at
        plan time: bucket bytes over the all-reduce bus bandwidth against the launches' algorithmic FLOPs at the
        model's typical 700 TFLOP/s; those launches are capped to (SM count) - FVIT_NCCL_CTAS SMs (default 16 =
        NCCL_MAX_CTAS set by enable_grad_allreduce callers such as bench.py)."""
        import os
        reserve = int(os.environ.get("FVIT_NCCL_CTAS", "16"))
        if world <= 1 or reserve <= 0:
            return {}
        sms = _sm_count()
        cap = max(8, sms - reserve)
        shadow: dict[int, int] = {}
        # all-reduce bus bandwidth: measured once per plan on the idle fabric (GradBucketReducer.measure_busbw); the
        # table is the fallback
        if not busbw or busbw <= 0:
            busbw = {2: 200e9, 3: 300e9, 4: 400e9}.get(world, 600e9)
        self.ar_busbw = busbw
        for i, op in enumerate(self.bwd_ops):
            if op[0] != "bucket":
                continue
            lo, hi = op[1]
            t_need = 1.5 * 2.0 * (world - 1) / world * (hi - lo) * 4 / busbw   # seconds, with margin
            t = 0.0
            for j in range(i + 1, len(self.bwd_ops)):
                if t >= t_need:
                    break
                shadow[j] = cap
                t += max(self.bwd_flops.get(j, 0.0) / 700e12, 8e-6)
        return shadow

    def profile(self, x: torch.Tensor) -> list[dict]:
        """Per-launch CUDA-event timing of one training step (forward list, then backward list with the
        gradient of sum(logits)/B as a stand-in loss gradient)."""
        def timed(name, fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            torch.cuda._sleep(int(2e8))
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            return dict(name=name, ms=e0.elapsed_time(e1), flops=0.0, phase="step")

        for t in self.fwd_zero:
            t.zero_()
        # per-step work around the two launch lists: weight re-packing (parameters change every optimizer step),
        # accumulator clears, the copy that hands the flat gradient buffer to autograd
        out = [timed("prep: repack weights to fp16 operands", lambda: self.run_ops(self.prep_ops, None)),
               timed("backward prologue: clear gradient buffers", lambda: self.run_ops(self._bwd_prologue, None)),
               timed("gradient hand-off copy", lambda: self.grad_views())]
        for ops, flops, tag in ((self.ops, self.op_flops, ""), (self.bwd_ops, self.bwd_flops, "")):
            if ops is self.bwd_ops:
                self._bwd_start(torch.full((self.B, self._ncls), 1.0 / self.B, device=self._dlogits.device))
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(ops) + 1)]
            torch.cuda.synchronize()
            torch.cuda._sleep(int(8e8))
            evs[0].record()
            for i, op in enumerate(ops):
                self.run_ops([op], x)
                evs[i + 1].record()
            torch.cuda.synchronize()
            out += [dict(name=op[2], ms=evs[i].elapsed_time(evs[i + 1]), flops=flops.get(i, 0.0),
                         phase="bwd" if ops is self.bwd_ops else "fwd", **self._op_desc(op))
                    for i, op in enumerate(ops) if op[0] not in ("wait_side", "bucket")]   # (markers launch nothing)
        return out


class GradBucketReducer:
    """Asynchronous mean all-reduce of slices of the flat gradient buffer (train.py:542-551's DDP, restated for
    a single autograd node): `reduce(lo, hi)` is called from the backward launch list at the points where the
    slice [lo, hi) is final; `finish` reduces whatever was not covered and waits for all of them."""

    def __init__(self, flat: torch.Tensor, group=None):
        import torch.distributed as dist
        if not dist.is_available() or not dist.is_initialized():
            raise L.FvitError("enable_grad_allreduce() needs an initialised torch.distributed process group")
        self.dist, self.flat, self.group = dist, flat, group
        self.world = dist.get_world_size(group)
        self.avg = dist.get_backend(group) == "nccl"   # gloo has no AVG
        self.pending: list = []
        self.done: list[tuple[int, int]] = []

    def reduce(self, lo: int, hi: int) -> None:
        if self.world == 1 or hi <= lo:
            return
        op = self.dist.ReduceOp.AVG if self.avg else self.dist.ReduceOp.SUM
        self.pending.append(self.dist.all_reduce(self.flat[lo:hi], op=op, group=self.group, async_op=True))
        self.done.append((lo, hi))

    def measure_busbw(self, nbytes: int = 64 << 20) -> float | None:
        """All-reduce bus bandwidth (bytes/s) of this group as configured (NCCL_MAX_CTAS, topology), timed once on a
        slice of the flat buffer before the backward pass zeroes it: sizes the SM cap windows of the launch list."""
        if self.world == 1 or not self.avg or not self.flat.is_cuda:
            return None
        n = min(self.flat.numel(), nbytes // 4)
        buf = self.flat[:n]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for i in range(3):   # two warm-ups (channel setup), one timed
            if i == 2:
                ev[0].record()
            self.dist.all_reduce(buf, op=self.dist.ReduceOp.AVG, group=self.group)
        ev[1].record()
        ev[1].synchronize()
        ms = ev[0].elapsed_time(ev[1])
        bw = torch.tensor([2.0 * (self.world - 1) / self.world * n * 4 / (ms * 1e-3)], device=self.flat.device)
        self.dist.all_reduce(bw, op=self.dist.ReduceOp.MIN, group=self.group)   # every rank plans the same windows
        return float(bw.item())

    def finish(self, buckets: list[tuple[int, int]]) -> None:
        for lo, hi in buckets:
            if (lo, hi) not in self.done:
                self.reduce(lo, hi)
        for w in self.pending:
            w.wait()
        if not self.avg and self.world > 1:
            self.flat.div_(self.world)


def allreduce_mean_(flat: torch.Tensor, group=None) -> torch.Tensor:
    """Data parallel (train.py:542-551): the ONE exchange of the path — the flat gradient buffer is averaged
    over the ranks with a single all-reduce (NCCL over NVLink / NVSwitch on GPUs; gloo in the CPU
    tests). BatchNorm statistics stay per-GPU like the reference (sync_bn: false)."""
    import torch.distributed as dist
    if not dist.is_available() or not dist.is_initialized():
        raise L.FvitError("enable_grad_allreduce() needs an initialised torch.distributed process group")
    world = dist.get_world_size(group)
    if world == 1:
        return flat
    if dist.get_backend(group) == "nccl":
        dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=group)
    else:  # gloo has no AVG
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.div_(world)
    return flat


class _Claim:
    """the token by which an autograd node holds its train plan instance (TrainPlan.claim)"""
    __slots__ = ("__weakref__",)


def _check_fresh(ctx, plan: TrainPlan, what: str) -> None:
    if ctx.generation != plan.fwd_generation:
        raise L.FvitError(
            f"backward of a stale forward: another train-mode forward of the same {what} ran in between and overwrote "
            "the saved activations of this one. Call backward before the next forward, or let several forwards await "
            "their backward with model.set_train_forwards_in_flight(n) (multi-view losses, clips of frames; each "
            "costs one more set of activations on the device)")


class _FasterViTFunction(torch.autograd.Function):
    """One autograd node for the whole network: forward runs the train plan, backward runs the backward
    plan and hands out views of the flat gradient buffer (one per nn.Parameter, in .parameters() order).
    The node holds its plan instance (TrainPlan.claim) until its backward has run."""

    @staticmethod
    def forward(ctx, plan: TrainPlan, x: torch.Tensor, *params):
        ctx.plan = plan
        logits = plan.run_forward(x)
        ctx.generation = plan.fwd_generation
        ctx.claim = plan.claim()
        return logits.clone()

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dlogits):
        plan: TrainPlan = ctx.plan
        _check_fresh(ctx, plan, "input shape")
        plan.run_backward(dlogits.contiguous().float())
        res = (None, _train_dx(ctx, plan), *plan.grad_views())
        plan.release(ctx.claim)
        return res


class _DenseFunction(torch.autograd.Function):
    """Autograd node of a pooled / levels-mode train plan: the outputs are copies of the plan's static output buffers;
    backward copies their gradients into the plan's static gradient buffers and runs the backward launch list.
    Parameters off the path of the outputs (and the frozen prefix) get None."""

    @staticmethod
    def forward(ctx, plan: TrainPlan, x: torch.Tensor, *params):
        ctx.plan = plan
        plan.run_forward(x)
        ctx.generation = plan.fwd_generation
        ctx.claim = plan.claim()
        return tuple(o.clone() for o in plan.outputs)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        plan: TrainPlan = ctx.plan
        _check_fresh(ctx, plan, "input shape and outputs")
        plan.run_backward([None if g is None else g.contiguous().float() for g in grads])
        res = (None, _train_dx(ctx, plan), *plan.grad_views_on_path())
        plan.release(ctx.claim)
        return res


def _train_dx(ctx, plan: TrainPlan):
    """the image gradient of a train-mode step: a copy of the plan's static buffer (local to this rank: the gradient
    all-reduce covers parameters only), or None when the plan was built for an input without a gradient"""
    if not ctx.needs_input_grad[1]:
        return None
    if not plan.want_dx:
        raise L.FvitError("the input requires grad but this train plan was built without the image gradient")
    return plan.dx.clone()


class _EvalGradFunction(torch.autograd.Function):
    """Autograd node of a grad-enabled eval()-mode forward (logits, or the pooled features of a num_classes = 0 model).
    forward runs the inference launch list unchanged -- bitwise the output of the same call under no_grad, at its speed
    and memory -- and keeps x. backward recomputes: the eval-grad plan (Engine.eval_grad_plan) runs a saving forward on
    x with every BatchNorm on its running statistics, then its backward from the output gradient, which yields the
    parameter gradients and the image gradient. Which of them autograd asks for (ctx.needs_input_grad) selects the plan:
    a stage none of whose parameters needs a gradient runs the data-only backward, and is skipped when x needs none
    either. Each node recomputes on its own, so several forwards may feed one
    backward; nothing is built until the first backward. First order only: the gradients come from raw kernel buffers
    and carry no graph, so a backward through them (create_graph=True, then differentiating dx) raises."""

    @classmethod
    def apply_fast(cls, *args):
        """Function.apply without its functorch dead-wrapper pass: that pass walks every argument in Python (about
        150 us for a model's few hundred parameters, a third of the node's host cost). It only matters while functorch
        transforms are active, and then the ordinary apply runs."""
        if torch._C._are_functorch_transforms_active():
            return cls.apply(*args)
        return super(torch.autograd.Function, cls).apply(*args)   # (the C implementation underneath)

    @staticmethod
    def forward(ctx, engine, plan, x: torch.Tensor, *params):
        ctx.engine, ctx.plan = engine, plan
        out = engine._run_eval(plan, x)
        ctx.weights_key = engine._prepped[id(plan)]    # (what _run_eval just checked the packed weights against)
        ctx.save_for_backward(x)    # (autograd then rejects a backward after an in-place change of x)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        (x,) = ctx.saved_tensors
        engine, plan = ctx.engine, ctx.plan
        _check_eval_backward(engine.model, plan.weights_key() != ctx.weights_key)
        with torch.cuda.device(x.device):
            needs = dict(zip(map(id, engine._params), ctx.needs_input_grad[3:]))
            gp = engine.eval_grad_plan(x, ctx.needs_input_grad[2], stage_mask(engine.model, lambda p: needs[id(p)]))
            gp.run_forward(x)
            g = gout.contiguous().float()
            gp.run_backward(g if gp.kind is None else [g])
            dx = gp.dx.clone() if ctx.needs_input_grad[2] else None
            return (None, None, dx, *gp.grad_views())


def _check_eval_backward(m, weights_changed: bool, recomputes: bool = True) -> None:
    """what makes the recompute of an eval-mode forward impossible or different from the forward that ran
    (recomputes=False: a backward that reads only its saved input and the head, where deploy mode does not matter)"""
    if weights_changed:
        raise L.FvitError(
            "backward of an eval-mode forward after a weight change: this model's parameters or buffers changed, "
            "or any model's fused optimizer step, EMA update or train-mode forward ran in between (those write "
            "through raw pointers and advance one library-wide epoch, so they count even for another model); the "
            "recomputed forward might not be the one that ran: call backward before them")
    if getattr(m, "_grad_allreduce", None) is not None:
        raise L.FvitError("eval-mode gradients are not all-reduced across ranks: the gradient all-reduce "
                          "(enable_grad_allreduce) only covers train-mode steps")
    if recomputes and any(getattr(mod, "deploy", False) for mod in m.modules()):
        raise L.FvitError("eval-mode gradients need the relative-position-bias MLPs: a module was switched to "
                          "deploy mode (switch_to_deploy caches their output), so they have no gradient path")


def _norm_versions(outs) -> tuple:
    """autograd versions of the level norms' tensors (the backbone's norm{i} are not part of the model's weights key)"""
    return tuple(t._version for _, bn in outs if bn is not None
                 for t in (getattr(bn, n, None) for n in ("weight", "bias", "running_mean", "running_var"))
                 if t is not None)


class _EvalDenseGradFunction(torch.autograd.Function):
    """Autograd node of grad-enabled eval()-mode dense outputs: forward_levels, forward_features and the backbone's
    forward_raw. forward runs the inference extraction unchanged (bitwise the no_grad outputs) and keeps x. backward
    recomputes through the eval levels plan (Engine.eval_dense_plan: a levels-mode TrainPlan with every BatchNorm, the
    level norms included, on running statistics and no stochastic depth), loads the output gradients (an unused output
    is a zero gradient) and runs its backward. The frozen prefix, and every stage none of whose parameters needs a
    gradient, is data-only: crossed by the activation gradient alone when x needs one, not emitted otherwise. Guards
    and first-order restriction as _EvalGradFunction."""

    @staticmethod
    def forward(ctx, engine, plan, spec, x: torch.Tensor, *params):
        outs, frozen, features = spec
        ctx.engine, ctx.plan, ctx.outs, ctx.frozen, ctx.params = engine, plan, outs, frozen, params
        res = engine._eval_dense_fwd(plan, x, outs, features)
        ctx.weights_key = (engine._prepped[id(plan)], _norm_versions(outs))
        ctx.save_for_backward(x)
        ctx.set_materialize_grads(False)   # (an unused output stays None: the plan zeroes its gradient buffer)
        return res

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        (x,) = ctx.saved_tensors
        engine, plan = ctx.engine, ctx.plan
        _check_eval_backward(engine.model, (plan.weights_key(), _norm_versions(ctx.outs)) != ctx.weights_key)
        want_dx = ctx.needs_input_grad[3]
        with torch.cuda.device(x.device):
            needs = dict(zip(map(id, ctx.params), ctx.needs_input_grad[4:]))
            gp = engine.eval_dense_plan(x, ctx.outs, ctx.frozen, want_dx, stage_mask(engine.model, lambda p: needs[id(p)]))
            if len(gp.params) != len(ctx.params) or any(a is not b for a, b in zip(gp.params, ctx.params)):
                raise L.FvitError("the model's parameters changed between an eval-mode forward and its backward")
            gp.run_forward(x)
            gp.run_backward([None if g is None else g.contiguous().float() for g in grads])
            dx = gp.dx.clone() if want_dx else None
            views = [g if p.requires_grad else None for p, g in zip(gp.params, gp.grad_views_on_path())]
            return (None, None, None, dx, *views)


class _EvalHeadFunction(torch.autograd.Function):
    """Autograd node of forward_head under .eval(): forward is the inference helper (fp16 pooling + GEMM) unchanged;
    backward is fvit_head_eval_bwd in fp32 -- the feature gradient through the pooling and the Linear, the head's weight
    gradient from the pooled features recomputed from the saved input, and the bias gradient. First order only."""

    @staticmethod
    def forward(ctx, engine, feats: torch.Tensor, *params):
        ctx.engine = engine
        ctx.key = (tuple(p._version for p in params), L.weights_epoch())
        ctx.save_for_backward(feats)
        return engine._head_fwd(feats)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        (feats,) = ctx.saved_tensors
        m = ctx.engine.model
        head = m.head if isinstance(m.head, torch.nn.Linear) else None
        params = tuple(head.parameters()) if head is not None else ()
        _check_eval_backward(m, (tuple(p._version for p in params), L.weights_epoch()) != ctx.key, recomputes=False)
        B, nf = feats.shape[0], m.num_features
        T = feats.shape[2] * feats.shape[3] if feats.dim() == 4 else 1
        dl = gout.contiguous().float()
        dev = feats.device
        want = ctx.needs_input_grad
        f32 = feats.contiguous()
        dfeats = torch.empty(f32.shape, dtype=torch.float32, device=dev) if want[1] else None
        dW = torch.zeros_like(head.weight) if head is not None and want[2] else None
        db = torch.zeros_like(head.bias) if head is not None and head.bias is not None and want[3] else None
        ws = torch.empty(B * nf, dtype=torch.float32, device=dev) if dW is not None and T > 1 else None
        with torch.cuda.device(dev):
            L.call("fvit_head_eval_bwd", dl.data_ptr(), dl.stride(0), B, dl.shape[1], f32.data_ptr(), nf, T,
                   head.weight.data_ptr() if head is not None else None, L.ptr(ws), L.ptr(dfeats), L.ptr(dW), L.ptr(db))
        return (None, dfeats, dW, db)[:2 + len(params)]
