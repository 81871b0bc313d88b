"""Geometry classes of the attention entry points, the table of GPU cases that covers them, and an fp64 reference with a
per-element error bound. Imports without a GPU: tests/test_attn_geometry_cpu.py checks on the CPU that every attention
launch of the plans the package builds falls in a class some case covers; tests/test_attn_geometry_gpu.py runs the
cases.

Entry points (include/fvit.h) and where each one's dispatch is decided:
  fvit_attn_tc_fwd        attn_sm100.cu:273 window slot 16 / 32 / 64 / 128 rows (gpt = 128 / slot windows per 128-row
                          tile, the last tile partial when groups % gpt != 0); attn_sm100.cu:284-286 hdp 32 / 64 / 80
  fvit_attn_tc_bwd        attn_sm100.cu:601 slot 16 / 32 / 64; attn_sm100.cu:348-361 the CTA walk: one head per CTA when
                          the grid has at least one CTA per head, head-major items otherwise (grid < heads: only under
                          fvit_set_sm_limit)
  fvit_attn_loop_fwd      attn_loop_sm100.cu:304 nqt = nkt = ceil(S / 128) key tiles; attn_loop_sm100.cu:182, 207 a
                          partial last key tile when S % 128 != 0; attn_loop_sm100.cu:266 the optional lse rows
  fvit_attn_loop_bwd_long attn_loop_sm100.cu:677 nt key / query tiles, attn_loop_sm100.cu:482 partial last tile
  fvit_hat_attn_fwd       hat_sm100.cu:350 slot (hdp 64 only, hat_sm100.cu:342); qkv_out saved or not
  fvit_attn_core_fwd      ops_sm100.cu:1034-1059 one-shot kernel with its [S, S] score matrix in <= 48 KB of shared
                          memory (the default limit), one-shot above 48 KB (opt-in up to 227 KB), or the streaming
                          kernel past 227 KB; block of 256 threads from S * S >= 4096 (the streaming kernel: always);
                          ops_sm100.cu:491 shared rows of hd + 1 floats: head widths <= 80, or the SIMT-only widths
                          above 80 (multiples of 8 such as 96 and 128, or not, such as 81)
  fvit_attn_core_bwd      train_sm100.cu:1771-1776 the whole window in shared memory, <= 48 KB or above (refused past
                          227 KB); train_sm100.cu:713-717 head-pad columns zeroed when hdp > hd
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import NamedTuple

import torch

U16 = 2.0 ** -11        # unit roundoff of fp16
U32 = 2.0 ** -24        # unit roundoff of fp32
HALF_SUB = 2.0 ** -25   # half the fp16 subnormal spacing: absolute rounding error near zero
SUB = HALF_SUB / U16    # the same in units of U16 (the bound's magnitudes M are multiplied by U16)
LOG2E = 1.4426950408889634
H100_SMS = 132          # SM count of an H100 SXM: the persistent grids' width at full size
SMEM_MAX = 227 * 1024   # opt-in shared memory per block on sm_90
SMEM_DEFAULT = 48 * 1024
# Per-element bound: |got - ref| <= C_ATTN * U16 * M + U16 * |ref| + HALF_SUB for fp16 results, with M the reference
# formula evaluated on absolute values (out: |P||V|, dv: |P|^T |dO|, dq / dk: |dS| through |K| / |Q|, |dS| bounded by
# P o (|dO||V|^T + |delta|); dbias: summed over windows; plus HALF_SUB per fp16 probability or dS operand, for the ones
# that fall into fp16's subnormal range). Worst |err| / (U16 M) measured over every case and softmax edge of
# tests/test_attn_geometry_gpu.py (after the U16 |ref| output rounding; H100 80GB HBM3, 700 W): loop_bwd_long 0.96 (dv,
# bias std 20), tc_bwd 0.87 (dv), tc_fwd 0.67, loop_fwd 0.62, hat_attn_fwd 0.19, core_fwd 0.008, core_bwd 0.005 (fp32
# throughout). C_ATTN = 2 keeps a factor 2 of margin over the worst.
C_ATTN = 2.0
# whole-tensor bars of tests/test_attn_gpu.py, kept so that the per-element check is never weaker
FWD_BAR, BWD_BAR = 2e-3, 4e-3

TC = ("fvit_attn_tc_fwd", "fvit_attn_tc_bwd", "fvit_attn_loop_fwd", "fvit_attn_loop_bwd_long", "fvit_hat_attn_fwd")
SIMT = ("fvit_attn_core_fwd", "fvit_attn_core_bwd")
ENTRIES = TC + SIMT
BWD = ("fvit_attn_tc_bwd", "fvit_attn_loop_bwd_long", "fvit_attn_core_bwd")


# ---------------------------------------------------------------------------------------------- plan launches
class Launch(NamedTuple):
    entry: str
    S: int
    hdp: int        # padded head width (the SIMT forward: its unpadded head_dim, the only width it takes)
    groups: int
    heads: int
    bias: bool
    dbias: bool
    hd: int         # unpadded head width where the entry point takes it (the backward kernels), else hdp
    lse: bool       # fvit_attn_loop_fwd: log-sum-exp rows written
    save_qkv: bool  # fvit_hat_attn_fwd: qkv_out given


# argument positions per entry point (include/fvit.h): groups, S, heads, hdp, bias, and dbias / hd / lse / qkv_out
_ARGS = {
    "fvit_attn_tc_fwd": dict(g=2, S=3, h=4, d=5, b=6),
    "fvit_attn_loop_fwd": dict(g=2, S=3, h=4, d=5, b=6, lse=10),
    "fvit_hat_attn_fwd": dict(g=6, S=7, h=8, d=9, b=10, qkv=14),
    "fvit_attn_tc_bwd": dict(g=4, S=5, h=6, hd=7, d=8, b=9, db=13),
    "fvit_attn_loop_bwd_long": dict(g=7, S=8, h=9, d=10, b=11, db=15),
    "fvit_attn_core_fwd": dict(g=2, S=3, h=4, d=5, b=6),
    "fvit_attn_core_bwd": dict(g=4, S=5, h=6, hd=7, d=8, b=9, db=13),
}


def attention_launches(plan):
    """Launch(...) of every attention-core launch in the plan's launch lists."""
    for lst in (v for v in vars(plan).values() if isinstance(v, list)):
        for op in lst:
            if isinstance(op, tuple) and len(op) == 3 and isinstance(op[2], str) and op[2] in _ARGS:
                args = op[1][2] if op[0] == "unless_deploy" else op[1]
                a = _ARGS[op[2]]
                hdp = args[a["d"]]
                yield Launch(op[2], args[a["S"]], hdp, args[a["g"]], args[a["h"]], args[a["b"]] is not None,
                             "db" in a and args[a["db"]] is not None, args[a["hd"]] if "hd" in a else hdp,
                             "lse" in a and args[a["lse"]] is not None, "qkv" in a and args[a["qkv"]] is not None)


# ---------------------------------------------------------------------------------------------- geometry classes
def slot_of(S: int) -> int:
    return 16 if S <= 16 else (32 if S <= 32 else (64 if S <= 64 else 128))


def simt_fwd_smem(S: int, hd: int) -> int:
    """one-shot kernel's shared memory (ops_sm100.cu:1034)"""
    return (3 * S * (hd + 1) + S * (S + 1)) * 4


def simt_bwd_smem(S: int, hd: int) -> int:
    """fvit_attn_core_bwd's shared memory (train_sm100.cu:1771): the whole window"""
    return (4 * S * (hd + 1) + S * (S + 1) + S) * 4


def _tiles(S: int) -> str:
    n = (S + 127) // 128
    return "1 tile" if n == 1 else ("2 tiles" if n == 2 else "3+ tiles")


def geometry_class(entry: str, S: int, hdp: int, groups: int, heads: int, *, hd: int | None = None, lse: bool = False,
                   save_qkv: bool = False, sms: int = H100_SMS) -> tuple:
    """The dispatch decisions a launch of `entry` at this geometry takes (see the module docstring); `sms` is the width
    the persistent grids are capped at (fvit_set_sm_limit, default the H100's SM count)."""
    hd = hdp if hd is None else hd
    if entry == "fvit_attn_tc_fwd":
        slot = slot_of(S)
        return entry, hdp, f"slot {slot}", "partial tile" if groups % (128 // slot) else "full tiles"
    if entry == "fvit_attn_tc_bwd":
        slot = slot_of(S)
        tiles = -(-groups // (128 // slot))
        grid = min(tiles * heads, sms)
        return entry, hdp, f"slot {slot}", "one head per CTA" if grid >= heads else "head-major"
    if entry == "fvit_attn_loop_fwd":
        return entry, hdp, _tiles(S), "S % 128 == 0" if S % 128 == 0 else "partial key tile", "lse" if lse else "no lse"
    if entry == "fvit_attn_loop_bwd_long":
        return entry, hdp, _tiles(S), "S % 128 == 0" if S % 128 == 0 else "partial key tile"
    if entry == "fvit_hat_attn_fwd":
        return entry, hdp, f"slot {slot_of(S)}", "qkv_out" if save_qkv else "no qkv_out"
    if entry == "fvit_attn_core_fwd":
        sm = simt_fwd_smem(S, hdp)
        kind = "streaming" if sm > SMEM_MAX else ("one-shot > 48 KB" if sm > SMEM_DEFAULT else "one-shot <= 48 KB")
        block = 256 if kind == "streaming" or S * S >= 4096 else 128
        width = "hd <= 80" if hdp <= 80 else ("hd > 80, % 8 == 0" if hdp % 8 == 0 else "hd > 80, % 8 != 0")
        return entry, kind, f"block {block}", width
    if entry == "fvit_attn_core_bwd":
        sm = simt_bwd_smem(S, hd)
        kind = "refused (> 227 KB)" if sm > SMEM_MAX else ("> 48 KB" if sm > SMEM_DEFAULT else "<= 48 KB")
        return entry, kind, "hdp == hd" if hdp == hd else "hdp > hd (pad columns)"
    raise ValueError(entry)


def launch_class(a: Launch, sms: int = H100_SMS) -> tuple:
    return geometry_class(a.entry, a.S, a.hdp, a.groups, a.heads, hd=a.hd, lse=a.lse, save_qkv=a.save_qkv, sms=sms)


def required_classes() -> set:
    """Every class the issue-level contract names, minus the impossible combinations: what CASES must cover."""
    req = set()
    for hdp in (32, 64, 80):
        for slot in (16, 32, 64, 128):
            req.add(("fvit_attn_tc_fwd", hdp, f"slot {slot}", "full tiles"))
            if slot < 128:          # one window per tile at slot 128: never partial
                req.add(("fvit_attn_tc_fwd", hdp, f"slot {slot}", "partial tile"))
        for slot in (16, 32, 64):
            for walk in ("one head per CTA", "head-major"):
                req.add(("fvit_attn_tc_bwd", hdp, f"slot {slot}", walk))
        for t in ("1 tile", "2 tiles", "3+ tiles"):
            for m in ("S % 128 == 0", "partial key tile"):
                req.add(("fvit_attn_loop_bwd_long", hdp, t, m))
                for lse in ("lse", "no lse"):
                    req.add(("fvit_attn_loop_fwd", hdp, t, m, lse))
    for slot in (16, 32, 64, 128):
        for q in ("qkv_out", "no qkv_out"):
            req.add(("fvit_hat_attn_fwd", 64, f"slot {slot}", q))
    for w in ("hd <= 80", "hd > 80, % 8 == 0", "hd > 80, % 8 != 0"):
        req.add(("fvit_attn_core_fwd", "one-shot <= 48 KB", "block 128", w))
        req.add(("fvit_attn_core_fwd", "one-shot > 48 KB", "block 128", w))
        req.add(("fvit_attn_core_fwd", "one-shot > 48 KB", "block 256", w))
        req.add(("fvit_attn_core_fwd", "streaming", "block 256", w))
    # 256 threads need S >= 64, which puts a window of hd > 80 above 48 KB
    req.add(("fvit_attn_core_fwd", "one-shot <= 48 KB", "block 256", "hd <= 80"))
    for k in ("<= 48 KB", "> 48 KB"):
        for p in ("hdp == hd", "hdp > hd (pad columns)"):
            req.add(("fvit_attn_core_bwd", k, p))
    return req


# ---------------------------------------------------------------------------------------------- GPU cases
@dataclass(frozen=True)
class Case:
    entry: str
    S: int
    heads: int
    hd: int
    groups: int
    hdp: int = 0            # 0: Plan._head_pad(hd) for the tensor-core kernels, hd for the SIMT forward
    bias: str = "bias"      # "bias" (and dbias), "no_dbias" (bias, dbias = NULL) or "no_bias" (neither)
    lse: bool = True        # fvit_attn_loop_fwd: write the log-sum-exp rows
    save_qkv: bool = False  # fvit_hat_attn_fwd: qkv_out
    C: int = 64             # fvit_hat_attn_fwd: input width
    sm_limit: int = 0       # fvit_set_sm_limit for the call (0: full grid)

    @property
    def width(self) -> int:
        if self.hdp:
            return self.hdp
        if self.entry == "fvit_attn_core_fwd" or self.hd > 80:
            return self.hd
        return 32 if self.hd <= 32 else (64 if self.hd <= 64 else 80)

    @property
    def cls(self) -> tuple:
        return geometry_class(self.entry, self.S, self.width, self.groups, self.heads, hd=self.hd,
                              lse=self.lse, save_qkv=self.save_qkv, sms=self.sm_limit or H100_SMS)

    @property
    def id(self) -> str:
        e = self.entry.replace("fvit_", "").replace("_attn", "")
        extra = "".join([f"-{self.bias}" if self.bias != "bias" else "", "" if self.lse else "-nolse",
                         "-qkvout" if self.save_qkv else "", f"-sm{self.sm_limit}" if self.sm_limit else ""])
        return f"{e}-S{self.S}-h{self.heads}-d{self.hd}p{self.width}-g{self.groups}{extra}"


def _c(entry, S, heads, hd, groups, **kw):
    return Case(entry, S, heads, hd, groups, **kw)


_F, _B, _LF, _LB, _H, _SF, _SB = ENTRIES[0], ENTRIES[1], ENTRIES[2], ENTRIES[3], ENTRIES[4], ENTRIES[5], ENTRIES[6]

CASES: list[Case] = [
    # -- tile forward: slot 16 (carriers S = 4 .. 16), 32 (S = 25), 64 (S = 49 / 53), 128 (S = 85 / 100 / 128); group
    #    counts that fill the last tile or leave it partial; hd below the padded width (pad columns)
    _c(_F, 16, 4, 32, 16), _c(_F, 13, 2, 24, 11), _c(_F, 16, 8, 49, 8), _c(_F, 4, 4, 64, 5, bias="no_bias"),
    _c(_F, 16, 2, 80, 24), _c(_F, 9, 3, 72, 7),
    _c(_F, 25, 4, 32, 8), _c(_F, 32, 2, 16, 9, bias="no_bias"), _c(_F, 25, 4, 49, 12), _c(_F, 29, 2, 64, 7),
    _c(_F, 32, 2, 80, 4), _c(_F, 25, 2, 80, 5, bias="no_bias"),
    _c(_F, 49, 8, 32, 10), _c(_F, 53, 4, 32, 37), _c(_F, 53, 4, 49, 6), _c(_F, 64, 2, 64, 9),
    _c(_F, 49, 4, 80, 12), _c(_F, 53, 2, 72, 5),
    _c(_F, 85, 2, 16, 5), _c(_F, 128, 2, 49, 3, bias="no_bias"), _c(_F, 100, 2, 80, 3), _c(_F, 128, 2, 80, 2),
    # -- tile backward: the three slots at every width, full grid (one head per CTA), dbias NULL / bias NULL at 32 / 64;
    #    the head-major walk under a grid narrower than the head count (tiles < heads)
    _c(_B, 16, 4, 32, 16), _c(_B, 8, 4, 49, 10), _c(_B, 16, 2, 80, 9), _c(_B, 13, 2, 72, 8, bias="no_dbias"),
    _c(_B, 25, 4, 24, 8), _c(_B, 32, 2, 64, 7, bias="no_bias"), _c(_B, 29, 4, 80, 6),
    _c(_B, 53, 4, 32, 11), _c(_B, 49, 2, 49, 9, bias="no_dbias"), _c(_B, 53, 4, 80, 5), _c(_B, 64, 2, 32, 4),
    _c(_B, 49, 8, 32, 6, sm_limit=3), _c(_B, 53, 6, 49, 5, sm_limit=5), _c(_B, 49, 8, 80, 4, sm_limit=7),
    _c(_B, 16, 8, 32, 12, sm_limit=3), _c(_B, 16, 6, 64, 9, sm_limit=1), _c(_B, 13, 8, 80, 5, sm_limit=7),
    _c(_B, 25, 8, 32, 10, sm_limit=7), _c(_B, 32, 6, 64, 6, sm_limit=3), _c(_B, 20, 8, 80, 7, sm_limit=1),
    # -- key-loop forward: one tile (65 .. 128, the training plans' single-tile case), two (S = 148 / 196 / 256), many
    #    (S = 384 / 576); S % 128 == 0 or a partial last tile; with and without the lse rows; bias NULL at 32 / 64
    _c(_LF, 68, 4, 16, 6), _c(_LF, 68, 2, 32, 4, lse=False), _c(_LF, 128, 2, 32, 5, lse=False), _c(_LF, 128, 2, 32, 3),
    _c(_LF, 68, 2, 49, 5, lse=False), _c(_LF, 100, 3, 64, 4), _c(_LF, 128, 2, 64, 3, lse=False),
    _c(_LF, 128, 2, 49, 4, bias="no_bias"),
    _c(_LF, 64, 4, 80, 6), _c(_LF, 85, 2, 80, 3, bias="no_bias", lse=False), _c(_LF, 128, 2, 80, 3),
    _c(_LF, 128, 2, 80, 2, lse=False),
    _c(_LF, 148, 8, 32, 6), _c(_LF, 148, 4, 32, 3, lse=False), _c(_LF, 256, 2, 32, 2), _c(_LF, 256, 2, 24, 2, lse=False, bias="no_bias"),
    _c(_LF, 196, 4, 49, 3), _c(_LF, 150, 2, 64, 2, bias="no_bias", lse=False), _c(_LF, 256, 2, 64, 2),
    _c(_LF, 256, 2, 49, 2, lse=False, bias="no_bias"),
    _c(_LF, 148, 4, 80, 4), _c(_LF, 148, 2, 72, 3, lse=False), _c(_LF, 256, 2, 80, 2), _c(_LF, 256, 1, 80, 2, lse=False),
    _c(_LF, 576, 2, 32, 1), _c(_LF, 420, 2, 16, 1, lse=False), _c(_LF, 384, 2, 32, 1), _c(_LF, 384, 1, 32, 2, lse=False),
    _c(_LF, 576, 2, 49, 1), _c(_LF, 388, 1, 64, 2, lse=False), _c(_LF, 384, 2, 64, 1), _c(_LF, 384, 1, 49, 1, lse=False),
    _c(_LF, 576, 2, 80, 1), _c(_LF, 388, 1, 80, 1, lse=False), _c(_LF, 384, 1, 80, 1), _c(_LF, 384, 1, 72, 1, lse=False),
    # -- key-loop backward (S % 4 == 0): same tile counts; dbias NULL / bias NULL at 32 / 64
    _c(_LB, 68, 4, 16, 6), _c(_LB, 128, 2, 32, 3), _c(_LB, 100, 3, 49, 4, bias="no_dbias"), _c(_LB, 128, 2, 64, 3),
    _c(_LB, 64, 4, 80, 5), _c(_LB, 128, 2, 80, 2),
    _c(_LB, 148, 8, 32, 5), _c(_LB, 256, 2, 32, 2, bias="no_bias"), _c(_LB, 196, 4, 49, 3), _c(_LB, 256, 2, 64, 2),
    _c(_LB, 148, 4, 80, 4), _c(_LB, 256, 1, 72, 2),
    _c(_LB, 576, 2, 32, 1), _c(_LB, 384, 2, 24, 1), _c(_LB, 388, 1, 64, 2, bias="no_bias"), _c(_LB, 384, 2, 49, 1),
    _c(_LB, 420, 1, 80, 1), _c(_LB, 384, 1, 80, 1),
    # -- fused qkv projection + attention (hdp 64): every slot, with and without the saved qkv
    _c(_H, 16, 4, 49, 11), _c(_H, 4, 2, 64, 6, save_qkv=True, C=128), _c(_H, 25, 2, 49, 7, save_qkv=True),
    _c(_H, 32, 2, 40, 4), _c(_H, 53, 4, 49, 9, C=192), _c(_H, 49, 2, 64, 6, save_qkv=True),
    _c(_H, 85, 2, 49, 3, save_qkv=True), _c(_H, 128, 2, 64, 2),
    # -- SIMT forward: one-shot <= 48 KB (block 128 / 256), one-shot > 48 KB (block 128 / 256), streaming; head widths
    #    <= 80, above 80 multiples of 8 (96, 128) and not (81, 100); bias NULL
    _c(_SF, 53, 4, 24, 7), _c(_SF, 64, 2, 16, 5), _c(_SF, 36, 2, 81, 5), _c(_SF, 20, 2, 96, 4),
    _c(_SF, 40, 2, 81, 3, bias="no_bias"), _c(_SF, 53, 4, 80, 4), _c(_SF, 53, 2, 96, 5), _c(_SF, 53, 2, 81, 6), _c(_SF, 64, 2, 81, 3),
    _c(_SF, 49, 2, 128, 3, bias="no_bias"),
    _c(_SF, 148, 4, 32, 3), _c(_SF, 125, 2, 96, 3), _c(_SF, 173, 2, 81, 2), _c(_SF, 85, 2, 128, 2),
    _c(_SF, 229, 2, 16, 2), _c(_SF, 300, 2, 96, 1), _c(_SF, 260, 2, 81, 1, bias="no_bias"), _c(_SF, 576, 1, 128, 1),
    # -- SIMT backward: <= 48 KB or above, hdp = hd or head-padded (the 65 .. 128-token windows with S % 4 != 0)
    _c(_SB, 53, 2, 24, 5, hdp=24), _c(_SB, 36, 2, 16, 4, hdp=32), _c(_SB, 85, 4, 16, 3, hdp=32),
    _c(_SB, 125, 2, 24, 3, hdp=32, bias="no_dbias"), _c(_SB, 173, 2, 16, 2, hdp=16), _c(_SB, 85, 2, 96, 2),
    _c(_SB, 53, 2, 96, 3, bias="no_bias"), _c(_SB, 101, 2, 49, 2, hdp=64), _c(_SB, 121, 2, 72, 2, hdp=80),
]


# ---------------------------------------------------------------------------------------------- fp64 reference
def _chunks(groups: int, S: int, heads: int):
    step = max(1, min(groups, (1 << 24) // (heads * S * S)))
    for g0 in range(0, groups, step):
        yield g0, min(groups, g0 + step)


def reference(q, k, v, bias, scale, do=None, qk_err=None):
    """fp64 attention on [groups, heads, S, hd] operands (bias [heads, S, S] or None, do like q or None).
    Returns out, lse (log2 units, [groups, heads, S]) and the magnitudes M_out; with do also dq, dk, dv, dbias (summed over
    windows) and M_dq, M_dk, M_dv, M_dbias (see C_ATTN). qk_err (optional, [groups, heads, S, S]) bounds each logit's
    error in units of U16 (q and k that were themselves rounded to fp16), propagated into M_out."""
    groups, heads, S, _ = q.shape
    res = {n: torch.zeros_like(q) for n in ("out", "M_out")}
    res["lse"] = torch.zeros(groups, heads, S, dtype=torch.float64, device=q.device)
    if do is not None:
        for n in ("dq", "dk", "dv", "M_dq", "M_dk", "M_dv"):
            res[n] = torch.zeros_like(q)
        res["dbias"] = torch.zeros(heads, S, S, dtype=torch.float64, device=q.device)
        res["M_dbias"] = torch.zeros_like(res["dbias"])
    for g0, g1 in _chunks(groups, S, heads):
        qc, kc, vc = q[g0:g1], k[g0:g1], v[g0:g1]
        att = (qc @ kc.transpose(-2, -1)) * scale
        if bias is not None:
            att = att + bias
        lse = torch.logsumexp(att, -1)
        p = torch.exp(att - lse[..., None])
        o = p @ vc
        res["out"][g0:g1], res["lse"][g0:g1] = o, lse * LOG2E
        m = p @ vc.abs()
        if qk_err is not None:
            pe = p * qk_err[g0:g1]
            m = m + pe @ vc.abs() + pe.sum(-1, keepdim=True) * o.abs()
        # + the kernels' fp16 probabilities (unnormalised, max 1) that fall into fp16's subnormal range: an absolute
        # HALF_SUB each
        res["M_out"][g0:g1] = m + SUB * vc.abs().sum(-2, keepdim=True)
        if do is None:
            continue
        dc = do[g0:g1]
        dp = dc @ vc.transpose(-2, -1)
        delta = (p * dp).sum(-1, keepdim=True)
        ds = p * (dp - delta)
        a_dp = dc.abs() @ vc.abs().transpose(-2, -1)
        a_ds = p * (a_dp + (p * a_dp).sum(-1, keepdim=True))
        res["dv"][g0:g1] = p.transpose(-2, -1) @ dc
        res["dq"][g0:g1] = scale * (ds @ kc)
        res["dk"][g0:g1] = scale * (ds.transpose(-2, -1) @ qc)
        res["dbias"] += ds.sum(0)
        # (+ the subnormal floor of the fp16 P and dS operands of the tensor-core gradient MMAs)
        res["M_dv"][g0:g1] = p.transpose(-2, -1) @ dc.abs() + SUB * dc.abs().sum(-2, keepdim=True)
        res["M_dq"][g0:g1] = scale * (a_ds @ kc.abs() + SUB * kc.abs().sum(-2, keepdim=True))
        res["M_dk"][g0:g1] = scale * (a_ds.transpose(-2, -1) @ qc.abs() + SUB * qc.abs().sum(-2, keepdim=True))
        res["M_dbias"] += a_ds.sum(0)
    return res


def bound16(ref: torch.Tensor, mag: torch.Tensor, c: float = None) -> torch.Tensor:
    """per-element bound of an fp16 result"""
    return (C_ATTN if c is None else c) * U16 * mag + U16 * ref.abs() + HALF_SUB


def needed_c(got: torch.Tensor, ref: torch.Tensor, mag: torch.Tensor) -> float:
    """the smallest C_ATTN this fp16 result would pass with"""
    over = ((got.double() - ref).abs() - U16 * ref.abs() - HALF_SUB).clamp_min(0)
    return float((over / (U16 * mag).clamp_min(1e-300)).max()) if over.numel() else 0.0


def assert_within(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str) -> None:
    """every element within its own bound (NaN fails)"""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, e.g. {i}: got "
                             f"{got[i].item()!r} want {ref[i].item()!r} (|err| {err[i].item():.3g} > {bound[i].item():.3g})")


def assert_whole(got: torch.Tensor, ref: torch.Tensor, bar: float, what: str, mag: torch.Tensor | None = None) -> None:
    """the whole-tensor max-rel bar of tests/test_attn_gpu.py. With `mag` (the bound's M), a result that cancels to
    less than 1 % of its magnitude (the gradients of one-hot softmax rows: dS ~ P (dP - delta) ~ 0) is left to the
    per-element bound: relative to a maximum near zero the bar measures nothing but rounding noise."""
    den = ref.abs().max().item()
    if mag is not None and den < 1e-2 * mag.max().item():
        return
    err = (got.double() - ref).abs().max().item() / den if den > 0 else (got.double() - ref).abs().max().item()
    assert err < bar, (what, err)


def heads_view(x: torch.Tensor, groups: int, S: int, n: int, heads: int, hdp: int, hd: int) -> torch.Tensor:
    """[groups * S, n * heads * hdp] -> fp64 [n, groups, heads, S, hd] (pad columns dropped)"""
    return x.double().reshape(groups, S, n, heads, hdp)[..., :hd].permute(2, 0, 3, 1, 4)


def rows_view(x: torch.Tensor, hdp: int) -> torch.Tensor:
    """fp64 [n, groups, heads, S, hd] -> [groups * S, n * heads * hdp] (pad columns zero)"""
    n, groups, heads, S, hd = x.shape
    out = torch.zeros(groups, S, n, heads, hdp, dtype=x.dtype, device=x.device)
    out[..., :hd] = x.permute(1, 3, 0, 2, 4)
    return out.reshape(groups * S, n * heads * hdp)


def largest_simt_bwd_S(hd: int) -> int:
    S = 1
    while simt_bwd_smem(S + 1, hd) <= SMEM_MAX:
        S += 1
    return S

