"""Host-side checks of the dense-prediction train plans (built on the CPU, nothing launched): stochastic depth and the
backward launch list at the frozen prefix of FasterViTBackbone (fastervit.py:801-812)."""
import torch

KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[2, 2, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7])


def _plan(fs, out_indices=(1, 2, 3), drop_path_rate=0.3):
    from fastervit_b200.backbone import FasterViTBackbone
    from fastervit_b200.engine_train import TrainPlan
    bb = FasterViTBackbone("faster_vit_0_any_res", out_indices=out_indices, frozen_stages=fs,
                           drop_path_rate=drop_path_rate, **KW).train()
    norms = [getattr(bb, f"norm{i}") for i in out_indices]
    spec = dict(kind="levels", outs=tuple(zip(out_indices, norms)), frozen=fs)
    return TrainPlan(bb.body, 2, 160, 224, torch.device("cpu"), spec=spec)


def test_frozen_levels_run_without_stochastic_depth():
    """the reference eval()s the frozen prefix, so DropPath is the identity there: no masks are drawn for its blocks"""
    names = {fs: [d["name"] for d in _plan(fs).drop_specs] for fs in (-1, 2, 3)}
    assert any(n.startswith("levels.0.") for n in names[-1])
    assert not any(n.startswith("levels.0.") for n in names[2]) and any(n.startswith("levels.1.") for n in names[2])
    assert not any(n.startswith(("levels.0.", "levels.1.")) for n in names[3])
    assert any(n.startswith("levels.2.") for n in names[3])


def _gemms_into(plan, buf):
    return sum(1 for fn, args, name in plan.bwd_ops if name == "fvit_gemm" and args[0]._obj.out_f32 == buf.data_ptr())


def test_backward_ends_at_the_frozen_prefix():
    """no data gradient is computed for the frozen part: the conv1 data-gradient GEMM of the lowest trained level's
    first block (which only feeds the frozen stem / Downsample) is not emitted, nor anything of the frozen levels"""
    full, fs1, fs2 = _plan(-1), _plan(1), _plan(2)
    assert _gemms_into(full, full.conv_lv[0]["g"]) == 2          # (two blocks per conv level in this config)
    assert _gemms_into(fs1, fs1.conv_lv[1]["g"]) == 2
    assert _gemms_into(fs1, fs1.conv_lv[0]["g"]) == 1
    assert _gemms_into(fs2, fs2.conv_lv[1]["g"]) == 1 and _gemms_into(fs2, fs2.conv_lv[0]["g"]) == 0
    assert len(fs2.bwd_ops) < len(fs1.bwd_ops) < len(full.bwd_ops)


def test_outputs_inside_the_frozen_prefix_add_their_norm_gradients_once():
    plan = _plan(4, out_indices=(1, 2))    # both requested levels are frozen: only the norms train
    fmb = [args for fn, args, name in plan.bwd_ops if name == "fvit_feature_map_bwd"]
    assert len(fmb) == 2 and all(a[14] is None for a in fmb)     # one per output, no level gradient written
    assert not [op for op in plan.bwd_ops if op[2] == "fvit_gemm"]
