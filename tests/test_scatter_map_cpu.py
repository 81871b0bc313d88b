"""fvit_scatter_add_rows adds with a plain read-modify-write (no atomics), so it is only correct for a map that is
injective on its non-negative entries (include/fvit.h). Host-side check, on plans built on the CPU (nothing launched),
that every map the training plans pass to it -- the carrier-token ct_dewindow backward -- is injective."""
import pytest
import torch


def _plan(case, B):
    import fastervit_b200 as F
    from fastervit_b200.engine_train import TrainPlan
    from oracle.configs import CASES, cfg_of
    entry, kw, _ = CASES[case]
    model = F.create_model(entry, drop_path_rate=0.0, **kw).train()
    res = cfg_of(case)["resolution"]
    H, W = (res, res) if isinstance(res, int) else res
    return TrainPlan(model, B, H, W, torch.device("cpu"))


@pytest.mark.parametrize("case,B", [("tiny_a", 3), ("tiny_ar", 2), ("tiny_ar148", 2), ("fv0", 2)])
def test_scatter_add_maps_are_injective(case, B):
    plan = _plan(case, B)
    by_ptr = {t.data_ptr(): t for t in plan.bufs.named.values()}
    calls = [args for ops in (plan.ops, plan.bwd_ops) for fn, args, name in ops if name == "fvit_scatter_add_rows"]
    assert calls, "the plan has carrier tokens: its backward scatters them back"
    for args in calls:
        rows = args[5]
        mp = by_ptr[args[4]].flatten()[:rows]
        valid = mp[mp >= 0]
        assert valid.numel() == torch.unique(valid).numel(), (case, "map repeats a destination row")
