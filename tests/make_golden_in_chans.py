"""Generate the in_chans != 3 golden fixtures (tests/golden/tiny_c4.pt, tiny_ar_c1.pt) with oracle/make_golden.py.

    FASTERVIT_REFERENCE=<path to the reference checkout> python tests/make_golden_in_chans.py

The cases are reduced models built with `in_chans` by the unmodified reference. make_golden.run_case draws its
images with oracle.synth_input, which makes 3-channel images; here it draws the same normal samples with the case's
channel count (`synth_input` below, which the tests use too). Everything else is make_golden's recipe: fp64 eval
and train-mode forward + backward of the reference, checked against the oracle on the same weights.
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

_TINY = dict(dim=32, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])
_TINY_AR = dict(resolution=[240, 336], window_size=[7, 7, 5, 6], ct_size=2, dim=16, in_dim=16, depths=[1, 1, 2, 1],
                num_heads=[1, 2, 4, 8])
CASES = {
    # name: (reference entrypoint, override kwargs, oracle cfg, (eval batch, train batch))
    "tiny_c4": ("faster_vit_0_224", dict(_TINY, in_chans=4), dict(
        _TINY, window_size=[7, 7, 7, 7], ct_size=2, mlp_ratio=4, resolution=224, hat=[False, False, True, False],
        do_propagation=False), (2, 3)),
    "tiny_ar_c1": ("faster_vit_0_any_res", dict(_TINY_AR, in_chans=1), dict(
        _TINY_AR, mlp_ratio=4, hat=[False, False, True, False], do_propagation=False, any_res=True), (2, 2)),
}


def synth_input(batch: int, hw, seed: int, cin: int, dtype=torch.float32) -> torch.Tensor:
    """oracle.synth_input with `cin` channels (cin = 3 gives exactly oracle.synth_input's image)"""
    g = torch.Generator().manual_seed(seed)
    hw = (hw, hw) if isinstance(hw, int) else tuple(hw)
    return torch.randn((batch, cin) + hw, generator=g, dtype=torch.float64).to(dtype)


if __name__ == "__main__":
    import oracle.make_golden as MG
    from oracle import fastervit_oracle as O
    torch.set_num_threads(8)
    for case in sys.argv[1:] or list(CASES):
        entry, kwargs, cfg, batches = CASES[case]
        MG.CASES[case] = (entry, kwargs, cfg)
        MG.batch_for = lambda c, b=batches: b
        O.synth_input = lambda batch, hw, seed, dtype=torch.float32, c=kwargs["in_chans"]: synth_input(
            batch, hw, seed, c, dtype)
        MG.run_case(case)
