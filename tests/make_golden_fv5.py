"""Generate the full-size FasterViT-5 golden fixture (tests/golden/fv5.pt) with oracle/make_golden.py.

    FASTERVIT_REFERENCE=<path to the reference checkout> python tests/make_golden_fv5.py

faster_vit_5_224 at the entrypoint's defaults (dim 320: level 3 is 2560 channels wide, every transformer head 80
wide), built by the unmodified reference. The recipe is make_golden's fv4 case: fp64 eval at batch 1, a train-mode
forward + backward at batch 2, both checked against the oracle on the same weights, and every second point of each
gradient sample kept so the fixture stays under 1 MB. It takes about 40 GiB of host memory.
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

CASE = ("faster_vit_5_224", {}, dict(
    dim=320, in_dim=64, depths=[3, 3, 12, 5], num_heads=[4, 8, 16, 32], window_size=[7, 7, 7, 7],
    ct_size=2, mlp_ratio=4, resolution=224, hat=[False, False, True, False], do_propagation=True))


if __name__ == "__main__":
    import oracle.make_golden as MG
    torch.set_num_threads(8)
    MG.CASES["fv5"] = CASE
    MG.batch_for = lambda case: (1, 2)
    MG.GRAD_SAMPLE_STEP["fv5"] = 2
    MG.run_case("fv5")
