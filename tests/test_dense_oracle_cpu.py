"""The fp64 reference of the dense-prediction tests (tests/_dense_oracle.py) against the oracle's pinned forward
(oracle/fastervit_oracle.py, itself checked against the reference's golden outputs): same level outputs, same
`norm` map and the same logits through the head, in train and eval mode, with and without stochastic-depth masks,
with and without the ConvBlock layer scale."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/_dense_oracle.py
import _dense_oracle as DO  # noqa: E402


@pytest.mark.parametrize("case", ["tiny_a", "tiny_b", "tiny_ar", "tiny_21k224"])
@pytest.mark.parametrize("training", [True, False])
def test_dense_forward_matches_oracle_forward(case, training):
    import fastervit_b200 as F
    from oracle import fastervit_oracle as O
    from oracle.configs import CASES, cfg_of
    entry, kw, _ = CASES[case]
    cfg = cfg_of(case)
    model = F.create_model(entry, drop_path_rate=0.0, **kw)
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    O.synth_fill_(sd, 77)
    if case == "tiny_b":   # a ConvBlock layer scale (layer_scale_conv) in one block: the gamma branch of both forwards
        sd["levels.1.blocks.0.gamma"] = torch.rand(sd["levels.1.blocks.0.conv2.bias"].shape, dtype=torch.float64) + 0.5
    x = O.synth_input(2, cfg["resolution"], 5, torch.float64)
    masks = None
    if training:
        cap0 = {}
        O.forward(sd, cfg, x, training=True, capture=cap0)
        n_win = cap0["levels.2.blocks.1"].shape[0]   # one draw per window at the level-2 window sites
        g = torch.Generator().manual_seed(3)
        masks = {"levels.0.blocks.0": torch.tensor([0.0, 2.0], dtype=torch.float64),
                 "levels.2.blocks.1.attn": torch.rand(n_win, generator=g).double() + 0.5}
    cap = {}
    stats_ref, stats = {}, {}
    logits = O.forward(sd, cfg, x, training=training, capture=cap, bn_stats=stats_ref, drop_masks=masks)
    out = DO.dense_forward(sd, cfg, x, final="norm", training=training, bn_stats=stats, drop_masks=masks)
    for i in range(4):
        assert torch.equal(out["levels"][i], cap[f"levels.{i}.out"]), i
    assert torch.equal(out["norm"], cap["norm"])
    assert torch.equal(torch.nn.functional.linear(out["pooled"], sd["head.weight"], sd["head.bias"]), logits)
    assert stats.keys() == stats_ref.keys()
    for k in stats:
        assert all(torch.equal(a, b) for a, b in zip(stats[k], stats_ref[k])), k
