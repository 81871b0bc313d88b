"""CPU tests: the oracle against golden vectors of reduced models built with in_chans = 4 and 1 by the unmodified
reference (fp64; tests/make_golden_in_chans.py): eval logits and level activations, train-mode loss, logits and
gradient samples. This pins the oracle, which the GPU in_chans tests compare against, at the channel counts the stem
kernels now take."""
import sys
from pathlib import Path

import pytest
import torch

from oracle import fastervit_oracle as O

sys.path.insert(0, str(Path(__file__).resolve().parent))   # tests/make_golden_in_chans.py
from make_golden_in_chans import synth_input  # noqa: E402

GOLDEN = Path(__file__).parent / "golden"
CASES = ["tiny_c4", "tiny_ar_c1"]


def _load(case):
    return torch.load(GOLDEN / f"{case}.pt", weights_only=False)


def _state_dict(g, dtype):
    sd = {}
    for k, shape, dt in g["state_keys"]:
        sd[k] = torch.zeros(shape, dtype=dtype if dt.startswith("float") else getattr(torch, dt))
    for k in list(sd):
        if k.endswith("relative_coords_table"):
            sd[k] = O.rel_coords_table((sd[k].shape[1] + 1) // 2, dtype)
        elif k.endswith("relative_position_index"):
            sd[k] = O.rel_position_index(int(round(sd[k].shape[0] ** 0.5)))
    return O.synth_fill_(sd, g["seeds"]["w"])


def _sample(t, n=512):
    f = t.detach().flatten()
    return f[::max(1, (f.numel() + n - 1) // n)].float()


@pytest.mark.parametrize("case", CASES)
def test_golden_was_made_with_in_chans(case):
    g = _load(case)
    cin = g["kwargs"]["in_chans"]
    assert cin != 3
    shapes = {k: s for k, s, _ in g["state_keys"]}
    assert shapes["patch_embed.conv_down.0.weight"] == (g["cfg"]["in_dim"], cin, 3, 3)
    assert g["train"]["grads"]["patch_embed.conv_down.0.weight"]["shape"] == (g["cfg"]["in_dim"], cin, 3, 3)


@pytest.mark.parametrize("case", CASES)
def test_oracle_eval_matches_reference_fp64(case):
    g = _load(case)
    sd = _state_dict(g, torch.float64)
    x = synth_input(g["eval"]["batch"], g["cfg"]["resolution"], g["seeds"]["x"], g["kwargs"]["in_chans"], torch.float64)
    cap = {}
    with torch.no_grad():
        logits = O.forward(sd, g["cfg"], x, capture=cap)
    ref = g["eval"]["logits"]
    assert logits.shape == ref.shape
    assert ((logits - ref).abs().max() / ref.abs().max()).item() < 1e-9
    want = g["eval"]["acts"]["patch_embed"]
    assert tuple(cap["patch_embed"].shape) == tuple(want["shape"])
    assert (_sample(cap["patch_embed"]) - want["sample"]).abs().max() / want["amax"] < 1e-5
    for i in range(4):
        got = cap[f"levels.{i}.down"] if i < 3 else cap[f"levels.{i}.out"]
        want = g["eval"]["acts"][f"levels.{i}"]
        assert tuple(got.shape) == tuple(want["shape"])
        assert (_sample(got) - want["sample"]).abs().max() / want["amax"] < 1e-5, i


@pytest.mark.parametrize("case", CASES)
def test_oracle_train_grads_match_reference(case):
    g = _load(case)
    sd = _state_dict(g, torch.float64)
    tr = g["train"]
    x = synth_input(tr["batch"], g["cfg"]["resolution"], g["seeds"]["x"] + 100, g["kwargs"]["in_chans"], torch.float64)
    loss, logits, grads = O.loss_and_grads(sd, g["cfg"], x, tr["target"], training=True)
    assert abs(loss.item() - tr["loss"]) < 1e-9 * max(1.0, abs(tr["loss"]))
    assert ((logits - tr["logits"]).abs().max() / tr["logits"].abs().max()).item() < 1e-9
    floor = tr["grad_floor"]
    assert set(grads) == set(tr["grads"])
    for k, want in tr["grads"].items():
        got = grads[k]
        assert tuple(got.shape) == tuple(want["shape"])
        assert abs(got.norm().item() - want["l2"]) <= 1e-6 * max(want["l2"], floor), k
        assert (_sample(got) - want["sample"]).abs().max().item() <= 2e-6 * max(want["amax"], floor), k
