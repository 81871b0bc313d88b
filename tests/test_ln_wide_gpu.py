"""The LayerNorm kernels at the widths of FasterViT-5 / -6 level 3 (2560 channels): the existing kernel tests run again
at widths past the bounds they had before. fvit_ln_fwd's widest instantiation, ln_fwd_kernel<32, 20>, takes
2048 < C <= 2560; the vectorised backward's ln_bwd_dx_kernel<10, false> takes 1792 < C <= 2560 with C % 8 == 0, and
C = 2564 (a multiple of 4, not of 8) stays on the generic backward kernels. Bars are those of the tests reused."""
import pytest
import torch

import test_data_only_backward_gpu as data_only
import test_glue_kernels_gpu as glue
import test_train_ops_gpu as train_ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C", [2052, 2560])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_ln_fwd_wide(C, eps):
    glue.test_ln_fwd_maps_posadd_writeback(C, eps)


@pytest.mark.parametrize("rows,C", [(98, 1800), (53, 2056), (245, 2560), (37, 2564)])
@pytest.mark.parametrize("mapped", [False, True])
def test_ln_bwd_wide(rows, C, mapped):
    train_ops.test_ln_bwd_matches_autograd(rows, C, mapped)


@pytest.mark.parametrize("C", [1800, 2056, 2560, 2564])
@pytest.mark.parametrize("routed", [False, True])
def test_ln_dgrad_wide(C, routed):
    """bitwise equal to the dx of fvit_ln_bwd on the vectorised path (C % 8 == 0), to rounding at 2564"""
    data_only.test_ln_dgrad_equals_the_dx_of_ln_bwd(C, routed)


def test_ln_fwd_rejects_rows_past_2560():
    from fastervit_b200 import lib as L
    C, rows = 2564, 4
    x = torch.randn(rows, C, device="cuda")
    gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    out = torch.empty(rows, C, device="cuda", dtype=torch.half)
    with pytest.raises(L.FvitError, match="C=2564"):
        L.call("fvit_ln_fwd", x.data_ptr(), C, None, rows, C, None, 1, 0, None, 0, gamma.data_ptr(), beta.data_ptr(),
               1e-6, out.data_ptr(), C, None, None, None, None, 0)
