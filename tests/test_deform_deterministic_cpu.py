"""The deterministic backward of multi-scale deformable attention without a GPU: fvit_msda_bwd_deterministic is
exported and bound with the argument list of its declaration in include/fvit.h, the ABI version is unchanged, the
scratch is sized from the shapes alone, and the entry point rejects bad sizes and null pointers before it touches a
device."""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

import pytest

from fastervit_b200 import deform, lib

HEADER = (Path(__file__).resolve().parent.parent / "include" / "fvit.h").read_text()
NAME = "fvit_msda_bwd_deterministic"


def _declared_argtypes(name):
    """ctypes types of a declaration in fvit.h: pointers -> c_void_p, int32_t -> c_int32, int64_t -> c_int64"""
    params = re.search(rf"\bint {name}\(([^)]*)\);", HEADER).group(1)
    out = []
    for p in params.split(","):
        p = " ".join(p.split())
        out.append(C.c_void_p if "*" in p else {"int32_t": C.c_int32, "int64_t": C.c_int64}[p.split()[0]])
    return out


def test_exported_and_bound_as_declared():
    cdll = lib.load()
    fn = getattr(cdll, NAME)
    assert fn.argtypes == lib._OP_SIGS[NAME] == _declared_argtypes(NAME)
    assert fn.restype == C.c_int
    # the same leading arguments as fvit_msda_bwd, then scratch and workspace before the stream
    assert lib._OP_SIGS[NAME] == lib._OP_SIGS["fvit_msda_bwd"][:-1] + [C.c_void_p] * 3


def test_abi_version_unchanged():
    assert lib.load().fvit_abi_version() == 1


def test_workspace_size_matches_header():
    assert int(re.search(r"#define FVIT_MSDA_DET_WORKSPACE (\d+)", HEADER).group(1)) == lib.MSDA_DET_WORKSPACE


@pytest.mark.parametrize("shape", [(2, 22223, 8, 32), (2, 89023, 8, 32), (1, 25512, 8, 32), (3, 1, 1, 1)])
def test_scratch_sized_from_shapes(shape):
    N, S, M, D = shape
    n_scratch, n_workspace = deform.deterministic_scratch_sizes(N, S, M, D)
    assert n_scratch == N * S * M * D and n_workspace == lib.MSDA_DET_WORKSPACE
    # DINO's 5-scale encoder at 800 x 1333, batch 2: twice grad_value's bytes
    if shape == (2, 89023, 8, 32):
        assert n_scratch * 8 == 364_638_208


def _call(N=1, S=4, M=1, D=4, Lq=2, L=1, P=1, ptr=None):
    cdll = lib.load()
    rc = getattr(cdll, NAME)(*[ptr] * 6, N, S, M, D, Lq, L, P, *[ptr] * 5, None)
    return rc, cdll.fvit_last_error().decode()


def test_rejects_bad_sizes_and_null_pointers_on_the_host():
    rc, msg = _call(L=17)
    assert rc != 0 and "at most 16" in msg and NAME in msg
    rc, msg = _call(D=0)
    assert rc != 0 and "bad sizes" in msg
    rc, msg = _call()
    assert rc != 0 and "null pointer" in msg
    assert _call(N=0)[0] == 0          # nothing to do and nothing to write: no device needed
