"""The product's per-face expansion maths (csrc/gms_expand.cuh, compiled for the CPU by tests/hostshim) on the edge cases of
tests/expansion_cases.py -- trained-like parameters, every quaternion branch, slivers, mesh scales 1e-3 / 1e3, a 2003-face
fan, K up to 40, the animated path, zero-area faces -- against float64 autograd of oracle/expansion.py, per element."""
import ctypes as C

import numpy as np
import pytest

import expansion_cases as ec
from hostshim import build_shim

CASES = ec.build_cases()


@pytest.fixture(scope="module")
def shim():
    return C.CDLL(build_shim.build())


def _run(shim, case):
    put = lambda arr: (arr, arr.ctypes.data)
    get = lambda arr: arr
    fwd = lambda a: shim.shim_expand_forward(C.byref(a)) == 0 or pytest.fail("shim_expand_forward")
    bwd = lambda a, g: shim.shim_expand_backward(C.byref(a), C.byref(g)) == 0 or pytest.fail("shim_expand_backward")
    return ec.run_abi(case, put, get, fwd, bwd)


@pytest.fixture(scope="module")
def refs():
    return {c.name: ec.Reference(c) for c in CASES}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_expansion_edge_case_vs_float64(shim, refs, case):
    ec.check_case(refs[case.name], _run(shim, case), ec.TOL, f"cpu {case.name}")


def test_cases_cover_every_quaternion_branch(refs):
    ec.branch_coverage(list(refs.values()))


def test_zero_area_faces_finite_and_match_fp32_oracle(shim):
    case = ec.degenerate_case()
    ec.check_degenerate(ec.Reference(case), _run(shim, case), ec.TOL_DEGENERATE, "cpu degenerate")
