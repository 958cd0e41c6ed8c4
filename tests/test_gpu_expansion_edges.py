"""-m gpu: k_expand_fwd / k_expand_bwd on the edge cases of tests/expansion_cases.py -- trained-like parameters, every
quaternion branch, slivers, mesh scales 1e-3 / 1e3, a 2003-face fan (2003 atomics into one vertex), K up to 40 (direct
kernel), the animated path, zero-area faces -- against float64 autograd of oracle/expansion.py, per element.  Each case runs
the kernels its K selects: the forward staged through shared memory up to the 48 KB limit, direct beyond it."""
import ctypes as C

import numpy as np
import pytest
import torch

import expansion_cases as ec
from gms_b200 import _lib

pytestmark = pytest.mark.gpu

CASES = ec.build_cases()


def _run(case):
    stream = torch.cuda.current_stream().cuda_stream

    def put(arr):
        t = torch.from_numpy(arr).cuda()
        return t, t.data_ptr()

    def call(fn, *args):
        _lib.check(fn(*[C.byref(x) for x in args], stream), fn.__name__)

    L = _lib.lib()
    return ec.run_abi(case, put, lambda t: t.cpu().numpy(), lambda a: call(L.gms_expand_forward, a),
                      lambda a, g: call(L.gms_expand_backward, a, g))


@pytest.fixture(scope="module")
def refs():
    return {c.name: ec.Reference(c) for c in CASES}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_expansion_kernels_edge_case_vs_float64(refs, case):
    ec.check_case(refs[case.name], _run(case), ec.TOL, f"gpu {case.name}")


def test_expansion_kernels_zero_area_faces():
    case = ec.degenerate_case()
    ec.check_degenerate(ec.Reference(case), _run(case), ec.TOL_DEGENERATE, "gpu degenerate", frame_outputs=False)
