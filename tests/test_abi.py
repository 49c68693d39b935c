"""CPU-only checks of the C-ABI boundary: the CUDA library builds for sm_90a, loads without a GPU and
exports every symbol include/trajopt_b200.h declares; the product fails loudly (never falls back) when no
device is present."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import __graft_entry__ as entry
from trajopt_b200 import capi, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    entry.build()
    return C.CDLL(capi.library_path())


def test_header_symbols_exported(lib):
    header = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    declared = set(re.findall(r"\b(tb200_[a-z_]+)\s*\(", header))
    assert declared == set(capi.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), f"{name} missing from libtrajopt_b200.so"


def test_struct_sizes_match_header(lib):
    """ctypes mirrors must have the C layout (spot check through the defaults entry points)."""
    s = capi.SqpParams()
    lib.tb200_default_sqp_params(C.byref(s))
    assert (s.improve_ratio_threshold, s.max_iter, s.trust_box_size, s.inflate_constraints_individually) == (0.25, 50, 0.1, 1)
    q = capi.QpSettings()
    lib.tb200_default_qp_settings(C.byref(q))
    assert (q.eps_abs, q.eps_rel, q.max_iter, q.polishing, q.warm_starting) == (1e-4, 1e-6, 8192, 1, 1)


def test_no_cpu_fallback_without_device(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    d = problems.config0()
    h = C.c_void_p()
    lib.tb200_problem_create.argtypes = [C.POINTER(capi.ProblemDescC), C.c_int, C.POINTER(C.c_void_p)]
    rc = lib.tb200_problem_create(C.byref(d.c), 0, C.byref(h))
    lib.tb200_last_error.restype = C.c_char_p
    assert rc == 4 and b"no CPU fallback" in lib.tb200_last_error()
