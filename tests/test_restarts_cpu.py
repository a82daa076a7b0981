"""CPU tests of k-means restarts (kmeans_cuda(..., n_init=, inertia=); include/kmcuda_b200.h
kmcuda_b200_kmeans_restarts, DESIGN.md §4n): the argument checks of both Python surfaces and of the C entry point, which
all run before any device is touched, and the NumPy model of the seed schedule and of the pick."""
import ctypes
import importlib.util
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import restarts_model as M  # noqa: E402


def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_check_n_init_and_inertia(which):
    f = _surfaces()[which].kmeans_cuda
    X = np.zeros((10, 4), np.float32)
    for bad in ("2", 2.0, True, None):
        with pytest.raises(TypeError, match="n_init"):
            f(X, 2, n_init=bad)
    for bad in (0, -1, 1 << 32):
        with pytest.raises(ValueError, match="n_init"):
            f(X, 2, n_init=bad)
    for bad in (1, 0, "yes", None):
        with pytest.raises(TypeError, match="inertia"):
            f(X, 2, inertia=bad)
    with pytest.raises(ValueError, match="n_init"):              # imported centroids: every restart is the same run
        f(X, 2, init=np.zeros((2, 4), np.float32), n_init=2)
    with pytest.raises(ValueError, match="batch_size"):
        f(X, 2, batch_size=4, n_init=2)
    with pytest.raises(ValueError, match="batch_size"):
        f(X, 2, batch_size=4, inertia=True)


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_accept_valid_restart_arguments(which):
    """valid arguments get past the checks: without a GPU the call ends at the device lookup"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    f = _surfaces()[which].kmeans_cuda
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    for kw in ({"n_init": 3}, {"n_init": np.uint32(2), "inertia": True}, {"inertia": np.bool_(True)},
               {"n_init": 1, "init": np.zeros((2, 4), np.float32), "inertia": True}):
        with pytest.raises(ValueError, match="No such CUDA device"):
            f(X, 2, **kw)


def _c_call(n_init, init, inertia=True):
    km, _ = _surfaces()
    X = np.random.default_rng(5).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    e = ctypes.c_double(0)
    return km._lib.kmcuda_b200_kmeans_restarts(
        init, None, 0.01, 0.1, 0, 100, 8, 5, 1, 1, -1, 0, 0, X.ctypes.data, None, 0, n_init, C.ctypes.data,
        A.ctypes.data, None, ctypes.byref(e) if inertia else None)


def test_c_entry_rejects_zero_restarts_and_repeated_imports():
    km, _ = _surfaces()
    assert _c_call(0, km.INIT_PLUSPLUS) == km.INVALID_ARGUMENTS
    assert _c_call(0, km.INIT_PLUSPLUS, inertia=False) == km.INVALID_ARGUMENTS
    assert _c_call(2, km.INIT_IMPORT) == km.INVALID_ARGUMENTS
    assert _c_call(2 ** 32 - 1, km.INIT_IMPORT) == km.INVALID_ARGUMENTS


def test_seed_schedule():
    s = M.seeds(7, 4)
    assert s.dtype == np.uint32 and s[0] == 7
    assert [int(v) for v in s] == [(7 + r * 0x9E3779B9) % 2 ** 32 for r in range(4)]
    w = M.seeds(0xFFFFFFF0, 3)                                   # wraps around 2^32
    assert int(w[1]) == (0xFFFFFFF0 + 0x9E3779B9) - 2 ** 32
    assert int(w[2]) == (0xFFFFFFF0 + 2 * 0x9E3779B9) % 2 ** 32
    assert len(set(int(v) for v in M.seeds(12345, 64))) == 64   # no repeats over many restarts


def test_selection_rule():
    nan = math.nan
    assert M.select([3.0]) == 0
    assert M.select([3.0, 2.0, 1.0]) == 2
    assert M.select([2.0, 1.0, 1.0]) == 1                       # ties keep the earlier restart
    assert M.select([1.0, 1.0]) == 0
    assert M.select([2.0, nan, 1.5]) == 2                       # NaN never wins
    assert M.select([nan, 1.0, 0.5]) == 0                       # ... and restart 0 is the first best, NaN or not
    assert M.select([1.0, math.inf, nan]) == 0


def test_inertia_model_rules():
    X = np.array([[0.0, 0], [1, 0], [3, 4], [np.nan, 0], [2, 0]])
    C = np.array([[0.0, 0], [2, 0]])
    a = np.array([0, 0, 0, 0, 2])                               # row 4 has no centroid, row 3 is NaN
    assert M.inertia(X, C, a) == 0 + 1 + 25
    assert M.inertia(X, C, a, w=[1, 2, 0, 1, 1]) == 2
    U = np.array([[1.0, 0], [0, 1]])
    assert abs(M.inertia(U, np.array([[1.0, 0]]), [0, 0], metric=1) - (math.pi / 2) ** 2) < 1e-12
