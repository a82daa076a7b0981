"""CPU tests of scikit-learn's stopping rule (kmeans_cuda(..., tol=, max_iter=, n_iter=True); include/kmcuda_b200.h
kmcuda_b200_kmeans_center_shift, DESIGN.md §4p): the model against scikit-learn's KMeans, and the argument checks of
both Python surfaces and of the C entry."""
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import center_shift_model as M  # noqa: E402

sklearn = pytest.importorskip("sklearn")
from sklearn.cluster import KMeans  # noqa: E402
from sklearn.cluster._kmeans import _tolerance  # noqa: E402


def _blobs(n, d, k, seed=0, spread=1.0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)) * 3
    return (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)


def _start(X, k, seed=1):
    return X[np.random.default_rng(seed).choice(len(X), k, replace=False)].copy()


def test_tolerance_is_scikit_learns():
    X = _blobs(3000, 7, 5)
    for tol in (0.0, 1e-4, 0.3):
        assert M.tolerance_abs(X, tol) == pytest.approx(_tolerance(X.astype(np.float64), tol), rel=1e-12, abs=0)


def test_shift_total_skips_non_finite_centroids():
    a = np.zeros((3, 2), np.float32)
    b = np.array([[1, 0], [np.nan, 0], [0, np.inf]], np.float32)
    assert M.shift_total(a, b) == 1.0
    assert M.shift_total(b, b) == 0.0


CASES = {
    # name: (tol, max_iter, weights, relocate, expected reason)
    "equal_labels": (0.0, 300, False, False, "equal labels"),
    "tolerance": (1e-3, 300, False, False, "tolerance"),
    "max_iter": (0.0, 2, False, False, "max_iter"),
    "weighted": (1e-4, 300, True, False, None),
    "relocate": (1e-4, 300, False, True, None),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_model_matches_scikit_learn(case):
    tol, max_iter, weighted, reloc, reason = CASES[case]
    X = _blobs(4000, 6, 8, seed=3, spread=1.5)
    k = 8
    C0 = _start(X, k, seed=4)
    if reloc:   # a duplicated start row: the second copy wins no row and is relocated after the first pass
        C0[1] = C0[0]
    w = np.random.default_rng(5).uniform(0.5, 2, len(X)).astype(np.float32) if weighted else None
    m = M.run(X, C0, M.argmin64, tol, max_iter=max_iter, w=w, relocate_empty=reloc)
    if reason:
        assert m["reason"] == reason
    km = KMeans(k, init=C0.astype(np.float64), n_init=1, algorithm="lloyd", tol=tol, max_iter=max_iter).fit(
        X.astype(np.float64), sample_weight=None if w is None else w.astype(np.float64))
    assert m["n_iter"] == km.n_iter_
    assert np.array_equal(m["labels"], km.labels_)
    np.testing.assert_allclose(m["C"], km.cluster_centers_, rtol=1e-5, atol=1e-5)


# --------------------------------------------------------------------------------------------- argument checks
def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_check_tol(which):
    f = _surfaces()[which].kmeans_cuda
    X = np.zeros((10, 4), np.float32)
    for bad in ("0.1", True, np.bool_(False), [0.1], 1j):
        with pytest.raises(TypeError, match="tol"):
            f(X, 2, tol=bad)
    for bad in (-1e-4, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="tol"):
            f(X, 2, tol=bad)
    with pytest.raises(ValueError, match="tol"):
        f(X, 2, tol=1e-4, batch_size=4)
    with pytest.raises(ValueError, match="tol"):
        f(X, 2, init="random", tol=1e-4, bisecting="biggest_inertia")
    for bad in (1, "yes", None):
        with pytest.raises(TypeError, match="n_iter"):
            f(X, 2, tol=1e-4, n_iter=bad)
    with pytest.raises(ValueError, match="n_iter"):
        f(X, 2, n_iter=True)
    with pytest.raises(ValueError, match="max_iter"):
        f(X, 2, max_iter=5)
    with pytest.raises(ValueError, match="max_iter"):
        f(X, 2, tol=1e-4, max_iter=-1)


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_accept_valid_tol_arguments(which):
    """valid arguments get past the checks: without a GPU the call ends at the device lookup"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    f = _surfaces()[which].kmeans_cuda
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    w = np.ones(100, np.float32)
    for kw in ({"tol": 0}, {"tol": 1e-4, "max_iter": 300, "n_iter": True}, {"tol": np.float32(0.5), "n_init": 3},
               {"tol": np.int64(1), "sample_weight": w, "relocate_empty_clusters": True, "inertia": True},
               {"tol": 1e-4, "tolerance": 100.0, "average_distance": True, "n_iter": np.bool_(True)}):
        with pytest.raises(ValueError, match="No such CUDA device"):
            f(X, 2, **kw)


def _c_call(tol=1e-4, **over):
    km, _ = _surfaces()
    a = dict(init=km.INIT_RANDOM, metric=0, device=1, n_init=1, max_iter=0, yy=0.1)
    a.update(over)
    X = np.random.default_rng(5).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    e = ctypes.c_double(0)
    it = ctypes.c_uint32(0)
    return km._lib.kmcuda_b200_kmeans_center_shift(
        a["init"], None, tol, a["yy"], a["metric"], 100, 8, 5, 1, a["device"], -1, 0, 0, X.ctypes.data, None, 0,
        a["n_init"], a["max_iter"], C.ctypes.data, A.ctypes.data, None, ctypes.byref(e), ctypes.byref(it))


def test_c_entry_checks_tol():
    km, _ = _surfaces()
    for bad in (-1e-4, float("nan"), float("inf")):
        assert _c_call(tol=bad) == km.INVALID_ARGUMENTS
    assert _c_call(n_init=0) == km.INVALID_ARGUMENTS
    assert _c_call(n_init=2, init=km.INIT_IMPORT) == km.INVALID_ARGUMENTS
    assert _c_call(yy=0.7) == km.INVALID_ARGUMENTS
    import torch
    if not torch.cuda.is_available():
        for tol in (0.0, 1e-4, 1e30):
            assert _c_call(tol=tol) == km.NO_SUCH_DEVICE
