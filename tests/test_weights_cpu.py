"""CPU tests of the sample_weight argument of kmeans_cuda: both Python surfaces (the ctypes module kmcuda_b200 and the
libKMCUDA extension module) reject a malformed sample_weight before any device call."""
import importlib.util

import numpy as np
import pytest


def _modules():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return [km, mod]


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_sample_weight_errors_are_raised_before_the_device(which):
    m = _modules()[which]
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    with pytest.raises(ValueError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=np.ones(99, np.float32))          # wrong length
    with pytest.raises(ValueError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=np.ones((100, 1), np.float32))    # 2-D
    with pytest.raises(ValueError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=np.ones((10, 10), np.float32))    # 2-D with N elements
    with pytest.raises(ValueError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=1.0)                              # a scalar is 0-D
    with pytest.raises(TypeError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=["a"] * 100)                      # non-numeric
    with pytest.raises(TypeError, match="sample_weight"):
        m.kmeans_cuda(X, 5, sample_weight=np.array([object()] * 100))
    with pytest.raises(TypeError, match="sample_weight"):                   # device-pointer samples: an int pointer
        m.kmeans_cuda((12345, 0, (100, 4)), 5, sample_weight=np.ones(100, np.float32))


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_sample_weight_is_the_last_keyword(which):
    m = _modules()[which]
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    with pytest.raises(ValueError, match="sample_weight"):   # positional: after verbosity
        m.kmeans_cuda(X, 5, 0.01, "k-means++", 0.1, "L2", False, 3, 0, 0, np.ones(7, np.float32))


def test_weighted_entry_point_rejects_bad_arguments_like_kmeans_cuda():
    """the C entry point validates the plain arguments first, with the same codes as kmeans_cuda"""
    import kmcuda_b200 as km
    X = np.zeros((100, 4), np.float32)
    W = np.ones(100, np.float32)
    C = np.zeros((5, 4), np.float32)
    A = np.zeros(100, np.uint32)
    f = km._lib.kmcuda_b200_kmeans_weighted
    assert f(1, None, 0.01, 0.1, 0, 100, 4, 1, 0, 1, -1, 0, 0, X.ctypes.data, W.ctypes.data, C.ctypes.data,
             A.ctypes.data, None) == km.INVALID_ARGUMENTS                                   # clusters < 2
    assert f(1, None, 0.01, 0.1, 0, 3, 4, 5, 0, 1, -1, 0, 0, X.ctypes.data, W.ctypes.data, C.ctypes.data,
             A.ctypes.data, None) == km.INVALID_ARGUMENTS                                   # N < K
    assert f(1, None, 5.0, 0.1, 0, 100, 4, 5, 0, 1, -1, 0, 0, X.ctypes.data, W.ctypes.data, C.ctypes.data,
             A.ctypes.data, None) == km.INVALID_ARGUMENTS                                   # tolerance > 1
