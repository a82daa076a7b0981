"""CPU tests of the init stage of mini-batch k-means (kmeans_cuda(..., batch_size=b, init_size=, n_init=);
include/kmcuda_b200.h kmcuda_b200_kmeans_minibatch_init, DESIGN.md §4q): the model (tests/minibatch_init_model.py)
against scikit-learn's MiniBatchKMeans, and the arguments both Python surfaces and the C entry reject before any device
is touched."""
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import minibatch_init_model as M  # noqa: E402
import minibatch_model as MB  # noqa: E402


def _rows_only(N):
    """an N x 1 array that takes no memory: scikit-learn's size rule reads X.shape only"""
    return np.lib.stride_tricks.as_strided(np.zeros(1, np.float32), shape=(N, 1), strides=(0, 4))


@pytest.mark.parametrize("N,b,K", [(8000000, 65536, 1024), (50000, 1024, 200), (20000, 1024, 50), (1000, 16, 100),
                                   (1000, 16, 400), (1000, 2000, 10), (250, 64, 100), (3000, 1, 2), (5000, 333, 1000)])
def test_auto_size_is_scikit_learns(N, b, K):
    from sklearn.cluster import MiniBatchKMeans
    km = MiniBatchKMeans(n_clusters=K, batch_size=b, tol=0.0)
    km._check_params_vs_input(_rows_only(N))
    assert M.init_size(N, b, K) == km._init_size
    if (N, b, K) == (8000000, 65536, 1024):
        assert km._init_size == 196608


def test_auto_size_branches():
    assert M.init_size(8000000, 65536, 1024) == 3 * 65536    # 3 b
    assert M.init_size(1000, 16, 100) == 300                 # 3 b < K: 3 K
    assert M.init_size(1000, 16, 400) == 1000                # 3 K > N: N
    assert M.init_size(1000, 2000, 10) == 1000               # b is first capped at N, 3 N at N
    assert M.init_size(1000, 16, 10, 5000) == 1000           # an explicit size is capped at N
    assert M.init_size(1000, 16, 10, 123) == 123


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("weighted", [False, True])
def test_validation_inertia_is_scikit_learns(seed, weighted):
    from sklearn.cluster._kmeans import _labels_inertia
    rng = np.random.default_rng(seed)
    N, D, K, m = 3000, 7, 25, 900
    X = rng.standard_normal((N, D))
    C = rng.standard_normal((K, D))
    w = rng.random(N) * 3 if weighted else None
    rows = M.valid_rows(100 + seed, N, m)
    assert len(np.unique(rows)) < m   # drawn with replacement: duplicates count once per entry
    wv = np.ones(m) if w is None else w[rows]
    _, sk = _labels_inertia(X[rows], wv, C)
    got = M.validation_inertia(X, C, rows, w)
    assert abs(got - sk) <= 1e-12 * sk


def test_draws_have_their_own_tags():
    seed, N, m = 12345, 1000003, 500
    a, b, v = M.init_rows(seed, 0, N, m), M.init_rows(seed, 1, N, m), M.valid_rows(seed, N, m)
    for rows in (a, b, v):
        assert rows.min() >= 0 and rows.max() < N
    assert not np.array_equal(a, b) and not np.array_equal(a, v)
    assert not np.array_equal(a, MB.draw(seed, 0, N, m)) and not np.array_equal(v, MB.draw(seed, 0, N, m))
    key = MB.mix((MB.mix(M.TAG_INIT ^ seed) + 1) & MB.M64)
    for j in (0, 1, 499):
        assert b[j] == int((MB.mix(key ^ j) >> 11) * 2.0 ** -53 * N)
    assert len({M.TAG_INIT, M.TAG_VALID, MB.TAG_BATCH, MB.TAG_REASSIGN, 0x677265656479212B}) == 5


def test_pick_is_the_restarts_rule():
    nan = float("nan")
    assert M.select([3.0, 2.0, 2.0]) == 1
    assert M.select([2.0, nan, 1.0]) == 2
    assert M.select([nan, 1.0]) == 0
    assert [int(s) for s in M.seeds(7, 3)] == [(7 + r * 0x9E3779B9) % 2 ** 32 for r in range(3)]


def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_check_init_size(which):
    f = _surfaces()[which].kmeans_cuda
    X = np.zeros((100, 4), np.float32)
    for bad in (True, 2.5, [30], b"auto"):
        with pytest.raises(TypeError, match="init_size"):
            f(X, 10, batch_size=8, init_size=bad)
    for bad in (0, -1, "Auto", "all"):
        with pytest.raises(ValueError, match="init_size"):
            f(X, 10, batch_size=8, init_size=bad)
    with pytest.raises(ValueError, match="init_size"):           # below K
        f(X, 10, batch_size=8, init_size=9)
    with pytest.raises(ValueError, match="init_size"):           # an imported init reads no rows
        f(X, 10, batch_size=8, init=np.zeros((10, 4), np.float32), init_size=50)
    with pytest.raises(ValueError, match="init_size"):           # not without batch_size
        f(X, 10, init_size=50)
    with pytest.raises(ValueError, match="init_size"):           # not with bisecting
        f(X, 10, init="random", bisecting="biggest_inertia", init_size=50)
    with pytest.raises(ValueError, match="batch_size"):          # several inits need an init size
        f(X, 10, batch_size=8, n_init=3)
    with pytest.raises(ValueError, match="batch_size"):          # inertia stays a Lloyd / bisecting output
        f(X, 10, batch_size=8, init_size="auto", inertia=True)


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_accept_valid_init_size_arguments(which):
    """valid arguments get past the checks: without a GPU the call ends at the device lookup"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    f = _surfaces()[which].kmeans_cuda
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    for kw in ({"init_size": "auto"}, {"init_size": 10}, {"init_size": np.int64(10 ** 12), "n_init": 3},
               {"init_size": "auto", "n_init": np.uint32(2), "init": "random"}, {"init_size": None}):
        with pytest.raises(ValueError, match="No such CUDA device"):
            f(X, 10, batch_size=8, **kw)


def _c_call(init_size, n_init=1, init=None, batch_size=8, weights=None):
    km, _ = _surfaces()
    X = np.random.default_rng(5).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    return km._lib.kmcuda_b200_kmeans_minibatch_init(
        km.INIT_RANDOM if init is None else init, None, 0.0, 0, 100, 8, 5, 1, 1, -1, 0, 0, X.ctypes.data,
        None if weights is None else weights.ctypes.data, batch_size, 0, init_size, n_init, C.ctypes.data,
        A.ctypes.data, None)


def test_c_entry_rejects_bad_init_stages():
    km, _ = _surfaces()
    assert _c_call(4) == km.INVALID_ARGUMENTS                              # below K
    assert _c_call(1) == km.INVALID_ARGUMENTS
    assert _c_call(50, init=km.INIT_IMPORT) == km.INVALID_ARGUMENTS        # an imported init
    assert _c_call(km.INIT_SIZE_AUTO, init=km.INIT_IMPORT) == km.INVALID_ARGUMENTS
    assert _c_call(0, n_init=2) == km.INVALID_ARGUMENTS                    # several inits without an init size
    assert _c_call(50, n_init=0) == km.INVALID_ARGUMENTS
    assert _c_call(50, batch_size=0) == km.INVALID_ARGUMENTS               # not without a batch size
    import torch
    if not torch.cuda.is_available():
        for size, n in ((0, 1), (5, 1), (50, 3), (km.INIT_SIZE_AUTO, 2), (10 ** 9, 1)):
            assert _c_call(size, n) == km.NO_SUCH_DEVICE
        assert _c_call(0, init=km.INIT_IMPORT) == km.NO_SUCH_DEVICE       # today's mini-batch call
