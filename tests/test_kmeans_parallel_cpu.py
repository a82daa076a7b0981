"""CPU tests of the k-means|| seeding: the draw rule's NumPy model (which the GPU tests use as the reference), the model's
row distances against the oracle, and the init="k-means||" intake of both Python surfaces."""
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import kmeans_parallel_model as M  # noqa: E402
from oracle import oracle as O  # noqa: E402


def test_hash_matches_the_scalar_definition():
    rows = np.array([0, 1, 2, 12345, 2 ** 32 - 1], np.uint64)
    key = M.mix((7 << 8) | 3)
    want = [(M.mix(key ^ int(i)) >> 11) * 2.0 ** -53 for i in rows]
    assert np.array_equal(M.uniform(7, 3, rows), np.array(want))
    u = M.uniform(1, 1, np.arange(200000))
    assert 0 <= u.min() and u.max() < 1 and abs(u.mean() - 0.5) < 0.005


def test_expected_draws_per_round_are_at_most_ell():
    rng = np.random.default_rng(0)
    for w in (None, rng.integers(0, 5, 50000).astype(np.float32)):
        d = rng.lognormal(0, 2, 50000).astype(np.float32)
        ell = 2.0 * 200
        m = M.mass(d, w)
        expected = np.minimum(1.0, ell * m / m.sum()).sum()
        assert expected <= ell
        drawn = sum(M.draws(d, w, 3, r, ell, m.sum()).sum() for r in range(1, 6)) / 5
        assert drawn <= ell * 1.2


def test_zero_weight_and_zero_distance_rows_are_never_drawn():
    rng = np.random.default_rng(1)
    d = rng.random(100000).astype(np.float32)
    w = rng.random(100000).astype(np.float32)
    d[::3] = 0
    w[1::3] = 0
    d[5] = np.nan
    m = M.mass(d, w)
    for r in range(1, 33):
        f = M.draws(d, w, 9, r, 1e9, m.sum())   # an l this large draws every row with mass
        assert not f[::3].any() and not f[1::3].any() and not f[5]
        assert f[2::3][:-1].all() or m[2::3].min() == 0


def test_draws_do_not_depend_on_the_shard_split():
    rng = np.random.default_rng(2)
    d = rng.random(30000).astype(np.float32)
    phi = M.mass(d).sum()
    whole = M.draws(d, None, 11, 2, 400.0, phi)
    for cuts in ([10000], [512, 20000], [7, 8, 29999]):
        parts = np.split(np.arange(30000), cuts)
        split = np.concatenate([M.draws(d[p], None, 11, 2, 400.0, phi, offset=int(p[0])) for p in parts])
        assert np.array_equal(whole, split)


@pytest.mark.parametrize("metric", [0, 1])
def test_row_distances_agree_with_average_distance(metric):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((3000, 30)).astype(np.float32)
    if metric:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    C = X[:17].copy()
    a = O.assign_lloyd(X, C, metric=metric)[0]
    d = M.row_distances(X, C, a, metric)
    assert d[0] == 0 or metric
    avg = O.average_distance(X, C, a, metric=metric)
    assert np.float32(np.float64(d.astype(np.float64).sum()) / len(X)) == np.float32(avg)


def test_model_without_draws_falls_back_to_the_fill_walk():
    X = np.repeat(np.eye(4, dtype=np.float32), [10000, 1, 1, 1], axis=0)   # one row repeated, three single rows
    rows, log, nearest = M.candidates(X, 20, seed=5, rounds=5)
    assert len(rows) == 4 and len(set(map(tuple, X[rows]))) == 4   # round 1 takes the three, then phi = 0 stops
    assert [rec[:2] for rec in log] == [(1, 3)] and abs(log[0][2] - 6.0) < 1e-6   # three times sqrt(2)^2
    C = M.fill(X, rows, 20, seed=5)
    assert C.shape == (20, 4) and np.array_equal(C[:len(rows)], X[rows])


def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


def test_both_python_surfaces_accept_k_means_parallel():
    import torch
    km, mod = _surfaces()
    assert km.INIT_KMEANS_PARALLEL == 4
    X = np.random.default_rng(4).random((100, 8), dtype=np.float32)
    for f in (km.kmeans_cuda, mod.kmeans_cuda):
        for init in ("k-means||", "kmeans||", ("k-means||", 3), ("kmeans||", 0), ("k-means||", np.int64(32))):
            if not torch.cuda.is_available():
                with pytest.raises(ValueError, match="No such CUDA device"):
                    f(X, 5, init=init)
        for bad in (33, -1, 2.5, "3", True, None):
            with pytest.raises(ValueError):
                f(X, 5, init=("k-means||", bad))


def test_c_abi_rejects_more_than_32_rounds_before_touching_a_device():
    km, _ = _surfaces()
    X = np.random.default_rng(5).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    for fn in (km._lib.kmeans_cuda, km._lib.kmcuda_b200_kmeans_weighted):
        r = ctypes.c_uint32(33)
        args = [4, ctypes.byref(r), 0.01, 0.1, 0, 100, 8, 5, 1, 0, -1, 0, 0, X.ctypes.data]
        if fn is km._lib.kmcuda_b200_kmeans_weighted:
            args.append(None)
        assert fn(*args, C.ctypes.data, A.ctypes.data, None) == km.INVALID_ARGUMENTS
