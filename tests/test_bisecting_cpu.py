"""CPU tests of bisecting k-means (kmeans_cuda(..., bisecting=...); include/kmcuda_b200.h kmcuda_b200_kmeans_bisecting,
DESIGN.md §4o): the NumPy model against scikit-learn's own BisectingKMeans, the draw keys, the wave schedule, and the
argument checks of both Python surfaces and of the C entry point, which all run before any device is touched."""
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bisecting_model as M  # noqa: E402


def _blobs(n, d, k, seed=0, spread=0.5):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 4
    return (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)


def _sklearn(X, K, inits, strategy, n_init, tol, max_iter, w):
    """scikit-learn's BisectingKMeans, each init taken from `inits` in call order (scikit-learn centres X first)"""
    from sklearn.cluster import BisectingKMeans

    class Pinned(BisectingKMeans):
        def _init_centroids(self, X, *args, **kwargs):
            return inits.pop(0).astype(np.float64) - self._X_mean

    km = Pinned(n_clusters=K, init="random", n_init=n_init, tol=tol, max_iter=max_iter, bisecting_strategy=strategy,
                algorithm="lloyd", random_state=0)
    km.fit(X.astype(np.float64), sample_weight=None if w is None else w.astype(np.float64))
    assert not inits
    return km


CASES = {
    "inertia-1": dict(strategy="biggest_inertia", n_init=1, w=None),
    "inertia-3-w": dict(strategy="biggest_inertia", n_init=3, w="int"),
    "largest-1-w": dict(strategy="largest_cluster", n_init=1, w="int"),
    "largest-3": dict(strategy="largest_cluster", n_init=3, w=None),
    "maxiter2": dict(strategy="biggest_inertia", n_init=1, w=None, max_iter=2),
    "greedy-inertia-1": dict(strategy="biggest_inertia", n_init=1, w=None, init="greedy-k-means++"),
    "greedy-inertia-3-w": dict(strategy="biggest_inertia", n_init=3, w="int", init=("greedy-k-means++", 5)),
    "greedy-largest-1-w": dict(strategy="largest_cluster", n_init=1, w="int", init=("greedy-k-means++", 1)),
    "greedy-largest-3": dict(strategy="largest_cluster", n_init=3, w=None, init="greedy-k-means++"),
}


def _recording(monkeypatch, X, inits):
    """the model's init centres, recorded in call order"""
    real_random, real_greedy = M.random_init, M.greedy_init

    def random_init(rows, wn, seed, lo, hi, r):
        pair = real_random(rows, wn, seed, lo, hi, r)
        inits.append(X[list(pair)].copy())
        return pair

    def greedy_init(Xn, rows, wn, seed, lo, hi, r, L):
        pair = real_greedy(Xn, rows, wn, seed, lo, hi, r, L)
        inits.append(X[list(pair)].copy())
        return pair

    monkeypatch.setattr(M, "random_init", random_init)
    monkeypatch.setattr(M, "greedy_init", greedy_init)


@pytest.mark.parametrize("case", sorted(CASES))
def test_model_matches_sklearn(case, monkeypatch):
    pytest.importorskip("sklearn")
    c = CASES[case]
    X = _blobs(1500, 6, 8, seed=len(case))
    w = None if c["w"] is None else np.random.default_rng(1).integers(1, 4, len(X)).astype(np.float32)
    max_iter = c.get("max_iter", 300)
    tol = 1e-4
    inits = []
    _recording(monkeypatch, X, inits)
    C, labels, lines, inertia, _, _ = M.bisecting(X, 8, 11, c["strategy"], c["n_init"], tol, max_iter, w, waves=False,
                                                  init=c.get("init", "random"))
    km = _sklearn(X, 8, list(inits), c["strategy"], c["n_init"], M.tolerance_abs(X, tol), max_iter, w)
    np.testing.assert_array_equal(labels, km.labels_)
    np.testing.assert_allclose(C, km.cluster_centers_, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(inertia, km.inertia_, rtol=1e-5)
    if case == "maxiter2":
        assert any("stopped on max_iter" in ln for ln in lines)


def test_model_matches_sklearn_through_an_empty_child_relocation(monkeypatch):
    """five distinct rows, duplicated: some inits put both centres on equal rows, so the first E step leaves child 1
    empty and scikit-learn's _relocate_empty_clusters_dense runs, in the model and in scikit-learn alike"""
    pytest.importorskip("sklearn")
    rng = np.random.default_rng(31)
    base = (rng.standard_normal((5, 3)) * 3).astype(np.float32)
    X = base[rng.integers(0, 5, 60)]
    X[:3] += (0.01 * rng.standard_normal((3, 3))).astype(np.float32)
    inits, relocations = [], []
    _recording(monkeypatch, X, inits)
    real = M.two_means

    def two_means(*a):
        run = real(*a)
        relocations.append(run["relocations"])
        return run

    monkeypatch.setattr(M, "two_means", two_means)
    C, labels, _, inertia, _, _ = M.bisecting(X, 4, 31, "biggest_inertia", 1, 1e-4, 300, None, waves=False)
    assert sum(relocations) >= 2
    km = _sklearn(X, 4, list(inits), "biggest_inertia", 1, M.tolerance_abs(X, 1e-4), 300, None)
    np.testing.assert_array_equal(labels, km.labels_)
    np.testing.assert_allclose(C, km.cluster_centers_, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(inertia, km.inertia_, rtol=1e-5, atol=1e-9)


def test_model_relocates_an_empty_child():
    """two distinct points, one duplicated: the first E step leaves child 1 empty and it takes the farthest row"""
    X = np.array([[0, 0], [0, 0], [0, 0], [1, 0], [0, 0]], np.float32)
    rows = np.arange(5)
    run = M.two_means(X, np.ones(5, np.float32), rows, X[[0, 1]], 0.0, 300)
    assert run["cnt"] == [4, 1] and run["W"] == [4.0, 1.0]
    assert (run["C"][1] == [1, 0]).all()


def test_model_marks_a_node_without_two_positive_rows_unsplittable():
    X = _blobs(40, 3, 2)
    w = np.zeros(40, np.float32)
    w[7] = 1
    assert M.bisect(X, w, np.arange(40), 0, 40, 1, 1, 0.0, 10, 0) == (None, [])
    with pytest.raises(ValueError):
        M.bisecting(X, 2, 1, w=w)


def test_waves_change_nothing_but_the_schedule():
    X = _blobs(3000, 5, 9, seed=3)
    a = M.bisecting(X, 9, 5, "biggest_inertia", 2, 1e-4, 300)
    b = M.bisecting(X, 9, 5, "biggest_inertia", 2, 1e-4, 300, waves=False)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    assert a[3] == b[3]
    assert a[5] < b[5]   # fewer waves than sequential bisections


def test_draw_keys_depend_on_the_node_init_stage_and_row_only():
    rows = np.arange(100, 140)
    w = np.ones(40, np.float32)
    k = M.draw_keys(7, 10, 90, 1, 0, rows, w)
    np.testing.assert_array_equal(k, M.draw_keys(7, 10, 90, 1, 0, rows, w))
    np.testing.assert_array_equal(k[5:], M.draw_keys(7, 10, 90, 1, 0, rows[5:], w[5:]))   # not on the row's place
    for other in ((8, 10, 90, 1, 0), (7, 11, 90, 1, 0), (7, 10, 91, 1, 0), (7, 10, 90, 2, 0), (7, 10, 90, 1, 1)):
        assert not np.array_equal(k, M.draw_keys(*other, rows, w))
    np.testing.assert_array_equal(M.draw_keys(7, 10, 90, 1, 0, rows, 2 * w), k / 2)
    assert np.isinf(M.draw_keys(7, 10, 90, 1, 0, rows[:1], [0.0])).all()
    assert M.node_key(7 + (1 << 32), 10, 90, 1, 0) == M.node_key(7, 10, 90, 1, 0)   # the seed is 32 bits


def test_fixed_sum_order():
    v = np.array([1e16, 1.0, -1e16, 1.0] * 1000)
    assert M.fixed_sum(v) == np.cumsum(np.concatenate([[0.0], v[:M.CHUNK]]))[-1] + \
        np.cumsum(np.concatenate([[0.0], v[M.CHUNK:]]))[-1]


def test_wave_schedule_on_hand_made_scores():
    """children scores: node [lo, hi) splits in half, child scores from a table; the waves bisect the top K - #leaves
    uncached leaves and the picks follow (score desc, lo asc)"""
    scores = {(0, 16): (5.0, 3.0), (0, 8): (1.0, 4.0), (8, 16): (2.0, 2.0), (4, 8): (0.5, 0.5),
              (8, 12): (0.1, 0.1), (12, 16): (0.2, 0.2), (0, 4): (0.3, 0.3)}
    calls = []

    def fn(lo, hi):
        calls.append((lo, hi))
        s = scores[(lo, hi)]
        return {"splittable": (lo, hi) != (12, 16), "cnt": [(hi - lo) // 2, (hi - lo) // 2], "score": list(s)}

    leaves, events = M.schedule(5, 16, fn)
    assert sorted(leaves.items()) == [(0, 4), (4, 6), (6, 8), (8, 12), (12, 16)]
    waves = [e[1] for e in events if e[0] == "wave"]
    # round 1: the root; round 2: both children (K - 2 = 3 >= 2); [0, 8) splits; then [4, 8) (score 4) is uncached:
    # the wave takes the top K - 3 = 2 leaves, [4, 8) and the cached [8, 16) is skipped
    assert waves == [[(0, 16)], [(0, 8), (8, 16)], [(4, 8)]]
    splits = [(e[1], e[2]) for e in events if e[0] == "split"]
    assert splits == [(0, 16), (0, 8), (4, 8), (8, 16)]
    assert calls == [(0, 16), (0, 8), (8, 16), (4, 8)]   # every node bisected once
    leaves_seq, events_seq = M.schedule(5, 16, fn, waves=False)
    assert leaves_seq == leaves
    assert [e[:3] for e in events_seq if e[0] == "split"] == [e[:3] for e in events if e[0] == "split"]


def test_wave_schedule_skips_unsplittable_leaves():
    def fn(lo, hi):
        return None if (lo, hi) == (0, 8) else {"splittable": True, "cnt": [(hi - lo) // 2] * 2,
                                                "score": [9.0, 1.0] if hi - lo == 16 else [0.5, 0.5]}

    leaves, events = M.schedule(3, 16, fn)
    assert ("not split", 0, 8) in events
    assert sorted(leaves.items()) == [(0, 8), (8, 12), (12, 16)]
    assert M.schedule(4, 16, lambda lo, hi: None)[0] is None


# --------------------------------------------------------------------------------------------- argument checks
def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_check_bisecting(which):
    f = _surfaces()[which].kmeans_cuda
    X = np.zeros((10, 4), np.float32)
    for bad in (1, True, b"biggest_inertia"):
        with pytest.raises(TypeError, match="bisecting"):
            f(X, 2, init="random", bisecting=bad)
    with pytest.raises(ValueError, match="bisecting"):
        f(X, 2, init="random", bisecting="biggest")
    for kw in ({"batch_size": 4}, {"relocate_empty_clusters": True}):
        with pytest.raises(ValueError, match="bisecting"):
            f(X, 2, init="random", bisecting="largest_cluster", **kw)
    for init in ("k-means++", "afkmc2", "k-means||", ("random", 2), ("k-means++", 2), np.zeros((2, 4), np.float32)):
        with pytest.raises(ValueError, match="random"):
            f(X, 2, init=init, bisecting="biggest_inertia")
    with pytest.raises(ValueError, match="trials"):
        f(X, 2, init=("greedy-k-means++", 33), bisecting="biggest_inertia")
    with pytest.raises(ValueError, match="max_iter"):
        f(X, 2, max_iter=5)
    for bad in ("5", 5.0, None):
        with pytest.raises(TypeError, match="max_iter"):
            f(X, 2, init="random", bisecting="biggest_inertia", max_iter=bad)
    with pytest.raises(ValueError, match="max_iter"):
        f(X, 2, init="random", bisecting="biggest_inertia", max_iter=-1)


@pytest.mark.parametrize("which", [0, 1], ids=["ctypes", "libKMCUDA"])
def test_python_surfaces_accept_valid_bisecting_arguments(which):
    """valid arguments get past the checks: without a GPU the call ends at the device lookup"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    f = _surfaces()[which].kmeans_cuda
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    for kw in ({"bisecting": "biggest_inertia"}, {"bisecting": "largest_cluster", "n_init": 3, "inertia": True},
               {"bisecting": "biggest_inertia", "max_iter": np.uint32(4), "average_distance": True}):
        for init in ("random", "greedy-k-means++", ("greedy-k-means++", 5), ("greedy-kmeans++", 0)):
            with pytest.raises(ValueError, match="No such CUDA device"):
                f(X, 2, init=init, **kw)


def _c_call(**over):
    km, _ = _surfaces()
    a = dict(init=km.INIT_RANDOM, metric=0, device=1, strategy=0, n_init=1, trials=None)
    a.update(over)
    trials = None if a["trials"] is None else ctypes.byref(ctypes.c_uint32(a["trials"]))
    X = np.random.default_rng(5).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    e = ctypes.c_double(0)
    return km._lib.kmcuda_b200_kmeans_bisecting(
        a["init"], trials, 0.01, a["metric"], 100, 8, 5, 1, a["device"], -1, 0, 0, X.ctypes.data, None,
        a["strategy"], a["n_init"], 0, C.ctypes.data, A.ctypes.data, None, ctypes.byref(e))


def test_c_entry_rejects_invalid_bisecting_arguments(monkeypatch):
    km, _ = _surfaces()
    assert _c_call(metric=1) == km.INVALID_ARGUMENTS
    assert _c_call(device=3) in (km.INVALID_ARGUMENTS, km.NO_SUCH_DEVICE)   # no such device without two GPUs
    assert _c_call(strategy=2) == km.INVALID_ARGUMENTS
    assert _c_call(strategy=-1) == km.INVALID_ARGUMENTS
    assert _c_call(n_init=0) == km.INVALID_ARGUMENTS
    for init in (km.INIT_PLUSPLUS, km.INIT_AFKMC2, km.INIT_IMPORT, km.INIT_KMEANS_PARALLEL):
        assert _c_call(init=init) == km.INVALID_ARGUMENTS
    assert _c_call(init=km.INIT_GREEDY_PLUSPLUS, trials=33) == km.INVALID_ARGUMENTS
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    assert _c_call() == km.INVALID_ARGUMENTS
