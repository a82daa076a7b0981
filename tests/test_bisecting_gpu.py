"""GPU tests of bisecting k-means (kmeans_cuda(..., bisecting=...); include/kmcuda_b200.h, DESIGN.md §4o).

The library is pinned to its NumPy model (tests/bisecting_model.py): centroids, assignments, the inertia (%.17g) and the
verbosity-2 lines that start with "bisecting" are identical to the model's with the library's wave schedule, and the
centroids, assignments and inertia also to the model's sequential schedule (one node bisected per round, as
scikit-learn does), which shows that the waves change nothing but the speed."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bisecting_model as M  # noqa: E402

pytestmark = pytest.mark.gpu

SEED = 5


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _blobs(n, d, k, seed=0, spread=0.6):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    return (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)


def _weights(kind, n, seed=3):
    rng = np.random.default_rng(seed)
    if kind is None:
        return None
    if kind == "int":
        return rng.integers(1, 5, n).astype(np.float32)
    if kind == "lognormal":
        return rng.lognormal(0, 1, n).astype(np.float32)
    w = rng.lognormal(0, 1, n).astype(np.float32)   # "zeros": 30 % of the rows carry no weight
    w[rng.random(n) < 0.3] = 0
    return w


def _run(km, capfd, X, K, strategy, n_init=1, tolerance=1e-4, max_iter=0, w=None, init="random", **kw):
    capfd.readouterr()
    C, A, e = km.kmeans_cuda(X, K, tolerance=tolerance, init=init, seed=SEED, verbosity=2, sample_weight=w,
                             bisecting=strategy, n_init=n_init, max_iter=max_iter, inertia=True, **kw)
    out = capfd.readouterr().out
    return C, A, e, [ln for ln in out.splitlines() if ln.startswith("bisecting: ")]


def _pin(km, capfd, X, K, strategy, n_init=1, tolerance=1e-4, max_iter=0, w=None, init="random"):
    C, A, e, lines = _run(km, capfd, X, K, strategy, n_init, tolerance, max_iter, w, init)
    # the device's tolerance comes from Job::mean_variance; the model's numpy variance agrees with it to rounding, which
    # no stop decision of these cases lies within
    for waves in (True, False):
        mC, mA, mlines, me, _, _ = M.bisecting(X, K, SEED, strategy, n_init, tolerance, max_iter, w, waves, init=init)
        np.testing.assert_array_equal(A, mA)
        np.testing.assert_array_equal(C.view(np.uint32), mC.view(np.uint32))
        assert "%.17g" % e == "%.17g" % me
        if waves:
            assert lines == mlines
            wave_lines = mlines
    return wave_lines


SHAPES = {"d64": (4000, 64), "d67": (3000, 67), "d768": (1200, 768), "d1100": (900, 1100)}
CASES = [  # (shape, K, strategy, n_init, weights)
    ("d64", 16, "biggest_inertia", 1, None),
    ("d64", 16, "largest_cluster", 3, "int"),
    ("d64", 100, "biggest_inertia", 1, "lognormal"),
    ("d64", 100, "largest_cluster", 1, None),
    ("d67", 16, "biggest_inertia", 3, "zeros"),
    ("d67", 2, "largest_cluster", 1, "lognormal"),
    ("d768", 16, "biggest_inertia", 1, "int"),
    ("d768", 2, "biggest_inertia", 3, None),
    ("d1100", 16, "largest_cluster", 1, "zeros"),
    ("d1100", 2, "biggest_inertia", 1, None),
]


@pytest.mark.parametrize("shape,K,strategy,n_init,weights", CASES,
                         ids=["%s-K%d-%s-n%d-%s" % (c[0], c[1], c[2][:7], c[3], c[4]) for c in CASES])
def test_bit_identical_to_the_model(km, capfd, shape, K, strategy, n_init, weights):
    n, d = SHAPES[shape]
    X = _blobs(n, d, 12, seed=d)
    _pin(km, capfd, X, K, strategy, n_init, w=_weights(weights, n))


GREEDY = [  # (shape, K, strategy, n_init, weights, init)
    ("d64", 16, "biggest_inertia", 1, None, "greedy-k-means++"),
    ("d64", 100, "largest_cluster", 3, "int", ("greedy-k-means++", 5)),
    ("d67", 16, "largest_cluster", 3, "zeros", ("greedy-k-means++", 1)),
    ("d768", 16, "biggest_inertia", 1, "int", ("greedy-k-means++", 5)),
    ("d1100", 16, "largest_cluster", 1, "lognormal", "greedy-k-means++"),
    ("d1100", 2, "biggest_inertia", 3, None, ("greedy-k-means++", 1)),
]


@pytest.mark.parametrize("shape,K,strategy,n_init,weights,init", GREEDY,
                         ids=["%s-K%d-%s-n%d-%s-L%s" % (c[0], c[1], c[2][:7], c[3], c[4],
                                                        c[5][1] if isinstance(c[5], tuple) else "default")
                              for c in GREEDY])
def test_greedy_init_bit_identical_to_the_model(km, capfd, shape, K, strategy, n_init, weights, init):
    n, d = SHAPES[shape]
    X = _blobs(n, d, 12, seed=d + 2)
    _pin(km, capfd, X, K, strategy, n_init, w=_weights(weights, n), init=init)


@pytest.mark.parametrize("shape", ["d64", "d67", "d1100"])
def test_tolerance_zero_max_iter_three(km, capfd, shape):
    n, d = SHAPES[shape]
    X = _blobs(n, d, 12, seed=d + 1, spread=2.0)
    lines = _pin(km, capfd, X, 16, "biggest_inertia", 1, tolerance=0.0, max_iter=3, w=_weights("int", n))
    assert any("stopped on max_iter" in ln for ln in lines)


def test_many_small_leaves(km, capfd):
    """waves of hundreds of segments"""
    X = _blobs(20000, 8, 40, seed=9, spread=1.0)
    lines = _pin(km, capfd, X, 500, "largest_cluster", 1)
    assert int(lines[-1].split(" waves")[0].split()[-1]) < 100
    lines = _pin(km, capfd, X, 500, "biggest_inertia", 1, init="greedy-k-means++")
    assert int(lines[-1].split(" waves")[0].split()[-1]) < 100


def test_duplicated_rows_relocate_an_empty_child(km, capfd, monkeypatch):
    rng = np.random.default_rng(4)
    base = rng.standard_normal((6, 5)).astype(np.float32)
    X = base[rng.integers(0, 6, 300)]
    relocations = []
    real = M.two_means

    def two_means(*a):
        run = real(*a)
        relocations.append(run["relocations"])
        return run

    monkeypatch.setattr(M, "two_means", two_means)
    _pin(km, capfd, X, 6, "biggest_inertia", 2)
    assert sum(relocations) > 0


def test_unsplittable_node(km, capfd):
    """4 distinct rows, K = 4: the two largest leaves hold one distinct row each, and every split of them leaves a child
    empty, so they are not split and the smallest leaf is"""
    rng = np.random.default_rng(2)
    base = np.array([[0, 0], [10, 0], [0, 10], [10, 10]], np.float32)
    X = base[rng.permutation(np.repeat(np.arange(4), [50, 30, 5, 5]))]
    lines = _pin(km, capfd, X, 4, "largest_cluster", 1)
    assert any(ln.endswith("is not split") for ln in lines)


def test_fewer_distinct_rows_than_clusters(km):
    X = np.repeat(np.eye(3, dtype=np.float32), 20, axis=0)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 4, init="random", seed=1, bisecting="biggest_inertia")


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_sample(km, bad):
    X = _blobs(500, 4, 3)
    X[77, 2] = bad
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 4, init="random", seed=1, bisecting="biggest_inertia")


def test_all_ones_weights_equal_unweighted(km, capfd):
    X = _blobs(3000, 67, 10, seed=1)
    a = _run(km, capfd, X, 12, "biggest_inertia", 2)
    b = _run(km, capfd, X, 12, "biggest_inertia", 2, w=np.ones(len(X), np.float32))
    np.testing.assert_array_equal(a[0].view(np.uint32), b[0].view(np.uint32))
    np.testing.assert_array_equal(a[1], b[1])
    assert a[2] == b[2] and a[3] == b[3]


def test_fp16_and_device_pointers_match_host_fp32(km, capfd):
    import torch
    X = _blobs(2000, 64, 10, seed=2).astype(np.float16)
    Xf = X.astype(np.float32)
    C, A, e, lines = _run(km, capfd, Xf, 10, "largest_cluster")
    C16, A16, e16, lines16 = _run(km, capfd, X.view(np.float16).reshape(2000, 64), 10, "largest_cluster")
    np.testing.assert_array_equal(A16, A)
    np.testing.assert_array_equal(C16, C.astype(np.float16))
    assert lines16 == lines
    Xt = torch.from_numpy(Xf).cuda()
    Ct = torch.empty((10, 64), dtype=torch.float32, device="cuda")
    At = torch.empty(2000, dtype=torch.int32, device="cuda")
    km.kmeans_cuda((Xt.data_ptr(), 0, (2000, 64), Ct.data_ptr(), At.data_ptr()), 10, tolerance=1e-4, init="random",
                   seed=SEED, bisecting="largest_cluster")
    torch.cuda.synchronize()
    np.testing.assert_array_equal(Ct.cpu().numpy().view(np.uint32), C.view(np.uint32))
    np.testing.assert_array_equal(At.cpu().numpy().view(np.uint32), A)


def test_quality_against_sklearn(km):
    sk = pytest.importorskip("sklearn.cluster")
    X = _blobs(50000, 32, 32, seed=7, spread=1.0)
    _, _, e = km.kmeans_cuda(X, 32, tolerance=1e-4, init="random", seed=3, bisecting="biggest_inertia",
                             inertia=True)
    ref = sk.BisectingKMeans(n_clusters=32, init="random", n_init=1, tol=M.tolerance_abs(X, 1e-4),
                             bisecting_strategy="biggest_inertia", random_state=0).fit(X.astype(np.float64))
    assert e <= 1.05 * ref.inertia_
