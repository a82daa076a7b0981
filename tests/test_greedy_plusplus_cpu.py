"""CPU tests of the greedy k-means++ seeding (init="greedy-k-means++"): its NumPy model (which the GPU tests use as the
reference) pinned to scikit-learn's _kmeans_plusplus, the d^2 draw, the shard merge, and the intake of both Python
surfaces."""
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import greedy_plusplus_model as G  # noqa: E402
import kmeans_parallel_model as KP  # noqa: E402


def _blobs(n, d, k, seed=0, spread=0.6):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    return X


@pytest.mark.parametrize("metric", [0, 1])
def test_model_distances_are_the_oracles(metric):
    rng = np.random.default_rng(0)
    X = rng.standard_normal((600, 67)).astype(np.float32)
    if metric:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    X[3, 5] = np.nan
    E = G.distances(X, X[[7, 9]], metric)
    for j, c in enumerate([7, 9]):
        ref = KP.row_distances(X, X[[c]], np.zeros(len(X), np.uint32), metric)
        if metric == 0:
            assert np.array_equal(E[j].view(np.uint32), ref.view(np.uint32))
        else:   # acosf: the model rounds the float64 arccos, libm's acosf may differ by an ulp
            ok = np.isfinite(ref)
            assert np.array_equal(np.isnan(E[j]), np.isnan(ref))
            assert np.max(np.abs(E[j][ok].astype(np.float64) - ref[ok])) <= 2 * np.spacing(np.float32(np.pi))


def test_block_sum_is_the_device_order():
    rng = np.random.default_rng(1)
    m = rng.lognormal(0, 3, 300000)
    assert abs(G.block_sum(m) - m.sum()) <= 1e-12 * m.sum()
    assert G.block_sum(np.ones(5)) == 5.0 and G.block_sum([]) == 0.0
    # a block partial: the shuffle tree over 32 lanes, then the four warps in order
    v = rng.random(128)
    a = v.reshape(4, 32)
    while a.shape[1] > 1:
        a = a[:, :a.shape[1] // 2] + a[:, a.shape[1] // 2:]
    assert G.block_sum(v) == ((0.0 + a[0, 0]) + a[1, 0] + a[2, 0]) + a[3, 0]


# ------------------------------------------------------------------------------------------ the model = scikit-learn
class _Pinned:
    """random_state for sklearn's _kmeans_plusplus whose draws land on the model's picks: choice() returns c0, and
    uniform(size=L) returns the midpoints of the model's trial rows' intervals in scikit-learn's own CDF (its running
    minimum of squared distances over the model's picks so far, times w), divided by its potential"""

    def __init__(self, X64, w, rows, drawn):
        from sklearn.metrics.pairwise import _euclidean_distances
        sq = (X64 ** 2).sum(1)
        self.dist = lambda i: _euclidean_distances(X64[[i]], X64, Y_norm_squared=sq, squared=True)[0]
        self.w, self.rows, self.drawn, self.r = w, rows, drawn, 0
        self.closest = None

    def choice(self, n, p=None):
        self.closest = self.dist(int(self.rows[0]))
        return int(self.rows[0])

    def uniform(self, size):
        if self.r > 0:   # scikit-learn chose the previous round's best trial: the model's pick, if they agree
            self.closest = np.minimum(self.closest, self.dist(int(self.rows[self.r])))
        cdf = np.cumsum(self.w * self.closest)
        pot = self.closest @ self.w
        lo = np.concatenate([[0.0], cdf[:-1]])
        u = np.array([(lo[i] + cdf[i]) / 2 / pot for i in self.drawn[self.r]])
        assert len(u) == size
        self.r += 1
        return u


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("L", [1, None, 7])
def test_model_picks_what_scikit_learn_picks(weighted, L):
    from sklearn.cluster._kmeans import _kmeans_plusplus
    X = _blobs(3000, 16, 30, seed=2)
    K = 30
    w = np.random.default_rng(3).integers(0, 4, len(X)).astype(np.float32) if weighted else None
    rows, pots, drawn, filled, _ = G.greedy(X, K, seed=5, L=L, w=w)
    assert filled == K and len(drawn) == K - 1
    X64 = X.astype(np.float64)
    w64 = np.ones(len(X)) if w is None else w.astype(np.float64)
    _, idx = _kmeans_plusplus(X64, K, (X64 ** 2).sum(1), w64, _Pinned(X64, w64, rows, drawn), n_local_trials=L)
    assert np.array_equal(idx, rows)
    # the potentials agree to float32 distance precision
    ref = ((X64[:, None, :] - X64[rows][None]) ** 2).sum(-1).min(1) @ w64
    assert abs(pots[-1] - ref) <= 1e-5 * ref


def test_default_trials_are_scikit_learns():
    assert [G.default_trials(k) for k in (2, 7, 8, 200, 1024)] == [2, 3, 4, 7, 8]


# ------------------------------------------------------------------------------------------------------ the draws
def test_trial_draws_are_proportional_to_w_d_squared():
    from scipy import stats
    rng = np.random.default_rng(4)
    n = 40
    d = rng.random(n).astype(np.float32) + 0.1
    w = rng.integers(0, 4, n).astype(np.float32)
    d[5] = 0
    d[6] = np.nan
    m = KP.mass(d, w)
    counts = np.zeros(n)
    for r in range(1, 1501):
        for t in range(8):
            counts[G.keys(m, 9, r, t).argmin()] += 1
    assert counts[m == 0].sum() == 0 and m[5] == 0 and m[6] == 0
    live = m > 0
    expected = m[live] / m[live].sum() * counts.sum()
    assert stats.chisquare(counts[live], expected).pvalue > 1e-3


def test_trials_do_not_depend_on_the_shard_split():
    rng = np.random.default_rng(5)
    m = KP.mass(rng.random(30000).astype(np.float32), rng.integers(0, 3, 30000).astype(np.float32))
    for r in (1, 2, 77):
        whole = G.trials(m, 11, r, 9)
        for cuts in ([10000], [512, 20000], [7, 8, 29999]):
            assert G.trials(m, 11, r, 9, cuts) == whole


def test_model_over_shards_picks_the_same_rows():
    X = _blobs(2000, 8, 10, seed=6)
    one = G.greedy(X, 12, seed=3)[0]
    for cuts in ([1000], [300, 1700]):
        assert np.array_equal(G.greedy(X, 12, seed=3, cuts=cuts)[0], one)


def test_model_without_mass_takes_the_fill_walk():
    base = np.random.default_rng(7).standard_normal((4, 30)).astype(np.float32)
    X = np.repeat(base, [200, 1, 1, 1], axis=0)
    rows, pots, _, filled, C = G.greedy(X, 20, seed=5)
    assert filled == 4 and len(set(rows.tolist())) == 4 and pots[-1] == 0
    assert C.shape == (20, 30) and np.array_equal(C[:4], X[rows])
    assert G.log_lines(3, rows, pots, filled, 20)[-1].endswith("after 4 centroids, the rest from the random walk")


# -------------------------------------------------------------------------------------------------- argument intake
def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


def test_both_python_surfaces_accept_greedy_k_means_plus_plus():
    import torch
    km, mod = _surfaces()
    assert km.INIT_GREEDY_PLUSPLUS == 5
    X = np.random.default_rng(8).random((100, 8), dtype=np.float32)
    for f in (km.kmeans_cuda, mod.kmeans_cuda):
        for init in ("greedy-k-means++", "greedy-kmeans++", ("greedy-k-means++", 1), ("greedy-kmeans++", 0),
                     ("greedy-k-means++", np.int64(32))):
            if not torch.cuda.is_available():
                with pytest.raises(ValueError, match="No such CUDA device"):
                    f(X, 5, init=init)
        for bad in (33, -1, 2.5, "3", True, None):
            with pytest.raises(ValueError, match="greedy k-means\\+\\+ trials"):
                f(X, 5, init=("greedy-k-means++", bad))
        with pytest.raises(ValueError, match="Unknown centroids initialization"):
            f(X, 5, init="greedy")


def test_c_abi_rejects_more_than_32_trials_before_touching_a_device():
    km, _ = _surfaces()
    X = np.random.default_rng(9).random((100, 8), dtype=np.float32)
    C = np.zeros((5, 8), np.float32)
    A = np.zeros(100, np.uint32)
    for fn in (km._lib.kmeans_cuda, km._lib.kmcuda_b200_kmeans_weighted, km._lib.kmcuda_b200_kmeans_relocate):
        t = ctypes.c_uint32(33)
        args = [5, ctypes.byref(t), 0.01, 0.1, 0, 100, 8, 5, 1, 0, -1, 0, 0, X.ctypes.data]
        if fn is not km._lib.kmeans_cuda:
            args.append(None)
        assert fn(*args, C.ctypes.data, A.ctypes.data, None) == km.INVALID_ARGUMENTS
