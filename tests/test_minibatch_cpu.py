"""CPU tests of the mini-batch k-means model (tests/minibatch_model.py) against scikit-learn, and of the Python
arguments of kmeans_cuda(..., batch_size=...) that are rejected before any device work."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import minibatch_model as M  # noqa: E402

sklearn_kmeans = pytest.importorskip("sklearn.cluster._kmeans")


def _case(seed, b=64, K=12, D=5, zero_w=True):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((b, D))
    w = rng.random(b) + 0.1
    C = rng.standard_normal((K, D))
    W = rng.random(K) * 20 + 0.5
    if zero_w:
        W[rng.random(K) < 0.3] = 0.0
    return X, w, C, W


def _labels(X, C):
    return np.argmin(((X[:, None, :] - C[None, :, :]) ** 2).sum(2), axis=1)


@pytest.mark.parametrize("seed", range(6))
def test_step_equals_scikit_learn(seed):
    X, w, C, W = _case(seed)
    labels = _labels(X, C)
    Cn, Wn, inertia, shift, _ = M.step(X, w, labels, C, W)
    sk_C, sk_W = np.empty_like(C), W.copy()
    sk_inertia = sklearn_kmeans._mini_batch_step(X, w, C, sk_C, sk_W, np.random.RandomState(0), random_reassign=False)
    sk_labels, _ = sklearn_kmeans._labels_inertia(X, w, C)
    assert np.array_equal(labels, sk_labels)
    assert abs(inertia - sk_inertia) <= 1e-12 * abs(sk_inertia)
    np.testing.assert_allclose(Cn, sk_C, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(Wn, sk_W, rtol=1e-12, atol=0)
    assert abs(shift - ((sk_C - C) ** 2).sum()) <= 1e-12 * max(1.0, shift)


@pytest.mark.parametrize("seed,b,K", [(0, 64, 12), (1, 64, 40), (2, 20, 50), (3, 8, 30), (4, 200, 300)])
def test_reassigned_set_equals_scikit_learn(seed, b, K):
    """The set of reassigned centroids (scikit-learn's to_reassign, cut to floor(b / 2)) and the weight they get."""
    X, w, C, W = _case(seed, b=b, K=K, zero_w=False)
    W *= np.random.default_rng(seed + 100).random(K) ** 8   # spread: many centroids below 1 % of the largest
    labels = _labels(X, C)
    keys = M.reassign_keys(7, 1, w)
    Cn, Wn, _, _, cidx = M.step(X, w, labels, C, W, reassign=True, keys=keys)
    plain_W = W.copy()
    sklearn_kmeans._mini_batch_step(X, w, C, np.empty_like(C), plain_W, np.random.RandomState(0),
                                    random_reassign=False)
    sk_W = W.copy()
    sklearn_kmeans._mini_batch_step(X, w, C, np.empty_like(C), sk_W, np.random.RandomState(0), random_reassign=True,
                                    reassignment_ratio=M.REASSIGNMENT_RATIO)
    sk_set = set(np.nonzero(sk_W != plain_W)[0].tolist())
    assert len(sk_set) > 0
    assert set(cidx.tolist()) == sk_set
    np.testing.assert_array_equal(Wn, sk_W)
    # the reassigned centroids are distinct batch rows
    rows = [int(np.nonzero((X == Cn[c]).all(1))[0][0]) for c in cidx]
    assert len(set(rows)) == len(rows)


def _sk_convergence(b, N, tol_abs, seq, n_steps):
    km = sklearn_kmeans.MiniBatchKMeans(n_clusters=2, batch_size=b, max_no_improvement=M.MAX_NO_IMPROVEMENT)
    km._batch_size, km._tol, km.verbose = b, tol_abs, 0
    km._ewa_inertia = km._ewa_inertia_min = None
    km._no_improvement = 0
    out = []
    for i, (inertia, shift) in enumerate(seq):
        stop = km._mini_batch_convergence(i, n_steps, N, shift, inertia)
        out.append((stop, km._ewa_inertia))
        if stop:
            break
    return out


@pytest.mark.parametrize("kind", ["plateau", "tolerance", "noisy", "first_step_tiny_shift"])
def test_stop_rule_equals_scikit_learn(kind):
    rng = np.random.default_rng(3)
    b, N, n = 256, 10000, 60
    inertia = 1000 * np.exp(-np.arange(n) / 5.0) + 50
    shift = 10 * np.exp(-np.arange(n) / 3.0)
    tol_abs = 0.0
    if kind == "tolerance":
        tol_abs = 0.05
    if kind == "noisy":
        inertia = inertia + rng.normal(0, 30, n)
    if kind == "first_step_tiny_shift":   # step 1 never stops, whatever its shift
        shift[0] = 0.0
        tol_abs = 1e-3
    seq = list(zip(inertia, shift))
    want = _sk_convergence(b, N, tol_abs, seq, n)
    conv = M.Convergence(b, N, tol_abs)
    got = []
    for s, (i_, sh) in enumerate(seq, 1):
        r = conv.update(s, i_, sh)
        got.append((r is not None, conv.ewa))
        if r:
            break
    assert len(got) == len(want)
    for (gs, ge), (ws, we) in zip(got, want):
        assert gs == ws
        assert (ge is None and we is None) or abs(ge - we) <= 1e-12 * abs(we)
    if kind == "tolerance":
        assert len(got) < n


def test_tolerance_scales_by_the_unweighted_mean_variance():
    X = np.random.default_rng(0).standard_normal((500, 7)).astype(np.float32) * np.arange(1, 8, dtype=np.float32)
    assert M.tolerance(X, 0.01) == pytest.approx(sklearn_kmeans._tolerance(X.astype(np.float64), np.float32(0.01)),
                                                 rel=1e-12)
    assert M.tolerance(X, 0) == 0


def test_draws_match_the_scalar_hash_formula():
    seed, s, N, b = 12345, 17, 1000003, 500
    rows = M.draw(seed, s, N, b)
    key = M.mix((M.mix(M.TAG_BATCH ^ seed) + s) & M.M64)
    for j in (0, 1, 2, 255, 499):
        u = (M.mix(key ^ j) >> 11) * 2.0 ** -53
        assert rows[j] == int(u * N)
    assert rows.min() >= 0 and rows.max() < N
    assert not np.array_equal(rows, M.draw(seed, s + 1, N, b))
    assert not np.array_equal(rows, M.draw(seed + 1, s, N, b))
    # the reassignment draw uses its own tag: its uniforms differ from the batch draw's
    kb = M.reassign_keys(seed, s, np.ones(b))
    assert not np.allclose(np.exp(-kb), (M.mix_np(np.uint64(key) ^ np.arange(b, dtype=np.uint64)) >> np.uint64(11))
                           * 2.0 ** -53)


def test_reassignment_keys_never_pick_a_zero_weight_entry():
    rng = np.random.default_rng(1)
    b, K = 40, 30
    X = rng.standard_normal((b, 3))
    w = rng.integers(0, 3, b).astype(np.float64)   # about a third are 0
    C = rng.standard_normal((K, 3))
    W = np.zeros(K)
    for seed in range(20):
        keys = M.reassign_keys(seed, 1, w)
        assert np.all(np.isinf(keys[w == 0])) and np.all(np.isfinite(keys[w > 0]))
        Cn, _, _, _, cidx = M.step(X, w, _labels(X, C), C, W, reassign=True, keys=keys)
        assert 0 < len(cidx) <= min(b // 2, int((w > 0).sum()))
        for c in cidx:
            j = np.nonzero((X == Cn[c]).all(1))[0]
            assert w[j[0]] > 0
    # fewer positive-weight entries than centroids to reassign: each of them is taken once
    w3 = np.zeros(b)
    w3[[4, 17, 33]] = 1.0
    Cn, _, _, _, cidx = M.step(X, w3, _labels(X, C), C, W, reassign=True, keys=M.reassign_keys(0, 1, w3))
    assert len(cidx) == 3
    assert sorted(int(np.nonzero((X == Cn[c]).all(1))[0][0]) for c in cidx) == [4, 17, 33]


def test_python_arguments_are_checked_before_the_call():
    import kmcuda_b200 as km
    X = np.zeros((10, 4), np.float32)
    for bad in ("8", 2.0, True):
        with pytest.raises(TypeError):
            km.kmeans_cuda(X, 2, batch_size=bad)
    for bad in (0, -1, 1 << 32):
        with pytest.raises(ValueError):
            km.kmeans_cuda(X, 2, batch_size=bad)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 2, batch_size=4, max_steps=-1)
    with pytest.raises(TypeError):
        km.kmeans_cuda(X, 2, batch_size=4, max_steps=1.5)
    with pytest.raises(ValueError, match="max_steps"):   # a step count without a batch size is not a Lloyd option
        km.kmeans_cuda(X, 2, max_steps=50)


def test_libkmcuda_module_checks_the_arguments():
    import importlib.util

    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    X = np.zeros((10, 4), np.float32)
    with pytest.raises(TypeError):
        mod.kmeans_cuda(X, 2, batch_size="8")
    with pytest.raises(ValueError):
        mod.kmeans_cuda(X, 2, batch_size=0)
    with pytest.raises(ValueError):
        mod.kmeans_cuda(X, 2, batch_size=4, max_steps=-2)
    with pytest.raises(ValueError):
        mod.kmeans_cuda(X, 2, max_steps=50)
