"""CPU checks of the relocation model (tests/relocate_model.py) against scikit-learn's own empty-cluster relocation
(sklearn.cluster._k_means_common._relocate_empty_clusters_dense) and Lloyd run (_kmeans_single_lloyd), and of the
Yinyang bound argument for a relocating update (DESIGN.md §4l)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import relocate_model as R  # noqa: E402

common = pytest.importorskip("sklearn.cluster._k_means_common")
kmeans_mod = pytest.importorskip("sklearn.cluster._kmeans")


def _blobs(n, d, k, seed=0, spread=0.5):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)) * 4
    lab = rng.integers(0, k, n)
    return centers[lab] + spread * rng.standard_normal((n, d)), lab


def _totals(X, w, labels, K):
    sums = np.zeros((K, X.shape[1]))
    np.add.at(sums, labels, w[:, None] * X)
    return sums, np.bincount(labels, weights=w, minlength=K)


def _sklearn(X, w, C_old, labels, K):
    sums, W = _totals(X, w, labels, K)
    common._relocate_empty_clusters_dense(X, w, C_old, sums, W, labels.astype(np.int32))
    return sums, W


def _model(X, w, C_old, labels, K):
    sums, W = _totals(X, w, labels, K)
    d = R.distances(X, C_old, labels)
    counts = np.bincount(labels, minlength=K)
    return R.relocate(X, w, labels, d, sums.astype(np.float32), counts, W.astype(np.float32))


def _case(n_empty, seed=0, n=400, d=5, k=8):
    X, lab = _blobs(n, d, k, seed)
    K = k + n_empty
    C_old = np.vstack([np.array([X[lab == c].mean(0) for c in range(k)]), 100 + np.arange(n_empty)[:, None] +
                       np.zeros((n_empty, d))])
    labels = np.argmin(((X[:, None] - C_old[None]) ** 2).sum(-1), 1)
    assert set(range(k, K)).isdisjoint(labels)
    return X.astype(np.float32).astype(np.float64), C_old, labels, K


def test_one_empty_cluster_matches_scikit_learn():
    X, C_old, labels, K = _case(1)
    w = np.ones(len(X))
    sk_sums, sk_W = _sklearn(X, w, C_old, labels, K)
    sums, counts, W, rec, left = _model(X, w, C_old, labels, K)
    assert left == 0 and len(rec) == 1
    np.testing.assert_allclose(sums, sk_sums, rtol=1e-6, atol=1e-4)
    np.testing.assert_array_equal(W, sk_W)
    assert rec[0][1] == int(np.argmax(R.distances(X, C_old, labels)))


@pytest.mark.parametrize("weighted", [False, True])
def test_several_empty_clusters_take_the_same_rows(weighted):
    X, C_old, labels, K = _case(4, seed=3)
    w = np.random.default_rng(1).uniform(0.5, 2, len(X)) if weighted else np.ones(len(X))
    sk_sums, sk_W = _sklearn(X, w, C_old, labels, K)
    sums, counts, W, rec, left = _model(X, w, C_old, labels, K)
    assert left == 0 and len(rec) == 4
    empties = list(range(K - 4, K))
    # the same rows, paired in another order (scikit-learn: argpartition order): the same multiset of new centroids
    mine = np.array(sorted(map(tuple, (sums[empties] / W[empties, None]).astype(np.float64))))
    theirs = np.array(sorted(map(tuple, sk_sums[empties] / sk_W[empties, None])))
    np.testing.assert_allclose(mine, theirs, rtol=1e-5, atol=1e-5)
    rows = sorted(r[1] for r in rec)
    assert np.allclose(np.array(sorted(map(tuple, X[rows]))), theirs, atol=1e-5)
    donors = sorted(set(range(K - 4)))
    np.testing.assert_allclose(sums[donors], sk_sums[donors], rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(W[donors], sk_W[donors], rtol=1e-6)


def test_a_donor_is_protected_by_the_walk():
    """the two farthest rows are a cluster's only members: the model takes one and skips the other (scikit-learn
    takes both and leaves that cluster empty)"""
    X, C_old, labels, K = _case(2)
    lone = np.flatnonzero(labels == 0)
    X = np.vstack([X, [[50, 0, 0, 0, 0], [50, 0, 0, 0, 49]]])
    C_old = np.vstack([C_old, [[50, 0, 0, 0, 25]]])
    K += 1
    labels = np.concatenate([labels, [K - 1, K - 1]])
    w = np.ones(len(X))
    sk_sums, sk_W = _sklearn(X, w, C_old, labels, K)
    sums, counts, W, rec, left = _model(X, w, C_old, labels, K)
    assert sk_W[K - 1] == 0                                  # scikit-learn empties the donor
    assert W[K - 1] == 1 and counts[K - 1] == 1              # the walk keeps its last member
    assert [r[3] for r in rec].count(K - 1) == 1 and len(rec) == 2 and lone.size


def test_zero_weight_rows_are_never_taken():
    X, C_old, labels, K = _case(1)
    w = np.ones(len(X))
    far = int(np.argmax(R.distances(X, C_old, labels)))
    w[far] = 0
    sums, counts, W, rec, left = _model(X, w, C_old, labels, K)
    assert rec[0][1] != far
    sk_sums, sk_W = _sklearn(X, w, C_old, labels, K)
    assert sk_W[K - 1] == 0                                  # scikit-learn picks the zero-weight row


def test_more_empty_clusters_than_eligible_rows():
    X = np.array([[0.0, 0], [1, 0], [5, 5], [6, 5]])
    C_old = np.array([[0.5, 0], [5.5, 5], [100, 100], [200, 200], [300, 300], [400, 400]])
    labels = np.array([0, 0, 1, 1])
    sums, counts, W, rec, left = _model(X, np.ones(4), C_old, labels, 6)
    assert len(rec) == 2 and left == 2                       # one row per donor can go
    with np.errstate(invalid="ignore", divide="ignore"):
        C = sums * (np.float32(1) / W)[:, None]
    assert np.isnan(C[4:]).all() and not np.isnan(C[:4]).any()


def test_ties_take_the_lowest_row_first():
    X = np.array([[0.0], [0], [9], [9], [9]])
    C_old = np.array([[0.0], [100], [200]])
    labels = np.zeros(5, np.int64)
    _, _, _, rec, _ = _model(X, np.ones(5), C_old, labels, 3)
    assert [r[1] for r in rec] == [2, 3]


def _labeler64(X, C):
    d = ((X.astype(np.float64)[:, None] - C.astype(np.float64)[None]) ** 2).sum(-1)
    d = np.where(np.isnan(d), np.inf, d)
    return np.argmin(d, 1)


def test_whole_run_matches_scikit_learn_lloyd():
    X, lab = _blobs(3000, 6, 10, seed=7, spread=0.3)
    X = X.astype(np.float32)
    rng = np.random.default_rng(2)
    C0 = X[rng.choice(len(X), 10, replace=False)].astype(np.float64)
    C0[[2, 5, 8]] = 1e3 + np.arange(3)[:, None]             # three clusters empty from the start
    sk_labels, _, _, _ = kmeans_mod._kmeans_single_lloyd(X.astype(np.float64), np.ones(len(X)), C0.copy(), max_iter=300,
                                                         tol=0.0, n_threads=1)
    C, labels, log = R.run(X, C0.astype(np.float32), _labeler64)
    assert sum(len(e[2]) for e in log) >= 3
    assert not np.isnan(C).any()
    np.testing.assert_array_equal(labels, sk_labels)


def test_yinyang_bounds_stay_valid_through_a_relocating_update():
    """ub += drift(own), lb_g -= max drift over group g keeps ub >= d(x, c_own) and lb_g <= min over g of d(x, c)
    because both old and new centroids are finite for a relocated cluster and for its donor"""
    X, _ = _blobs(2000, 4, 6, seed=5)
    rng = np.random.default_rng(0)
    C_old = np.vstack([X[rng.choice(len(X), 6, replace=False)], [[500, 500, 500, 500]]])
    K = len(C_old)
    groups = np.array([0, 0, 1, 1, 2, 2, 2])
    labels = _labeler64(X, C_old)
    dist = np.sqrt(((X[:, None] - C_old[None]) ** 2).sum(-1))
    ub = dist[np.arange(len(X)), labels]
    lb = np.array([[dist[i, (groups == g) & (np.arange(K) != labels[i])].min(initial=np.inf) for g in range(3)]
                   for i in range(len(X))])
    sums, W = _totals(X, np.ones(len(X)), labels, K)
    d = R.distances(X, C_old, labels)
    sums, counts, W, rec, _ = R.relocate(X, None, labels, d, sums.astype(np.float32), np.bincount(labels, minlength=K),
                                         W.astype(np.float32))
    assert len(rec) == 1
    C_new = sums.astype(np.float64) / W.astype(np.float64)[:, None]
    drift = np.sqrt(((C_new - C_old) ** 2).sum(1))
    assert np.isfinite(drift).all()
    maxdrift = np.array([drift[groups == g].max() for g in range(3)])
    ub2 = ub + drift[labels]
    lb2 = lb - maxdrift[None]
    dn = np.sqrt(((X[:, None] - C_new[None]) ** 2).sum(-1))
    assert (ub2 >= dn[np.arange(len(X)), labels] - 1e-9).all()
    for g in range(3):
        true = np.where((groups[None] == g) & (np.arange(K)[None] != labels[:, None]), dn, np.inf).min(1)
        assert (lb2[:, g] <= true + 1e-9).all()
