"""GPU tests of the greedy k-means++ seeding (init="greedy-k-means++"; include/kmcuda_b200.h, DESIGN.md §4m).

The seeding is pinned to its NumPy model (tests/greedy_plusplus_model.py): the init centroids, read from a tolerance=1.0
call that stops after the first assignment pass without touching them, are bit-identical to the model's, and so is the
verbosity-2 log (angular: the potentials to 1e-6, as the host's acosf and the device's may differ by an ulp).  Shapes
cover D % 4 == 0, D % 4 != 0 and D > 1024."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import greedy_plusplus_model as G  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {"d64": (4000, 64, 40), "d768": (1500, 768, 12), "d67": (3000, 67, 30), "d1100": (1200, 1100, 10)}
SEED = 7
INIT = "greedy-k-means++"


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _blobs(n, d, k, seed=0, spread=0.6, cos=False):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if cos:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _weights(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "none":
        return None
    w = rng.integers(1, 5, n).astype(np.float32)
    if kind == "zeros":
        w[rng.random(n) < 0.3] = 0
    return w


def _init(km, capfd, X, k, trials=None, **kw):
    """init centroids (tolerance=1.0 returns them untouched) and the greedy k-means++ log lines"""
    capfd.readouterr()
    kw.setdefault("seed", SEED)
    init = INIT if trials is None else (INIT, trials)
    c, _ = km.kmeans_cuda(X, k, init=init, tolerance=1.0, yinyang_t=0, device=1, verbosity=2, **kw)
    lines = [ln.lstrip("\r") for ln in capfd.readouterr().out.splitlines()]
    return c, [ln for ln in lines if ln.startswith("greedy k-means++")]


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _check_log(got, want, rel=0.0):
    assert len(got) == len(want), (got[:3], want[:3])
    for g, w in zip(got, want):
        gh, _, gp = g.partition("potential ")
        wh, _, wp = w.partition("potential ")
        assert gh == wh, (g, w)
        if rel == 0.0 or not gp[:1].isdigit():
            assert gp == wp, (g, w)
        else:
            assert abs(float(gp) - float(wp)) <= rel * abs(float(wp)), (g, w)


def _model(X, k, metric, w, trials=None, seed=SEED):
    L = trials or G.default_trials(k)
    rows, pots, _, filled, C = G.greedy(X, k, seed, L=L, w=w, metric=1 if metric == "cos" else 0)
    return C, G.log_lines(L, rows, pots, filled, k), rows


# ------------------------------------------------------------------------------------------------ 1. model equality
CASES = [(shape, metric, weights, None) for shape in SHAPES for metric, weights in
         (("L2", "integer"), ("cos", "zeros"))]
CASES += [("d64", "L2", weights, trials) for trials in (1, 32) for weights in ("none", "zeros")]
CASES += [("d64", "L2", "none", None), ("d1100", "L2", "none", 32), ("d67", "cos", "none", 1), ("d768", "L2", "zeros", 1)]


@pytest.mark.parametrize("shape,metric,weights,trials", CASES)
def test_seeding_matches_the_model(km, capfd, shape, metric, weights, trials):
    n, d, k = SHAPES[shape]
    X = _blobs(n, d, k, seed=1, cos=metric == "cos")
    w = _weights(weights, n, 2)
    kw = {} if w is None else {"sample_weight": w}
    c, log = _init(km, capfd, X, k, trials=trials, metric=metric, **kw)
    cm, lines, _ = _model(X, k, metric, w, trials)
    _check_log(log, lines, rel=0.0 if metric == "L2" else 1e-6)
    assert _same(c, cm)


# ------------------------------------------------------------------------------------------------------ 2. edge cases
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_all_ones_weights_are_bit_identical_to_unweighted(km, capfd, metric):
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=3, cos=metric == "cos")
    c0, l0 = _init(km, capfd, X, k, metric=metric)
    c1, l1 = _init(km, capfd, X, k, metric=metric, sample_weight=np.ones(n, np.float32))
    assert l0 == l1 and _same(c0, c1)
    r0 = km.kmeans_cuda(X, k, init=INIT, metric=metric, seed=SEED, device=1, average_distance=True)
    r1 = km.kmeans_cuda(X, k, init=INIT, metric=metric, seed=SEED, device=1, average_distance=True,
                        sample_weight=np.ones(n, np.float32))
    assert _same(r0[0], r1[0]) and np.array_equal(r0[1], r1[1]) and r0[2] == r1[2]


def test_nan_zero_weight_and_duplicated_rows_are_never_chosen_twice(km, capfd):
    rng = np.random.default_rng(4)
    base = _blobs(600, 32, 30, seed=4)
    X = np.concatenate([base, base[:300], base[:100]])   # every one of the first 100 rows three times
    X[rng.choice(len(X), 40, replace=False), 0] = np.nan
    w = rng.integers(1, 4, len(X)).astype(np.float32)
    w[rng.random(len(X)) < 0.2] = 0
    k = 60
    c, log = _init(km, capfd, X, k, sample_weight=w)
    cm, lines, rows = _model(X, k, "L2", w)
    _check_log(log, lines)
    assert _same(c, cm)
    assert len(set(map(bytes, c))) == k and not np.isnan(c).any()
    assert (w[rows] > 0).all()


def test_fewer_distinct_rows_than_k_take_the_fill_walk(km, capfd):
    base = np.random.default_rng(8).standard_normal((4, 30)).astype(np.float32)
    X = np.repeat(base, [5000, 1, 1, 1], axis=0)
    c, log = _init(km, capfd, X, 20)
    cm, lines, _ = _model(X, 20, "L2", None)
    _check_log(log, lines)
    assert log[-1].endswith("the rest from the random walk")
    assert _same(c, cm)


def test_fp16_samples_equal_fp32_on_the_widened_values(km, capfd):
    n, d, k = SHAPES["d64"]
    X16 = _blobs(n, d, k, seed=6).astype(np.float16)
    c16, l16 = _init(km, capfd, X16, k)
    c32, l32 = _init(km, capfd, X16.astype(np.float32), k)
    assert l16 == l32
    assert np.array_equal(c16.view(np.uint16), c32.astype(np.float16).view(np.uint16))


def test_device_pointers_equal_host_input(km, capfd):
    import torch
    n, d, k = SHAPES["d67"]
    X = _blobs(n, d, k, seed=7)
    w = _weights("zeros", n, 7)
    ch, lh = _init(km, capfd, X, k, sample_weight=w)
    Xt = torch.from_numpy(X).cuda()
    wt = torch.from_numpy(w).cuda()
    capfd.readouterr()
    cp, ap = km.kmeans_cuda((Xt.data_ptr(), 0, X.shape), k, init=INIT, tolerance=1.0, yinyang_t=0, seed=SEED,
                            device=1, verbosity=2, sample_weight=wt.data_ptr())
    ld = [ln.lstrip("\r") for ln in capfd.readouterr().out.splitlines()]
    ld = [ln for ln in ld if ln.startswith("greedy k-means++")]
    cd = np.empty((k, d), np.float32)
    km._cuda_memcpy_d2h(0, cd.ctypes.data, cp, cd.nbytes)
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    assert lh == ld and _same(ch, cd)


# -------------------------------------------------------------------------------------------------------- 3. quality
def test_greedy_seeds_beat_k_means_plus_plus_and_k_means_parallel(km):
    """The blob set of test_k_means_parallel_seeds_no_worse_than_k_means_plus_plus: the seeded average distance is at
    most 0.7 x k-means++'s and at most k-means||'s, and the Lloyd run from it ends within 2 % of scikit-learn's
    KMeans(init="k-means++", n_init=1)."""
    from sklearn.cluster import KMeans
    n, d, k = 50000, 64, 200
    X = _blobs(n, d, k, seed=10, spread=0.3)
    seeded = {init: km.kmeans_cuda(X, k, init=init, tolerance=1.0, yinyang_t=0, seed=SEED, device=1,
                                   average_distance=True)[2] for init in (INIT, "k-means++", "k-means||")}
    assert seeded[INIT] <= 0.7 * seeded["k-means++"] and seeded[INIT] <= seeded["k-means||"]
    final = km.kmeans_cuda(X, k, init=INIT, tolerance=0.01, yinyang_t=0, seed=SEED, device=1, average_distance=True)[2]
    sk = KMeans(k, init="k-means++", n_init=1, random_state=0).fit(X.astype(np.float64))
    ref = np.linalg.norm(X - sk.cluster_centers_[sk.labels_], axis=1).mean()
    assert final <= 1.02 * ref, (final, ref, seeded)


# ------------------------------------------------------------------------------------------ 4. with the run options
def test_composes_with_minibatch_and_relocation(km, capfd):
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=11)
    C0, _ = _init(km, capfd, X, k)
    for kw in ({"batch_size": 512, "max_steps": 40}, {"relocate_empty_clusters": True, "tolerance": 0.01}):
        a = km.kmeans_cuda(X, k, init=INIT, seed=SEED, device=1, **kw)
        b = km.kmeans_cuda(X, k, init=C0, seed=SEED, device=1, **kw)
        assert _same(a[0], b[0]) and np.array_equal(a[1], b[1]), kw


# ------------------------------------------------------------------------------------------------------- 5. two GPUs
def test_two_gpus_match_one_gpu(km, capfd):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=12, spread=0.1)
    capfd.readouterr()
    c1, a1 = km.kmeans_cuda(X, k, init=INIT, tolerance=1.0, yinyang_t=0, seed=SEED, device=1)
    c2, a2 = km.kmeans_cuda(X, k, init=INIT, tolerance=1.0, yinyang_t=0, seed=SEED, device=3)
    assert _same(c1, c2) and np.array_equal(a1, a2)
