"""GPU tests of the k-means|| seeding (init="k-means||"; include/kmcuda_b200.h, DESIGN.md §4g).

The seeding is pinned to its NumPy model (tests/kmeans_parallel_model.py): the per-round log (drawn counts exactly,
costs to 1e-12) and the init centroids, which must be bit-identical to the library's own weighted run on the model's
candidates and weights.  The init centroids are read from a tolerance=1.0 call, which stops after the first
assignment pass without touching them.  Shapes as in test_weights_gpu.py: 50000 x 64 @ 200 takes the tensor-core
assignment path, 20000 x 30 @ 50 the exact one."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import kmeans_parallel_model as M  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {"tc": (50000, 64, 200), "exact": (20000, 30, 50)}
SEED = 7


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _blobs(n, d, k, seed=0, spread=0.6, cos=False):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    label = rng.integers(0, k, n)
    X = (centers[label] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if cos:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X, centers, label


def _weights(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "none":
        return None
    w = rng.integers(1, 5, n).astype(np.float32)
    if kind == "zeros":
        w[rng.random(n) < 0.3] = 0
    return w


def _run(km, capfd, X, k, init=("k-means||", 0), **kw):
    capfd.readouterr()
    kw.setdefault("seed", SEED)
    out = km.kmeans_cuda(X, k, init=init, device=1, verbosity=1, **kw)
    lines = capfd.readouterr().out.splitlines()
    return out, [ln for ln in lines if ln.startswith("k-means||")], [ln for ln in lines if ln.startswith("iteration")]


def _init(km, capfd, X, k, **kw):
    """init centroids (tolerance=1.0 returns them untouched) and the k-means|| log"""
    (c, _), klog, _ = _run(km, capfd, X, k, tolerance=1.0, yinyang_t=0, **kw)
    return c, klog


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _check_log(got, want, rel=1e-12):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        gh, wh = g.rsplit("cost", 1) if "cost" in g else (g, None), w.rsplit("cost", 1) if "cost" in w else (w, None)
        assert gh[0] == wh[0], (g, w)
        if gh[1] is not None:
            gc, wc = float(gh[1]), float(wh[1])
            assert abs(gc - wc) <= rel * abs(wc), (g, w)


def _model_centroids(km, X, k, metric, w, seed=SEED, samples=None):
    """the model's candidates, log lines and init centroids (through the library's weighted run when C_n > K).
    samples: what the weighted run is given (default X), e.g. the fp16 rows whose widened values X holds"""
    mid = 1 if metric == "cos" else 0
    rows, log, nearest = M.candidates(X, k, seed, w=w, metric=mid)
    lines = M.log_lines(log, len(rows), k)
    if len(rows) <= k:
        return rows, lines, M.fill(X, rows, k, seed, w=w)
    W = M.candidate_weights(nearest, len(rows), w)
    C, _ = km.kmeans_cuda((X if samples is None else samples)[rows], k, init="k-means++", tolerance=0.01,
                          yinyang_t=0, metric=metric, seed=seed, device=1, sample_weight=W)
    return rows, lines, C


# ------------------------------------------------------------------------------------------------ 1. model equality
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("metric", ["L2", "cos"])
@pytest.mark.parametrize("weights", ["none", "integer", "zeros"])
def test_seeding_matches_the_model(km, capfd, shape, metric, weights):
    n, d, k = SHAPES[shape]
    X, _, _ = _blobs(n, d, k, seed=1, cos=metric == "cos")
    w = _weights(weights, n, 2)
    kw = {} if w is None else {"sample_weight": w}
    c, klog = _init(km, capfd, X, k, metric=metric, **kw)
    rows, lines, cm = _model_centroids(km, X, k, metric, w)
    # angular: the host's acosf and the device's may differ by an ulp, which moves the cost in its 8th digit
    _check_log(klog, lines, rel=1e-12 if metric == "L2" else 1e-6)
    assert len(rows) > k
    assert _same(c, cm)


# ------------------------------------------------------------------------------- 2. all-ones weights = unweighted
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_all_ones_weights_are_bit_identical_to_unweighted(km, capfd, shape, metric):
    n, d, k = SHAPES[shape]
    X, _, _ = _blobs(n, d, k, seed=3, cos=metric == "cos")
    (c0, a0, avg0), k0, it0 = _run(km, capfd, X, k, metric=metric, tolerance=0.01, yinyang_t=0.1,
                                   average_distance=True)
    (c1, a1, avg1), k1, it1 = _run(km, capfd, X, k, metric=metric, tolerance=0.01, yinyang_t=0.1,
                                   average_distance=True, sample_weight=np.ones(n, np.float32))
    assert len(k0) >= 2 and k0 == k1 and len(it0) >= 2 and it0 == it1
    assert _same(c0, c1) and np.array_equal(a0, a1) and avg0 == avg1


# --------------------------------------------------------------------------------------------- 3. determinism, seed
def test_same_seed_same_result_other_seed_other_result(km, capfd):
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=4)
    (c0, a0), l0, _ = _run(km, capfd, X, k, tolerance=0.01)
    (c1, a1), l1, _ = _run(km, capfd, X, k, tolerance=0.01)
    assert l0 == l1 and _same(c0, c1) and np.array_equal(a0, a1)
    c2, l2 = _init(km, capfd, X, k, seed=SEED + 1)
    c3, _ = _init(km, capfd, X, k)
    assert l2 != l0 or not _same(c2, c3)


# -------------------------------------------------------------------------------- 4. exact route = tensor-core route
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_forced_exact_route_is_bit_identical(km, capfd, monkeypatch, metric):
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=5, cos=metric == "cos")
    c0, l0 = _init(km, capfd, X, k, metric=metric)
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1")
    c1, l1 = _init(km, capfd, X, k, metric=metric)
    assert l0 == l1 and _same(c0, c1)


# ---------------------------------------------------------------------------------------- 5. fp16, device pointers
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fp16_samples_equal_fp32_on_the_widened_values(km, capfd, shape):
    n, d, k = SHAPES[shape]
    X, _, _ = _blobs(n, d, k, seed=6)
    X16 = X.astype(np.float16)
    (c16, a16), l16, _ = _run(km, capfd, X16, k, tolerance=0.01, yinyang_t=0)
    (c32, a32), l32, _ = _run(km, capfd, X16.astype(np.float32), k, tolerance=0.01, yinyang_t=0)
    assert l16 == l32 and np.array_equal(a16, a32)
    assert np.array_equal(c16.view(np.uint16), c32.astype(np.float16).view(np.uint16))


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fp16_angular_samples_match_the_model(km, capfd, shape):
    """fp16x2 angular input: widened unit vectors are unit length only to fp16 precision, which the call accepts (it
    probes unit length on fp32 input only); the reclustering of the candidates must accept them too"""
    n, d, k = SHAPES[shape]
    X, _, _ = _blobs(n, d, k, seed=12, cos=True)
    X16 = X.astype(np.float16)
    c16, klog = _init(km, capfd, X16, k, metric="cos")
    rows, lines, cm = _model_centroids(km, X16.astype(np.float32), k, "cos", None, samples=X16)
    _check_log(klog, lines, rel=1e-6)
    assert len(rows) > k and c16.dtype == np.float16
    assert np.array_equal(c16.view(np.uint16), cm.view(np.uint16))


def test_strict_update_mode_leaves_the_seeding_alone(km, capfd, monkeypatch):
    """KMCUDA_B200_STRICT_UPDATE=1 replays the reference's unweighted update for the caller's run; the weighted
    reclustering of the candidates must not take it (the init centroids come out of a tolerance=1.0 call unchanged)"""
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=13)
    c0, l0 = _init(km, capfd, X, k)
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    c1, l1 = _init(km, capfd, X, k)
    assert l0 == l1 and _same(c0, c1)


@pytest.mark.parametrize("weighted", [False, True])
def test_device_pointers_equal_host_input(km, capfd, weighted):
    import torch
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=7)
    w = _weights("zeros", n, 7) if weighted else None
    kw = {} if w is None else {"sample_weight": w}
    (ch, ah), lh, _ = _run(km, capfd, X, k, tolerance=0.01, yinyang_t=0.1, **kw)
    Xt = torch.from_numpy(X).cuda()
    wt = None if w is None else torch.from_numpy(w).cuda()
    kw = {} if w is None else {"sample_weight": wt.data_ptr()}
    (cp, ap), ld, _ = _run(km, capfd, (Xt.data_ptr(), 0, X.shape), k, tolerance=0.01, yinyang_t=0.1, **kw)
    cd = np.empty((k, d), np.float32)
    ad = np.empty(n, np.uint32)
    km._cuda_memcpy_d2h(0, cd.ctypes.data, cp, cd.nbytes)
    km._cuda_memcpy_d2h(0, ad.ctypes.data, ap, ad.nbytes)
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    assert lh == ld and _same(ch, cd) and np.array_equal(ah, ad)


# ----------------------------------------------------------------------------------------- 6. at most K candidates
def test_few_candidates_take_the_fill_walk(km, capfd):
    rng = np.random.default_rng(8)
    base = rng.standard_normal((4, 30)).astype(np.float32)
    X = np.repeat(base, [20000, 1, 1, 1], axis=0)   # the repeated row is c0, round 1 draws the other three
    c, klog = _init(km, capfd, X, 50)
    rows, lines, cm = _model_centroids(km, X, 50, "L2", None)
    assert len(rows) <= 50
    _check_log(klog, lines)
    assert _same(c, cm)


@pytest.mark.parametrize("weights", ["none", "zeros"])
def test_k_plus_five_rows(km, capfd, weights):
    n, d, k = 55, 30, 50
    X, _, _ = _blobs(n, d, 10, seed=9)
    w = None if weights == "none" else _weights("integer", n, 9)
    if w is not None:
        w[:3] = 0   # 52 rows of positive weight, enough for 50 centroids
    kw = {} if w is None else {"sample_weight": w}
    c, klog = _init(km, capfd, X, k, **kw)
    _, lines, cm = _model_centroids(km, X, k, "L2", w)
    _check_log(klog, lines)
    assert _same(c, cm)


# -------------------------------------------------------------------------------------------------------- 7. quality
def test_k_means_parallel_seeds_no_worse_than_k_means_plus_plus(km, capfd):
    """Well-separated blobs: the seeded average distance (tolerance 1.0, no update) is no higher than k-means++'s, and
    the Lloyd run from it ends within 20 % of the one from k-means++.  Not every blob is guaranteed a seed: the recluster
    is k-means++, which draws proportionally to W * d (DESIGN.md §4g)."""
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=10, spread=0.3)
    avg = {}
    for init in ("k-means||", "k-means++"):
        seeded = km.kmeans_cuda(X, k, init=init, tolerance=1.0, yinyang_t=0, seed=SEED, device=1,
                                average_distance=True)[2]
        final = km.kmeans_cuda(X, k, init=init, tolerance=0.01, yinyang_t=0, seed=SEED, device=1,
                               average_distance=True)[2]
        avg[init] = (seeded, final)
    assert avg["k-means||"][0] <= avg["k-means++"][0]
    assert avg["k-means||"][1] <= avg["k-means++"][1] * 1.2


# ------------------------------------------------------------------------------------------------------- 8. two GPUs
@pytest.mark.parametrize("weights", ["none", "integer"])
def test_two_gpus_match_one_gpu(km, capfd, weights):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n, d, k = SHAPES["tc"]
    X, _, _ = _blobs(n, d, k, seed=11)
    w = _weights(weights, n, 11)
    kw = {} if w is None else {"sample_weight": w}
    capfd.readouterr()
    c1, a1 = km.kmeans_cuda(X, k, init="k-means||", tolerance=1.0, yinyang_t=0, seed=SEED, device=1, verbosity=1, **kw)
    l1 = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("k-means||")]
    c2, a2 = km.kmeans_cuda(X, k, init="k-means||", tolerance=1.0, yinyang_t=0, seed=SEED, device=3, verbosity=1, **kw)
    l2 = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("k-means||")]
    _check_log(l2, l1)
    assert _same(c1, c2) and np.array_equal(a1, a2)
