"""GPU tests of k-means restarts (kmeans_cuda(..., n_init=, inertia=); include/kmcuda_b200.h
kmcuda_b200_kmeans_restarts, DESIGN.md §4n).

A restart must be exactly a fresh call with its seed: the inertia each restart logs is compared, to the last printed
digit, with the inertia of a separate n_init=1 call with that seed, and the returned run with that call's centroid bits
and assignments.  That catches any state one restart leaves to the next (the Lloyd iteration timing, relocation
records, the angular update's cached sums, Yinyang bounds and tables)."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import restarts_model as M  # noqa: E402

pytestmark = pytest.mark.gpu

RESTART = re.compile(r"restart (\d+)/(\d+): seed (\d+), inertia (\S+)$")
KEPT = re.compile(r"restarts: kept restart (\d+), inertia (\S+)$")


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _out(capfd):
    """what the calls since the last read printed (the library printf's: flush the C stdio buffer first)"""
    ctypes.CDLL(None).fflush(None)
    return capfd.readouterr().out


def _blobs(n, d, k, seed=0, spread=0.6, metric=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if metric == 1:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _duplicated(n, d, distinct, seed=0, metric=0):
    """n rows that repeat `distinct` blob rows: random seeding often draws one row twice, and the second of the two
    centroids then wins no row (an empty cluster for the relocation)"""
    base = _blobs(distinct, d, 20, seed=seed, metric=metric)
    return base[np.random.default_rng(seed + 1).integers(0, distinct, n)].copy()


def _weights(n, seed=2):
    return np.random.default_rng(seed).uniform(0.5, 2, n).astype(np.float32)


def _bits(a):
    return np.asarray(a).view(np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _metric(m):
    return "cos" if m else "L2"


def _logged(lines):
    rs = [m.groups() for m in map(RESTART.match, lines) if m]
    kept = [m.groups() for m in map(KEPT.match, lines) if m]
    return [(int(r), int(n), int(s), e) for r, n, s, e in rs], kept


# ------------------------------------------------------------------------------------------------ 1. n_init=1 = old call
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("variant", ["plain", "weighted", "relocate"])
def test_one_restart_is_the_old_call(km, capfd, metric, variant):
    X = _blobs(20000, 64, 50, metric=metric, spread=3.0 if metric else 0.6)
    w = _weights(len(X)) if variant == "weighted" else None
    kw = dict(init="k-means++", seed=5, device=1, metric=_metric(metric), average_distance=True, sample_weight=w,
              verbosity=1, relocate_empty_clusters=variant == "relocate")
    _out(capfd)
    c0, a0, d0 = km.kmeans_cuda(X, 50, **kw)
    log0 = _out(capfd)
    c1, a1, d1, e1 = km.kmeans_cuda(X, 50, inertia=True, **kw)
    log1 = _out(capfd)
    assert _same(c0, c1) and np.array_equal(a0, a1) and d0 == d1
    assert log0 == log1 and "iteration" in log0 and "restart" not in log1
    assert isinstance(e1, float) and e1 > 0
    np.testing.assert_allclose(e1, M.inertia(X, c1, a1, w, metric), rtol=1e-6)


# ------------------------------------------------------------------------------------------------ 2. restart = fresh call
CASES = {
    # id: (init, metric, yinyang_t, D, weighted, relocate)
    "random-l2-yy-d64": ("random", 0, 0.1, 64, False, False),
    "kmpp-cos-lloyd-d64": ("k-means++", 1, 0.0, 64, False, False),
    "afkmc2-l2-lloyd-d64-w": ("afk-mc2", 0, 0.0, 64, True, False),
    "kmpar-cos-yy-d64-w": ("k-means||", 1, 0.1, 64, True, False),
    "greedy-l2-yy-d768": ("greedy-k-means++", 0, 0.1, 768, False, False),
    "greedy-cos-yy-d30": ("greedy-k-means++", 1, 0.1, 30, False, False),
    "kmpp-l2-yy-d30-w": ("k-means++", 0, 0.1, 30, True, False),
    "random-l2-yy-d64-reloc": ("random", 0, 0.1, 64, False, True),
    "random-cos-lloyd-d30-reloc": ("random", 1, 0.0, 30, False, True),
    "random-l2-lloyd-d768-w-reloc": ("random", 0, 0.0, 768, True, True),
}


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_each_restart_is_a_fresh_call(km, capfd, case):
    init, metric, yy, d, weighted, relocate = CASES[case]
    n, k, R, seed = (8000 if d == 768 else 20000), 50, 4, 0xFFFFFF00 + d   # the schedule wraps around 2^32
    if relocate:
        X = _duplicated(n, d, 400, metric=metric)
    else:
        X = _blobs(n, d, 40, metric=metric, spread=3.0 if metric else 0.6)
    w = _weights(n) if weighted else None
    kw = dict(init=init, tolerance=0.001, yinyang_t=yy, device=1, metric=_metric(metric), sample_weight=w,
              relocate_empty_clusters=relocate, inertia=True, average_distance=True)
    _out(capfd)
    C, a, dist, e = km.kmeans_cuda(X, k, seed=seed, n_init=R, verbosity=1, **kw)
    lines = _out(capfd).splitlines()
    logged, kept = _logged(lines)
    seeds = M.seeds(seed, R)
    assert [(r, nn, s) for r, nn, s, _ in logged] == [(r, R, int(seeds[r])) for r in range(R)]
    if relocate:
        assert any("empty clusters relocated" in ln for ln in lines)
    singles = [km.kmeans_cuda(X, k, seed=int(s), n_init=1, **kw) for s in seeds]
    for (_, _, _, text), (_, _, _, es) in zip(logged, singles):
        assert text == "%.17g" % es
    inertias = [es for _, _, _, es in singles]
    best = M.select(inertias)
    assert kept == [(str(best), "%.17g" % inertias[best])]
    Cb, ab, db, eb = singles[best]
    assert _same(C, Cb) and np.array_equal(a, ab) and dist == db and e == eb


# ------------------------------------------------------------------------------------------------ 3. input forms
def test_fp16_samples_equal_the_widened_fp32_call(km):
    X = _blobs(20000, 64, 40).astype(np.float16)
    kw = dict(init="greedy-k-means++", seed=11, device=1, n_init=3, inertia=True, yinyang_t=0.1)
    C16, a16, e16 = km.kmeans_cuda(X, 40, **kw)
    C32, a32, e32 = km.kmeans_cuda(X.astype(np.float32), 40, **kw)
    assert np.array_equal(a16, a32) and e16 == e32
    assert C16.dtype == np.float16 and np.array_equal(C16, C32.astype(np.float16))


def test_device_pointer_samples_equal_the_host_call(km):
    import torch
    X = _blobs(20000, 64, 40, seed=4)
    kw = dict(init="k-means++", seed=12, device=1, n_init=3, inertia=True, yinyang_t=0.1, average_distance=True)
    Ch, ah, dh, eh = km.kmeans_cuda(X, 40, **kw)
    Xd = torch.from_numpy(X).cuda()
    Cd = torch.empty((40, 64), dtype=torch.float32, device="cuda")
    Ad = torch.empty(len(X), dtype=torch.int32, device="cuda")
    cp, ap, dd, ed = km.kmeans_cuda((Xd.data_ptr(), 0, X.shape, Cd.data_ptr(), Ad.data_ptr()), 40, **kw)
    torch.cuda.synchronize()
    assert (cp, ap) == (Cd.data_ptr(), Ad.data_ptr())
    assert _same(Cd.cpu().numpy(), Ch) and np.array_equal(Ad.cpu().numpy().view(np.uint32), ah)
    assert dd == dh and ed == eh


# ------------------------------------------------------------------------------------------------ 4. rows that add nothing
@pytest.mark.parametrize("metric", [0, 1])
def test_nan_and_zero_weight_rows_add_nothing(km, metric):
    X = _blobs(20000, 64, 40, seed=6, metric=metric, spread=3.0 if metric else 0.6)
    X[17] = np.nan
    w = _weights(len(X), seed=7)
    w[::97] = 0
    C, a, e = km.kmeans_cuda(X, 40, init="k-means++", seed=13, device=1, n_init=2, inertia=True,
                             metric=_metric(metric), sample_weight=w)
    assert np.isfinite(e)
    np.testing.assert_allclose(e, M.inertia(X, C, a, w, metric), rtol=1e-6)


# ------------------------------------------------------------------------------------------------ 5. two GPUs
def test_two_gpus_equal_the_separate_calls(km):
    if km.device_count() < 2:
        pytest.skip("needs two GPUs")
    X = _blobs(40000, 64, 40, seed=8)
    kw = dict(init="greedy-k-means++", device=3, inertia=True, yinyang_t=0.1, average_distance=True)
    C, a, dist, e = km.kmeans_cuda(X, 40, seed=21, n_init=3, **kw)
    singles = [km.kmeans_cuda(X, 40, seed=int(s), n_init=1, **kw) for s in M.seeds(21, 3)]
    Cb, ab, db, eb = singles[M.select([s[3] for s in singles])]
    assert _same(C, Cb) and np.array_equal(a, ab) and dist == db and e == eb


# ------------------------------------------------------------------------------------------------ 6. quality
def test_restarts_keep_the_lowest_inertia_and_match_scikit_learn(km, capfd):
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(9)
    centers = rng.uniform(0, 10, (60, 8))
    X = (centers[rng.integers(0, 60, 30000)] + 0.7 * rng.standard_normal((30000, 8))).astype(np.float32)
    _out(capfd)
    C, a, e = km.kmeans_cuda(X, 30, init="greedy-k-means++", seed=17, device=1, n_init=8, inertia=True,
                             tolerance=0.0, yinyang_t=0, verbosity=1)
    logged, _ = _logged(_out(capfd).splitlines())
    inertias = [float(t) for _, _, _, t in logged]
    assert len(inertias) == 8 and len(set(inertias)) > 1, "every seeding reached the same minimum"
    assert e == min(inertias)
    np.testing.assert_allclose(e, M.inertia(X, C, a), rtol=1e-6)
    sk = KMeans(n_clusters=30, init="k-means++", n_init=8, random_state=0).fit(X.astype(np.float64))
    assert e <= 1.02 * sk.inertia_, (e, sk.inertia_)
