"""GPU tests of the AFK-MC² seeding (init="afkmc2" / ("afkmc2", m); Job::init_afkmc2 in seeding.cu, DESIGN.md §4f).

The seeding is pinned to its NumPy model (tests/afkmc2_model.py): the init centroids, read from a tolerance=1.0 call
that stops after the first assignment pass without touching them, are bit-identical to the model's, and the logged c0
is the model's.  Angular cases first check that no decision of the model lies within 1e-6 (relative) of flipping, as
the host's acosf and the device's may differ by an ulp; the seed is the first from a fixed start that passes.  Shapes
cover D % 4 == 0 (D = 64, and D = 768 where the run takes 64-row tensor-core tiles), D % 4 != 0 and D > 1024; chains
of 1, 7, 200 (the default) and N / 2 candidates (angular: 1 and 7); no, integer, lognormal and 30 %-zero weights; fp16
samples; the restart seed schedule across 2^32; fewer distinct rows than clusters; rows with a NaN feature, which must
never be drawn."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import afkmc2_model as A  # noqa: E402
import restarts_model as RM  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {"d64": (4000, 64, 40), "d768": (1500, 768, 12), "d67": (3000, 67, 30), "d1100": (1200, 1100, 10)}
SEED = 7
C0 = re.compile(r"afkmc2: calculating q \(c0 = (\d+)\)")
KEPT = re.compile(r"restarts: kept restart (\d+), inertia (\S+)")


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


def _blobs(n, d, k, seed=0, spread=0.6, cos=False):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if cos:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _weights(kind, n, seed):
    """integer and lognormal weights sum exactly in double, in any order, so the device's total is the model's"""
    rng = np.random.default_rng(seed)
    if kind == "none":
        return None
    if kind == "lognormal":
        return rng.lognormal(0, 1, n).astype(np.float32)
    w = rng.integers(1, 5, n).astype(np.float32)
    if kind == "zeros":
        w[rng.random(n) < 0.3] = 0
    return w


def _init(km, capfd, X, k, m=None, **kw):
    """init centroids (tolerance=1.0 returns them untouched) and the logged c0 of every seeding"""
    _out(capfd)
    kw.setdefault("seed", SEED)
    init = "afkmc2" if m is None else ("afkmc2", m)
    c, _ = km.kmeans_cuda(X, k, init=init, tolerance=1.0, yinyang_t=0, device=1, verbosity=2, **kw)
    return c, [int(v) for v in C0.findall(_out(capfd))]


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _where_they_part(c, r, X):
    """the first centroid where the device left the model, with the model's step for it"""
    for k in range(len(r.rows)):
        if not np.array_equal(np.asarray(c[k]).view(np.uint32), X[r.rows[k]].view(np.uint32)):
            same = np.nonzero((X.view(np.uint32) == np.asarray(c[k]).view(np.uint32)).all(axis=1))[0]
            if k == 0:
                return "c0: device row %s, model row %d" % (same[:3].tolist(), r.rows[0])
            s = r.trace[k - 1]
            inside = [int(j) for j in np.nonzero(np.isin(s.cand, same))[0]][:5]
            return ("centroid %d: device row %s (chain slots %s), model row %d; model accepted slots %s"
                    % (k, same[:3].tolist(), inside, r.rows[k], np.nonzero(s.accepted)[0][-5:].tolist()))
    return "no centroid differs"


def _pinned(X, k, metric, m=0, w=None, start=SEED):
    """(seed, model) for the first seed from `start` whose seeding the model pins: c0 has no NaN feature (c0 is only
    redrawn on an x[0] NaN) and, angular, no draw or chain decision lies within 1e-6 (relative) of flipping.  Angular
    chains stay short: over thousands of draws some draw always comes closer than that to a CDF boundary."""
    for seed in range(start, start + 20):
        r = A.afkmc2(X, k, seed, m=m, w=w, metric=1 if metric == "cos" else 0)
        if np.isnan(X[r.c0]).any():
            continue
        if metric == "cos" and not (r.margin_draw > 1e-6 and r.margin_accept > 1e-6):
            continue
        return seed, r
    pytest.fail("no seed in [%d, %d) gives a clean c0 and margins above 1e-6" % (start, start + 20))


def _check(c, c0s, r, X):
    assert c0s == [r.c0]
    assert _same(c, r.C), _where_they_part(c, r, X)


# ------------------------------------------------------------------------------------------------ 1. model equality
CASES = [(shape, metric, weights, m) for shape in SHAPES
         for metric, weights, m in (("L2", "integer", 0), ("cos", "zeros", 7))]
CASES += [("d64", "L2", weights, m) for m in (1, 7, "half") for weights in ("none", "lognormal")]
CASES += [("d67", "cos", "lognormal", 7), ("d1100", "L2", "none", "half"), ("d768", "L2", "zeros", 1),
          ("d64", "cos", "none", 1), ("d1100", "cos", "lognormal", 1), ("d67", "L2", "lognormal", "half")]


@pytest.mark.parametrize("shape,metric,weights,m", CASES)
def test_seeding_matches_the_model(km, capfd, shape, metric, weights, m):
    n, d, k = SHAPES[shape]
    m = n // 2 if m == "half" else m
    X = _blobs(n, d, k, seed=1, cos=metric == "cos")
    w = _weights(weights, n, 2)
    seed, r = _pinned(X, k, metric, m=m, w=w)
    kw = {} if w is None else {"sample_weight": w}
    c, c0s = _init(km, capfd, X, k, m=m or None, metric=metric, seed=seed, **kw)
    _check(c, c0s, r, X)


def test_a_chain_longer_than_half_the_samples_is_refused(km):
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=1)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, k, init=("afkmc2", n // 2 + 1), tolerance=1.0, yinyang_t=0, seed=SEED, device=1)


# ------------------------------------------------------------------------------------------------------ 2. edge cases
def test_fp16_samples_equal_the_model_on_the_widened_values(km, capfd):
    n, d, k = SHAPES["d64"]
    X16 = _blobs(n, d, k, seed=6).astype(np.float16)
    c16, c0s = _init(km, capfd, X16, k)
    r = A.afkmc2(X16.astype(np.float32), k, SEED)
    assert c0s == [r.c0]
    assert np.array_equal(c16.view(np.uint16), r.C.astype(np.float16).view(np.uint16))


def test_restart_seeds_wrap_into_the_generator(km, capfd):
    """n_init=3 at seed 0xFFFFFFF0: restart r seeds with (seed + r * 0x9E3779B9) mod 2^32, which must reach
    std::mt19937_64 wrapped; each restart's seeding is read from a tolerance=1.0 call at its own seed"""
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=9)
    seed = 0xFFFFFFF0
    seeds = [int(s) for s in RM.seeds(seed, 3)]
    assert seeds[1] < seed and seeds[2] < seed
    _out(capfd)
    C, _, _ = km.kmeans_cuda(X, k, init="afkmc2", tolerance=1.0, yinyang_t=0, seed=seed, device=1, n_init=3,
                             inertia=True, verbosity=2)
    out = _out(capfd)
    kept = [int(g[1]) for g in KEPT.finditer(out)]
    models = [A.afkmc2(X, k, s) for s in seeds]
    assert [int(v) for v in C0.findall(out)] == [r.c0 for r in models]
    for s, r in zip(seeds, models):
        c, c0s = _init(km, capfd, X, k, seed=s)
        assert c0s == [r.c0] and _same(c, r.C), (s, _where_they_part(c, r, X))
    assert len(kept) == 1 and _same(C, models[kept[0]].C)


def test_fewer_distinct_rows_than_clusters(km, capfd):
    """once every distinct row is a centroid, p = 0 for every candidate and each chain takes its last one"""
    base = np.random.default_rng(8).standard_normal((4, 30)).astype(np.float32)
    X = np.repeat(base, [5000, 1, 1, 1], axis=0)
    c, c0s = _init(km, capfd, X, 20)
    r = A.afkmc2(X, 20, SEED)
    _check(c, c0s, r, X)
    assert len(set(map(bytes, c))) == 4
    flat = [s for s in r.trace if (s.p == 0).all()]
    assert flat and all(s.chosen == s.cand[-1] for s in flat)


@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_rows_with_a_nan_feature_never_become_centroids(km, capfd, metric):
    """2 % of the rows carry a NaN: 40 in feature 0 (plusplus_kernel gives them distance 0 in k-means++), 40 in feature
    5 (a NaN distance).  A drawn NaN row has no finite distance to any centroid, p = +inf, and a chain that meets one
    takes it; with q = 0 on those rows none is ever drawn.  L2 runs the default chain of 200, angular one of 7 (see
    _pinned)."""
    n, d, k = SHAPES["d64"]
    X = _blobs(n, d, k, seed=13, cos=metric == "cos")
    rng = np.random.default_rng(14)
    pool = np.setdiff1d(np.arange(n), [0, n // 2, n - 1])   # (the angular probe rows stay unit length)
    rows = rng.choice(pool, 80, replace=False)
    X[rows[:40], 0] = np.nan
    X[rows[40:], 5] = np.nan
    m = 0 if metric == "L2" else 7
    seed, r = _pinned(X, k, metric, m=m, start=21)
    c, c0s = _init(km, capfd, X, k, m=m or None, metric=metric, seed=seed)
    bad = int(np.isnan(c).any(axis=1).sum())
    assert bad == 0, "%d of %d centroids are NaN" % (bad, k)
    _check(c, c0s, r, X)
