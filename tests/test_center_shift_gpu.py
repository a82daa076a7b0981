"""GPU tests of scikit-learn's stopping rule (kmeans_cuda(..., tol=, max_iter=, n_iter=True); include/kmcuda_b200.h
kmcuda_b200_kmeans_center_shift, DESIGN.md §4p).

- tol = 0 with a large max_iter stops where tolerance = 0 stops, bit for bit, on every route.
- The library is pinned to tests/center_shift_model.py with the oracle's argmin as labels: every stop reason on the
  tensor-core route (D = 256), the 64-row-tile route (D = 768) and the exact route (D = 13, 1100).  The tolerance is
  chosen so that no model shift lies within a factor 2 of it, so fp32 rounding cannot flip a decision unseen.
- Against scikit-learn, the cap, non-finite data, device-pointer and fp16 input, restarts and two GPUs."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import center_shift_model as M  # noqa: E402

pytestmark = pytest.mark.gpu

ITER = re.compile(r"iteration (\d+): (\d+) reassignments$")
STOP = re.compile(r"stopped at iteration (\d+): (.+)$")
RESTART = re.compile(r"restart (\d+)/(\d+): seed (\d+), inertia (\S+)$")


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _out(capfd):
    ctypes.CDLL(None).fflush(None)
    return capfd.readouterr().out


def _iters(out):
    return [ln for ln in out.splitlines() if ITER.match(ln)]


def _stop(out):
    s = [STOP.match(ln).groups() for ln in out.splitlines() if STOP.match(ln)]
    assert len(s) == 1, out[-2000:]
    return int(s[0][0]), s[0][1]


def _blobs(n, d, k, seed=0, spread=0.6, metric=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if metric == 1:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _bits(a):
    return np.asarray(a).view(np.uint32)


# ------------------------------------------------------------------------------------------------ 1. tol = 0 equivalence
EQUIV = [  # (metric, yinyang_t, adaptive, weights, relocate, n_init)
    (0, 0.0, True, False, False, 1),
    (1, 0.0, True, False, False, 1),
    (0, 0.1, False, False, False, 1),
    (1, 0.1, False, False, False, 1),
    (0, 0.1, True, False, False, 1),
    (0, 0.1, False, True, False, 1),
    (0, 0.0, True, False, True, 1),
    (0, 0.1, False, True, True, 3),
    (1, 0.1, True, False, False, 3),
]


@pytest.mark.parametrize("metric,yy,adaptive,weighted,reloc,n_init", EQUIV)
def test_tol_zero_is_tolerance_zero(km, capfd, monkeypatch, metric, yy, adaptive, weighted, reloc, n_init):
    if not adaptive:
        monkeypatch.setenv("KMCUDA_B200_YY_ADAPTIVE", "0")
    X = _blobs(60000, 64, 40, seed=7, spread=1.2, metric=metric)
    if reloc:   # repeated rows: random seeding draws one twice and its second copy is relocated
        X = X[np.random.default_rng(8).integers(0, 300, len(X))].copy()
    w = np.random.default_rng(9).uniform(0.5, 2, len(X)).astype(np.float32) if weighted else None
    kw = dict(init="k-means++" if not reloc else "random", seed=11, yinyang_t=yy, metric="cos" if metric else "L2",
              device=1, verbosity=1, sample_weight=w, relocate_empty_clusters=reloc, n_init=n_init, inertia=True)
    _out(capfd)
    Ca, Aa, ea = km.kmeans_cuda(X, 40, tolerance=0.0, **kw)
    ref = _out(capfd)
    Cb, Ab, eb, it = km.kmeans_cuda(X, 40, tol=0, max_iter=10_000, n_iter=True, **kw)
    new = _out(capfd)
    assert np.array_equal(_bits(Ca), _bits(Cb))
    assert np.array_equal(Aa, Ab)
    assert ea == eb
    assert _iters(ref) == _iters(new)
    if n_init == 1:
        at, why = _stop(new)
        assert at == it and why in ("equal labels", "tolerance")
        if yy == 0:   # (Yinyang's grouping is a nested run with iteration lines of its own)
            assert len(_iters(new)) == it + (why == "tolerance")


# ------------------------------------------------------------------------------------------------ 2. pinned to the model
def _oracle_labeler(metric=0):
    from oracle import oracle as O
    return lambda X, C: O.assign_lloyd(X, C, metric)[0].astype(np.int64)


def _pick_tol(shifts, var_mean):
    """a tol whose tol_abs stops the run at a shift S_j > 0 with every shift up to S_j more than 2x away from it"""
    for j in range(1, len(shifts)):
        t = np.sqrt(shifts[j - 1] * shifts[j])
        if shifts[j] > 0 and all(s > 2 * t for s in shifts[:j]) and shifts[j] < t / 2:
            return float(t / var_mean)
    pytest.fail("no shift sequence with a 4x gap: %r" % (shifts,))


PIN = [(256, 64), (768, 32), (13, 32), (1100, 16)]


@pytest.mark.parametrize("D,K", PIN)
@pytest.mark.parametrize("reason", M.REASONS)
def test_pinned_to_model(km, capfd, D, K, reason):
    n = 20000 if D <= 256 else 8000
    X = _blobs(n, D, K, seed=D)
    C0 = X[np.random.default_rng(1).choice(n, K, replace=False)].copy()
    lab = _oracle_labeler()
    free = M.run(X, C0, lab, 0.0, max_iter=10_000)
    var_mean = M.tolerance_abs(X, 1.0)
    if reason == "equal labels":
        tol, max_iter = 0.0, 10_000
    elif reason == "tolerance":
        tol, max_iter = _pick_tol(free["shifts"], var_mean), 10_000
    else:
        assert free["n_iter"] >= 2, free["n_iter"]
        tol, max_iter = 0.0, free["n_iter"] - 1
    m = M.run(X, C0, lab, tol, max_iter=max_iter)
    assert m["reason"] == reason
    for s in m["shifts"]:
        assert not (m["tol_abs"] / 2 <= s <= 2 * m["tol_abs"]) or m["tol_abs"] == 0, (s, m["tol_abs"])
    _out(capfd)
    C, A, it = km.kmeans_cuda(X, K, init=C0, yinyang_t=0, tol=tol, max_iter=max_iter, n_iter=True, device=1,
                              verbosity=1)
    out = _out(capfd)
    assert it == m["n_iter"]
    assert _stop(out) == (m["n_iter"], reason)
    assert [int(ITER.match(ln).group(2)) for ln in _iters(out)] == m["passes"]
    assert np.array_equal(A.astype(np.int64), m["labels"])
    scale = max(1.0, float(np.nanmax(np.abs(m["C"]))))   # dead clusters keep NaN centroids in both
    np.testing.assert_allclose(C, m["C"], rtol=1e-5, atol=1e-5 * scale)


# ------------------------------------------------------------------------------------------------ 3. scikit-learn
@pytest.mark.parametrize("tol,max_iter", [(1e-4, 300), (0.0, 300), (1e-2, 300), (0.0, 3)])
def test_against_scikit_learn(km, tol, max_iter):
    KMeans = pytest.importorskip("sklearn.cluster").KMeans
    rng = np.random.default_rng(21)
    centers = rng.standard_normal((20, 32)) * 3
    X = (centers[rng.integers(0, 20, 50000)] + rng.standard_normal((50000, 32))).astype(np.float32)
    C0 = (centers + 0.5 * rng.standard_normal((20, 32))).astype(np.float32)
    C, A, e, it = km.kmeans_cuda(X, 20, init=C0, yinyang_t=0, tol=tol, max_iter=max_iter, n_iter=True, inertia=True,
                                 device=1)
    sk = KMeans(20, init=C0.astype(np.float64), n_init=1, algorithm="lloyd", tol=tol, max_iter=max_iter).fit(
        X.astype(np.float64))
    assert it == sk.n_iter_
    assert np.array_equal(A, sk.labels_)
    assert e == pytest.approx(sk.inertia_, rel=1e-5)


# ------------------------------------------------------------------------------------------------ 4. the cap
@pytest.mark.parametrize("yy", [0.0, 0.1])
@pytest.mark.parametrize("max_iter", [1, 2])
def test_cap(km, capfd, yy, max_iter):
    X = np.random.default_rng(3).random((30000, 24), dtype=np.float32)
    _out(capfd)
    _, _, it = km.kmeans_cuda(X, 64, init="random", seed=5, yinyang_t=yy, tol=0, max_iter=max_iter, n_iter=True,
                              device=1, verbosity=1)
    out = _out(capfd)
    assert it == max_iter
    assert len(_iters(out)) == max_iter + 1
    assert _stop(out) == (max_iter, "max_iter")


# ------------------------------------------------------------------------------------------------ 5. non-finite data
def test_nan_row_stops_on_max_iter(km, capfd):
    X = np.random.default_rng(4).random((20000, 16), dtype=np.float32)
    X[123, 5] = np.nan
    _out(capfd)
    _, _, it = km.kmeans_cuda(X, 50, init="random", seed=1, yinyang_t=0, tol=1e-4, max_iter=4, n_iter=True,
                              device=1, verbosity=1)
    out = _out(capfd)
    assert "center shift tolerance: nan" in out.lower()
    assert (it, "max_iter") == _stop(out)


def test_dead_cluster_does_not_block_tolerance(km, capfd):
    X = _blobs(20000, 16, 8, seed=5)
    C0 = X[np.random.default_rng(6).choice(len(X), 9, replace=False)].copy()
    C0[8] = 50.0   # wins no row: its centroid turns NaN after the first update
    _out(capfd)
    C, _, it = km.kmeans_cuda(X, 9, init=C0, yinyang_t=0, tol=1e-3, n_iter=True, device=1, verbosity=1)
    out = _out(capfd)
    assert np.isnan(C[8]).all()
    assert _stop(out)[1] in ("tolerance", "equal labels") and it < 300


# ------------------------------------------------------------------------------------------------ 6. other inputs
def test_device_pointers_and_fp16_equal_host_fp32(km):
    import torch
    X = _blobs(40000, 32, 16, seed=12)
    kw = dict(init="k-means++", seed=3, yinyang_t=0.1, tol=1e-4, n_iter=True, device=1)
    C, A, it = km.kmeans_cuda(X, 16, **kw)
    Xd = torch.from_numpy(X).cuda()
    Cd, Ad, itd = km.kmeans_cuda((Xd.data_ptr(), 0, tuple(Xd.shape)), 16, **kw)
    hc = np.empty_like(C)
    ha = np.empty_like(A)
    km._cuda_memcpy_d2h(0, hc.ctypes.data, Cd, hc.nbytes)
    km._cuda_memcpy_d2h(0, ha.ctypes.data, Ad, ha.nbytes)
    km._cuda_free(0, Cd)
    km._cuda_free(0, Ad)
    assert itd == it and np.array_equal(_bits(hc), _bits(C)) and np.array_equal(ha, A)
    Xh = X.astype(np.float16)
    Ch, Ah, ith = km.kmeans_cuda(Xh, 16, **kw)
    Cf, Af, itf = km.kmeans_cuda(Xh.astype(np.float32), 16, **kw)
    assert ith == itf and np.array_equal(Ah, Af)
    assert np.array_equal(Ch, Cf.astype(np.float16))


# ------------------------------------------------------------------------------------------------ 7. restarts
def test_each_restart_is_a_fresh_call(km, capfd):
    X = _blobs(30000, 32, 24, seed=13, spread=1.5)
    kw = dict(init="k-means++", yinyang_t=0.1, tol=1e-4, max_iter=50, device=1, inertia=True, n_iter=True)
    _out(capfd)
    C, A, e, it = km.kmeans_cuda(X, 24, seed=17, n_init=3, verbosity=1, **kw)
    lines = _out(capfd).splitlines()
    rs = [RESTART.match(ln).groups() for ln in lines if RESTART.match(ln)]
    assert len(rs) == 3
    fresh = []
    for r, _, s, er in rs:
        Cr, Ar, e1, it1 = km.kmeans_cuda(X, 24, seed=int(s), **kw)
        assert "%.17g" % e1 == er
        fresh.append((e1, it1, Cr, Ar))
    best = min(range(3), key=lambda r: (fresh[r][0], r))
    assert e == fresh[best][0] and it == fresh[best][1]
    assert np.array_equal(_bits(C), _bits(fresh[best][2])) and np.array_equal(A, fresh[best][3])


# ------------------------------------------------------------------------------------------------ 8. two GPUs
@pytest.mark.parametrize("yy", [0.0, 0.1])
def test_two_gpus_equal_one(km, yy):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    X = _blobs(100000, 64, 32, seed=14, spread=1.5)
    kw = dict(init="k-means++", seed=9, yinyang_t=yy, tol=1e-4, n_iter=True)
    C1, A1, it1 = km.kmeans_cuda(X, 32, device=1, **kw)
    C2, A2, it2 = km.kmeans_cuda(X, 32, device=3, **kw)
    assert it1 == it2 and np.array_equal(A1, A2)
    np.testing.assert_allclose(C2, C1, rtol=1e-5, atol=1e-5)
