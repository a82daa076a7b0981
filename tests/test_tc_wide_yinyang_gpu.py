"""The Yinyang local step (MODE 1) and bounds refresh (MODE 3) on 64-row tiles at 512 < D <= 1024 (assign_tc.cu, NKB
9..16, DESIGN §4k).  Run on an H100: `pytest -m gpu`.

D in {516, 576, 768, 1024} (NKB 9 with a ragged last K-block, 9, 12, 16) unless a test says otherwise.  Covered here:
- whole Yinyang runs, tensor-core local step against the reference-order scan (both with the exact refresh): the same
  iteration lines, assignments and centroids, L2 and cosine;
- Shard.debug_yy_bounds, tensor-core refresh against the exact one: identical upper / own-group bounds and exact-row
  refresh, every other bound valid and within 1e-3;
- rows whose best and second-best centroids sit in the second warpgroup's column half above a lower first-half
  maximum (the emitters' second-best merge);
- whole default calls (yinyang_t = 0.1, adaptive switch on and off) against yinyang_t = 0;
- ragged shapes (N = 1, 100, fewer tiles than SMs, more than two per SM) with a clean pipeline;
- that the MODE 1 and MODE 3 kernels of the 64-row layout ran (torch.profiler).
"""
import os

import numpy as np
import pytest

import tc_sweep_cases as T
from oracle import oracle as O
from test_tc_sweep_gpu import c_kmeans, run_pass
from test_tc_wide_gpu import TR, _blobs, wide_n

pytestmark = pytest.mark.gpu

YY_D = [516, 576, 768, 1024]


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    O.set_threads(os.cpu_count())
    return kmcuda_b200


@pytest.fixture(scope="module")
def lib(km):
    return O.load_c_api(km.LIB_PATH)


@pytest.fixture(scope="module")
def sms(km):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _structureless(n, d, k, seed, metric):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32) if metric == 0 else T.unit(rng.standard_normal((n, d)))
    C0 = X[rng.choice(n, k, replace=False)].copy()
    return np.ascontiguousarray(X, np.float32), C0


def _yy_runs(lib, X, C0, metric, monkeypatch, capfd, tol=1e-3):
    """the same Yinyang run with the tensor-core local step and with the reference-order scan, both refreshing their
    bounds exactly: {force_exact: (C, A, log lines)}"""
    monkeypatch.setenv("KMCUDA_B200_YY_EXACT_REFRESH", "1")
    runs = {}
    for fe in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", fe)
        capfd.readouterr()
        C, A = c_kmeans(lib, X, C0, tol, 0.1, metric, verbosity=1)
        out = capfd.readouterr().out
        runs[fe] = C, A, [ln for ln in out.splitlines() if ln.startswith("iteration") or "refreshing" in ln]
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "0")
    monkeypatch.delenv("KMCUDA_B200_YY_EXACT_REFRESH")
    return runs


def _assert_same_runs(runs):
    assert any("refreshing" in ln for ln in runs["0"][2]) and len(runs["0"][2]) > 3, runs["0"][2]
    assert runs["0"][2] == runs["1"][2]
    assert np.array_equal(runs["0"][1], runs["1"][1]), int((runs["0"][1] != runs["1"][1]).sum())
    np.testing.assert_array_equal(runs["0"][0], runs["1"][0])


# ------------------------------------------------------------------------------------------- MODE 1: whole runs
YY = [(d, 0) for d in YY_D] + [(516, 1), (1024, 1)]


@pytest.mark.parametrize("D,metric", YY, ids=["D%d-%s" % (d, "cos" if m else "L2") for d, m in YY])
def test_wide_yinyang_runs_tc_equal_exact(lib, D, metric, monkeypatch, capfd):
    X, C0 = _structureless(20000, D, 300, D, metric)
    runs = _yy_runs(lib, X, C0, metric, monkeypatch, capfd)
    _assert_same_runs(runs)
    C_last, A_last = runs["0"][:2]
    assert (c_kmeans(lib, X, C_last, 1.0, 0.0, metric)[1] == A_last).mean() > 0.9995


# ------------------------------------------------------------------------------------------- MODE 3: bounds
def _groups(k, G, rng):
    """groups 0-3 with 1, 2, 3 and 5 members, the other centroids spread at random over groups 4 .. G - 1"""
    if G == 1:
        return np.zeros(k, np.uint32)
    fixed = np.repeat(np.arange(4), [1, 2, 3, 5])
    g = np.concatenate([fixed, rng.integers(4, G, k - len(fixed))])
    return g[rng.permutation(k)].astype(np.uint32)


def _bounds_case(n, D, k, seed):
    rng = np.random.default_rng(seed)
    centers = rng.random((k, D), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.1 * rng.standard_normal((n, D), dtype=np.float32)).astype(np.float32)
    C = (centers + 0.02 * rng.standard_normal((k, D), dtype=np.float32)).astype(np.float32)
    return X, C, rng


def _check_bounds(X, C, groups, G, nan_row):
    """tensor-core refresh against the exact one; returns the largest relative slack of the other-group bounds"""
    import torch
    from kmcuda_b200.shard import Shard
    n, D = X.shape
    k = len(C)
    a = run_pass(X, C)[0].astype(np.int32)
    Xt, Ct, at = torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda(), torch.from_numpy(a).cuda()
    sh = Shard(n, D, k)
    bt = sh.debug_yy_bounds(Xt, Ct, at, groups, G, True).cpu().numpy()
    be = sh.debug_yy_bounds(Xt, Ct, at, groups, G, False).cpu().numpy()
    torch.cuda.synchronize()
    assert sh.last_error() == 0
    sh.close()
    an = a.astype(np.uint32)
    ok = an < k
    np.testing.assert_array_equal(bt[ok, 0], be[ok, 0])                                  # upper bound: exact
    own = groups[np.minimum(an, k - 1)]
    rows = np.flatnonzero(ok)
    np.testing.assert_array_equal(bt[rows, 1 + own[rows]], be[rows, 1 + own[rows]])     # own group: exact
    if nan_row is not None:
        np.testing.assert_array_equal(bt[nan_row], be[nan_row])                        # exact row refresh
    lt, le = bt[:, 1:], be[:, 1:]
    finite = np.isfinite(le) & (le < 1e30)
    assert (lt[finite] <= le[finite]).all(), float((lt[finite] - le[finite]).max())
    assert np.array_equal(lt[~finite], le[~finite])                                      # empty groups stay FLT_MAX
    return float(((le[finite] - lt[finite]) / np.maximum(1.0, le[finite])).max()) if finite.any() else 0.0


@pytest.mark.parametrize("G", ["1", "7", "K/4"])
@pytest.mark.parametrize("D", YY_D)
def test_wide_yinyang_refresh_bounds(km, D, G):
    n, k = 20000, 300
    X, C, rng = _bounds_case(n, D, k, D)
    G = {"1": 1, "7": 7, "K/4": k // 4}[G]
    groups = _groups(k, G, rng)
    C[5] = np.nan
    groups[5] = G                                            # dead centroid: no group
    X[11, 3] = np.nan                                        # a row the filter cannot bound -> exact row refresh
    slack = _check_bounds(X, C, groups, G, 11)
    assert slack <= 1e-3, slack


# ------------------------------------------------------------------------------------------- MODE 1: split columns
def _second_half_case(D, seed=0):
    """K = 256 (two n-tiles).  The real centroids sit at columns 64 .. 127 of both n-tiles (the second warpgroup's half);
    columns 0 .. 63 hold decoys far from the uniform rows, each owning a few far rows of its own.  Every uniform row has
    its best and second best in the second half and a lower maximum in the first."""
    rng = np.random.default_rng(seed + D)
    n_main, k = 12000, 256
    second = np.array([c for c in range(k) if c % 128 >= 64])
    first = np.array([c for c in range(k) if c % 128 < 64])
    X_main = rng.random((n_main, D), dtype=np.float32)
    decoy = (3.0 + rng.random((len(first), D), dtype=np.float32)).astype(np.float32)
    X_decoy = np.repeat(decoy, 4, axis=0) + 1e-3 * rng.standard_normal((4 * len(first), D), dtype=np.float32)
    X = np.ascontiguousarray(np.concatenate([X_main, X_decoy]), np.float32)
    C0 = np.zeros((k, D), np.float32)
    C0[second] = X_main[rng.choice(n_main, len(second), replace=False)]
    C0[first] = decoy
    return X, C0, n_main, second


@pytest.mark.parametrize("D", [768, 1024])
def test_wide_yinyang_second_half(lib, D, monkeypatch, capfd):
    X, C0, n_main, second = _second_half_case(D)
    runs = _yy_runs(lib, X, C0, 0, monkeypatch, capfd)
    _assert_same_runs(runs)
    assert np.isin(runs["0"][1][:n_main], second).all()


# ------------------------------------------------------------------------------------------- whole default calls
@pytest.mark.parametrize("adaptive", ["1", "0"])
def test_wide_default_call_same_clustering(km, adaptive, monkeypatch):
    n, d, k = 30000, 768, 1000
    X = _blobs(n, d, k)
    C0 = X[np.random.default_rng(1).choice(n, k, replace=False)].copy()
    kw = dict(init=C0, tolerance=1e-3, device=1, seed=5)
    C_l, A_l = km.kmeans_cuda(X, k, yinyang_t=0.0, **kw)
    monkeypatch.setenv("KMCUDA_B200_YY_ADAPTIVE", adaptive)
    C_y, A_y = km.kmeans_cuda(X, k, yinyang_t=0.1, **kw)
    assert (A_y == A_l).mean() > 0.9999, float((A_y == A_l).mean())
    np.testing.assert_allclose(C_y, C_l, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------- ragged shapes
@pytest.mark.parametrize("nl", ["1", "100", "few", "many"])
def test_wide_yinyang_ragged_refresh(km, sms, nl):
    """MODE 3 with N = 1, 100, fewer 64-row tiles than SMs and more than two per SM"""
    n, D, k = wide_n(nl, sms), 576, 129
    X, C, rng = _bounds_case(max(n, 2), D, k, n)
    X = X[:n]
    G = 13
    groups = _groups(k, G, rng)
    _check_bounds(X, C, groups, G, None)


@pytest.mark.parametrize("nl", ["100", "few", "many"])
def test_wide_yinyang_ragged_runs(lib, sms, nl, monkeypatch, capfd):
    """MODE 1 on survivor lists of every length a run goes through (most rows early, a ragged tile or two late):
    100 rows, fewer 64-row tiles than SMs, more than two per SM.  A pipeline error fails the call."""
    n = wide_n(nl, sms)
    X, C0 = _structureless(n, 576, min(300, n // 2), n, 0)
    runs = _yy_runs(lib, X, C0, 0, monkeypatch, capfd)
    assert runs["0"][2] == runs["1"][2]
    assert np.array_equal(runs["0"][1], runs["1"][1])
    np.testing.assert_array_equal(runs["0"][0], runs["1"][0])


# ------------------------------------------------------------------------------------------- the kernels ran
def test_wide_yinyang_kernels_ran(km, monkeypatch):
    """a silent exact fallback cannot pass: the MODE 1 and MODE 3 kernels of the 64-row layout show up in the trace"""
    from torch.profiler import ProfilerActivity, profile
    X, C0 = _structureless(20000, 768, 300, 3, 0)
    monkeypatch.setenv("KMCUDA_B200_YY_ADAPTIVE", "0")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        km.kmeans_cuda(X, 300, init=C0, tolerance=1e-2, yinyang_t=0.1, device=1)
    names = {e.name for e in prof.events() if "tc_assign" in e.name}
    assert any("tc_assign_kernel<12, 1>" in nm for nm in names), names
    assert any("tc_assign_kernel<12, 3>" in nm for nm in names), names
