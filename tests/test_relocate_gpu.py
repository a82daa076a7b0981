"""GPU tests of the empty-cluster relocation (kmeans_cuda(..., relocate_empty_clusters=True);
include/kmcuda_b200.h kmcuda_b200_kmeans_relocate, DESIGN.md §4l).

Runs are pinned to the NumPy model (tests/relocate_model.py) with the oracle's argmin as labels: centroids to 1e-5,
assignments and the relocation log lines exactly.  Every pinned L2 case first checks that the same call without
relocation leaves a NaN centroid, so the test exercises what it claims to."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import relocate_model as R  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

SUMMARY = re.compile(r"iteration (\d+): (\d+) empty clusters relocated(?:, (\d+) left empty)?$")
DETAIL = re.compile(r"relocated cluster (\d+): sample (\d+), key (\S+), donor (\d+)$")


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _blobs(n, d, k, seed=0, spread=0.6, metric=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    if metric == 1:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _init_with_empties(X, k, n_far, seed=1, metric=0):
    """k rows of X, the last n_far of them moved far from every sample (they win no row in the first pass)"""
    C = X[np.random.default_rng(seed).choice(len(X), k, replace=False)].copy()
    far = -C[:n_far] if metric == 1 else C[:n_far] + 1e3
    C[k - n_far:] = far
    return C


def _run(km, capfd, X, k, C0, metric=0, **kw):
    capfd.readouterr()
    kw.setdefault("tolerance", 0.0)
    kw.setdefault("yinyang_t", 0)
    out = km.kmeans_cuda(X, k, init=C0, device=1, verbosity=2, metric="cos" if metric else "L2", seed=3, **kw)
    return out, capfd.readouterr().out.splitlines()


def _log(lines):
    """[(iteration, relocated, left, [(cluster, sample, key, donor)])] from the library's log"""
    out = []
    for ln in lines:
        m = SUMMARY.match(ln)
        if m:
            out.append((int(m.group(1)), int(m.group(2)), int(m.group(3) or 0), []))
            continue
        m = DETAIL.match(ln)
        if m:
            out[-1][3].append((int(m.group(1)), int(m.group(2)), float(m.group(3)), int(m.group(4))))
    return out


def _model_log(mlog):
    return [(it, len(rec), left, rec) for it, _, rec, left in mlog if rec or left]


def _labeler(metric):
    return lambda X, C: O.assign_lloyd(X, C, metric)[0].astype(np.int64)


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _check_against_model(got_log, mlog, C, mC, a, ma):
    g, m = _log(got_log), _model_log(mlog)
    assert [x[:3] for x in g] == [x[:3] for x in m]
    for (_, _, _, gr), (_, _, _, mr) in zip(g, m):
        assert [(c, s, dn) for c, s, _, dn in gr] == [(c, s, dn) for c, s, _, dn in mr]
        for (_, _, gk, _), (_, _, mk, _) in zip(gr, mr):
            assert abs(gk - mk) <= 1e-4 * abs(mk) + 1e-6
    scale = max(1.0, float(np.nanmax(np.abs(mC))))
    np.testing.assert_allclose(C, mC, rtol=1e-5, atol=1e-5 * scale)
    assert np.array_equal(a.astype(np.int64), ma)


# ------------------------------------------------------------------------------------------------ 1. off = plain call
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("weighted", [False, True])
def test_off_is_bit_identical_to_the_plain_call(km, metric, weighted):
    X = _blobs(20000, 64, 50, metric=metric)
    C0 = _init_with_empties(X, 50, 3, metric=metric)
    w = np.random.default_rng(2).uniform(0.5, 2, len(X)).astype(np.float32) if weighted else None
    c1, a1 = km.kmeans_cuda(X, 50, init=C0, device=1, metric="cos" if metric else "L2", sample_weight=w, seed=3)
    c2, a2 = km.kmeans_cuda(X, 50, init=C0, device=1, metric="cos" if metric else "L2", sample_weight=w, seed=3,
                            relocate_empty_clusters=False)
    assert _same(c1, c2) and np.array_equal(a1, a2)


# ------------------------------------------------------------------------------------------------ 2. model pin
SHAPES = [(20000, 64, 60), (20000, 256, 60), (8000, 768, 40), (20000, 30, 60)]   # tensor core, 64-row tiles, exact


@pytest.mark.parametrize("shape", SHAPES, ids=["d64", "d256", "d768", "d30_exact"])
@pytest.mark.parametrize("metric", [0, 1])
def test_run_matches_the_model(km, capfd, shape, metric):
    n, d, k = shape
    X = _blobs(n, d, k, metric=metric)
    C0 = _init_with_empties(X, k, 4, metric=metric)
    (cp, _), _ = _run(km, capfd, X, k, C0, metric)
    if metric == 0:
        assert np.isnan(cp).any()
    (C, a), lines = _run(km, capfd, X, k, C0, metric, relocate_empty_clusters=True)
    assert not np.isnan(C).any()
    mC, ma, mlog = R.run(X, C0, _labeler(metric), metric=metric)
    _check_against_model(lines, mlog, C, mC, a, ma)
    assert any(rec for _, _, rec, _ in mlog)


def test_fp16_samples_match_the_model(km, capfd):
    """fp16x2 samples are widened on ingest: the run equals the fp32 run on the widened values (imported centroids
    travel as packed halves in fp16 mode)"""
    X = _blobs(20000, 64, 60).astype(np.float16)
    Xw = X.astype(np.float32)
    C0 = _init_with_empties(Xw, 60, 4).astype(np.float16)
    (C, a), lines = _run(km, capfd, X, 60, C0.view(np.float32), relocate_empty_clusters=True)
    (Cw, aw), lw = _run(km, capfd, Xw, 60, C0.astype(np.float32), relocate_empty_clusters=True)
    assert np.array_equal(a, aw) and _log(lines) == _log(lw) and _log(lw)
    assert np.array_equal(C.view(np.uint16), Cw.astype(np.float16).view(np.uint16))
    mC, ma, mlog = R.run(Xw, C0.astype(np.float32), _labeler(0))
    _check_against_model(lw, mlog, Cw, mC, aw, ma)


def test_imported_nan_rows_are_relocated_at_the_first_update(km, capfd):
    X = _blobs(20000, 64, 40)
    C0 = _init_with_empties(X, 40, 2)
    C0[5] = np.nan
    C0[17] = np.nan
    (C, a), lines = _run(km, capfd, X, 40, C0, relocate_empty_clusters=True)
    g = _log(lines)
    assert g[0][0] == 1 and sorted(c for c, _, _, _ in g[0][3]) == [5, 17, 38, 39]
    assert not np.isnan(C).any()


# ------------------------------------------------------------------------------------------------ 3. weights
def test_all_ones_weights_are_bit_identical(km, capfd):
    X = _blobs(20000, 64, 50)
    C0 = _init_with_empties(X, 50, 3)
    (c1, a1), l1 = _run(km, capfd, X, 50, C0, relocate_empty_clusters=True)
    (c2, a2), l2 = _run(km, capfd, X, 50, C0, relocate_empty_clusters=True, sample_weight=np.ones(len(X)))
    assert _same(c1, c2) and np.array_equal(a1, a2) and _log(l1) == _log(l2) and _log(l1)


def test_zero_weight_rows_are_never_taken(km, capfd):
    X = _blobs(20000, 64, 50)
    X[[10, 20, 30]] += 40                       # the farthest rows, of weight 0
    w = np.random.default_rng(4).uniform(0.5, 2, len(X)).astype(np.float32)
    w[[10, 20, 30]] = 0
    C0 = _init_with_empties(X, 50, 3)
    (C, a), lines = _run(km, capfd, X, 50, C0, relocate_empty_clusters=True, sample_weight=w)
    taken = [s for it in _log(lines) for _, s, _, _ in it[3]]
    assert taken and not {10, 20, 30} & set(taken)
    mC, ma, mlog = R.run(X, C0, _labeler(0), w=w)
    _check_against_model(lines, mlog, C, mC, a, ma)


def test_the_walk_protects_a_donor_and_logs_clusters_left_empty(km, capfd):
    rng = np.random.default_rng(6)
    X = (rng.standard_normal((4000, 32)) * 0.1).astype(np.float32)
    X[:2000, 0] += 10                            # two tight blobs, two centroids, four far ones
    C0 = np.vstack([X[:2000].mean(0), X[2000:].mean(0), np.full((4, 32), 1e3, np.float32) + np.arange(4)[:, None]])
    C0 = C0.astype(np.float32)
    # one more cluster holding a single far row: the walk may not take its only member
    X = np.vstack([X, np.full((1, 32), 60, np.float32)])
    C0 = np.vstack([C0, np.full((1, 32), 55, np.float32)])
    (C, a), lines = _run(km, capfd, X, 7, C0, relocate_empty_clusters=True)
    g = _log(lines)
    assert all(s != len(X) - 1 for _, s, _, _ in g[0][3])
    mC, ma, mlog = R.run(X, C0, _labeler(0))
    _check_against_model(lines, mlog, C, mC, a, ma)
    # more empty clusters than rows that may go (NaN rows have no centroid): the rest stay NaN and are logged
    Xs = np.zeros((6, 32), np.float32)
    Xs[1, 0], Xs[2, 0], Xs[3, 0] = 1, 5, 6
    Xs[4:] = np.nan
    C1 = np.vstack([Xs[:2].mean(0), Xs[2:4].mean(0), np.full((4, 32), 1e3, np.float32)]).astype(np.float32)
    (C, a), lines = _run(km, capfd, Xs, 6, C1, relocate_empty_clusters=True)
    g = _log(lines)
    assert g[0][1] == 2 and g[0][2] == 2, lines
    assert np.isnan(C).any()


def test_duplicate_far_rows_go_lowest_index_first(km, capfd):
    X = _blobs(20000, 64, 50)
    X[[900, 300, 600]] = X[100] + 30
    C0 = _init_with_empties(X, 50, 2)
    (C, a), lines = _run(km, capfd, X, 50, C0, relocate_empty_clusters=True)
    assert [s for _, s, _, _ in _log(lines)[0][3]] == [300, 600]


# ------------------------------------------------------------------------------------------------ 4. selection at scale
@pytest.mark.parametrize("m", [1, 17, 1000])
def test_selection_at_scale_equals_a_stable_sort(km, m):
    import torch
    n, d, K = 2_000_000, 32, 1000
    g = torch.Generator(device="cuda").manual_seed(m)
    X = torch.randn(n, d, device="cuda", generator=g)
    C = torch.randn(K, d, device="cuda", generator=g)
    a = torch.randint(0, K, (n,), device="cuda", generator=g, dtype=torch.int32)
    a[::97] = K                                   # rows without a centroid are not eligible
    T = 2 * m + 32
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    top = torch.empty(T, dtype=torch.int64, device="cuda")
    f = km._lib.kmcuda_b200_debug_relocate_select
    f.restype = ctypes.c_int64
    f.argtypes = [ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint16] + [ctypes.c_void_p] * 2 + \
        [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
    torch.cuda.synchronize()
    elig = f(0, n, d, X.data_ptr(), C.data_ptr(), K, a.data_ptr(), None, T, keys.data_ptr(), top.data_ptr())
    kh = keys.cpu().numpy().view(np.uint64)
    assert elig == int((kh != 0).sum()) == n - len(range(0, n, 97))
    hi = (kh >> np.uint64(32)).astype(np.uint32)
    dist = np.where(hi & 0x80000000, hi & 0x7FFFFFFF, ~hi).astype(np.uint32).view(np.float32)
    row = np.arange(n)
    ok = kh != 0
    order = row[ok][np.lexsort((row[ok], -dist[ok].astype(np.float64)))][:T]
    got = ~(top.cpu().numpy().view(np.uint64).astype(np.uint32))
    assert np.array_equal(got.astype(np.int64), order)
    # the keys are the exact squared distances of the inertia pass
    ref = ((X[:1000] - C[a[:1000].clamp(max=K - 1).long()]) ** 2).sum(1).cpu().numpy()
    np.testing.assert_allclose(dist[:1000][ok[:1000]], ref[ok[:1000]], rtol=1e-5)


# ------------------------------------------------------------------------------------------------ 5. Yinyang
def test_yinyang_relocation_after_the_bounds_exist(km, capfd):
    """Two far init centroids take two identical far rows at the first update; both then sit on the same point, the
    second pass gives the rows to the lower index, and the other cluster empties again in the first Yinyang iteration."""
    n, d, k = 60000, 64, 100
    rng = np.random.default_rng(9)
    centers = rng.standard_normal((k - 2, d)).astype(np.float32) * 6
    X = (centers[rng.integers(0, k - 2, n)] + 0.3 * rng.standard_normal((n, d))).astype(np.float32)
    X[[123, 4567]] = centers[0] + 40
    C0 = np.vstack([centers, np.full((2, d), 1e3, np.float32)]).astype(np.float32)
    (c1, a1), l1 = _run(km, capfd, X, k, C0, yinyang_t=0.1, relocate_empty_clusters=True)
    (c0, a0), l0 = _run(km, capfd, X, k, C0, yinyang_t=0, relocate_empty_clusters=True)
    first = next(i for i, ln in enumerate(l1) if ln.startswith("refreshing Yinyang bounds"))
    assert any(SUMMARY.match(ln) for ln in l1[first:]), l1
    assert _same(c1, c0) and np.array_equal(a1, a0)


# ------------------------------------------------------------------------------------------------ 6. quality
def test_quality_against_scikit_learn_and_lloyd(km):
    """The data and init of tests/test_minibatch_gpu.py's quality test (50000 x 64 @ 200 blobs, 200 rows as init).
    Full-data inertia of the relocating Lloyd run against the plain Lloyd run and scikit-learn's KMeans from the same
    centroids (algorithm="lloyd", tol=0).  Measured on an H100 80GB HBM3 at 700 W: 0.9768 x the plain Lloyd run (which
    keeps the init's empty clusters as NaN) and 1.0000 x scikit-learn.  Bounds: <= the plain run, 1.01 x scikit-learn."""
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(0)
    n, d, k = 50000, 64, 200
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + 0.6 * rng.standard_normal((n, d))).astype(np.float32)
    C0 = X[np.random.default_rng(1).choice(len(X), k, replace=False)].copy()
    CR, aR = km.kmeans_cuda(X, k, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3, relocate_empty_clusters=True)
    CL, aL = km.kmeans_cuda(X, k, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3)
    assert not np.isnan(CR).any()
    mine = float(((X.astype(np.float64) - CR[aR]) ** 2).sum())
    lloyd = float(np.nansum((X.astype(np.float64) - CL[aL]) ** 2))
    sk = KMeans(n_clusters=k, init=C0, n_init=1, algorithm="lloyd", tol=0.0).fit(X)
    sk_inertia = float(((X.astype(np.float64) - sk.cluster_centers_[sk.labels_]) ** 2).sum())
    print("relocating Lloyd / plain Lloyd = %.4f, relocating Lloyd / scikit-learn = %.4f" % (mine / lloyd,
                                                                                            mine / sk_inertia))
    assert mine <= lloyd
    assert mine <= 1.01 * sk_inertia


# ------------------------------------------------------------------------------------------------ 7. two GPUs
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_two_gpus_take_the_same_rows(km, capfd, monkeypatch, exchange):
    if km.device_count() < 2:
        pytest.skip("needs two GPUs")
    if exchange == "nccl":
        monkeypatch.setenv("KMCUDA_B200_EXCHANGE", "nccl")
    X = _blobs(40000, 64, 60)
    C0 = _init_with_empties(X, 60, 5)
    (c1, a1), l1 = _run(km, capfd, X, 60, C0, relocate_empty_clusters=True)
    capfd.readouterr()
    c2, a2 = km.kmeans_cuda(X, 60, init=C0, device=3, verbosity=2, tolerance=0.0, yinyang_t=0, seed=3,
                            relocate_empty_clusters=True)
    l2 = capfd.readouterr().out.splitlines()
    g1, g2 = _log(l1), _log(l2)
    assert [[(c, s, dn) for c, s, _, dn in x[3]] for x in g1] == [[(c, s, dn) for c, s, _, dn in x[3]] for x in g2]
    assert not np.isnan(c2).any()


# ------------------------------------------------------------------------------------------------ 8. arguments
def test_rejected_arguments(km, monkeypatch):
    X = _blobs(2000, 16, 10)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, batch_size=256, device=1, relocate_empty_clusters=True)
    with pytest.raises(TypeError):
        km.kmeans_cuda(X, 10, device=1, relocate_empty_clusters=1)
    with pytest.raises(TypeError):
        km.kmeans_cuda(X, 10, device=1, relocate_empty_clusters="yes")
    C = np.zeros((10, 16), np.float32)
    A = np.zeros(2000, np.uint32)
    lib = km._lib
    args = (1, None, ctypes.c_float(0.01), ctypes.c_float(0.0), 0, 2000, 16, 10, 3, 1, -1, 0, 0, X.ctypes.data)
    assert lib.kmcuda_b200_kmeans_relocate(*args, None, C.ctypes.data, A.ctypes.data, None) == km.SUCCESS
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    assert lib.kmcuda_b200_kmeans_relocate(*args, None, C.ctypes.data, A.ctypes.data, None) == km.INVALID_ARGUMENTS
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, device=1, relocate_empty_clusters=True)


def test_cpython_module_takes_the_argument(km, capfd):
    sys.path.insert(0, os.path.dirname(km.LIB_PATH))
    import libKMCUDA
    X = _blobs(20000, 64, 50)
    C0 = _init_with_empties(X, 50, 3)
    c1, a1 = libKMCUDA.kmeans_cuda(X, 50, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3,
                                   relocate_empty_clusters=True)
    c2, a2 = km.kmeans_cuda(X, 50, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3, relocate_empty_clusters=True)
    assert _same(c1, c2) and np.array_equal(a1, a2)
    with pytest.raises(TypeError):
        libKMCUDA.kmeans_cuda(X, 50, device=1, relocate_empty_clusters=1)
    with pytest.raises(ValueError):
        libKMCUDA.kmeans_cuda(X, 50, device=1, batch_size=100, relocate_empty_clusters=True)
