"""GPU tests of per-sample weights (kmcuda_b200_kmeans_weighted / kmeans_cuda(..., sample_weight=...)).

The rule that pins the design: with every weight 1.0 a weighted call is bit-identical to the unweighted one (centroids,
assignments, the per-iteration log, the seeding picks, average_distance).  Beyond that the weighted update is checked
against duplicated rows, float64, scikit-learn and zero weights.  Each property runs on a shape that takes the
tensor-core assignment path (D % 4 == 0) and one that takes the exact SIMT path (D = 30)."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import cases  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {"tc": (50000, 64, 200), "exact": (20000, 30, 50)}


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
    C0 = X[rng.choice(n, k, replace=False)].copy()
    return X, C0


def _run(km, capfd, X, k, init, **kw):
    capfd.readouterr()
    out = km.kmeans_cuda(X, k, init=init, device=1, seed=7, verbosity=1, average_distance=True, **kw)
    log = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("iteration")]
    return out, log


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


# ------------------------------------------------------------------------------------------------ 1. all-ones weights
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("metric", ["L2", "cos"])
@pytest.mark.parametrize("yy", [0.0, 0.1])
@pytest.mark.parametrize("init", ["import", "k-means++", "afkmc2", "random"])
def test_all_ones_weights_are_bit_identical_to_unweighted(km, capfd, shape, metric, yy, init):
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=1, cos=metric == "cos")
    init_arg = C0 if init == "import" else init
    (c0, a0, avg0), log0 = _run(km, capfd, X, k, init_arg, metric=metric, yinyang_t=yy, tolerance=0.01)
    (c1, a1, avg1), log1 = _run(km, capfd, X, k, init_arg, metric=metric, yinyang_t=yy, tolerance=0.01,
                                sample_weight=np.ones(n, np.float32))
    assert len(log0) >= 2 and log0 == log1
    assert _same(c0, c1) and np.array_equal(a0, a1)
    assert _same(np.float32(avg0), np.float32(avg1))


@pytest.mark.parametrize("shape", list(SHAPES))
def test_weighted_entry_point_with_null_weights_is_kmeans_cuda(km, shape):
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=2)
    outs = []
    for fn in ("kmeans_cuda", "weighted"):
        C = C0.copy()
        A = np.zeros(n, np.uint32)
        avg = ctypes.c_float(0)
        args = [3, None, 0.01, 0.1, 0, n, d, k, 3, 1, -1, 0, 0, X.ctypes.data]
        if fn == "weighted":
            rc = km._lib.kmcuda_b200_kmeans_weighted(*args, None, C.ctypes.data, A.ctypes.data, ctypes.byref(avg))
        else:
            rc = km._lib.kmeans_cuda(*args, C.ctypes.data, A.ctypes.data, ctypes.byref(avg))
        assert rc == 0
        outs.append((C, A, avg.value))
    assert _same(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2]


# ------------------------------------------------------------------------------------- 2. integer weights = duplicates
def _tie_exempt(X, C, rel=1e-6):
    """rows whose fp64 best and second-best squared distances are within `rel` of each other"""
    X64, C64 = X.astype(np.float64), C.astype(np.float64)
    d2 = (X64 ** 2).sum(1)[:, None] - 2 * X64 @ C64.T + (C64 ** 2).sum(1)[None]
    part = np.partition(d2, 1, axis=1)
    return (part[:, 1] - part[:, 0]) <= rel * np.maximum(np.abs(part[:, 1]), 1e-30)


def _close(a, b, rtol):
    scale = np.abs(b).max(1, keepdims=True)
    return (np.abs(a - b) <= rtol * scale).all()


@pytest.mark.parametrize("shape", list(SHAPES))
def test_integer_weights_equal_duplicated_rows_after_one_update(km, shape):
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=3, spread=2.0)
    w = np.random.default_rng(3).integers(1, 4, n)
    Xd = np.repeat(X, w, axis=0)
    cw, aw = km.kmeans_cuda(X, k, init=C0, tolerance=0.99, yinyang_t=0, device=1, sample_weight=w)
    cd, ad = km.kmeans_cuda(Xd, k, init=C0, tolerance=0.99, yinyang_t=0, device=1)
    assert _close(cw, cd, 1e-6)
    first = np.concatenate([[0], np.cumsum(w)[:-1]])
    for r in range(3):   # every copy of a row
        sel = w > r
        mism = (aw[sel] != ad[first[sel] + r]) & ~_tie_exempt(X[sel], cd)
        assert mism.sum() == 0


@pytest.mark.parametrize("yy", [0.0, 0.1])
def test_integer_weights_equal_duplicated_rows_whole_runs(km, yy):
    for n, d, k in [(30000, 64, 40), (20000, 30, 25)]:
        rng = np.random.default_rng(4)
        centers = rng.standard_normal((k, d)).astype(np.float32) * 3
        label = np.arange(n) % k                          # well separated blobs, one initial centroid in each
        X = (centers[label] + 0.3 * rng.standard_normal((n, d))).astype(np.float32)
        C0 = X[:k].copy()
        w = rng.integers(1, 4, n)
        Xd = np.repeat(X, w, axis=0)
        _, aw = km.kmeans_cuda(X, k, init=C0, tolerance=0.0, yinyang_t=yy, device=1, sample_weight=w)
        _, ad = km.kmeans_cuda(Xd, k, init=C0, tolerance=0.0, yinyang_t=yy, device=1)
        assert np.array_equal(np.repeat(aw, w), ad)


# ------------------------------------------------------------------------------------------- 3. real weights, float64
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_lognormal_weights_first_update_matches_float64(km, shape, metric):
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=5, spread=2.0, cos=metric == "cos")
    w = np.random.default_rng(5).lognormal(0.0, 1.0, n).astype(np.float32)
    c, _ = km.kmeans_cuda(X, k, init=C0, tolerance=0.99, yinyang_t=0, metric=metric, device=1, sample_weight=w)
    a1 = O.assign_lloyd(X, C0, metric=1 if metric == "cos" else 0)[0]   # the pass the update was computed from
    S = np.zeros((k, d))
    np.add.at(S, a1, w[:, None].astype(np.float64) * X)
    if metric == "L2":
        W = np.bincount(a1, weights=w.astype(np.float64), minlength=k)
        ref = S / W[:, None]
    else:
        ref = S / np.linalg.norm(S, axis=1, keepdims=True)
    assert _close(c, ref, 1e-5)


# -------------------------------------------------------------------------------------------------- 4. scikit-learn
def test_final_labels_match_scikit_learn(km):
    sk = pytest.importorskip("sklearn.cluster")
    X = cases.blobs()
    rng = np.random.default_rng(6)
    C0 = X[[0, 2000, 4000, 6000, 8000, 10000]].copy()   # one row of each of the six blobs
    w = rng.lognormal(0.0, 0.5, len(X)).astype(np.float32)
    _, a = km.kmeans_cuda(X, 6, init=C0, tolerance=0.0, yinyang_t=0, device=1, sample_weight=w)
    ref = sk.KMeans(6, init=C0.astype(np.float64), n_init=1, algorithm="lloyd", tol=0, max_iter=1000)
    ref.fit(X.astype(np.float64), sample_weight=w.astype(np.float64))
    assert np.array_equal(a, ref.labels_.astype(np.uint32))


# -------------------------------------------------------------------------------------------------- 5. zero weights
@pytest.mark.parametrize("shape", list(SHAPES))
def test_zero_weight_rows_do_not_move_centroids(km, shape):
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=8, spread=2.0)
    m = 777
    far = (1000.0 + np.random.default_rng(8).standard_normal((m, d))).astype(np.float32)
    Xa = np.concatenate([X, far])
    wa = np.concatenate([np.ones(n, np.float32), np.zeros(m, np.float32)])
    c0, a0 = km.kmeans_cuda(X, k, init=C0, tolerance=0.99, yinyang_t=0, device=1)
    c1, a1 = km.kmeans_cuda(Xa, k, init=C0, tolerance=0.99, yinyang_t=0, device=1, sample_weight=wa)
    assert _close(c1, c0, 1e-6)
    assert np.array_equal(a1[:n], a0)
    assert np.array_equal(a1, O.assign_lloyd(Xa, c1)[0])   # zero-weight rows are still assigned (argmin)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("init", ["k-means++", "afkmc2", "random"])
def test_seeding_never_picks_a_zero_weight_row(km, shape, init):
    n, d, k = SHAPES[shape]
    X, _ = _blobs(n, d, k, seed=9)
    w = np.random.default_rng(9).lognormal(0.0, 1.0, n).astype(np.float32)
    w[np.random.default_rng(10).random(n) < 0.4] = 0
    w[:n // 10] = 0                                     # and a solid run of zeros at the start
    c, _ = km.kmeans_cuda(X, k, init=init, tolerance=1.0, yinyang_t=0, device=1, seed=11, sample_weight=w)
    rows = {X[i].tobytes(): i for i in range(n)}
    picked = [rows[row.tobytes()] for row in c]
    assert (w[picked] > 0).all()


# ----------------------------------------------------------------------------------------------------- 6. validation
def test_invalid_weights_are_rejected(km, monkeypatch):
    X, C0 = _blobs(5000, 16, 10, seed=12)
    for bad in (np.nan, np.inf, -1.0):
        w = np.ones(5000, np.float32)
        w[1234] = bad
        with pytest.raises(ValueError):
            km.kmeans_cuda(X, 10, init=C0, device=1, sample_weight=w)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, init=C0, device=1, sample_weight=np.zeros(5000, np.float32))
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, init=C0, device=1, sample_weight=np.ones(5000, np.float32))


# ------------------------------------------------------------------------------------------ 7. device pointers, fp16
@pytest.mark.parametrize("shape", list(SHAPES))
def test_device_pointer_weights_equal_host_weights(km, shape):
    import torch
    n, d, k = SHAPES[shape]
    X, C0 = _blobs(n, d, k, seed=13)
    w = np.random.default_rng(13).lognormal(0.0, 1.0, n).astype(np.float32)
    ch, ah, avgh = km.kmeans_cuda(X, k, init=C0, tolerance=0.01, yinyang_t=0.1, device=1, average_distance=True,
                                  sample_weight=w)
    Xt, wt = torch.from_numpy(X).cuda(), torch.from_numpy(w).cuda()
    cp, ap, avgd = km.kmeans_cuda((Xt.data_ptr(), 0, X.shape), k, init=C0, tolerance=0.01, yinyang_t=0.1, device=1,
                                  average_distance=True, sample_weight=wt.data_ptr())
    cd = np.empty((k, d), np.float32)
    ad = np.empty(n, np.uint32)
    km._cuda_memcpy_d2h(0, cd.ctypes.data, cp, cd.nbytes)
    km._cuda_memcpy_d2h(0, ad.ctypes.data, ap, ad.nbytes)
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    assert _same(ch, cd) and np.array_equal(ah, ad) and avgh == avgd


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fp16_samples_with_weights_equal_fp32_on_the_widened_samples(km, shape):
    n, d, k = SHAPES[shape]
    X, _ = _blobs(n, d, k, seed=14)
    X16 = X.astype(np.float16)
    w = np.random.default_rng(14).lognormal(0.0, 1.0, n).astype(np.float32)
    c16, a16 = km.kmeans_cuda(X16, k, init="k-means++", seed=5, tolerance=0.01, yinyang_t=0, device=1,
                              sample_weight=w)
    c32, a32 = km.kmeans_cuda(X16.astype(np.float32), k, init="k-means++", seed=5, tolerance=0.01, yinyang_t=0,
                              device=1, sample_weight=w)
    assert c16.dtype == np.float16
    assert np.array_equal(a16, a32)
    assert np.array_equal(c16.view(np.uint16), c32.astype(np.float16).view(np.uint16))


# ------------------------------------------------------------------------------------------------------- 8. two GPUs
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_two_gpus_weighted_match_one_gpu(km, monkeypatch, exchange):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    if exchange == "nccl":
        monkeypatch.setenv("KMCUDA_B200_EXCHANGE", "nccl")
    n, d, k = SHAPES["tc"]
    X, C0 = _blobs(n, d, k, seed=15, spread=2.0)
    w = np.random.default_rng(15).lognormal(0.0, 1.0, n).astype(np.float32)
    _, a1 = km.kmeans_cuda(X, k, init=C0, tolerance=1.0, yinyang_t=0, device=1, sample_weight=w)
    _, a2 = km.kmeans_cuda(X, k, init=C0, tolerance=1.0, yinyang_t=0, device=3, sample_weight=w)
    assert np.array_equal(a1, a2)
    c1, a1 = km.kmeans_cuda(X, k, init=C0, tolerance=0.99, yinyang_t=0, device=1, sample_weight=w)
    c2, a2 = km.kmeans_cuda(X, k, init=C0, tolerance=0.99, yinyang_t=0, device=3, sample_weight=w)
    assert _close(c2, c1, 1e-5)
    assert (a1 != a2).mean() < 1e-4
    _, a1 = km.kmeans_cuda(X, k, init=C0, tolerance=0.001, yinyang_t=0.1, device=1, sample_weight=w)
    _, a2 = km.kmeans_cuda(X, k, init=C0, tolerance=0.001, yinyang_t=0.1, device=3, sample_weight=w)
    assert (a1 == a2).mean() > 0.98
