"""Round-2 GPU parity tests: the gaps VERDICT r01 named, all through the C ABI and all against the UNMODIFIED
reference library (oracle/_ref) or scikit-learn (the reference's own pins, src/test.py).

  * centroid update vs the reference itself (rtol 1e-5) and the oracle's `adjust` pinned to it
  * per-iteration log of whole runs next to the reference (first differing iteration is reported)
  * 8M x 256 @ 1024: the full output of one pass equal to the exact pass's, a fixed row sample to the reference's
  * angular k-NN, k = 50, C5-shaped k-NN against sklearn on a query subset
  * the pipeline error word surfaces as kmcudaRuntimeError; outliers far beyond the sentinel score
  * `import libKMCUDA` (the CPython entry of the same .so) running a real clustering
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import cases  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
IMPORT = 3


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


@pytest.fixture(scope="module")
def ours(km):
    return O.load_c_api(km.LIB_PATH)


@pytest.fixture(scope="module")
def ref():
    if not O.reference_available():
        pytest.skip("oracle/_ref/libKMCUDA.so not built")
    return O.reference_lib()


def c_kmeans(lib, X, C0, tol, yy, metric=0, verbosity=0, device=1):
    X = np.ascontiguousarray(X)
    N, D = X.shape
    K = C0.shape[0]
    C = np.array(C0, copy=True, order="C")
    A = np.zeros(N, np.uint32)
    m = ctypes.c_uint32(0)
    rc = lib.kmeans_cuda(IMPORT, ctypes.byref(m), tol, yy, metric, N, D, K, 3, device, -1, 0, verbosity,
                         X.ctypes.data, C.ctypes.data, A.ctypes.data, None)
    assert rc == 0, rc
    return C, A


def _unit(a):
    return (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)


def _tie_exempt(X, C, rows, metric=0, rel=1e-6):
    """rows whose best and second-best float64 distances differ by less than `rel` (SURVEY.md 8c)"""
    Xd, Cd = X[rows].astype(np.float64), C.astype(np.float64)
    if metric == 0:
        d = (Cd ** 2).sum(1)[None, :] - 2 * Xd @ Cd.T + (Xd ** 2).sum(1)[:, None]
    else:
        d = np.arccos(np.clip(Xd @ Cd.T, -1, 1))
    part = np.partition(d, 1, axis=1)
    return (part[:, 1] - part[:, 0]) <= rel * np.maximum(1.0, np.abs(part[:, 1]))


# ------------------------------------------------------------------------------------------- (a) update
@pytest.mark.parametrize("n,d,k,metric", [(100000, 256, 1024, 0), (60000, 128, 300, 1), (30011, 100, 77, 0)])
def test_update_matches_reference_library(ours, ref, n, d, k, metric):
    """assign -> update -> assign (tolerance 0.99, reference src/test.py:512-519 trick): centroids after ONE update
    within 1e-5 relative of the reference's (north_star), second-pass assignments equal (fp64 near-ties exempt)"""
    rng = np.random.default_rng(n + d)
    X = rng.random((n, d), dtype=np.float32) if metric == 0 else _unit(rng.standard_normal((n, d)))
    C0 = X[rng.choice(n, k, replace=False)].copy()
    Co, Ao = c_kmeans(ours, X, C0, 0.99, 0.0, metric)
    Cr, Ar = c_kmeans(ref, X, C0, 0.99, 0.0, metric)
    ok = ~np.isnan(Cr).any(1)
    assert ok.sum() >= k - 2 and np.array_equal(np.isnan(Co).any(1), ~ok)
    scale = np.abs(Cr[ok]).max(1, keepdims=True)      # relative to the centroid's largest coordinate
    assert (np.abs(Co[ok] - Cr[ok]) / scale).max() < 1e-5
    diff = np.flatnonzero(Ao != Ar)
    if len(diff):
        assert len(diff) < 1e-4 * n
        assert _tie_exempt(X, Cr[ok], diff, metric, rel=1e-5).all()


def test_oracle_adjust_pinned_to_reference(ref):
    """oracle/kmcuda_oracle.c::ko_adjust (restating src/kmeans.cu:366-429) == the reference kernel, bit for bit"""
    rng = np.random.default_rng(12)
    X = rng.random((20000, 64), dtype=np.float32)
    C0 = X[:100].copy()
    a, prev, _ = O.assign_lloyd(X, C0)
    Cexp, cnt = O.adjust(X, C0, prev, a, np.zeros(100, np.uint32))
    Cr, Ar = c_kmeans(ref, X, C0, 0.99, 0.0)
    np.testing.assert_array_equal(Cr, Cexp)
    a2, _, _ = O.assign_lloyd(X, Cexp)
    np.testing.assert_array_equal(Ar, a2)


# ------------------------------------------------------------------------------------------- (b) whole runs
def _iteration_log(lib, X, C0, tol, yy, capfd, metric=0):
    capfd.readouterr()
    C, A = c_kmeans(lib, X, C0, tol, yy, metric, verbosity=1)
    out = capfd.readouterr().out
    return [int(ln.split(":")[1].split()[0]) for ln in out.splitlines() if ln.startswith("iteration")], C, A


def test_whole_run_next_to_reference_c1(ours, ref, capfd):
    """C1 (100 000 x 256 @ 1024, U[0,1), Lloyd to 0.2 %): per-iteration reassignment counts of both libraries.
    The assignment step is bit-identical; the update differs in the last ulps (this library: sorted compensated
    sums; reference: running sum in sample order with one compensation term shared by all features), so on
    structureless data near-tie samples flip after a few iterations and the trajectories separate.  The test pins
    what IS guaranteed: identical first iterations, counts that stay close, and a result of the same quality."""
    rng = np.random.default_rng(777)
    X = rng.random((100000, 256), dtype=np.float32)
    C0 = X[rng.choice(len(X), 1024, replace=False)].copy()
    lo, Co, Ao = _iteration_log(ours, X, C0, 0.002, 0.0, capfd)
    lr, Cr, Ar = _iteration_log(ref, X, C0, 0.002, 0.0, capfd)
    first_diff = next((i for i, (a, b) in enumerate(zip(lo, lr)) if a != b), min(len(lo), len(lr)))
    print("ours", lo)
    print("ref ", lr)
    print("first differing iteration:", first_diff + 1)
    assert lo[0] == lr[0] == len(X)
    assert first_diff >= 1                       # iteration 1 is the same pass on the same centroids; from iteration 2
                                                 # on a handful of near-tie samples may flip (measured: 29181 vs 29180)
    assert abs(len(lo) - len(lr)) <= 3
    for a, b in zip(lo, lr):
        assert abs(a - b) <= 0.02 * len(X)
    # same objective to 1e-4 relative
    def inertia(C, A):
        ok = ~np.isnan(C).any(1)
        return float(((X.astype(np.float64) - C[A].astype(np.float64)) ** 2).sum())
    assert abs(inertia(Co, Ao) - inertia(Cr, Ar)) < 2e-4 * inertia(Cr, Ar)


# ------------------------------------------------------------------------------------------- (c) 8M one pass
def test_headline_8m_one_pass_equals_reference(ours, monkeypatch):
    """BASELINE configs[1] shape, full output: every one of the 8 000 000 assignments of the tensor-core pass equals
    the exact pass's (the reference's arithmetic restated), and the rows of a fixed sample equal the reference
    library's own assignments, stored in golden/headline_8m.npz (golden/make_golden.py --headline)"""
    X, C0 = cases.headline_8m()
    expected = np.load(os.path.join(HERE, "golden", "headline_8m.npz"))["assign"].astype(np.uint32)
    rows = cases.headline_rows()
    _, Ao = c_kmeans(ours, X, C0, 1.0, 0.0)
    assert np.array_equal(Ao[rows], expected), int((Ao[rows] != expected).sum())
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1")
    _, Ae = c_kmeans(ours, X, C0, 1.0, 0.0)
    assert np.array_equal(Ao, Ae), int((Ao != Ae).sum())


# ------------------------------------------------------------------------------------------- robustness
def test_far_outliers_and_dead_centroids(ours, ref):
    """ADVICE r01: rows whose every score lies below the -65504 sentinel of padded / dead centroid columns (an
    outlier far away and opposite to all centroids, K % 128 != 0, a NaN centroid) must take the exact pass"""
    rng = np.random.default_rng(3)
    n, d, k = 5000, 64, 200                      # 200 % 128 != 0: 56 padded columns
    X = (1.0 + 0.05 * rng.standard_normal((n, d))).astype(np.float32)
    C = (1.0 + 0.05 * rng.standard_normal((k, d))).astype(np.float32)
    C[17] = np.nan
    X[3] = -40.0
    X[77] = -900.0
    X[1234] = 3000.0
    X[99, :] = 0.0
    for lib_metric in (0,):
        _, Ao = c_kmeans(ours, X, C, 1.0, 0.0, lib_metric)
        _, Ar = c_kmeans(ref, X, C, 1.0, 0.0, lib_metric)
        assert np.array_equal(Ao, Ar), np.flatnonzero(Ao != Ar)[:10]
        assert not (Ao == 17).any() and Ao.max() < k


@pytest.mark.parametrize("offset", [3.0, 100.0])
def test_offset_data_is_exact(km, offset):
    """data far from the origin relative to its spread.  The centred operands keep the fp16 scores precise, but the
    REFERENCE's own fp32 ranking score ||c||^2 - 2 x.c then lives at ~offset^2 * D with an ulp comparable to the
    distance gaps, so a bit-identical filter must (and does) hand the rows it cannot separate from that noise to the
    exact kernels: the result has to equal the oracle either way."""
    import torch
    from kmcuda_b200.shard import assign_once
    rng = np.random.default_rng(8)
    X = (offset + rng.random((50000, 128))).astype(np.float32)
    C = X[rng.choice(len(X), 512, replace=False)].copy()
    a, _, _, info = assign_once(torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda())
    assert info[0]
    print("offset %.0f: re-checked %d, full exact pass %d of %d rows" % (offset, info[1], info[2], len(X)))
    if offset <= 3.0:
        assert info[2] < len(X) // 10
    exp = O.assign_lloyd(X, C)[0]
    assert np.array_equal(a.cpu().numpy().astype(np.uint32), exp)


def test_unaligned_centroid_pointer_is_rejected(km):
    """ADVICE r01: a centroid pointer that is not 16-byte aligned must give an error code, not a fault"""
    import torch
    from kmcuda_b200.shard import Shard
    n, d, k = 4096, 64, 64
    X = torch.rand((n, d), device="cuda")
    Cbig = torch.rand((k * d + 1,), device="cuda")
    C = Cbig[1:].view(k, d)                      # 4-byte aligned only
    assert C.data_ptr() % 16 != 0
    sh = Shard(n, d, k)
    a = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    with pytest.raises(Exception):
        sh.assign(X, C, a, a.clone(), torch.zeros(1, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()                     # the context is still alive
    sh.assign(X, Cbig[:k * d].view(k, d), a, a.clone(), torch.zeros(1, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- k-NN
def _knn(lib, k, X, C, A, metric=0, device=1):
    out = np.zeros((len(X), k), np.uint32)
    rc = lib.knn_cuda(k, metric, X.shape[0], X.shape[1], C.shape[0], device, -1, 0, 0, X.ctypes.data, C.ctypes.data,
                      A.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    return out


def test_knn_k50_blobs_matches_sklearn(km):
    """reference src/test.py:608-609: k = 50 on the blobs, at most 2 differing entries vs sklearn"""
    from sklearn.neighbors import NearestNeighbors
    X = cases.blobs()
    cent, asg = km.kmeans_cuda(X, 50, init="k-means++", device=1, seed=777, yinyang_t=0)
    nb = km.knn_cuda(50, X, cent, asg, device=1)
    exp = NearestNeighbors(n_neighbors=51, algorithm="brute").fit(X).kneighbors(X, return_distance=False)[:, 1:]
    diff = nb != exp.astype(np.uint32)
    rows = np.unique(np.argwhere(diff)[:, 0])
    bad = 0
    for r in rows:                               # exact distance ties may swap places
        dg = np.sort(np.linalg.norm(X[nb[r]].astype(np.float64) - X[r], axis=1))
        de = np.sort(np.linalg.norm(X[exp[r]].astype(np.float64) - X[r], axis=1))
        bad += not np.allclose(dg, de, atol=1e-7)
    assert bad <= 2, bad


def test_knn_angular_matches_reference_and_bruteforce(ours, ref):
    """reference src/test.py:735-745 (cosine k-NN): same neighbours as the reference library up to angle ties, and
    as a float64 brute force on a query sample"""
    rng = np.random.default_rng(31)
    n, d, kc, k = 20000, 48, 100, 10
    X = _unit(rng.standard_normal((n, d)) + 2.0 * rng.standard_normal((1, d)))
    C0 = X[rng.choice(n, kc, replace=False)].copy()
    C, A = c_kmeans(ref, X, C0, 0.05, 0.0, metric=1)
    got = _knn(ours, k, X, C, A, metric=1)
    exp = _knn(ref, k, X, C, A, metric=1)
    assert (got != exp).mean() < 2e-3, (got != exp).mean()
    qs = rng.choice(n, 300, replace=False)
    Xd = X.astype(np.float64)
    bad = 0
    for q in qs:
        ang = np.arccos(np.clip(Xd @ Xd[q], -1, 1))
        ang[q] = np.inf
        order = np.argsort(ang, kind="stable")[:k + 1]
        if abs(ang[order[k]] - ang[order[k - 1]]) < 1e-6:
            continue
        got_ang = np.sort(np.arccos(np.clip(Xd[got[q]] @ Xd[q], -1, 1)))
        bad += not np.allclose(got_ang, np.sort(ang[order[:k]]), atol=2e-4)   # acosf resolution near 0
    assert bad == 0, bad


def test_knn_c5_shape_vs_sklearn_subset(ours, ref):
    """BASELINE configs[4] shape scaled to what the reference library finishes in seconds: clustered data,
    k = 10; full output equal to the reference (ties aside) and equal to sklearn brute force on 10 000 queries"""
    from sklearn.neighbors import NearestNeighbors
    rng = np.random.default_rng(55)
    n, d, kc, k = 300000, 256, 100, 10
    centers = rng.random((kc, d), dtype=np.float32)
    X = (centers[rng.integers(0, kc, n)] + 0.05 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    C, A = c_kmeans(ours, X, centers, 0.01, 0.0)
    got = _knn(ours, k, X, C, A)
    exp = _knn(ref, k, X, C, A)
    assert (got != exp).mean() < 1e-4, (got != exp).mean()
    qs = rng.choice(n, 10000, replace=False)
    nn = NearestNeighbors(n_neighbors=k + 1, algorithm="brute").fit(X)
    dist, idx = nn.kneighbors(X[qs])
    bad = 0
    for j, q in enumerate(qs):
        e = idx[j][idx[j] != q][:k]
        if set(got[q].tolist()) != set(e.tolist()):
            # sklearn works in float64 on ||x||^2 - 2xy + ||y||^2: accept differences at fp32 distance ties only
            dg = np.sort(np.linalg.norm(X[got[q]].astype(np.float64) - X[q], axis=1))
            de = np.sort(np.linalg.norm(X[e].astype(np.float64) - X[q], axis=1))
            bad += not np.allclose(dg, de, rtol=1e-6)
    assert bad == 0, bad


# ------------------------------------------------------------------------------------------- CPython entry
def test_import_libkmcuda_runs_a_clustering(km):
    """`import libKMCUDA` (PyInit_libKMCUDA of the SAME shared object, reference python.cc:33) in a fresh
    interpreter: k-means + k-NN on the blobs, validated like the reference's own test (src/test.py:176-183)"""
    code = r'''
import sys, numpy as np
sys.path.insert(0, %r); sys.path.insert(0, %r)
import cases
import libKMCUDA
X = cases.blobs()
cent, asg = libKMCUDA.kmeans_cuda(X, 50, init="k-means++", device=1, seed=3, tolerance=0.01, yinyang_t=0.1)
assert cent.shape == (50, 2) and asg.dtype == np.uint32 and asg.shape == (13000,)
d = ((X[:, None, :].astype(np.float64) - cent[None].astype(np.float64)) ** 2).sum(-1)
assert (d.argmin(1) != asg).mean() < 0.01
nb = libKMCUDA.knn_cuda(10, X, cent, asg, device=1)
assert nb.shape == (13000, 10) and libKMCUDA.supports_fp16
print("IMPORT_OK")
''' % (os.path.dirname(km.LIB_PATH), os.path.join(HERE, "golden"))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=300)
    assert "IMPORT_OK" in r.stdout, r.stdout[-800:]


# ------------------------------------------------------------------------------------------- >= 2 GPUs
def _ngpu():
    import torch
    return torch.cuda.device_count()


def test_multi_gpu_single_process_matches_one_gpu(ours):
    """device mask 0x3 vs 0x1 (reference README.md:126-131): one assignment pass is identical, one update agrees
    to 1e-5 (different summation order), k-NN is identical, a Yinyang run has the same quality"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    rng = np.random.default_rng(21)
    n, d, k = 200000, 128, 256
    centers = rng.random((k, d), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.2 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    C0 = X[rng.choice(n, k, replace=False)].copy()
    _, A1 = c_kmeans(ours, X, C0, 1.0, 0.0, device=1)
    _, A2 = c_kmeans(ours, X, C0, 1.0, 0.0, device=3)
    assert np.array_equal(A1, A2)
    C1, A1 = c_kmeans(ours, X, C0, 0.99, 0.0, device=1)
    C2, A2 = c_kmeans(ours, X, C0, 0.99, 0.0, device=3)
    assert (np.abs(C1 - C2) / np.abs(C1).max(1, keepdims=True)).max() < 1e-5
    assert (A1 != A2).mean() < 1e-4
    C1, A1 = c_kmeans(ours, X, C0, 0.001, 0.1, device=1)
    C2, A2 = c_kmeans(ours, X, C0, 0.001, 0.1, device=3)
    assert (A1 == A2).mean() > 0.98
    nb1 = _knn(ours, 10, X, C1, A1, device=1)
    nb2 = _knn(ours, 10, X, C1, A1, device=3)
    assert (nb1 != nb2).mean() < 1e-5


# ------------------------------------------------------------------------------------------- error surfacing
def test_pipeline_error_is_reported_not_swallowed(km):
    """VERDICT r01 / ADVICE: a timed-out barrier in the tensor-core pipeline (injected here) must turn into
    kmcudaRuntimeError at the C ABI (AssertionError in the Python surface, reference python.cc:365-381) instead
    of kmcudaSuccess with garbage assignments"""
    code = r'''
import os, sys, ctypes, numpy as np
os.environ["KMCUDA_B200_INJECT_PIPELINE_ERROR"] = "1"
sys.path.insert(0, %r)
import kmcuda_b200
rng = np.random.default_rng(0)
X = rng.random((20000, 64), dtype=np.float32)
C = X[:64].copy(); A = np.zeros(len(X), np.uint32); m = ctypes.c_uint32(0)
rc = kmcuda_b200._lib.kmeans_cuda(3, ctypes.byref(m), 1.0, 0.0, 0, len(X), 64, 64, 0, 1, -1, 0, 0,
                                  X.ctypes.data, C.ctypes.data, A.ctypes.data, None)
print("RC", rc)
try:
    kmcuda_b200.kmeans_cuda(X, 64, init=C, tolerance=0.01, yinyang_t=0.1, device=1)
    print("NOEXC")
except AssertionError:
    print("ASSERTION")
''' % ROOT
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=300)
    assert "RC 4" in r.stdout and "ASSERTION" in r.stdout, r.stdout[-800:]


# ------------------------------------------------------------------------------------------- Yinyang bounds refresh
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_yinyang_refresh_bounds_are_valid_and_tight(km, metric):
    """the tensor-core bounds refresh (assign_tc.cu MODE 3) against the exact pass (reference kmeans_yy_init,
    src/kmeans.cu:431-485): identical upper bound and own-group bound, every other lower bound valid (never above
    the exact value) and tight (within 1e-3 of it)"""
    import torch
    from kmcuda_b200.shard import Shard, assign_once
    rng = np.random.default_rng(17)
    n, d, k, G = 40000, 96, 300, 30
    centers = rng.random((k, d), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.1 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    C = (centers + 0.02 * rng.standard_normal((k, d), dtype=np.float32)).astype(np.float32)
    if metric == "cos":
        X, C = _unit(X - 0.5), _unit(C - 0.5)
    groups = (rng.permutation(k) % G).astype(np.uint32)      # uneven, non-contiguous groups
    groups[rng.choice(k, 9, replace=False)] = 7              # one larger group
    C[5] = np.nan
    groups[5] = G                                            # dead centroid: no group (kmeans.cu:464-468)
    X[11, 3] = np.nan                                        # a row the filter cannot bound -> exact row refresh
    Xt, Ct = torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda()
    a, _, _, _ = assign_once(Xt, Ct, metric=metric)
    sh = Shard(n, d, k, metric)
    bt = sh.debug_yy_bounds(Xt, Ct, a, groups, G, True).cpu().numpy()
    be = sh.debug_yy_bounds(Xt, Ct, a, groups, G, False).cpu().numpy()
    an = a.cpu().numpy()
    ok = an < k
    np.testing.assert_array_equal(bt[ok, 0], be[ok, 0])                       # upper bound: exact
    own = groups[np.minimum(an, k - 1)]
    rows = np.flatnonzero(ok)
    np.testing.assert_array_equal(bt[rows, 1 + own[rows]], be[rows, 1 + own[rows]])   # own group: exact
    np.testing.assert_array_equal(bt[11], be[11])                             # exact row refresh
    lt, le = bt[:, 1:], be[:, 1:]
    finite = np.isfinite(le) & (le < 1e30)
    assert (lt[finite] <= le[finite]).all(), float((lt[finite] - le[finite]).max())
    assert (lt[finite] >= le[finite] - 1e-3 * np.maximum(1.0, le[finite])).all(), float((le[finite] - lt[finite]).max())
    assert np.array_equal(lt[~finite], le[~finite])                           # empty groups stay FLT_MAX


def test_yinyang_run_same_with_tensor_core_and_exact_refresh(ours, monkeypatch):
    """whole Yinyang runs with the tensor-core refresh and with the exact refresh give the same clustering: valid
    bounds do not change what Lloyd's algorithm computes"""
    rng = np.random.default_rng(23)
    n, d, k = 60000, 64, 200
    centers = rng.random((k, d), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.15 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    C0 = (centers + 0.1 * rng.standard_normal((k, d), dtype=np.float32)).astype(np.float32)
    runs = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_YY_EXACT_REFRESH", mode)
        runs[mode] = c_kmeans(ours, X, C0, 0.0005, 0.1)
    monkeypatch.delenv("KMCUDA_B200_YY_EXACT_REFRESH")
    assert (runs["0"][1] == runs["1"][1]).mean() > 0.9999
    np.testing.assert_allclose(runs["0"][0], runs["1"][0], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------- strict parity mode
@pytest.mark.parametrize("n,d,k,metric,tol,yy", [(100000, 256, 1024, 0, 0.002, 0.0), (30000, 32, 64, 1, 0.001, 0.0),
                                                 (60000, 64, 256, 0, 0.001, 0.1)])
def test_strict_update_mode_reproduces_reference_runs_bit_for_bit(ours, ref, monkeypatch, capfd, n, d, k, metric, tol,
                                                                  yy):
    """KMCUDA_B200_STRICT_UPDATE=1 replays the reference's running-sum centroid update in sample order
    (src/kmeans.cu:366-429).  With it, WHOLE runs -- every iteration's reassignment count, the final assignments and
    the final centroids -- are identical to the reference library's, which bisects the default mode's trajectory
    drift to exactly one cause: the summation order of the update (1e-7 relative), not the assignment step."""
    rng = np.random.default_rng(n + k)
    X = rng.random((n, d), dtype=np.float32) if metric == 0 else _unit(rng.standard_normal((n, d)))
    C0 = X[rng.choice(n, k, replace=False)].copy()
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    lo, Co, Ao = _iteration_log(ours, X, C0, tol, yy, capfd, metric)
    monkeypatch.delenv("KMCUDA_B200_STRICT_UPDATE")
    lr, Cr, Ar = _iteration_log(ref, X, C0, tol, yy, capfd, metric)
    print("ours", lo)
    print("ref ", lr)
    if metric == 0 and yy == 0.0:
        assert lo == lr
        assert np.array_equal(Ao, Ar), int((Ao != Ar).sum())
        np.testing.assert_array_equal(Co, Cr)
    elif metric == 0:
        # Yinyang: both libraries compute Lloyd's assignments, but with different (valid) bounds a sample sitting on
        # an fp32 tie between two centroids may be re-evaluated by one and skipped by the other
        assert lo[:4] == lr[:4] and abs(len(lo) - len(lr)) <= 1
        assert (Ao == Ar).mean() > 0.9999
        np.testing.assert_allclose(Co, Cr, rtol=1e-5, atol=1e-6)
    else:   # device acosf ties aside (the reference's own cosine tests are statistical, src/test.py:437-457)
        assert lo[:3] == lr[:3] and abs(len(lo) - len(lr)) <= 1
        assert (Ao == Ar).mean() > 0.9995
        assert np.abs(Co - Cr).max() < 1e-5


# ------------------------------------------------------------------------------------------- k-means++ on the device
@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_device_kmeanspp_picks_the_same_centroids_as_the_host_walk(km, monkeypatch, metric):
    """k-means++ with the rounds resident on the device (distances, CDF walk and row copy never leave the GPU) picks
    the same samples as the reference-shaped host loop (kmcuda.cc:262-333: D2H of all distances + sequential walk
    per round), because both consume the same rand() draws with the same walk semantics.  tolerance=1 returns the
    initial centroids (the run stops after the first assignment pass)."""
    rng = np.random.default_rng(40)
    n, d, k = 30000, 24, 80
    centers = rng.random((k, d), dtype=np.float32) * 4
    X = (centers[rng.integers(0, k, n)] + 0.2 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    if metric == "cos":
        X = _unit(X - X.mean(0))
    got = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_HOST_PLUSPLUS", mode)
        got[mode] = km.kmeans_cuda(X, k, init="k-means++", tolerance=1.0, yinyang_t=0, metric=metric, seed=11, device=1)
    monkeypatch.delenv("KMCUDA_B200_HOST_PLUSPLUS")
    np.testing.assert_array_equal(got["0"][0], got["1"][0])
    assert np.array_equal(got["0"][1], got["1"][1])
    # every centroid is one of the samples, and they are spread (k-means++): no duplicates
    cent = got["0"][0]
    assert len({tuple(np.round(c, 5)) for c in cent}) == k


def test_cuda_graph_replay_of_the_assignment_pass(ours, monkeypatch):
    """KMCUDA_B200_GRAPH=1: the launches of an assignment pass are captured once and replayed as one CUDA graph per
    iteration; a whole Lloyd run must not change"""
    rng = np.random.default_rng(61)
    for n in (70000, 90000):             # single CTAs / CTA pairs (cluster launch inside the captured graph)
        X = rng.random((n, 128), dtype=np.float32)
        C0 = X[rng.choice(len(X), 300, replace=False)].copy()
        runs = {}
        for mode in ("0", "1"):
            monkeypatch.setenv("KMCUDA_B200_GRAPH", mode)
            runs[mode] = c_kmeans(ours, X, C0, 0.005, 0.0)
        monkeypatch.delenv("KMCUDA_B200_GRAPH")
        assert np.array_equal(runs["0"][1], runs["1"][1])
        np.testing.assert_array_equal(runs["0"][0], runs["1"][0])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [75776 + 2 * 128 + 17, 75776 + 4 * 128])   # 595 tiles (ragged last tile) and 596
def test_multi_tile_pass_with_ragged_tiles_and_padded_ntiles_equals_reference(ours, ref, n):
    """A Lloyd pass over several tiles per CTA, a ragged last sample tile and K % 128 != 0 (padded table rows in the
    last n-tile): the reference's assignments (reference src/kmeans.cu:293-364)"""
    rng = np.random.default_rng(4242)
    d, k = 256, 1000
    X = rng.random((n, d), dtype=np.float32)
    C = X[rng.choice(n, k, replace=False)].copy()
    _, a_ref = c_kmeans(ref, X, C, 1.0, 0.0)
    _, a = c_kmeans(ours, X, C, 1.0, 0.0)
    assert np.array_equal(a, a_ref), "%d assignments differ from the reference" % int((a != a_ref).sum())


def test_adaptive_yinyang_switch_and_fast_refresh_keep_the_clustering(ours, monkeypatch, capfd):
    """yinyang_t > 0 on a shape where a tensor-core Lloyd pass beats a Yinyang iteration (K = 1024): with the adaptive
    switch the run finishes with Lloyd passes, without it Yinyang runs to the end; Yinyang being exact, both give the
    assignments of the plain Lloyd run from the same start.  Also covers the pair-queue form of the exact own-group
    bounds and the evening-out of a degenerate grouping (near-equidistant random centres)."""
    rng = np.random.default_rng(99)
    n, d, k = 200000, 256, 1024
    centers = rng.random((k, d), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.05 * rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    C0 = X[rng.choice(n, k, replace=False)].copy()
    runs = {}
    for name, yy, adaptive in (("lloyd", 0.0, "0"), ("yinyang", 0.1, "0"), ("adaptive", 0.1, "1")):
        monkeypatch.setenv("KMCUDA_B200_YY_ADAPTIVE", adaptive)
        runs[name] = c_kmeans(ours, X, C0, 0.0005, yy, verbosity=1 if name == "adaptive" else 0)
    out = capfd.readouterr().out
    monkeypatch.setenv("KMCUDA_B200_YY_ADAPTIVE", "0")
    for name in ("yinyang", "adaptive"):
        assert (runs[name][1] == runs["lloyd"][1]).mean() > 0.9999, name
        np.testing.assert_allclose(runs[name][0], runs["lloyd"][0], rtol=1e-4, atol=1e-5)
    assert "iteration" in out


def test_staged_pageable_ingest_delivers_the_same_bytes(ours, monkeypatch):
    """host buffers >= 256 MB that are not pinned are copied by several host threads through pinned staging buffers
    (transfer.cu::host_to_device); the result must be the one of the plain cudaMemcpy (ragged last chunk included)"""
    rng = np.random.default_rng(5)
    n, d, k = 280001, 260, 300           # 291 MB (staged from 256 MB upwards), not a multiple of the 16 MB chunk
    X = rng.random((n, d), dtype=np.float32)
    C0 = X[rng.choice(n, k, replace=False)].copy()
    out = {}
    for threads in ("6", "1"):
        monkeypatch.setenv("KMCUDA_B200_INGEST_THREADS", threads)
        out[threads] = c_kmeans(ours, X, C0, 0.01, 0.0)
    assert np.array_equal(out["6"][1], out["1"][1])
    assert np.array_equal(out["6"][0], out["1"][0])


@pytest.mark.parametrize("D,K", [(256, 1024), (96, 37), (480, 300)])
def test_member_sums_with_skewed_empty_and_unassigned_clusters(km, D, K):
    """The member-sum kernel walks fixed chunks of the cluster-sorted order (simt_kernels.cu::cluster_sums_kernel):
    one giant cluster spanning hundreds of chunks, clusters smaller than the unroll depth, empty clusters, runs that
    end exactly on a chunk boundary and rows with the "unassigned" key K must all give the fp64 sums to fp32
    accuracy and the exact counts (reference semantics: kmeans.cu:366-429 sums the members of every cluster)."""
    import torch
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D * 1000 + K)
    n = 300000
    X = (rng.standard_normal((n, D)) * 3 + 1).astype(np.float32)
    a = np.empty(n, np.int64)
    a[:150000] = 5                                     # giant cluster
    a[150000:151024] = 7                               # exactly one chunk's worth
    a[151024:151027] = 9                               # below the unroll depth
    a[151027:200000] = rng.integers(10, K // 2, 48973)
    a[200000:299000] = rng.integers(K // 2 + 3, K, 99000)   # K//2 .. K//2+2 stay empty
    a[299000:] = K                                     # unassigned
    a = a[rng.permutation(n)]
    sh = Shard(n, D, K)
    sums = torch.full((K, D), 7.0, device="cuda")
    counts = torch.full((K,), 7, dtype=torch.int32, device="cuda")
    sh.partial_sums(torch.from_numpy(X).cuda(), torch.from_numpy(a.astype(np.int32)).cuda(), sums, counts)
    torch.cuda.synchronize()
    exp = np.zeros((K, D), np.float64)
    valid = a < K
    np.add.at(exp, a[valid], X[valid].astype(np.float64))
    cnt = np.bincount(a[valid], minlength=K)
    assert np.array_equal(counts.cpu().numpy(), cnt)
    got = sums.cpu().numpy().astype(np.float64)
    scale = np.zeros((K, D), np.float64)
    np.add.at(scale, a[valid], np.abs(X[valid]).astype(np.float64))
    assert np.all(np.abs(got - exp) <= 4e-7 * scale + 1e-30), float(np.max(np.abs(got - exp) / (scale + 1e-30)))
    assert np.all(got[cnt == 0] == 0)


def test_multi_gpu_peer_memory_exchange_one_process_per_gpu():
    """the CUDA-IPC exchange of the centroid update (csrc/exchange.cu) under torchrun: tests/_peer_exchange_worker.py"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(_ngpu(), 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(HERE, "_peer_exchange_worker.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert "PEER_EXCHANGE_OK" in r.stdout, r.stdout[-3000:]
