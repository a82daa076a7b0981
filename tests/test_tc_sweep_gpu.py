"""Sweep of the tensor-core filter `tc_assign_kernel<NKB, MODE>` (assign_tc.cu) over every K-block count, all four
modes and the filter's slow paths (run on an H100: `pytest -m gpu`).

Checkers (no reference library needed): the CPU oracle (`oracle.assign_lloyd`, the C restatement of the reference
arithmetic, pinned to the reference by `test_oracle_matches_reference`), this library's exact path
(`KMCUDA_B200_FORCE_EXACT=1`, which shares no code with the filter's candidate logic), fp64 truth for cosine near-ties
and k-NN.  After every tensor-core pass the pipeline status is clean and the pass really ran on the tensor cores.

Which instantiation is checked where (NKB = K-blocks of 64 features, D 4..512):

| mode | NKB | checked by |
|---|---|---|
| 0 Lloyd | 1-8, full and ragged last K-block (D = 4, 60..512) | `test_lloyd_pass_sweep`: K in {2, 127, 128, 129, 1000} (+ 5000), fewer sample tiles than SMs / more than two per SM, N = 1 and 100; cosine at one D per NKB; near-tie pairs; `test_lloyd_pass_bookkeeping` (prev / changed) per NKB |
| 0 Lloyd, slow paths | 1, 4, 8 | `test_filter_slow_paths`: list compaction (rising threshold), candidate counts that pin the margin's width, full per-lane list, > 32 candidates, pair queue full, duplicate centroids; `test_non_finite_and_far_rows` |
| 1 Yinyang local step | 1 (D 64), 2 (128), 3 (132; cosine 192), 4 (256), 5 (260), 6 (384), 7 (388), 8 (512; cosine 512) | `test_yinyang_runs_tc_equal_exact`: whole runs, TC route == reference-order scan |
| 3 bounds refresh | 1 (D 4), 2 (128), 3 (132), 4 (256), 5 (260), 6 (384), 7 (388), 8 (512) | `test_yinyang_refresh_bounds_sweep`: G in {1, 7, K/4}, groups of 1 / 2 / 3 / 5, dead centroid, NaN row |
| 2 k-NN | 1 (D 4), 2 (128), 3 (132), 4 (256), 5 (260), 6 (384), 7 (388), 8 (512) | `test_knn_sweep` (k in {1, 15}, N = 4096 tensor-core / 4095 exact), `test_knn_cluster_shapes` (NKB 3, 7) |

NKB = ceil(D / 64).  Every row above is run by this file alone and needs no reference library.  With
KMB_SWEEP_COUNTERS=<file> the per-case `(rechecked, overflowed)` counters of the tensor-core passes (and the largest
bounds-refresh slack per case) are written to that file as JSON at the end of the module.
"""
import ctypes
import functools
import json
import os

import numpy as np
import pytest

import tc_sweep_cases as T
from oracle import oracle as O

pytestmark = pytest.mark.gpu

IMPORT = 3
COUNTERS = []


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    O.set_threads(os.cpu_count())
    yield kmcuda_b200
    if os.environ.get("KMB_SWEEP_COUNTERS"):
        with open(os.environ["KMB_SWEEP_COUNTERS"], "w") as f:
            json.dump(COUNTERS, f, indent=0)


@pytest.fixture(scope="module")
def lib(km):
    return O.load_c_api(km.LIB_PATH)


@pytest.fixture(scope="module")
def sms(km):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_pass(X, C, metric="L2", force_exact=False, assign=None, tc=True):
    """one Shard pass: (assign, prev, changed, (used_tc, rechecked, overflowed)); the pipeline status must be clean.
    tc: whether the shape is one the tensor-core route takes (checked unless force_exact)"""
    import torch
    from kmcuda_b200.shard import Shard
    old = os.environ.get("KMCUDA_B200_FORCE_EXACT")
    os.environ["KMCUDA_B200_FORCE_EXACT"] = "1" if force_exact else "0"     # read when the shard is created
    try:
        n = len(X)
        sh = Shard(n, X.shape[1], C.shape[0], metric)
    finally:
        if old is None:
            os.environ.pop("KMCUDA_B200_FORCE_EXACT", None)
        else:
            os.environ["KMCUDA_B200_FORCE_EXACT"] = old
    Xt, Ct = torch.from_numpy(np.ascontiguousarray(X)).cuda(), torch.from_numpy(np.ascontiguousarray(C)).cuda()
    a = (torch.full((n,), -1, dtype=torch.int32, device="cuda") if assign is None
         else torch.from_numpy(assign.astype(np.int32)).cuda())
    prev = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ch = torch.zeros(1, dtype=torch.int32, device="cuda")
    sh.assign(Xt, Ct, a, prev, ch)
    torch.cuda.synchronize()
    err, info = sh.last_error(), sh.last_pass_info()
    sh.close()
    assert err == 0, "pipeline error 0x%x" % err
    if not force_exact:
        assert info[0] == tc, "tensor-core path taken: %s, expected %s" % (info[0], tc)
    return (a.cpu().numpy().astype(np.uint32), prev.cpu().numpy().astype(np.uint32), int(ch.item()), info)


def check_oracle(X, C, got, metric, rows=None):
    rows = np.arange(len(X)) if rows is None else rows
    exp = O.assign_lloyd(X[rows], C, metric=1 if metric == "cos" else 0)[0]
    keep = exp != T.UNTOUCHED                        # rows the oracle leaves untouched (every score NaN)
    bad = np.flatnonzero(keep & (got[rows] != exp))
    if metric == "cos" and len(bad):                  # device acosf vs glibc acosf: only fp64 near-ties may differ
        _, best, second = O.assign_truth(X[rows[bad]], C, metric=1)
        bad = bad[~O.tie_exempt(best, second)]
    assert len(bad) == 0, "%d oracle mismatches, rows %s" % (len(bad), rows[bad][:8])
    return exp


# ------------------------------------------------------------------------------------------- MODE 0 sweep
SWEEP_D = [4, 60, 64, 68, 128, 132, 192, 196, 256, 260, 320, 324, 384, 388, 448, 452, 508, 512]
SWEEP_K = [2, 127, 128, 129, 1000]
NKB_D = [64, 128, 192, 256, 320, 384, 448, 512]      # one full-K-block D per NKB


def _sweep_cases():
    out = []
    for D in SWEEP_D:
        for nl in ("few", "many"):
            for K in SWEEP_K + ([5000] if D in (132, 388) else []):
                out.append((D, K, nl, "L2", "plain"))
            if D in NKB_D and nl == "many":
                out += [(D, K, nl, "cos", "plain") for K in (129, 1000)]
                out.append((D, 1000, nl, "L2", "near_ties"))
        if D in (64, 260):
            out += [(D, K, nl, "L2", "plain") for nl in ("1", "100") for K in SWEEP_K]
    return out


SWEEP = _sweep_cases()


@functools.lru_cache(maxsize=2)
def _samples(N, D, metric):
    X = T.clustered(N, D, seed=D)
    return T.unit(X) if metric == "cos" else X


@functools.lru_cache(maxsize=4)
def _centroids(N, D, K, metric, variant):
    # drawn from at least 4096 samples of the same clusters: with N = 1 or 100 and K = 1000, perturbed copies of the
    # same few samples would leave most rows with more than 32 candidates
    pool = _samples(max(N, 4096), D, metric)
    C = T.perturbed_centroids(pool, K, seed=K + D, near_ties=variant == "near_ties")
    return T.unit(C) if metric == "cos" else C


@pytest.mark.parametrize("D,K,nl,metric,variant", SWEEP, ids=["D%d-K%d-N%s-%s-%s" % c for c in SWEEP])
def test_lloyd_pass_sweep(km, sms, D, K, nl, metric, variant):
    N = T.sweep_n(nl, sms)
    X, C = _samples(N, D, metric), _centroids(N, D, K, metric, variant)
    a, prev, changed, info = run_pass(X, C, metric)
    COUNTERS.append(("sweep D%d K%d N%d %s %s" % (D, K, N, metric, variant), info[1], info[2]))
    assert changed == N and (prev == T.UNTOUCHED).all()
    e, _, _, info_e = run_pass(X, C, metric, force_exact=True)
    assert not info_e[0]
    assert np.array_equal(a, e), "%d rows differ from the exact pass" % int((a != e).sum())
    rows = None if N <= 4096 else np.sort(np.random.default_rng(N + D + K).choice(N, 512, replace=False))
    check_oracle(X, C, a, metric, rows)
    if variant == "plain":
        assert info[2] <= max(1, N // 20), "too many rows fell back to the exact pass: %d of %d" % (info[2], N)
    else:
        assert info[1] > 0, "the near-tie pairs never reached the re-check queue"


@pytest.mark.parametrize("D", NKB_D)
def test_lloyd_pass_bookkeeping(km, sms, D):
    """a second pass from a given assignment: prev = the input, changed = the oracle's count (warp-aggregated counter,
    rows finished by the emitters, the re-check and the exact pass alike)"""
    N, K = T.sweep_n("few", sms), 129
    X = _samples(N, D, "L2")
    C = T.perturbed_centroids(X, K, seed=D, near_ties=True)
    C2 = C + (0.05 * np.abs(C).mean() * np.random.default_rng(D).standard_normal(C.shape)).astype(np.float32)
    a_in = O.assign_lloyd(X, C2)[0]
    a_exp, _, ch_exp = O.assign_lloyd(X, C, assign=a_in)
    a, prev, changed, info = run_pass(X, C, assign=a_in)
    COUNTERS.append(("bookkeeping D%d" % D, info[1], info[2]))
    assert np.array_equal(prev, a_in)
    assert np.array_equal(a, a_exp), int((a != a_exp).sum())
    assert changed == ch_exp and 0 < changed < N


# ------------------------------------------------------------------------------------------- MODE 0 slow paths
SLOW = [(k, D, "L2") for k in T.LIST_CASES for D in (64, 256, 512)]
SLOW += [(k, D, "cos") for k in ("rise", "list_overflow") for D in (64, 256)]


@pytest.mark.parametrize("kind,D,metric", SLOW, ids=["%s-D%d-%s" % c for c in SLOW])
def test_filter_slow_paths(km, kind, D, metric):
    """inputs built to reach list compaction, a full per-lane list, > MAX_CAND candidates, a full pair queue and exact
    duplicates (test_tc_sweep_cases_cpu.py proves they do); the exact winner is placed where a kernel that mishandles
    the path picks another index"""
    X, C, info = T.list_case(kind, D, metric)
    a, prev, changed, pi = run_pass(X, C, metric)
    COUNTERS.append(("%s D%d %s" % (kind, D, metric), pi[1], pi[2]))
    e = run_pass(X, C, metric, force_exact=True)[0]
    assert np.array_equal(a, e), "%d rows differ from the exact pass" % int((a != e).sum())
    check_oracle(X, C, a, metric)
    for rows, win in zip(info["rows"], info["winner"]):
        assert (a[rows] == win).all(), (win, np.unique(a[rows]))
    rechecked, overflowed = pi[1], pi[2]
    if kind in ("rise", "rise_pair", "rise_coarse"):
        assert rechecked == 0 and overflowed == 0            # compaction leaves exactly one candidate per row
    elif kind == "rise_wide":
        assert rechecked == len(X) and overflowed == 0       # every row: the winner and the runner-up 0.75 margins below
    elif kind in ("rise_margin", "dupes"):
        assert rechecked > 0 and overflowed == 0
    elif kind in ("list_overflow", "max_cand"):
        assert overflowed > 0
    else:   # queue: the first rows fit into the pair queue, the rest go to the exact pass
        assert rechecked > 0 and overflowed > 0


@pytest.mark.parametrize("D", [64, 256, 512])
def test_non_finite_and_far_rows(km, D):
    X, C = T.nonfinite_case(D)
    a, _, _, info = run_pass(X, C)
    COUNTERS.append(("non-finite D%d" % D, info[1], info[2]))
    e = run_pass(X, C, force_exact=True)[0]
    assert np.array_equal(a, e), np.flatnonzero(a != e)[:10]
    exp = check_oracle(X, C, a, "L2")
    assert info[2] > 0
    assert (a[10:20] == 6).all() and (a[20:30] == 3).all()   # duplicates: the lowest index wins
    assert not np.isin(a[exp != T.UNTOUCHED], [40, 41, 170]).any()


# ------------------------------------------------------------------------------------------- MODE 1
_libc = ctypes.CDLL(None)


def c_kmeans(lib, X, C0, tol, yy, metric=0, verbosity=0):
    X = np.ascontiguousarray(X)
    N, D = X.shape
    C = np.array(C0, copy=True, order="C")
    A = np.zeros(N, np.uint32)
    m = ctypes.c_uint32(0)
    rc = lib.kmeans_cuda(IMPORT, ctypes.byref(m), tol, yy, metric, N, D, C.shape[0], 3, 1, -1, 0, verbosity,
                         X.ctypes.data, C.ctypes.data, A.ctypes.data, None)
    _libc.fflush(None)      # the log lines are printf'ed: out of the C stdio buffer before the caller reads them
    assert rc == 0, rc
    return C, A


def _structureless(n, d, k, seed, metric):
    """uniform (L2) / isotropic unit (cosine) samples, centroids = samples: dozens of slow iterations, so the run
    leaves the Lloyd draft phase and the Yinyang local step does most of the work"""
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32) if metric == 0 else T.unit(rng.standard_normal((n, d)))
    C0 = X[rng.choice(n, k, replace=False)].copy()
    return np.ascontiguousarray(X, np.float32), C0


YY = [(64, 0), (128, 0), (132, 0), (256, 0), (260, 0), (384, 0), (388, 0), (512, 0), (192, 1), (512, 1)]


@pytest.mark.parametrize("D,metric", YY, ids=["D%d-%s" % (d, "cos" if m else "L2") for d, m in YY])
def test_yinyang_runs_tc_equal_exact(lib, D, metric, monkeypatch, capfd):
    """whole Yinyang runs: the tensor-core local step (MODE 1) and the reference-order scan give the same iteration
    lines, assignments and centroids.  Both runs refresh their bounds exactly: the tensor-core refresh (MODE 3, checked
    by test_yinyang_refresh_bounds_sweep) gives valid but looser bounds, so fewer rows pass the global filter and the
    run's refresh heuristic fires at other iterations -- same clustering, other log lines."""
    X, C0 = _structureless(20000, D, 300, D, metric)
    monkeypatch.setenv("KMCUDA_B200_YY_EXACT_REFRESH", "1")
    runs = {}
    for fe in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", fe)
        capfd.readouterr()
        C, A = c_kmeans(lib, X, C0, 1e-3, 0.1, metric, verbosity=1)
        out = capfd.readouterr().out
        runs[fe] = C, A, [ln for ln in out.splitlines() if ln.startswith("iteration") or "refreshing" in ln]
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "0")
    assert any("refreshing" in ln for ln in runs["0"][2]) and len(runs["0"][2]) > 3, runs["0"][2]
    assert runs["0"][2] == runs["1"][2]
    assert np.array_equal(runs["0"][1], runs["1"][1]), int((runs["0"][1] != runs["1"][1]).sum())
    np.testing.assert_array_equal(runs["0"][0], runs["1"][0])
    C_last, A_last = runs["0"][:2]
    assert (c_kmeans(lib, X, C_last, 1.0, 0.0, metric)[1] == A_last).mean() > 0.9995


# ------------------------------------------------------------------------------------------- MODE 3
def _groups(k, G, rng):
    """groups 0-3 with 1, 2, 3 and 5 members, the other centroids spread at random over groups 4 .. G - 1"""
    if G == 1:
        return np.zeros(k, np.uint32)
    fixed = np.repeat(np.arange(4), [1, 2, 3, 5])
    g = np.concatenate([fixed, rng.integers(4, G, k - len(fixed))])
    return g[rng.permutation(k)].astype(np.uint32)


@pytest.mark.parametrize("G", ["1", "7", "K/4"])
@pytest.mark.parametrize("D", [4, 128, 132, 256, 260, 384, 388, 512])
def test_yinyang_refresh_bounds_sweep(km, D, G):
    """MODE 3 against the exact refresh: identical upper bound, own-group bound and exact-row refresh; every other
    bound valid (<= exact) and within 1e-3 of it"""
    import torch
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D)
    n, k = 20000, 300
    G = {"1": 1, "7": 7, "K/4": k // 4}[G]
    centers = rng.random((k, D), dtype=np.float32)
    X = (centers[rng.integers(0, k, n)] + 0.1 * rng.standard_normal((n, D), dtype=np.float32)).astype(np.float32)
    C = (centers + 0.02 * rng.standard_normal((k, D), dtype=np.float32)).astype(np.float32)
    groups = _groups(k, G, rng)
    C[5] = np.nan
    groups[5] = G                                            # dead centroid: no group
    X[11, min(3, D - 1)] = np.nan                            # a row the filter cannot bound -> exact row refresh
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
    np.testing.assert_array_equal(bt[ok, 0], be[ok, 0])
    own = groups[np.minimum(an, k - 1)]
    rows = np.flatnonzero(ok)
    np.testing.assert_array_equal(bt[rows, 1 + own[rows]], be[rows, 1 + own[rows]])
    np.testing.assert_array_equal(bt[11], be[11])
    lt, le = bt[:, 1:], be[:, 1:]
    finite = np.isfinite(le) & (le < 1e30)
    assert (lt[finite] <= le[finite]).all(), float((lt[finite] - le[finite]).max())
    slack = float(((le[finite] - lt[finite]) / np.maximum(1.0, le[finite])).max())
    COUNTERS.append(("refresh D%d G%d slack" % (D, G), slack, 0))
    # D = 4: the margin E counts 64 features per K-block (the accumulation term is 16x what 4 features need) and the
    # distances to other groups are short, so a bound sits up to ~6e-3 below the exact one (measured on an H100)
    tight = 1e-3 if D > 4 else 1e-2
    assert slack <= tight, slack
    assert np.array_equal(lt[~finite], le[~finite])


# ------------------------------------------------------------------------------------------- MODE 2
def _knn(km, k, X, C, A, monkeypatch, capfd, force_exact=False):
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1" if force_exact else "0")
    monkeypatch.setenv("KMCUDA_B200_TIMING", "1")
    capfd.readouterr()
    nb = km.knn_cuda(k, X, C, A, device=1)
    err = capfd.readouterr().err
    monkeypatch.delenv("KMCUDA_B200_TIMING")
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "0")
    line = [ln for ln in err.splitlines() if "knn tensor-core path" in ln]
    if not line:
        return nb, 0, 0
    # a pipeline error of the tensor-core pass makes the library search every query exactly: the answer stays right,
    # so the error word is the only trace of it
    assert "error word 0x0;" in line[0], line[0]
    served = int(line[0].split("path:")[1].split("rows")[0])
    list_full = int(line[0].split("list full")[1].split(",")[0])
    return nb, served, list_full


def _check_knn(X, nb, queries, k, ref=None):
    """the neighbours' fp64 distances are the k smallest (so the sets agree unless the k-th and (k+1)-th distances
    are within 1e-6); ref: a second answer whose sets must equal nb's wherever there is no such near-tie"""
    truth = T.knn_truth(X, queries, k)
    Xd = X.astype(np.float64)
    got = nb[queries].astype(np.int64)
    assert (got < len(X)).all() and (got != queries[:, None]).all()
    assert all(len(set(r)) == k for r in got.tolist())
    d = np.sort(((Xd[got] - Xd[queries][:, None, :]) ** 2).sum(-1), axis=1)
    np.testing.assert_allclose(d, truth[:, :k], rtol=1e-6, atol=1e-12)
    if ref is not None:
        clear = truth[:, k] - truth[:, k - 1] > 1e-6 * np.maximum(truth[:, k], 1e-30)
        for q, a, b in zip(queries[clear], got[clear], ref[queries[clear]]):
            assert set(a.tolist()) == set(b.tolist()), q


KNN = [(D, k, N) for D in (4, 128, 132, 256, 260, 384, 388, 512) for k in (1, 15) for N in (4096, 4095)]


@pytest.mark.parametrize("D,k,N", KNN, ids=["D%d-k%d-N%d" % c for c in KNN])
def test_knn_sweep(km, D, k, N, monkeypatch, capfd):
    """N = 4096 is the smallest input the tensor-core route takes, N = 4095 runs the exact search"""
    X = T.clustered(N, D, seed=D + k, n_centers=40, sigma=0.3)
    C = T.perturbed_centroids(X, 40, seed=D)
    A = T.nearest(X, C)
    nb, served, _ = _knn(km, k, X, C, A, monkeypatch, capfd)
    if N >= 4096:
        assert served > 0.5 * N, served
    else:
        assert served == 0
    ex, served_e, _ = _knn(km, k, X, C, A, monkeypatch, capfd, force_exact=True)
    assert served_e == 0
    _check_knn(X, nb, np.arange(N), k, ref=ex)


@pytest.mark.parametrize("kind", ["tiny_clusters", "giant", "duplicates"])
@pytest.mark.parametrize("D", [132, 388])
def test_knn_cluster_shapes(km, kind, D, monkeypatch, capfd):
    X, C, A = T.knn_shape(kind, D)
    k = 15
    nb, served, list_full = _knn(km, k, X, C, A, monkeypatch, capfd)
    assert served > 0, "tensor-core k-NN path not taken"
    if kind == "duplicates":
        assert list_full > 0, "no half-row filled its KNN_CAP entries"
    ex, _, _ = _knn(km, k, X, C, A, monkeypatch, capfd, force_exact=True)
    rng = np.random.default_rng(D)
    queries = np.sort(np.concatenate([rng.choice(len(X) - 6000, 400, replace=False),
                                      len(X) - 6000 + rng.choice(6000, 100, replace=False)]))
    _check_knn(X, nb, queries, k, ref=ex)


# ------------------------------------------------------------------------------------------- fp16x2 samples
@pytest.mark.parametrize("D", [64, 256])
def test_fp16_samples_on_the_tensor_core_path(km, D):
    """fp16 samples are widened at ingest: the same assignments as the fp32 call on the widened arrays, bit for bit,
    and the fp16 call's assignment pass runs the MODE 0 tensor-core kernel"""
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(D)
    X16 = T.clustered(20000, D, seed=D).astype(np.float16)
    C16 = (X16[rng.choice(20000, 300, replace=False)].astype(np.float32)
           + 0.05 * rng.standard_normal((300, D)).astype(np.float32)).astype(np.float16)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, a16 = km.kmeans_cuda(X16, 300, init=C16.view(np.float32), tolerance=1.0, yinyang_t=0.0, device=1)
    kernels = {e.name for e in prof.events() if "tc_assign_kernel" in e.name}
    nkb = (D + 63) // 64
    assert any("tc_assign_kernel<%d, 0>" % nkb in k for k in kernels), kernels
    X32, C32 = X16.astype(np.float32), C16.astype(np.float32)
    _, a32 = km.kmeans_cuda(X32, 300, init=C32, tolerance=1.0, yinyang_t=0.0, device=1)
    exp = O.assign_lloyd(X32, C32)[0]
    assert np.array_equal(a32, exp), int((a32 != exp).sum())
    assert np.array_equal(a16, exp), int((a16 != exp).sum())
