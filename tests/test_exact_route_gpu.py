"""Sweep of the exact SIMT route (simt_kernels.cu, yinyang.cu, knn_kernels.cu) beyond the tensor-core envelope: D % 4 != 0
and 1024 < D <= 65535, the feature counts every call outside 4 <= D <= 1024, D % 4 == 0 runs on (run on an H100:
`pytest -m gpu`).

Checkers (no reference library needed): the CPU oracle (`oracle.assign_lloyd`, `kmeans`, `knn`, the C restatement of the
reference arithmetic, pinned to the reference by `test_oracle_matches_reference`), bit for bit where the reference
arithmetic is replayed; fp64 truth for sums, distances and bounds; the NumPy models of mini-batch, k-means|| and the
relocation.  Every shape list below straddles the configuration switches of the kernels, which
test_exact_route_cases_cpu.py derives from the sources and checks against these lists.  A Shard pass on every shape
checks that the tensor-core route did not take it (`last_pass_info()[0]` is false), so that a wider tensor-core envelope
cannot silently empty this file; the one shape inside the envelope (D = 772) runs with KMCUDA_B200_FORCE_EXACT=1.

| kernel | switch | shapes | checked by |
|---|---|---|---|
| `exact_pass_kernel<.., 0>` Lloyd pass | 128 / 64 / 32-row tiles, no staging above D = 1536 | D 1 .. 2049 x K {2, 3, 33, 129, 1000}, D 11264 .. 65535 x K {2, 3, 33}; N = 1, ragged against the tile; NaN / Inf rows, NaN and duplicate centroids; cosine at one D per tier | `test_lloyd_pass` (oracle), `test_lloyd_pass_bookkeeping` (prev / changed) |
| `exact_rows_few_kernel` / `exact_pass_kernel` list mode | <= 8192 rows / more; row in shared memory up to D = 16384 | lists of 1, 8192 and 8193 rows (duplicates, longer than N) at D 5 .. 65535 | `test_row_lists` (oracle on X[rows]) |
| `exact_pass_kernel<.., 1>` bounds refresh | tiers as above | D 5 .. 12287, G {1, 7, 32}, empty group, dead centroid | `test_exact_bounds_refresh` (fp64) |
| `yy_rows_cta_kernel` Yinyang local step | row in shared memory up to D = 16384 | D 5 .. 16385, cosine at D 126 and 1025 | `test_yinyang_rows_kernel_equals_reference_order_scan` (against `yy_local_scan_kernel`, bits and logs) |
| `strict_adjust_kernel` | D <= 1600 | D 7 .. 1600; 1601 rejected | `test_strict_runs_equal_the_oracle`, `test_strict_mode_rejects_wide_samples` |
| `cluster_sums_kernel` | VEC 4 (D % 4 == 0, aligned), VEC 1 | D 5 .. 2049, unaligned X, several float4 columns per thread | `test_member_sums` (fp64) |
| `average_distance_kernel` | - | D 5 .. 12287 | `test_average_distance` (fp64) |
| `knn_warp_search_kernel` | query in shared memory up to D = 2048 | D 1025 .. 12287 x k {1, 16, 31, 32, 33, 65} | `test_knn` (oracle, fp64) |
| weights, mini-batch, k-means||, relocation, k-means++, fp16x2 | - | D 1026, 1030, 11265 | `test_*` below (bits, models) |
| default and mini-batch calls | - | D 11265, 12287, 65535 | `test_every_accepted_d_runs` (oracle) |
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import kmeans_parallel_model as KPM  # noqa: E402
import minibatch_model as MBM  # noqa: E402
import relocate_model as RM  # noqa: E402
import tc_sweep_cases as T  # noqa: E402
import test_kmeans_parallel_gpu as KPG  # noqa: E402
import test_minibatch_gpu as MBG  # noqa: E402
import test_relocate_gpu as RG  # noqa: E402
import test_tc_sweep_gpu as S  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

FLT_MAX = np.finfo(np.float32).max

# the shape lists (test_exact_route_cases_cpu.py checks that they straddle every switch of the kernels)
LLOYD_D = [1, 3, 5, 33, 126, 381, 382, 771, 772, 1025, 1026, 1028, 1536, 1537, 2048, 2049]
LLOYD_WIDE_D = [11264, 11265, 12287, 65535]
LLOYD_K = [2, 3, 33, 129, 1000]
LLOYD_WIDE_K = [2, 3, 33]
COS_D = [126, 382, 1025, 2049]                     # one D per tier of the Lloyd pass
BOOKKEEPING_D = [5, 382, 772, 1025, 1537, 12287]
LIST_D = [5, 382, 772, 1025, 1537, 2049, 11264, 11265, 12287, 16384, 16385, 65535]
LIST_LENGTHS = [1, 8192, 8193]
REFRESH_D = [5, 382, 772, 1025, 1537, 2049, 12287]
YY_D = [5, 126, 382, 1025, 1537, 2049, 11264, 11265, 12287, 16384, 16385]
YY_COS_D = [126, 1025]
STRICT_D = [7, 1025, 1536, 1537, 1600]
STRICT_REJECTED_D = 1601
SUMS = [(5, 37, False), (33, 37, False), (126, 300, False), (1028, 300, False), (1028, 300, True), (2048, 100, False),
        (2049, 100, False)]
AVG_D = [5, 1025, 2049, 12287]
KNN_D = [1025, 2048, 2049, 12287]
KNN_K = [1, 16, 31, 32, 33, 65]
EXT_D = [1030, 11265]
FP16_D = 1026
ACCEPT_D = [11265, 12287, 65535]


def tc_shape(D):
    """the tensor-core route's envelope (assign_tc.cu::tc_supported)"""
    return 4 <= D <= 1024 and D % 4 == 0


def tile_rows(D):
    """rows per CTA of exact_pass_kernel (simt_kernels.cu::exact_cfg)"""
    for rb in (128, 64, 32):
        if (rb + 1) * D * 4 + 8 * rb * 8 <= 200 * 1024:
            return rb
    return 128


def ragged_n(D):
    return 2 * tile_rows(D) + 7


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


def _pass(X, C, metric="L2", assign=None):
    """one Shard pass on the exact route: D = 772 is forced there, every other shape must not take the tensor cores"""
    return S.run_pass(X, C, metric, force_exact=tc_shape(X.shape[1]), assign=assign, tc=False)


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _lines(out, prefix="iteration"):
    return [ln for ln in out.splitlines() if ln.startswith(prefix)]


def _edge_rows(X, C):
    """NaN in the first feature (an insane row), NaN elsewhere, +-Inf rows, a NaN centroid and a duplicate centroid whose
    lower index must win for the row sitting on it"""
    X, C = X.copy(), C.copy()
    K, D = C.shape
    X[0, 0] = np.nan
    X[1, D - 1] = np.nan
    X[2] = np.inf
    X[3] = -np.inf
    if K >= 3:
        C[K - 1] = np.nan
        C[1] = C[0]
        X[4] = C[0]
    return X, C


# ------------------------------------------------------------------------------------------- Lloyd pass
def _lloyd_cases():
    out = [(D, K, "ragged", "L2") for D in LLOYD_D for K in LLOYD_K]
    out += [(D, K, "ragged", "L2") for D in LLOYD_WIDE_D for K in LLOYD_WIDE_K]
    out += [(D, 3, "1", "L2") for D in (5, 1025, 65535)]
    out += [(D, 129, "ragged", "cos") for D in COS_D]
    return out


LLOYD = _lloyd_cases()


@pytest.mark.parametrize("D,K,nl,metric", LLOYD, ids=["D%d-K%d-N%s-%s" % c for c in LLOYD])
def test_lloyd_pass(km, D, K, nl, metric):
    N = ragged_n(D) if nl == "ragged" else int(nl)
    X = T.clustered(N, D, seed=D + K, n_centers=16)
    C = T.perturbed_centroids(X, K, seed=K + D)
    if metric == "cos":
        X, C = T.unit(X), T.unit(C)
    edges = N >= 16 and metric == "L2"
    if edges:
        X, C = _edge_rows(X, C)
    a, prev, changed, _ = _pass(X, C, metric)
    exp = S.check_oracle(X, C, a, metric)
    assert (a[exp == T.UNTOUCHED] == T.UNTOUCHED).all()
    assert (prev == T.UNTOUCHED).all()
    if edges:
        assert a[0] == K
        if K >= 3:
            assert a[4] == 0 and not (a == K - 1).any()
    if metric == "L2":
        assert changed == O.assign_lloyd(X, C)[2]


@pytest.mark.parametrize("D", BOOKKEEPING_D)
def test_lloyd_pass_bookkeeping(km, D):
    """a second pass from a given assignment: prev = the input, changed = the oracle's count"""
    N, K = ragged_n(D), 33
    X = T.clustered(N, D, seed=D, n_centers=16)
    C = T.perturbed_centroids(X, K, seed=D, near_ties=True)
    C2 = C + (0.05 * np.abs(C).mean() * np.random.default_rng(D).standard_normal(C.shape)).astype(np.float32)
    a_in = O.assign_lloyd(X, C2)[0]
    a_exp, prev_exp, ch_exp = O.assign_lloyd(X, C, assign=a_in)
    a, prev, changed, _ = _pass(X, C, assign=a_in)
    assert np.array_equal(prev, a_in) and np.array_equal(prev, prev_exp)
    assert np.array_equal(a, a_exp), int((a != a_exp).sum())
    assert changed == ch_exp and 0 < changed < N


# ------------------------------------------------------------------------------------------- row lists
@pytest.mark.parametrize("D", LIST_D)
def test_row_lists(km, monkeypatch, D):
    """Shard.debug_assign_rows without a tensor-core plan: lists of up to kFewRows rows go to exact_rows_few_kernel,
    longer ones to exact_pass_kernel's list mode; duplicates, lists longer than N and an insane row"""
    import torch
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D)
    N, K = (700 if D <= 2049 else 64), 33
    X = T.clustered(N, D, seed=D, n_centers=16)
    C = T.perturbed_centroids(X, K, seed=D)
    X, C = _edge_rows(X, C)
    exp = O.assign_lloyd(X, C)[0]
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1" if tc_shape(D) else "0")
    sh = Shard(max(LIST_LENGTHS), D, K)
    Xt, Ct = torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda()
    for n in LIST_LENGTHS:
        rows = np.array([0]) if n == 1 else np.concatenate([[0, 4], rng.integers(0, N, n - 2)])
        got = sh.debug_assign_rows(Xt, Ct, torch.from_numpy(rows.astype(np.int32))).cpu().numpy().view(np.uint32)
        assert sh.last_error() == 0 and not sh.last_pass_info()[0]
        keep = exp[rows] != T.UNTOUCHED
        assert np.array_equal(got[keep], exp[rows][keep]), (n, int((got[keep] != exp[rows][keep]).sum()))
        assert got[0] == K
    sh.close()


# ------------------------------------------------------------------------------------------- exact bounds refresh
@pytest.mark.parametrize("G", [1, 7, 32])
@pytest.mark.parametrize("D", REFRESH_D)
def test_exact_bounds_refresh(km, monkeypatch, D, G):
    """debug_yy_bounds(use_tc=False): the upper bound is the exact own distance, every group bound the fp64 minimum over
    the group's other live members, a group without one stays FLT_MAX, the dead centroid counts nowhere"""
    import torch
    from scipy.spatial.distance import cdist
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D + G)
    n, k = (600 if D <= 2049 else 200), 129
    X = T.clustered(n, D, seed=D, n_centers=16)
    C = T.perturbed_centroids(X, k, seed=D)
    groups = S._groups(k, G, rng)
    if G >= 7:
        groups[groups == G - 1] = 4                          # an empty group
    C[5] = np.nan
    groups[5] = G                                            # dead centroid: no group
    a = O.assign_lloyd(X, C)[0]
    assert (a < k).all()
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1" if tc_shape(D) else "0")
    sh = Shard(n, D, k)
    b = sh.debug_yy_bounds(torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda(),
                           torch.from_numpy(a.astype(np.int32)).cuda(), groups, G, False).cpu().numpy()
    torch.cuda.synchronize()
    assert sh.last_error() == 0
    sh.close()
    np.testing.assert_array_equal(b[:, 0], KPM.row_distances(X, C, a))
    d = cdist(X.astype(np.float64), np.nan_to_num(C.astype(np.float64)))
    d[np.arange(n), a] = np.inf                              # the own centroid goes to the upper bound only
    d[:, 5] = np.inf
    exp = np.full((n, G), np.inf)
    for g in range(G):
        members = np.flatnonzero(groups == g)
        if len(members):
            exp[:, g] = d[:, members].min(1)
    got = b[:, 1:].astype(np.float64)
    none = ~np.isfinite(exp)
    assert (got[none] == FLT_MAX).all()
    if G >= 7:
        assert none[:, G - 1].all()                           # the empty group
    assert np.all(np.abs(got[~none] - exp[~none]) <= 2e-6 * exp[~none] + 1e-30), \
        float(np.max(np.abs(got[~none] - exp[~none]) / np.maximum(exp[~none], 1e-30)))


# ------------------------------------------------------------------------------------------- Yinyang local step
YY = [(D, 0) for D in YY_D] + [(D, 1) for D in YY_COS_D]


def _slow_data(n, D, k, seed, metric=0):
    """uniform (L2) / isotropic unit (cosine) samples of at most 8 dimensions, embedded in D features, and centroids =
    samples: dozens of slow iterations whatever D, so the run leaves the Lloyd draft phase and the Yinyang local step
    does most of the work (uniform samples in thousands of dimensions are almost equidistant and converge at once)"""
    rng = np.random.default_rng(seed)
    r = min(D, 8)
    Z = rng.random((n, r)) if metric == 0 else rng.standard_normal((n, r))
    X = Z @ rng.standard_normal((r, D)) if D > r else Z
    X = T.unit(X) if metric else np.ascontiguousarray(X, np.float32)
    return X, X[rng.choice(n, k, replace=False)].copy()


def _yy_shape(D):
    return (4000, 100) if D <= 1537 else (2000, 60) if D <= 2049 else (1000, 40)


@pytest.mark.parametrize("D,metric", YY, ids=["D%d-%s" % (d, "cos" if m else "L2") for d, m in YY])
def test_yinyang_rows_kernel_equals_reference_order_scan(lib, D, metric, monkeypatch, capfd):
    """whole Yinyang runs: without a tensor-core plan, KMCUDA_B200_FORCE_EXACT 0 and 1 differ only in the local step --
    yy_rows_cta_kernel against the reference-order yy_local_scan_kernel.  Same iteration lines, assignments and
    centroids, bit for bit; the result is a Lloyd fixed point (ties aside)"""
    n, k = _yy_shape(D)
    X, C0 = _slow_data(n, D, k, D, metric)
    _pass(X[:64], C0, "cos" if metric else "L2")
    runs = {}
    for fe in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", fe)
        capfd.readouterr()
        C, A = S.c_kmeans(lib, X, C0, 1e-3, 0.1, metric, verbosity=1)
        out = capfd.readouterr().out
        runs[fe] = C, A, [ln for ln in out.splitlines() if ln.startswith("iteration") or "refreshing" in ln]
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "0")
    log = runs["0"][2]
    first = next(i for i, ln in enumerate(log) if "refreshing" in ln)
    assert any(ln.startswith("iteration") for ln in log[first:]), log
    assert runs["0"][2] == runs["1"][2]
    assert np.array_equal(runs["0"][1], runs["1"][1]), int((runs["0"][1] != runs["1"][1]).sum())
    np.testing.assert_array_equal(runs["0"][0], runs["1"][0])
    C_last, A_last = runs["0"][:2]
    assert (S.c_kmeans(lib, X, C_last, 1.0, 0.0, metric)[1] == A_last).mean() > 0.9995


# ------------------------------------------------------------------------------------------- strict runs
def _strict_data(D):
    X = T.clustered(2000, D, seed=D, n_centers=24, sigma=0.6)
    C0 = X[np.random.default_rng(D).choice(len(X), 20, replace=False)].copy()
    return X, C0


@pytest.mark.parametrize("D", STRICT_D)
def test_strict_runs_equal_the_oracle(lib, D, monkeypatch, capfd):
    """KMCUDA_B200_STRICT_UPDATE=1 Lloyd runs replay the reference's update: iteration lines, assignments and
    centroids equal the oracle's whole run bit for bit"""
    X, C0 = _strict_data(D)
    _pass(X[:64], C0)
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    capfd.readouterr()
    C, A = S.c_kmeans(lib, X, C0, 1e-3, 0.0, 0, verbosity=1)
    got = _lines(capfd.readouterr().out)
    Co, Ao, _ = O.kmeans(X, C0, tolerance=1e-3, yinyang_t=0.0, log=True)
    S._libc.fflush(None)
    want = _lines(capfd.readouterr().out)
    assert len(want) > 2 and got == want, (got, want)
    assert np.array_equal(A, Ao), int((A != Ao).sum())
    np.testing.assert_array_equal(C, Co)


def test_strict_mode_rejects_wide_samples(km, monkeypatch, capfd):
    """the strict update keeps a [D][32] centroid tile in shared memory: wider samples are rejected up front, fp16x2
    counted in features"""
    X, C0 = _strict_data(STRICT_REJECTED_D)
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    X16 = np.concatenate([X, X[:, :1]], axis=1).astype(np.float16)        # 801 pairs of halves: D = 1602
    for samples in (X, X16):
        capfd.readouterr()
        with pytest.raises(ValueError):
            km.kmeans_cuda(samples, 20, init="random", tolerance=0.01, yinyang_t=0, device=1, verbosity=1)
        assert "KMCUDA_B200_STRICT_UPDATE=1 takes at most 1600 features" in capfd.readouterr().out
    monkeypatch.delenv("KMCUDA_B200_STRICT_UPDATE")
    C, A = km.kmeans_cuda(X, 20, init=C0, tolerance=1.0, yinyang_t=0, device=1)
    assert np.array_equal(A, O.assign_lloyd(X, C0)[0])


# ------------------------------------------------------------------------------------------- member sums
@pytest.mark.parametrize("D,K,unaligned", SUMS, ids=["D%d-K%d%s" % (d, k, "-unaligned" if u else "") for d, k, u in SUMS])
def test_member_sums(km, D, K, unaligned):
    """the layout of test_member_sums_with_skewed_empty_and_unassigned_clusters at the exact route's feature counts: one
    giant cluster over many chunks, one chunk's worth, fewer rows than the unroll depth, empty clusters, unassigned
    rows; VEC 1 (D % 4 != 0 or an X that is not 16-byte aligned) and VEC 4 with several float4 columns per thread"""
    import torch
    from scipy import sparse
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D * 1000 + K)
    n = 40000 if D <= 126 else 12000
    X = (rng.standard_normal((n, D)) * 3 + 1).astype(np.float32)
    a = np.empty(n, np.int64)
    h = n // 2
    a[:h] = 5                                          # giant cluster
    a[h:h + 512] = 7                                   # one chunk's worth (kSumChunk)
    a[h + 512:h + 515] = 9                             # below the unroll depth
    q = (n - h - 515 - n // 300) // 3
    a[h + 515:h + 515 + q] = rng.integers(10, K // 2, q)
    a[h + 515 + q:n - n // 300] = rng.integers(K // 2 + 3, K, n - n // 300 - h - 515 - q)   # K//2 .. K//2+2 empty
    a[n - n // 300:] = K                               # unassigned
    a = a[rng.permutation(n)]
    flat = torch.empty(n * D + 1, device="cuda")
    Xt = flat[1:] if unaligned else flat[:-1]
    Xt = Xt.view(n, D)
    Xt.copy_(torch.from_numpy(X))
    assert (Xt.data_ptr() % 16 != 0) == unaligned
    sh = Shard(n, D, K)
    sums = torch.full((K, D), 7.0, device="cuda")
    counts = torch.full((K,), 7, dtype=torch.int32, device="cuda")
    sh.partial_sums(Xt, torch.from_numpy(a.astype(np.int32)).cuda(), sums, counts)
    torch.cuda.synchronize()
    sh.close()
    valid = np.flatnonzero(a < K)
    onehot = sparse.csr_matrix((np.ones(len(valid)), (a[valid], valid)), shape=(K, n))
    exp = onehot @ X.astype(np.float64)
    scale = onehot @ np.abs(X).astype(np.float64)
    cnt = np.bincount(a[valid], minlength=K)
    assert np.array_equal(counts.cpu().numpy(), cnt)
    got = sums.cpu().numpy().astype(np.float64)
    assert np.all(np.abs(got - exp) <= 4e-7 * scale + 1e-30), float(np.max(np.abs(got - exp) / (scale + 1e-30)))
    assert np.all(got[cnt == 0] == 0)


# ------------------------------------------------------------------------------------------- average distance
@pytest.mark.parametrize("D", AVG_D)
def test_average_distance(km, D):
    n, k = (3000 if D <= 2049 else 500), 33
    X = T.clustered(n, D, seed=D, n_centers=16)
    C0 = T.perturbed_centroids(X, k, seed=D)
    _pass(X[:64], C0)
    C, a, avg = km.kmeans_cuda(X, k, init=C0, tolerance=1.0, yinyang_t=0, device=1, average_distance=True)
    assert np.array_equal(C, C0) and np.array_equal(a, O.assign_lloyd(X, C0)[0])
    truth = np.sqrt(((X.astype(np.float64) - C0[a].astype(np.float64)) ** 2).sum(1)).mean()
    assert abs(avg - truth) <= 1e-6 * truth, (avg, truth)


# ------------------------------------------------------------------------------------------- k-NN
KNN = [(D, k) for D in KNN_D for k in KNN_K]


@pytest.mark.parametrize("D,k", KNN, ids=["D%d-k%d" % c for c in KNN])
def test_knn(km, D, k, monkeypatch, capfd):
    """the warp-per-query exact search, its sorted list crossing the 32-entry chunks of knn_list_insert (k 31 .. 65), the
    query row in shared memory (D <= 2048) or read from global memory"""
    N = 700 if D <= 2049 else 300
    X = T.clustered(N, D, seed=D + k, n_centers=12, sigma=0.3)
    C = T.perturbed_centroids(X, 12, seed=D)
    A = T.nearest(X, C)
    nb, served, _ = S._knn(km, k, X, C, A, monkeypatch, capfd)
    assert served == 0
    exp, _ = O.knn(k, X, C, A)
    # rows that differ from the oracle must list the same sequence of exact fp32 distances: the two differ only in the
    # order of samples at equal distance, or in which of them fills the last place
    for q in np.flatnonzero((nb != exp).any(1)):
        xq = np.repeat(X[q:q + 1], k, 0)
        got_d, exp_d = KPM.row_distances(xq, X, nb[q]), KPM.row_distances(xq, X, exp[q])
        assert np.array_equal(got_d, exp_d), (q, nb[q], exp[q], got_d, exp_d)
    S._check_knn(X, nb, np.arange(N), k)


# ------------------------------------------------------------------------------------------- extensions
def _ext_data(D, n=None, k=20, seed=0):
    n = n or (3000 if D <= 2049 else 800)
    X = T.clustered(n, D, seed=D + seed, n_centers=k, sigma=0.8)
    C0 = X[np.random.default_rng(D + seed).choice(n, k, replace=False)].copy()
    _pass(X[:64], C0)
    return X, C0


def _run(km, capfd, X, k, **kw):
    capfd.readouterr()
    out = km.kmeans_cuda(X, k, device=1, verbosity=1, **kw)
    return out, capfd.readouterr().out


@pytest.mark.parametrize("D", EXT_D)
def test_all_ones_weights_are_bit_identical(km, capfd, D):
    X, C0 = _ext_data(D)
    kw = dict(init=C0, tolerance=0.001, yinyang_t=0.1, seed=7, average_distance=True)
    (c1, a1, d1), o1 = _run(km, capfd, X, 20, **kw)
    (c2, a2, d2), o2 = _run(km, capfd, X, 20, sample_weight=np.ones(len(X)), **kw)
    assert _same(c1, c2) and np.array_equal(a1, a2) and d1 == d2
    assert _lines(o1) == _lines(o2) and len(_lines(o1)) > 2


@pytest.mark.parametrize("D", EXT_D)
def test_minibatch_matches_the_model(km, capfd, D):
    X, C0 = _ext_data(D)
    b, steps, seed = 256, 6, 11
    (C, a), out = _run(km, capfd, X, 20, init=C0, yinyang_t=0, tolerance=0.0, seed=seed, batch_size=b,
                       max_steps=steps)
    got = MBG._steps(_lines(out, "mini-batch"))
    mc, mlog, _, _ = MBM.run(X, C0, b, steps, 0.0, seed, lambda Xb, Cm: O.assign_lloyd(Xb, Cm)[0].astype(np.int64))
    assert len(got) == len(mlog) == steps
    for g, m in zip(got, mlog):
        assert g[0] == m[0] and abs(g[1] - m[1]) <= 1e-5 * abs(m[1]), (g, m)
        assert (g[2] is None) == (m[2] is None)
        if m[2] is not None:
            assert abs(g[2] - m[2]) <= 1e-5 * abs(m[2]), (g, m)
    np.testing.assert_allclose(C, mc, rtol=1e-5, atol=1e-5 * float(np.abs(mc).max()))
    assert np.array_equal(a, O.assign_lloyd(X, C)[0])


def test_kmeans_parallel_matches_the_model(km, capfd):
    D = EXT_D[0]
    X = T.clustered(3000, D, seed=D, n_centers=20, sigma=0.8)
    _pass(X[:64], X[:20])
    c, klog = KPG._init(km, capfd, X, 20)
    rows, lines, cm = KPG._model_centroids(km, X, 20, "L2", None)
    KPG._check_log(klog, lines)
    assert len(rows) > 20
    assert _same(c, cm)


def test_relocation_matches_the_model(km, capfd):
    """D = 1030: the relocation keys (staged_own_sum) end in a slice of 6 features, off the float4 path"""
    D = EXT_D[0]
    X = RG._blobs(3000, D, 20)
    C0 = RG._init_with_empties(X, 20, 3)
    _pass(X[:64], C0)
    (C, a), lines = RG._run(km, capfd, X, 20, C0, relocate_empty_clusters=True)
    mC, ma, mlog = RM.run(X, C0, RG._labeler(0))
    RG._check_against_model(lines, mlog, C, mC, a, ma)
    assert any(rec for _, _, rec, _ in mlog)


@pytest.mark.parametrize("D", EXT_D)
def test_device_kmeanspp_picks_the_host_walks_rows(km, monkeypatch, D):
    X, _ = _ext_data(D)
    got = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_HOST_PLUSPLUS", mode)
        got[mode] = km.kmeans_cuda(X, 20, init="k-means++", tolerance=1.0, yinyang_t=0, seed=11, device=1)
    monkeypatch.delenv("KMCUDA_B200_HOST_PLUSPLUS")
    assert _same(got["0"][0], got["1"][0]) and np.array_equal(got["0"][1], got["1"][1])
    rows = {X[i].tobytes(): i for i in range(len(X))}
    assert len({rows[c.tobytes()] for c in got["0"][0]}) == 20     # 20 distinct sample rows


def test_fp16_samples_with_an_odd_feature_count(km, capfd):
    """fp16x2 samples of 513 packed pairs (D = 1026, D % 4 == 2): the run equals the fp32 run on the widened samples"""
    X, _ = _ext_data(FP16_D)
    X16 = X.astype(np.float16)
    kw = dict(init="random", tolerance=0.001, yinyang_t=0.1, seed=5)
    (c16, a16), o16 = _run(km, capfd, X16, 20, **kw)
    (c32, a32), o32 = _run(km, capfd, X16.astype(np.float32), 20, **kw)
    assert np.array_equal(a16, a32) and _lines(o16) == _lines(o32) and len(_lines(o32)) > 2
    assert np.array_equal(c16.view(np.uint16), c32.astype(np.float16).view(np.uint16))


# ------------------------------------------------------------------------------------------- every accepted D
@pytest.mark.parametrize("D", ACCEPT_D)
def test_every_accepted_d_runs(km, capfd, D):
    """a default call (k-means++, Yinyang) and a mini-batch call at the widest feature counts return 0 and end on the
    oracle's assignment of their centroids"""
    n, k = (1200 if D < 65535 else 400), 33
    X, _ = _slow_data(n, D, k, D)
    _pass(X[:64], X[:k])
    (C, a), out = _run(km, capfd, X, k, seed=3)
    log = out.splitlines()
    first = next(i for i, ln in enumerate(log) if ln.startswith("refreshing Yinyang bounds"))
    assert any(ln.startswith("iteration") for ln in log[first:]), log
    assert (a == O.assign_lloyd(X, C)[0]).mean() > 0.999
    (C, a), out = _run(km, capfd, X, k, seed=3, yinyang_t=0, batch_size=128, max_steps=3)
    assert len(_lines(out, "mini-batch step")) == 3
    assert np.array_equal(a, O.assign_lloyd(X, C)[0])

