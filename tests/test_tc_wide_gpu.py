"""The tensor-core Lloyd pass at 512 < D <= 1024 (assign_tc.cu, NKB 9..16: 64-row tiles, the two consumer warpgroups on
the same rows and one 64-column half of every n-tile each).  Run on an H100: `pytest -m gpu`.

Checkers as in test_tc_sweep_gpu.py: the CPU oracle (`oracle.assign_lloyd`), this library's exact route
(`KMCUDA_B200_FORCE_EXACT=1`) and fp64 truth for cosine near-ties.  Covered here:
- MODE 0 at both ends of every NKB range (D 516 / 576 .. 964 / 1024), K in {2, 127, 128, 129, 1000} (+ 5000), fewer
  64-row tiles than SMs, more than two per SM, N = 1 and N = 100; cosine and near-tie pairs once per NKB;
- the filter's slow paths at NKB 12 and 16 (tc_sweep_cases' adversarial inputs, whose special centroids all sit in the
  first warpgroup's half), duplicates across the two halves, and a winner in the second half whose rows' first-half
  maximum is lower (the emitters' threshold must use the larger of the two warpgroup maxima);
- the row-list pass (Shard::assign_rows) over the same D range;
- whole runs at D = 768, each bit-identical to the forced-exact run, logs included;
- that the 64-row kernels ran (torch.profiler), and, with oracle/_ref built, one pass equal to the reference library.
"""
import functools
import os
import re

import numpy as np
import pytest

import tc_sweep_cases as T
from oracle import oracle as O
from test_tc_sweep_gpu import check_oracle, run_pass

pytestmark = pytest.mark.gpu

TR = 64                                           # sample rows per tile at NKB 9..16
WIDE_D = [d for nkb in range(9, 17) for d in (64 * (nkb - 1) + 4, 64 * nkb)]   # 516, 576, 580, 640, ..., 964, 1024
NKB_D = [64 * nkb for nkb in range(9, 17)]
K_SET = [2, 127, 128, 129, 1000]


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    O.set_threads(os.cpu_count())
    return kmcuda_b200


@pytest.fixture(scope="module")
def sms(km):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def wide_n(label, num_sms):
    """'few': fewer 64-row tiles than SMs; 'many': more than two per SM plus a ragged last tile"""
    if label == "few":
        return TR * max(1, num_sms // 2) + 37
    if label == "many":
        return TR * (2 * num_sms + 5) + 45
    return int(label)


# ------------------------------------------------------------------------------------------- MODE 0 sweep
def _sweep_cases():
    out = []
    for D in WIDE_D:
        for nl in ("few", "many"):
            out += [(D, K, nl, "L2", "plain") for K in K_SET + ([5000] if D in (580, 1024) else [])]
        if D in NKB_D:
            out += [(D, K, "many", "cos", "plain") for K in (129, 1000)]
            out.append((D, 1000, "many", "L2", "near_ties"))
            out.append((D, 1000, "many", "cos", "near_ties"))
        if D in (516, 1024):
            out += [(D, K, nl, "L2", "plain") for nl in ("1", "100") for K in K_SET]
    return out


SWEEP = _sweep_cases()


@functools.lru_cache(maxsize=2)
def _samples(N, D, metric):
    X = T.clustered(N, D, seed=D)
    return T.unit(X) if metric == "cos" else X


@functools.lru_cache(maxsize=4)
def _centroids(N, D, K, metric, variant):
    pool = _samples(max(N, 4096), D, metric)
    C = T.perturbed_centroids(pool, K, seed=K + D, near_ties=variant == "near_ties")
    return T.unit(C) if metric == "cos" else C


@pytest.mark.parametrize("D,K,nl,metric,variant", SWEEP, ids=["D%d-K%d-N%s-%s-%s" % c for c in SWEEP])
def test_wide_lloyd_pass_sweep(km, sms, D, K, nl, metric, variant):
    N = wide_n(nl, sms)
    X, C = _samples(N, D, metric), _centroids(N, D, K, metric, variant)
    a, prev, changed, info = run_pass(X, C, metric)
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


@pytest.mark.parametrize("D", [576, 768, 1024])
def test_wide_lloyd_pass_bookkeeping(km, sms, D):
    N, K = wide_n("few", sms), 129
    X = _samples(N, D, "L2")
    C = T.perturbed_centroids(X, K, seed=D, near_ties=True)
    C2 = C + (0.05 * np.abs(C).mean() * np.random.default_rng(D).standard_normal(C.shape)).astype(np.float32)
    a_in = O.assign_lloyd(X, C2)[0]
    a_exp, _, ch_exp = O.assign_lloyd(X, C, assign=a_in)
    a, prev, changed, _ = run_pass(X, C, assign=a_in)
    assert np.array_equal(prev, a_in)
    assert np.array_equal(a, a_exp), int((a != a_exp).sum())
    assert changed == ch_exp and 0 < changed < N


# ------------------------------------------------------------------------------------------- slow paths
SLOW = [(k, D) for k in T.LIST_CASES for D in (768, 1024)]


@pytest.mark.parametrize("kind,D", SLOW, ids=["%s-D%d" % c for c in SLOW])
def test_wide_filter_slow_paths(km, kind, D):
    """list compaction, a full per-lane list (flag bit 2), > MAX_CAND candidates, a full pair queue, duplicates: the
    exact winner is placed where a kernel that mishandles the path picks another index"""
    X, C, info = T.list_case(kind, D)
    a, _, _, pi = run_pass(X, C)
    e = run_pass(X, C, force_exact=True)[0]
    assert np.array_equal(a, e), "%d rows differ from the exact pass" % int((a != e).sum())
    check_oracle(X, C, a, "L2")
    for rows, win in zip(info["rows"], info["winner"]):
        assert (a[rows] == win).all(), (win, np.unique(a[rows]))
    rechecked, overflowed = pi[1], pi[2]
    if kind in ("rise", "rise_pair", "rise_coarse"):
        assert rechecked == 0 and overflowed == 0
    elif kind == "rise_wide":
        assert rechecked == len(X) and overflowed == 0
    elif kind in ("rise_margin", "dupes"):
        assert rechecked > 0 and overflowed == 0
    elif kind in ("list_overflow", "max_cand"):
        assert overflowed > 0
    else:
        assert rechecked > 0 and overflowed > 0


def _halves_case(kind, D, seed=0):
    """8 groups of 32 near-identical rows, special centroids placed as in tc_sweep_cases.list_case.
    'split': the winner at column 64 + 8 g + 5 of n-tile 3 (second warpgroup); in the first half, column 8 g + 5 of
    n-tiles 0..3 sits 4 margins below it and is its half's maximum, so the first warpgroup keeps it as a candidate of
    its own (lower) threshold and only the merged threshold drops it: exactly one candidate per row.
    'dupes': one centroid at three indices, the lowest (64 + 8 g + 7, second half, emitted last) must win."""
    rng = np.random.default_rng(seed + D + len(kind))
    n_groups, rows_per, K = 8, 32, T.LIST_K
    C = rng.standard_normal((K, D))
    xg = rng.standard_normal((n_groups, D))
    gid = np.repeat(np.arange(n_groups), rows_per)
    X = np.ascontiguousarray(xg[gid] + 1e-6 * rng.standard_normal((len(gid), D)), np.float32)
    if kind == "split":
        layout = [[(8 * g + 5 + T.TN * t, 0.0) for t in range(4)] + [(T.TN * 3 + 64 + 8 * g + 5, 4.0)]
                  for g in range(n_groups)]
    else:
        layout = [[(64 + 8 * g + 7, 1.0), (T.TN + 8 * g + 1, 0.0), (2 * T.TN + 8 * g + 3, 0.0)] for g in range(n_groups)]
    rows = [np.flatnonzero(gid == g) for g in range(n_groups)]
    place_seed = int(rng.integers(1 << 31))

    def build(delta):
        Cb = C.copy()
        grng = np.random.default_rng(place_seed)
        for g, spec in enumerate(layout):
            R2 = (max(f for _, f in spec) + 40.0) * delta[g]
            for idx, f in spec:
                Cb[idx] = T._place(xg[g], R2 - f * delta[g], grng, "L2")
            if kind == "dupes":
                for idx, _ in spec[1:]:
                    Cb[idx] = Cb[spec[0][0]]
        return np.ascontiguousarray(Cb, np.float32)

    delta = np.full(n_groups, 1e-3 * D)
    for _ in range(2):
        mg, s = T.margins(X, build(delta))
        delta = np.array([np.median(2.0 * mg[r] / (s * s)) for r in rows])
    winner = [spec[0][0] if kind == "dupes" else spec[-1][0] for spec in layout]
    return X, build(delta), rows, winner


@pytest.mark.parametrize("kind", ["split", "dupes"])
@pytest.mark.parametrize("D", [768, 1024])
def test_wide_column_halves(km, kind, D):
    X, C, rows, winner = _halves_case(kind, D)
    a, _, _, pi = run_pass(X, C)
    e = run_pass(X, C, force_exact=True)[0]
    assert np.array_equal(a, e), "%d rows differ from the exact pass" % int((a != e).sum())
    check_oracle(X, C, a, "L2")
    for r, win in zip(rows, winner):
        assert (a[r] == win).all(), (win, np.unique(a[r]))
    if kind == "split":
        assert pi[1] == 0 and pi[2] == 0, pi          # one candidate per row: the first half's entries were dropped
    else:
        assert pi[1] > 0 and pi[2] == 0, pi


@pytest.mark.parametrize("D", [768, 1024])
def test_wide_non_finite_and_far_rows(km, D):
    X, C = T.nonfinite_case(D)
    a, _, _, info = run_pass(X, C)
    e = run_pass(X, C, force_exact=True)[0]
    assert np.array_equal(a, e), np.flatnonzero(a != e)[:10]
    exp = check_oracle(X, C, a, "L2")
    assert info[2] > 0
    assert (a[10:20] == 6).all() and (a[20:30] == 3).all()
    assert not np.isin(a[exp != T.UNTOUCHED], [40, 41, 170]).any()


# ------------------------------------------------------------------------------------------- row-list pass
@pytest.mark.parametrize("D", WIDE_D)
@pytest.mark.parametrize("K", [2, 129, 1000])
def test_wide_assign_rows(km, monkeypatch, D, K):
    import torch
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D * 7 + K)
    N = 900
    X = rng.standard_normal((N, D)).astype(np.float32)
    C = (X[rng.choice(N, K, replace=K > N)] + 0.01 * rng.standard_normal((K, D))).astype(np.float32)
    X[5, 0] = np.nan
    X[7] *= 1e4
    lists = {
        "overflow_dupes": np.array([5, 5, 7, 3, 5, 7]),
        "dupes_ragged": rng.integers(0, N, 517),
        "one": np.array([N - 1]),
        "longer_than_n": np.concatenate([np.arange(N), rng.integers(0, N, 300)]),
    }
    Xt, Ct = torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda()
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "0")
    tc = Shard(1200, D, K)
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1")
    ex = Shard(1200, D, K)
    for name, rows in lists.items():
        r = torch.from_numpy(rows.astype(np.int32))
        got = tc.debug_assign_rows(Xt, Ct, r).cpu().numpy().view(np.uint32)
        want = ex.debug_assign_rows(Xt, Ct, r).cpu().numpy().view(np.uint32)
        assert np.array_equal(got, want), name
        assert np.array_equal(got, O.assign_lloyd(X[rows], C)[0]), name
        assert tc.last_error() == 0
    assert tc.last_pass_info()[0], "the tensor-core route did not run"
    tc.close()
    ex.close()


# ------------------------------------------------------------------------------------------- whole runs, D = 768
RUN_LINE = re.compile(r"^(iteration \d+: \d+ reassignments|mini-batch .*|refreshing.*|.*=> Lloyd)$")


def _blobs(n, d, k, seed=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k // 4, d)).astype(np.float32)
    return (centers[rng.integers(0, len(centers), n)] + 0.8 * rng.standard_normal((n, d))).astype(np.float32)


RUNS = ["lloyd", "yinyang", "weighted", "kmeans_parallel", "minibatch", "fp16"]


@pytest.mark.parametrize("run", RUNS)
def test_wide_runs_equal_forced_exact(km, run, monkeypatch, capfd):
    n, d, k = 30000, 768, 1000
    X = _blobs(n, d, k)
    C0 = X[np.random.default_rng(1).choice(n, k, replace=False)].copy()
    kw = dict(init=C0, tolerance=1e-3, yinyang_t=0.0, device=1, verbosity=1, seed=5)
    if run == "yinyang":
        kw["yinyang_t"] = 0.1
    elif run == "weighted":
        kw["sample_weight"] = np.random.default_rng(2).integers(0, 4, n).astype(np.float32)
    elif run == "kmeans_parallel":
        kw["init"] = "k-means||"
    elif run == "minibatch":
        kw.update(batch_size=4096, max_steps=40, tolerance=0.0)
    elif run == "fp16":
        X = X.astype(np.float16)
        kw["init"] = C0.astype(np.float16).view(np.float32)
    out = {}
    for fe in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", fe)
        capfd.readouterr()
        C, A = km.kmeans_cuda(X, k, **kw)
        lines = [ln for ln in capfd.readouterr().out.splitlines() if RUN_LINE.match(ln)]
        out[fe] = C, A, lines
    assert len(out["0"][2]) > 2, out["0"][2]
    assert out["0"][2] == out["1"][2]
    assert np.array_equal(out["0"][1], out["1"][1]), int((out["0"][1] != out["1"][1]).sum())
    assert np.array_equal(np.asarray(out["0"][0]).view(np.uint32), np.asarray(out["1"][0]).view(np.uint32))


def test_wide_kernels_ran(km):
    """a silent exact fallback cannot pass: the MODE 0 and row-list kernels of the 64-row layout show up in the trace"""
    from torch.profiler import ProfilerActivity, profile
    X = _blobs(20000, 768, 300)
    C0 = X[:300].copy()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        km.kmeans_cuda(X, 300, init=C0, tolerance=1e-2, yinyang_t=0.0, device=1)
        km.kmeans_cuda(X, 300, init=C0, tolerance=0.0, yinyang_t=0.0, device=1, batch_size=2048, max_steps=3)
    names = {e.name for e in prof.events() if "tc_assign" in e.name}
    assert any("tc_assign_kernel<12, 0>" in nm for nm in names), names
    assert any("tc_assign_rows_kernel<12>" in nm for nm in names), names


def test_wide_pass_matches_reference():
    if not O.reference_available():
        pytest.skip("oracle/_ref/libKMCUDA.so not built")
    import ctypes
    ref = O.reference_lib()
    rng = np.random.default_rng(768)
    n, d, k = 100000, 768, 1000
    X = _blobs(n, d, k, seed=3)
    C = X[rng.choice(n, k, replace=False)].copy()
    a, prev, changed, info = run_pass(X, C)
    assert info[2] < n // 20, info
    A = np.zeros(n, np.uint32)
    Cr = C.copy()
    m = ctypes.c_uint32(0)
    rc = ref.kmeans_cuda(3, ctypes.byref(m), 1.0, 0.0, 0, n, d, k, 3, 1, -1, 0, 0, X.ctypes.data, Cr.ctypes.data,
                         A.ctypes.data, None)
    assert rc == 0, rc
    assert np.array_equal(a, A), int((a != A).sum())
