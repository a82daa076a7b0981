"""GPU tests of mini-batch k-means (kmeans_cuda(..., batch_size=b); include/kmcuda_b200.h, DESIGN.md §4h).

The run is pinned to its NumPy model (tests/minibatch_model.py), which takes its batch labels from the oracle: every
logged mean batch inertia and EWA, and the final centroids, to 1e-5 relative.  Shapes as in
test_kmeans_parallel_gpu.py: 50000 x 64 @ 200 takes the tensor-core assignment, 20000 x 30 @ 50 the exact one."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import minibatch_model as M  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {"tc": (50000, 64, 200), "exact": (20000, 30, 50)}
SEED = 11
BATCH = 1024
STEP = re.compile(r"mini-batch step (\d+)/(\d+): mean batch inertia ([^,\s]+)(?:, ewa inertia (\S+))?")


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


def _blobs(n, d, k, seed=0, spread=0.6):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)
    return X


def _init(X, k, seed=1):
    return X[np.random.default_rng(seed).choice(len(X), k, replace=False)].copy()


def _weights(kind, n):
    if kind == "none":
        return None
    rng = np.random.default_rng(5)
    w = rng.integers(1, 5, n).astype(np.float32)
    if kind == "zeros":
        w[rng.random(n) < 0.3] = 0
    return w


def _run(km, capfd, X, k, C0, **kw):
    capfd.readouterr()
    kw.setdefault("seed", SEED)
    kw.setdefault("batch_size", BATCH)
    kw.setdefault("tolerance", 0.0)
    out = km.kmeans_cuda(X, k, init=C0, device=1, verbosity=1, yinyang_t=0, **kw)
    lines = capfd.readouterr().out.splitlines()
    return out, [ln for ln in lines if ln.startswith("mini-batch")], lines


def _steps(log):
    return [(int(m.group(1)), float(m.group(3)), None if m.group(4) is None else float(m.group(4)))
            for m in map(STEP.match, log) if m]


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _oracle_labels(Xb, C):
    return O.assign_lloyd(Xb.astype(np.float32), C)[0].astype(np.int64)


# ------------------------------------------------------------------------------------------------ 1. model pin
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("steps", [1, 3, 20])
@pytest.mark.parametrize("weights", ["none", "zeros"])
def test_run_matches_the_model(km, capfd, shape, steps, weights):
    n, d, k = SHAPES[shape]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    w = _weights(weights, n)
    (C, a), log, _ = _run(km, capfd, X, k, C0, max_steps=steps, sample_weight=w)
    mc, mlog, reason, done = M.run(X, C0, BATCH, steps, 0.0, SEED, _oracle_labels, w=w)
    got = _steps(log)
    assert len(got) == len(mlog), (log[-3:], reason)
    for g, m in zip(got, mlog):
        assert g[0] == m[0]
        assert abs(g[1] - m[1]) <= 1e-5 * abs(m[1]), "first differing step %d: %r vs %r" % (g[0], g, m)
        assert (g[2] is None) == (m[2] is None)
        if m[2] is not None:
            assert abs(g[2] - m[2]) <= 1e-5 * abs(m[2]), "first differing step %d: %r vs %r" % (g[0], g, m)
    scale = float(np.abs(mc).max())
    np.testing.assert_allclose(C, mc, rtol=1e-5, atol=1e-5 * scale)
    assert np.array_equal(a, O.assign_lloyd(X, C)[0])


# ------------------------------------------------------------------------------------------------ 2. routes, bits
@pytest.mark.parametrize("weights", ["none", "zeros"])
def test_forced_exact_route_is_bit_identical(km, capfd, monkeypatch, weights):
    n, d, k = SHAPES["tc"]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    w = _weights(weights, n)
    (c1, a1), l1, _ = _run(km, capfd, X, k, C0, max_steps=30, sample_weight=w)
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1")
    (c2, a2), l2, _ = _run(km, capfd, X, k, C0, max_steps=30, sample_weight=w)
    assert _same(c1, c2) and np.array_equal(a1, a2) and l1 == l2


@pytest.mark.parametrize("shape", list(SHAPES))
def test_all_ones_weights_and_same_seed_are_bit_identical(km, capfd, shape):
    n, d, k = SHAPES[shape]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    (c1, a1, d1), l1, _ = _run(km, capfd, X, k, C0, max_steps=25, average_distance=True)
    (c2, a2, d2), l2, _ = _run(km, capfd, X, k, C0, max_steps=25, average_distance=True, sample_weight=np.ones(n))
    (c3, a3, d3), l3, _ = _run(km, capfd, X, k, C0, max_steps=25, average_distance=True)
    (c4, _), l4, _ = _run(km, capfd, X, k, C0, max_steps=25, seed=SEED + 1)
    assert _same(c1, c2) and np.array_equal(a1, a2) and d1 == d2 and l1 == l2
    assert _same(c1, c3) and np.array_equal(a1, a3) and d1 == d3 and l1 == l3
    assert not _same(c1, c4)


# ------------------------------------------------------------------------------------------------ 3. stopping
def test_stopping_rules(km, capfd):
    n, d, k = SHAPES["tc"]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    _, log, _ = _run(km, capfd, X, k, C0, max_steps=7)
    assert [s for s, _, _ in _steps(log)] == list(range(1, 8))
    assert log[-1] == "mini-batch: 7 steps"
    _, log, _ = _run(km, capfd, X, k, C0, tolerance=0.5)
    assert re.fullmatch(r"mini-batch: converged \(small centers change\) at step \d+/%d" % (100 * n // BATCH), log[-1])
    # runs with the default max_steps (0: 100 epochs) on converged data: the default tolerance (0.01) ends them by the
    # small centre change (measured: step 123 of 4882), and without a tolerance only the lack of improvement ends them
    C1, _ = km.kmeans_cuda(X, k, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3)
    capfd.readouterr()
    km.kmeans_cuda(X, k, init=C1, device=1, verbosity=1, yinyang_t=0, seed=SEED, batch_size=BATCH)
    log = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("mini-batch")]
    assert re.fullmatch(r"mini-batch: converged \(small centers change\) at step \d+/%d" % (100 * n // BATCH), log[-1])
    assert len(_steps(log)) < 100 * n // BATCH
    _, log, _ = _run(km, capfd, X, k, C1, tolerance=0.0)
    assert "lack of improvement in inertia" in log[-1], log[-1]
    assert len(_steps(log)) < 100 * n // BATCH


def test_batch_larger_than_n_is_clamped(km, capfd):
    n, d, k = 3000, 32, 20
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    (c1, a1), l1, _ = _run(km, capfd, X, k, C0, max_steps=4, batch_size=10 ** 6)
    (c2, a2), l2, _ = _run(km, capfd, X, k, C0, max_steps=4, batch_size=n)
    assert _same(c1, c2) and l1 == l2
    mc, mlog, _, _ = M.run(X, C0, n, 4, 0.0, SEED, _oracle_labels)
    np.testing.assert_allclose(c1, mc, rtol=1e-5, atol=1e-5 * float(np.abs(mc).max()))


# ------------------------------------------------------------------------------------------------ 4. row-list pass
D_ENDS = [4, 64, 68, 128, 132, 192, 196, 256, 260, 320, 324, 384, 388, 448, 452, 512]


@pytest.mark.parametrize("D", D_ENDS)
@pytest.mark.parametrize("K", [2, 129, 1000])
def test_assign_rows_matches_exact_and_oracle(km, monkeypatch, D, K):
    import torch
    from kmcuda_b200.shard import Shard
    rng = np.random.default_rng(D * 7 + K)
    N = 900
    X = rng.standard_normal((N, D)).astype(np.float32)
    C = (X[rng.choice(N, K, replace=K > N)] + 0.01 * rng.standard_normal((K, D))).astype(np.float32)
    X[5, 0] = np.nan      # overflow path: a non-finite row goes to the exact list pass, resolved by position
    X[7] *= 1e4           # far from every centroid
    lists = {
        "overflow_dupes": np.array([5, 5, 7, 3, 5, 7]),
        "dupes_ragged": rng.integers(0, N, 517),                          # duplicates, last tile of 5 rows
        "one": np.array([N - 1]),
        "longer_than_n": np.concatenate([np.arange(N), rng.integers(0, N, 300)]),
    }
    Xt, Ct = torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda()
    tc = Shard(1200, D, K)
    monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", "1")
    ex = Shard(1200, D, K)
    for name, rows in lists.items():
        r = torch.from_numpy(rows.astype(np.int32))
        got = tc.debug_assign_rows(Xt, Ct, r).cpu().numpy().view(np.uint32)
        want = ex.debug_assign_rows(Xt, Ct, r).cpu().numpy().view(np.uint32)
        oracle = O.assign_lloyd(X[rows], C)[0]
        assert np.array_equal(got, want), name
        assert np.array_equal(got, oracle), name
        assert tc.last_error() == 0
    assert tc.last_pass_info()[0], "the tensor-core route did not run"


# ------------------------------------------------------------------------------------------------ 5. quality
def test_quality_against_scikit_learn_and_lloyd(km, capfd):
    """Final full-data inertia from the same init, tol = 0, both with max_no_improvement = 10 and at most 195 steps
    (4 epochs of 50000 x 64 @ 200 blobs, b = 1024); either run may stop early by that rule.  Measured on an H100 80GB
    HBM3: the library stopped after 161 steps, scikit-learn after 176; 1.0134 x scikit-learn's MiniBatchKMeans and
    0.4917 x the library's full Lloyd run from the same centroids (Lloyd keeps the init's empty and doubled blobs; the
    random reassignment moves them).  Bounds: 1.05 x and 0.6 x."""
    from sklearn.cluster import MiniBatchKMeans
    n, d, k = SHAPES["tc"]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    epochs = 4
    steps = epochs * n // BATCH   # scikit-learn's step count for max_iter = epochs
    (C, a), log, _ = _run(km, capfd, X, k, C0, max_steps=steps)
    taken = len(_steps(log))
    assert taken == steps or "lack of improvement" in log[-1], log[-1]
    mine = float(((X.astype(np.float64) - C[a]) ** 2).sum())
    sk = MiniBatchKMeans(n_clusters=k, batch_size=BATCH, max_iter=epochs, tol=0.0, init=C0, n_init=1,
                         max_no_improvement=10, random_state=0, reassignment_ratio=0.01).fit(X)
    sk_inertia = float(((X.astype(np.float64) - sk.cluster_centers_[sk.labels_]) ** 2).sum())
    CL, aL = km.kmeans_cuda(X, k, init=C0, tolerance=0.0, yinyang_t=0, device=1, seed=3)
    lloyd = float(((X.astype(np.float64) - CL[aL]) ** 2).sum())
    print("steps %d (scikit-learn %d); mini-batch / scikit-learn = %.4f, mini-batch / Lloyd = %.4f"
          % (taken, sk.n_steps_, mine / sk_inertia, mine / lloyd))
    assert mine <= 1.05 * sk_inertia
    assert mine <= 0.6 * lloyd


# ------------------------------------------------------------------------------------------------ 6. arguments
def test_rejected_arguments(km, monkeypatch):
    X = _blobs(2000, 16, 10)
    Xn = X / np.linalg.norm(X, axis=1, keepdims=True)
    with pytest.raises(ValueError):
        km.kmeans_cuda(Xn, 10, metric="cos", batch_size=256, device=1)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, batch_size=256, device=3)
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, batch_size=0, device=1)
    monkeypatch.setenv("KMCUDA_B200_STRICT_UPDATE", "1")
    with pytest.raises(ValueError):
        km.kmeans_cuda(X, 10, batch_size=256, device=1)


def test_fp16_and_device_pointer_samples_run(km, capfd):
    import torch
    n, d, k = SHAPES["tc"]
    X = _blobs(n, d, k)
    C0 = _init(X, k)
    Xh = X.astype(np.float16)
    # fp16x2 samples are widened on ingest: the run equals the fp32 run on the widened values (random init: same rows)
    (ch, ah), lh, _ = _run(km, capfd, Xh, k, "random", max_steps=10)
    (cf, af), lf, _ = _run(km, capfd, Xh.astype(np.float32), k, "random", max_steps=10)
    assert lh == lf and np.array_equal(ah, af)
    assert np.array_equal(ch.view(np.uint16), cf.astype(np.float16).view(np.uint16))
    Xt = torch.from_numpy(X).cuda()
    Ct = torch.from_numpy(C0).cuda()
    at = torch.empty(n, dtype=torch.int32, device="cuda")
    capfd.readouterr()
    km.kmeans_cuda((Xt.data_ptr(), 0, (n, d), Ct.data_ptr(), at.data_ptr()), k, init=C0, device=1, verbosity=1,
                   yinyang_t=0, tolerance=0.0, seed=SEED, batch_size=BATCH, max_steps=10)
    torch.cuda.synchronize()
    ld = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("mini-batch")]
    (c, a), l2, _ = _run(km, capfd, X, k, C0, max_steps=10)
    assert ld == l2
    assert _same(Ct.cpu().numpy(), c) and np.array_equal(at.cpu().numpy().view(np.uint32), a)
