"""knn_cuda on the tensor cores at 512 < D <= 1024 (assign_tc.cu MODE 2 on 64-row tiles, DESIGN §4j).  Run on an
H100: `pytest -m gpu`.

The neighbour lists are exact on both routes, so every check compares with fp64 truth (`_check_knn`) and with the
forced-exact search (`KMCUDA_B200_FORCE_EXACT=1`) wherever the k-th and (k+1)-th neighbours are not near-ties.
Covered here:
- both ends of every NKB range (D 516 / 576 .. 964 / 1024) x k in {1, 15} x N in {4096 (the tensor-core route), 4095
  (the exact search)};
- the cluster shapes of test_tc_sweep_gpu (tiny clusters, one giant cluster, duplicates that fill the entry lists) at
  D = 768 and 1024;
- clusters whose sizes leave the second 64-row half of a 128-row table block empty or partly filled;
- unit-length data with the angular metric (served through the L2 pass), fp16 samples and device-pointer inputs;
- that `tc_assign_kernel<12, 2>` ran (torch.profiler); with oracle/_ref built, one call equal to the reference
  library; with two GPUs, the query-tile shards equal the one-GPU answer.
"""
import os

import numpy as np
import pytest

import tc_sweep_cases as T
from oracle import oracle as O
from test_tc_sweep_gpu import _check_knn, _knn

pytestmark = pytest.mark.gpu

WIDE_D = [d for nkb in range(9, 17) for d in (64 * (nkb - 1) + 4, 64 * nkb)]   # 516, 576, 580, 640, ..., 964, 1024


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    O.set_threads(os.cpu_count())
    return kmcuda_b200


def _served(capfd_err):
    line = [ln for ln in capfd_err.splitlines() if "knn tensor-core path" in ln]
    if not line:
        return 0
    assert "error word 0x0;" in line[0], line[0]
    return int(line[0].split("path:")[1].split("rows")[0])


KNN = [(D, k, N) for D in WIDE_D for k in (1, 15) for N in (4096, 4095)]


@pytest.mark.parametrize("D,k,N", KNN, ids=["D%d-k%d-N%d" % c for c in KNN])
def test_wide_knn_sweep(km, D, k, N, monkeypatch, capfd):
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
@pytest.mark.parametrize("D", [768, 1024])
def test_wide_knn_cluster_shapes(km, kind, D, monkeypatch, capfd):
    X, C, A = T.knn_shape(kind, D)
    if kind == "duplicates":
        # a part records one 32-column chunk per n-tile (two per half at 128 rows), so the 4000 copies (32 blocks) do
        # not fill its KNN_CAP = 40 entries: 2000 more copies make the tie group 47 blocks long
        X = np.concatenate([X, np.repeat(X[-1:], 2000, axis=0)])
        A = T.nearest(X, C)
    k = 15
    nb, served, list_full = _knn(km, k, X, C, A, monkeypatch, capfd)
    assert served > 0, "tensor-core k-NN path not taken"
    if kind == "duplicates":
        assert list_full > 0, "no row part filled its KNN_CAP entries"
    ex, _, _ = _knn(km, k, X, C, A, monkeypatch, capfd, force_exact=True)
    rng = np.random.default_rng(D)
    queries = np.sort(np.concatenate([rng.choice(len(X) - 6000, 400, replace=False),
                                      len(X) - 6000 + rng.choice(6000, 100, replace=False)]))
    _check_knn(X, nb, queries, k, ref=ex)


def _sized_clusters(sizes, D, seed):
    """well separated clusters of the given sizes: the fp64 nearest centroid is the planned one"""
    rng = np.random.default_rng(seed)
    centers = (rng.standard_normal((len(sizes), D)) * 4.0).astype(np.float32)
    lab = np.repeat(np.arange(len(sizes)), sizes)
    X = (centers[lab] + 0.3 * rng.standard_normal((len(lab), D))).astype(np.float32)
    A = T.nearest(X, centers)
    assert np.array_equal(A, lab)
    return X, centers, A


@pytest.mark.parametrize("fill", ["empty", "partial"])
def test_wide_knn_half_filled_blocks(km, fill, monkeypatch, capfd):
    """a cluster's last 128-row block holds size % 128 rows: 1..64 leave its second 64-row query tile without live
    rows (skipped), 65..127 leave it partly filled"""
    D, k = 768, 15
    if fill == "empty":
        sizes = [1, 17, 63, 64, 128 + 1, 128 + 40, 256 + 64] * 6
    else:
        sizes = [65, 66, 100, 127, 128 + 65, 128 + 120, 256 + 99] * 6
    X, C, A = _sized_clusters(sizes, D, seed=len(fill))
    assert len(X) >= 4096
    nb, served, _ = _knn(km, k, X, C, A, monkeypatch, capfd)
    assert served > 0.5 * len(X), served
    ex, _, _ = _knn(km, k, X, C, A, monkeypatch, capfd, force_exact=True)
    _check_knn(X, nb, np.arange(len(X)), k, ref=ex)


def test_wide_knn_angular_unit_length(km, monkeypatch, capfd):
    """angular metric on unit-length samples: served through the L2 pass, the same neighbours as the exact search"""
    D, k, N = 768, 10, 8000
    X = T.unit(T.clustered(N, D, seed=7, n_centers=40, sigma=0.3))
    C = T.unit(T.perturbed_centroids(X, 40, seed=7))
    A = T.nearest(X, C)
    out = {}
    for fe in ("0", "1"):
        monkeypatch.setenv("KMCUDA_B200_FORCE_EXACT", fe)
        monkeypatch.setenv("KMCUDA_B200_TIMING", "1")
        capfd.readouterr()
        out[fe] = km.knn_cuda(k, X, C, A, metric="cos", device=1), _served(capfd.readouterr().err)
    monkeypatch.delenv("KMCUDA_B200_TIMING")
    assert out["0"][1] > 0.5 * N, out["0"][1]
    assert out["1"][1] == 0
    # unit vectors: the L2 order is the angular order, so fp64 L2 truth checks both answers
    _check_knn(X, out["0"][0], np.arange(N), k, ref=out["1"][0])


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
def test_wide_knn_device_and_fp16_inputs_equal_host_fp32(km, fp16, monkeypatch, capfd):
    import torch
    D, k, N = 768, 8, 6000
    X = T.clustered(N, D, seed=11, n_centers=30, sigma=0.3)
    C = T.perturbed_centroids(X, 30, seed=11)
    A = T.nearest(X, C)
    src, Cin = (X.astype(np.float16), C.astype(np.float16)) if fp16 else (X, C)
    host, served, _ = _knn(km, k, src.astype(np.float32), Cin.astype(np.float32), A, monkeypatch, capfd)
    assert served > 0.5 * N, served
    Xt = torch.from_numpy(np.ascontiguousarray(src.view(np.float32) if fp16 else src)).cuda(0)
    Ct = torch.from_numpy(np.ascontiguousarray(Cin.view(np.float32) if fp16 else Cin)).cuda(0)
    At = torch.from_numpy(A.view(np.int32)).cuda(0)
    shape = (N, D // 2, 1) if fp16 else (N, D)
    ptr = km.knn_cuda(k, (Xt.data_ptr(), 0, shape), (Ct.data_ptr(), len(C)), At.data_ptr(), device=1)
    got = np.empty((N, k), np.uint32)
    km._cuda_memcpy_d2h(0, got.ctypes.data, ptr, got.nbytes)
    km._cuda_free(0, ptr)
    assert np.array_equal(got, host), int((got != host).sum())


def test_wide_knn_kernel_ran(km):
    """a silent exact fallback cannot pass: the MODE 2 kernel of the 64-row layout shows up in the trace"""
    from torch.profiler import ProfilerActivity, profile
    X = T.clustered(8000, 768, seed=3, n_centers=30, sigma=0.3)
    C = T.perturbed_centroids(X, 30, seed=3)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        km.knn_cuda(10, X, C, T.nearest(X, C), device=1)
    names = {e.name for e in prof.events() if "tc_assign" in e.name}
    assert any("tc_assign_kernel<12, 2>" in nm for nm in names), names


def test_wide_knn_matches_reference(km):
    if not O.reference_available():
        pytest.skip("oracle/_ref/libKMCUDA.so not built")
    lib = O.load_c_api(km.LIB_PATH)
    ref = O.reference_lib()
    D, k, N = 768, 10, 20000
    X = T.clustered(N, D, seed=5, n_centers=100, sigma=0.3)
    C = T.perturbed_centroids(X, 100, seed=5)
    A = T.nearest(X, C)
    outs = []
    for L in (lib, ref):
        out = np.zeros((N, k), np.uint32)
        rc = L.knn_cuda(k, 0, N, D, len(C), 1, -1, 0, 0, X.ctypes.data, C.ctypes.data, A.ctypes.data, out.ctypes.data)
        assert rc == 0, rc
        outs.append(out)
    assert (outs[0] != outs[1]).mean() < 1e-4, (outs[0] != outs[1]).mean()
    _check_knn(X, outs[0], np.arange(0, N, 40), k, ref=outs[1])


def test_wide_knn_two_gpu_shards_equal_one_gpu(km, monkeypatch, capfd):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    D, k, N = 768, 10, 30000
    X = T.clustered(N, D, seed=9, n_centers=60, sigma=0.3)
    C = T.perturbed_centroids(X, 60, seed=9)
    A = T.nearest(X, C)
    one, served, _ = _knn(km, k, X, C, A, monkeypatch, capfd)
    assert served > 0.5 * N
    two = km.knn_cuda(k, X, C, A, device=3)
    assert np.array_equal(one, two), int((one != two).sum())
