"""GPU tests of the copy routes between the caller's memory and the devices (csrc/transfer.cu: copy_in / copy_out).

Every route must give the bits of the host fp32 route: device-pointer inputs (borrowed in place on their own device,
peer-copied to another), fp16 inputs widened on the device (compared with fp32 inputs widened from the same halves),
imported centroids from device memory, and device-pointer outputs.  `device` selects the GPU that runs the call: 1 is
the pointers' own GPU, 2 another one (peer copies; skipped with one GPU)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, DIM, K = 20000, 32, 40
RUN = dict(tolerance=0.01, seed=3, average_distance=True)


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    return kmcuda_b200


@pytest.fixture(params=[1, 2], ids=["same-gpu", "peer-gpu"])
def device(request):
    import torch
    if request.param == 2 and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    return request.param


def _data(seed=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((K, DIM)).astype(np.float32) * 3
    X16 = (centers[rng.integers(0, K, N)] + 0.6 * rng.standard_normal((N, DIM))).astype(np.float16)
    w = rng.lognormal(0.0, 1.0, N).astype(np.float32)
    C16 = X16[rng.choice(N, K, replace=False)].copy()
    return X16, w, C16


def _on_gpu(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).cuda(0)


def _fetch(km, ptr, shape, dtype):
    out = np.empty(shape, dtype)
    km._cuda_memcpy_d2h(0, out.ctypes.data, ptr, out.nbytes)
    km._cuda_free(0, ptr)
    return out


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _kmeans_dev(km, X, k, device, fp16, weights=None, **kw):
    """kmeans_cuda on samples (and weights) in device memory of GPU 0; the outputs come back from there"""
    Xt = _on_gpu(X.view(np.float32) if fp16 else X)
    shape = (X.shape[0], X.shape[1] // 2, 1) if fp16 else X.shape
    wt = _on_gpu(weights) if weights is not None else None
    cp, ap, avg = km.kmeans_cuda((Xt.data_ptr(), 0, shape), k, device=device,
                                 sample_weight=None if wt is None else wt.data_ptr(), **kw)
    c = _fetch(km, cp, (k, X.shape[1]), np.float16 if fp16 else np.float32)
    return c, _fetch(km, ap, X.shape[0], np.uint32), avg


def _same_run(dev, host, fp16):
    (cd, ad, avgd), (ch, ah, avgh) = dev, host
    if fp16:
        ch = ch.astype(np.float16)
    assert np.array_equal(_bits(cd), _bits(ch))
    assert np.array_equal(ad, ah)
    assert avgd == avgh


@pytest.mark.parametrize("entry", ["plain", "weighted", "minibatch"])
def test_fp16_device_samples_equal_host_fp32_of_the_widened_samples(km, device, entry):
    X16, w, _ = _data(1)
    kw = dict(RUN, init="k-means++")
    if entry == "weighted":
        kw["yinyang_t"] = 0.1
    if entry == "minibatch":
        kw.update(batch_size=2048, max_steps=30)
    weights = w if entry != "plain" else None
    host = km.kmeans_cuda(X16.astype(np.float32), K, device=device, sample_weight=weights, **kw)
    _same_run(_kmeans_dev(km, X16, K, device, True, weights, **kw), host, True)


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
def test_imported_device_centroids_equal_host_import(km, device, fp16):
    X16, _, C16 = _data(2)
    X = X16 if fp16 else X16.astype(np.float32)
    # the binding's import takes float32 rows of the pointer width: fp16 centroids travel as their raw bytes
    init = C16.view(np.float32) if fp16 else C16.astype(np.float32)
    host = km.kmeans_cuda(X16.astype(np.float32), K, init=C16.astype(np.float32), device=device, yinyang_t=0.1, **RUN)
    _same_run(_kmeans_dev(km, X, K, device, fp16, init=init, yinyang_t=0.1, **RUN), host, fp16)


@pytest.mark.parametrize("entry", ["weighted", "minibatch"])
def test_device_outputs_equal_host_outputs(km, device, entry):
    X16, w, C16 = _data(3)
    X = X16.astype(np.float32)
    kw = dict(RUN, init=C16.astype(np.float32))
    if entry == "minibatch":
        kw.update(batch_size=2048, max_steps=30)
    host = km.kmeans_cuda(X, K, device=device, sample_weight=w, **kw)
    _same_run(_kmeans_dev(km, X, K, device, False, w, **kw), host, False)


@pytest.mark.parametrize("metric", ["L2", "cos"])
@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
def test_knn_device_inputs_equal_host_fp32(km, device, fp16, metric):
    X16, _, _ = _data(4)
    X = X16.astype(np.float32)
    if metric == "cos":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    C, A = km.kmeans_cuda(X, K, init="k-means++", metric=metric, device=device, tolerance=0.01, seed=4)
    k = 8
    host = km.knn_cuda(k, X, C, A, metric=metric, device=device)
    src = X.astype(np.float16) if fp16 else X
    Cin = C.astype(np.float16) if fp16 else C
    if fp16:   # the fp32 reference on the same halves
        host = km.knn_cuda(k, src.astype(np.float32), Cin.astype(np.float32), A, metric=metric, device=device)
    Xt = _on_gpu(src.view(np.float32) if fp16 else src)
    Ct = _on_gpu(Cin.view(np.float32) if fp16 else Cin)
    At = _on_gpu(A.view(np.int32))
    shape = (N, DIM // 2, 1) if fp16 else (N, DIM)
    nptr = km.knn_cuda(k, (Xt.data_ptr(), 0, shape), (Ct.data_ptr(), K), At.data_ptr(), metric=metric, device=device)
    assert np.array_equal(_fetch(km, nptr, (N, k), np.uint32), host)
