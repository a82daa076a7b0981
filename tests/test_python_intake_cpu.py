"""CPU tests of the Python intake: the kmcuda_b200 package converts a few inputs that `import libKMCUDA` rejects as the
reference does, and both surfaces reject a malformed device-pointer tuple or AFK-MC² chain length before any device
call."""
import importlib.util

import numpy as np
import pytest


def _surfaces():
    import kmcuda_b200 as km
    spec = importlib.util.spec_from_file_location("libKMCUDA", km.LIB_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return km, mod


def _permissive_calls():
    X = np.random.default_rng(0).random((100, 4))   # float64
    X32 = X.astype(np.float32)
    C = X32[:5].copy()
    A = (np.arange(100) % 5).astype(np.uint32)
    return {
        "float64 samples": lambda f: f.kmeans_cuda(X, 5, seed=3),
        "float64 init": lambda f: f.kmeans_cuda(X32, 5, init=C.astype(np.float64), seed=3),
        "seed None": lambda f: f.kmeans_cuda(X32, 5, seed=None),
        "float clusters": lambda f: f.kmeans_cuda(X32, 5.0, seed=3),
        "float verbosity": lambda f: f.kmeans_cuda(X32, 5, seed=3, verbosity=1.5),
        "float k": lambda f: f.knn_cuda(3.0, X32, C, A),
        "int64 k-NN assignments": lambda f: f.knn_cuda(3, X32, C, A.astype(np.int64)),
        "float64 k-NN centroids": lambda f: f.knn_cuda(3, X32, C.astype(np.float64), A),
    }


@pytest.mark.parametrize("case", sorted(_permissive_calls()))
def test_package_converts_what_the_extension_rejects(case):
    """without a GPU a call that got past the intake ends at the device lookup"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    km, ext = _surfaces()
    call = _permissive_calls()[case]
    with pytest.raises(ValueError, match="No such CUDA device"):
        call(km)
    with pytest.raises(TypeError):
        call(ext)


T = (0x1000, 0, (100, 4))
BAD_TUPLES = {
    "kmeans device": lambda f: f.kmeans_cuda((0x1000, 0.0, (100, 4)), 5),
    "kmeans device str": lambda f: f.kmeans_cuda((0x1000, "0", (100, 4)), 5),
    "kmeans n": lambda f: f.kmeans_cuda((0x1000, 0, (100.0, 4)), 5),
    "kmeans d": lambda f: f.kmeans_cuda((0x1000, 0, (100, "4")), 5),
    "kmeans centroids": lambda f: f.kmeans_cuda((0x1000, 0, (100, 4), 1.5, 0x3000), 5),
    "kmeans assignments": lambda f: f.kmeans_cuda((0x1000, 0, (100, 4), 0x2000, "x"), 5),
    "kmeans afkmc2 m": lambda f: f.kmeans_cuda(np.zeros((100, 4), np.float32), 5, init=("afkmc2", 2.5)),
    "kmeans afkmc2 m str": lambda f: f.kmeans_cuda(np.zeros((100, 4), np.float32), 5, init=("afkmc2", "x")),
    "knn samples": lambda f: f.knn_cuda(3, (1.5, 0, (100, 4)), (0x2000, 5), 0x3000),
    "knn device": lambda f: f.knn_cuda(3, (0x1000, 0.5, (100, 4)), (0x2000, 5), 0x3000),
    "knn n": lambda f: f.knn_cuda(3, (0x1000, 0, (100.0, 4)), (0x2000, 5), 0x3000),
    "knn centroids": lambda f: f.knn_cuda(3, T, (1.5, 5), 0x3000),
    "knn clusters": lambda f: f.knn_cuda(3, T, (0x2000, 5.0), 0x3000),
    "knn assignments": lambda f: f.knn_cuda(3, T, (0x2000, 5), 1.5),
    "knn neighbors": lambda f: f.knn_cuda(3, T, (0x2000, 5), (0x3000, 1.5)),
    "knn assignments 3-tuple": lambda f: f.knn_cuda(3, T, (0x2000, 5), (0x3000, 0x4000, 5)),
}


@pytest.mark.parametrize("which", [0, 1], ids=["package", "libKMCUDA"])
@pytest.mark.parametrize("case", sorted(BAD_TUPLES))
def test_malformed_tuples_are_rejected_before_the_device(which, case):
    """these members used to reach the library as garbage with a Python error pending; the fake pointers are never
    dereferenced because the call stops in the intake"""
    f = _surfaces()[which]
    with pytest.raises((TypeError, ValueError)) as e:
        BAD_TUPLES[case](f)
    assert "CUDA device" not in str(e.value)


@pytest.mark.parametrize("which", [0, 1], ids=["package", "libKMCUDA"])
def test_out_of_range_counts_are_not_wrapped(which):
    f = _surfaces()[which]
    X = np.zeros((100, 4), np.float32)
    for clusters in (2 ** 32 + 5, -3):
        with pytest.raises(ValueError, match="clusters"):
            f.kmeans_cuda(X, clusters)
    for k in (2 ** 32 + 3, -1):
        with pytest.raises(ValueError, match="k"):
            f.knn_cuda(k, X, X[:5], np.zeros(100, np.uint32))


def test_bisecting_says_yinyang_t_is_ignored(capfd):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU tests run these calls")
    _, ext = _surfaces()
    X = np.random.default_rng(0).random((100, 4), dtype=np.float32)
    with pytest.raises(ValueError, match="No such CUDA device"):
        ext.kmeans_cuda(X, 2, init="random", bisecting="biggest_inertia", verbosity=1)
    assert "bisecting k-means: yinyang_t is ignored" in capfd.readouterr().out
