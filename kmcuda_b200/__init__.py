"""kmcuda_b200 -- H100-native (sm_90a) implementation of kmcuda's batched-distance hot path.

Python surface = the reference's `libKMCUDA` module (reference src/python.cc:33-54):

    kmeans_cuda(samples, clusters, tolerance=.01, init="k-means++", yinyang_t=.1, metric="L2",
                average_distance=False, seed=time(), device=0, verbosity=0,   # python.cc:159-410
                sample_weight=None,                                           # extension: per-sample weights
                batch_size=None, max_steps=0,                                 # extension: mini-batch k-means
                relocate_empty_clusters=False,                                # extension: scikit-learn's relocation
                n_init=1, inertia=False,                                      # extension: restarts, inertia
                bisecting=None, max_iter=0,                                   # extension: bisecting k-means
                tol=None, n_iter=False,                                       # extension: scikit-learn's stop rule
                init_size=None)                                               # extension: mini-batch init stage
                init="k-means||" / ("k-means||", rounds)                      # extension: k-means|| seeding
    knn_cuda(k, samples, centroids, assignments, metric="L2", device=0, verbosity=0)  # python.cc:412-632
    supports_fp16                                                             # python.cc:52

Same argument meaning, same return types, same exceptions.  `libKMCUDA.so` exports the C ABI (include/kmcuda.h,
include/kmcuda_b200.h) and `PyInit_libKMCUDA` (csrc/py_module.cc), so `import libKMCUDA` works when its directory is
on sys.path.  This package loads that extension from the same file and calls it; the extension checks every argument.
In front of it the package converts a few inputs the reference module rejects, and nothing else:
- ndarray-like samples other than float16, and ndarray-like `init` centroids, become C-contiguous float32;
- knn_cuda's host centroids take the samples' dtype, and its host assignments become uint32;
- seed=None becomes the current time; clusters, k, seed, device and verbosity go through int().
A conversion that fails leaves the argument as it was, for the extension to reject.  `_lib` binds the same library
with ctypes for the C-ABI callers (shard.py, bench.py, tests).

kmeans_cuda returns (centroids, assignments[, avg_distance][, inertia][, n_iter]).  The extension keywords:

sample_weight: one non-negative weight per sample (include/kmcuda_b200.h, kmcuda_b200_kmeans_weighted), a 1-D
array-like of length N, or an int device pointer when `samples` is the device-pointer tuple; None = unweighted.

batch_size: an int >= 1 runs mini-batch k-means (kmcuda_b200_kmeans_minibatch, scikit-learn's MiniBatchKMeans)
with batches of min(batch_size, N) rows for at most max_steps steps (0 = 100 * N // batch size) on one GPU, L2
only; yinyang_t is ignored.  None = the Lloyd / Yinyang run.

init_size: with batch_size, the number of rows the seeding reads (kmcuda_b200_kmeans_minibatch_init, scikit-learn's
MiniBatchKMeans init_size): an int >= clusters, or "auto" for scikit-learn's default 3 * batch size (3 * clusters
when that is smaller than clusters), at most N.  Init r seeds with (seed + r * 0x9E3779B9) mod 2^32 on that many rows
drawn uniformly with replacement, with their weights, exactly as a call on those rows would seed; n_init such inits
are ranked by their inertia on as many validation rows and the lowest is kept, then the mini-batch steps run as
without init_size.  Not with an ndarray init or bisecting.  None = seed on all rows, and then n_init must be 1.

relocate_empty_clusters: True moves every cluster that ends an update without members to one of the samples
farthest from their centroids (kmcuda_b200_kmeans_relocate, scikit-learn's KMeans rule) instead of leaving a NaN
centroid; not with batch_size (mini-batch has its own reassignment).

n_init: an int >= 1, the number of restarts (kmcuda_b200_kmeans_restarts, scikit-learn's KMeans n_init): restart r
seeds with (seed + r * 0x9E3779B9) mod 2^32 and runs Lloyd / Yinyang as a fresh call would, on one ingest of the
samples; the run of lowest inertia is returned (ties keep the earlier restart).  Not with an ndarray init (every
restart would be the same run).  With batch_size it needs init_size and counts the inits of the mini-batch run.

inertia: True appends the returned run's inertia, sum w * ||x - c||^2 (angular: w * angle^2) as a float, to the
result; not with batch_size.

bisecting: "biggest_inertia" or "largest_cluster" runs bisecting k-means (kmcuda_b200_kmeans_bisecting,
scikit-learn's BisectingKMeans with that bisecting_strategy) on one GPU, L2 only, with init "random",
"greedy-k-means++" or ("greedy-k-means++", L) (L = 0: 2 trials, scikit-learn's 2 + floor(ln 2)); n_init is then
the number of inits per bisection and max_iter (0 = 300) the Lloyd iterations per 2-means run; yinyang_t is
ignored.  Not with batch_size, max_steps or relocate_empty_clusters.  None = the other routes.

tol: a real number >= 0 stops Lloyd / Yinyang runs by scikit-learn's KMeans rule (kmcuda_b200_kmeans_center_shift):
when the centroids of an update move by at most tol * (the mean per-feature variance of the samples) in total
squared distance, when an update is the max_iter-th (max_iter 0 = 300; one final assignment pass follows either),
or when a pass reassigns no sample.  `tolerance` is then ignored.  Works with sample_weight,
relocate_empty_clusters, n_init and inertia; not with batch_size or bisecting.  None = the reference's rule, a run
ends when at most tolerance * N samples were reassigned.

n_iter: True appends the number of iterations of the returned run (scikit-learn's n_iter_) as an int, last; needs
tol.

There is no CPU fallback: if the CUDA library cannot be loaded the import fails loudly.
"""
import ctypes
import importlib.machinery
import importlib.util
import os
import time

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KMCUDA_B200_LIB") or os.path.join(_HERE, "libKMCUDA.so")   # override: A/B timing of builds

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "kmcuda_b200: %s is missing -- build it with `python kmcuda_b200/build.py` "
        "(there is no CPU fallback)" % LIB_PATH)

_lib = ctypes.CDLL(LIB_PATH, mode=os.RTLD_LOCAL | os.RTLD_NOW)

_lib.kmeans_cuda.restype = ctypes.c_int
_lib.kmeans_cuda.argtypes = [
    ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_uint32,
    ctypes.c_uint16, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int32, ctypes.c_int32,
    ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
_lib.kmcuda_b200_kmeans_weighted.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_weighted.argtypes = _lib.kmeans_cuda.argtypes[:14] + [ctypes.c_void_p] + \
    _lib.kmeans_cuda.argtypes[14:]
_lib.kmcuda_b200_kmeans_relocate.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_relocate.argtypes = _lib.kmcuda_b200_kmeans_weighted.argtypes
_lib.kmcuda_b200_kmeans_minibatch.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_minibatch.argtypes = _lib.kmeans_cuda.argtypes[:3] + _lib.kmeans_cuda.argtypes[4:14] + \
    [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32] + _lib.kmeans_cuda.argtypes[14:]
_lib.kmcuda_b200_kmeans_minibatch_init.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_minibatch_init.argtypes = _lib.kmcuda_b200_kmeans_minibatch.argtypes[:16] + \
    [ctypes.c_uint32, ctypes.c_uint32] + _lib.kmeans_cuda.argtypes[14:]
_lib.kmcuda_b200_kmeans_restarts.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_restarts.argtypes = _lib.kmeans_cuda.argtypes[:14] + \
    [ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint32] + _lib.kmeans_cuda.argtypes[14:] + [ctypes.c_void_p]
_lib.kmcuda_b200_kmeans_bisecting.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_bisecting.argtypes = _lib.kmcuda_b200_kmeans_minibatch.argtypes[:13] + \
    [ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint32] + _lib.kmeans_cuda.argtypes[14:] + \
    [ctypes.c_void_p]
_lib.kmcuda_b200_kmeans_center_shift.restype = ctypes.c_int
_lib.kmcuda_b200_kmeans_center_shift.argtypes = _lib.kmcuda_b200_kmeans_restarts.argtypes[:-4] + [ctypes.c_uint32] + \
    _lib.kmcuda_b200_kmeans_restarts.argtypes[-4:] + [ctypes.c_void_p]
_lib.knn_cuda.restype = ctypes.c_int
_lib.knn_cuda.argtypes = [
    ctypes.c_uint16, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint16, ctypes.c_uint32, ctypes.c_uint32,
    ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
    ctypes.c_void_p]

# enums of include/kmcuda.h and include/kmcuda_b200.h
SUCCESS, INVALID_ARGUMENTS, NO_SUCH_DEVICE, MEMORY_ALLOCATION_FAILURE, RUNTIME_ERROR, MEMORY_COPY_ERROR = range(6)
INIT_RANDOM, INIT_PLUSPLUS, INIT_AFKMC2, INIT_IMPORT = range(4)
INIT_KMEANS_PARALLEL = 4   # kmcudaInitMethodKMeansParallel
INIT_GREEDY_PLUSPLUS = 5   # kmcudaInitMethodGreedyPlusPlus
METRIC_L2, METRIC_COSINE = range(2)
INIT_SIZE_AUTO = 0xFFFFFFFF   # KMCUDA_B200_INIT_SIZE_AUTO

# `import libKMCUDA` from the same file: one dlopen, so _lib and the extension share the library's state
_loader = importlib.machinery.ExtensionFileLoader("libKMCUDA", LIB_PATH)
_ext = importlib.util.module_from_spec(importlib.util.spec_from_loader("libKMCUDA", _loader))
_loader.exec_module(_ext)
supports_fp16 = _ext.supports_fp16


def _raise_for(result, fn):
    if result == SUCCESS:
        return
    if result == INVALID_ARGUMENTS:
        raise ValueError("Invalid arguments were passed to %s" % fn)
    if result == NO_SUCH_DEVICE:
        raise ValueError("No such CUDA device exists")
    if result == MEMORY_ALLOCATION_FAILURE:
        raise MemoryError("Failed to allocate memory on GPU")
    if result == MEMORY_COPY_ERROR:
        raise RuntimeError("cudaMemcpy failed")
    if result == RUNTIME_ERROR:
        raise AssertionError("%s failure (bug?)" % fn)
    raise AssertionError("Unknown error code returned from %s" % fn)


def _converted(convert, value):
    """convert(value), or value unchanged when the conversion fails: the extension then raises its own error"""
    try:
        return convert(value)
    except Exception:
        return value


def _float32_unless_half(samples):
    arr = np.asarray(samples)
    return arr if arr.dtype == np.float16 else np.ascontiguousarray(arr, np.float32)


def kmeans_cuda(samples, clusters, tolerance=.01, init="k-means++", yinyang_t=.1, metric="L2",
                average_distance=False, seed=None, device=0, verbosity=0, *args, **kwargs):
    """K-means on the GPU(s): libKMCUDA's kmeans_cuda after the conversions of the module docstring, which also
    describes the keywords after verbosity."""
    if not isinstance(samples, tuple):
        samples = _converted(_float32_unless_half, samples)
    if init is not None and not isinstance(init, (str, tuple)):
        init = _converted(lambda c: np.ascontiguousarray(c, np.float32), init)
    if seed is None:
        seed = int(time.time()) & 0xFFFFFFFF
    clusters, seed, device, verbosity = (_converted(int, v) for v in (clusters, seed, device, verbosity))
    return _ext.kmeans_cuda(samples, clusters, tolerance, init, yinyang_t, metric, average_distance, seed, device,
                            verbosity, *args, **kwargs)


def knn_cuda(k, samples, centroids, assignments, metric="L2", device=0, verbosity=0):
    """Exact k nearest neighbours accelerated by a clustering; returns uint32 [N][k] (python.cc:412-632).
    libKMCUDA's knn_cuda after the conversions of the module docstring."""
    if not isinstance(samples, tuple):
        samples = _converted(_float32_unless_half, samples)
        if isinstance(samples, np.ndarray):
            centroids = _converted(lambda c: np.ascontiguousarray(c, samples.dtype), centroids)
        assignments = _converted(lambda a: np.ascontiguousarray(a, np.uint32), assignments)
    k, device, verbosity = (_converted(int, v) for v in (k, device, verbosity))
    return _ext.knn_cuda(k, samples, centroids, assignments, metric, device, verbosity)


# ---- device-memory helpers for the raw-pointer forms (include/kmcuda_b200.h) ----
_lib.kmcuda_b200_device_malloc.restype = ctypes.c_int
_lib.kmcuda_b200_device_malloc.argtypes = [ctypes.c_int32, ctypes.c_uint64, ctypes.POINTER(ctypes.c_void_p)]
_lib.kmcuda_b200_device_free.restype = ctypes.c_int
_lib.kmcuda_b200_device_free.argtypes = [ctypes.c_int32, ctypes.c_void_p]
_lib.kmcuda_b200_device_memcpy.restype = ctypes.c_int
_lib.kmcuda_b200_device_memcpy.argtypes = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64,
                                           ctypes.c_int32]
_lib.kmcuda_b200_device_synchronize.restype = ctypes.c_int
_lib.kmcuda_b200_device_synchronize.argtypes = [ctypes.c_int32]
_lib.kmcuda_b200_device_count.restype = ctypes.c_int32
_lib.kmcuda_b200_device_count.argtypes = []


def _cuda_free(device, ptr):
    _raise_for(_lib.kmcuda_b200_device_free(int(device), ctypes.c_void_p(ptr)), "cudaFree")


def _cuda_memcpy_d2h(device, dst, src, nbytes):
    _raise_for(_lib.kmcuda_b200_device_memcpy(int(device), ctypes.c_void_p(dst), ctypes.c_void_p(src),
                                              int(nbytes), 2), "cudaMemcpy")


def device_count():
    return int(_lib.kmcuda_b200_device_count())


__all__ = ["kmeans_cuda", "knn_cuda", "supports_fp16", "LIB_PATH"]
