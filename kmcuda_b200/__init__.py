"""kmcuda_b200 -- H100-native (sm_90a) implementation of kmcuda's batched-distance hot path.

Python surface = the reference's `libKMCUDA` module (reference src/python.cc:33-54):

    kmeans_cuda(samples, clusters, tolerance=.01, init="k-means++", yinyang_t=.1, metric="L2",
                average_distance=False, seed=time(), device=0, verbosity=0,   # python.cc:159-410
                sample_weight=None)                                           # extension: per-sample weights
                init="k-means||" / ("k-means||", rounds)                      # extension: k-means|| seeding
    knn_cuda(k, samples, centroids, assignments, metric="L2", device=0, verbosity=0)  # python.cc:412-632
    supports_fp16                                                             # python.cc:52

Same argument meaning, same return types, same exceptions.  This module binds the C ABI of
`libKMCUDA.so` (include/kmcuda.h) with ctypes; the same shared object also exports
`PyInit_libKMCUDA`, so `import libKMCUDA` works when its directory is on sys.path.

There is no CPU fallback: if the CUDA library cannot be loaded the import fails loudly.
"""
import ctypes
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
_lib.knn_cuda.restype = ctypes.c_int
_lib.knn_cuda.argtypes = [
    ctypes.c_uint16, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint16, ctypes.c_uint32, ctypes.c_uint32,
    ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
    ctypes.c_void_p]

supports_fp16 = True

# enums of include/kmcuda.h
SUCCESS, INVALID_ARGUMENTS, NO_SUCH_DEVICE, MEMORY_ALLOCATION_FAILURE, RUNTIME_ERROR, MEMORY_COPY_ERROR = range(6)
INIT_RANDOM, INIT_PLUSPLUS, INIT_AFKMC2, INIT_IMPORT = range(4)
INIT_KMEANS_PARALLEL = 4   # include/kmcuda_b200.h: kmcudaInitMethodKMeansParallel
KMEANS_PARALLEL_MAX_ROUNDS = 32
METRIC_L2, METRIC_COSINE = range(2)

_INIT_METHODS = {"kmeans++": INIT_PLUSPLUS, "k-means++": INIT_PLUSPLUS, "afkmc2": INIT_AFKMC2,
                 "afk-mc2": INIT_AFKMC2, "random": INIT_RANDOM, "k-means||": INIT_KMEANS_PARALLEL,
                 "kmeans||": INIT_KMEANS_PARALLEL}
_METRICS = {"euclidean": METRIC_L2, "L2": METRIC_L2, "l2": METRIC_L2, "cos": METRIC_COSINE,
            "cosine": METRIC_COSINE, "angular": METRIC_COSINE}


def _get_metric(metric):
    if metric is None:
        return METRIC_L2
    if not isinstance(metric, str):
        raise TypeError("\"metric\" must be either None or string.")
    if metric not in _METRICS:
        raise ValueError("Unknown metric. Supported values are \"L2\" and \"cos\".")
    return _METRICS[metric]


def _get_samples(samples):
    """ndarray intake of python.cc:120-157: float16 -> fp16x2, else float32; must be 2-D."""
    try:
        arr = np.asarray(samples)
    except Exception:
        raise TypeError("\"samples\" must be a 2D float32 or float16 numpy array")
    fp16x2 = arr.dtype == np.float16
    if not fp16x2:
        try:
            arr = np.ascontiguousarray(arr, dtype=np.float32)
        except Exception:
            raise TypeError("\"samples\" must be a 2D float32 or float16 numpy array")
    else:
        arr = np.ascontiguousarray(arr)
    if arr.ndim != 2:
        raise ValueError("\"samples\" must be a 2D numpy array")
    n, d = arr.shape
    if fp16x2:
        if d % 2 != 0:
            raise ValueError("the number of features must be even in fp16 mode")
        d //= 2
    return arr, fp16x2, int(n), int(d)


def _get_sample_weight(sample_weight, n, device_ptrs):
    """sample_weight intake: with ndarray samples a 1-D array-like of length n (kept alive by the caller as float32),
    with device-pointer samples an int device pointer on the samples' device.  Returns (keep, pointer)."""
    if device_ptrs >= 0:
        if isinstance(sample_weight, bool) or not isinstance(sample_weight, int):
            raise TypeError("\"sample_weight\" must be a device pointer (integer) when \"samples\" is a pointer tuple")
        if sample_weight == 0:
            raise ValueError("\"sample_weight\" is null")
        return None, sample_weight
    try:
        arr = np.asarray(sample_weight)
    except Exception:
        raise TypeError("\"sample_weight\" must be a 1D numeric array")
    if arr.dtype.kind not in "biuf":
        raise TypeError("\"sample_weight\" must be a 1D numeric array")
    if arr.ndim != 1:
        raise ValueError("\"sample_weight\" must be a 1D array")
    if arr.shape[0] != n:
        raise ValueError("\"sample_weight\" must be of the same length as \"samples\"")
    arr = np.ascontiguousarray(arr, dtype=np.float32)
    return arr, arr.ctypes.data


def _kmeans_parallel_rounds(rounds):
    """the rounds of init=("k-means||", rounds): an integer in [0, 32], 0 = the default (5)"""
    if isinstance(rounds, bool) or not isinstance(rounds, (int, np.integer)):
        raise ValueError("k-means|| rounds must be an integer, got %r" % (rounds,))
    if not 0 <= rounds <= KMEANS_PARALLEL_MAX_ROUNDS:
        raise ValueError("k-means|| rounds must be in [0, %d], got %d" % (KMEANS_PARALLEL_MAX_ROUNDS, rounds))
    return int(rounds)


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


def kmeans_cuda(samples, clusters, tolerance=.01, init="k-means++", yinyang_t=.1, metric="L2",
                average_distance=False, seed=None, device=0, verbosity=0, sample_weight=None):
    """K-means on the GPU(s); see the module docstring.  Returns (centroids, assignments[, avg_distance]).

    sample_weight: one non-negative weight per sample (include/kmcuda_b200.h, kmcuda_b200_kmeans_weighted), a 1-D
    array-like of length N, or an int device pointer when `samples` is the device-pointer tuple; None = unweighted."""
    clusters = int(clusters)
    if seed is None:
        seed = int(time.time()) & 0xFFFFFFFF
    afkmc2_m = ctypes.c_uint32(0)
    if init is None:
        init_method = INIT_PLUSPLUS
    elif isinstance(init, str):
        if init not in _INIT_METHODS:
            raise ValueError("Unknown centroids initialization method. Supported values are "
                             "\"kmeans++\", \"random\" and <numpy array>.")
        init_method = _INIT_METHODS[init]
    elif isinstance(init, tuple):
        if len(init) == 0 or init[0] is None:
            raise ValueError("centroid initialization method may not be null.")
        if init[0] not in _INIT_METHODS:
            raise ValueError("Unknown centroids initialization method. Supported values are "
                             "\"kmeans++\", \"random\" and <numpy array>.")
        init_method = _INIT_METHODS[init[0]]
        if len(init) > 1 and init_method == INIT_AFKMC2:
            afkmc2_m = ctypes.c_uint32(int(init[1]))
        if len(init) > 1 and init_method == INIT_KMEANS_PARALLEL:
            afkmc2_m = ctypes.c_uint32(_kmeans_parallel_rounds(init[1]))
    else:
        init_method = INIT_IMPORT
    metric_id = _get_metric(metric)
    if clusters < 2 or clusters >= 0xFFFFFFFF:
        raise ValueError("\"clusters\" must be greater than 1 and less than (1 << 32) - 1")
    device_ptrs = -1
    centroids_ptr = assignments_ptr = None
    if isinstance(samples, tuple):
        if len(samples) not in (3, 5):
            raise ValueError("len(\"samples\") must be either 3 or 5")
        ptr, device_ptrs, shape = samples[0], int(samples[1]), samples[2]
        if not isinstance(ptr, int):
            raise ValueError("\"samples\"[0] is not a pointer (integer)")
        if ptr == 0:
            raise ValueError("\"samples\"[0] is null")
        if not isinstance(shape, tuple) or len(shape) not in (2, 3):
            raise TypeError("\"samples\"[2] must be a shape tuple")
        n, d = int(shape[0]), int(shape[1])
        fp16x2 = bool(shape[2]) if len(shape) == 3 else False
        samples_ptr = ptr
        if len(samples) == 5:
            centroids_ptr, assignments_ptr = int(samples[3]), int(samples[4])
        keep = None
    else:
        keep, fp16x2, n, d = _get_samples(samples)
        samples_ptr = keep.ctypes.data
    if d > 0xFFFF:
        raise ValueError("\"samples\": more than %d features is not supported" % d)
    keep_w = weights_ptr = None
    if sample_weight is not None:
        keep_w, weights_ptr = _get_sample_weight(sample_weight, n, device_ptrs)
    owned = []
    if device_ptrs < 0:
        centroids = np.empty((clusters, d * 2 if fp16x2 else d), dtype=np.float16 if fp16x2 else np.float32)
        assignments = np.empty(n, dtype=np.uint32)
        centroids_ptr, assignments_ptr = centroids.ctypes.data, assignments.ctypes.data
    elif centroids_ptr is None:
        # the binding allocates the outputs on the caller's device; the caller owns them afterwards
        centroids_ptr = _cuda_malloc(device_ptrs, clusters * d * 4)
        assignments_ptr = _cuda_malloc(device_ptrs, n * 4)
    if init_method == INIT_IMPORT:
        try:
            imp = np.ascontiguousarray(init, dtype=np.float32)
        except Exception:
            raise TypeError("\"init\" centroids must be a 2D numpy array")
        if imp.ndim != 2:
            raise ValueError("\"init\" centroids must be a 2D numpy array")
        if imp.shape[0] != clusters:
            raise ValueError("\"init\" centroids shape[0] does not match the number of clusters")
        if imp.shape[1] != d:
            raise ValueError("\"init\" centroids shape[1] does not match the number of features")
        if device_ptrs < 0:
            ctypes.memmove(centroids_ptr, imp.ctypes.data, clusters * d * 4)
        else:
            _cuda_memcpy_h2d(device_ptrs, centroids_ptr, imp.ctypes.data, clusters * d * 4)
    avg = ctypes.c_float(0)
    common = (init_method, ctypes.byref(afkmc2_m), tolerance, yinyang_t, metric_id, n, d, clusters,
              int(seed) & 0xFFFFFFFF, int(device), device_ptrs, int(fp16x2), int(verbosity), samples_ptr)
    outputs = (centroids_ptr, assignments_ptr, ctypes.byref(avg) if average_distance else None)
    if weights_ptr is None:
        result = _lib.kmeans_cuda(*common, *outputs)
    else:
        result = _lib.kmcuda_b200_kmeans_weighted(*common, weights_ptr, *outputs)
    del owned, keep_w
    _raise_for(result, "kmeans_cuda")
    if device_ptrs < 0:
        return (centroids, assignments, avg.value) if average_distance else (centroids, assignments)
    return (centroids_ptr, assignments_ptr, avg.value) if average_distance else (centroids_ptr, assignments_ptr)


def knn_cuda(k, samples, centroids, assignments, metric="L2", device=0, verbosity=0):
    """Exact k nearest neighbours accelerated by a clustering; returns uint32 [N][k] (python.cc:412-632)."""
    k = int(k)
    metric_id = _get_metric(metric)
    if k <= 0 or k > 0xFFFF:
        raise ValueError("\"k\" must be greater than 0 and less than (1 << 16)")
    device_ptrs = -1
    neighbors_ptr = None
    if isinstance(samples, tuple):
        if len(samples) != 3:
            raise ValueError("len(\"samples\") must be 3")
        if not isinstance(centroids, tuple) or len(centroids) != 2:
            raise ValueError("\"centroids\" must be a tuple of length 2")
        if not isinstance(assignments, (tuple, int)):
            raise ValueError("\"assignments\" must be a pointer or a tuple of length 2")
        samples_ptr, device_ptrs, shape = int(samples[0]), int(samples[1]), samples[2]
        n, d = int(shape[0]), int(shape[1])
        fp16x2 = bool(shape[2]) if len(shape) == 3 else False
        centroids_ptr, clusters = int(centroids[0]), int(centroids[1])
        if isinstance(assignments, tuple):
            assignments_ptr, neighbors_ptr = int(assignments[0]), int(assignments[1])
        else:
            assignments_ptr = int(assignments)
        if samples_ptr == 0 or centroids_ptr == 0 or assignments_ptr == 0:
            raise ValueError("null pointer")
        keep = None
    else:
        keep_s, fp16x2, n, d = _get_samples(samples)
        samples_ptr = keep_s.ctypes.data
        cdtype = np.float16 if fp16x2 else np.float32
        try:
            keep_c = np.ascontiguousarray(centroids, dtype=cdtype)
        except Exception:
            raise TypeError("\"centroids\" must be a 2D float32 or float16 numpy array")
        if keep_c.ndim != 2:
            raise ValueError("\"centroids\" must be a 2D numpy array")
        clusters = keep_c.shape[0]
        if keep_c.shape[1] != (d * 2 if fp16x2 else d):
            raise ValueError("\"centroids\" must have same number of features as \"samples\"")
        try:
            keep_a = np.ascontiguousarray(assignments, dtype=np.uint32)
        except Exception:
            raise TypeError("\"assignments\" must be a 1D uint32 numpy array")
        if keep_a.ndim != 1:
            raise ValueError("\"assignments\" must be a 1D numpy array")
        if keep_a.shape[0] != n:
            raise ValueError("\"assignments\" must be of the same length as \"samples\"")
        centroids_ptr, assignments_ptr = keep_c.ctypes.data, keep_a.ctypes.data
    if d > 0xFFFF:
        raise ValueError("\"samples\": more than %d features is not supported" % d)
    if device_ptrs < 0:
        neighbors = np.empty((n, k), dtype=np.uint32)
        neighbors_ptr = neighbors.ctypes.data
    elif neighbors_ptr is None:
        neighbors_ptr = _cuda_malloc(device_ptrs, n * k * 4)
    result = _lib.knn_cuda(k, metric_id, n, d, clusters, int(device), device_ptrs, int(fp16x2), int(verbosity),
                           samples_ptr, centroids_ptr, assignments_ptr, neighbors_ptr)
    _raise_for(result, "knn_cuda")
    return neighbors if device_ptrs < 0 else neighbors_ptr


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


def _cuda_malloc(device, nbytes):
    p = ctypes.c_void_p()
    _raise_for(_lib.kmcuda_b200_device_malloc(int(device), int(nbytes), ctypes.byref(p)), "cudaMalloc")
    return p.value


def _cuda_free(device, ptr):
    _raise_for(_lib.kmcuda_b200_device_free(int(device), ctypes.c_void_p(ptr)), "cudaFree")


def _cuda_memcpy_h2d(device, dst, src, nbytes):
    _raise_for(_lib.kmcuda_b200_device_memcpy(int(device), ctypes.c_void_p(dst), ctypes.c_void_p(src),
                                              int(nbytes), 1), "cudaMemcpy")


def _cuda_memcpy_d2h(device, dst, src, nbytes):
    _raise_for(_lib.kmcuda_b200_device_memcpy(int(device), ctypes.c_void_p(dst), ctypes.c_void_p(src),
                                              int(nbytes), 2), "cudaMemcpy")


def device_count():
    return int(_lib.kmcuda_b200_device_count())


__all__ = ["kmeans_cuda", "knn_cuda", "supports_fp16", "LIB_PATH"]
