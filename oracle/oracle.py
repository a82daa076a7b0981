"""ctypes front-end of the CPU oracle (oracle/kmcuda_oracle.c) and of the rebuilt reference library
(oracle/_ref/libKMCUDA.so).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (kmcuda_b200) never imports this module.
"""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libkmoracle.so")
REF_PATH = os.path.join(HERE, "_ref", "libKMCUDA.so")

_u32p = ctypes.POINTER(ctypes.c_uint32)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)


def build(force=False):
    """Compile the C restatement with gcc (no fast-math, no FP contraction)."""
    src = os.path.join(HERE, "kmcuda_oracle.c")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(
            ["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-ffp-contract=off", "-o", LIB_PATH, src, "-lm"])
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(LIB_PATH)
        L.ko_set_threads.restype = ctypes.c_int
        L.ko_set_threads.argtypes = [ctypes.c_int]
        L.ko_fma_rd.restype = ctypes.c_float
        L.ko_fma_rd.argtypes = [ctypes.c_float] * 3
        L.ko_fma_rd_fenv.restype = ctypes.c_float
        L.ko_fma_rd_fenv.argtypes = [ctypes.c_float] * 3
        L.ko_kahan_dot.restype = ctypes.c_float
        L.ko_kahan_dot.argtypes = [_f32p, _f32p, ctypes.c_int]
        L.ko_distance.restype = ctypes.c_float
        L.ko_distance.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_int]
        L.ko_assign_lloyd.restype = ctypes.c_uint32
        L.ko_assign_lloyd.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int,
                                      ctypes.c_uint32, _u32p, _u32p, _f32p, _f32p]
        L.ko_assign_truth.restype = None
        L.ko_assign_truth.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int,
                                      ctypes.c_uint32, _u32p, _f64p, _f64p]
        L.ko_adjust.restype = None
        L.ko_adjust.argtypes = [ctypes.c_int, _f32p, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint32,
                                _u32p, _u32p, _f32p, _u32p]
        L.ko_average_distance.restype = ctypes.c_float
        L.ko_average_distance.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int, _u32p]
        L.ko_kmeans.restype = ctypes.c_int
        L.ko_kmeans.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_uint32, _f32p, ctypes.c_uint32,
                                ctypes.c_int, ctypes.c_uint32, _f32p, _u32p, ctypes.c_int, ctypes.c_int]
        L.ko_yy_init.restype = None
        L.ko_yy_init.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint32,
                                 ctypes.c_uint32, _u32p, _u32p, _f32p]
        L.ko_yy_drifts.restype = None
        L.ko_yy_drifts.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint32,
                                   _u32p, _f32p, _f32p]
        L.ko_yy_step.restype = ctypes.c_uint32
        L.ko_yy_step.argtypes = [ctypes.c_int, _f32p, _f32p, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint32,
                                 ctypes.c_uint32, _u32p, _f32p, _f32p, _u32p, _u32p, _f32p, _u32p, _u32p]
        L.ko_knn.restype = None
        L.ko_knn.argtypes = [ctypes.c_int, ctypes.c_int, _f32p, ctypes.c_uint32, ctypes.c_int, _f32p,
                             ctypes.c_uint32, _u32p, _u32p, ctypes.c_uint32, _u32p, _f64p]
        _lib = L
    return _lib


def set_threads(n):
    """OpenMP threads used by the oracle (returns the effective count)"""
    return int(lib().ko_set_threads(int(n)))


def _f(a):
    return a.ctypes.data_as(_f32p)


def _u(a):
    return a.ctypes.data_as(_u32p)


def _d(a):
    return a.ctypes.data_as(_f64p)


def _c32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def assign_lloyd(X, C, metric=0, assign=None, with_scores=False):
    """One Lloyd assignment pass (kmeans.cu:293-364). Returns (assign, prev, changed[, best, second])."""
    X, C = _c32(X), _c32(C)
    N, D = X.shape
    K = C.shape[0]
    a = np.full(N, 0xFFFFFFFF, dtype=np.uint32) if assign is None else np.array(assign, dtype=np.uint32)
    prev = np.full(N, 0xFFFFFFFF, dtype=np.uint32)
    best = np.empty(N, np.float32)
    second = np.empty(N, np.float32)
    changed = lib().ko_assign_lloyd(metric, _f(X), _f(C), N, D, K, _u(a), _u(prev), _f(best), _f(second))
    if with_scores:
        return a, prev, changed, best, second
    return a, prev, changed


def assign_truth(X, C, metric=0):
    """float64 argmin with best / second-best values (tie detector)."""
    X, C = _c32(X), _c32(C)
    N, D = X.shape
    K = C.shape[0]
    arg = np.empty(N, np.uint32)
    best = np.empty(N, np.float64)
    second = np.empty(N, np.float64)
    lib().ko_assign_truth(metric, _f(X), _f(C), N, D, K, _u(arg), _d(best), _d(second))
    return arg, best, second


def tie_exempt(best, second, rel=1e-6):
    """SURVEY.md 8c: a sample is tie-exempt iff fp64 best/second-best differ by < rel (relative)."""
    scale = np.maximum(np.abs(best), np.abs(second))
    scale = np.where(scale > 0, scale, 1.0)
    return (second - best) <= rel * scale


def adjust(X, C, prev, cur, ccounts, metric=0):
    """Centroid update (kmeans.cu:366-429). Returns (C_new, ccounts_new)."""
    X = _c32(X)
    C = np.array(C, dtype=np.float32, order="C")
    cc = np.array(ccounts, dtype=np.uint32)
    prev = np.ascontiguousarray(prev, dtype=np.uint32)
    cur = np.ascontiguousarray(cur, dtype=np.uint32)
    lib().ko_adjust(metric, _f(X), X.shape[0], X.shape[1], C.shape[0], _u(prev), _u(cur), _f(C), _u(cc))
    return C, cc


def average_distance(X, C, assign, metric=0):
    X, C = _c32(X), _c32(C)
    a = np.ascontiguousarray(assign, dtype=np.uint32)
    return float(lib().ko_average_distance(metric, _f(X), _f(C), X.shape[0], X.shape[1], _u(a)))


def kmeans(X, C0, tolerance=0.01, yinyang_t=0.1, metric=0, log=False, max_iter=0):
    """Whole run from imported centroids (kmeans.cu:1028-1263). Returns (C, assign, iteration_lines)."""
    X = _c32(X)
    C = np.array(C0, dtype=np.float32, order="C")
    N, D = X.shape
    K = C.shape[0]
    a = np.empty(N, np.uint32)
    G = int(np.float32(yinyang_t) * np.float32(K))
    lines = lib().ko_kmeans(metric, tolerance, G, _f(X), N, D, K, _f(C), _u(a), int(log), int(max_iter))
    return C, a, lines


# Yinyang pieces (kmeans.cu:431-672).  Bounds are row-major [N][G + 1] here, the library's layout (column 0 the upper
# bound, column 1 + g the lower bound of group g); the C side keeps the reference's [(G + 1)][N] planes.
def yy_init(X, C, assign, groups, G, metric=0):
    """bounds refresh (kmeans_yy_init): [N][G + 1] float32"""
    X, C = _c32(X), _c32(C)
    N, D = X.shape
    a = np.ascontiguousarray(assign, dtype=np.uint32)
    g = np.ascontiguousarray(groups, dtype=np.uint32)
    planes = np.empty((G + 1, N), np.float32)
    lib().ko_yy_init(metric, _f(X), _f(C), N, D, C.shape[0], G, _u(g), _u(a), _f(planes))
    return np.ascontiguousarray(planes.T)


def yy_drifts(C_new, C_old, groups, G, metric=0):
    """(drift [K], maxdrift [G]): distance of each centroid from its old position, largest per group (-FLT_MAX if
    the group has no member)"""
    Cn, Co = _c32(C_new), _c32(C_old)
    K, D = Cn.shape
    g = np.ascontiguousarray(groups, dtype=np.uint32)
    drift = np.empty(K, np.float32)
    maxdrift = np.empty(max(G, 1), np.float32)
    lib().ko_yy_drifts(metric, _f(Cn), _f(Co), K, D, G, _u(g), _f(drift), _f(maxdrift))
    return drift, maxdrift[:G]


def yy_step(X, C, groups, G, drift, maxdrift, assign, bounds, metric=0):
    """global + local filter after a centroid update.  Returns (assign, prev, bounds, changed, tight, passed); the
    inputs are not modified"""
    X, C = _c32(X), _c32(C)
    N, D = X.shape
    g = np.ascontiguousarray(groups, dtype=np.uint32)
    a = np.array(assign, dtype=np.uint32)
    prev = np.empty(N, np.uint32)
    planes = np.ascontiguousarray(np.asarray(bounds, np.float32).reshape(N, G + 1).T)
    dr, md = _c32(drift), _c32(maxdrift)
    tight, passed = ctypes.c_uint32(0), ctypes.c_uint32(0)
    changed = lib().ko_yy_step(metric, _f(X), _f(C), N, D, C.shape[0], G, _u(g), _f(dr), _f(md), _u(a), _u(prev),
                               _f(planes), ctypes.byref(tight), ctypes.byref(passed))
    return a, prev, np.ascontiguousarray(planes.T), int(changed), tight.value, passed.value


def knn(k, X, C, assign, metric=0, queries=None):
    """Cluster-pruned exact k-NN (knn.cu). Returns ([nq][k] uint32, evaluated_pairs)."""
    X, C = _c32(X), _c32(C)
    a = np.ascontiguousarray(assign, dtype=np.uint32)
    N, D = X.shape
    if queries is None:
        q, nq, qp = None, N, None
    else:
        q = np.ascontiguousarray(queries, dtype=np.uint32)
        nq, qp = len(q), _u(q)
    out = np.empty((nq, k), np.uint32)
    pairs = ctypes.c_double(0)
    lib().ko_knn(metric, k, _f(X), N, D, _f(C), C.shape[0], _u(a), qp, nq, _u(out), ctypes.byref(pairs))
    return out, pairs.value


# ---------------------------------------------------------------------------------------------
# The rebuilt, unmodified reference library (CUDA; needs a GPU to do anything but load).
# ---------------------------------------------------------------------------------------------
def reference_available():
    return os.path.exists(REF_PATH)


_KM_ARGTYPES = [ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                ctypes.c_uint32, ctypes.c_uint16, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32,
                ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p,
                ctypes.c_void_p, ctypes.c_void_p]
_KNN_ARGTYPES = [ctypes.c_uint16, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint16, ctypes.c_uint32,
                 ctypes.c_uint32, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]


def load_c_api(path):
    """Bind kmeans_cuda / knn_cuda (kmcuda.h:118-123,150-155) of any libKMCUDA.so by file path."""
    L = ctypes.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.kmeans_cuda.restype = ctypes.c_int
    L.kmeans_cuda.argtypes = _KM_ARGTYPES
    L.knn_cuda.restype = ctypes.c_int
    L.knn_cuda.argtypes = _KNN_ARGTYPES
    return L


def reference_lib():
    return load_c_api(REF_PATH)
