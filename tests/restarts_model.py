"""NumPy restatement of the restart rules of kmcuda_b200_kmeans_restarts (include/kmcuda_b200.h, DESIGN.md §4n):
the seed schedule, the inertia of a run and the pick among the restarts."""
import numpy as np

SEED_STEP = 0x9E3779B9


def seeds(seed, n_init):
    """seed_r = seed + r * 0x9E3779B9 (mod 2^32), r = 0 .. n_init - 1, in uint32 arithmetic"""
    r = np.arange(n_init, dtype=np.uint64)
    return ((np.uint64(seed) + r * np.uint64(SEED_STEP)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def select(inertias):
    """index of the kept restart: restart 0 is the first best, a later one wins only with a strictly lower inertia
    (ties keep the earlier restart, NaN never wins)"""
    best = 0
    for r in range(1, len(inertias)):
        if inertias[r] < inertias[best]:
            best = r
    return best


def inertia(X, C, a, w=None, metric=0):
    """sum w_i e_i in fp64: L2 e = ||x - c_a||^2, angular e = angle(x, c_a)^2; rows with a >= K or a non-finite e add 0"""
    X = np.asarray(X, np.float64)
    C = np.asarray(C, np.float64)
    a = np.asarray(a, np.int64)
    K = len(C)
    live = a < K
    e = np.zeros(len(X))
    c = C[np.where(live, a, 0)]
    with np.errstate(invalid="ignore", over="ignore"):
        if metric == 1:
            e = np.arccos(np.clip((X * c).sum(1), -1.0, 1.0)) ** 2
        else:
            e = ((X - c) ** 2).sum(1)
    ok = live & np.isfinite(e)
    wv = np.ones(len(X)) if w is None else np.asarray(w, np.float64)
    return float((wv[ok] * e[ok]).sum())
