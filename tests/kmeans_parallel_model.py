"""NumPy restatement of the k-means|| seeding (include/kmcuda_b200.h, DESIGN.md §4g), used by the CPU and GPU tests.

The draw of round r is u(seed, r, i) < l * w_i d_i^2 / phi with u a SplitMix64-style counter hash of the global row
index; the distances are the oracle's ko_distance (the reference's true distance, bit for bit with the device) and the
per-round argmin is the oracle's Lloyd assignment.  The host RNG steps (first centroid, the fill walk) are glibc's
rand() through ctypes, as the library calls it.
"""
import ctypes

import numpy as np

from oracle import oracle as O

_M64 = (1 << 64) - 1
_libc = ctypes.CDLL("libc.so.6")
_libc.rand.restype = ctypes.c_int
_libc.srand.argtypes = [ctypes.c_uint]
RAND_MAX = 2147483647


def mix(z):
    """the hash's finaliser on uint64 (scalars as Python ints, arrays as np.uint64)"""
    if isinstance(z, np.ndarray):
        with np.errstate(over="ignore"):
            z = z + np.uint64(0x9E3779B97F4A7C15)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            return z ^ (z >> np.uint64(31))
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def uniform(seed, r, rows):
    """u(seed, r, i) for the global row indices `rows`"""
    key = np.uint64(mix(((int(seed) & 0xFFFFFFFF) << 8) | int(r)))
    z = mix(key ^ np.asarray(rows, dtype=np.uint64))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def mass(d, w=None):
    """w_i d_i^2 in double; rows with a non-finite distance carry none"""
    d64 = np.asarray(d, np.float32).astype(np.float64)
    w64 = np.ones_like(d64) if w is None else np.asarray(w, np.float32).astype(np.float64)
    m = w64 * (d64 * d64)
    m[~np.isfinite(d64)] = 0.0
    return m


def draws(d, w, seed, r, ell, phi, offset=0):
    """the draw flags of rows offset .. offset + len(d) - 1"""
    return uniform(seed, r, np.arange(offset, offset + len(d))) < (ell * mass(d, w)) / phi


def row_distances(X, C, assign, metric=0):
    """ko_distance of every row to its assigned row of C (the library's true distance)"""
    X = np.ascontiguousarray(X, np.float32)
    C = np.ascontiguousarray(C, np.float32)
    N, D = X.shape
    L = O.lib()
    fp = ctypes.POINTER(ctypes.c_float)
    xb, cb, step = X.ctypes.data, C.ctypes.data, 4 * D
    out = np.empty(N, np.float32)
    for i, a in enumerate(np.asarray(assign)):
        out[i] = L.ko_distance(metric, ctypes.cast(xb + i * step, fp), ctypes.cast(cb + int(a) * step, fp), D)
    return out


def first_centroid(X, seed, w=None):
    """draw_first_centroid: srand(seed), rand() % N redrawn while the row is NaN or of weight 0"""
    _libc.srand(seed & 0xFFFFFFFF)
    N = len(X)
    while True:
        i = _libc.rand() % N
        if w is not None and not w[i] > 0:
            continue
        if X[i, 0] == X[i, 0]:
            return i


def random_order(N):
    """init_random's shuffle (the caller seeds rand())"""
    order = np.arange(N, dtype=np.int64)
    for i in range(1, N):
        j = _libc.rand() % (i + 1)
        if i != j:
            order[i], order[j] = order[j], order[i]
    return order


def candidates(X, K, seed, rounds=5, w=None, metric=0):
    """Returns (candidate rows in list order, [(round, drawn, phi)], nearest list index of every row)."""
    X = np.ascontiguousarray(X, np.float32)
    N = len(X)
    ell = 2.0 * K
    rows = [first_centroid(X, seed, w)]
    d = row_distances(X, X[rows[0]][None], np.zeros(N, np.uint32), metric)
    d[X[:, 0] != X[:, 0]] = 0
    nearest = np.zeros(N, np.int64)
    log = []
    for r in range(1, rounds + 1):
        phi = float(np.sum(mass(d, w)))
        if not phi > 0:
            break
        new = np.nonzero(draws(d, w, seed, r, ell, phi))[0]
        log.append((r, len(new), phi))
        if len(new) == 0:
            continue
        base = len(rows)
        rows.extend(int(i) for i in new)
        a = O.assign_lloyd(X, X[new], metric=metric)[0]
        e = row_distances(X, X[new], np.minimum(a, len(new) - 1), metric)
        upd = (a < len(new)) & (e < d)
        d[upd] = e[upd]
        nearest[upd] = base + a[upd].astype(np.int64)
    return np.array(rows, np.int64), log, nearest


def candidate_weights(nearest, n_cand, w=None):
    """W_j = sum of w_i over the rows nearest to candidate j (exact for integer weights)"""
    return np.bincount(nearest, weights=None if w is None else np.asarray(w, np.float64),
                       minlength=n_cand).astype(np.float32)


def fill(X, rows, K, seed, w=None):
    """at most K candidates: the candidates, then init_random's walk over the rows not chosen yet"""
    _libc.srand(seed & 0xFFFFFFFF)
    taken = set(int(i) for i in rows)
    out = list(rows)
    for i in random_order(len(X)):
        if len(out) == K:
            break
        if int(i) in taken or (w is not None and not w[i] > 0):
            continue
        out.append(int(i))
    return X[np.array(out)]


def log_lines(log, n_cand, K):
    lines = ["k-means|| round %d: %d candidates, cost %.17g" % rec for rec in log]
    return lines + ["k-means||: %d candidates -> %d centroids" % (n_cand, K)]
