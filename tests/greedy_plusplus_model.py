"""NumPy restatement of the greedy k-means++ seeding (include/kmcuda_b200.h, DESIGN.md §4m), used by the CPU and GPU
tests.

c0 is kmeans_parallel_model.first_centroid, the masses are kmeans_parallel_model.mass, the fill walk is
kmeans_parallel_model.fill.  The true distances are the reference's Kahan chain (fma rounded down, "inverted c"),
restated over all rows at once from the oracle's ko_fma_rd, and are checked against the oracle's ko_distance in the CPU
tests.  The potentials are summed as the device sums them: a warp's shuffle tree, the four warps of a 128-row block in
order, then kmp_sum_kernel's fold of the block partials, so they match the device bit for bit.
"""
import numpy as np

import kmeans_parallel_model as KP

TAG_TRIAL = 0x677265656479212B   # kernels.h: kGppTagTrial
MAX_TRIALS = 32
_M64 = (1 << 64) - 1


def default_trials(K):
    """scikit-learn's n_local_trials: 2 + floor(ln K)"""
    return 2 + int(np.log(K))


# ------------------------------------------------------------------------------------------------ exact distances
def fma_rd(a, b, c):
    """float32 fma rounded toward -inf, element-wise (the oracle's ko_fma_rd: the product is exact in double and TwoSum
    gives the exact error of the double addition)"""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    c = np.asarray(c, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        cd = c.astype(np.float64)
        s = p + cd
        bb = s - p
        e = (p - (s - bb)) + (cd - bb)
        f = s.astype(np.float32)
        fd = f.astype(np.float64)
        down = (fd > s) | ((fd == s) & (e < 0.0))
        f = np.where(down, np.nextafter(f, np.float32(-np.inf)), f)
        zero = (s == 0.0) & (e == 0.0)
        pos_zero = (p == 0.0) & (cd == 0.0) & ~np.signbit(p) & ~np.signbit(cd)
        f = np.where(zero, np.where(pos_zero, np.float32(0.0), np.float32(-0.0)), f)
        finite = np.isfinite(s)
        return np.where(finite, f, s.astype(np.float32)).astype(np.float32)


def distances(X, Y, metric=0):
    """[len(Y), len(X)] true distances of every row of X to every row of Y (exact.cuh's distance_exact)"""
    X = np.ascontiguousarray(X, np.float32)
    Y = np.ascontiguousarray(Y, np.float32)
    s = np.zeros((len(Y), len(X)), np.float32)
    r = np.zeros_like(s)
    with np.errstate(invalid="ignore", over="ignore"):
        for f in range(X.shape[1]):
            x = X[:, f][None, :]
            y = Y[:, f][:, None]
            if metric == 1:
                v = fma_rd(x, y, r)
            else:
                dd = (x - y).astype(np.float32)
                v = fma_rd(dd, dd, r)
            t = (s + v).astype(np.float32)
            r = (v - (t - s)).astype(np.float32)
            s = t
        if metric == 1:
            # acosf: float64 arccos rounded to float32 (the device's acosf and libm's may still differ by an ulp)
            out = np.arccos(np.clip(s, -1, 1).astype(np.float64)).astype(np.float32)
            out[s >= 1] = 0
            out[s <= -1] = np.float32(np.pi)
            return out
        return np.sqrt(s).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the device's sums
def block_sum(m):
    """sum of the masses m in the device's order: per 128-row block a warp shuffle tree and the 4 warps in order, then
    kmp_sum_kernel's fold (contiguous chunks of ceil(nb / 1024) partials, then the chunks in order)"""
    m = np.asarray(m, np.float64)
    nb = max(1, -(-len(m) // 128))
    a = np.zeros(nb * 128)
    a[:len(m)] = m
    a = a.reshape(nb, 4, 32)
    while a.shape[-1] > 1:
        h = a.shape[-1] // 2
        a = a[..., :h] + a[..., h:]
    part = np.cumsum(a[..., 0], axis=1)[:, -1]   # 0.0 + p0 + p1 + p2 + p3
    per = -(-nb // 1024)
    chunks = np.zeros(1024 * per)
    chunks[:nb] = part
    chunk = np.cumsum(chunks.reshape(1024, per), axis=1)[:, -1]
    return float(np.cumsum(chunk)[-1])


# ------------------------------------------------------------------------------------------------------- the draws
def round_key(seed, r):
    """gpp_round_key: mb_step_key(seed, r, kGppTagTrial) = mix(mix(tag ^ seed) + r)"""
    return KP.mix((KP.mix(TAG_TRIAL ^ (int(seed) & 0xFFFFFFFF)) + int(r)) & _M64)


def keys(m, seed, r, t, offset=0):
    """-ln(u) / m of rows offset .. offset + len(m) - 1 in trial t of round r (inf where m = 0)"""
    kt = np.uint64(KP.mix((round_key(seed, r) + int(t)) & _M64))
    z = KP.mix(kt ^ np.arange(offset, offset + len(m), dtype=np.uint64))
    u = ((z >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    m = np.asarray(m, np.float64)
    with np.errstate(divide="ignore"):
        return np.where(m > 0, -np.log(u) / np.where(m > 0, m, 1.0), np.inf)


def trials(m, seed, r, L, cuts=()):
    """the L trial rows of round r (None when no row has mass): the smallest (key, row) per trial; `cuts` splits the rows
    into shards whose minima are merged as the host merges the devices' (minimum key, lowest row on ties)"""
    if not (np.asarray(m) > 0).any():
        return None
    bounds = [0] + list(cuts) + [len(m)]
    out = []
    for t in range(L):
        best = (np.inf, None)
        for lo, hi in zip(bounds[:-1], bounds[1:]):
            k = keys(m[lo:hi], seed, r, t, offset=lo)
            if len(k) == 0:
                continue
            j = int(np.argmin(k))   # the first of equal keys: the lowest row
            if k[j] < best[0] or (k[j] == best[0] and best[1] is not None and lo + j < best[1]):
                best = (k[j], lo + j)
        out.append(best[1])
    return out


# --------------------------------------------------------------------------------------------------- the seeding
def greedy(X, K, seed, L=None, w=None, metric=0, cuts=()):
    """Returns (chosen rows, potentials after each round, trial rows per round, filled, centroids).  filled = the number
    of centroids chosen before the potential reached 0 (K when it never did); the rest come from the fill walk."""
    X = np.ascontiguousarray(X, np.float32)
    N = len(X)
    L = L or default_trials(K)
    nan_row = X[:, 0] != X[:, 0]
    rows = [KP.first_centroid(X, seed, w)]
    d = distances(X, X[rows[0]][None], metric)[0]
    d[nan_row] = 0
    d[rows[0]] = 0
    pots, drawn = [], []
    filled = K
    for r in range(1, K):
        tr = trials(KP.mass(d, w), seed, r, L, cuts)
        if tr is None:
            filled = r
            break
        drawn.append(tr)
        E = distances(X, X[tr], metric)
        dp = np.where(E < d[None, :], E, d[None, :])
        dp[:, nan_row] = d[nan_row]
        dp[np.arange(L), tr] = 0
        phis = [block_sum(KP.mass(dp[t], w)) for t in range(L)]
        best = int(np.argmin(phis))   # the lowest t on equal potentials
        d = dp[best]
        rows.append(tr[best])
        pots.append(phis[best])
    if filled < K:
        C = KP.fill(X, rows, K, seed, w=w)
    else:
        C = X[np.array(rows)]
    return np.array(rows, np.int64), pots, drawn, filled, C


def log_lines(L, rows, pots, filled, K):
    """the verbosity-2 lines that start with "greedy k-means++" """
    lines = ["greedy k-means++: %d trials per round" % L]
    lines += ["greedy k-means++ round %d: row %d, potential %.17g" % (r, rows[r], pots[r - 1]) for r in range(1, filled)]
    if filled == K:
        lines.append("greedy k-means++: potential %.17g" % pots[-1])
    else:
        lines.append("greedy k-means++: potential 0 after %d centroids, the rest from the random walk" % filled)
    return lines
