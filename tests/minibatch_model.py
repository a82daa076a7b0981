"""NumPy model of mini-batch k-means (kmeans_cuda(..., batch_size=b); include/kmcuda_b200.h, DESIGN.md §4h).

It restates the library's draws (csrc/minibatch.cu) and scikit-learn's MiniBatchKMeans rules: the centroid update of
_mini_batch_update_dense, the random reassignment of _mini_batch_step, _random_reassign and _mini_batch_convergence.
tests/test_minibatch_cpu.py checks it against scikit-learn itself; tests/test_minibatch_gpu.py pins the library to it.
Batch labels come from the caller (the oracle's argmin for the GPU pin), so the model holds no assignment rule."""
import numpy as np

M64 = (1 << 64) - 1
TAG_BATCH = 0x6D696E6962617463      # kernels.h: kMbTagBatch
TAG_REASSIGN = 0x7265617373696721   # kernels.h: kMbTagReassign
REASSIGNMENT_RATIO = 0.01
MAX_NO_IMPROVEMENT = 10


def mix(z):
    """SplitMix64 finaliser on a Python int"""
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def mix_np(z):
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def step_key(seed, step, tag):
    return mix((mix(tag ^ (seed & 0xFFFFFFFF)) + step) & M64)


def draw(seed, step, N, b):
    """row_j = floor(u(seed, step, j) * N), j < b"""
    h = mix_np(np.uint64(step_key(seed, step, TAG_BATCH)) ^ np.arange(b, dtype=np.uint64))
    u = (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return np.minimum(np.floor(u * N).astype(np.int64), N - 1)


def reassign_keys(seed, step, wb):
    """Efraimidis-Spirakis keys -log(u) / w of the batch entries (+inf for weight 0); the smallest are drawn"""
    h = mix_np(np.uint64(step_key(seed, step, TAG_REASSIGN)) ^ np.arange(len(wb), dtype=np.uint64))
    u = ((h >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    wb = np.asarray(wb, np.float64)
    with np.errstate(divide="ignore"):
        return np.where(wb > 0, -np.log(u) / np.where(wb > 0, wb, 1.0), np.inf)


def step(Xb, wb, labels, C, W, reassign=False, keys=None):
    """one mini-batch step in float64.  labels[j] >= K: no member.  Returns (C_new, W_new, inertia, shift,
    reassigned centroid indices)"""
    Xb = np.asarray(Xb, np.float64)
    C = np.asarray(C, np.float64)
    W = np.asarray(W, np.float64)
    wb = np.asarray(wb, np.float64)
    K, D = C.shape
    b = len(Xb)
    live = labels < K
    lab = np.where(live, labels, 0)
    inertia = float(np.sum(np.where(live, wb * ((Xb - C[lab]) ** 2).sum(1), 0.0)))
    S = np.zeros((K, D))
    Wb = np.zeros(K)
    np.add.at(S, lab[live], Xb[live] * wb[live, None])
    np.add.at(Wb, lab[live], wb[live])
    Cn = C.copy()
    Wn = W + Wb
    upd = Wb > 0
    Cn[upd] = (C[upd] * W[upd, None] + S[upd]) / Wn[upd, None]
    cidx = np.zeros(0, np.int64)
    if reassign:
        order = np.argsort(Wn, kind="stable")
        cnt = int(np.sum(Wn < REASSIGNMENT_RATIO * Wn.max()))
        m = min(cnt, b // 2, int(np.sum(wb > 0)))
        picks = np.argsort(keys, kind="stable")[:m]
        cidx = order[:m]
        minkept = Wn[order[m]] if m < K else Wn[order[-1]]
        Cn[cidx] = Xb[picks]
        Wn[cidx] = minkept
    shift = float(((Cn - C) ** 2).sum())
    return Cn, Wn, inertia, shift, cidx


class Convergence:
    """scikit-learn's _mini_batch_convergence; update() returns None or the stop reason"""

    def __init__(self, b, N, tol_abs):
        self.b, self.N, self.tol = b, N, tol_abs
        self.ewa = self.ewa_min = None
        self.no_improvement = 0

    def update(self, s, inertia, shift):
        mean = inertia / self.b
        self.mean = mean
        if s == 1:
            return None
        if self.ewa is None:
            self.ewa = mean
        else:
            alpha = min(1.0, self.b * 2.0 / (self.N + 1))
            self.ewa = self.ewa * (1 - alpha) + mean * alpha
        if self.tol > 0 and shift <= self.tol:
            return "small centers change"
        if self.ewa_min is None or self.ewa < self.ewa_min:
            self.no_improvement = 0
            self.ewa_min = self.ewa
        else:
            self.no_improvement += 1
        if self.no_improvement >= MAX_NO_IMPROVEMENT:
            return "lack of improvement in inertia"
        return None


def tolerance(X, tol):
    """scikit-learn's _tolerance with the float32 tolerance the C ABI takes"""
    if tol == 0:
        return 0.0
    return float(np.asarray(X, np.float64).var(0).mean()) * float(np.float32(tol))


def run(X, C0, b, max_steps, tol, seed, labels_fn, w=None):
    """the whole loop; labels_fn(Xb, C) -> labels.  The centroids are kept in fp32 between steps, as the library keeps
    them (each blend is computed in double and rounded), so labels_fn sees the centroids the library assigns against
    up to the rounding of the member sums.  Returns (centroids, log of (step, mean, ewa or None), stop reason, steps
    taken)"""
    X = np.asarray(X)
    N = len(X)
    K = len(C0)
    b = min(b, N)
    steps = max_steps if max_steps else 100 * N // b
    C = np.asarray(C0, np.float32)
    W = np.zeros(K)
    conv = Convergence(b, N, tolerance(X, tol))
    since = 0
    log = []
    reason = None
    s = 0
    for s in range(1, steps + 1):
        since += b
        reassign = bool(np.any(W == 0)) or since >= 10 * K
        if reassign:
            since = 0
        rows = draw(seed, s, N, b)
        Xb = X[rows]
        wb = np.ones(b) if w is None else np.asarray(w, np.float64)[rows]
        labels = labels_fn(Xb, C)
        keys = reassign_keys(seed, s, wb) if reassign else None
        Cn, W, inertia, _, _ = step(Xb, wb, labels, C, W, reassign, keys)
        Cn = Cn.astype(np.float32)
        shift = float(((Cn.astype(np.float64) - C) ** 2).sum())
        C = Cn
        reason = conv.update(s, inertia, shift)
        log.append((s, conv.mean, conv.ewa if s > 1 else None))
        if reason:
            break
    return C, log, reason, s
