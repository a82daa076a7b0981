"""NumPy model of bisecting k-means (kmeans_cuda(..., bisecting=...); include/kmcuda_b200.h, DESIGN.md §4o).

It restates scikit-learn's BisectingKMeans.fit / _bisect / _kmeans_single_lloyd with this library's draws and
arithmetic, and the host's wave schedule (Job::bisecting), so that the result and the logs can be compared bit for bit:
  * the E step is the oracle's assign_lloyd between the two centres (the reference argmin), e the Kahan sum of
    (x - c)^2 to the winner;
  * every double total is a sequential sum in position order inside chunks of CHUNK positions of the node's range,
    the chunks then added in order (np.cumsum, never np.sum, which adds pairwise);
  * the draws of a node depend on (seed, lo, hi, init r, stage, row) only.
tests/test_bisecting_cpu.py checks it against scikit-learn itself; tests/test_bisecting_gpu.py pins the library to it."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import kmeans_parallel_model as KP  # noqa: E402
import greedy_plusplus_model as GP  # noqa: E402
from oracle import oracle as O  # noqa: E402

TAG_NODE = 0x6269736563742121   # kernels.h: kBkTagNode
CHUNK = 2048                    # kernels.h: kBkChunk
STRATEGIES = {"biggest_inertia": 0, "largest_cluster": 1}
STOP = ("equal labels", "tolerance", "max_iter")
_M64 = (1 << 64) - 1


def node_key(seed, lo, hi, r, stage):
    k = KP.mix(TAG_NODE ^ (int(seed) & 0xFFFFFFFF))
    k = KP.mix((k + int(lo)) & _M64)
    k = KP.mix((k + int(hi)) & _M64)
    return KP.mix((k + ((int(r) << 8) | int(stage))) & _M64)


def draw_keys(seed, lo, hi, r, stage, rows, w):
    """-ln(u) / w of the rows (inf where w <= 0)"""
    z = KP.mix(np.uint64(node_key(seed, lo, hi, r, stage)) ^ np.asarray(rows, np.uint64))
    u = ((z >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    w = np.asarray(w, np.float64)
    with np.errstate(divide="ignore"):
        return np.where(w > 0, -np.log(u) / np.where(w > 0, w, 1.0), np.inf)


def fixed_sum(v, mask=None):
    """sum over the first axis in position order: 0.0 + each CHUNK-position chunk sequentially, the chunks in order"""
    v = np.asarray(v, np.float64)
    total = np.zeros(v.shape[1:])
    for c0 in range(0, max(len(v), 1), CHUNK):
        blk = v[c0:c0 + CHUNK]
        if mask is not None:
            blk = blk[np.asarray(mask)[c0:c0 + CHUNK]]
        total = total + np.cumsum(np.concatenate([np.zeros((1,) + v.shape[1:]), blk]), axis=0)[-1]
    return total


def sqdiff(X, c):
    """Kahan sum of (x - c)^2 per row in feature order (exact.cuh's Kahan::sqdiff), float32"""
    s = np.zeros(len(X), np.float32)
    r = np.zeros_like(s)
    with np.errstate(invalid="ignore", over="ignore"):
        for f in range(X.shape[1]):
            dd = (X[:, f] - c[f]).astype(np.float32)
            y = GP.fma_rd(dd, dd, r)
            t = (s + y).astype(np.float32)
            r = (y - (t - s)).astype(np.float32)
            s = t
    return s


def random_init(rows, w, seed, lo, hi, r):
    """the two positive-weight rows of smallest key (ties: the lower row), or None"""
    k = draw_keys(seed, lo, hi, r, 0, rows, w)
    order = np.lexsort((rows, k))
    if len(order) < 2 or not np.isfinite(k[order[1]]):
        return None
    return int(rows[order[0]]), int(rows[order[1]])


def greedy_init(Xn, rows, w, seed, lo, hi, r, L):
    """greedy k-means++ (§4m's round 1 restricted to the node): c0 = the row of smallest -ln(u) / w, d the true distance
    to it, mass m = w d^2, trial t = the row of smallest -ln(u_t) / m (stage 1 + t), phi_t = the fixed-order sum of
    mass(min(d, e_t)); the lowest phi_t (then t) is c1.  Returns the two rows, or None when no row has mass."""
    k = draw_keys(seed, lo, hi, r, 0, rows, w)
    first = np.lexsort((rows, k))[0]
    if not np.isfinite(k[first]):
        return None
    d = GP.distances(Xn, Xn[first][None])[0]
    m = KP.mass(d, w)
    if not (m > 0).any():
        return None
    trial, phis = [], []
    for t in range(L):
        kt = draw_keys(seed, lo, hi, r, 1 + t, rows, m)
        j = np.lexsort((rows, kt))[0]
        e = GP.distances(Xn, Xn[j][None])[0]
        trial.append(j)
        phis.append(float(fixed_sum(KP.mass(np.where(e < d, e, d), w))))
    best = int(np.argmin(phis))   # the first of equal potentials
    return int(rows[first]), int(rows[trial[best]])


def estep(X, w, C):
    lab = O.assign_lloyd(X, C)[0].astype(np.int64)
    e0, e1 = sqdiff(X, C[0]), sqdiff(X, C[1])
    e = np.where(lab == 1, e1, e0)
    return lab, e, w.astype(np.float64) * e.astype(np.float64)


def two_means(X, w, rows, C, tol_abs, max_iter):
    """_kmeans_single_lloyd on the node's rows X (position order) from centres C.  Returns a dict with the final labels,
    centres, inertia, per-child W / I / counts, iterations and stop reason."""
    C = np.array(C, np.float32)
    prev = None
    it = 0
    stop = 2
    wd = w.astype(np.float64)
    relocations = 0
    for i in range(max_iter):
        lab, e, we = estep(X, w, C)
        it = i + 1
        if prev is not None and np.array_equal(lab, prev):
            return _final(lab, e, we, wd, C, it, 0, relocations)
        W = [fixed_sum(wd, lab == j) for j in range(2)]
        S = [fixed_sum(wd[:, None] * X.astype(np.float64), lab == j) for j in range(2)]
        for j in range(2):   # _relocate_empty_clusters_dense for k = 2
            donor = (lab == 1 - j) & (w > 0)
            if W[j] == 0.0 and donor.sum() >= 2:
                cand = np.flatnonzero(donor)
                best = cand[np.lexsort((rows[cand], -e[cand].astype(np.float64)))[0]]
                v = np.float64(w[best]) * X[best].astype(np.float64)
                S[1 - j] = S[1 - j] - v
                S[j] = v
                W[1 - j] = W[1 - j] - np.float64(w[best])
                W[j] = np.float64(w[best])
                relocations += 1
                break
        Cn = np.array([(S[j] / W[j]).astype(np.float32) if W[j] > 0 else C[j] for j in range(2)], np.float32)
        d = Cn.astype(np.float64).ravel() - C.astype(np.float64).ravel()
        shift = np.cumsum(np.concatenate([[0.0], d * d]))[-1]
        C = Cn
        prev = lab
        if shift <= tol_abs:
            stop = 1
            break
    lab, e, we = estep(X, w, C)
    return _final(lab, e, we, wd, C, it, stop, relocations)


def _final(lab, e, we, wd, C, it, stop, relocations):
    return {"labels": lab, "C": C, "iters": it, "stop": stop, "inertia": float(fixed_sum(we)), "relocations": relocations,
            "W": [float(fixed_sum(wd, lab == j)) for j in range(2)],
            "I": [float(fixed_sum(we, lab == j)) for j in range(2)],
            "cnt": [int((lab == j).sum()) for j in range(2)]}


def tolerance_abs(X, tolerance):
    """tolerance times the mean of the unweighted per-feature variances (Job::mean_variance's arithmetic is checked on
    the GPU; numpy's two-pass variance agrees with it to rounding, so the CPU tests keep away from the boundary)"""
    Xd = X.astype(np.float64)
    var = ((Xd - Xd.mean(axis=0)) ** 2).mean(axis=0)
    return float(np.cumsum(var)[-1] / X.shape[1] * float(np.float32(tolerance)))   # the C ABI's tolerance is a float


def bisect(X, w, perm, lo, hi, seed, n_init, tol_abs, max_iter, strategy, L=0):
    """one node's bisection: (result dict or None when the node cannot be split, per-init runs); L = 0 random init,
    else greedy k-means++ with L trials"""
    rows = perm[lo:hi]
    Xn, wn = X[rows], w[rows]
    runs = []
    for r in range(n_init):
        pair = greedy_init(Xn, rows, wn, seed, lo, hi, r, L) if L else random_init(rows, wn, seed, lo, hi, r)
        if pair is None:
            return None, []
        runs.append(two_means(Xn, wn, rows, X[list(pair)], tol_abs, max_iter))
    best = 0
    for r in range(1, n_init):
        if runs[r]["inertia"] < runs[best]["inertia"] * (1 - 1e-6):
            best = r
    b = dict(runs[best])
    b["r"] = best
    b["splittable"] = b["W"][0] > 0 and b["W"][1] > 0
    b["score"] = b["I"] if strategy == 0 else [float(c) for c in b["cnt"]]
    return b, runs


def schedule(K, N, bisect_fn, on_split=None, waves=True):
    """the host's rounds (Job::bisecting).  bisect_fn(lo, hi) -> a result with "splittable", "cnt" and "score", or None
    when the node cannot be split; on_split(lo, hi, result) is called when a split is applied.  Returns (leaves
    {lo: hi} or None when fewer than K clusters can be made, events in order: ("wave", [(lo, hi), ...]),
    ("split", lo, hi, result), ("not split", lo, hi))."""
    leaves = {0: N}
    pick = {0: 0.0}          # lo -> score of the pickable leaves
    cache = {}
    events = []
    while len(leaves) < K:
        if not pick:
            return None, events
        top = sorted(pick, key=lambda lo: (-pick[lo], lo))
        lo = top[0]
        if lo not in cache:
            nodes = [p for p in top[:K - len(leaves)] if p not in cache] if waves else [lo]
            for p in nodes:
                cache[p] = bisect_fn(p, leaves[p])
            events.append(("wave", [(p, leaves[p]) for p in nodes]))
            continue
        res = cache.pop(lo)
        del pick[lo]
        hi = leaves[lo]
        if res is None or not res["splittable"]:
            events.append(("not split", lo, hi))
            continue
        mid = lo + res["cnt"][0]
        events.append(("split", lo, hi, res))
        if on_split:
            on_split(lo, hi, res)
        leaves[lo] = mid
        leaves[mid] = hi
        pick[lo] = res["score"][0]
        pick[mid] = res["score"][1]
    return leaves, events


def bisecting(X, K, seed, strategy="biggest_inertia", n_init=1, tolerance=1e-4, max_iter=300, w=None, waves=True,
              tol_abs=None, init="random"):
    """Returns (centroids [K][D], labels [N], the log lines of verbosity 2 that start with "bisecting", the final
    inertia, nodes bisected, waves); raises ValueError when fewer than K clusters can be made.  init: "random",
    "greedy-k-means++" or ("greedy-k-means++", L) with L = 0 for the default 2 + floor(ln 2) trials."""
    X = np.ascontiguousarray(X, np.float32)
    N, D = X.shape
    w = np.ones(N, np.float32) if w is None else np.asarray(w, np.float32)
    st = STRATEGIES[strategy] if isinstance(strategy, str) else strategy
    max_iter = max_iter or 300
    if tol_abs is None:
        tol_abs = tolerance_abs(X, tolerance)
    L = 0 if init == "random" else ((init[1] if isinstance(init, tuple) else 0) or GP.default_trials(2))
    perm = np.arange(N)
    runs_log = {}
    centres = {}

    def fn(lo, hi):
        res, runs = bisect(X, w, perm, lo, hi, seed, n_init, tol_abs, max_iter, st, L)
        runs_log[(lo, hi)] = runs
        return res

    def split(lo, hi, res):
        rows = perm[lo:hi]
        lab = res["labels"]
        perm[lo:hi] = np.concatenate([rows[lab == 0], rows[lab == 1]])
        centres[lo] = res["C"][0]
        centres[lo + res["cnt"][0]] = res["C"][1]

    leaves, events = schedule(K, N, fn, split, waves)
    if leaves is None:
        raise ValueError("fewer than K clusters can be made")
    lines = []
    nwaves = bisected = 0
    for ev in events:
        if ev[0] == "wave":
            nwaves += 1
            bisected += len(ev[1])
            for lo, hi in ev[1]:
                runs = runs_log[(lo, hi)]
                if not runs:
                    lines.append("bisecting: node [%d, %d) has no init" % (lo, hi))
                for r, run in enumerate(runs):
                    lines.append("bisecting: node [%d, %d) init %d: %d iterations, stopped on %s, inertia %.17g"
                                 % (lo, hi, r, run["iters"], STOP[run["stop"]], run["inertia"]))
        elif ev[0] == "not split":
            lines.append("bisecting: [%d, %d) is not split" % ev[1:])
        else:
            lo, hi, res = ev[1:]
            n0 = res["cnt"][0]
            lines.append("bisecting: split [%d, %d) into %d + %d rows, scores %.17g %.17g"
                         % (lo, hi, n0, hi - lo - n0, res["score"][0], res["score"][1]))
    los = sorted(leaves)
    C = np.array([centres[lo] for lo in los], np.float32)
    labels = np.zeros(N, np.uint32)
    for i, lo in enumerate(los):
        labels[perm[lo:leaves[lo]]] = i
    inertia = final_inertia(X, C, labels, w)
    lines.append("bisecting: %d waves, %d nodes bisected, inertia %.17g" % (nwaves, bisected, inertia))
    return C, labels, lines, inertia, bisected, nwaves


def final_inertia(X, C, labels, w):
    """Job::inertia: sum w e with e the Kahan sum of (x - c)^2 to the row's centroid, added as launch_inertia adds it"""
    e = np.zeros(len(X), np.float32)
    for i in range(len(C)):
        m = labels == i
        e[m] = sqdiff(X[m], C[i])
    return GP.block_sum(np.where(w > 0, w.astype(np.float64) * e.astype(np.float64), 0.0))
