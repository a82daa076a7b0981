"""NumPy restatement of the AFK-MC² seeding (Job::init_afkmc2 in seeding.cu; DESIGN.md §4f), used by the CPU and GPU
tests.

c0 is kmeans_parallel_model.first_centroid (srand(seed), rand() % N, redrawn on an x[0] NaN and on weight 0) and the
true distances are greedy_plusplus_model.distances (exact.cuh's distance_exact, pinned to the oracle's ko_distance).
The rest is the host's own arithmetic:

* q_i = w_i / 2W + w_i d_i² / (2 Σ w d²) in double (unweighted: w = 1, W = N), d_i the distance to c0; rows whose
  distance to c0 is not finite (every row with a NaN feature) have q_i = 0 and add nothing to Σ w d².  The sums and the
  CDF are sequential left-to-right double sums (np.cumsum, not the pairwise np.sum); the chain reads q_i as float32.
* std::mt19937_64(seed) drives the chain; uniform() = ((g >> 11) + 0.5) 2⁻⁵³.  Each of the m chain steps draws the
  candidate first (part = uniform() · cdf[N - 1], the first row whose cdf reaches it, clamped to N - 1), then rand_a =
  (float) uniform().
* d_min of a candidate is afkmc2_min_dist_kernel's atomicMin on float bits: the smallest fmaxf(d, 0) over the first k
  centroids, NaN skipped, starting from the 0x7f7f7f7f sentinel (3.39e38); p = w · (d_min · d_min) in float32, so a
  candidate with no finite distance has p = +inf.
* A candidate replaces the current one when curr_prob == 0 or (p / q) / curr_prob > rand_a, in float32.

The model also returns its smallest decision margins.  The angular tests need them: the device's acosf and the float64
arccos the model rounds may differ by an ulp (about 1.2e-7 relative), which moves the d² terms of q and the p of the
chain by about twice that.
* A draw's margin is its distance to the CDF boundaries on either side of the drawn row, relative to the d² terms that
  boundary and the draw carry: |part - cdf_b| / (T_b + u T_N), T_b the sum of w_i d_i² / (2 Σ w d²) up to the boundary.
  It is the smallest common relative change of those terms that could move the draw to another row.
* A chain decision's margin is |ratio - rand_a| / rand_a.
"""
from collections import namedtuple
import math

import numpy as np

import greedy_plusplus_model as G
import kmeans_parallel_model as KP

DEFAULT_M = 200
SENTINEL = np.array([0x7F7F7F7F], np.uint32).view(np.float32)[0]   # afkmc2_min_dist's "no centroid yet"
_M64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------------------ std::mt19937_64
class MT19937_64:
    """std::mt19937_64 (the C++ standard's parameters), the twist vectorised over uint64 arrays"""
    NN, MM = 312, 156
    _A = np.uint64(0xB5026F5AA96619E9)
    _UP = np.uint64(0xFFFFFFFF80000000)
    _LO = np.uint64(0x7FFFFFFF)

    def __init__(self, seed=5489):
        mt = [int(seed) & _M64]
        for i in range(1, self.NN):
            mt.append((6364136223846793005 * (mt[-1] ^ (mt[-1] >> 62)) + i) & _M64)
        self.mt = np.array(mt, np.uint64)
        self.out = np.empty(0, np.uint64)

    def _mix(self, hi, lo):
        y = (hi & self._UP) | (lo & self._LO)
        return (y >> np.uint64(1)) ^ np.where((y & np.uint64(1)) != 0, self._A, np.uint64(0))

    def _twist(self):
        mt, m = self.mt, self.MM
        mt[:m] = mt[m:] ^ self._mix(mt[:m], mt[1:m + 1])                            # rows 156 ahead: old
        mt[m:-1] = mt[:self.NN - m - 1] ^ self._mix(mt[m:-1], mt[m + 1:])           # rows 156 behind: new
        mt[-1:] = mt[m - 1:m] ^ self._mix(mt[-1:], mt[:1])
        y = mt.copy()
        y ^= (y >> np.uint64(29)) & np.uint64(0x5555555555555555)
        y ^= (y << np.uint64(17)) & np.uint64(0x71D67FFFEDA60000)
        y ^= (y << np.uint64(37)) & np.uint64(0xFFF7EEE000000000)
        y ^= y >> np.uint64(43)
        return y

    def next(self, n):
        """the next n outputs (uint64)"""
        parts = [self.out]
        have = len(self.out)
        while have < n:
            parts.append(self._twist())
            have += self.NN
        buf = np.concatenate(parts)
        self.out = buf[n:]
        return buf[:n]

    def uniform(self, n):
        """n draws of init_afkmc2's uniform(): ((g >> 11) + 0.5) * 2^-53, in (0, 1)"""
        return ((self.next(n) >> np.uint64(11)).astype(np.float64) + 0.5) * (1.0 / 9007199254740992.0)


# ---------------------------------------------------------------------------------------------------- the seeding
Result = namedtuple("Result", "rows C c0 q cdf trace margin_draw margin_accept")
Step = namedtuple("Step", "cand part rand_a dmin p accepted chosen")


def chain_length(m, N):
    """init_centroids' rule for m: 0 is 200, more than N / 2 is refused (kmcudaInvalidArguments)"""
    if m == 0:
        return DEFAULT_M
    if m > N // 2:
        raise ValueError("afkmc2: m > %d is not supported (got %d)" % (N // 2, m))
    return m


def proposal(d, w=None):
    """(q as float32, cdf, running sum of the d² terms of q) from the distances d to c0: the host's double arithmetic,
    rows of non-finite d at q = 0"""
    N = len(d)
    d2 = np.asarray(d, np.float32).astype(np.float64) ** 2
    live = np.isfinite(d2)
    wi = np.ones(N) if w is None else np.asarray(w, np.float32).astype(np.float64)
    W = float(N) if w is None else math.fsum(wi)   # check_weights' total (exact for the weights the tests use)
    with np.errstate(invalid="ignore"):
        mass = np.where(live, wi * d2, 0.0)
    dsum = float(np.cumsum(mass)[-1])
    base = wi / (2.0 * W)
    with np.errstate(invalid="ignore"):
        qi = base + (wi * d2 / (2.0 * dsum) if dsum > 0 else base)
    qi = np.where(live, qi, 0.0)
    return qi.astype(np.float32), np.cumsum(qi), np.cumsum(np.where(live, qi - base, 0.0))


def min_dist(E):
    """afkmc2_min_dist_kernel over E [k, m] (distances of m candidates to k centroids): the smallest fmaxf(d, 0) that
    is not NaN, or the sentinel when it is smaller"""
    E = np.asarray(E, np.float32)
    v = np.where(np.isnan(E), SENTINEL, np.maximum(E, np.float32(0)))
    return np.minimum(v.min(axis=0), SENTINEL).astype(np.float32)


def afkmc2(X, K, seed, m=0, w=None, metric=0):
    """The seeding of init="afkmc2" (init_params m, 0 = 200).  Returns a Result: the chosen rows (c0 first), the
    centroids, c0, q, the CDF, one Step per centroid after c0 and the two smallest decision margins."""
    X = np.ascontiguousarray(X, np.float32)
    N = len(X)
    m = chain_length(m, N)
    wf = None if w is None else np.asarray(w, np.float32)
    c0 = KP.first_centroid(X, seed, wf)
    cols = [G.distances(X, X[c0][None], metric)[0]]   # distance of every row to each chosen centroid
    q, cdf, tcum = proposal(cols[0], wf)
    total = cdf[-1]
    gen = MT19937_64(seed & 0xFFFFFFFF)
    rows, trace = [c0], []
    margin_draw = margin_accept = np.inf
    for k in range(1, K):
        u = gen.uniform(2 * m)
        part = u[0::2] * total
        rand_a = u[1::2].astype(np.float32)
        cand = np.minimum(np.searchsorted(cdf, part, "left"), N - 1)
        below = np.maximum(cand - 1, 0)
        lo, t_lo = np.where(cand > 0, cdf[below], 0.0), np.where(cand > 0, tcum[below], 0.0)
        ut = u[0::2] * tcum[-1]
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.minimum((part - lo) / (t_lo + ut), (cdf[cand] - part) / (tcum[cand] + ut))
        margin_draw = min(margin_draw, float(np.min(np.where(np.isnan(rel), np.inf, rel))))
        dmin = min_dist(np.stack([c[cand] for c in cols]))
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            p = dmin * dmin if wf is None else wf[cand] * (dmin * dmin)
            cand_prob = (p / q[cand]).astype(np.float32)
            curr_prob, curr = np.float32(0), 0
            accepted = np.zeros(m, bool)
            for j in range(m):
                if curr_prob == 0:
                    take = True
                else:
                    ratio = cand_prob[j] / curr_prob
                    take = bool(ratio > rand_a[j])
                    if np.isfinite(ratio):
                        margin_accept = min(margin_accept, abs(float(ratio) - float(rand_a[j])) / float(rand_a[j]))
                if take:
                    curr, curr_prob = j, cand_prob[j]
                    accepted[j] = True
        chosen = int(cand[curr])
        trace.append(Step(cand, part, rand_a, dmin, p.astype(np.float32), accepted, chosen))
        rows.append(chosen)
        if k < K - 1:
            cols.append(G.distances(X, X[chosen][None], metric)[0])
    rows = np.array(rows, np.int64)
    return Result(rows, X[rows], c0, q, cdf, trace, margin_draw, margin_accept)


def log_line(c0):
    """the verbosity >= 1 line that opens the seeding"""
    return "afkmc2: calculating q (c0 = %d)... " % c0
