"""Seeded inputs of one Yinyang iteration for `test_yinyang_step_gpu.py` (the library's step against the oracle's
`ko_yy_step`, bit for bit) and `test_yinyang_step_cpu.py` (the oracle step equals Lloyd's assignment, and each input
reaches the edge it is built for).

`build(name, D, metric)` returns `(X, C_old, C_new, groups, G, assign, bounds)`: the state right after a centroid update
of a Yinyang run -- `bounds` ([n][G + 1], the library's layout) were refreshed at `C_old` for `assign`, and the step
measures the drifts from `C_old` to `C_new`, runs the global filter and the local step.

Every input bound is valid: `ko_yy_init` at `C_old`, then pulled in by a relative 1e-5 (lower bounds down, the upper bound
up) so that the fp32 triangle inequality cannot break it by an ulp after the decay, or loosened on purpose (`lb = 0`,
`lb x U(0.5, 1)`).  The library's tensor-core and CTA routes equal the reference-order scan only for valid bounds
(yinyang.cu, header).  Exact equalities are used only where they hold by construction: `C_new == C_old` for every
member of a group gives drift 0 and maxdrift 0, so decayed bounds keep their bits.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402

FLT_MAX = np.float32(np.finfo(np.float32).max)
H100_SMS = 132
# surviving-row counts at the 64 / 128-row tile edges of MODE 1; "few": fewer 128-row tiles than an H100 has SMs
SURVIVORS = {"0": 0, "1": 1, "63": 63, "64": 64, "65": 65, "127": 127, "128": 128, "129": 129,
             "few": 128 * (H100_SMS // 2) + 37}
CASES = (["natural"] + ["survivors_" + s for s in SURVIVORS] +
         ["ties", "groups_1", "groups_7", "groups_quarter", "groups_half", "nonfinite", "overflow", "queue", "k5000"])
DUPES = 40           # exact copies of one centroid: more candidates than MAX_CAND = 32


def _unit(a):
    a = np.asarray(a, np.float64)
    return (a / np.linalg.norm(a, axis=-1, keepdims=True)).astype(np.float32)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _metric(metric):
    return 1 if metric == "cos" else 0


def _groups(K, G, rng, empty=0):
    """every group 0 .. G - empty - 1 gets at least one member; the last `empty` groups none"""
    live = G - empty
    g = np.concatenate([np.arange(live), rng.integers(0, live, K - live)])
    return g[rng.permutation(K)].astype(np.uint32)


def _blobs(n, D, K, rng, metric, sigma):
    """K centres, n rows around them (sigma per feature), C_old = the centres moved by 0.02 per feature"""
    centres = rng.standard_normal((K, D))
    lab = rng.integers(0, K, n)
    X = centres[lab] + sigma * rng.standard_normal((n, D))
    C = centres + 0.02 * rng.standard_normal((K, D))
    if metric == "cos":
        return _unit(X), _unit(C)
    return _f32(X), _f32(C)


def _moved(C, rng, metric, scale=0.01):
    Cn = C + scale * rng.standard_normal(C.shape)
    return _unit(Cn) if metric == "cos" else _f32(Cn)


def init_bounds(X, C, assign, groups, G, metric):
    return O.yy_init(X, C, assign, groups, G, _metric(metric))


def pull_in(b):
    """lower bounds x (1 - 1e-5), finite upper bounds x (1 + 1e-5)"""
    b = b.copy()
    lb = b[:, 1:]
    fin = np.isfinite(lb) & (lb < FLT_MAX)
    lb[fin] = (lb[fin].astype(np.float64) * (1 - 1e-5)).astype(np.float32)
    ub = b[:, 0]
    fin = np.isfinite(ub) & (ub < FLT_MAX)
    ub[fin] = (ub[fin].astype(np.float64) * (1 + 1e-5)).astype(np.float32)
    return b


def adjust_sequence(X, C0, steps, metric):
    """a Lloyd start and `steps` oracle centroid updates: [(C, assign, prev, ccounts)] where C is the table the
    assignments were made against and the next entry's C = ko_adjust(C, prev, assign)"""
    m = _metric(metric)
    a, prev, _ = O.assign_lloyd(X, C0, metric=m)
    C, cnt = O.adjust(X, C0, prev, a, np.zeros(len(C0), np.uint32), metric=m)
    a, prev, _ = O.assign_lloyd(X, C, metric=m, assign=a)
    out = [(C, a, prev, cnt)]
    for _ in range(steps):
        C, cnt = O.adjust(X, C, prev, a, cnt, metric=m)
        out.append((C, None, None, cnt))
    return out


def natural(D, metric, seed, n=1024, K=200, G=None):
    """C_new = one ko_adjust from C_old: the state of a real run"""
    rng = np.random.default_rng(seed)
    X, C0 = _blobs(n, D, K, rng, metric, sigma=0.7)
    C0 = X[rng.choice(n, K, replace=False)].copy()
    (C_old, a, _, _), (C_new, _, _, _) = adjust_sequence(X, C0, 1, metric)
    G = G or K // 10
    groups = _groups(K, G, rng)
    b = pull_in(init_bounds(X, C_old, a, groups, G, metric))
    return X, C_old, C_new, groups, G, a, b


def survivors(D, metric, seed, count):
    """C_new == C_old, exact bounds, well separated rows (every row pruned), lb = 0 on exactly `count` rows"""
    rng = np.random.default_rng(seed)
    n, K, G = max(512, count + 256), 100, 7
    X, C = _blobs(n, D, K, rng, metric, sigma=0.05)
    a = O.assign_lloyd(X, C, metric=_metric(metric))[0]
    groups = _groups(K, G, rng)
    b = init_bounds(X, C, a, groups, G, metric)
    rows = np.sort(rng.choice(n, count, replace=False))
    b[rows, 1:] = 0.0
    return X, C, C.copy(), groups, G, a, b


def tie_rows(n):
    """row sets of `ties`: candidate at ub, two tied candidates below ub, lb == ub after decay"""
    return np.arange(0, 40), np.arange(40, 80), np.arange(80, 120)


def ties(D, metric, seed):
    """C_new == C_old (drift 0).  Rows 0-39: centroid 2 is an exact copy of their own centroid 5 (a candidate at
    exactly ub with the lower index: the own centroid stays, strict '<').  Rows 40-79: own centroid 9, two exact copies
    11 and 300 of a closer point (the lower index wins, through yy_finish_kernel on the tensor-core route).  Rows
    80-119: `DUPES` exact copies of a closer point, at indices one CTA kernel thread apart and across its 4-chain loop,
    so the row has more than 32 candidates and reaches yy_rows_cta_kernel on every route.  Rows 120-159: every lower
    bound == the upper bound (valid: the own centroid is the nearest), so min lb == ub after the decay and the row is
    pruned (filter #1 uses '>=')."""
    rng = np.random.default_rng(seed)
    n, K, G = 512, 1500, 13
    X, C = _blobs(n, D, K, rng, metric, sigma=0.05)
    r_at, r_two, r_many = tie_rows(n)
    r_eq = np.arange(120, 160)
    far = 3.0 if metric == "L2" else 0.3
    # rows 0-39 sit near centroid 5, its copy at 2
    C[2] = C[5]
    X[r_at] = C[5] + 0.05 * rng.standard_normal((len(r_at), D))
    # rows 40-79: a point p, copies at 11 and 300, own centroid 9 farther away
    p = C[9].astype(np.float64) + far * 0.2 * rng.standard_normal(D)
    X[r_two] = p + 0.01 * rng.standard_normal((len(r_two), D))
    C[11] = C[300] = p
    # rows 80-119: DUPES copies of a point q (indices 17 + 37 j: never a multiple of 256 apart, up to 1460)
    dup_idx = 17 + 37 * np.arange(DUPES)
    q = C[40].astype(np.float64) + far * 0.2 * rng.standard_normal(D)
    X[r_many] = q + 0.01 * rng.standard_normal((len(r_many), D))
    C[dup_idx] = q
    if metric == "cos":
        X, C = _unit(X), _unit(C)
    X, C = _f32(X), _f32(C)
    a = O.assign_lloyd(X, C, metric=_metric(metric))[0]
    a[r_at] = 5
    a[r_two] = 9
    a[r_many] = 40
    groups = _groups(K, G, rng)
    groups[2], groups[5] = 0, 1                 # the copy at ub and the own centroid in different groups
    b = init_bounds(X, C, a, groups, G, metric)
    b[r_at, 1:] = 0.0                           # every group unpruned: the copy at 2 is evaluated
    b[r_two, 1:] = np.minimum(b[r_two, 1:], 0.5 * b[r_two, :1])
    b[r_many, 1:] = 0.0
    b[r_eq, 1:] = b[r_eq, :1]
    return X, C, C.copy(), groups, G, a, b


def group_edges(D, metric, seed, G_kind):
    """G = 1, 7, K / 4 or K / 2 (the largest G the API accepts).  Centroids move (drift > 0) except those of the
    singleton groups; dead centroids (groups[c] = G); one empty group (maxdrift -FLT_MAX, its bounds decay to inf) for
    G > 1.  Rows of the singleton groups' centroids (the own group has no other member, yy_finish_kernel must not take
    its bound) carry lb = 1.5 ub on the own group -- valid, there is nothing else in it, and pruned yet below every
    other candidate -- and lb = 0 on one other group, so they reach the local step."""
    rng = np.random.default_rng(seed)
    n, K = 1024, 300
    G = {"1": 1, "7": 7, "quarter": K // 4, "half": K // 2}[G_kind]
    X, C_old = _blobs(n, D, K, rng, metric, sigma=0.5)
    a = O.assign_lloyd(X, C_old, metric=_metric(metric))[0]
    empty = 1 if G > 1 else 0
    groups = _groups(K, G, rng, empty=empty)
    dead = np.array([7, 8, 150])
    singles = np.array([], np.int64)
    if G >= 7:
        singles = np.array([3, 4, 5])
        for j, c in enumerate(singles):     # groups 0, 1, 2 become {3}, {4}, {5}; their other members go to group 3
            groups[groups == j] = 3
            groups[c] = j
    groups[dead] = G
    C_new = _moved(C_old, rng, metric)
    C_new[singles] = C_old[singles]
    b = pull_in(init_bounds(X, C_old, a, groups, G, metric))
    own = np.flatnonzero(np.isin(a, singles))
    if len(own):
        b[own, 1 + groups[a[own]]] = 1.5 * b[own, 0]
        other = (groups[a[own]] + 3) % (G - empty)
        b[own, 1 + other] = 0.0
    loose = rng.random(n) < 0.3                 # looser lower bounds on some rows: lb x U(0.5, 1)
    loose[own] = False
    b[loose, 1:] *= rng.uniform(0.5, 1.0, (int(loose.sum()), G)).astype(np.float32)
    return X, C_old, C_new, groups, G, a, b


def nonfinite(D, metric, seed):
    """centroids 11 and 12 NaN in C_new only (L2 empty clusters), 12 the own centroid of rows 0-29; rows 30-39 NaN in
    a feature other than the first; rows 40-49 NaN in the first feature and assigned K; the rest natural"""
    rng = np.random.default_rng(seed)
    n, K, G = 1024, 300, 20
    X, C_old = _blobs(n, D, K, rng, metric, sigma=0.4)
    X[:30] = C_old[12] + 0.05 * rng.standard_normal((30, D)).astype(np.float32)
    if metric == "cos":
        X = _unit(X)
    X[30:40, min(1, D - 1) if D > 1 else 0] = np.nan
    X[30:40, D // 2] = np.nan
    X[40:50, 0] = np.nan
    a = O.assign_lloyd(X, C_old, metric=_metric(metric))[0]
    a[:30] = 12
    a[30:40] = 20               # (the Lloyd pass leaves these rows untouched: every score is NaN)
    a[40:50] = K
    groups = _groups(K, G, rng)
    C_new = _moved(C_old, rng, metric)
    C_new[11] = np.nan
    C_new[12] = np.nan
    b = pull_in(init_bounds(X, C_old, a, groups, G, metric))
    return X, C_old, C_new, groups, G, a, b


def _rings(D, metric, seed, n_points, per_point, rows_per, K):
    """n_points points, `per_point` centroids nearly equidistant from each (more candidates than the tensor-core
    margin can tell apart), every other centroid far; rows near the points, lb = 0 everywhere"""
    rng = np.random.default_rng(seed)
    P = 4.0 * rng.standard_normal((n_points, D))
    C = 4.0 * rng.standard_normal((K, D)) + 40.0
    for j in range(n_points):
        u = rng.standard_normal((per_point, D))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        C[j * per_point:(j + 1) * per_point] = P[j] + u
    lab = np.repeat(np.arange(n_points), rows_per)
    X = P[lab] + 1e-4 * rng.standard_normal((len(lab), D))
    if metric == "cos":
        X, C = _unit(X), _unit(C)
    X, C = _f32(X), _f32(C)
    a = O.assign_lloyd(X, C, metric=_metric(metric))[0]
    G = 16
    groups = _groups(K, G, rng)
    C_new = C.copy()
    C_new[n_points * per_point:] = _moved(C[n_points * per_point:], rng, metric)
    b = pull_in(init_bounds(X, C, a, groups, G, metric))
    b[:, 1:] = 0.0
    return X, C, C_new, groups, G, a, b


def overflow(D, metric, seed):
    """rows with 40 near-equidistant centroids: more than 32 candidates, the overflow list of MODE 1"""
    return _rings(D, metric, seed, n_points=8, per_point=40, rows_per=64, K=400)


def queue(D, metric, seed):
    """every row survives with 24 candidates: 2048 x 24 pairs > 10 n + 1024, the pair queue fills part-way"""
    return _rings(D, metric, seed, n_points=32, per_point=24, rows_per=64, K=800)


def k5000(D, metric, seed):
    """K = 5000 (the CTA kernel's outer loop over c0 += 1024): natural rows, lb = 0 on 300 of them, and `DUPES` copies
    of one point at indices spread over all five 1024-blocks for rows 0-39"""
    rng = np.random.default_rng(seed)
    n, K, G = 2048, 5000, 50
    X, C_old = _blobs(n, D, K, rng, metric, sigma=0.3)
    dup_idx = 29 + 125 * np.arange(DUPES)
    q = C_old[1].astype(np.float64) + 0.3 * rng.standard_normal(D)
    if metric == "cos":
        q = _unit(q[None])[0]
    C_old[dup_idx] = q
    X[:40] = q + 0.01 * rng.standard_normal((40, D))
    if metric == "cos":
        X = _unit(X)
    X = _f32(X)
    a = O.assign_lloyd(X, C_old, metric=_metric(metric))[0]
    a[:40] = 1
    groups = _groups(K, G, rng)
    C_new = _moved(C_old, rng, metric, scale=0.002)
    C_new[dup_idx] = C_old[dup_idx]
    b = pull_in(init_bounds(X, C_old, a, groups, G, metric))
    b[:40, 1:] = 0.0
    b[rng.choice(np.arange(40, n), 300, replace=False), 1:] = 0.0
    return X, C_old, C_new, groups, G, a, b


def build(name, D, metric="L2", seed=0):
    s = seed * 7919 + D * 31 + len(name) + (0 if metric == "L2" else 5000)
    if name == "natural":
        return natural(D, metric, s)
    if name.startswith("survivors_"):
        return survivors(D, metric, s, SURVIVORS[name.split("_", 1)[1]])
    if name == "ties":
        return ties(D, metric, s)
    if name.startswith("groups_"):
        return group_edges(D, metric, s, name.split("_", 1)[1])
    return {"nonfinite": nonfinite, "overflow": overflow, "queue": queue, "k5000": k5000}[name](D, metric, s)


def chain(D, metric="L2", seed=0, steps=4):
    """4 consecutive steps without a refresh: (X, groups, G, assign, bounds, [C_0 .. C_steps]) with C_{k+1} =
    ko_adjust(C_k) over the oracle's own step results.  The caller carries assign / bounds across the steps."""
    rng = np.random.default_rng(seed + D)
    n, K = 1024, 200
    X, _ = _blobs(n, D, K, rng, metric, sigma=0.7)
    C0 = X[rng.choice(n, K, replace=False)].copy()
    (C, a, prev, cnt), = adjust_sequence(X, C0, 0, metric)
    G = K // 10
    groups = _groups(K, G, rng)
    b = pull_in(init_bounds(X, C, a, groups, G, metric))
    m = _metric(metric)
    Cs = [C]
    aa, bb, pp = a, b, prev
    for _ in range(steps):
        Cn, cnt = O.adjust(X, Cs[-1], pp, aa, cnt, metric=m)
        dr, md = O.yy_drifts(Cn, Cs[-1], groups, G, m)
        aa, pp, bb = O.yy_step(X, Cn, groups, G, dr, md, aa, bb, m)[:3]
        Cs.append(Cn)
    return X, groups, G, a, b, Cs


def oracle_step(X, C_old, C_new, groups, G, assign, bounds, metric="L2"):
    """(drift, maxdrift, assign, prev, bounds, changed, tight, passed) of ko_yy_drifts + ko_yy_step"""
    m = _metric(metric)
    dr, md = O.yy_drifts(C_new, C_old, groups, G, m)
    return (dr, md) + O.yy_step(X, C_new, groups, G, dr, md, assign, bounds, m)
