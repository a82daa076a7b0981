"""The oracle's single Yinyang iteration (`ko_yy_init` / `ko_yy_drifts` / `ko_yy_step`, oracle/kmcuda_oracle.c) and the
inputs of `yinyang_step_cases.py` (no GPU needed).

- The split oracle reproduces whole runs recorded before the split (tests/golden/yinyang_runs.npz): log lines,
  assignments and centroids, bit for bit.
- One step from valid bounds gives Lloyd's assignment (`ko_assign_lloyd` at C_new, fp64 near-ties exempt) and leaves
  valid bounds (fp64 distances, up to fp32 rounding): the step oracle is pinned to Lloyd's semantics, not only to itself.
- Each case reaches the edge it is built for, counted on the oracle step.  The edges only the GPU can count (more than
  32 candidates, a full pair queue) are asserted on the library's counters in test_yinyang_step_gpu.py.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_yinyang_runs as R  # noqa: E402
import yinyang_step_cases as Y  # noqa: E402
from oracle import oracle as O  # noqa: E402

D_CPU = 12
CPU_CASES = [(c, m) for c in Y.CASES for m in ("L2", "cos")]


@pytest.mark.parametrize("name", list(R.RUNS))
def test_split_oracle_reproduces_recorded_runs(name):
    rec = np.load(os.path.join(HERE, "golden", "yinyang_runs.npz"))
    C, a, log = R.logged_run(name)
    assert log == list(rec[name + "/log"])
    assert np.array_equal(a, rec[name + "/assign"])
    assert np.array_equal(C.view(np.uint32), rec[name + "/C"].view(np.uint32))


_memo = {}


def _step(name, metric):
    if (name, metric) not in _memo:
        case = Y.build(name, D_CPU, metric)
        _memo[(name, metric)] = case, Y.oracle_step(*case, metric=metric)
    return _memo[(name, metric)]


def _dist64(X, C, metric):
    Xd, Cd = X.astype(np.float64), C.astype(np.float64)
    if metric == "cos":
        return np.arccos(np.clip(Xd @ Cd.T, -1.0, 1.0))
    return np.sqrt(np.maximum((Xd ** 2).sum(1)[:, None] + (Cd ** 2).sum(1)[None] - 2.0 * Xd @ Cd.T, 0.0))


@pytest.mark.parametrize("name,metric", CPU_CASES, ids=["%s-%s" % c for c in CPU_CASES])
def test_step_gives_lloyd_assignment_and_valid_bounds(name, metric):
    (X, C_old, C_new, groups, G, a_in, b_in), (dr, md, a, prev, b, changed, tight, passed) = _step(name, metric)
    K = len(C_new)
    m = 1 if metric == "cos" else 0
    assert np.array_equal(prev, a_in)
    assert changed == int((a != a_in).sum()) and passed <= tight
    exp = O.assign_lloyd(X, C_new, metric=m)[0]
    arg, best, second = O.assign_truth(X, C_new, metric=m)
    bad_c = ~np.isfinite(C_new).all(1)
    # the reference's semantics that Lloyd does not share: a row whose own centroid turned NaN keeps it (no distance is
    # below a NaN upper bound); no row moves to a centroid outside every group
    keep = (exp != 0xFFFFFFFF) & (a_in < K)
    keep &= ~bad_c[np.minimum(a_in, K - 1)]
    keep &= groups[np.minimum(exp, K - 1)] < G
    keep &= ~O.tie_exempt(best, second)
    diff = np.flatnonzero(keep & (a != exp))
    assert len(diff) == 0, (len(diff), diff[:8], a[diff[:8]], exp[diff[:8]])
    assert np.array_equal(a[a_in >= K], a_in[a_in >= K])
    # bounds valid in fp64: ub >= d(x, own), lb[g] <= min over the other members of g
    rows = np.flatnonzero(np.isfinite(X).all(1) & (a < K))
    rows = rows[~bad_c[a[rows]]]
    d = _dist64(X[rows], C_new, metric)
    rel, tol = (1e-5, 1e-6) if metric == "L2" else (1e-4, 2e-3)   # fp32 rounding; acos near 0 amplifies it
    ub = b[rows, 0].astype(np.float64)
    own = d[np.arange(len(rows)), a[rows]]
    assert (ub >= own * (1 - rel) - tol).all(), float((own - ub).max())
    d[np.arange(len(rows)), a[rows]] = np.inf
    d[:, bad_c | (groups >= G)] = np.inf
    for g in range(G):
        members = np.flatnonzero(groups == g)
        if len(members) == 0:
            continue
        lo = d[:, members].min(1)
        lb = b[rows, 1 + g].astype(np.float64)
        fin = np.isfinite(lo)
        assert (lb[fin] <= lo[fin] * (1 + rel) + tol).all(), (g, float((lb[fin] - lo[fin]).max()))


@pytest.mark.parametrize("count", list(Y.SURVIVORS))
def test_survivor_counts_are_exact(count):
    for metric in ("L2", "cos"):
        (X, *_), (_, _, a, _, _, changed, tight, passed) = _step("survivors_" + count, metric)
        assert tight == passed == Y.SURVIVORS[count], (metric, tight, passed)


@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_ties_reach_their_edges(metric):
    (X, C_old, C_new, groups, G, a_in, b_in), (dr, md, a, prev, b, changed, tight, passed) = _step("ties", metric)
    r_at, r_two, r_many = Y.tie_rows(len(X))
    # a candidate at exactly ub with a lower index: copy 2 of the own centroid 5; the row stays
    d2 = np.array([O.lib().ko_distance(1 if metric == "cos" else 0, O._f(X[r]), O._f(C_new[2]), X.shape[1])
                   for r in r_at], np.float32)
    assert np.array_equal(d2.view(np.uint32), b[r_at, 0].view(np.uint32))
    assert (a[r_at] == 5).all()
    assert (a[r_two] == 11).all() and (a[r_many] == 17).all()
    if metric == "L2":   # drift 0 exactly (a cosine self-distance is acos of a dot that may round below 1)
        assert (dr == 0).all() and (md == 0).all()
        r_eq = np.arange(120, 160)
        minlb = (b_in[r_eq, 1:] - md[None]).min(1)
        ub = b_in[r_eq, 0] + dr[a_in[r_eq]]
        assert np.array_equal(minlb, ub)
        # pruned with '>=': the upper bound is the decayed one, and the tight count has none of these rows
        assert np.array_equal(b[r_eq, 0], ub)
        assert tight == len(r_at) + len(r_two) + len(r_many)


@pytest.mark.parametrize("kind", ["7", "quarter", "half"])
def test_group_edges_reach_their_edges(kind):
    for metric in ("L2", "cos"):
        (X, C_old, C_new, groups, G, a_in, b_in), (dr, md, a, prev, b, *_) = _step("groups_" + kind, metric)
        K = len(C_new)
        assert md[G - 1] == -Y.FLT_MAX and not (groups == G - 1).any()          # the empty group
        assert np.isinf(b[:, G]).all()                                            # FLT_MAX - (-FLT_MAX)
        assert (groups == G).sum() == 3                                           # dead centroids
        singles = [3, 4, 5]                                                       # built as singleton groups
        assert all((groups == groups[c]).sum() == 1 for c in singles)
        rows = np.flatnonzero(np.isin(a_in, singles) & (a == a_in))
        assert len(rows) > 0
        pg = groups[a_in[rows]]
        # the own-only group's bound is pruned and below the second smallest distance the step wrote for it: a local
        # step that took it as a candidate bound would have written it instead
        lb_pg = b_in[rows, 1 + pg] - md[pg]
        assert (lb_pg >= b[rows, 0]).all()
        assert (b[rows, 1 + pg] > lb_pg).sum() >= 1, metric
        assert (b[rows, 1 + pg] != b_in[rows, 1 + pg]).all()                      # the rows reached the local step
    assert G == K // 2 if kind == "half" else True


@pytest.mark.parametrize("metric", ["L2", "cos"])
def test_nonfinite_reaches_its_edges(metric):
    (X, C_old, C_new, groups, G, a_in, b_in), (dr, md, a, prev, b, *_) = _step("nonfinite", metric)
    K = len(C_new)
    assert np.isnan(dr[[11, 12]]).all() and np.isfinite(md).all()
    assert (a[:30] == 12).all() and np.isnan(b[:30, 0]).all()                    # own centroid NaN: stays, ub NaN
    assert (a[40:50] == K).all() and (prev[40:50] == K).all()
    np.testing.assert_array_equal(b[40:50], b_in[40:50])                          # assign >= K: bounds untouched
    assert np.isnan(b[30:40, 0]).all()                                            # NaN feature: NaN upper bound


def test_chain_states_stay_valid():
    X, groups, G, a, b, Cs = Y.chain(D_CPU)
    for k in range(len(Cs) - 1):
        dr, md, a2, prev, b, changed, tight, passed = Y.oracle_step(X, Cs[k], Cs[k + 1], groups, G, a, b)
        assert np.array_equal(prev, a) and passed > 0
        a = a2
    assert (a == O.assign_lloyd(X, Cs[-1])[0]).mean() > 0.999
