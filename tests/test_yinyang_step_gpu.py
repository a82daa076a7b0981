"""One Yinyang iteration of the library against the oracle's `ko_yy_drifts` + `ko_yy_step`, bit for bit (run on an H100:
`pytest -m gpu`).

`Shard.debug_yy_step` runs `Shard::yy_step` -- the code the k-means Job calls -- from a given state (samples, old and new
centroids, groups, assignments, bounds) on a chosen route of the local step:

| route | upper bounds of the rows filter #1 keeps | local step |
|---|---|---|
| 0 | tensor-core exact distances | MODE 1 candidates (`tc_assign_kernel<NKB, 1>`) + `yy_finish_kernel`; rows it cannot bound to `yy_rows_cta_kernel` |
| 1 | `yy_tight_scan_kernel` | `yy_rows_cta_kernel` |
| 2 | `yy_tight_scan_kernel` | `yy_local_scan_kernel` (reference order) |

All three share the drift kernels (`yy_drifts_kernel`, `yy_group_max_kernel`) and the global filter (`yy_decay_kernel`,
`yy_pass_kernel`).  L2: drift, maxdrift, assignments, prev, the reassignment / tightened / passed counts and the whole
[n][G + 1] bounds array equal the oracle's bits (any NaN equals any NaN).  Cosine: the device acosf is not glibc's, so
assignments match the oracle up to fp64 near-ties and the three routes equal each other bit for bit.  Inputs:
`yinyang_step_cases.py`, whose edges `test_yinyang_step_cpu.py` proves are reached.  On route 0 the MODE 1 pass's
counters show that it received every surviving row (`check_counters`, `test_route_0_runs_the_mode_1_kernel`).

D covers every K-block count of the tensor-core pass (NKB 1-8 on 128-row tiles, 9-16 on 64-row tiles) and two shapes
outside it (D = 1027, 1600: routes 1 and 2 only).
"""
import os

import numpy as np
import pytest

import yinyang_step_cases as Y
from oracle import oracle as O

pytestmark = pytest.mark.gpu

TC_D = [4, 64, 128, 132, 256, 260, 384, 388, 512, 516, 640, 644, 768, 772, 896, 900, 1024]
PLANLESS_D = [1027, 1600]
COS_D = [192, 512, 772]
EVERY_D = ["natural", "ties"]
SOME_D = [c for c in Y.CASES if c not in EVERY_D and c != "k5000"]

SWEEP = [(c, D, "L2") for D in (64, 772, 1027) for c in SOME_D if not (c == "queue" and D == 1027)]
SWEEP += [(c, D, "L2") for D in TC_D + PLANLESS_D for c in EVERY_D]
SWEEP += [("k5000", 132, "L2")]
SWEEP += [(c, D, "cos") for D in COS_D for c in EVERY_D + ["nonfinite", "groups_7", "overflow"]]


@pytest.fixture(scope="module")
def km():
    import torch
    assert torch.cuda.is_available()
    import kmcuda_b200
    O.set_threads(os.cpu_count())
    return kmcuda_b200


def tc_shape(D):
    return 4 <= D <= 1024 and D % 4 == 0


def _cuda(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.view(dtype)
    return t.cuda()


def _new_shard(n, D, K, metric):
    from kmcuda_b200.shard import Shard
    return Shard(n, D, K, metric)


def device_step(sh, X, C_old, C_new, groups, G, assign, bounds, route):
    """(drift, maxdrift, assign, prev, bounds, counts) of one Shard::yy_step; inputs are host arrays or device tensors"""
    import torch
    a = assign.clone() if torch.is_tensor(assign) else _cuda(assign.astype(np.uint32), torch.int32)
    b = bounds.clone() if torch.is_tensor(bounds) else _cuda(bounds)
    prev, dr, md, cnt = sh.debug_yy_step(X, C_old, C_new, a, groups, G, b, route)
    return dr, md, a, prev, b, cnt


def _host(r):
    dr, md, a, prev, b, cnt = r
    u = np.uint32
    return (dr.cpu().numpy(), md.cpu().numpy(), a.cpu().numpy().view(u), prev.cpu().numpy().view(u), b.cpu().numpy(),
            cnt)


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _differ(x, y):
    """elementwise: the fp32 bits differ, except that any two NaNs are equal (the device's NaN is 0x7fffffff, the x86
    default NaN 0xffc00000; no comparison in the step can tell them apart)"""
    return (_bits(x) != _bits(y)) & ~(np.isnan(x) & np.isnan(y))


def assert_equal_state(got, exp, what):
    """got: host tuple of device_step; exp: oracle_step"""
    dr, md, a, prev, b, cnt = got
    edr, emd, ea, eprev, eb, ech, etight, epassed = exp
    assert not _differ(dr, edr).any(), (what, "drift", np.flatnonzero(_differ(dr, edr))[:8])
    assert not _differ(md, emd).any(), (what, "maxdrift", np.flatnonzero(_differ(md, emd))[:8])
    assert (cnt["tight"], cnt["passed"]) == (etight, epassed), (what, cnt, etight, epassed)
    bad = np.flatnonzero(a != ea)
    assert len(bad) == 0, (what, "assign", len(bad), bad[:8], a[bad[:8]], ea[bad[:8]])
    assert np.array_equal(prev, eprev), (what, "prev")
    assert cnt["changed"] == ech, (what, cnt["changed"], ech)
    rows = np.flatnonzero(_differ(b, eb).any(1))
    assert len(rows) == 0, (what, "bounds", len(rows), rows[:4], b[rows[:2]], eb[rows[:2]])


def check_counters(cnt, route, name, what):
    assert cnt["error"] == 0, (what, "pipeline error 0x%x" % cnt["error"])
    if route != 0:
        return
    # every row MODE 1 receives is either queued for the exact re-check or put on the overflow list (a row the full pair
    # queue turns away is both): the counters show that the MODE 1 pass ran on every surviving row
    if name != "queue":   # the pair queue only fills on that input
        assert cnt["rechecked"] + cnt["overflowed"] == cnt["passed"], (what, cnt)
    assert cnt["rechecked"] <= cnt["passed"], (what, cnt)
    if name in ("overflow", "ties", "k5000"):
        assert cnt["overflowed"] > 0, (what, cnt)
    if name == "queue":
        assert cnt["rechecked"] > 0 and cnt["overflowed"] > 0 and cnt["rechecked"] + cnt["overflowed"] > cnt["passed"], \
            (what, cnt)


def check_cos_oracle(X, C_new, a_in, a, ea):
    """assignments equal the oracle's except fp64 near-ties (device acosf vs glibc acosf)"""
    bad = np.flatnonzero(a != ea)
    if len(bad):
        _, best, second = O.assign_truth(X[bad], C_new, metric=1)
        bad = bad[~O.tie_exempt(best, second)]
    assert len(bad) == 0, ("cos assign", bad[:8], a[bad], ea[bad])


@pytest.mark.parametrize("name,D,metric", SWEEP, ids=["%s-D%d-%s" % c for c in SWEEP])
def test_yinyang_step(km, name, D, metric):
    import torch
    X, C_old, C_new, groups, G, assign, bounds = Y.build(name, D, metric)
    n, K = len(X), len(C_new)
    sh = _new_shard(n, D, K, metric)
    Xt, Co, Cn = _cuda(X), _cuda(C_old), _cuda(C_new)
    routes = [0, 1, 2] if tc_shape(D) else [1, 2]
    got = {}
    for r in routes:
        got[r] = _host(device_step(sh, Xt, Co, Cn, groups, G, assign, bounds, r))
        check_counters(got[r][5], r, name, "%s D%d %s route %d" % (name, D, metric, r))
    torch.cuda.synchronize()
    sh.close()
    exp = Y.oracle_step(X, C_old, C_new, groups, G, assign, bounds, metric)
    if metric == "L2":
        for r in routes:
            assert_equal_state(got[r], exp, "route %d" % r)
        return
    check_cos_oracle(X, C_new, assign, got[routes[0]][2], exp[2])
    keys = ("changed", "tight", "passed")
    for r in routes[1:]:
        for i, what in enumerate(("drift", "maxdrift", "assign", "prev", "bounds")):
            x, y = got[r][i], got[routes[0]][i]
            same = np.array_equal(x, y) if x.dtype == np.uint32 else not _differ(x, y).any()
            assert same, ("route %d vs %d" % (r, routes[0]), what)
        assert [got[r][5][k] for k in keys] == [got[routes[0]][5][k] for k in keys]


@pytest.mark.parametrize("D", [256, 772, 1027])
def test_yinyang_chain_of_steps(km, D):
    """4 steps without a refresh: assignments and bounds carried on the device, the oracle's centroid sequence"""
    X, groups, G, a0, b0, Cs = Y.chain(D)
    n, K = len(X), len(Cs[0])
    sh = _new_shard(n, D, K, "L2")
    Xt = _cuda(X)
    Ct = [_cuda(C) for C in Cs]
    for r in ([0, 1, 2] if tc_shape(D) else [1, 2]):
        a, b = a0, b0
        import torch
        at, bt = _cuda(a0.astype(np.uint32), torch.int32), _cuda(b0)
        for k in range(len(Cs) - 1):
            exp = Y.oracle_step(X, Cs[k], Cs[k + 1], groups, G, a, b)
            res = device_step(sh, Xt, Ct[k], Ct[k + 1], groups, G, at, bt, r)
            got = _host(res)
            check_counters(got[5], r, "chain", "chain step %d route %d" % (k, r))
            assert_equal_state(got, exp, "chain step %d route %d" % (k, r))
            a, b = exp[2], exp[4]
            at, bt = res[2], res[4]
    sh.close()


@pytest.mark.parametrize("D", [256, 772])
def test_route_0_runs_the_mode_1_kernel(km, D):
    """the tensor-core route's local step is the MODE 1 pass: on a fresh shard (its plan's counters start at 0) the
    re-check queue and the overflow list are written only by the MODE 1 emitter, so every surviving row must show up in
    exactly one of them (the pair queue does not fill on this input)"""
    X, C_old, C_new, groups, G, assign, bounds = Y.build("natural", D)
    sh = _new_shard(len(X), D, len(C_new), "L2")
    cnt = device_step(sh, _cuda(X), _cuda(C_old), _cuda(C_new), groups, G, assign, bounds, 0)[5]
    sh.close()
    assert cnt["error"] == 0 and cnt["passed"] > 0, cnt
    assert cnt["rechecked"] > 0 and cnt["rechecked"] + cnt["overflowed"] == cnt["passed"], cnt


@pytest.mark.parametrize("D", [4, 132, 772, 1027, 1600])
def test_exact_refresh_equals_oracle_bits(km, D):
    """debug_yy_bounds(use_tc=False), the exact refresh, against ko_yy_init: every bound bit for bit (natural rows;
    NaN rows, a row assigned K and NaN centroids in the second input)"""
    for name in ("natural", "nonfinite"):
        X, C_old, C_new, groups, G, assign, _ = Y.build(name, D)
        C = C_new if name == "nonfinite" else C_old
        import torch
        sh = _new_shard(len(X), D, len(C), "L2")
        got = sh.debug_yy_bounds(_cuda(X), _cuda(C), _cuda(assign.astype(np.uint32), torch.int32), groups, G,
                                 False).cpu().numpy()
        sh.close()
        exp = O.yy_init(X, C, assign, groups, G)
        rows = np.flatnonzero(_differ(got, exp).any(1))
        assert len(rows) == 0, (name, len(rows), rows[:4], got[rows[:2]], exp[rows[:2]])
