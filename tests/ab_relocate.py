"""Timing of the empty-cluster relocation (relocate_empty_clusters=True, DESIGN.md §4l) on 8M x 256 @ 1024 device data.

    python tests/ab_relocate.py [--n 8000000] [--out relocate.json]

* the relocation keys + top-T selection alone (kmcuda_b200_debug_relocate_select, CUDA events) for m in {1, 64}, against
  the HBM floor of reading the samples once (n * D * 4 bytes at 3.35 TB/s);
* one relocating update, as the difference of two whole calls that stop after one update (tolerance 0.999): the same
  init with m far centroids, relocation on and off, m in {1, 64};
* relocation on against off when no cluster empties (init = sample rows), three alternated rounds each.
The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8_000_000)
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--k", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import kmcuda_b200 as km
    n, d, k = a.n, a.d, a.k
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.rand(n, d, device="cuda", generator=g)
    base = X[torch.randperm(n, device="cuda", generator=g)[:k]].cpu().numpy()
    res = {"card": card, "power_limit": power, "n": n, "d": d, "k": k}

    def call(C0, relocate, tol):
        Cd = torch.empty(k, d, device="cuda")
        Ad = torch.empty(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        t = time.perf_counter()
        km.kmeans_cuda((X.data_ptr(), 0, (n, d), Cd.data_ptr(), Ad.data_ptr()), k, init=C0, tolerance=tol,
                       yinyang_t=0, device=1, seed=3, relocate_empty_clusters=relocate)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    # keys + selection alone
    f = km._lib.kmcuda_b200_debug_relocate_select
    f.restype = ctypes.c_int64
    f.argtypes = [ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint16] + [ctypes.c_void_p] * 2 + \
        [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
    Ct = torch.from_numpy(base).cuda()
    assign = torch.randint(0, k, (n,), device="cuda", dtype=torch.int32, generator=g)
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    for m in (1, 64):
        T = 2 * m + 32
        top = torch.empty(T, dtype=torch.int64, device="cuda")
        args = (0, n, d, X.data_ptr(), Ct.data_ptr(), k, assign.data_ptr(), None, T, keys.data_ptr(), top.data_ptr())
        f(*args)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        reps = 10
        ev[0].record()
        for _ in range(reps):
            f(*args)
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / reps
        res["keys_select_ms_m%d" % m] = ms
    res["hbm_floor_ms"] = n * d * 4 / 3.35e12 * 1e3

    # one relocating update: the same one-update call with relocation on and off
    for m in (1, 64):
        C0 = base.copy()
        C0[k - m:] = 1e3
        call(C0, True, 0.999)
        on, off = [], []
        for _ in range(a.rounds):
            on.append(call(C0, True, 0.999))
            off.append(call(C0, False, 0.999))
        res["update_extra_ms_m%d" % m] = (float(np.median(on)) - float(np.median(off))) * 1e3
        res["calls_on_off_s_m%d" % m] = [on, off]

    # no empty cluster: on against off, whole runs
    call(base, True, 0.01)
    on, off = [], []
    for _ in range(a.rounds):
        on.append(call(base, True, 0.01))
        off.append(call(base, False, 0.01))
    res["no_empty_on_s"], res["no_empty_off_s"] = on, off
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
