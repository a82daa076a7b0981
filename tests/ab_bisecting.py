"""Timing of bisecting k-means (kmeans_cuda(..., bisecting=...), DESIGN.md §4o) against Lloyd from greedy k-means++ at
the same K, on device-resident data.  Not collected by pytest.

    python tests/ab_bisecting.py --n 8000000 --d 256 --k 1024 16384 --rounds 3 [--no-lloyd-above 1024] [--out DIR]

For every data set (U[0,1) and a 1024-blob mixture) and K it prints, per variant, the median call time with its spread
over the alternated rounds and the final inertia; for the bisecting runs also the waves, nodes bisected and
wave-iterations (host round trips), from the verbosity-2 log.  A separate profiled call per data set and K gives the
device time of bk_step_kernel, and its share of the HBM floor for the rows it read (sum over (node, init) of the node's
rows times its E steps, 4 D bytes per row, at 3.35 TB/s).  The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def data(kind, n, d, seed=0):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "uniform":
        return torch.rand((n, d), generator=g, device="cuda")
    centers = torch.randn((1024, d), generator=g, device="cuda") * 3
    idx = torch.randint(0, 1024, (n,), generator=g, device="cuda")
    return centers[idx] + torch.randn((n, d), generator=g, device="cuda")


def call(km, X, K, variant, verbosity=0):
    import torch
    n, d = X.shape
    C = torch.empty((K, d), device="cuda")
    A = torch.empty(n, dtype=torch.int32, device="cuda")
    kw = dict(tolerance=1e-4, seed=3, verbosity=verbosity, inertia=True)
    if variant == "lloyd":
        kw.update(init="greedy-k-means++", yinyang_t=0.0)
    else:
        kw.update(init="random", bisecting=variant)
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = km.kmeans_cuda((X.data_ptr(), 0, (n, d), C.data_ptr(), A.data_ptr()), K, **kw)
    torch.cuda.synchronize()
    return time.perf_counter() - t, out[-1]


def log_counts(text, d):
    lines = [ln for ln in text.splitlines() if ln.startswith("bisecting")]
    rows = 0
    for ln in lines:
        m = re.match(r"bisecting: node \[(\d+), (\d+)\) init \d+: (\d+) iterations, stopped on (.*), inertia", ln)
        if m:
            lo, hi, it, why = int(m.group(1)), int(m.group(2)), int(m.group(3)), m.group(4)
            rows += (hi - lo) * (it + (0 if why == "equal labels" else 1))
    m = re.search(r"(\d+) waves, (\d+) nodes bisected", lines[-1])
    return int(m.group(1)), int(m.group(2)), rows


def step_split(km, X):
    """bk_step_kernel with and without the member sums: K = 2, tolerance 0, max_iter 3 runs three E + M steps and one
    final E step (which skips the S columns) over all of X; returns the device ms of each launch"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    n, d = X.shape
    C = torch.empty((2, d), device="cuda")
    A = torch.empty(n, dtype=torch.int32, device="cuda")
    args = ((X.data_ptr(), 0, (n, d), C.data_ptr(), A.data_ptr()), 2)
    kw = dict(tolerance=0.0, max_iter=3, seed=3, init="random", bisecting="biggest_inertia")
    km.kmeans_cuda(*args, **kw)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        km.kmeans_cuda(*args, **kw)
        torch.cuda.synchronize()
    return [e.device_time_total / 1e3 for e in prof.events() if "bk_step_kernel" in e.name]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8_000_000)
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--k", type=int, nargs="+", default=[1024, 16384])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-lloyd-above", type=int, default=1 << 30)
    ap.add_argument("--data", nargs="+", default=["uniform", "blobs"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import kmcuda_b200 as km
    res = {"card": card(), "n": a.n, "d": a.d, "runs": []}
    print("card:", res["card"], flush=True)
    for kind in a.data:
        X = data(kind, a.n, a.d)
        ms = step_split(km, X)
        floor_ms = a.n * 4.0 * a.d / HBM * 1e3
        row = {"data": kind, "step_ms_e_and_m": ms[:-1], "step_ms_e_only": ms[-1:], "hbm_floor_ms": floor_ms}
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
        for K in a.k:
            variants = ["biggest_inertia", "largest_cluster"] + (["lloyd"] if K <= a.no_lloyd_above else [])
            call(km, X, K, variants[0])   # warm-up: module load, memory pool
            times = {v: [] for v in variants}
            inert = {}
            for _ in range(a.rounds):
                for v in variants:
                    t, e = call(km, X, K, v)
                    times[v].append(t)
                    inert[v] = e
            for v in variants:
                ts = sorted(times[v])
                row = {"data": kind, "K": K, "variant": v, "median_s": ts[len(ts) // 2], "min_s": ts[0],
                       "max_s": ts[-1], "inertia": inert[v]}
                if v != "lloyd":
                    with tempfile.TemporaryFile() as f:   # the library logs to fd 1
                        sys.stdout.flush()
                        saved = os.dup(1)
                        os.dup2(f.fileno(), 1)
                        try:
                            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                                call(km, X, K, v, verbosity=2)
                        finally:
                            ctypes.CDLL(None).fflush(None)
                            os.dup2(saved, 1)
                            os.close(saved)
                        f.seek(0)
                        text = f.read().decode(errors="replace")
                    waves, nodes, rows = log_counts(text, a.d)
                    step = [e for e in prof.events() if "bk_step_kernel" in e.name]
                    dev_us = sum(e.device_time_total for e in step) if step else 0.0
                    row.update(waves=waves, nodes_bisected=nodes, wave_iterations=len(step),
                               step_device_ms=dev_us / 1e3, step_rows_read=rows,
                               step_hbm_share=(rows * 4.0 * a.d / HBM) / (dev_us / 1e6) if dev_us else None)
                res["runs"].append(row)
                print(json.dumps(row), flush=True)
        del X
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ab_bisecting.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
