"""A/B of the mini-batch init stage (DESIGN.md §4q): seeding on all rows against init_size="auto".

    python tests/ab_minibatch_init.py [--rounds 3] [--points 8000000] [--batch 65536] [--out DIR]

Data as in tests/ab_init.py, generated on the device and passed as device pointers: uniform [0, 1) samples (8M x 256,
K = 1024) and a mixture of 1024 Gaussian blobs of the same shape.  Every arm is one mini-batch call, b = 2^16,
tolerance 0 (the steps stop by scikit-learn's no-improvement rule), seed 3, with KMCUDA_B200_TIMING=1:
  greedy-full / greedy-auto         init="greedy-k-means++" on all rows / with init_size="auto"
  kmeans++-full / kmeans++-auto     init="k-means++" on all rows / with init_size="auto"
  random-auto-n3                    init="random", n_init=3, init_size="auto" (MiniBatchKMeans(init="random"))
Per arm: the wall time of the call (it ends in a synchronisation), the seeding time (the library's "init centroids"
phase, or its "mini-batch init: seeding" phase) and validation time, and the final full-data inertia sum ||x - c||^2
in double.  The arms are alternated `--rounds` times.  Prints one JSON line: card, power limit, medians and spreads
(max - min) of the times; the inertia of a seeded call does not change between rounds.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ARMS = {"greedy-full": dict(init="greedy-k-means++"),
        "greedy-auto": dict(init="greedy-k-means++", init_size="auto"),
        "kmeans++-full": dict(init="k-means++"),
        "kmeans++-auto": dict(init="k-means++", init_size="auto"),
        "random-auto-n3": dict(init="random", init_size="auto", n_init=3)}
PHASE = re.compile(r"\[kmcuda_b200 timing\]\s+(.+?)\s+([0-9.]+) ms$")


def make_data(kind, points, dim, seed=777):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "uniform":
        return torch.rand((points, dim), generator=g, device="cuda", dtype=torch.float32)
    centers = torch.rand((1024, dim), generator=g, device="cuda", dtype=torch.float32) * 4
    label = torch.randint(0, 1024, (points,), generator=g, device="cuda")
    X = centers[label]
    X += 0.1 * torch.randn((points, dim), generator=g, device="cuda", dtype=torch.float32)
    return X


def inertia(X, cp, ap, k):
    """sum ||x - c||^2 in double over every row, from the call's device outputs"""
    import torch
    n, d = X.shape
    C = torch.empty((k, d), dtype=torch.float32, device="cuda")
    A = torch.empty(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    import kmcuda_b200 as km
    km._lib.kmcuda_b200_device_memcpy(0, C.data_ptr(), cp, C.numel() * 4, 3)
    km._lib.kmcuda_b200_device_memcpy(0, A.data_ptr(), ap, A.numel() * 4, 3)
    km._lib.kmcuda_b200_device_synchronize(0)
    total = 0.0
    for s in range(0, n, 1 << 20):
        diff = X[s:s + (1 << 20)].double() - C[A[s:s + (1 << 20)].long()].double()
        total += float((diff * diff).sum())
    return total


def call(X, k, b, kw):
    """(seconds, phases in ms, final inertia); the library's timing table goes to fd 2"""
    import kmcuda_b200 as km
    n, d = X.shape
    with tempfile.TemporaryFile(mode="w+") as err:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(err.fileno(), 2)
        try:
            t0 = time.perf_counter()
            cp, ap = km.kmeans_cuda((X.data_ptr(), 0, (n, d)), k, batch_size=b, tolerance=0.0, yinyang_t=0, seed=3,
                                    device=1, **kw)
            sec = time.perf_counter() - t0
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        err.seek(0)
        phases = {}
        for line in err:
            m = PHASE.match(line.strip())
            if m:
                phases[m.group(1)] = phases.get(m.group(1), 0.0) + float(m.group(2))
    e = inertia(X, cp, ap, k)
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    return sec, phases, e


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, default=8000000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    os.environ["KMCUDA_B200_TIMING"] = "1"
    res = {"card": card(), "points": a.points, "dim": a.dim, "clusters": a.clusters, "batch": a.batch}
    res["power_limit"] = res["card"].split(", ")[1] if ", " in res["card"] else "unknown"
    for kind in ("uniform", "blobs"):
        X = make_data(kind, a.points, a.dim)
        torch.cuda.synchronize()
        call(X, a.clusters, a.batch, ARMS["random-auto-n3"])   # warm-up: modules, the memory pool
        rec = {arm: {"call_s": [], "seed_s": [], "valid_s": [], "inertia": None} for arm in ARMS}
        for _ in range(a.rounds):
            for arm, kw in ARMS.items():
                sec, ph, e = call(X, a.clusters, a.batch, kw)
                rec[arm]["call_s"].append(sec)
                rec[arm]["seed_s"].append((ph.get("init centroids", 0.0) + ph.get("mini-batch init: seeding", 0.0))
                                          / 1e3)
                rec[arm]["valid_s"].append(ph.get("mini-batch init: validation", 0.0) / 1e3)
                rec[arm]["inertia"] = e
        for arm in ARMS:
            for key in ("call_s", "seed_s", "valid_s"):
                v = rec[arm].pop(key)
                rec[arm][key + "_median"] = round(statistics.median(v), 4)
                rec[arm][key + "_spread"] = round(max(v) - min(v), 4)
        for base in ("greedy", "kmeans++"):
            full, auto = rec[base + "-full"], rec[base + "-auto"]
            auto["call_vs_full"] = round(auto["call_s_median"] / full["call_s_median"], 4)
            auto["inertia_vs_full"] = round(auto["inertia"] / full["inertia"], 5)
        rec["random-auto-n3"]["inertia_vs_greedy_full"] = round(rec["random-auto-n3"]["inertia"] /
                                                                rec["greedy-full"]["inertia"], 5)
        res[kind] = rec
        del X
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ab_minibatch_init.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
