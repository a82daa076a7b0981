#!/usr/bin/env python
"""Timing of whole default kmeans_cuda calls (Yinyang, yinyang_t=0.1) at 512 < D <= 1024, where the Yinyang local step
and bounds refresh run on 64-row tensor-core tiles, against Lloyd calls (yinyang_t=0) and against another build of the
library (--parent-lib, loaded through KMCUDA_B200_LIB).  Run on an H100.  Checker script, not collected by pytest.

    python tests/ab_wide_yinyang.py --parent-lib variants/parent/libKMCUDA.so [--n 2000000] [--k 1024]
                                    [--dims 576,768,1024] [--blobs] [--rounds 3] [--out results/x.json]

Shapes: N x D @ K on U[0, 1) samples (the reference's benchmark distribution) for every D in --dims, initial centroids
= K random rows; with --blobs also 1M x 768 @ 1000 on the Gaussian-blob data of ab_wide_knn.py (1000 unit-normal
centres, spread 0.1), initial centroids = random rows.  Each call runs in its own process (the library and its
environment are chosen at load time): data generated on the GPU from a fixed seed, one small warm-up call, then the
timed call with KMCUDA_B200_TIMING=1 (host clock around a call that returns after the device is done).  The phase
totals of the timing report give the per-stage split: assignment passes, centroid updates, grouping, bounds refreshes,
Yinyang filter + local step; the log lines give the iteration count, the number of refreshes and whether the adaptive
switch sent the run back to Lloyd.  Arms alternate within each of --rounds rounds; medians and spreads over the rounds.
Every arm's assignments are compared with the Lloyd arm's.  Prints the card's name, power limit and max SM clock
first, then one JSON line per shape.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0]


def make_data(shape, n, k):
    """(X, C0) as host float32 arrays, deterministic per shape"""
    import torch
    if shape == "blobs":
        n, D, K = 1000000, 768, 1000
        g = torch.Generator(device="cuda").manual_seed(D)
        centers = torch.randn((K, D), generator=g, device="cuda")
        lab = torch.randint(0, K, (n,), generator=g, device="cuda")
        X = centers[lab] + 0.1 * torch.randn((n, D), generator=g, device="cuda")
    else:
        D, K = int(shape), k
        g = torch.Generator(device="cuda").manual_seed(D)
        X = torch.rand((n, D), generator=g, device="cuda", dtype=torch.float32)
    C0 = X[torch.randperm(len(X), generator=g, device="cuda")[:K]]
    return X.cpu().numpy(), C0.cpu().numpy(), K


PHASE = re.compile(r"^\[kmcuda_b200 timing\]\s{3}(\S.*?)\s+([\d.]+) ms$")


def worker(a):
    """one timed call: prints a JSON line"""
    import numpy as np
    import kmcuda_b200 as km
    X, C0, K = make_data(a.shape, a.n, a.k)
    yy = 0.0 if a.arm == "lloyd" else 0.1
    km.kmeans_cuda(X[:100000], K, init=C0, tolerance=0.5, yinyang_t=0.0, device=1)   # warm-up (modules, pool)
    os.environ["KMCUDA_B200_TIMING"] = "1"
    log_out, log_err = a.log + ".out", a.log + ".err"
    sys.stdout.flush()
    sys.stderr.flush()
    saved = os.dup(1), os.dup(2)
    with open(log_out, "w") as fo, open(log_err, "w") as fe:
        os.dup2(fo.fileno(), 1)
        os.dup2(fe.fileno(), 2)
    try:
        t0 = time.perf_counter()
        C, A = km.kmeans_cuda(X, K, init=C0, yinyang_t=yy, device=1, verbosity=1)
        dt = time.perf_counter() - t0
    finally:
        import ctypes
        ctypes.CDLL(None).fflush(None)
        os.dup2(saved[0], 1)
        os.dup2(saved[1], 2)
    out = open(log_out).read().splitlines()
    phases = {}
    for ln in open(log_err):
        m = PHASE.match(ln.rstrip("\n"))
        if m:
            phases[m.group(1)] = phases.get(m.group(1), 0.0) + float(m.group(2))
    np.save(a.log + ".npy", A)
    iters = [int(m.group(1)) for m in (re.match(r"^iteration (\d+):", ln) for ln in out) if m]
    print(json.dumps({"s": dt, "iterations": max(iters) if iters else 0,
                      "refreshes": sum("refreshing Yinyang bounds" in ln for ln in out),
                      "switched_to_lloyd": any("=> Lloyd" in ln and "Yinyang iteration" in ln for ln in out),
                      "phases_ms": phases}), flush=True)


def run_arm(a, shape, arm, tmp):
    env = dict(os.environ)
    env.pop("KMCUDA_B200_LIB", None)
    if arm == "parent":
        env["KMCUDA_B200_LIB"] = os.path.abspath(a.parent_lib)
    log = os.path.join(tmp, "%s_%s" % (shape, arm))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--shape", shape, "--arm", arm,
                        "--n", str(a.n), "--k", str(a.k), "--log", log], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("%s / %s failed:\n%s" % (shape, arm, r.stdout[-3000:]))
    return json.loads(lines[-1]), log + ".npy"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000000)
    ap.add_argument("--k", type=int, default=1024)
    ap.add_argument("--dims", default="576,768,1024")
    ap.add_argument("--blobs", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--shape")
    ap.add_argument("--arm")
    ap.add_argument("--log")
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    import numpy as np
    results = [{"card": card()}]
    print(json.dumps(results[0]), flush=True)
    arms = ["yinyang", "lloyd"] + (["parent"] if a.parent_lib else [])
    shapes = [d for d in a.dims.split(",") if d] + (["blobs"] if a.blobs else [])
    tmp = tempfile.mkdtemp()
    for shape in shapes:
        runs = {arm: [] for arm in arms}
        agree = {}
        for _ in range(a.rounds):
            for arm in arms:
                r, npy = run_arm(a, shape, arm, tmp)
                runs[arm].append(r)
                print("# %s %s: %.2f s" % (shape, arm, r["s"]), flush=True)
                agree[arm] = npy
        ref = np.load(agree["lloyd"])
        out = {"shape": "blobs 1000000 x 768 @ 1000" if shape == "blobs" else "%d x %s @ %d U[0,1)" % (a.n, shape, a.k)}
        for arm in arms:
            ts = [r["s"] for r in runs[arm]]
            last = runs[arm][-1]
            out[arm] = {"s": float(np.median(ts)), "spread_s": float(np.ptp(ts)), "rounds_s": ts,
                        "iterations": last["iterations"], "refreshes": last["refreshes"],
                        "switched_to_lloyd": last["switched_to_lloyd"],
                        "phases_ms": {k: float(np.median([r["phases_ms"].get(k, 0.0) for r in runs[arm]]))
                                      for k in last["phases_ms"]},
                        "labels_equal_to_lloyd": float((np.load(agree[arm]) == ref).mean())}
        results.append(out)
        print(json.dumps(out), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
