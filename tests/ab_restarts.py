"""Timing of k-means restarts (n_init=, DESIGN.md §4n) from pageable NumPy samples.

    python tests/ab_restarts.py [--shapes 8000000x256,2000000x768] [--k 1024] [--rounds 3] [--out restarts.json]

* per shape, one n_init=4 call against four separate n_init=1 calls with the restarts' seeds, alternated for `rounds`
  rounds (medians and spread); the n_init=4 result must equal the separate call of lowest inertia, bit for bit;
* the inertia pass alone (inertia_kernel + its fixed-order fold, torch.profiler over one n_init=2 call on device
  samples), against the HBM floor of reading the samples and assignments once (n (4 D + 4) bytes at 3.35 TB/s).
The card's name, power limit and top SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import restarts_model as M  # noqa: E402


def blobs(n, d, k, seed=0):
    """well-separated blobs in float32, generated in chunks (no float64 temporaries of the full size)"""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d), dtype=np.float32) * 3
    X = np.empty((n, d), np.float32)
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        X[s:e] = centers[rng.integers(0, k, e - s)] + 0.6 * rng.standard_normal((e - s, d), dtype=np.float32)
    return X


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="8000000x256,2000000x768")
    ap.add_argument("--k", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n-init", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import kmcuda_b200 as km
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        q = "unknown"
    res = {"card": torch.cuda.get_device_name(0), "nvidia_smi": q, "k": a.k, "n_init": a.n_init, "shapes": {}}
    R, k = a.n_init, a.k
    kw = dict(init="k-means||", tolerance=0.01, yinyang_t=0, device=1, inertia=True)
    for shape in a.shapes.split(","):
        n, d = map(int, shape.split("x"))
        X = blobs(n, d, k)
        seeds = [int(s) for s in M.seeds(7, R)]

        def timed(f):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = f()
            torch.cuda.synchronize()
            return time.perf_counter() - t, out

        one = lambda: km.kmeans_cuda(X, k, seed=7, n_init=R, **kw)   # noqa: E731
        sep = lambda: [km.kmeans_cuda(X, k, seed=s, n_init=1, **kw) for s in seeds]   # noqa: E731
        timed(lambda: km.kmeans_cuda(X, k, seed=7, n_init=1, **kw))   # warm-up: module load, workspace cache
        t_one, t_sep = [], []
        for _ in range(a.rounds):
            t, (C, A, e) = timed(one)
            t_one.append(t)
            t, singles = timed(sep)
            t_sep.append(t)
            best = M.select([s[2] for s in singles])
            Cb, Ab, eb = singles[best]
            assert np.array_equal(C.view(np.uint32), Cb.view(np.uint32)) and np.array_equal(A, Ab) and e == eb, \
                "n_init=%d differs from the separate calls" % R
        r = {"n_init_call_s": t_one, "separate_calls_s": t_sep,
             "n_init_call_median_s": float(np.median(t_one)), "separate_calls_median_s": float(np.median(t_sep)),
             "n_init_call_spread_s": float(np.ptp(t_one)), "separate_calls_spread_s": float(np.ptp(t_sep)),
             "inertias": [s[2] for s in singles], "kept": best}
        # the inertia pass alone, on device samples (the pass does not depend on where the samples came from)
        Xd = torch.from_numpy(X).cuda()
        Cd = torch.empty(k, d, device="cuda")
        Ad = torch.empty(n, dtype=torch.int32, device="cuda")
        dev = (Xd.data_ptr(), 0, (n, d), Cd.data_ptr(), Ad.data_ptr())
        km.kmeans_cuda(dev, k, seed=7, n_init=2, **kw)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            km.kmeans_cuda(dev, k, seed=7, n_init=2, **kw)
            torch.cuda.synchronize()
        passes = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "inertia_kernel" in ev.name:
                passes.setdefault("inertia_kernel", []).append(ev.device_time_total / 1e3)
        r["inertia_kernel_ms"] = passes.get("inertia_kernel", [])
        r["hbm_floor_ms"] = n * (4 * d + 4) / 3.35e12 * 1e3
        del Xd, Cd, Ad, X
        torch.cuda.empty_cache()
        res["shapes"][shape] = r
        print(json.dumps({shape: r}), flush=True)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
