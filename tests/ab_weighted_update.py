"""A/B timing of the weighted centroid update (DESIGN.md §4f): unweighted vs all-ones weights vs lognormal weights.

    python tests/ab_weighted_update.py [--rounds 3] [--points 8000000] [--tolerance 0.05]

bench.py's distribution (uniform [0, 1) samples, 8M x 256, K = 1024 sample rows as centroids) is generated on the
device and passed as device pointers, init=import, yinyang_t=0 (Lloyd).  Every arm runs in its own child process with
KMCUDA_B200_TIMING=1; the library's "centroid update" phase total is divided by the number of updates of the run
(iterations - 1).  The arms are alternated `--rounds` times.  Prints one JSON line: card, power limit, per-arm medians
and spreads (max - min) in ms per update.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("unweighted", "ones", "lognormal")


def child(arm, points, dim, k, tolerance):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import kmcuda_b200 as km
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(777)
    X = torch.rand((points, dim), generator=g, device="cuda", dtype=torch.float32)
    C0 = X[torch.randperm(points, generator=g, device="cuda")[:k]].cpu().numpy()
    w = None
    if arm == "ones":
        w = torch.ones(points, device="cuda", dtype=torch.float32)
    elif arm == "lognormal":
        w = torch.empty(points, device="cuda", dtype=torch.float32).log_normal_(0.0, 1.0, generator=g)
    torch.cuda.synchronize()
    cp, ap = km.kmeans_cuda((X.data_ptr(), 0, (points, dim)), k, init=C0, tolerance=tolerance, yinyang_t=0,
                            device=1, verbosity=1, sample_weight=None if w is None else w.data_ptr())
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        out["power_limit_w"] = None
    return out


def run_arm(arm, a):
    env = dict(os.environ, KMCUDA_B200_TIMING="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, "--points", str(a.points),
                        "--dim", str(a.dim), "--clusters", str(a.clusters), "--tolerance", str(a.tolerance)],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("%s arm failed:\n%s" % (arm, r.stderr[-2000:]))
    iters = sum(1 for ln in r.stdout.splitlines() if ln.startswith("iteration"))
    m = re.search(r"centroid update\s+([0-9.]+) ms", r.stderr)
    updates = iters - 1
    if not m or updates < 1:
        raise RuntimeError("%s arm: no update timed (%d iterations)" % (arm, iters))
    return float(m.group(1)) / updates, updates


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, default=8_000_000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--tolerance", type=float, default=0.05)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.points, a.dim, a.clusters, a.tolerance)
        return
    import numpy as np
    ms = {arm: [] for arm in ARMS}
    updates = {arm: [] for arm in ARMS}
    for _ in range(a.rounds):
        for arm in ARMS:
            t, u = run_arm(arm, a)
            ms[arm].append(t)
            updates[arm].append(u)
    res = {"what": "weighted centroid update, ms per update", "card": card(),
           "shape": [a.points, a.dim, a.clusters], "tolerance": a.tolerance, "rounds": a.rounds}
    for arm in ARMS:
        res[arm] = {"median_ms": float(np.median(ms[arm])), "spread_ms": float(max(ms[arm]) - min(ms[arm])),
                    "runs_ms": [round(x, 4) for x in ms[arm]], "updates": updates[arm]}
    base = res["unweighted"]["median_ms"]
    res["ones_over_unweighted"] = res["ones"]["median_ms"] / base
    res["lognormal_over_unweighted"] = res["lognormal"]["median_ms"] / base
    print(json.dumps(res))


if __name__ == "__main__":
    main()
