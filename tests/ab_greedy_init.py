"""A/B of the seedings (DESIGN.md §4m): k-means++, k-means|| (5 rounds) and greedy k-means++ (default trials).

    python tests/ab_greedy_init.py [--rounds 2] [--points 8000000] [--lloyd-points 1000000] [--out DIR]

Data as in tests/ab_init.py, generated on the device and passed as device pointers: uniform [0, 1) samples (8M x 256,
K = 1024) and a mixture of 1024 Gaussian blobs of the same shape.  Per data set and arm: the wall time of a tolerance=1.0
call (the seeding plus one assignment pass; the host clock stops after the call, which synchronises), its average
distance (the seeding's quality), and the final average distance of a tolerance=0.01 Lloyd run on the first
`--lloyd-points` rows.  The arms are alternated `--rounds` times (`--profile-only` skips this part).  Then
torch.profiler times the kernels of a greedy k-means++ call with 8 trials per round (K = 64) on the uniform data;
the trial pass is set against the HBM floor of one read of X (N * D * 4 bytes / 3.35 TB/s).  Prints one JSON line: card, power limit, medians and spreads (max - min).
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ARMS = {"k-means++": "k-means++", "k-means||": ("k-means||", 5), "greedy-k-means++": "greedy-k-means++"}


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


def call(km, X, k, init, tolerance):
    n, d = X.shape
    cp, ap, avg = km.kmeans_cuda((X.data_ptr(), 0, (n, d)), k, init=init, tolerance=tolerance, yinyang_t=0, seed=3,
                                 device=1, average_distance=True)
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    return avg


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--points", type=int, default=8000000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--lloyd-points", type=int, default=1000000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile-only", action="store_true", help="only the kernel times")
    a = ap.parse_args()
    import torch
    import kmcuda_b200 as km
    res = {"card": card(), "points": a.points, "dim": a.dim, "clusters": a.clusters}
    for kind in () if a.profile_only else ("uniform", "blobs"):
        X = make_data(kind, a.points, a.dim)
        torch.cuda.synchronize()
        rec = {arm: {"seed_s": [], "seeded": None, "final": None} for arm in ARMS}
        for _ in range(a.rounds):
            for arm, init in ARMS.items():
                t0 = time.perf_counter()
                avg = call(km, X, a.clusters, init, 1.0)
                rec[arm]["seed_s"].append(time.perf_counter() - t0)
                rec[arm]["seeded"] = avg
        Xl = X[:a.lloyd_points].contiguous()
        for arm, init in ARMS.items():
            rec[arm]["final"] = call(km, Xl, a.clusters, init, 0.01)
        for arm in ARMS:
            s = rec[arm].pop("seed_s")
            rec[arm]["seed_s_median"] = statistics.median(s)
            rec[arm]["seed_s_spread"] = max(s) - min(s)
        res[kind] = rec
        del X, Xl
        torch.cuda.empty_cache()
    res["power_limit"] = res["card"].split(", ")[1] if ", " in res["card"] else "unknown"
    # kernel times of the greedy rounds (8 trials, 63 rounds) on the uniform data
    X = make_data("uniform", a.points, a.dim)
    call(km, X, 64, ("greedy-k-means++", 8), 1.0)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(km, X, 64, ("greedy-k-means++", 8), 1.0)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "gpp_" in e.key or "kmp_update" in e.key:
            name = re.search(r"(gpp_\w+|kmp_update_kernel)", e.key).group(1)
            t = kern.setdefault(name, [0.0, 0])
            t[0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            t[1] += e.count
    res["kernels_us_per_launch"] = {k: round(v[0] / max(v[1], 1), 1) for k, v in kern.items()}
    floor_ms = a.points * a.dim * 4 / 3.35e12 * 1e3
    res["trial_pass_hbm_floor_ms"] = round(floor_ms, 3)
    if "gpp_trial_kernel" in res["kernels_us_per_launch"]:
        res["trial_pass_ms"] = res["kernels_us_per_launch"]["gpp_trial_kernel"] / 1e3
        res["trial_pass_share_of_floor"] = round(floor_ms / res["trial_pass_ms"], 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ab_greedy_init.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
