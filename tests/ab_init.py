"""A/B of the seeding (DESIGN.md §4g): init="k-means++" against init="k-means||" (5 rounds).

    python tests/ab_init.py [--rounds 3] [--points 8000000] [--lloyd-points 1000000]

Data, generated on the device and passed as device pointers: bench.py's uniform [0, 1) samples (8M x 256, K = 1024)
and a mixture of 1024 Gaussian blobs of the same shape.  Every arm runs in its own child process with
KMCUDA_B200_TIMING=1 and reports, per data set, the init phase time (the library's phases whose name starts with
"init"), the average distance after a tolerance=1.0 call (the seeding's quality: one assignment pass, no update), and
the iterations and final average distance of a tolerance=0.01 Lloyd run on the first `--lloyd-points` rows.  The arms
are alternated `--rounds` times; one more k-means|| child runs under torch.profiler and lists the device time per
kernel of its init on the uniform data and on a weighted, skewed variant (90 % of the rows one repeated row;
`--profile-only` runs just that child).  Prints one JSON line: card, power limit, per-arm medians and spreads (max - min).
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = {"k-means++": "k-means++", "k-means||": ("k-means||", 5)}
DATA = ("uniform", "blobs")


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


def call(km, X, k, init, tolerance, w=None):
    n, d = X.shape
    cp, ap, avg = km.kmeans_cuda((X.data_ptr(), 0, (n, d)), k, init=init, tolerance=tolerance, yinyang_t=0, seed=3,
                                 device=1, verbosity=1, average_distance=True,
                                 sample_weight=None if w is None else w.data_ptr())
    km._cuda_free(0, cp)
    km._cuda_free(0, ap)
    return avg


def child(arm, a):
    sys.path.insert(0, ROOT)
    import torch
    import kmcuda_b200 as km
    torch.cuda.set_device(0)
    for kind in DATA:
        X = make_data(kind, a.points, a.dim)
        torch.cuda.synchronize()
        print("@data %s" % kind, flush=True)
        sys.stderr.write("@data %s\n" % kind)
        sys.stderr.flush()
        avg = call(km, X, a.clusters, ARMS[arm], 1.0)
        sys.stderr.write("@seeded %r\n" % avg)
        sys.stderr.flush()
        print("@lloyd", flush=True)
        avg = call(km, X[:a.lloyd_points].contiguous(), a.clusters, ARMS[arm], 0.01)
        print("@final %r" % avg, flush=True)
        del X
        torch.cuda.empty_cache()


def profile_child(a):
    sys.path.insert(0, ROOT)
    import torch
    import kmcuda_b200 as km
    torch.cuda.set_device(0)
    from torch.profiler import ProfilerActivity, profile
    X = make_data("uniform", a.points, a.dim)
    # second case: weighted, 90 % of the rows one repeated row, so one candidate's weight total covers most rows
    w = torch.empty(a.points, device="cuda", dtype=torch.float32).log_normal_(0.0, 1.0)
    for tag in ("uniform", "skewed_weighted"):
        if tag == "skewed_weighted":
            X[:a.points * 9 // 10] = X[0]
        ww = w if tag == "skewed_weighted" else None
        call(km, X, a.clusters, ARMS["k-means||"], 1.0, ww)   # warm-up: module load, pooled allocations
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(km, X, a.clusters, ARMS["k-means||"], 1.0, ww)
            torch.cuda.synchronize()
        rows = {}
        for ev in prof.key_averages():
            t = getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0)
            if t > 0:
                rows[ev.key[:90]] = {"ms": t / 1000.0, "calls": ev.count}
        print("@profile %s %s" % (tag, json.dumps(rows)), flush=True)


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


def _spawn(args, a):
    env = dict(os.environ, KMCUDA_B200_TIMING="1")
    cmd = [sys.executable, os.path.abspath(__file__)] + args + [
        "--points", str(a.points), "--dim", str(a.dim), "--clusters", str(a.clusters),
        "--lloyd-points", str(a.lloyd_points)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("%s failed:\n%s" % (args, r.stderr[-3000:]))
    return r


def run_arm(arm, a):
    r = _spawn(["--child", arm], a)
    res = {}
    err = r.stderr.split("@data ")[1:]
    out = r.stdout.split("@data ")[1:]
    for e, o in zip(err, out):
        kind = e.split("\n", 1)[0]
        first = e.split("[kmcuda_b200 timing] kmeans_cuda")[1]   # the table of the tolerance=1.0 call
        first = first.split("@seeded")[0]
        phases = {m.group(1).strip(): float(m.group(2))
                  for m in re.finditer(r"\[kmcuda_b200 timing\]\s{3}(\S.*?)\s+([0-9.]+) ms", first)}
        lloyd = o.split("@lloyd", 1)[1]
        res[kind] = {
            "init_ms": sum(v for k, v in phases.items() if k.startswith("init")),
            "init_phases_ms": {k: v for k, v in phases.items() if k.startswith("init")},
            "seeded_avg": float(re.search(r"@seeded (\S+)", e).group(1)),
            "lloyd_iterations": sum(1 for ln in lloyd.splitlines() if ln.startswith("iteration")),
            "lloyd_final_avg": float(re.search(r"@final (\S+)", lloyd).group(1)),
            "candidates": [int(x) for x in re.findall(r"k-means\|\|: (\d+) candidates", o.split("@lloyd")[0])],
        }
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", default=None)
    ap.add_argument("--profile-child", action="store_true")
    ap.add_argument("--profile-only", action="store_true", help="only the per-kernel profile (one JSON line)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, default=8_000_000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--lloyd-points", type=int, default=1_000_000)
    a = ap.parse_args()
    if a.child:
        child(a.child, a)
        return
    if a.profile_child:
        profile_child(a)
        return
    if a.profile_only:
        print(json.dumps(dict(card=card(), **profile(a))))
        return
    import numpy as np
    runs = {arm: [] for arm in ARMS}
    for _ in range(a.rounds):
        for arm in ARMS:
            runs[arm].append(run_arm(arm, a))
    res = {"what": "seeding A/B: init time, seeded and final average distance", "card": card(),
           "shape": [a.points, a.dim, a.clusters], "lloyd_points": a.lloyd_points, "rounds": a.rounds}
    for arm in ARMS:
        res[arm] = {}
        for kind in DATA:
            rec = [r[kind] for r in runs[arm]]
            out = {}
            for key in ("init_ms", "seeded_avg", "lloyd_iterations", "lloyd_final_avg"):
                v = [x[key] for x in rec]
                out[key] = {"median": float(np.median(v)), "spread": float(max(v) - min(v)), "runs": v}
            out["init_phases_ms_last"] = rec[-1]["init_phases_ms"]
            out["candidates_last"] = rec[-1]["candidates"]
            res[arm][kind] = out
    for kind in DATA:
        res["init_speedup_" + kind] = res["k-means++"][kind]["init_ms"]["median"] / \
            res["k-means||"][kind]["init_ms"]["median"]
    res.update(profile(a))
    print(json.dumps(res))


def profile(a):
    """device time per kernel of one k-means|| init, uniform data and the skewed weighted case"""
    p = _spawn(["--profile-child"], a)
    return {"kmeans_parallel_kernels_" + m.group(1): json.loads(m.group(2))
            for m in re.finditer(r"@profile (\S+) (.*)", p.stdout)}


if __name__ == "__main__":
    main()
