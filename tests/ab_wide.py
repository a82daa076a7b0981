#!/usr/bin/env python
"""Timing of the assignment pass at 512 < D <= 1024 (64-row tensor-core tiles) against the forced-exact pass, run on
an H100.  Checker script, not collected by pytest.

    python tests/ab_wide.py [--n 2000000] [--k 1024] [--out results/ab_wide.json]

For N x D @ K on U[0, 1) samples (the reference's benchmark distribution), D in {512, 576, 768, 1024}: one Shard per
route (KMCUDA_B200_FORCE_EXACT is read when a shard is created), both passes' assignments compared, then CUDA-event
timing of whole passes (`Shard.assign`: preparation, filter, re-check, exact rows, bookkeeping) -- a warm-up, then
three rounds that alternate the routes, 20 passes each; medians and spreads over the rounds.  Then whole Lloyd
(`yinyang_t=0`) and default (Yinyang, adaptive) calls at N x 768 @ K from the same initial centroids, host-timed.
Prints one JSON line per measurement and the card's name and power limit first.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%r)" % e


def make_shard(n, D, K, exact):
    from kmcuda_b200.shard import Shard
    os.environ["KMCUDA_B200_FORCE_EXACT"] = "1" if exact else "0"
    try:
        return Shard(n, D, K)
    finally:
        os.environ.pop("KMCUDA_B200_FORCE_EXACT", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000000)
    ap.add_argument("--k", type=int, default=1024)
    ap.add_argument("--dims", default="512,576,768,1024")
    ap.add_argument("--passes", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import kmcuda_b200
    results = [{"card": card(), "torch": torch.__version__}]
    print(json.dumps(results[0]), flush=True)
    n, K = a.n, a.k
    for D in [int(d) for d in a.dims.split(",")]:
        g = torch.Generator(device="cuda").manual_seed(D)
        X = torch.rand((n, D), generator=g, device="cuda", dtype=torch.float32)
        C = X[torch.randperm(n, generator=g, device="cuda")[:K]].contiguous()
        shards = {"tc": make_shard(n, D, K, False), "exact": make_shard(n, D, K, True)}
        ch = torch.zeros(1, dtype=torch.int32, device="cuda")
        out, info = {}, {}
        for name, sh in shards.items():
            asg = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            prev = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            sh.assign(X, C, asg, prev, ch)          # first pass from -1: every row decided (also the warm-up)
            torch.cuda.synchronize()
            out[name] = (asg, prev)
            info[name] = sh.last_pass_info()
            assert sh.last_error() == 0
        mism = int((out["tc"][0] != out["exact"][0]).sum().item())
        times = {"tc": [], "exact": []}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for name in ("tc", "exact"):
                asg, prev = out[name]
                e0.record()
                for _ in range(a.passes):
                    shards[name].assign(X, C, asg, prev, ch)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / a.passes)
        kt = shards["tc"].kernel_times(a.passes)
        med = {k: float(np.median(v)) for k, v in times.items()}
        r = {"what": "pass", "n": n, "D": D, "K": K, "tc_ms": med["tc"], "exact_ms": med["exact"],
             "tc_spread_ms": float(np.ptp(times["tc"])), "exact_spread_ms": float(np.ptp(times["exact"])),
             "tc_rounds_ms": times["tc"], "exact_rounds_ms": times["exact"], "speedup": med["exact"] / med["tc"],
             "tc_kernel_ms": float(np.median(kt)), "tc_kernel_tflops": 2.0 * n * K * D / (np.median(kt) * 1e-3) / 1e12,
             "tc_route": bool(info["tc"][0]), "exact_route": bool(info["exact"][0]),
             "rows_rechecked_exactly": int(info["tc"][1]), "rows_full_exact_fallback": int(info["tc"][2]),
             "assignment_mismatches": mism, "pipeline_error": hex(shards["tc"].last_error())}
        results.append(r)
        print(json.dumps(r), flush=True)
        for sh in shards.values():
            sh.close()
        del X, C, out, shards
        torch.cuda.empty_cache()
    # whole runs at N x 768 @ K, the same initial centroids; host clock around calls that return after the device is done
    rng = np.random.default_rng(768)
    Xh = rng.random((n, 768), dtype=np.float32)
    C0 = Xh[rng.choice(n, K, replace=False)].copy()
    kmcuda_b200.kmeans_cuda(Xh[:100000], K, init=C0, tolerance=0.5, yinyang_t=0.0, device=1)   # warm-up (modules, pool)
    runs = {}
    for label, yy in (("lloyd", 0.0), ("default_yinyang", 0.1)):
        t0 = time.perf_counter()
        Cr, Ar = kmcuda_b200.kmeans_cuda(Xh, K, init=C0, yinyang_t=yy, device=1)
        runs[label] = (time.perf_counter() - t0, Ar)
    r = {"what": "runs", "n": n, "D": 768, "K": K, "lloyd_s": runs["lloyd"][0],
         "default_yinyang_s": runs["default_yinyang"][0],
         "assignments_equal": bool(np.array_equal(runs["lloyd"][1], runs["default_yinyang"][1]))}
    results.append(r)
    print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
