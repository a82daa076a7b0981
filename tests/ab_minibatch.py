"""A/B of mini-batch k-means (DESIGN.md §4h) against the full Lloyd run, from the same init=import centroids.

    python tests/ab_minibatch.py [--rounds 3] [--points 8000000] [--profile-steps 20]

Data: bench.py's shape, 8M x 256 uniform [0, 1) samples generated on the device and passed as device pointers, K = 1024,
the init centroids 1024 random rows (seed 3).  Arms: full Lloyd (yinyang_t = 0, tolerance = 0.01) and mini-batch with
b = 2^16 and 2^18 (tolerance = 0, max_steps = 0: the run ends by the lack-of-improvement rule).  Each arm reports the
wall time of the call (host clock around a call that ends in a device synchronise) and the final average distance;
the arms are alternated `--rounds` times.  Two more mini-batch runs (b = 2^16, `--profile-steps` and twice as many
steps) under torch.profiler give the device time of every kernel per step (their difference divided by the extra
steps).  Last, the assignment of one batch alone, b = 2^16 and 2^18, the same drawn rows and the init centroids: the
row-list tensor-core pass (Shard.debug_assign_rows) against X[rows] gathered by torch followed by the contiguous
Shard.assign, CUDA events around 20 calls of each, alternated `--rounds` times.  Prints one JSON line: card, power
limit, per-arm medians and spreads (max - min), per-step kernel times, per-call ms of the two assignment routes.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, default=8_000_000)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--profile-only", action="store_true", help="skip the timed arms")
    a = ap.parse_args()
    import numpy as np
    import torch
    import kmcuda_b200 as km
    n, d, k = a.points, 256, 1024
    g = torch.Generator(device="cuda").manual_seed(777)
    X = torch.rand((n, d), generator=g, device="cuda", dtype=torch.float32)
    C0 = X[torch.from_numpy(np.random.default_rng(3).choice(n, k, replace=False)).cuda()].cpu().numpy()
    arms = {"lloyd": None, "mb_65536": 1 << 16, "mb_262144": 1 << 18}

    def call(b, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cp, ap_, avg = km.kmeans_cuda((X.data_ptr(), 0, (n, d)), k, init=C0, yinyang_t=0, seed=3, device=1,
                                      average_distance=True, tolerance=0.01 if b is None else 0.0,
                                      batch_size=b, **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        km._cuda_free(0, cp)
        km._cuda_free(0, ap_)
        return dt, avg

    call(1 << 16, max_steps=3)   # warm-up: module load, pools
    res = {name: {"s": [], "avg": []} for name in arms}
    for _ in range(0 if a.profile_only else a.rounds):
        for name, b in arms.items():
            dt, avg = call(b)
            res[name]["s"].append(dt)
            res[name]["avg"].append(avg)
    summary = {name: {"median_s": float(np.median(v["s"])), "spread_s": float(max(v["s"]) - min(v["s"])),
                      "avg_distance": float(np.median(v["avg"])),
                      "avg_spread": float(max(v["avg"]) - min(v["avg"]))} for name, v in res.items() if v["s"]}
    from torch.profiler import ProfilerActivity, profile

    def kernels(steps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(1 << 16, max_steps=steps)
        out = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                name = re.sub(r"\(anonymous namespace\)::", "", e.key)
                name = re.sub(r"<cub::.*", "", re.sub(r"\(.*", "", name))[:70]
                t, c = out.get(name, (0.0, 0))
                out[name] = (t + e.device_time_total / 1000.0, c + e.count)
        return out

    # two runs of different length: the difference per step leaves out the setup and the final full assignment pass
    short, long_ = kernels(a.profile_steps), kernels(2 * a.profile_steps)
    per_step = {k_: round((long_[k_][0] - short.get(k_, (0.0, 0))[0]) / a.profile_steps * 1000.0, 1)
                for k_ in long_}
    per_step = dict(sorted(((k_, v) for k_, v in per_step.items() if v > 0.05), key=lambda kv: -kv[1]))
    from kmcuda_b200.shard import Shard
    Ct = torch.from_numpy(C0).cuda()
    passes = {}
    for b in (1 << 16, 1 << 18):
        rows = torch.from_numpy(np.random.default_rng(5).integers(0, n, b).astype(np.int32)).cuda()
        fused, contig = Shard(b, d, k), Shard(b, d, k)
        out = torch.empty(b, dtype=torch.int32, device="cuda")
        scratch = torch.empty(n, dtype=torch.int32, device="cuda")
        asg = torch.full((b,), -1, dtype=torch.int32, device="cuda")
        prev = torch.empty(b, dtype=torch.int32, device="cuda")
        ch = torch.zeros(1, dtype=torch.int32, device="cuda")

        def run_fused():
            fused.debug_assign_rows(X, Ct, rows, out=out, scratch=scratch, sync=False)

        def run_gather():
            contig.assign(X[rows.long()], Ct, asg, prev, ch)

        times = {"row_list": [], "gather_then_contiguous": []}
        for _ in range(a.rounds):
            for name, fn in (("row_list", run_fused), ("gather_then_contiguous", run_gather)):
                fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(20):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / 20)
        assert fused.last_error() == 0 and contig.last_error() == 0
        assert torch.equal(out, asg), "the two routes disagree"
        passes[str(b)] = {k_: {"median_ms": round(float(np.median(v)), 4), "spread_ms": round(max(v) - min(v), 4)}
                          for k_, v in times.items()}
    print(json.dumps({"card": card(), "points": n, "summary": summary, "per_step_us_b65536": per_step,
                      "profile_steps": [a.profile_steps, 2 * a.profile_steps], "assign_one_batch": passes}))


if __name__ == "__main__":
    main()
