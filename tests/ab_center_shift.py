"""Cost of scikit-learn's stopping rule (kmeans_cuda(..., tol=); DESIGN.md §4p) against the reference rule.

    python tests/ab_center_shift.py [--rounds 3]

For each shape, a blob mixture on the device (device-pointer input, so no host copy is timed) is clustered from the
same imported centroids by three calls, alternated over the rounds after one warm-up round, each timed with a device
synchronisation on both sides:
    ref    tolerance = 0 (the reference rule)
    rule0  tol = 0, max_iter = 10000: the same passes and updates, plus the centroid copy, the shift and its fold per
           update and the shift read back with each pass; no variance pass (tol == 0)
    rule   tol = 1e-12: rule0 plus the variance pass (two reads of X); the shift test stops it where rule0 stops
The three results are checked bit-equal.  (rule0 - ref) / n_iter is the per-iteration overhead, rule - rule0 the
variance pass.  Prints one line per shape and the card's name, power limit and max SM clock."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers still stand; the card line says why it is missing
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import kmcuda_b200 as km
    print("card:", _card(), flush=True)
    for n, d, k in ((8 << 20, 256, 1024), (2 << 20, 768, 1024)):
        g = torch.Generator(device="cuda").manual_seed(0)
        centers = torch.randn(k, d, device="cuda", generator=g) * 3
        X = centers[torch.randint(0, k, (n,), device="cuda", generator=g)] + \
            0.3 * torch.randn(n, d, device="cuda", generator=g)
        C0 = (centers + 0.05 * torch.randn(k, d, device="cuda", generator=g)).cpu().numpy()
        samples = (X.data_ptr(), 0, (n, d))
        arms = {"ref": dict(tolerance=0.0), "rule0": dict(tol=0, max_iter=10_000, n_iter=True),
                "rule": dict(tol=1e-12, max_iter=10_000, n_iter=True)}
        times = {name: [] for name in arms}
        outs = {}
        for r in range(a.rounds + 1):
            for name, kw in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = km.kmeans_cuda(samples, k, init=C0, yinyang_t=0, device=1, **kw)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                c = np.empty((k, d), np.float32)
                asg = np.empty(n, np.uint32)
                km._cuda_memcpy_d2h(0, c.ctypes.data, res[0], c.nbytes)
                km._cuda_memcpy_d2h(0, asg.ctypes.data, res[1], asg.nbytes)
                km._cuda_free(0, res[0])
                km._cuda_free(0, res[1])
                outs[name] = (c.view(np.uint32), asg, res[2] if len(res) > 2 else None)
                if r > 0:
                    times[name].append(dt)
            same = all(np.array_equal(outs[x][0], outs["ref"][0]) and np.array_equal(outs[x][1], outs["ref"][1])
                       for x in ("rule0", "rule"))
            assert same, "the three arms differ"
        it = outs["rule0"][2]
        assert outs["rule"][2] == it
        med = {x: float(np.median(v)) * 1e3 for x, v in times.items()}
        var_ms = med["rule"] - med["rule0"]
        floor_ms = 2 * n * d * 4 / 3.35e12 * 1e3
        print("%dx%d @ %d: n_iter %d, ref %.1f ms, rule0 %.1f ms, rule %.1f ms (medians of %d); per-iteration "
              "overhead %.3f ms, variance pass %.2f ms (2 reads of X at 3.35 TB/s: %.2f ms)"
              % (n, d, k, it, med["ref"], med["rule0"], med["rule"], a.rounds, (med["rule0"] - med["ref"]) / it,
                 var_ms, floor_ms), flush=True)
        del X, centers
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
