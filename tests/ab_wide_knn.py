#!/usr/bin/env python
"""Timing of knn_cuda on the tensor-core route against the forced-exact search, run on an H100.  Checker script,
not collected by pytest.

    python tests/ab_wide_knn.py [--n 1000000] [--k 1000] [--nn 10] [--dims 512,576,768,1024] [--out results/x.json]

For each D: N rows in K Gaussian blobs (unit-normal centres, per-feature spread --sigma; with the default 0.1 the
cluster skip test prunes most clusters, as it does on clustered embeddings -- with wide blobs every query visits
every cluster and the exact search at this N runs for many minutes per call), centroids and assignments from one kmeans_cuda run, then
knn_cuda(nn)
on the tensor-core route (KMCUDA_B200_FORCE_EXACT=0) and the exact search (=1), alternated over --rounds rounds after
one warm-up call of each.  Call times are host-clocked (knn_cuda returns after the neighbours are on the host).  The
MODE 2 kernel time (both passes) comes from a torch.profiler trace of one more tensor-core call per round, taken
separately.  The `knn tensor-core path:` timing line gives the rows served, candidate pairs and fallback reasons.
The two routes' neighbour sets are compared; rows that differ are checked in fp64 and counted as near-ties when their
sorted neighbour distances agree to 1e-6.  Prints the card's name, power limit and max SM clock first, then one JSON
line per D.
"""
import argparse
import contextlib
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


@contextlib.contextmanager
def stderr_to(path):
    """the library prints its timing lines from C++ on fd 2"""
    sys.stderr.flush()
    saved = os.dup(2)
    with open(path, "w") as f:
        os.dup2(f.fileno(), 2)
    try:
        yield
    finally:
        sys.stderr.flush()
        os.dup2(saved, 2)
        os.close(saved)


def knn_call(km, nn, X, C, A, exact, log):
    os.environ["KMCUDA_B200_FORCE_EXACT"] = "1" if exact else "0"
    os.environ["KMCUDA_B200_TIMING"] = "1"
    with stderr_to(log):
        t0 = time.perf_counter()
        nb = km.knn_cuda(nn, X, C, A, device=1)
        dt = time.perf_counter() - t0
    os.environ.pop("KMCUDA_B200_TIMING")
    os.environ["KMCUDA_B200_FORCE_EXACT"] = "0"
    line = [ln for ln in open(log) if "knn tensor-core path" in ln]
    return nb, dt, (line[0].strip() if line else None)


def parse_line(line):
    if line is None:
        return {"served": 0}
    nums = lambda key: int(re.search(key + r" (\d+)", line).group(1))
    return {"served": int(line.split("path:")[1].split("rows")[0]), "pairs": int(line.split("rows,")[1].split("candidate")[0]),
            "to_exact": int(line.split("pairs,")[1].split("rows")[0]), "error_word": line.split("error word")[1].split(";")[0].strip(),
            "nan_inf": nums("nan/inf"), "list_full": nums("list full"), "no_threshold": nums("no threshold"),
            "gt64_cand": int(re.search(r">64 cand (\d+)", line).group(1)), "lt_k_cand": int(re.search(r"<k cand (\d+)", line).group(1))}


def mode2_kernel_ms(km, nn, X, C, A, log):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        knn_call(km, nn, X, C, A, False, log)
    ev = [e for e in prof.events() if "tc_assign_kernel<" in e.name and ", 2>" in e.name]
    return sum(e.device_time for e in ev) / 1e3, sorted({e.name.split("(")[0] for e in ev})


def near_tie_check(X, nb_a, nb_b):
    """rows whose neighbour sets differ: (count, count not explained by fp64 near-ties)"""
    import numpy as np
    import torch
    diff = np.flatnonzero((np.sort(nb_a, 1) != np.sort(nb_b, 1)).any(1))
    if len(diff) == 0:
        return 0, 0
    Xt = torch.from_numpy(X).cuda()
    xa = Xt[torch.from_numpy(diff).cuda()].double()
    da = ((Xt[torch.from_numpy(nb_a[diff].astype(np.int64)).cuda()].double() - xa[:, None]) ** 2).sum(-1).sort(1)[0]
    db = ((Xt[torch.from_numpy(nb_b[diff].astype(np.int64)).cuda()].double() - xa[:, None]) ** 2).sum(-1).sort(1)[0]
    bad = int((~torch.isclose(da, db, rtol=1e-6, atol=1e-12)).any(1).sum().item())
    return int(len(diff)), bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--sigma", type=float, default=0.1)
    ap.add_argument("--nn", type=int, default=10)
    ap.add_argument("--dims", default="512,576,768,1024")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import kmcuda_b200 as km
    results = [{"card": card(), "torch": torch.__version__}]
    print(json.dumps(results[0]), flush=True)
    log = os.path.join(tempfile.mkdtemp(), "knn_timing.log")
    for D in [int(d) for d in a.dims.split(",")]:
        rng = np.random.default_rng(D)
        g = torch.Generator(device="cuda").manual_seed(D)
        centers = torch.randn((a.k, D), generator=g, device="cuda")
        lab = torch.randint(0, a.k, (a.n,), generator=g, device="cuda")
        X = (centers[lab] + a.sigma * torch.randn((a.n, D), generator=g, device="cuda")).cpu().numpy()
        # k-means from the blob centres: one cluster per blob (from random rows, blobs without a seed merge into wide
        # clusters that the skip test cannot prune)
        C0 = centers.cpu().numpy()
        del centers, lab
        t0 = time.perf_counter()
        C, A = km.kmeans_cuda(X, a.k, init=C0, tolerance=0.01, yinyang_t=0.0, device=1)
        t_km = time.perf_counter() - t0
        print("# D=%d: data and kmeans_cuda in %.1f s" % (D, t_km), flush=True)
        out = {}
        for exact in (False, True):                                   # warm-up of both routes, and their answers
            out[exact] = knn_call(km, a.nn, X, C, A, exact, log)
            print("# D=%d: warm-up %s call %.2f s" % (D, "exact" if exact else "tc", out[exact][1]), flush=True)
        times = {False: [], True: []}
        kms, info = [], None
        for _ in range(a.rounds):
            for exact in (False, True):
                nb, dt, line = knn_call(km, a.nn, X, C, A, exact, log)
                print("# D=%d: %s call %.2f s" % (D, "exact" if exact else "tc", dt), flush=True)
                times[exact].append(dt)
                if not exact:
                    info = parse_line(line)
                assert np.array_equal(nb, out[exact][0]), "a route's answer changed between calls"
            ms, names = mode2_kernel_ms(km, a.nn, X, C, A, log)
            kms.append(ms)
        ndiff, nbad = near_tie_check(X, out[False][0], out[True][0])
        r = {"D": D, "n": a.n, "K": a.k, "k": a.nn, "kmeans_s": t_km,
             "tc_call_s": float(np.median(times[False])), "tc_call_spread_s": float(np.ptp(times[False])),
             "exact_call_s": float(np.median(times[True])), "exact_call_spread_s": float(np.ptp(times[True])),
             "tc_rounds_s": times[False], "exact_rounds_s": times[True],
             "mode2_kernel_ms": float(np.median(kms)), "mode2_kernel_spread_ms": float(np.ptp(kms)), "mode2_kernels": names,
             "timing_line": info, "rows_with_different_sets": ndiff, "differences_not_near_ties": nbad}
        results.append(r)
        print(json.dumps(r), flush=True)
        del X, out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
