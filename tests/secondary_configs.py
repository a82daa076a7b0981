#!/usr/bin/env python
"""Secondary configurations of BASELINE.json (C1, C2, C3, C5) on one H100: this library next to the
unmodified reference (oracle/_ref/libKMCUDA.so), same inputs, same C-ABI call, wall clock around the call.

    python tests/secondary_configs.py [c1 c2 c3 c5 ...] [--out gpurun_out/secondary.json]

Measurement / checker script (lives under tests/ because it loads oracle/_ref); not collected by pytest.
Where the reference would take minutes it runs on a stated sub-sample and the rate is compared.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

IMPORT, RANDOM, PLUSPLUS = 3, 0, 1


def kmeans(lib, X, K, init, tol, yy, metric=0, seed=777, C0=None, verbosity=0, fp16x2=0):
    N, D = X.shape
    Dcall = D // 2 if fp16x2 else D
    esz = 2 if fp16x2 else 4
    C = np.zeros((K, D), X.dtype) if C0 is None else np.array(C0, copy=True, order="C")
    assert C.itemsize == esz and X.itemsize == esz
    A = np.zeros(N, np.uint32)
    m = ctypes.c_uint32(0)
    t = time.perf_counter()
    rc = lib.kmeans_cuda(init, ctypes.byref(m), tol, yy, metric, N, Dcall, K, seed, 1, -1, fp16x2, verbosity,
                         X.ctypes.data, C.ctypes.data, A.ctypes.data, None)
    dt = time.perf_counter() - t
    assert rc == 0, rc
    return dt, C, A


def knn(lib, k, X, C, A, metric=0):
    N, D = X.shape
    out = np.zeros((N, k), np.uint32)
    t = time.perf_counter()
    rc = lib.knn_cuda(k, metric, N, D, C.shape[0], 1, -1, 0, 0, X.ctypes.data, C.ctypes.data, A.ctypes.data,
                      out.ctypes.data)
    dt = time.perf_counter() - t
    assert rc == 0, rc
    return dt, out


def c1(ours, ref, res):
    """C1: Lloyd L2 fp32 100000x256 @ 1024 (the reference README benchmark shape, README.md:187-207)"""
    rng = np.random.default_rng(777)
    X = rng.random((100000, 256), dtype=np.float32)
    C0 = X[rng.choice(len(X), 1024, replace=False)].copy()
    out = {}
    for name, lib in (("ours", ours), ("reference", ref)):
        kmeans(lib, X[:20000], 1024, IMPORT, 1.0, 0.0, C0=C0)  # warm
        dt1, _, a1 = kmeans(lib, X, 1024, IMPORT, 1.0, 0.0, C0=C0)
        dtf, cf, af = kmeans(lib, X, 1024, IMPORT, 0.002, 0.0, C0=C0)
        out[name] = {"single_assign_s": dt1, "lloyd_tol0.002_s": dtf}
        out[name + "_a1"], out[name + "_af"], out[name + "_cf"] = a1, af, cf
    out["single_assign_equal"] = bool(np.array_equal(out["ours_a1"], out["reference_a1"]))
    out["final_assign_equal_frac"] = float((out["ours_af"] == out["reference_af"]).mean())
    out["final_centroid_max_rel"] = float(np.nanmax(np.abs(out["ours_cf"] - out["reference_cf"]) /
                                                    (np.abs(out["reference_cf"]) + 1e-12)))
    for k in [k for k in out if k.endswith(("_a1", "_af", "_cf"))]:
        del out[k]
    try:
        from sklearn.cluster import KMeans
        t = time.perf_counter()
        KMeans(n_clusters=1024, init="random", max_iter=15, random_state=0, n_init=1).fit(X)
        out["sklearn_15iter_s"] = time.perf_counter() - t
        out["host_cores"] = os.cpu_count()
    except Exception as e:  # pragma: no cover
        out["sklearn_15iter_s"] = repr(e)[:80]
    res["c1"] = out


def c2(ours, ref, res, n_full=8000000, n_ref=500000):
    """C2: Yinyang L2 fp32 8M x 256 @ 1024, tolerance 0.01, yinyang_t 0.1 (whole run, host buffers)"""
    rng = np.random.default_rng(777)
    X = rng.random((n_full, 256), dtype=np.float32)
    C0 = X[rng.choice(n_ref, 1024, replace=False)].copy()
    out = {}
    kmeans(ours, X[:20000], 1024, IMPORT, 1.0, 0.0, C0=C0)
    for yy in (0.0, 0.1):
        dt, c, a = kmeans(ours, X, 1024, IMPORT, 0.01, yy, C0=C0)
        out["ours_full_yy%.1f_s" % yy] = dt
    # the reference on a sub-sample (it needs minutes at 8M), ours on the same sub-sample
    Xs = X[:n_ref]
    for yy in (0.0, 0.1):
        dto, co, ao = kmeans(ours, Xs, 1024, IMPORT, 0.01, yy, C0=C0)
        dtr, cr, ar = kmeans(ref, Xs, 1024, IMPORT, 0.01, yy, C0=C0)
        out["sub%d_yy%.1f" % (n_ref, yy)] = {"ours_s": dto, "reference_s": dtr,
                                             "assign_equal_frac": float((ao == ar).mean()),
                                             "centroid_max_rel": float(np.nanmax(np.abs(co - cr) / (np.abs(cr) + 1e-12)))}
    res["c2"] = out


def c2c(ours, ref, res, n_full=8000000):
    """C2 on CLUSTERED data (SURVEY.md 8d's optional mixture: 1024 Gaussians, sigma 0.05, centres U[0,1)^256): the
    regime Yinyang is meant for.  Whole runs, host buffers; Lloyd vs Yinyang with this library."""
    rng = np.random.default_rng(778)
    centers = rng.random((1024, 256), dtype=np.float32)
    X = np.empty((n_full, 256), np.float32)
    step = 500000
    for i in range(0, n_full, step):
        m = min(step, n_full - i)
        X[i:i + m] = centers[rng.integers(0, 1024, m)] + 0.05 * rng.standard_normal((m, 256), dtype=np.float32)
    C0 = X[rng.choice(n_full, 1024, replace=False)].copy()
    out = {}
    kmeans(ours, X[:20000], 1024, IMPORT, 1.0, 0.0, C0=C0)
    for yy in (0.0, 0.1):
        dt, c, a = kmeans(ours, X, 1024, IMPORT, 0.01, yy, C0=C0)
        out["ours_full_yy%.1f_s" % yy] = dt
        out["clusters_used_yy%.1f" % yy] = int(len(np.unique(a)))
    res["c2_clustered"] = out


def _c3_data(n_full, n_ref, D, K, rng):
    X = np.empty((n_full, D), np.float16)
    step = 500000
    for i in range(0, n_full, step):
        blk = rng.standard_normal((min(step, n_full - i), D), dtype=np.float32)
        blk /= np.linalg.norm(blk, axis=1, keepdims=True)
        X[i:i + len(blk)] = blk.astype(np.float16)
    C0 = X[rng.choice(n_ref, K, replace=False)].astype(np.float32)
    C0 += 0.02 * rng.standard_normal(C0.shape).astype(np.float32)
    C0 = (C0 / np.linalg.norm(C0, axis=1, keepdims=True)).astype(np.float16)
    return X, C0


def c3_child(n_full, tol):
    """the C3 run itself (own process: the C library's stdout / stderr are parsed by the parent)"""
    import kmcuda_b200
    ours = O.load_c_api(kmcuda_b200.LIB_PATH)
    D, K = 480, 40000
    X, C0 = _c3_data(n_full, 100000, D, K, np.random.default_rng(777))
    t = time.perf_counter()
    dt, C, A = kmeans(ours, X, K, IMPORT, tol, 0.1, metric=1, C0=C0, fp16x2=1, verbosity=2)
    print("C3_WALL %.3f" % dt, flush=True)
    print("C3_USED_CLUSTERS %d" % len(np.unique(A)), flush=True)


def c3(ours, ref, res, n_full=2000000, n_ref=100000, tol=0.0005):
    """C3 sized for one 80 GB H100: Yinyang, angular, fp16 samples, 2M x 480 @ 40000, yinyang_t = 0.1 (G = 4000, 32 GB
    of bounds; the 4M rows of the original configuration would need 64 GB of bounds next to the samples, the
    centroids and the pass's work buffers).  The reference needs days to converge here (README.md:60-62); the run stops at `tol` reassignments so
    that a few Yinyang iterations (after the Lloyd draft phase and one bounds refresh) are timed."""
    import subprocess
    D, K = 480, 40000
    out = {}
    env = dict(os.environ, KMCUDA_B200_TIMING="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--c3-child", str(n_full), str(tol)], env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    log = r.stdout.splitlines()
    out["returncode"] = r.returncode
    out["iterations"] = [ln for ln in log if ln.startswith("iteration") or "refreshing" in ln or "Lloyd" in ln][:80]
    out["memory"] = [ln for ln in log if ln.startswith("GPU #")][:4]
    out["wall"] = [ln for ln in log if ln.startswith("C3_")]
    out["timing_table"] = [ln.replace("[kmcuda_b200 timing]", "").rstrip() for ln in r.stderr.splitlines()
                           if "[kmcuda_b200 timing]" in ln][-40:]
    if r.returncode != 0:
        out["stderr_tail"] = r.stderr[-1500:]
    out["hbm_floor_note"] = ("per Yinyang iteration the bounds stream is 2 * (G + 1) * 4 B per sample = %.1f GB; at the "
                             "H100 SXM data sheet's 3.35 TB/s that is %.1f ms" % (2 * 4001 * 4 * n_full / 1e9,
                                                                                 2 * 4001 * 4 * n_full / 3.35e12 * 1e3))
    # agreement with the reference on a sub-sample, one assignment step (the reference accumulates fp16 data in fp16,
    # this library works on the exactly widened values: statistical agreement, SURVEY.md a2)
    X, C0 = _c3_data(n_ref, n_ref, D, K, np.random.default_rng(777))
    dto, _, ao = kmeans(ours, X, K, IMPORT, 1.0, 0.0, metric=1, C0=C0, fp16x2=1)
    dtr, _, ar = kmeans(ref, X, K, IMPORT, 1.0, 0.0, metric=1, C0=C0, fp16x2=1)
    out["sub%d_single_assign" % n_ref] = {"ours_s": dto, "reference_s": dtr, "assign_equal_frac": float((ao == ar).mean())}
    res["c3"] = out


def c5(ours, ref, res, n_full=3000000, n_ref=200000):
    """C5: knn_cuda k=10, 3M x 256, 1000 precomputed clusters"""
    K, k = 1000, 10
    rng = np.random.default_rng(777)
    out = {}
    centers = rng.random((K, 256), dtype=np.float32)
    lab = rng.integers(0, K, n_full)
    X = centers[lab] + 0.05 * rng.standard_normal((n_full, 256), dtype=np.float32)
    for n, libs in ((n_ref, (("ours", ours), ("reference", ref))), (n_full, (("ours", ours),))):
        Xs = np.ascontiguousarray(X[:n])
        _, C, A = kmeans(ours, Xs, K, IMPORT, 0.01, 0.0, C0=centers)
        r = {}
        for name, lib in libs:
            dt, nb = knn(lib, k, Xs, C, A)
            r[name + "_s"] = dt
            r[name + "_queries_per_s"] = n / dt
            r[name + "_nb"] = nb
        if "reference_nb" in r:
            same = (r["ours_nb"] == r["reference_nb"]).all(1)
            r["rows_equal_frac"] = float(same.mean())
            # rows that differ: are the two answers the same multiset of exact (reference-arithmetic) distances?
            L = O.lib()
            fp = ctypes.POINTER(ctypes.c_float)
            ties = 0
            for q in np.nonzero(~same)[0][:200]:
                d = [sorted(L.ko_distance(0, Xs[q].ctypes.data_as(fp), Xs[int(j)].ctypes.data_as(fp), Xs.shape[1])
                            for j in r[name + "_nb"][q]) for name in ("ours", "reference")]
                ties += d[0] == d[1]
            r["differing_rows"] = int((~same).sum())
            r["differing_rows_checked_equal_distance_multisets"] = int(ties)
        for kk in [kk for kk in r if kk.endswith("_nb")]:
            del r[kk]
        out["n%d" % n] = r
    res["c5"] = out


def main():
    if len(sys.argv) >= 4 and sys.argv[1] == "--c3-child":
        c3_child(int(sys.argv[2]), float(sys.argv[3]))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="*", default=["c1", "c2", "c3", "c5"])
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "secondary.json"))
    args = ap.parse_args()
    import kmcuda_b200
    ours = O.load_c_api(kmcuda_b200.LIB_PATH)
    ref = O.reference_lib()
    res = {}
    if os.path.exists(args.out):
        try:
            res = json.load(open(args.out))
        except Exception:
            res = {}
    for w in args.which:
        t = time.perf_counter()
        {"c1": c1, "c2": c2, "c2c": c2c, "c3": c3, "c5": c5}[w](ours, ref, res)
        key = "c2_clustered" if w == "c2c" else w
        res[key]["script_wall_s"] = time.perf_counter() - t
        print(w, json.dumps(res[key]), flush=True)
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
