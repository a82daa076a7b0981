"""Output digests of every path that uses csrc/fixed_order.cuh, for comparing two builds of the library bit for bit.

    python tests/ab_fixed_order.py --parent-lib variants/parent/libKMCUDA.so [--out digests.json]

Fixed-seed calls through k-means++ (weighted and not), k-means||, greedy k-means++ (L = 1, the default and 32 at
D = 64, 67 and 768), mini-batch k-means, empty-cluster relocation on data whose initial centroids win no rows, and
n_init=3 with inertia=True, at D % 4 == 0 and D % 4 != 0, L2 and angular.  Each call runs once per library in a child
process (the library selected through KMCUDA_B200_LIB) at verbosity 2; the child prints one SHA-256 digest per call of
the returned arrays and numbers and of the log, without its "arguments:" line (it prints pointers).  Prints one JSON
line: the card, the power limit, the digests of both libraries and the calls whose digests differ; exits 1 if any
does.  Run on an H100.  Checker script, not collected by pytest."""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def blobs(n, d, k, seed=0, cos=False):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((k, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, k, n)] + 0.6 * rng.standard_normal((n, d))).astype(np.float32)
    if cos:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def with_empties(X, k, n_far, cos=False):
    """k rows of X, the last n_far of them moved away from every sample (they win no row in the first pass)"""
    C = X[np.random.default_rng(1).choice(len(X), k, replace=False)].copy()
    C[k - n_far:] = -C[:n_far] if cos else C[:n_far] + 1e3
    return C


def cases():
    """(name, samples, clusters, keyword arguments of kmeans_cuda)"""
    out = []
    w = lambda n: np.random.default_rng(5).uniform(0.1, 2.0, n).astype(np.float32)   # noqa: E731
    for d in (64, 67):
        X = blobs(200_000, d, 64)
        base = dict(tolerance=0.01, yinyang_t=0, seed=7, average_distance=True)
        out.append(("k-means++ D=%d" % d, X, 64, dict(base, init="k-means++")))
        out.append(("k-means++ weighted D=%d" % d, X, 64, dict(base, init="k-means++", sample_weight=w(len(X)))))
        out.append(("k-means|| D=%d" % d, X, 64, dict(base, init=("k-means||", 5))))
        out.append(("k-means|| weighted D=%d" % d, X, 64, dict(base, init=("k-means||", 5), sample_weight=w(len(X)))))
    for d in (64, 67, 768):
        X = blobs(50_000, d, 32, seed=2)
        for L in (1, 0, 32):
            out.append(("greedy L=%d D=%d" % (L, d), X, 32,
                        dict(init=("greedy-k-means++", L), tolerance=1.0, yinyang_t=0, seed=11, average_distance=True)))
    Xc = blobs(50_000, 67, 32, seed=2, cos=True)
    out.append(("greedy cos L=0 D=67", Xc, 32, dict(init=("greedy-k-means++", 0), tolerance=1.0, yinyang_t=0,
                                                     seed=11, metric="cos", average_distance=True)))
    for d in (64, 67):
        X = blobs(300_000, d, 128, seed=4)
        out.append(("mini-batch D=%d" % d, X, 128, dict(init="k-means++", batch_size=8192, max_steps=60, seed=13,
                                                        average_distance=True)))
        out.append(("mini-batch weighted D=%d" % d, X, 128,
                    dict(init="k-means++", batch_size=8192, max_steps=60, seed=13, sample_weight=w(len(X)))))
    for d, cos in ((64, False), (67, False), (64, True), (67, True)):
        X = blobs(100_000, d, 60, seed=6, cos=cos)
        out.append(("relocate %s D=%d" % ("cos" if cos else "L2", d), X, 60,
                    dict(init=with_empties(X, 60, 12, cos), tolerance=0.0, yinyang_t=0, seed=3,
                         relocate_empty_clusters=True, metric="cos" if cos else "L2")))
    for d, cos in ((64, False), (67, False), (67, True)):
        X = blobs(100_000, d, 48, seed=8, cos=cos)
        out.append(("n_init=3 %s D=%d" % ("cos" if cos else "L2", d), X, 48,
                    dict(init="k-means++", tolerance=0.01, yinyang_t=0, seed=17, n_init=3, inertia=True,
                         average_distance=True, metric="cos" if cos else "L2")))
    return out


def digest(obj):
    h = hashlib.sha256()
    for v in obj if isinstance(obj, tuple) else (obj,):
        h.update(np.ascontiguousarray(v).tobytes() if isinstance(v, np.ndarray) else repr(v).encode())
    return h.hexdigest()


def child():
    sys.path.insert(0, ROOT)
    import kmcuda_b200 as km
    libc = ctypes.CDLL(None)
    res = {}
    for name, X, k, kw in cases():
        with tempfile.TemporaryFile() as log:
            sys.stdout.flush()
            libc.fflush(None)
            saved = os.dup(1)
            os.dup2(log.fileno(), 1)
            try:
                out = km.kmeans_cuda(X, k, device=1, verbosity=2, **kw)
            finally:
                libc.fflush(None)
                os.dup2(saved, 1)
                os.close(saved)
            log.seek(0)
            lines = [ln for ln in log.read().decode().splitlines() if not ln.startswith("arguments:")]
        res[name] = {"out": digest(out), "log": hashlib.sha256("\n".join(lines).encode()).hexdigest(),
                     "log_lines": len(lines)}
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        return child()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    libs = {"parent": os.path.abspath(a.parent_lib), "new": os.path.join(ROOT, "kmcuda_b200", "libKMCUDA.so")}
    got = {}
    for tag, lib in libs.items():
        env = dict(os.environ, KMCUDA_B200_LIB=lib)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--parent-lib", a.parent_lib, "--child"],
                           env=env, capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit("%s library: child failed\n%s" % (tag, r.stderr[-4000:]))
        got[tag] = json.loads(r.stdout.strip().splitlines()[-1])
    differ = sorted(n for n in got["parent"] if got["parent"][n] != got["new"].get(n))
    res = {"card": card, "calls": len(got["parent"]), "differ": differ, "digests": got}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
