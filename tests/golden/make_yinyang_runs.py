"""Generates tests/golden/yinyang_runs.npz: whole Yinyang runs of the C oracle (`ko_kmeans`) -- log lines, assignments
and centroids -- recorded before the oracle's Yinyang iteration was split into `ko_yy_init` / `ko_yy_drifts` /
`ko_yy_step`.  `tests/test_yinyang_step_cpu.py::test_split_oracle_reproduces_recorded_runs` holds the split oracle to
them.

    python tests/golden/make_yinyang_runs.py

Inputs are regenerated from seeds by `yinyang_runs()` (no NaN rows, no empty clusters: the recorded oracle read out of
range on those, the split one restates the library's guard instead).
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402

OUT = os.path.join(HERE, "yinyang_runs.npz")

# name: (n, D, K, yinyang_t, metric, tolerance, max_iter, seed)
RUNS = {
    "l2_g4": (3000, 16, 40, 0.1, 0, 1e-3, 0, 1),
    "l2_g16": (4000, 33, 64, 0.25, 0, 1e-4, 0, 2),
    "l2_g1_maxiter": (2500, 8, 30, 0.04, 0, 0.0, 25, 3),
    "cos_g5": (3000, 24, 50, 0.1, 1, 1e-3, 0, 4),
}


def yinyang_run_inputs(name):
    n, D, K, yy, metric, tol, max_iter, seed = RUNS[name]
    rng = np.random.default_rng(seed)
    X = rng.random((n, D), dtype=np.float32)
    if metric == 1:
        X = X - np.float32(0.5)
        X = (X / np.linalg.norm(X.astype(np.float64), axis=1, keepdims=True)).astype(np.float32)
    C0 = X[rng.choice(n, K, replace=False)].copy()
    return np.ascontiguousarray(X), C0, dict(tolerance=tol, yinyang_t=yy, metric=metric, max_iter=max_iter)


def logged_run(name):
    """(C, assign, log lines) of one oracle run; the C stdout is read through a temporary file"""
    X, C0, kw = yinyang_run_inputs(name)
    import ctypes
    libc = ctypes.CDLL(None)
    with tempfile.TemporaryFile(mode="w+") as f:
        libc.fflush(None)
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(f.fileno(), 1)
        try:
            C, a, lines = O.kmeans(X, C0, log=True, **kw)
            libc.fflush(None)
        finally:
            os.dup2(saved, 1)
            os.close(saved)
        f.seek(0)
        log = [ln for ln in f.read().splitlines() if ln.startswith("iteration")]
    assert len(log) == lines, (len(log), lines)
    return C, a, log


def main():
    out = {}
    for name in RUNS:
        C, a, log = logged_run(name)
        out[name + "/C"] = C
        out[name + "/assign"] = a
        out[name + "/log"] = np.array(log)
        print(name, len(log), "lines")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
