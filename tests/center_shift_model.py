"""NumPy model of scikit-learn's stopping rule for Lloyd runs (kmeans_cuda(..., tol=, max_iter=, n_iter=True);
include/kmcuda_b200.h kmcuda_b200_kmeans_center_shift, DESIGN.md §4p).

`tolerance_abs` is scikit-learn's _tolerance; `shift_total` is S_i with its non-finite rule; `run` is a whole run, the
centroids kept in fp32 between iterations as the library keeps them, the update and the relocation those of
relocate_model.  Labels come from the caller (the oracle's argmin for the GPU pin, a float64 argmin for the scikit-learn
comparisons), so the model holds no assignment rule.  tests/test_center_shift_cpu.py checks it against scikit-learn;
tests/test_center_shift_gpu.py pins the library to it."""
import numpy as np

from relocate_model import distances, normalize_cos, relocate

REASONS = ("equal labels", "tolerance", "max_iter")


def tolerance_abs(X, tol):
    """tol times the mean of the unweighted population variances of the features, in double; 0 when tol == 0"""
    if tol == 0:
        return 0.0
    return float(np.mean(np.var(np.asarray(X, np.float64), axis=0)) * tol)


def shift_total(C_old, C_new):
    """sum_c ||c_new - c_old||^2 in double; a centroid whose term is not finite adds 0"""
    with np.errstate(invalid="ignore", over="ignore"):
        d = ((np.asarray(C_new, np.float64) - np.asarray(C_old, np.float64)) ** 2).sum(1)
    return float(d[np.isfinite(d)].sum())


def _update(X, C, labels, w, metric, relocate_empty, state):
    """one centroid update (fp32 result), with relocation if asked for; state carries the angular recurrence"""
    n, D = X.shape
    K = len(C)
    wf = np.ones(n, np.float64) if w is None else np.asarray(w, np.float64)
    own = labels < K
    sums = np.zeros((K, D), np.float64)
    np.add.at(sums, labels[own], wf[own, None] * X[own])
    counts = np.bincount(labels[own], minlength=K)
    Wt = np.bincount(labels[own], weights=wf[own], minlength=K)
    Wf = counts.astype(np.float32) if w is None else Wt.astype(np.float32)
    sums = sums.astype(np.float32)
    records = []
    if relocate_empty:
        d = distances(X, C, labels, metric)
        sums, counts, Wf, records, _ = relocate(X, w, labels, d, sums, counts, Wf)
    with np.errstate(invalid="ignore", divide="ignore"):
        if metric == 1:
            raw = (C.astype(np.float64) * state["ccounts"][:, None] +
                   (sums.astype(np.float64) - state["prev_sums"])).astype(np.float32)
            Cn = (raw / np.sqrt((raw.astype(np.float64) ** 2).sum(1, keepdims=True))).astype(np.float32)
            for e, i, _, _ in records:
                Cn[e] = normalize_cos(X[i])
            state["prev_sums"] = sums
            state["ccounts"] = Wf
        else:
            Cn = (sums * (np.float32(1) / Wf)[:, None]).astype(np.float32)
    return Cn


def run(X, C0, labeler, tol, max_iter=300, metric=0, w=None, relocate_empty=False):
    """A whole run under the rule.  labeler(X, C) -> labels (K for a row without a centroid).  Returns a dict with the
    final C and labels, n_iter, reason, shifts [S_1, ...] and passes [reassignments of pass 1, ...]."""
    X = np.asarray(X, np.float32)
    C = np.array(C0, np.float32)
    K, D = C.shape
    t = tolerance_abs(X, tol)
    state = {"ccounts": np.zeros(K, np.float32), "prev_sums": np.zeros((K, D), np.float32)}
    prev = np.full(len(X), -1, np.int64)
    labels = np.asarray(labeler(X, C), np.int64)
    passes = [int((labels != prev).sum())]
    shifts = []
    i = 1
    while True:
        if i > 1 and passes[-1] == 0:
            reason = "equal labels"
            break
        Cold = C
        C = _update(X, C, labels, w, metric, relocate_empty, state)
        shifts.append(shift_total(Cold, C))
        prev, labels = labels, np.asarray(labeler(X, C), np.int64)
        passes.append(int((labels != prev).sum()))
        if shifts[-1] <= t:
            reason = "tolerance"
            break
        if i == max_iter:
            reason = "max_iter"
            break
        i += 1
    return {"C": C, "labels": labels, "n_iter": i, "reason": reason, "shifts": shifts, "passes": passes,
            "tol_abs": t}


def argmin64(X, C):
    """float64 argmin of the squared L2 distances (first index on ties)"""
    X = np.asarray(X, np.float64)
    C = np.asarray(C, np.float64)
    d = (X * X).sum(1)[:, None] - 2 * X @ C.T + (C * C).sum(1)[None, :]
    return np.argmin(d, axis=1)
