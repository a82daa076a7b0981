"""NumPy model of the empty-cluster relocation (kmeans_cuda(..., relocate_empty_clusters=True);
include/kmcuda_b200.h kmcuda_b200_kmeans_relocate, DESIGN.md §4l).

`relocate` is one update's rule on the exchanged totals; `run` is a whole Lloyd run with it, the centroids kept in fp32
between iterations as the library keeps them.  Labels come from the caller (the oracle's argmin for the GPU pin, a
float64 argmin for the scikit-learn comparisons), so the model holds no assignment rule.
tests/test_relocate_cpu.py checks it against scikit-learn; tests/test_relocate_gpu.py pins the library to it."""
import numpy as np


def distances(X, C, labels, metric=0):
    """the relocation key d_i of every row against its own centroid (float64; L2: squared distance, the quantity the
    library orders by before its square root; angular: the angle), NaN where the row has no centroid"""
    X = np.asarray(X, np.float64)
    C = np.asarray(C, np.float64)
    K = len(C)
    labels = np.asarray(labels, np.int64)
    own = labels < K
    d = np.full(len(X), np.nan)
    c = C[labels[own]]
    with np.errstate(invalid="ignore"):
        if metric == 1:
            d[own] = np.arccos(np.clip((X[own] * c).sum(1), -1.0, 1.0))
        else:
            d[own] = ((X[own] - c) ** 2).sum(1)
    return d


def relocate(X, w, labels, d, sums, counts, W):
    """One update's relocation.  sums [K][D] fp32, counts [K], W [K] fp32 (the weight totals; the counts without
    weights) are the exchanged totals before normalisation.  Returns (sums, counts, W, records, left_empty) with records
    [(cluster, row, key, donor)] in walk order."""
    X = np.asarray(X, np.float32)
    K = len(W)
    n = len(X)
    w = np.ones(n, np.float32) if w is None else np.asarray(w, np.float32)
    sums = np.array(sums, np.float32)
    counts = np.array(counts, np.int64)
    W = np.array(W, np.float32)
    labels = np.asarray(labels, np.int64)
    E = np.flatnonzero(W == 0)
    if len(E) == 0:
        return sums, counts, W, [], 0
    elig = np.flatnonzero((labels < K) & (w > 0) & np.isfinite(d))
    order = elig[np.lexsort((elig, -d[elig]))]
    Wrun = W.copy()
    records = []
    for i in order:
        if len(records) == len(E):
            break
        a = labels[i]
        left = np.float32(Wrun[a] - w[i])
        if not left > 0:
            continue
        Wrun[a] = left
        records.append((int(E[len(records)]), int(i), float(d[i]), int(a)))
    for e, i, _, a in records:
        wx = (np.float32(w[i]) * X[i]).astype(np.float32)
        sums[a] = (sums[a] - wx).astype(np.float32)
        sums[e] = wx
        counts[a] -= 1
        counts[e] = 1
        W[a] = np.float32(W[a] - w[i])
        W[e] = w[i]
    return sums, counts, W, records, len(E) - len(records)


def normalize_cos(x):
    x = np.asarray(x, np.float32)
    return (x * np.float32(1.0 / np.sqrt(np.float64((x.astype(np.float64) ** 2).sum())))).astype(np.float32)


def run(X, C0, labeler, tolerance=0.0, metric=0, w=None, max_iter=300):
    """A whole Lloyd run with relocation.  labeler(X, C) -> labels (K for a row without a centroid).  Returns
    (C, labels, log) with log [(iteration, reassignments, records, left_empty)]."""
    X = np.asarray(X, np.float32)
    n, D = X.shape
    C = np.array(C0, np.float32)
    K = len(C)
    wf = np.ones(n, np.float64) if w is None else np.asarray(w, np.float64)
    prev = np.full(n, -1, np.int64)
    ccounts = np.zeros(K, np.float32)     # angular recurrence: the previous update's counts / weight totals
    prev_sums = np.zeros((K, D), np.float32)
    log = []
    for it in range(1, max_iter + 1):
        labels = np.asarray(labeler(X, C), np.int64)
        changed = int((labels != prev).sum())
        prev = labels
        entry = [it, changed, [], 0]
        log.append(entry)
        if changed <= tolerance * n:
            break
        own = labels < K
        sums = np.zeros((K, D), np.float64)
        np.add.at(sums, labels[own], wf[own, None] * X[own])
        counts = np.bincount(labels[own], minlength=K)
        Wt = np.bincount(labels[own], weights=wf[own], minlength=K)
        Wf = counts.astype(np.float32) if w is None else Wt.astype(np.float32)
        d = distances(X, C, labels, metric)
        sums, counts, Wf, records, left = relocate(X, w, labels, d, sums.astype(np.float32), counts, Wf)
        entry[2], entry[3] = records, left
        if metric == 1:
            with np.errstate(invalid="ignore", divide="ignore"):
                raw = (C.astype(np.float64) * ccounts[:, None] + (sums.astype(np.float64) - prev_sums)).astype(
                    np.float32)
                C = (raw / np.sqrt((raw.astype(np.float64) ** 2).sum(1, keepdims=True))).astype(np.float32)
            for e, i, _, _ in records:
                C[e] = normalize_cos(X[i])
            prev_sums = sums
            ccounts = Wf
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                C = (sums * (np.float32(1) / Wf)[:, None]).astype(np.float32)
    return C, prev, log
