"""Seeded input generators shared by make_golden.py and the tests (inputs are never stored)."""
import numpy as np

# name -> (n, d, k, seed, kind)
ASSIGN_CASES = {
    "uniform_3000x256_k1024": (3000, 256, 1024, 777, "uniform"),
    "uniform_5000x64_k100": (5000, 64, 100, 1, "uniform"),
    "normal_4000x128_k300": (4000, 128, 300, 2, "normal"),
    "ragged_1000x7_k3": (1000, 7, 3, 3, "uniform"),
    "ragged_4097x100_k33": (4097, 100, 33, 4, "uniform"),
    "blobs_13000x2_k50": (13000, 2, 50, 5, "blobs"),
    "wide_range_2000x32_k16": (2000, 32, 16, 6, "wide"),
    "dupes_1024x64_k64": (1024, 64, 64, 7, "dupes"),
}


def blobs():
    """reference src/test.py:158-169"""
    rng = np.random.RandomState(0)
    arr = np.empty((13000, 2), dtype=np.float32)
    arr[:2000] = rng.rand(2000, 2) + [0, 2]
    arr[2000:4000] = rng.rand(2000, 2) - [0, 2]
    arr[4000:6000] = rng.rand(2000, 2) + [2, 0]
    arr[6000:8000] = rng.rand(2000, 2) - [2, 0]
    arr[8000:10000] = rng.rand(2000, 2) - [2, 2]
    arr[10000:] = rng.rand(3000, 2) + [2, 2]
    return arr


def make_assign_case(n, d, k, seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "blobs":
        X = blobs()
    elif kind == "normal":
        X = rng.standard_normal((n, d)).astype(np.float32)
    elif kind == "wide":      # features spanning 12 orders of magnitude
        X = (rng.standard_normal((n, d)) * (10.0 ** rng.integers(-6, 6, size=d))).astype(np.float32)
    else:
        X = rng.random((n, d), dtype=np.float32)
    C = X[rng.choice(len(X), k, replace=False)].copy()
    if kind == "dupes":       # exact duplicate centroids: ties must resolve to the lowest index
        C[k // 2:] = C[:k - k // 2]
    else:
        C += (rng.standard_normal(C.shape) * 0.01 * np.abs(C).mean()).astype(np.float32)
    return np.ascontiguousarray(X), np.ascontiguousarray(C)


HEADLINE_SAMPLE = 65536     # rows of the 8M headline pass whose reference assignments are stored


def headline_8m():
    """8 000 000 x 256 U[0,1) samples (seed 777, the reference README's benchmark), 1024 centroids = rows of them"""
    n, d, k = 8000000, 256, 1024
    rng = np.random.default_rng(777)
    X = np.empty((n, d), np.float32)
    for i in range(0, n, 1000000):               # chunked generation keeps the host RSS at the matrix itself
        X[i:i + 1000000] = rng.random((1000000, d), dtype=np.float32)
    C0 = X[rng.choice(n, k, replace=False)].copy()
    return X, C0


def headline_rows():
    """the fixed sample of headline rows (sorted) that tests/golden/headline_8m.npz covers"""
    return np.sort(np.random.default_rng(2024).choice(8000000, HEADLINE_SAMPLE, replace=False))
