"""Generates the committed golden vectors:

    python tests/golden/make_golden.py               # golden.npz: needs the C oracle only
    python tests/golden/make_golden.py --headline    # headline_8m.npz: needs a GPU and oracle/_ref (the reference)

Inputs are regenerated from seeds by tests/golden/cases.py; only the expected OUTPUTS are stored.
Expected assignments come from the C oracle (oracle/kmcuda_oracle.c), which the GPU suite separately
pins bit-for-bit against the unmodified reference rebuilt for sm_90 (tests/test_parity_gpu.py::
test_oracle_matches_reference); expected neighbours come from scikit-learn, the reference's own pin
(reference src/test.py:598-606).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle import oracle as O  # noqa: E402
import cases  # noqa: E402


def main():
    out = {}
    for name, (n, d, k, seed, kind) in cases.ASSIGN_CASES.items():
        X, C = cases.make_assign_case(n, d, k, seed, kind)
        a, _, changed = O.assign_lloyd(X, C)
        _, best, second = O.assign_truth(X, C)
        out["assign/" + name] = a
        out["assign_ties/" + name] = O.tie_exempt(best, second)
        print(name, "changed", changed, "ties", int(out["assign_ties/" + name].sum()))
    X = cases.blobs()
    from sklearn.neighbors import NearestNeighbors
    nb = NearestNeighbors(n_neighbors=11).fit(X)
    out["knn/blobs_k10"] = nb.kneighbors(X)[1][:, 1:].astype(np.uint32)
    np.savez_compressed(os.path.join(HERE, "golden.npz"), **out)
    print("wrote", os.path.join(HERE, "golden.npz"), os.path.getsize(os.path.join(HERE, "golden.npz")), "bytes")


def headline(path):
    """The reference library's assignments of the headline pass (8M x 256 @ 1024, one Lloyd assignment) for the
    fixed row sample cases.headline_rows().  A row's assignment depends only on the row and the centroids, so the
    reference runs on the sampled rows alone: the full 8M-row call of the reference takes minutes."""
    import ctypes
    X, C0 = cases.headline_8m()
    rows = cases.headline_rows()
    Xs = np.ascontiguousarray(X[rows])
    del X
    ref = O.reference_lib()
    C = C0.copy()
    A = np.zeros(len(rows), np.uint32)
    m = ctypes.c_uint32(0)
    rc = ref.kmeans_cuda(3, ctypes.byref(m), 1.0, 0.0, 0, len(rows), Xs.shape[1], len(C0), 3, 1, -1, 0, 0,
                         Xs.ctypes.data, C.ctypes.data, A.ctypes.data, None)
    assert rc == 0, rc
    np.savez_compressed(path, assign=A.astype(np.uint16))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if "--headline" in sys.argv:
        headline(sys.argv[sys.argv.index("--headline") + 1] if len(sys.argv) > sys.argv.index("--headline") + 1
                 else os.path.join(HERE, "headline_8m.npz"))
    else:
        main()
