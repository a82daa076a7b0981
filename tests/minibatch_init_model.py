"""NumPy model of the init stage of mini-batch k-means (kmeans_cuda(..., batch_size=b, init_size=, n_init=);
include/kmcuda_b200.h kmcuda_b200_kmeans_minibatch_init, DESIGN.md §4q).

It restates the library's draws of the seeding subsets and of the validation rows (the counter hash of
tests/minibatch_model.py with their own tags), scikit-learn's default init size (MiniBatchKMeans._check_params_vs_input)
and the validation inertia and pick.  The seed schedule and the pick are those of the restarts
(tests/restarts_model.py).
tests/test_minibatch_init_cpu.py checks it against scikit-learn; tests/test_minibatch_init_gpu.py pins the library to
it."""
import numpy as np

import minibatch_model as MB
import restarts_model as RS

TAG_INIT = 0x6D62696E69747375    # kernels.h: kMbTagInit
TAG_VALID = 0x6D6276616C696421   # kernels.h: kMbTagValid
AUTO = 0xFFFFFFFF                # KMCUDA_B200_INIT_SIZE_AUTO

seeds = RS.seeds     # seed_r = seed + r * 0x9E3779B9 (mod 2^32)
select = RS.select   # init 0 is the first best; a later one wins only with a strictly lower inertia, NaN never


def _draw(key, N, m):
    """rows_j = floor(u(key, j) * N), j < m: launch_mb_draw"""
    h = MB.mix_np(np.uint64(key) ^ np.arange(m, dtype=np.uint64))
    u = (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return np.minimum(np.floor(u * N).astype(np.int64), N - 1)


def init_size(N, batch_size, K, init_size=AUTO):
    """the m of the init stage: an explicit size capped at N, or scikit-learn's default for AUTO"""
    b = min(batch_size, N)
    m = init_size
    if init_size == AUTO:
        m = 3 * b
        if m < K:
            m = 3 * K
    return min(m, N)


def init_rows(seed, r, N, m):
    """the seeding subset of init r (only drawn when m < N)"""
    return _draw(MB.step_key(seed, r, TAG_INIT), N, m)


def valid_rows(seed, N, m):
    """the validation rows (only drawn when n_init > 1)"""
    return _draw(MB.step_key(seed, 0, TAG_VALID), N, m)


def validation_inertia(X, C, rows, w=None, labels=None):
    """sum over the entries rows of w * ||x - c_label||^2 in float64, duplicates included; labels default to the
    float64 argmin, and an entry whose label is not a centroid adds 0"""
    Xv = np.asarray(X, np.float64)[rows]
    C = np.asarray(C, np.float64)
    wv = np.ones(len(rows)) if w is None else np.asarray(w, np.float64)[rows]
    if labels is None:
        labels = np.argmin(((Xv[:, None, :] - C[None, :, :]) ** 2).sum(2), axis=1)
    labels = np.asarray(labels)
    live = labels < len(C)
    e = ((Xv - C[np.where(live, labels, 0)]) ** 2).sum(1)
    return float(np.sum(np.where(live, wv * e, 0.0)))
