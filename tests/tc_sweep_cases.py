"""Seeded inputs for the tensor-core filter sweep (`test_tc_sweep_gpu.py`) and the CPU model that proves the adversarial
ones reach the filter's slow paths (`test_tc_sweep_cases_cpu.py`).

Adversarial Lloyd inputs (`list_case`): rows come in groups of near-identical samples x_g; next to each group a few
"special" centroids c = x_g + r u (u a random unit vector) sit at chosen table indices with chosen squared distances
r^2 = R^2 - f * delta, where delta is the group's filter margin expressed in squared-distance units (2 margin / s^2, from
the filter model of `test_margin_cpu.py`).  Every other centroid is a background point ~sqrt(2 D) away, far outside any
margin.  Index j + 128 t lies in n-tile t at column j, which the epilogue gives to lane (j % 8) // 2 (column 8 j' + 2 t'
+ e belongs to lane t'), so the indices decide which (row, lane) list receives which candidates.

`epilogue_model` replays the MODE 0 candidate epilogue of `assign_tc.cu` on the model's fp32 scores: the running row
maximum, the 32-bit lane masks, the 5-entry lists per epilogue thread with `compact_list`, the overflow flag and the
emitter's decode.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from test_margin_cpu import _filter_model  # noqa: E402

TM = TN = 128
LIST_LEN = 5
MAX_CAND = 32
SENTINEL = -65504.0
UNTOUCHED = 0xFFFFFFFF

# lane t holds the columns 8 j + 2 t + e of every n-tile, mask bit b = 2 j + e
LANE_COLS = np.array([[8 * (b >> 1) + 2 * t + (b & 1) for b in range(32)] for t in range(4)])


def lane_of(col):
    return (col % 8) // 2


# ------------------------------------------------------------------------------------------ sweep data (MODE 0)
def unit(a):
    a = np.asarray(a, np.float64)
    return (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)


def clustered(n, D, seed, n_centers=64, sigma=0.3):
    """Gaussian clusters around standard-normal centres"""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((n_centers, D))
    X = centers[rng.integers(0, n_centers, n)] + sigma * rng.standard_normal((n, D))
    return np.ascontiguousarray(X, dtype=np.float32)


def perturbed_centroids(X, K, seed, near_ties=False):
    """K perturbed samples; near_ties: centroid 2i + 1 = centroid 2i + delta with |delta| spread over 1e-6 .. 1e-2 of
    the centroid's feature scale, so that some pairs fall inside the filter margin and go to the re-check"""
    rng = np.random.default_rng(seed)
    base = rng.choice(len(X), K, replace=len(X) < K)
    C = X[base].astype(np.float64)
    C += rng.standard_normal(C.shape) * 0.05 * np.abs(X).mean()
    if near_ties:
        h = K // 2
        scale = np.abs(C[0:2 * h:2]).mean(1, keepdims=True) * 10.0 ** rng.uniform(-6, -2, (h, 1))
        C[1:2 * h:2] = C[0:2 * h:2] + scale * rng.standard_normal((h, C.shape[1]))
    return np.ascontiguousarray(C, dtype=np.float32)


def sweep_n(label, num_sms):
    """'few': fewer sample tiles than SMs; 'many': more than two tiles per SM plus a ragged last tile"""
    if label == "few":
        return TM * max(1, num_sms // 2) + 37
    if label == "many":
        return TM * (2 * num_sms + 5) + 77
    return int(label)


# ------------------------------------------------------------------------------------------ adversarial Lloyd inputs
LIST_K = 1100            # 9 n-tiles, the last one ragged (76 real columns)
LIST_CASES = ("rise", "rise_margin", "rise_wide", "rise_coarse", "rise_pair", "list_overflow", "max_cand", "queue",
              "dupes")


def _place(x, r2, rng, metric):
    """a centroid at squared distance r2 from x (L2) / at chord length^2 r2 on the unit sphere (cosine)"""
    u = rng.standard_normal(x.shape)
    u -= (u @ x) / (x @ x) * x if metric == "cos" else 0.0
    u /= np.linalg.norm(u)
    if metric == "cos":
        # unit x, c = (x + r u) / |x + r u| with u orthogonal to x: |x - c|^2 = 2 - 2 / sqrt(1 + r^2)
        cosang = 1.0 - r2 / 2.0
        r = np.sqrt(1.0 / cosang ** 2 - 1.0)
        c = x + r * u
        return c / np.linalg.norm(c)
    return x + np.sqrt(r2) * u


def _layout(kind, n_groups):
    """per group: list of (table index, f) -- r^2 = R^2 - f * delta; the largest f is the exact winner"""
    out = []
    for g in range(n_groups):
        if kind == "rise":            # the best column of n-tile t beats n-tile t - 1 by 4 margins, same lane, 9 n-tiles
            out.append([(8 * g + 5 + TN * t, 4.0 * t) for t in range(9)])      # column 8 g + 5: lane 2
        elif kind == "rise_margin":   # steps of 0.4 margins: compaction keeps the last two entries and moves them down
            out.append([(8 * g + 5 + TN * t, 0.4 * t) for t in range(9)])
        elif kind == "rise_wide":     # steps of 0.75 margins: exactly 2 candidates per row, 1 with half the margin
            out.append([(8 * g + 5 + TN * t, 0.75 * t) for t in range(9)])
        elif kind == "rise_coarse":   # steps of 1.25 margins: exactly 1 candidate per row, 2 with twice the margin
            out.append([(8 * g + 5 + TN * t, 1.25 * t) for t in range(9)])
        elif kind == "rise_pair":     # groups 0-7 rise as in "rise" (rows R0 of their epilogue threads); group 8 + g
            if g < 8:                 # (rows R1 of the same threads, scores far below) has its one candidate in the
                out.append([(8 * g + 5 + TN * t, 4.0 * t) for t in range(9)])    # same lane of n-tile 0: compaction
            else:                                                               # must test it against ITS threshold
                out.append([(8 * (g - 8) + 4, 0.0)])
        elif kind == "list_overflow":  # 8 candidates within 0.7 margins in one lane, the winner in the last n-tile
            out.append([(8 * g + 3 + TN * t, 0.1 * t) for t in range(8)])      # column 8 g + 3: lane 1
        elif kind == "max_cand":      # 40 candidates in n-tile g; the winner is column 39, the last in emitter order
            f = np.random.default_rng(100 + g).permutation(np.linspace(0.0, 0.45, 39))
            out.append([(g * TN + c, f[c]) for c in range(39)] + [(g * TN + 39, 0.5)])
        elif kind == "queue":         # 16 candidates per row in one n-tile: the pair queue fills part-way through
            base = 16 * g
            out.append([(base + i, 0.5 * i / 15.0) for i in range(16)])
        else:                         # "dupes": one centroid at three indices in three n-tiles; the lowest (lane 3)
            out.append([(7 + 8 * g, 1.0), (256 + 8 * g, 0.0), (515 + 8 * g, 0.0)])   # is listed after lanes 0 and 1
    return out


def list_case(kind, D, metric="L2", seed=0):
    """(X, C, info): info['rows'][g] = row indices of group g, info['winner'][g] = fp64-exact winner index"""
    rng = np.random.default_rng(seed * 1000 + D * 7 + len(kind) + (0 if metric == "L2" else 500))
    n_groups, rows_per = (64, 32) if kind == "queue" else (16, 16) if kind == "rise_pair" else (8, 32)
    K = LIST_K
    C = rng.standard_normal((K, D))
    xg = rng.standard_normal((n_groups, D))
    gid = np.repeat(np.arange(n_groups), rows_per)
    if kind == "rise_pair":
        xg[:8] *= 3.0             # |x - mu|^2 / 2 is part of every score: the R1 rows score far below the R0 rows
        xg[8:] *= 0.3
        i = np.arange(n_groups * rows_per)
        gid = (i // 16) % 8 + 8 * ((i % 16) >= 8)
    if metric == "cos":
        C, xg = unit(C).astype(np.float64), unit(xg).astype(np.float64)
    layout = _layout(kind, n_groups)
    eta = 1e-6 if metric == "L2" else 1e-7
    X = xg[gid] + eta * rng.standard_normal((len(gid), D))
    if metric == "cos":
        X = unit(X).astype(np.float64)
    rows = [np.flatnonzero(gid == g) for g in range(n_groups)]
    place_seed = int(rng.integers(1 << 31))

    def build(delta):
        Cb = C.copy()
        grng = np.random.default_rng(place_seed)
        for g, spec in enumerate(layout):
            fmax = max(f for _, f in spec)
            R2 = (fmax + 40.0) * delta[g]
            for idx, f in spec:
                Cb[idx] = _place(xg[g], R2 - f * delta[g], grng, metric)
        if kind == "dupes":
            for g, spec in enumerate(layout):
                for idx, _ in spec[1:]:
                    Cb[idx] = Cb[spec[0][0]]
        return np.ascontiguousarray(Cb, np.float32)

    # two rounds: the margin depends (weakly) on the centroid table through mu, cmax and dcmax
    delta = np.full(n_groups, 1e-3 * D if metric == "L2" else 1e-4)
    Xf = np.ascontiguousarray(X, np.float32)
    for _ in range(2):
        Cf = build(delta)
        mg, s = margins(Xf, Cf, metric)
        delta = np.array([np.median(2.0 * mg[r] / (s * s)) for r in rows])
    Cf = build(delta)
    if kind == "dupes":
        winner = [spec[0][0] for spec in layout]
    else:
        winner = [max(spec, key=lambda e: e[1])[0] for spec in layout]
    return Xf, Cf, {"rows": rows, "winner": winner, "layout": layout, "delta": delta}


def margins(X, C, metric="L2"):
    """per-row margin (2 E 1.001, score units) and scale s of the MODE 0 filter (centred for L2; the converters measure
    |x~| and the rounding residual, as the kernel does)"""
    _, E, s, _ = _filter_model(X, C, centred=(metric == "L2"), residual="measured")
    return (2.0 * E * 1.001 + 1e-30).astype(np.float32), s


def model_scores(X, C, metric="L2"):
    """the model's fp32 scores [n][nt * 128] (padded columns at the -65504 sentinel) and margins"""
    acc, E, s, _ = _filter_model(X, C, centred=(metric == "L2"), residual="measured")
    n, K = acc.shape
    nt = (K + TN - 1) // TN
    S = np.full((n, nt * TN), SENTINEL, np.float32)
    S[:, :K] = acc
    return S, (2.0 * E * 1.001 + 1e-30).astype(np.float32), s


def epilogue_model(S, mg, K):
    """Replay of the MODE 0 epilogue + emitter (L2: no cap) over sample tiles of 128 rows.

    Returns a dict of per-row arrays: 'cands' (decoded candidates in emitter order, i.e. lane, entry, bit), 'total',
    'overflow' (the row goes to the exact pass), 'list_full' (flag bit 2), 'lane_ntiles' [n][4] (n-tiles in which the
    row had candidates in that lane), 'lane_m' (running maxima at those n-tiles, per lane), 'compactions' and 'moves'
    (compact_list calls / entries moved down, summed over the row's four epilogue threads)."""
    n, ncols = S.shape
    nt = ncols // TN
    out = {"cands": [None] * n, "total": np.zeros(n, np.int64), "overflow": np.zeros(n, bool),
           "list_full": np.zeros(n, bool), "lane_ntiles": np.zeros((n, 4), np.int64),
           "lane_m": [[[] for _ in range(4)] for _ in range(n)],
           "compactions": np.zeros(n, np.int64), "moves": np.zeros(n, np.int64)}
    lid = np.arange(256)
    w, lane = lid // 32, lid % 32
    R = np.stack([16 * w + lane // 4, 16 * w + lane // 4 + 8])       # [hh][thread]
    T = lane % 4
    for t0 in range(0, n, TM):
        nr = min(TM, n - t0)
        St = np.full((TM, ncols), SENTINEL, np.float32)
        St[:nr] = S[t0:t0 + nr]
        m = np.ones(TM, np.float32)
        m[:nr] = mg[t0:t0 + nr]
        M = np.full(TM, -np.inf, np.float32)
        lists = [[] for _ in range(256)]
        full = np.zeros((2, 256), bool)
        comp = np.zeros(256, np.int64)
        moves = np.zeros(256, np.int64)
        for nn in range(nt):
            vals = St[:, nn * TN + LANE_COLS]                          # [row][lane][bit]
            cm = vals.max(-1)
            M = np.maximum(M, cm.max(1))
            thr = (M - m).astype(np.float32)
            bits = vals >= thr[:, None, None]
            for r in range(nr):
                for t in range(4):
                    if bits[r, t].any():
                        out["lane_ntiles"][t0 + r, t] += 1
                        out["lane_m"][t0 + r][t].append(float(M[r]))
            has = bits[R[0], T].any(1) | bits[R[1], T].any(1)
            for th in np.flatnonzero(has):
                r0, r1, t = R[0, th], R[1, th], T[th]
                lst = lists[th]
                if len(lst) >= LIST_LEN - 1:
                    keep = [i for i, e in enumerate(lst) if e[0] >= thr[r0] or e[1] >= thr[r1]]
                    comp[th] += 1
                    moves[th] += sum(1 for wi, i in enumerate(keep) if wi != i)
                    lst[:] = [lst[i] for i in keep]
                m0 = np.flatnonzero(bits[r0, t])
                m1 = np.flatnonzero(bits[r1, t])
                if len(lst) < LIST_LEN:
                    lst.append((cm[r0, t], cm[r1, t], m0, m1, nn))
                else:
                    full[0, th] |= len(m0) > 0
                    full[1, th] |= len(m1) > 0
        for r in range(nr):
            hh = (r >> 3) & 1
            lid0 = (r >> 4) * 32 + (r & 7) * 4
            thr = np.float32(M[r] - m[r])
            cands, fl = [], False
            for t in range(4):
                th = lid0 + t
                fl |= bool(full[hh, th])
                out["compactions"][t0 + r] += comp[th]
                out["moves"][t0 + r] += moves[th]
                for e in lists[th]:
                    if not e[hh] >= thr:
                        continue
                    cands += [c for c in (e[4] * TN + LANE_COLS[t][e[2 + hh]]).tolist() if c < K]
            out["cands"][t0 + r] = cands
            out["total"][t0 + r] = len(cands)
            out["list_full"][t0 + r] = fl
            out["overflow"][t0 + r] = fl or len(cands) > MAX_CAND
    return out


def max_pairs(n):
    return 10 * n + 1024


# ------------------------------------------------------------------------------------------ non-finite inputs
def nonfinite_case(D, seed=0):
    """K % 128 != 0, exact duplicate centroids in different n-tiles, NaN / +-Inf / 1e30 rows, NaN and Inf centroids,
    rows far from every centroid (their threshold falls below the padding sentinel)"""
    rng = np.random.default_rng(seed + D)
    n, K = 3000, 300
    X = clustered(n, D, seed + 1, n_centers=40, sigma=0.2)
    C = perturbed_centroids(X, K, seed + 2)
    C[200] = C[3]                 # exact duplicates: 200 and 129 (lane 0) reach the re-check queue before 3 (lane 1) and
    C[129] = C[6]                 # 6 (lane 3); the lowest index must win
    X[10:20] = C[6] + 1e-3 * rng.standard_normal((10, D)).astype(np.float32)
    X[20:30] = C[3]
    C[40] = np.nan
    C[41, D // 2] = np.inf
    C[170, 0] = -np.inf
    X[100, 0] = np.nan
    X[101, D - 1] = np.inf
    X[102, 1 % D] = -np.inf
    X[103] = 1e30
    X[104, D // 2] = 1e30
    X[105] = -40.0 * np.abs(X).max()
    X[106] = 900.0 * np.abs(X).max()
    X[107] = 0.0
    return np.ascontiguousarray(X, np.float32), np.ascontiguousarray(C, np.float32)


# ------------------------------------------------------------------------------------------ k-NN inputs
def knn_shape(kind, D, seed=0):
    """(X, C, A) at N ~ 20000: A = fp64 nearest centroid"""
    rng = np.random.default_rng(seed + D + len(kind))
    if kind == "tiny_clusters":   # 2000 centroids, 1-19 samples each, a quarter of them empty
        K = 2000
        centers = rng.standard_normal((K, D)) * 3.0
        sizes = rng.integers(1, 20, K)
        sizes[rng.random(K) < 0.25] = 0
        idx = np.repeat(np.arange(K), sizes)
        X = centers[idx] + 0.2 * rng.standard_normal((len(idx), D))
        C = centers
    elif kind == "giant":         # one cluster holds 90 % of the samples
        K = 64
        centers = rng.standard_normal((K, D)) * 2.0
        lab = np.where(rng.random(20000) < 0.9, 0, rng.integers(1, K, 20000))
        X = centers[lab] + 0.5 * rng.standard_normal((20000, D))
        C = centers
    else:   # "duplicates": 100 blocks of 20 identical samples, and one sample 4000 times -- every copy ties at distance
        K = 100   # 0, so the copies fill more than KNN_CAP = 40 (chunk, mask) entries of each other's half-rows
        centers = rng.standard_normal((K, D)) * 2.0
        base = centers[rng.integers(0, K, 14000)] + 0.4 * rng.standard_normal((14000, D))
        X = np.concatenate([base, np.repeat(base[:100], 20, axis=0), np.repeat(base[100:101], 4000, axis=0)])
        C = centers
    X = np.ascontiguousarray(X, np.float32)
    C = np.ascontiguousarray(C, np.float32)
    return X, C, nearest(X, C)


def nearest(X, C):
    Xd, Cd = X.astype(np.float64), C.astype(np.float64)
    out = np.empty(len(X), np.uint32)
    for i in range(0, len(X), 4096):
        d = (Cd ** 2).sum(1)[None] - 2.0 * Xd[i:i + 4096] @ Cd.T
        out[i:i + 4096] = d.argmin(1)
    return out


def knn_truth(X, queries, k):
    """fp64 distances of the k + 1 nearest other samples of each query (ascending), exact differences"""
    Xd = X.astype(np.float64)
    sq = (Xd ** 2).sum(1)
    res = np.empty((len(queries), k + 1))
    for i0 in range(0, len(queries), 512):
        q = queries[i0:i0 + 512]
        g = sq[None] - 2.0 * Xd[q] @ Xd.T
        g[np.arange(len(q)), q] = np.inf
        pre = np.argpartition(g, k + 24, axis=1)[:, :k + 25]
        for j, qi in enumerate(q):
            d = ((Xd[pre[j]] - Xd[qi]) ** 2).sum(1)
            res[i0 + j] = np.sort(d)[:k + 1]
    return res
