"""CPU models of the tensor-core Lloyd pass at 512 < D <= 1024 (assign_tc.cu, NKB 9..16: 64-row tiles; DESIGN.md
section 4).  No GPU needed.

1. The error bound still contains the fp32 winner at these widths: `test_margin_cpu._filter_model` (fp16 operands,
   fp32 accumulation, the margin exactly as the epilogue computes it, eps_acc = (D + 16) 2^-22 |x~| cmax) on
   adversarially scaled data at D in {516, 768, 1024}, centred and uncentred.
2. The split-column epilogue: consumer warpgroup g holds columns 64 g .. 64 g + 63 of every n-tile, lane t the columns
   64 g + 8 j + 2 t + e (16-bit masks, bit b = 2 j + e).  Each warpgroup's running row maximum covers its own columns
   only, so its threshold is <= the one of the true row maximum and its candidate set contains the true one; the
   emitter merges the 8 lists of a row (two warpgroups x four lanes) against the larger of the two maxima.  The
   model replays that on fp32 scores and checks that the merged set always contains every column within the margin
   of the row maximum (so the exact winner), and that the decode maps every (warpgroup, lane, bit) to its own column.
3. The A-slot / norms ring of the 64-row layout (16 slots of 8 KiB) for NKB 9..16 under random interleavings, with
   the simulator of test_a_ring_model_cpu.py: the slot / barrier protocol is the same as for NKB 1..8.
"""
import random

import numpy as np
import pytest

import tc_sweep_cases as T
from test_a_ring_model_cpu import ring_depths, simulate
from test_margin_cpu import _filter_model

TN, LIST_LEN, MAX_CAND = 128, 5, 32


# ------------------------------------------------------------------------------------------------ 1. error bound
def _wide_cases():
    rng = np.random.default_rng(2024)
    out = []
    for (n, d, k, kind) in [(120, 516, 40, "normal"), (120, 768, 60, "offset"), (100, 1024, 50, "wide"),
                            (120, 768, 64, "blobs"), (80, 1024, 30, "huge"), (100, 1024, 48, "embed")]:
        if kind == "normal":
            X = rng.standard_normal((n, d))
        elif kind == "offset":
            X = 50.0 + rng.standard_normal((n, d))
        elif kind == "wide":
            X = rng.standard_normal((n, d)) * (10.0 ** rng.integers(-6, 6, size=d))
        elif kind == "huge":
            X = rng.standard_normal((n, d)) * 1e15
        elif kind == "embed":            # unit-norm embedding-like rows with a shared offset direction
            X = rng.standard_normal((n, d)) + 3.0 * rng.standard_normal(d)[None]
            X /= np.linalg.norm(X, axis=1, keepdims=True)
        else:
            centers = rng.random((k, d))
            X = centers[rng.integers(0, k, n)] + 0.01 * rng.standard_normal((n, d))
        X = X.astype(np.float32)
        C = X[rng.choice(n, k, replace=False)] + (0.01 * np.abs(X).mean() * rng.standard_normal((k, d))).astype(np.float32)
        out.append(pytest.param(X, C.astype(np.float32), id="%s_%dx%d_k%d" % (kind, n, d, k)))
    return out


@pytest.mark.parametrize("centred", [False, True])
@pytest.mark.parametrize("X,C", _wide_cases())
def test_margin_contains_the_winner_up_to_d1024(X, C, centred):
    acc, E, s, mu = _filter_model(X, C, centred, "measured")
    Xd, Cd = X.astype(np.float64) - mu.astype(np.float64), C.astype(np.float64) - mu.astype(np.float64)
    exact = (s * s) * (Xd @ Cd.T - 0.5 * (Cd ** 2).sum(1)[None])
    assert np.isfinite(acc).all()
    worst = (np.abs(acc.astype(np.float64) - exact) / E[:, None]).max()
    assert worst <= 1.0, "error exceeds the bound: %.3f x E" % worst
    margin = 2.0 * E * 1.001 + 1e-30
    rows = np.arange(len(X))
    assert (acc[rows, exact.argmax(1)] >= acc.max(1) - margin).all()
    # the fp16 scale rule: s |c - mu| in [32, 64) for the largest centroid, and every score stays far above the
    # padding sentinel (-65504) relative to the guard at -65000
    cn = np.sqrt(((Cd * s) ** 2).sum(1)).max()
    assert 32.0 <= cn < 64.0 * 1.001
    assert (acc.max(1) - margin > -65000.0).all()


# ------------------------------------------------------------------------------------------------ 2. split epilogue
def decode(nn, wg, t, b):
    return nn * TN + 64 * wg + 8 * (b >> 1) + 2 * t + (b & 1)


LANE16 = np.array([[decode(0, 0, t, b) for b in range(16)] for t in range(4)])   # columns of lane t in a half


def test_decode_covers_the_ntile_once():
    cols = [decode(0, wg, t, b) for wg in range(2) for t in range(4) for b in range(16)]
    assert sorted(cols) == list(range(TN))
    # the 16-bit mask of the kernel: bit (15 - b) of (c0 << 8 | c1) is the sign of d_b, reversed after a shift by 16
    signs = np.random.default_rng(0).integers(0, 2, (200, 16))
    for sg in signs:
        c0 = int("".join(map(str, sg[:8])), 2)
        c1 = int("".join(map(str, sg[8:])), 2)
        x = (~((c0 << 8) | c1) << 16) & 0xFFFFFFFF
        mask = int(format(x, "032b")[::-1], 2)           # __brev
        assert mask == sum((1 - int(s)) << b for b, s in enumerate(sg))


def split_epilogue(S, mg, K):
    """the T64 MODE 0 epilogue + emitter on fp32 scores S [n][nt * 128] (one row per call of the inner loop; the two
    rows of a thread share a list entry in the kernel, which can only keep more entries).  Returns per row: the
    decoded candidates, the overflow flag, and the two warpgroup maxima."""
    n, ncols = S.shape
    nt = ncols // TN
    res = []
    for r in range(n):
        M = [-np.inf, -np.inf]
        lists = {(wg, t): [] for wg in range(2) for t in range(4)}
        full = False
        for nn in range(nt):
            for wg in range(2):
                vals = S[r, nn * TN + 64 * wg + LANE16]               # [lane][bit]
                cm = vals.max(1)
                M[wg] = max(M[wg], float(cm.max()))                   # quad all-reduce over the warpgroup's columns
                thr = np.float32(M[wg] - mg[r])
                bits = vals >= thr
                for t in range(4):
                    if not bits[t].any():
                        continue
                    lst = lists[(wg, t)]
                    if len(lst) >= LIST_LEN - 1:                      # compact_list against the risen threshold
                        lst[:] = [e for e in lst if e[0] >= thr]
                    if len(lst) < LIST_LEN:
                        lst.append((float(cm[t]), np.flatnonzero(bits[t]), nn))
                    else:
                        full = True
        thr = np.float32(max(M) - mg[r])                              # the emitter: the larger warpgroup maximum
        cands = []
        for wg in range(2):
            for t in range(4):
                for cmax, bits, nn in lists[(wg, t)]:
                    if cmax >= thr:
                        cands += [c for c in (decode(nn, wg, t, b) for b in bits) if c < K]
        res.append((cands, full or len(cands) > MAX_CAND, M))
    return res


def _adversarial_scores(seed, n=300, nt=6):
    """rows whose best column sits in one half while the other half holds near misses of a lower local maximum,
    rising maxima (compaction), ties and columns exactly at the threshold"""
    rng = np.random.default_rng(seed)
    S = (rng.standard_normal((n, nt * TN)) * 10.0 - 100.0).astype(np.float32)
    mg = rng.uniform(0.5, 4.0, n).astype(np.float32)
    for r in range(n):
        kind = r % 5
        win = int(rng.integers(0, nt * TN))
        top = np.float32(rng.uniform(-10, 10))
        if kind == 0:      # near misses in the other half, below the winner by 0.2 .. 3 margins
            other = [c for c in range(nt * TN) if (c % TN >= 64) != (win % TN >= 64)]
            for c in rng.choice(other, 12, replace=False):
                S[r, c] = top - np.float32(rng.uniform(0.2, 3.0)) * mg[r]
        elif kind == 1:    # rising maxima in one lane of one half, one per n-tile
            lane_cols = LANE16[rng.integers(0, 4)] + 64 * int(rng.integers(0, 2))
            for nn in range(nt):
                S[r, nn * TN + rng.choice(lane_cols)] = top - np.float32((nt - nn) * 0.45) * mg[r]
        elif kind == 2:    # exact ties in both halves
            S[r, rng.choice(nt * TN, 3, replace=False)] = top
        elif kind == 3:    # a column exactly at the threshold of the true maximum
            S[r, int(rng.integers(0, nt * TN))] = np.float32(top - mg[r])
        S[r, win] = top
    return S, mg


@pytest.mark.parametrize("seed", range(6))
def test_split_columns_contain_the_true_candidates(seed):
    S, mg = _adversarial_scores(seed)
    K = S.shape[1] - (seed * 7) % 40                                  # a ragged last n-tile for some seeds
    S[:, K:] = T.SENTINEL
    for r, (cands, ovf, M) in enumerate(split_epilogue(S, mg, K)):
        true_max = S[r, :K].max()
        assert max(M) == true_max and min(M) <= true_max
        want = set(np.flatnonzero(S[r, :K] >= np.float32(true_max - mg[r])).tolist())
        if not ovf:
            assert want <= set(cands), (r, sorted(want - set(cands)))
            assert len(set(cands)) == len(cands)                      # every column decoded once


@pytest.mark.parametrize("kind", ["rise", "list_overflow", "max_cand", "dupes"])
def test_split_columns_on_the_sweep_inputs(kind):
    """the adversarial inputs of the GPU sweep at D = 768, scores from the fp16 filter model: the merged split-column
    candidates contain the fp64 winner whenever the row does not take the exact pass"""
    X, C, info = T.list_case(kind, 768)
    S, mg, _ = T.model_scores(X, C)
    K = C.shape[0]
    res = split_epilogue(S, mg, K)
    truth = (((X.astype(np.float64)[:, None, :] - C.astype(np.float64)[None]) ** 2).sum(-1)).argmin(1)
    n_ovf = 0
    for r, (cands, ovf, _) in enumerate(res):
        n_ovf += ovf
        if not ovf:
            assert truth[r] in cands or kind == "dupes" and np.array_equal(C[truth[r]], C[cands[0]]), r
    if kind in ("list_overflow", "max_cand"):
        assert n_ovf > 0
    else:
        assert n_ovf == 0


# ------------------------------------------------------------------------------------------------ 3. A ring, NKB 9..16
@pytest.mark.parametrize("nkb", range(9, 17))
def test_a_ring_64_row_tiles(nkb):
    S, ND = ring_depths(nkb)
    assert S == 16 and nkb <= S and ND * nkb > S
    rng = random.Random(100 + nkb)
    for trial in range(40):
        segs = [rng.choice([1, 1, 2, 3, 8]) for _ in range(rng.randint(1, 7))]
        simulate(nkb, segs, seed=10000 * nkb + trial)
