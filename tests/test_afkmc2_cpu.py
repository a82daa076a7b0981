"""CPU tests of the AFK-MC² model (tests/afkmc2_model.py), which the GPU tests use as the reference: its
std::mt19937_64 against the C++ standard library, the vectorised model against a scalar, loop-by-loop transliteration
of Job::init_afkmc2 (seeding.cu) on the oracle's distances, and the seeding's properties."""
import bisect
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import afkmc2_model as A  # noqa: E402
import kmeans_parallel_model as KP  # noqa: E402
from oracle import oracle as O  # noqa: E402

_M64 = (1 << 64) - 1

_MT_PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include <random>
int main(int argc, char** argv) {
  std::mt19937_64 gen(std::strtoull(argv[1], nullptr, 10));
  for (int i = 0; i < 1000; i++) {
    const unsigned long long g = gen();
    std::printf("%llu %a\n", g, (static_cast<double>(g >> 11) + 0.5) * (1.0 / 9007199254740992.0));
  }
}
"""


class _ScalarMT:
    """std::mt19937_64 one output at a time, as the standard states it"""

    def __init__(self, seed=5489):
        self.mt = [seed & _M64]
        for i in range(1, 312):
            self.mt.append((6364136223846793005 * (self.mt[-1] ^ (self.mt[-1] >> 62)) + i) & _M64)
        self.i = 312

    def __call__(self):
        if self.i == 312:
            for k in range(312):
                y = (self.mt[k] & 0xFFFFFFFF80000000) | (self.mt[(k + 1) % 312] & 0x7FFFFFFF)
                self.mt[k] = self.mt[(k + 156) % 312] ^ (y >> 1) ^ (0xB5026F5AA96619E9 if y & 1 else 0)
            self.i = 0
        y = self.mt[self.i]
        self.i += 1
        y ^= (y >> 29) & 0x5555555555555555
        y ^= (y << 17) & 0x71D67FFFEDA60000
        y ^= (y << 37) & 0xFFF7EEE000000000
        return y ^ (y >> 43)


# --------------------------------------------------------------------------------------------------- mt19937_64
def test_mt19937_64_known_answer():
    """the C++ standard ([rand.predef]): the 10000th output of a default-constructed mt19937_64"""
    assert int(A.MT19937_64().next(10000)[-1]) == 9981545732273789042
    g = _ScalarMT()
    for _ in range(9999):
        g()
    assert g() == 9981545732273789042


@pytest.fixture(scope="module")
def mt_program(tmp_path_factory):
    """the 10-line C++ program above, built with the oracle's compiler (gcc, as C++)"""
    d = tmp_path_factory.mktemp("mt")
    src, exe = d / "mt.cc", d / "mt"
    src.write_text(_MT_PROGRAM)
    subprocess.check_call(["gcc", "-x", "c++", "-O2", "-o", str(exe), str(src), "-lstdc++"])
    return str(exe)


@pytest.mark.parametrize("seed", [0, 7, 2 ** 32 - 1])
def test_mt19937_64_matches_the_cpp_library(mt_program, seed):
    out = subprocess.check_output([mt_program, str(seed)], text=True).split()
    want = np.array([int(v) for v in out[0::2]], np.uint64)
    uni = np.array([float.fromhex(v) for v in out[1::2]])
    g = A.MT19937_64(seed)
    assert np.array_equal(g.next(1), want[:1]) and np.array_equal(g.next(700), want[1:701])   # across a twist
    assert np.array_equal(A.MT19937_64(seed).uniform(1000), uni)
    s = _ScalarMT(seed)
    assert [s() for _ in range(1000)] == [int(v) for v in want]
    assert (uni > 0).all() and (uni < 1).all()


# ---------------------------------------------------------------------------------- the literal transliteration
def _transliteration(X, K, seed, m, w, metric):
    """Job::init_afkmc2 statement by statement: host_dists from plusplus_kernel (NaN for a row whose x[0] is NaN),
    the two double loops, std::lower_bound, afkmc2_min_dist_kernel's atomicMin on float bits per (candidate,
    centroid) pair, the float chain.  Distances are the oracle's ko_distance."""
    L = O.lib()
    N, D = X.shape
    fp = ctypes.POINTER(ctypes.c_float)
    row = lambda i: X[i].ctypes.data_as(fp)   # noqa: E731
    f32 = np.float32
    m = m or 200
    c0 = KP.first_centroid(X, seed, w)
    host_dists = [float(L.ko_distance(metric, row(i), row(c0), D)) if X[i, 0] == X[i, 0] else float("nan")
                  for i in range(N)]
    W = float(N) if w is None else sum(float(v) for v in w)
    dsum = 0.0
    for i in range(N):
        d2 = host_dists[i] * host_dists[i]
        if np.isfinite(d2):
            dsum += (float(w[i]) * d2) if w is not None else d2
    q, cdf, acc = [], [], 0.0
    for i in range(N):
        d2 = host_dists[i] * host_dists[i]
        wi = float(w[i]) if w is not None else 1.0
        if not np.isfinite(d2):
            qi = 0.0
        else:
            qi = wi / (2.0 * W) + (wi * d2 / (2.0 * dsum) if dsum > 0 else wi / (2.0 * W))
        q.append(f32(qi))
        acc += qi
        cdf.append(acc)
    gen = _ScalarMT(seed)

    def uniform():
        return ((gen() >> 11) + 0.5) * (1.0 / 9007199254740992.0)

    chosen = [c0]
    for k in range(1, K):
        cand, rand_a = [], []
        for j in range(m):
            part = uniform() * cdf[N - 1]
            cand.append(min(bisect.bisect_left(cdf, part), N - 1))
            rand_a.append(f32(uniform()))
        p_cand = []
        for j in range(m):
            bits = 0x7F7F7F7F
            for c in range(k):
                d = f32(L.ko_distance(metric, row(cand[j]), row(chosen[c]), D))
                if d == d:
                    bits = min(bits, int(np.array([max(d, f32(0))], np.float32).view(np.uint32)[0]))
            dmin = np.array([bits], np.uint32).view(np.float32)[0]
            with np.errstate(over="ignore"):
                p_cand.append(f32(w[cand[j]]) * (dmin * dmin) if w is not None else dmin * dmin)
        curr_prob, curr_ind = f32(0), 0
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            for j in range(m):
                cand_prob = f32(p_cand[j] / q[cand[j]])
                if curr_prob == 0 or cand_prob / curr_prob > rand_a[j]:
                    curr_ind, curr_prob = j, cand_prob
        chosen.append(cand[curr_ind])
    return np.array(chosen, np.int64)


def _data(n, d, seed, metric=0, nan_rows=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((6, d)).astype(np.float32) * 3
    X = (centers[rng.integers(0, 6, n)] + 0.5 * rng.standard_normal((n, d))).astype(np.float32)
    if metric:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    if nan_rows:
        rows = rng.choice(np.arange(1, n), 2 * nan_rows, replace=False)
        X[rows[:nan_rows], 0] = np.nan
        X[rows[nan_rows:], min(5, d - 1)] = np.nan
    return X


TRANSLIT = {
    # id: (N, D, K, m, metric, weights, NaN rows of each kind)
    "l2": (300, 13, 8, 0, 0, None, 0),
    "cos": (300, 13, 8, 0, 1, None, 0),
    "l2-zero-weights": (300, 13, 8, 20, 0, "zeros", 0),
    "cos-lognormal": (240, 9, 6, 9, 1, "lognormal", 0),
    "l2-m1": (200, 8, 7, 1, 0, None, 0),
    "l2-m-half": (120, 6, 5, 60, 0, "zeros", 0),
    "l2-nan-rows": (300, 13, 8, 25, 0, None, 6),
}


def _weights(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind is None:
        return None
    if kind == "lognormal":
        return rng.lognormal(0, 1, n).astype(np.float32)
    w = rng.integers(1, 5, n).astype(np.float32)
    w[rng.random(n) < 0.3] = 0
    return w


@pytest.mark.parametrize("case", list(TRANSLIT), ids=list(TRANSLIT))
def test_model_equals_the_literal_transliteration(case):
    N, D, K, m, metric, wk, nans = TRANSLIT[case]
    X = _data(N, D, 1, metric, nans)
    w = _weights(wk, N, 2)
    for seed in (3, 11):
        r = A.afkmc2(X, K, seed, m=m, w=w, metric=metric)
        assert r.c0 == r.rows[0] and len(r.rows) == K
        if metric == 1:   # libm's acosf (the oracle) and the model's rounded arccos may differ by an ulp
            assert r.margin_draw > 1e-6 and r.margin_accept > 1e-6, (r.margin_draw, r.margin_accept)
        assert np.array_equal(r.rows, _transliteration(X, K, seed, m, w, metric)), (case, seed)
        assert np.array_equal(r.C.view(np.uint32), X[r.rows].view(np.uint32))


# -------------------------------------------------------------------------------------------------- properties
def _drawn(r):
    return np.unique(np.concatenate([s.cand for s in r.trace]))


def test_zero_weight_rows_are_never_drawn():
    X = _data(2000, 16, 4)
    w = _weights("zeros", len(X), 5)
    for seed in (1, 2, 3):
        r = A.afkmc2(X, 12, seed, m=50, w=w)
        assert (w[_drawn(r)] > 0).all() and (w[r.rows] > 0).all()
        assert (r.q[w == 0] == 0).all() and (r.q[w > 0] > 0).all()


def test_a_chain_of_one_accepts_its_candidate():
    X = _data(500, 8, 6)
    r = A.afkmc2(X, 10, 9, m=1)
    for s in r.trace:
        assert s.accepted.tolist() == [True] and s.chosen == s.cand[0]


def test_duplicated_rows_take_the_last_candidate():
    """every row the same: q is uniform and p = 0 for every candidate, so curr_prob stays 0 and the chain keeps
    replacing its current candidate"""
    X = np.repeat(np.random.default_rng(7).standard_normal((1, 12)).astype(np.float32), 400, axis=0)
    r = A.afkmc2(X, 6, 5, m=30)
    assert np.all(r.q == r.q[0]) and np.isclose(r.cdf[-1], 1.0)
    for s in r.trace:
        assert (s.p == 0).all() and s.accepted.all() and s.chosen == s.cand[-1]


@pytest.mark.parametrize("metric", [0, 1])
def test_rows_with_a_nan_feature_are_never_drawn(metric):
    X = _data(3000, 16, 8, metric, nan_rows=60)
    bad = np.isnan(X).any(axis=1)
    checked = 0
    for seed in (1, 2, 3, 4):
        r = A.afkmc2(X, 20, seed, m=200, metric=metric)
        if bad[r.c0]:
            continue   # c0 is only redrawn on an x[0] NaN (draw_first_centroid, shared by every seeding)
        checked += 1
        assert (r.q[bad] == 0).all() and (r.q[~bad] > 0).all()
        assert not bad[_drawn(r)].any() and not np.isnan(r.C).any()
        for s in r.trace:
            assert (s.dmin < A.SENTINEL).all()
    assert checked >= 3


def test_a_candidate_with_no_finite_distance_has_infinite_p():
    E = np.array([[np.nan, 1.5, 0.0], [np.nan, np.inf, 2.0]], np.float32)
    dmin = A.min_dist(E)
    assert dmin[0] == A.SENTINEL and dmin[1] == np.float32(1.5) and dmin[2] == 0
    with np.errstate(over="ignore"):
        assert np.isposinf(dmin[0] * dmin[0])


def test_chain_length_rule():
    assert A.chain_length(0, 10) == 200 and A.chain_length(5, 10) == 5
    with pytest.raises(ValueError):
        A.chain_length(6, 10)


def test_proposal_sums_are_sequential():
    """dsum and the CDF are left-to-right double sums, not np.sum's pairwise sum"""
    rng = np.random.default_rng(12)
    d = rng.lognormal(0, 4, 5000).astype(np.float32)
    q, cdf, _ = A.proposal(d)
    d2 = d.astype(np.float64) ** 2
    dsum = 0.0
    for v in d2:
        dsum += v
    qi = 1.0 / (2.0 * len(d)) + d2 / (2.0 * dsum)
    acc, want = 0.0, []
    for v in qi:
        acc += v
        want.append(acc)
    assert np.array_equal(cdf, np.array(want)) and np.array_equal(q, qi.astype(np.float32))
