"""The adversarial Lloyd inputs of `tc_sweep_cases.py` reach the filter paths they are built for (no GPU needed).

There is no device counter for list compaction or for a full per-lane list, so a GPU test built on these inputs could
pass without ever running those paths.  This file replays the MODE 0 epilogue (`tc_sweep_cases.epilogue_model`: the
centred filter model of `test_margin_cpu.py`, the lane / column map of `test_native_epilogue_model_cpu.py`, 5-entry lists
with `compact_list`, the emitter's decode) on the same inputs and asserts, per construction, what the kernel will see.
"""
import numpy as np
import pytest

import tc_sweep_cases as T

CASES = [(k, D, "L2") for k in T.LIST_CASES for D in (64, 256, 512)]
CASES += [(k, D, "cos") for k in ("rise", "list_overflow") for D in (64, 256)]


@pytest.fixture(scope="module")
def replay():
    memo = {}

    def get(kind, D, metric):
        if (kind, D, metric) not in memo:
            X, C, info = T.list_case(kind, D, metric)
            S, mg, _ = T.model_scores(X, C, metric)
            memo[(kind, D, metric)] = X, C, info, T.epilogue_model(S, mg, C.shape[0])
        return memo[(kind, D, metric)]
    return get


def _truth(X, C, metric):
    if metric == "L2":
        return T.nearest(X, C)
    return (X.astype(np.float64) @ C.astype(np.float64).T).argmax(1)


@pytest.mark.parametrize("kind,D,metric", CASES, ids=["%s-D%d-%s" % c for c in CASES])
def test_adversarial_case_reaches_its_path(replay, kind, D, metric):
    X, C, info, m = replay(kind, D, metric)
    truth = _truth(X, C, metric)
    for g, (rows, win) in enumerate(zip(info["rows"], info["winner"])):
        assert (truth[rows] == win).all(), (g, "the fp64 winner is not where the construction put it")
        spec = info["layout"][g]
        lane = T.lane_of(spec[0][0] % T.TN)
        for r in rows:
            cands, total = m["cands"][r], m["total"][r]
            if kind.startswith("rise") and (kind != "rise_pair" or g < 8):
                # >= 8 n-tiles with candidates in the same lane, each one raising the row maximum
                assert m["lane_ntiles"][r, lane] >= 8
                hist = m["lane_m"][r][lane]
                assert all(b > a for a, b in zip(hist, hist[1:])), hist
                assert m["compactions"][r] >= 2 and not m["overflow"][r]
                if kind == "rise_margin":
                    assert m["moves"][r] > 0 and 2 <= total <= 4 and win in cands   # compaction keeps and moves
                elif kind == "rise_wide":
                    assert total == 2 and win in cands                              # the winner and the last runner-up
                else:
                    assert cands == [win]                                           # compaction leaves one candidate
            elif kind == "rise_pair":
                # the R1 row's only candidate sits in the oldest entry of a list that its R0 partner keeps compacting
                partner = r - 8
                assert m["compactions"][partner] >= 2 and cands == [win]
                assert m["lane_ntiles"][r, lane] == 1
            elif kind == "list_overflow":
                # >= 6 n-tiles with candidates in one lane, <= 32 candidates in all; the winner's entry never fits
                assert m["lane_ntiles"][r, lane] >= 6 and m["list_full"][r] and m["overflow"][r]
                assert total <= T.MAX_CAND and win not in cands
            elif kind == "max_cand":
                # 40 candidates: more than MAX_CAND, and the winner lies beyond the first 32 in emitter order
                assert total == 40 and m["overflow"][r] and not m["list_full"][r]
                assert cands.index(win) >= T.MAX_CAND
            elif kind == "queue":
                assert 11 <= total <= T.MAX_CAND and not m["overflow"][r]
            else:   # dupes: all three copies reach the re-check, the lowest index is not the first one listed
                copies = sorted(idx for idx, _ in spec)
                assert sorted(cands) == copies and not m["overflow"][r]
                assert cands[0] != win
    pairs = int(m["total"][(m["total"] >= 2) & ~m["overflow"]].sum())
    if kind == "queue":
        # more than 10 candidates per row on average: the pair queue (10 n + 1024) fills part-way through the pass
        assert pairs > T.max_pairs(len(X)) and pairs < 2 * T.max_pairs(len(X))
    else:
        assert pairs <= T.max_pairs(len(X))


def test_epilogue_model_matches_the_plain_margin_rule():
    """without list pressure the replay yields exactly the columns within the margin of the row maximum"""
    rng = np.random.default_rng(3)
    X = rng.standard_normal((300, 64)).astype(np.float32)
    C = (X[rng.choice(300, 300, replace=False)] + 0.3 * rng.standard_normal((300, 64))).astype(np.float32)
    S, mg, _ = T.model_scores(X, C)
    m = T.epilogue_model(S, mg, 300)
    for r in range(300):
        want = set(np.flatnonzero(S[r, :300] >= np.float32(S[r].max() - mg[r])).tolist())
        if not m["overflow"][r]:
            assert set(m["cands"][r]) == want


@pytest.mark.parametrize("D", [64, 256, 512])
def test_candidate_counts_depend_on_the_margin_width(replay, D):
    """the rising cases with steps of 0.75 / 1.25 margins pin the margin's width: with half the margin every row of
    "rise_wide" has one candidate (no re-check), with twice the margin every row of "rise_coarse" has two"""
    for kind, scale, want in (("rise_wide", 0.5, 1), ("rise_coarse", 2.0, 2)):
        X, C, info, m = replay(kind, D, "L2")
        S, mg, _ = T.model_scores(X, C)
        alt = T.epilogue_model(S, (mg * scale).astype(np.float32), C.shape[0])
        assert (alt["total"] == want).all() and not alt["overflow"].any(), (kind, np.unique(alt["total"]))
        assert (m["total"] == 3 - want).all()
