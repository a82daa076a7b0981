"""CPU models of the Yinyang local step and bounds refresh on 64-row tiles (assign_tc.cu MODE 1 / 3 at NKB 9..16,
DESIGN §4k).

At 64 rows both consumer warpgroups hold the same rows, warpgroup g the columns 64g .. 64g + 63 of every 128-column
n-tile.  Checked here:
- MODE 1: each warpgroup keeps its own (largest, second largest) pair of chunk maxima per row and filters with its own
  threshold; the emitters merge the pairs into max(M2_0, M2_1, min(M1_0, M1_1)).  That value is <= the row's second
  best score, so the candidates contain every column within the margin of the second best -- with the best and second
  best in one half, in different halves, or both in the second half above a lower first-half maximum.  The merge the
  MODE 0 emitters use, max(M2_0, M1_1), loses candidates on the last of these;
- MODE 3: the (warp, lane) -> (row, part) map, the quads a part folds (table quads 8 part .. +7 of an n-tile), the
  single overflow emit per row, and the per-lane fold of quad maxima along group ids: with group runs that straddle
  quarters, warpgroups and n-tiles, the atomic-minimum merge of the pieces' bounds equals the bound of every group's
  true maximum.
"""
import numpy as np
import pytest

TR, TN = 64, 128
PAD_SCORE = -65504.0


def lane_row_part(e, lane):
    """consumer warp e (0..7) and lane -> (tile row, part), as in tc_assign_body's consumer branch at T64"""
    g, wq = e >> 2, e & 3
    h = (lane & 3) >> 1
    return wq * 16 + (lane >> 2) + 8 * (lane & 1), 2 * g + h


# ------------------------------------------------------------------------------------------- MODE 1
def lane_columns(g, t):
    """the 16 columns of an n-tile lane t (0..3 in its quad) of warpgroup g holds for each of its two rows"""
    return np.array([64 * g + 8 * j + 2 * t + e for j in range(8) for e in range(2)])


def warpgroup_pass(v, g, margin):
    """warpgroup g's epilogue over one row's scores v (n-tiles of 128 columns): the running pair (M1, M2) merged from the
    quad's four chunk maxima per n-tile, and the entries (chunk maximum, recorded columns) of its four lanes, each
    recorded against the warpgroup's own running threshold M2 - margin"""
    M1 = M2 = -np.inf
    entries = []
    for n in range(len(v) // TN):
        cols = [TN * n + lane_columns(g, t) for t in range(4)]
        cm = [float(v[c].max()) for c in cols]
        a1, a2 = max(cm[0], cm[1]), min(cm[0], cm[1])          # lanes t, t ^ 1
        b1, b2 = max(cm[2], cm[3]), min(cm[2], cm[3])          # the partner pair (xor 2)
        q1, q2 = max(a1, b1), max(min(a1, b1), max(a2, b2))
        M2 = max(M2, q2, min(M1, q1))
        M1 = max(M1, q1)
        thr = M2 - margin
        for t in range(4):
            rec = cols[t][v[cols[t]] >= thr]
            if len(rec):
                entries.append((cm[t], rec))
    return M1, M2, entries


def candidates(v, margin, merge):
    """the emitters' candidate set of one row at 64-row tiles with the given merge of the two warpgroups' pairs"""
    (m10, m20, e0), (m11, m21, e1) = warpgroup_pass(v, 0, margin), warpgroup_pass(v, 1, margin)
    Mf = merge(m10, m20, m11, m21)
    thr = Mf - margin
    cand = set()
    for cm, rec in e0 + e1:
        if cm >= thr:
            cand.update(int(c) for c in rec)
    return cand, Mf


def merge_split(m10, m20, m11, m21):
    return max(m20, m21, min(m10, m11))


def merge_mode0(m10, m20, m11, m21):      # what the MODE 0 emitters do with FIN_M2 in place of FIN_M of warpgroup 0
    return max(m20, m11)


def place(v, n, half, offset):
    """column of n-tile n in warpgroup `half`'s 64 columns"""
    return TN * n + 64 * half + offset


def adversarial_row(kind, rng, nt=4):
    """scores of one row: a best B and a second best S = B - 3 margins apart (margin 1), everything else far below.
    'same': both in the first half; 'split': best in the first, second in the second half; 'second_half': both in the
    second half while the first half holds a maximum F below S (the only shape where max(M2_0, M1_1) = B)"""
    v = rng.standard_normal(TN * nt) - 40.0
    B, S = 10.0, 7.0
    n1, n2 = int(rng.integers(0, nt)), int(rng.integers(0, nt))
    o1, o2 = rng.choice(64, 2, replace=False)
    if kind == "same":
        v[place(v, n1, 0, o1)], v[place(v, n2, 0, o2)] = B, S
    elif kind == "split":
        v[place(v, n1, 0, o1)], v[place(v, n2, 1, o2)] = B, S
    elif kind == "split_rev":
        v[place(v, n1, 1, o1)], v[place(v, n2, 0, o2)] = B, S
    else:
        v[place(v, n1, 1, o1)], v[place(v, n2, 1, o2)] = B, S
        v[place(v, int(rng.integers(0, nt)), 0, int(rng.integers(0, 64)))] = 5.0     # first-half maximum F < S
    return v


def true_set(v, margin):
    """the candidates the row's own second best gives: every column within the margin of it"""
    s2 = np.sort(v)[-2]
    return set(np.flatnonzero(v >= s2 - margin).tolist()), s2


@pytest.mark.parametrize("kind", ["same", "split", "split_rev", "second_half", "random", "ties"])
def test_split_column_second_best_bound(kind):
    rng = np.random.default_rng(len(kind))
    for _ in range(200):
        if kind == "random":
            v = rng.standard_normal(TN * int(rng.integers(1, 6)))
        elif kind == "ties":
            v = np.round(rng.standard_normal(TN * int(rng.integers(1, 6))) * 2) / 2
        else:
            v = adversarial_row(kind, rng)
        margin = 1.0
        want, s2 = true_set(v, margin)
        got, Mf = candidates(v, margin, merge_split)
        assert Mf <= s2, (kind, Mf, s2)
        assert want <= got, (kind, sorted(want - got))


def test_mode0_merge_misses_the_second_best():
    """both best and second best in the second warpgroup's half above a lower first-half maximum: max(M2_0, M1_1) is the
    best score, so the second best (3 margins below) is filtered out"""
    rng = np.random.default_rng(7)
    v = adversarial_row("second_half", rng)
    want, s2 = true_set(v, 1.0)
    got, Mf = candidates(v, 1.0, merge_mode0)
    assert Mf > s2
    assert not want <= got
    got_ok, _ = candidates(v, 1.0, merge_split)
    assert want <= got_ok


# ------------------------------------------------------------------------------------------- MODE 3
def test_part_map_quads_and_single_overflow_emit():
    seen = {}
    for e in range(8):
        for lane in range(32):
            row, part = lane_row_part(e, lane)
            assert (row, part) not in seen
            seen[(row, part)] = (e, lane)
    assert len(seen) == 256
    # part 2g + h = columns 64g + 32h .. +31 = table quads 8 part .. +7 of the n-tile; the kernel loads them as the uint4s
    # n * 8 + 2 part and + 1 of yy_qgroup (4 group ids each)
    for n in (0, 1, 5):
        for part in range(4):
            quads = n * 32 + 8 * part + np.arange(8)
            assert (quads // 4).tolist() == [n * 8 + 2 * part] * 4 + [n * 8 + 2 * part + 1] * 4
    # the overflow emit (kpart == 0) lists every row exactly once
    emit_rows = [r for (r, part) in seen if part == 0]
    assert sorted(emit_rows) == list(range(TR))


def yy_layout(sizes):
    """tc_yy_layout_host: groups padded to whole quads, table rows -> centroid (-1 = padding), group of every quad"""
    perm, qgroup = [], []
    c = 0
    for g, sz in enumerate(sizes):
        if sz == 0:
            continue
        padded = (sz + 3) // 4 * 4
        perm += list(range(c, c + sz)) + [-1] * (padded - sz)
        qgroup += [g] * (padded // 4)
        c += sz
    nt3 = max(1, (len(perm) + TN - 1) // TN)
    perm += [-1] * (nt3 * TN - len(perm))
    qgroup += [-1] * (nt3 * TN // 4 - len(qgroup))
    return np.array(perm), np.array(qgroup), nt3


def bound(run, xa2=5.0e4, E=0.25):
    """the L2 bound of yy_fold_groups (in s units): non-increasing in the group maximum"""
    t = xa2 - 2.0 * (run + E)
    return np.sqrt(t) if t > 0 else 0.0


def fold(qm, gq, G, gown, out):
    """yy_fold_groups: one lane's quad maxima folded along its group ids, each finished run merged with a minimum"""
    run = qm[0]
    for i in range(1, len(qm) + 1):
        if i == len(qm) or gq[i] != gq[i - 1]:
            g = gq[i - 1]
            if 0 <= g < G and g != gown:
                out[g] = min(out[g], bound(run))
            if i < len(qm):
                run = qm[i]
        else:
            run = max(run, qm[i])


def refresh_row(v_table, qgroup, nt3, G, gown, quads_per_lane):
    """one row's bounds: every lane (64-row tiles: 4 parts of 8 quads; 128-row: 2 halves of 16) of every n-tile folds
    its quads"""
    out = np.full(G, np.inf)
    nparts = 32 // quads_per_lane
    for n in range(nt3):
        for part in range(nparts):
            q0 = n * 32 + part * quads_per_lane
            cols = v_table[4 * q0: 4 * (q0 + quads_per_lane)].reshape(quads_per_lane, 4)
            fold(cols.max(axis=1), qgroup[q0:q0 + quads_per_lane], G, gown, out)
    return out


SIZES = {
    "straddle": [1, 2, 3, 5, 31, 33, 64, 100, 129, 7, 300, 2, 40],
    "one_big": [700],
    "singletons": [1] * 90,
    "with_empty": [9, 0, 70, 0, 1, 200, 3],
}


@pytest.mark.parametrize("kind", list(SIZES))
def test_fold_merges_to_the_true_group_bound(kind):
    rng = np.random.default_rng(len(kind))
    sizes = SIZES[kind]
    G = len(sizes)
    perm, qgroup, nt3 = yy_layout(sizes)
    K = int(sum(sizes))
    # runs of several groups must cross quarter (32 columns), warpgroup (64) and n-tile (128) boundaries
    if kind == "straddle":
        starts = np.cumsum([0] + [(s + 3) // 4 * 4 for s in sizes])
        ends = starts[1:] - 1
        crosses = [(a // b) != (e // b) for a, e in zip(starts[:-1], ends) for b in (32, 64, 128)]
        assert sum(crosses) >= 6
    for trial in range(20):
        scores = rng.standard_normal(K) * 50.0 + rng.standard_normal() * 10.0
        gown = int(rng.integers(0, G))
        v_table = np.where(perm >= 0, scores[np.maximum(perm, 0)], PAD_SCORE)
        got64 = refresh_row(v_table, qgroup, nt3, G, gown, 8)
        got128 = refresh_row(v_table, qgroup, nt3, G, gown, 16)
        gof = np.repeat(np.arange(G), sizes)
        for g in range(G):
            if g == gown or sizes[g] == 0:
                assert got64[g] == np.inf
                continue
            want = bound(scores[gof == g].max())
            assert got64[g] == want, (kind, g)
            assert got128[g] == want, (kind, g)
