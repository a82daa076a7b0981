"""CPU models of the k-NN candidate pass on 64-row tiles (assign_tc.cu MODE 2 at NKB 9..16, DESIGN §4j).

At 64 rows both consumer warpgroups hold the same rows, warpgroup g the columns 64g .. 64g + 63 of every 128-column
n-tile.  After the quad regroup (regroup_quad_t64) a thread holds 32 consecutive columns of one row, so a row has four
parts: part 2g + q covers columns 64g + 32q .. +31.  Checked here:
- the (warp, lane) -> (row, part) -> shared-memory slot map is a bijection onto the 256 slots of the [kk][256] scratch,
  and the global slot (table row * 4 + part) one onto the 4 x 128 slots of a table block;
- the quad regroup gives every lane the 32 consecutive columns of its (row, part), and chunk ids n * 4 + part decode
  (expand_kernel) to those columns;
- the four-part thresholds, merged as expand_kernel merges them, contain the true top-kk at every kk <= 16, whether
  the best columns are spread over the parts or all in one of them.
"""
import numpy as np
import pytest

TR = 64


def lane_row_part(e, lane):
    """consumer warp e (0..7) and lane -> (tile row, part), as in tc_assign_body's consumer branch at T64"""
    g, wq = e >> 2, e & 3
    h = (lane & 3) >> 1
    return wq * 16 + (lane >> 2) + 8 * (lane & 1), 2 * g + h


def test_slot_map_is_a_bijection():
    slots, pairs = [], set()
    for e in range(8):
        for lane in range(32):
            row, part = lane_row_part(e, lane)
            assert 0 <= row < TR and 0 <= part < 4
            pairs.add((row, part))
            slots.append(part * TR + row)
    assert sorted(slots) == list(range(256))
    assert len(pairs) == 256
    # the buckets of a row's four parts (knn_select_buckets4): slot row + 64 q
    for row in range(TR):
        assert sorted(part * TR + row for part in range(4)) == [row + 64 * q for q in range(4)]
    # global slots: query tile t is half t & 1 of block t >> 1, table row = t * 64 + row
    for blk in (0, 1, 7):
        ks = [((2 * blk + half) * TR + row) * 4 + part for half in (0, 1) for row in range(TR) for part in range(4)]
        assert sorted(ks) == list(range(blk * 512, blk * 512 + 512))


def regroup_quad_t64(acc):
    """acc[lane][32]: the m64n64 fragment of one warp; returns r[lane][32] as the kernel's shuffle rounds build it"""
    r = np.zeros((32, 32), acc.dtype)
    for lane in range(32):
        t = lane & 3
        for jj in range(4):
            for e2 in range(2):
                got = [None] * 4
                for k in range(4):
                    src = lane ^ k                       # __shfl_xor_sync(v, k): the value partner src computed for c
                    c = (src & 3) ^ k
                    b = {(0, 0): acc[src][jj * 4 + e2], (1, 0): acc[src][jj * 4 + 2 + e2],
                         (0, 1): acc[src][(4 + jj) * 4 + e2], (1, 1): acc[src][(4 + jj) * 4 + 2 + e2]}
                    got[k] = b[(c & 1, c >> 1)]
                for s in range(4):
                    r[lane][8 * jj + 2 * s + e2] = got[s ^ t]
    return r


def test_quad_regroup_gives_each_lane_its_parts_columns():
    # scores of one warp: rows wq*16 .. +15 at the 64 columns of warpgroup g's half; value = 1000 row + column
    for g in (0, 1):
        wq = 2
        acc = np.zeros((32, 32))
        for lane in range(32):
            t = lane & 3
            for j in range(8):
                for hh in range(2):
                    for e in range(2):
                        row = wq * 16 + hh * 8 + (lane >> 2)
                        acc[lane][j * 4 + hh * 2 + e] = 1000 * row + 64 * g + 8 * j + 2 * t + e
        r = regroup_quad_t64(acc)
        for lane in range(32):
            row, part = lane_row_part(4 * g + wq, lane)
            assert part >> 1 == g
            np.testing.assert_array_equal(r[lane], 1000 * row + 32 * part + np.arange(32))


def test_chunk_ids_decode_to_the_parts_columns():
    for n in (0, 1, 2, 3, 77, 16382):
        for g in (0, 1):
            for q in (0, 1):
                cid = n * 4 + 2 * g + q
                p0 = (cid >> 2) * 128 + ((cid >> 1) & 1) * 64 + (cid & 1) * 32
                assert p0 == 128 * n + 64 * g + 32 * q


def two_pass_candidates(v, n_own, kk):
    """one query row's scores v over the table columns (n-tiles 0 .. n_own-1: its own cluster, the rest: other
    clusters), swept as the kernel does at 64-row tiles with a zero margin.  Returns (candidates, merged kth)."""
    nt = len(v) // 128
    part_of = lambda c: (c % 128) // 32
    # pass 1, threshold sweep: buckets (part, n-tile % 4, 4-column group of the part) over the own cluster
    bmax = np.full((4, 32), -np.inf)
    own = np.arange(128 * n_own)
    np.maximum.at(bmax, (part_of(own), 8 * ((own // 128) % 4) + (own % 32) // 4), v[own])
    merged = np.sort(bmax.ravel())[::-1][:kk]             # knn_select_buckets4: every part adopts the merged list
    tops = [list(merged) for _ in range(4)]
    entries = [[] for _ in range(4)]                      # (chunk maximum, recorded columns) per part

    def sweep(n, record, insert):
        for part in range(4):
            cols = np.arange(128 * n + 32 * part, 128 * n + 32 * part + 32)
            if insert:
                for grp in range(8):
                    gm = v[cols[4 * grp:4 * grp + 4]].max()
                    if gm > tops[part][kk - 1]:
                        tops[part] = sorted(tops[part] + [gm], reverse=True)[:kk]
            if record:
                M = tops[part][kk - 1]
                rec = cols[v[cols] >= M]
                if len(rec):
                    entries[part].append((v[cols].max(), rec))

    for n in range(n_own):        # pass 1, recording sweep
        sweep(n, record=True, insert=False)
    for n in range(n_own, nt):    # pass 2: the other clusters' blocks
        sweep(n, record=True, insert=True)
    kth = max(t[kk - 1] for t in tops)                    # expand_kernel: the largest of the parts' kk-th values
    cand = set()
    for part in range(4):
        for cm, rec in entries[part]:
            if cm >= kth:
                cand.update(int(c) for c in rec)
    return cand, kth


@pytest.mark.parametrize("kind", ["random", "one_part", "all_parts", "ties", "pass2"])
def test_four_part_thresholds_contain_the_true_top_kk(kind):
    rng = np.random.default_rng(len(kind))
    for kk in range(1, 17):
        for _ in range(4):
            nt = int(rng.integers(2, 7))
            n_own = int(rng.integers(1, nt))
            v = rng.standard_normal(128 * nt)
            best = 8.0 + rng.random(kk)
            if kind == "one_part":             # the whole top-kk in one part of one n-tile
                n, part = int(rng.integers(0, nt)), int(rng.integers(0, 4))
                v[128 * n + 32 * part + rng.choice(32, kk, replace=False)] = best
            elif kind == "all_parts":          # spread round-robin over the four parts
                for i in range(kk):
                    part, n = i % 4, int(rng.integers(0, nt))
                    v[128 * n + 32 * part + int(rng.integers(0, 32))] = best[i]
            elif kind == "ties":               # many equal scores at the kk-th place
                v = np.round(v * 2) / 2
            elif kind == "pass2":              # the top-kk outside the own cluster only
                v[:128 * n_own] -= 10.0
            cand, kth = two_pass_candidates(v, n_own, kk)
            order = np.sort(v)[::-1]
            assert kth <= order[kk - 1]                     # each part's list holds kk distinct columns
            top = set(np.flatnonzero(v >= order[kk - 1]).tolist())
            assert top <= cand, (kind, kk, sorted(top - cand))
