"""CPU model of the Lloyd / Yinyang candidate epilogue of `assign_tc.cu::tc_assign_kernel` (MODE 0 / 1), which runs on
the wgmma m64n128 accumulator fragment as it lands (no GPU needed).

The model restates three things of the kernel:

* the fragment layout: warp w of the 8 consumer warps holds tile rows 16 w .. 16 w + 15; lane l holds rows
  R0 = 16 w + l // 4 and R1 = R0 + 8 at columns 8 j + 2 t + e (t = l % 4, j < 16, e < 2).  Mask bit b = 2 j + e of row
  R0 / R1 stands for column 8 j + 2 t + e;
* the epilogue per n-tile: the lane's chunk maximum over its 32 values, a quad all-reduce into the running ROW maximum,
  thr = M - margin, a 32-bit mask per row, and one list entry per n-tile in which either row has a candidate;
* the emitter's decode of an entry, col = n * 128 + 8 (b >> 1) + 2 t + (b & 1), over the 4 lanes of the row's quad.

It checks that the (lane, bit) map is a bijection of the 128 x 128 n-tile, that every row's decoded candidate set
contains its argmax (random scores with ties, ragged last n-tile), and that the masks built with full-row thresholds are
subsets of the masks built with the half-row thresholds the kernel used before (regrouped fragment).
"""
import numpy as np
import pytest

TM = TN = 128


def lane_bit_to_cell(w, lane, hh, b):
    """(tile row, n-tile column) of mask bit b of row hh (0: R0, 1: R1) held by lane `lane` of consumer warp w"""
    t = lane & 3
    row = 16 * w + (lane >> 2) + 8 * hh
    col = 8 * (b >> 1) + 2 * t + (b & 1)
    return row, col


def emitter_lanes(row):
    """the four (list column, hh) the emitter merges for tile row `row` (list column = consumer warp * 32 + lane)"""
    hh = (row >> 3) & 1
    lid0 = (row >> 4) * 32 + (row & 7) * 4
    return [(lid0 + t, t, hh) for t in range(4)]


def decode(n, t, b):
    return n * TN + 8 * (b >> 1) + 2 * t + (b & 1)


def test_lane_bit_map_is_a_bijection_and_decodes_back():
    seen = {}
    for w in range(8):
        for lane in range(32):
            for hh in range(2):
                for b in range(32):
                    cell = lane_bit_to_cell(w, lane, hh, b)
                    assert cell not in seen, "cell %r encoded twice" % (cell,)
                    seen[cell] = (w * 32 + lane, hh, b)
    assert len(seen) == TM * TN
    for (row, col), (lid, hh, b) in seen.items():
        # the emitter finds the cell among the lanes it merges for this row, and decodes the bit back to the column
        lanes = {l: (t, h) for l, t, h in emitter_lanes(row)}
        assert lid in lanes and lanes[lid][1] == hh
        assert decode(0, lanes[lid][0], b) == col
        assert decode(5, lanes[lid][0], b) == 5 * TN + col


def native_masks(S, margin):
    """S: [128 rows, nt * 128] scores of one sample tile.  Returns per row the decoded candidate set and per n-tile the
    masks[row][n] (as column sets, full-row thresholds), replaying the epilogue lane by lane and the emitter."""
    nrows, ncols = S.shape
    nt = ncols // TN
    M = np.full(nrows, -np.inf, np.float32)
    lists = {}                       # lid -> list of (max R0, max R1, mask R0, mask R1, n)
    masks = np.zeros((nrows, nt), dtype=object)
    for n in range(nt):
        blk = S[:, n * TN:(n + 1) * TN]
        # chunk maxima per (lane, row): the lane's 32 columns 8j + 2t + e
        cm = {}
        for w in range(8):
            for lane in range(32):
                t = lane & 3
                cols = np.array([8 * (b >> 1) + 2 * t + (b & 1) for b in range(32)])
                for hh in range(2):
                    r = 16 * w + (lane >> 2) + 8 * hh
                    cm[(w, lane, hh)] = (r, cols, blk[r, cols].max())
        # quad all-reduce -> running row maximum (identical in the quad)
        for w in range(8):
            for lane in range(0, 32, 4):
                for hh in range(2):
                    r = cm[(w, lane, hh)][0]
                    q = max(cm[(w, lane + k, hh)][2] for k in range(4))
                    M[r] = max(M[r], q)
        for w in range(8):
            for lane in range(32):
                mk = []
                for hh in range(2):
                    r, cols, _ = cm[(w, lane, hh)]
                    thr = np.float32(M[r] - margin[r])
                    bits = 0
                    for b in range(32):
                        if blk[r, cols[b]] >= thr:
                            bits |= 1 << b
                    mk.append(bits)
                    masks[r, n] = (masks[r, n] or set()) | {n * TN + cols[b] for b in range(32) if bits >> b & 1}
                if mk[0] | mk[1]:
                    lists.setdefault(w * 32 + lane, []).append(
                        (cm[(w, lane, 0)][2], cm[(w, lane, 1)][2], mk[0], mk[1], n))
    cands = []
    for r in range(nrows):
        thr = np.float32(M[r] - margin[r])
        got = set()
        for lid, t, hh in emitter_lanes(r):
            for ent in lists.get(lid, []):
                if not ent[hh] >= thr:
                    continue
                m = ent[2 + hh]
                for b in range(32):
                    if m >> b & 1:
                        got.add(decode(ent[4], t, b))
        cands.append(got)
    return cands, masks


def halfrow_masks(S, margin):
    """the parent's epilogue on the regrouped fragment: a thread owns one row and one 64-column half of every n-tile and
    keeps the running maximum of that half-row only"""
    nrows, ncols = S.shape
    nt = ncols // TN
    masks = np.zeros((nrows, nt), dtype=object)
    for r in range(nrows):
        for h in range(2):
            M = -np.inf
            for n in range(nt):
                v = S[r, n * TN + 64 * h:n * TN + 64 * h + 64]
                M = max(M, v.max())
                thr = np.float32(M - margin[r])
                sel = {n * TN + 64 * h + c for c in np.nonzero(v >= thr)[0]}
                masks[r, n] = (masks[r, n] or set()) | sel
    return masks


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_candidates_contain_argmax_and_shrink(seed):
    rng = np.random.default_rng(seed)
    K = 3 * TN + 37                                  # ragged last n-tile
    nt = (K + TN - 1) // TN
    # coarse values -> many exact ties; padded columns score the sentinel like the kernel's zero rows
    S = np.round(rng.normal(size=(TM, nt * TN)) * 4).astype(np.float32) / 4
    S += rng.normal(size=(TM, 1)).astype(np.float32) * 8   # per-row offsets, as |x|^2 / 2 gives
    S[:, K:] = -65504.0
    margin = rng.uniform(0.0, 0.6, size=TM).astype(np.float32)
    cands, masks = native_masks(S, margin)
    old = halfrow_masks(S, margin)
    for r in range(TM):
        got = {c for c in cands[r] if c < K}
        vals = S[r, :K]
        best = vals.max()
        # every column within the margin of the row maximum is a candidate, the argmax (and all its ties) included
        want = set(np.nonzero(vals >= np.float32(best - margin[r]))[0].tolist())
        assert int(np.argmax(vals)) in got
        assert want <= got
        for n in range(nt):
            assert (masks[r, n] or set()) <= (old[r, n] or set()), "row %d n-tile %d" % (r, n)

