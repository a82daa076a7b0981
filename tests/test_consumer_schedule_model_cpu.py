"""CPU model of the MODE 0 / 1 pipeline of `assign_tc.cu::tc_assign_kernel` on its 16-warp layout (no GPU needed).  The
model restates every role's schedule step by step, with the ring depths and warp counts parsed from the source:

- TMA producer (warp 3): per n-tile its NKB B stages, then the bias block.
- 4 converter warps: the A ring K-block by K-block; the last K-block of a tile also writes the tile's norms entry.
- 8 consumer warps: a tile starts with the wait for the emitters to have consumed its list parity (tile - 2); per n-tile
  one wgmma group per K-block (A slot + B stage) and one bias group; after issuing K-block kb, wgmma.wait_group 1
  retires K-block kb - 1 and releases its B stage (and, in the tile's last n-tile, its A slot); after the bias group,
  wait_group 0 releases the rest; the first n-tile's epilogue reads the norms entry, every epilogue writes the list
  parity, the last one publishes it.
- 3 emitter warps: thread = row with a stride of 96, so warp 0 reads two rows and arrives on the parity's EMPTY barrier
  only after its second row.

wgmma groups retire in order at random times, independently in each consumer warp.  Under random interleavings, for
NKB 1..8, n-tiles per tile nt in {1, 2, 8}, 1..5 tiles per CTA and a ragged last tile (rows past the end are not read
by the emitters), the model checks that
- no B stage, bias buffer or A slot is overwritten while a group that reads it is in flight, nor released before that
  group has retired;
- no norms entry or list parity is overwritten before its last reader has read it, and every read sees what it expects;
- the emitters read each live row of every tile exactly once;
- each wait passes in exactly the barrier phase it is meant for;
- nothing deadlocks.
"""
import os
import random
import re

import pytest

from test_a_ring_model_cpu import Barrier, ring_depths

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kmcuda_b200", "csrc", "assign_tc.cu")
TM, MAX_NKB = 128, 8


def _const(src, name):
    m = re.search(r"constexpr int %s = (\d+)(?: \* 32)?;" % name, src)
    assert m, name
    return int(m.group(1))


def layout(nkb):
    """(B stages, bias buffers, A slots, norms entries, converter / consumer / emitter warps) as the kernel has them"""
    src = open(SRC).read()
    assert re.search(r"constexpr int b_stages\(int nkb\) \{ return wide_nkb\(nkb\) \? 2 : B_STAGES; \}", src)
    assert re.search(r"constexpr int aug_bufs\(int nkb\) \{ return nkb <= 2 \? 2 : 1; \}", src)
    # the emitters' row walk and their EMPTY arrival after the warp's last row
    assert re.search(r"const int nrows = row0 \+ N_EMIT_WARPS \* 32 < TM \? 2 : 1;", src)
    assert re.search(r"const int row = row0 \+ ri \* N_EMIT_WARPS \* 32;", src)
    assert re.search(r"if \(ri == nrows - 1\) \{\s*__syncwarp\(\);\s*if \(lane == 0\) ptx::mbar_arrive\(&bars\[BAR_EMIT_EMPTY \+ par\]\);", src)
    assert re.search(r"ptx::mbar_init\(&bars\[BAR_EMIT_EMPTY \+ s\], N_EMIT_WARPS\);", src)
    bst = 2 if nkb > _const(src, "WIDE_NKB") else _const(src, "B_STAGES")
    slots, nd = ring_depths(nkb)
    n_emit, n_conv, n_epi = _const(src, "N_EMIT_WARPS"), _const(src, "N_CONV_WARPS"), _const(src, "N_EPI_WARPS")
    assert n_emit + n_conv + n_epi + 1 == _const(src, "N_THREADS")   # + the producer warp
    return bst, 2 if nkb <= 2 else 1, slots, nd, n_conv, n_epi, n_emit


class Sim:
    def __init__(self, nkb, nt, ntiles, last_rows):
        self.nkb, self.nt, self.ntiles, self.last_rows = nkb, nt, ntiles, last_rows
        self.BST, self.AUGB, self.S, self.ND, self.NC, self.NE, self.NM = layout(nkb)
        B = lambda n, c: [Barrier(c) for _ in range(n)]
        self.b_full, self.b_empty = B(self.BST, 1), B(self.BST, self.NE)
        self.aug_full, self.aug_empty = B(2, 1), B(2, self.NE)
        self.a_full, self.a_free = B(self.S, self.NC), B(self.S, self.NE)
        self.emit_full, self.emit_empty = B(2, self.NE), B(2, self.NM)
        self.content, self.readers = {}, {}
        self.norms = [[None] * self.NC for _ in range(self.ND)]
        self.norm_reads, self.lists, self.row_reads = {}, [[None] * self.NE for _ in range(2)], {}
        self.emit_done = {}
        self.queue = [[] for _ in range(self.NE)]
        self.retired = [0] * self.NE          # groups retired per consumer warp (in order)

    def live_rows(self, t):
        return self.last_rows if t == self.ntiles - 1 else TM

    def producer(self):
        g = ac = 0
        for _ in range(self.ntiles * self.nt):
            for _kb in range(self.nkb):
                s = g % self.BST
                yield ("wait", self.b_empty[s], ((g // self.BST) & 1) ^ 1)
                assert self.b_empty[s].phases == g // self.BST, ("B_EMPTY phase", g)
                assert not self.readers.get(("B", s)), ("B stage refilled while a group reads it", g)
                self.content[("B", s)] = g
                self.b_full[s].arrive()
                g += 1
                yield ("step",)
            a = ac % self.AUGB
            yield ("wait", self.aug_empty[a], ((ac // self.AUGB) & 1) ^ 1)
            assert self.aug_empty[a].phases == ac // self.AUGB, ("AUG_EMPTY phase", ac)
            assert not self.readers.get(("AUG", a)), ("bias buffer refilled while a group reads it", ac)
            self.content[("AUG", a)] = ac
            self.aug_full[a].arrive()
            ac += 1
            yield ("step",)

    def converter(self, w):
        g = 0
        for t in range(self.ntiles):
            for kb in range(self.nkb):
                s = g % self.S
                yield ("wait", self.a_free[s], ((g // self.S) & 1) ^ 1)
                assert self.a_free[s].phases == g // self.S, ("A_FREE phase", g)
                assert not self.readers.get(("A", s)), ("A slot overwritten while a group reads it", g)
                self.content[("A", s, w)] = g
                yield ("step",)
                if kb == self.nkb - 1:
                    e = t % self.ND
                    prev = self.norms[e][w]
                    if prev is not None:
                        assert self.norm_reads.get(prev, 0) == self.NE, ("norms overwritten before read", prev)
                    self.norms[e][w] = t
                    yield ("step",)
                self.a_full[s].arrive()
                g += 1

    def emitter(self, w):
        rows = list(range(w * 32, TM, self.NM * 32))   # thread = row: first row of each lane group
        for ti in range(self.ntiles):
            par = ti & 1
            yield ("wait", self.emit_full[par], (ti >> 1) & 1)
            assert self.emit_full[par].phases == (ti >> 1) + 1, ("EMIT_FULL phase", ti)
            for r0 in rows:
                for r in range(r0, r0 + 32):
                    if r < self.live_rows(ti):
                        assert self.lists[par] == [ti] * self.NE, ("lists content", ti, r, self.lists[par])
                        self.row_reads[(ti, r)] = self.row_reads.get((ti, r), 0) + 1
                yield ("step",)
            self.emit_done[ti] = self.emit_done.get(ti, 0) + 1
            self.emit_empty[par].arrive()

    def consumer(self, w):
        nkb, nt, BST, AUGB, S, ND = self.nkb, self.nt, self.BST, self.AUGB, self.S, self.ND
        q = self.queue[w]
        bs = bph = ac = a0 = aph0 = 0
        issued = 0                                   # groups issued by this warp
        g = 0                                        # B K-blocks issued

        def issue(res, expect):
            nonlocal issued
            for r in res:
                self.readers.setdefault(r, set()).add(w)
            q.append((res, expect))
            issued += 1

        def release_b(stage, gi):
            assert self.content[("B", stage)] == gi, ("released B stage holds", gi)
            self.b_empty[stage].arrive()

        for ti in range(self.ntiles):
            par = ti & 1
            yield ("wait", self.emit_empty[par], ((ti >> 1) & 1) ^ 1)
            assert self.emit_empty[par].phases == ti >> 1, ("EMIT_EMPTY phase", ti)
            prev = self.lists[par][w]
            if prev is not None:
                assert self.emit_done.get(prev, 0) == self.NM, ("lists overwritten before emitted", prev)
            for n in range(nt):
                need_a, free_a = n == 0, n == nt - 1
                prev_kb = None
                for kb in range(nkb):
                    wrap = a0 + kb >= S
                    sa = a0 + kb - S if wrap else a0 + kb
                    ga = ti * nkb + kb
                    if need_a:
                        yield ("wait", self.a_full[sa], aph0 ^ 1 if wrap else aph0)
                        assert self.a_full[sa].phases == ga // S + 1, ("A_FULL phase", ga)
                    assert all(self.content.get(("A", sa, c)) == ga for c in range(self.NC)), ("A slot content", ga)
                    yield ("wait", self.b_full[bs], bph)
                    assert self.b_full[bs].phases == g // BST + 1, ("B_FULL phase", g)
                    assert self.content[("B", bs)] == g, ("B stage content", g)
                    issue([("A", sa), ("B", bs)], {("B", bs): g, ("A", sa): ga})
                    yield ("step",)
                    if kb > 0:
                        yield ("wgwait", w, 1)
                        assert self.retired[w] >= issued - 1
                        pstage, pg, psa = prev_kb
                        release_b(pstage, pg)
                        if free_a:
                            self.a_free[psa].arrive()
                        yield ("step",)
                    prev_kb = (bs, g, sa)
                    g += 1
                    bs += 1
                    if bs == BST:
                        bs, bph = 0, bph ^ 1
                buf, aph = ac % AUGB, (ac // AUGB) & 1
                yield ("wait", self.aug_full[buf], aph)
                assert self.aug_full[buf].phases == ac // AUGB + 1, ("AUG_FULL phase", ac)
                issue([("AUG", buf)], {("AUG", buf): ac})
                yield ("wgwait", w, 0)
                assert self.retired[w] == issued
                pstage, pg, psa = prev_kb
                release_b(pstage, pg)
                self.aug_empty[buf].arrive()
                if free_a:
                    self.a_free[psa].arrive()
                    a0 += nkb
                    if a0 >= S:
                        a0, aph0 = a0 - S, aph0 ^ 1
                ac += 1
                if need_a:
                    e = ti % ND
                    assert self.norms[e] == [ti] * self.NC, ("norms content", ti, self.norms[e])
                    self.norm_reads[ti] = self.norm_reads.get(ti, 0) + 1
                self.lists[par][w] = ti
                yield ("step",)
            self.emit_full[par].arrive()

    def retire(self, w):
        res, expect = self.queue[w].pop(0)
        for r in res:
            self.readers[r].discard(w)
        for r, v in expect.items():
            if r[0] == "A":
                assert all(self.content[("A", r[1], c)] == v for c in range(self.NC)), ("A slot overwritten in flight", v)
            else:
                assert self.content[r] == v, ("operand overwritten while in flight", r, v)
        self.retired[w] += 1

    def run(self, seed):
        agents = ([self.producer()] + [self.converter(w) for w in range(self.NC)] +
                  [self.consumer(w) for w in range(self.NE)] + [self.emitter(w) for w in range(self.NM)])
        nxt = [next(a) for a in agents]
        rng = random.Random(seed)

        def ready(x):
            if x[0] == "step":
                return True
            if x[0] == "wgwait":
                return len(self.queue[x[1]]) <= x[2]
            return x[1].passes(x[2])

        while agents or any(self.queue):
            choices = [("a", i) for i, x in enumerate(nxt) if ready(x)] + [("r", w) for w in range(self.NE) if self.queue[w]]
            assert choices, ("deadlock", self.nkb, self.nt, self.ntiles)
            kind, i = rng.choice(choices)
            if kind == "r":
                self.retire(i)
                continue
            try:
                nxt[i] = next(agents[i])
            except StopIteration:
                del agents[i], nxt[i]
        assert all(self.norm_reads.get(t) == self.NE for t in range(self.ntiles))
        for t in range(self.ntiles):
            assert sorted(r for (tt, r) in self.row_reads if tt == t) == list(range(self.live_rows(t)))
        assert all(v == 1 for v in self.row_reads.values())


@pytest.mark.parametrize("nkb", range(1, MAX_NKB + 1))
@pytest.mark.parametrize("nt", [1, 2, 8])
def test_consumer_schedule_interleavings(nkb, nt):
    rng = random.Random(100 * nkb + nt)
    for trial in range(10):
        Sim(nkb, nt, rng.randint(1, 5), rng.choice([TM, 1, 33, 97])).run(seed=10000 * nkb + 100 * nt + trial)


def test_emitter_rows_cover_the_tile_once():
    *_, n_emit = layout(1)
    rows = [r0 + lane for w in range(n_emit) for r0 in range(w * 32, TM, n_emit * 32) for lane in range(32)]
    assert sorted(rows) == list(range(TM))
