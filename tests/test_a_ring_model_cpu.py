"""CPU model of the A-operand ring of `assign_tc.cu::tc_assign_kernel` (no GPU needed).  The model restates the kernel's
index arithmetic step by step, so a mistake in it shows up here.

The converters fill the A region K-block by K-block into a ring of `a_slots(nkb)` slots: running K-block g goes to slot
g % S, its waits use phase (g / S) & 1.  Each slot has a FULL barrier (one arrival per converter warp) and a FREE
barrier (one arrival per consumer warp).  A segment (one fill of the tile's A operand) also writes one entry of the
norms ring, read by every consumer warp in the segment's first n-tile; the consumers release the segment's slots in its
last n-tile, each as soon as the wgmma group that reads it has retired.

Under random interleavings of the 4 converter warps and the 8 consumer warps, for every NKB 1..8 with the kernel's own
ring depths (parsed from the source), the model checks that
- no slot or norms entry is overwritten before every consumer warp has read it;
- every read sees the K-block / segment it expects;
- each wait passes in exactly the barrier phase it is meant for (never a phase later);
- nothing deadlocks.
"""
import os
import random
import re

import pytest

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kmcuda_b200", "csrc", "assign_tc.cu")
N_CONV, N_EPI, MAX_NKB = 4, 8, 8


def _ternary_chain(expr, nkb):
    """evaluates `c1 ? v1 : c2 ? v2 : ... : v` (conditions on nkb, integer values)"""
    parts = [s.strip() for s in re.split(r"[?:]", expr)]
    env = {"nkb": nkb, "MAX_NKB": MAX_NKB}
    for i in range(0, len(parts) - 1, 2):
        if eval(parts[i], {}, env):
            return int(eval(parts[i + 1], {}, env))
    return int(eval(parts[-1], {}, env))


def ring_depths(nkb):
    src = open(SRC).read()
    m = re.search(r"constexpr int a_slots\(int nkb\) \{ return (.*?); \}", src)
    assert m, "a_slots() not found in assign_tc.cu"
    slots = _ternary_chain(m.group(1), nkb)
    assert re.search(r"constexpr int norm_depth\(int nkb\) \{ return a_slots\(nkb\) / nkb \+ 1; \}", src)
    return slots, slots // nkb + 1


class Barrier:
    def __init__(self, count):
        self.count, self.pending, self.phases = count, count, 0   # phases = completed phases

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phases += 1
            self.pending = self.count

    def passes(self, parity):   # mbarrier.try_wait.parity: the phase with this parity has completed
        return (self.phases & 1) != parity


def converter(w, st, segs, nkb, S, ND):
    """one converter warp: the kernel's `as` / `aph` counters"""
    as_, aph, g = 0, 0, 0
    for f in range(len(segs)):
        for kb in range(nkb):
            yield ("wait", st["free"][as_], aph ^ 1)
            # this is use (g // S) of the slot: every consumer warp has released use (g // S) - 1, and no later one
            assert st["free"][as_].phases == g // S, ("FREE phase", nkb, g)
            prev = st["slot"][as_][w]
            if prev is not None:
                assert st["slot_reads"].get((as_, prev), 0) == N_EPI, ("slot overwritten before it was read", nkb, as_, prev)
            st["slot"][as_][w] = g
            yield ("step",)
            if kb == nkb - 1:
                e = f % ND
                prevf = st["norms"][e][w]
                if prevf is not None:
                    assert st["norm_reads"].get((e, prevf), 0) == N_EPI, ("norms overwritten before read", nkb, e, prevf)
                st["norms"][e][w] = f
                yield ("step",)
            st["full"][as_].arrive()
            as_ += 1
            if as_ == S:
                as_, aph = 0, aph ^ 1
            g += 1


def consumer(st, segs, nkb, S, ND):
    """one consumer warp: the kernel's `a0` / `aph0` and per-K-block slot arithmetic"""
    a0, aph0 = 0, 0
    for f, nt in enumerate(segs):
        for j in range(nt):
            need_a, free_a = j == 0, j == nt - 1
            sa_prev = None
            for kb in range(nkb):
                wrap = a0 + kb >= S
                sa = a0 + kb - S if wrap else a0 + kb
                g = f * nkb + kb
                assert sa == g % S and (aph0 ^ wrap) == (g // S) & 1, ("slot / phase arithmetic", nkb, g)
                if need_a:
                    yield ("wait", st["full"][sa], aph0 ^ 1 if wrap else aph0)
                    assert st["full"][sa].phases == g // S + 1, ("FULL phase", nkb, g)
                    assert st["slot"][sa] == [g] * N_CONV, ("slot content", nkb, g, st["slot"][sa])
                    st["slot_reads"][(sa, g)] = st["slot_reads"].get((sa, g), 0) + 1
                    yield ("step",)
                else:
                    assert st["slot"][sa] == [g] * N_CONV, ("slot refilled while still in use", nkb, g)
                if kb > 0 and free_a:
                    st["free"][sa_prev].arrive()
                    yield ("step",)
                sa_prev = sa
            if free_a:
                st["free"][sa_prev].arrive()
                yield ("step",)
            if need_a:   # the epilogue of the segment's first n-tile reads its norms (after the releases above)
                e = f % ND
                assert st["norms"][e] == [f] * N_CONV, ("norms content", nkb, f, st["norms"][e])
                st["norm_reads"][(e, f)] = st["norm_reads"].get((e, f), 0) + 1
                yield ("step",)
            if free_a:
                a0 += nkb
                if a0 >= S:
                    a0, aph0 = a0 - S, aph0 ^ 1


def simulate(nkb, segs, seed):
    S, ND = ring_depths(nkb)
    st = {"full": [Barrier(N_CONV) for _ in range(S)], "free": [Barrier(N_EPI) for _ in range(S)],
          "slot": [[None] * N_CONV for _ in range(S)], "norms": [[None] * N_CONV for _ in range(ND)],
          "slot_reads": {}, "norm_reads": {}}
    agents = [converter(w, st, segs, nkb, S, ND) for w in range(N_CONV)] + [consumer(st, segs, nkb, S, ND)
                                                                            for _ in range(N_EPI)]
    nxt = [next(a) for a in agents]
    rng = random.Random(seed)
    while agents:
        ready = [i for i, x in enumerate(nxt) if x[0] == "step" or x[1].passes(x[2])]
        assert ready, ("deadlock", nkb, segs)
        i = rng.choice(ready)
        try:
            nxt[i] = next(agents[i])
        except StopIteration:
            del agents[i], nxt[i]
    assert all(v == N_EPI for v in st["slot_reads"].values())
    assert len(st["slot_reads"]) == len(segs) * nkb and len(st["norm_reads"]) == len(segs)


@pytest.mark.parametrize("nkb", range(1, MAX_NKB + 1))
def test_a_ring_interleavings(nkb):
    rng = random.Random(nkb)
    for trial in range(60):
        segs = [rng.choice([1, 1, 2, 3, 8]) for _ in range(rng.randint(1, 9))]   # n-tiles per segment
        simulate(nkb, segs, seed=1000 * nkb + trial)


@pytest.mark.parametrize("nkb", range(1, MAX_NKB + 1))
def test_a_ring_depths(nkb):
    S, ND = ring_depths(nkb)
    assert nkb <= S <= MAX_NKB           # a whole tile fits; the barrier arrays have MAX_NKB entries
    assert ND * nkb > S                  # the converters run fewer than ND segments ahead of the norms' readers
    if nkb <= 4:
        assert S > nkb                   # D <= 256: part of the next tile is converted during the current one
