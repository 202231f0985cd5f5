"""CPU emulation of the stage / phase schedule of ss_gemm_kernel (csrc/gvd_wgmma.cu).

Every actor of the kernel runs as a generator under a random scheduler: one producer thread and eight consumer warps (the two
warpgroups), plus the asynchronous TMA transfers, which land in any order.  The model also covers clusters of CTAs that share the W
slice (each loads a share and multicasts it, `empty` counts the consumer warps of every CTA); ncl = 2 is the variant measured in
DESIGN.md §3.  The mbarriers follow the PTX rules: a phase completes when its pending arrivals and its transaction bytes both reach zero,
the byte count may go below zero before the expecting arrival, and try_wait.parity(P) succeeds once the phase of parity P has completed.  The test checks, for K slice counts around the ring depth:
- the schedule ends (no deadlock) in every interleaving tried;
- a consumer warp only reads a stage whose parts (A slice, every CTA's share of the W slice) all hold the slice it expects;
- no transfer writes into a stage while a consumer warp of the destination CTA still reads it (between its wait on `full` and its
  arrival on `empty` after wgmma_wait<1>, or its final wgmma_wait<0>)."""
import random

import pytest

ST = 4                      # WG_STAGES
WARPS = 8                   # consumer warps per CTA
A_BYTES, W_BYTES = 128 * 128, 128 * 128


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _check(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0
        self.pending -= 1
        self._check()

    def expect_tx(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._check()

    def done(self, parity):
        return (self.phase & 1) != parity            # the phase of this parity has completed


def emulate(nk, ncl, seed):
    rng = random.Random(seed)
    full = [[Bar(1) for _ in range(ST)] for _ in range(ncl)]
    empty = [[Bar(ncl * WARPS) for _ in range(ST)] for _ in range(ncl)]
    slot = {}                                          # (cta, stage, part) -> slice held
    readers = {(c, s): set() for c in range(ncl) for s in range(ST)}
    transfers = []                                     # (dst cta, stage, part, slice, bytes)

    def producer(c):
        part = W_BYTES // ncl
        for i in range(nk):
            s = i % ST
            yield lambda: empty[c][s].done(((i // ST) & 1) ^ 1)
            full[c][s].expect_tx(A_BYTES + W_BYTES)
            transfers.append((c, s, "A", i, A_BYTES))
            for dst in range(ncl):                     # multicast of this CTA's share of the W slice
                transfers.append((dst, s, "W%d" % c, i, part))

    def consumer(c, w):
        def issue(i):
            s = i % ST
            yield lambda: full[c][s].done((i // ST) & 1)
            for part in ["A"] + ["W%d" % r for r in range(ncl)]:
                assert slot.get((c, s, part)) == i, (c, s, part, slot.get((c, s, part)), i)
            readers[(c, s)].add(w)

        def retire(i, arrive=True):
            s = i % ST
            readers[(c, s)].discard(w)
            if arrive:
                for dst in range(ncl):                 # local arrival, then the partner's barrier
                    empty[(c + dst) % ncl][s].arrive()

        for i in range(0, nk, 2):
            yield from issue(i)
            if i > 0:
                retire(i - 1)
            if i + 1 < nk:
                yield from issue(i + 1)
                retire(i)
        retire(nk - 1, arrive=False)

    actors = [producer(c) for c in range(ncl)] + [consumer(c, w) for c in range(ncl) for w in range(WARPS)]
    waits = [None] * len(actors)
    live = set(range(len(actors)))
    steps = 0
    while live or transfers:
        ready = [a for a in live if waits[a] is None or waits[a]()]
        choices = [("actor", a) for a in ready] + [("tma", k) for k in range(len(transfers))]
        assert choices, "deadlock: nk=%d ncl=%d seed=%d" % (nk, ncl, seed)
        kind, k = rng.choice(choices)
        if kind == "tma":
            c, s, part, i, nbytes = transfers.pop(k)
            assert not readers[(c, s)], "slice %d overwrites stage %d of CTA %d while it is read" % (i, s, c)
            slot[(c, s, part)] = i
            full[c][s].complete_tx(nbytes)
        else:
            try:
                waits[k] = next(actors[k])
            except StopIteration:
                live.discard(k)
        steps += 1
        assert steps < 200000
    # every expected phase completed: full barriers once per slice of each stage
    for c in range(ncl):
        for s in range(ST):
            assert full[c][s].phase == len(range(s, nk, ST))


@pytest.mark.parametrize("ncl", [1, 2])
@pytest.mark.parametrize("nk", [1, 2, 3, 4, 5, 7, 8, 9, 16, 17])
def test_ss_pipeline_schedule(nk, ncl):
    for seed in range(12):
        emulate(nk, ncl, seed)
