"""Discrete-event model of the stage ring of the tensor-core conv kernel (csrc/conv_tc.cu), persistent and split-K.

Actors: NP producer threads (thread 0 also issues the weight TMA) and two consumer warpgroups of four warps, interleaved
in a random order.  One CTA computes `tiles` output tiles of `chunks` K chunks each; the global chunk counter
g = j * chunks + it runs on across tiles, so stage g % STAGES and phase g // STAGES carry over tile boundaries.  With
`early` the B tiles of the first min(STAGES, tiles * chunks) chunks are requested before anything else (constant weights
fetched ahead of the grid dependency wait).  The producer threads keep the row tables of tiles j and j + 1 in two buffers;
as in the kernel, each gathers two half chunks ahead of its stores, and the gather of the first half of every tile after
the first passes a producer-only barrier and writes the table of tile j + 1, before the last chunk of tile j - 1 is stored.

mbarriers are waited on by parity, as the hardware does, and every successful wait checks that the barrier is at exactly
the phase the waiter means.  MMAs are asynchronous: a stage is "being read" from the issue of its MMAs until the wait
that covers them (wgmma.wait_group 1 inside a tile, 0 at its end).  Checked: no stage is overwritten while it is being
read, every MMA reads the A and B of the chunk it expects, every gather reads the row table of its own tile, the
persistent finish touches no stage, the split-K finish (which stages its tile in the operand stages) runs only when no
stage is being read and the producer has stored its last chunk, and the run terminates (no deadlock).

HaloSim models the halo kernel's two rings the same way (see its docstring).

    python scripts/conv_tc_protocol_sim.py        # a quick sweep
"""
import random


class Barrier:
    def __init__(self, count):
        self.count, self.pending, self.phases = count, count, 0

    def arrive(self, n=1):
        self.pending -= n
        assert self.pending >= 0, "more arrivals than the barrier's count"
        if self.pending == 0:
            self.phases += 1
            self.pending = self.count

    def ready(self, phase):              # try_wait.parity(phase & 1)
        return (self.phases & 1) != (phase & 1)


class Sim:
    def __init__(self, tiles, chunks, seed, stages=4, early=False, splitk=False, nprod=2, release_last=True):
        assert not splitk or tiles <= 1, "a split-K CTA computes one tile"
        self.J, self.C, self.S, self.NP = tiles, chunks, stages, nprod
        self.splitk, self.release_last = splitk, release_last      # release_last=False: a broken kernel, for the test
        self.rng = random.Random(seed)
        self.a_full = [Barrier(nprod) for _ in range(stages)]
        self.b_full = [Barrier(1) for _ in range(stages)]
        self.s_free = [Barrier(8) for _ in range(stages)]
        self.a_content = [None] * stages
        self.b_content = [None] * stages
        self.readers = [set() for _ in range(stages)]
        self.rows = [0, 1 if tiles > 1 else None]      # row-table buffers, written before the first barrier
        self.rows_readers = [set(), set()]
        self.pbar = {"arrived": 0, "gen": 0}           # producer-only named barrier
        self.npre = min(stages, tiles * chunks) if early else 0
        self.stored = 0 if tiles * chunks else nprod    # producer threads done with their last chunk
        self.staging = 0                               # consumer warpgroups at the split-K staging barrier
        for g in range(self.npre):                     # before the dependency wait: nothing can be in a stage yet
            self.issue_b(g)

    def issue_b(self, g):
        s = g % self.S
        assert not self.readers[s], f"TMA of chunk {g} overwrites stage {s} while {self.readers[s]} read it"
        self.b_content[s] = g
        self.b_full[s].arrive()                        # expect_tx + complete_tx folded into one arrival

    def wait(self, bar, phase):
        while not bar.ready(phase):
            yield False
        assert bar.phases == phase + 1, f"parity wait for phase {phase} passed at {bar.phases} completed phases"

    def producer_barrier(self):
        gen = self.pbar["gen"]
        self.pbar["arrived"] += 1
        if self.pbar["arrived"] == self.NP:
            self.pbar["arrived"], self.pbar["gen"] = 0, gen + 1
        while self.pbar["gen"] == gen:
            yield False

    def load_half(self, t, h):
        """Gather of half chunk h (registers only): the first half of tile j > 0 passes the producer-only barrier and
        writes the row table of tile j + 1, then every half of tile j reads the table of tile j."""
        g, part = divmod(h, 2)
        j, it = divmod(g, self.C)
        if part == 0 and it == 0:
            for b in (0, 1):                           # done with the row table of tile j - 1
                self.rows_readers[b].discard(t)
            if j > 0:
                yield from self.producer_barrier()
                buf = (j + 1) & 1
                assert not self.rows_readers[buf], f"row table {buf} rewritten while {self.rows_readers[buf]} read it"
                if j + 1 < self.J:
                    self.rows[buf] = j + 1
                yield True
        assert self.rows[j & 1] == j, f"thread {t} gathers tile {j} with the row table of tile {self.rows[j & 1]}"
        self.rows_readers[j & 1].add(t)                # the table is read whenever the tap changes during the tile
        yield True

    def store_half(self, t, h):
        """Store of half chunk h into its stage: part 0 waits for the stage to be free and issues the weight TMA, part 1
        arrives on "A full"."""
        S = self.S
        g, part = divmod(h, 2)
        s = g % S
        if part == 0:
            if g >= S:
                yield from self.wait(self.s_free[s], g // S - 1)
            if t == 0 and g >= self.npre:
                self.issue_b(g)
                yield True
        assert not self.readers[s], f"producer overwrites A of stage {s} while {self.readers[s]} read it"
        if t == 0 and part == 1:
            self.a_content[s] = g
        yield True
        if part == 1:
            self.a_full[s].arrive()
            if g == self.J * self.C - 1:
                self.stored += 1                       # this thread writes no shared memory after its last chunk
            yield True

    def producer(self, t):
        # the kernel's order: the gathers run two half chunks ahead of the stores (a ring of three register buffers), so
        # the barrier at the start of tile j is passed before the last chunk of tile j - 1 is stored
        nh = 2 * self.J * self.C
        for h in range(min(2, nh)):
            yield from self.load_half(t, h)
        for h in range(nh):
            if h + 2 < nh:
                yield from self.load_half(t, h + 2)
            yield from self.store_half(t, h)
        for b in (0, 1):
            self.rows_readers[b].discard(t)

    def consumer(self, wg):
        S, C = self.S, self.C
        groups = []                                  # committed wgmma groups, oldest first: (stage, chunk, key)

        def wait_group(keep):
            while len(groups) > keep:
                s, g, key = groups.pop(0)
                assert self.a_content[s] == g and self.b_content[s] == g, f"stage {s} changed under chunk {g}"
                self.readers[s].discard(key)

        def release(g):
            for _ in range(4):                       # one arrival per warp
                self.s_free[g % S].arrive()

        g = 0
        for j in range(self.J):
            for it in range(C):
                s = g % S
                yield from self.wait(self.a_full[s], g // S)
                yield from self.wait(self.b_full[s], g // S)
                assert self.a_content[s] == g and self.b_content[s] == g, \
                    f"warpgroup {wg} reads chunk {g} from stage {s} holding A {self.a_content[s]} / B {self.b_content[s]}"
                key = (wg, g)
                self.readers[s].add(key)
                groups.append((s, g, key))
                yield True
                wait_group(1)
                if it > 0:
                    release(g - 1)
                yield True
                g += 1
            wait_group(0)
            if C > 0 and self.release_last:
                release(g - 1)
            yield True
            if self.splitk:                          # bar.sync 1, 256, then the staging tile overwrites every stage
                self.staging += 1
                while self.staging < 2:
                    yield False
                assert all(not r for r in self.readers), "staging tile written while a stage is being read"
                assert self.stored == self.NP, "staging tile written before the producer stored its last chunk"
            yield True                               # finish: registers and global memory only (persistent)

    def run(self):
        actors = [self.producer(t) for t in range(self.NP)] + [self.consumer(w) for w in range(2)]
        steps = 0
        while actors:
            order = list(range(len(actors)))
            self.rng.shuffle(order)
            progressed = False
            for i in order:
                try:
                    if next(actors[i]):
                        progressed = True
                        break
                except StopIteration:
                    actors.pop(i)
                    progressed = True
                    break
            assert progressed, f"deadlock after {steps} steps"
            steps += 1
        assert all(not r for r in self.readers)
        return steps


class HaloSim:
    """The halo kernel of csrc/conv_tc.cu (conv3x3_halo_kernel): the weight ring beside a ring of two halo buffers.

    Actors: one weight lane (TMA of chunk g into stage g % STAGES after "b_free"), NP halo producer threads and two
    consumer warpgroups of four warps, interleaved in a random order.  One CTA computes `tiles` tiles of `slices` 64-channel
    slices; chunk g = (j * slices + sl) * 9 + tap and slice u = j * slices + sl run on across tiles, so the producers stage
    the halos of the next tile while the consumers finish this one.  A producer thread waits "h_free" of buffer u & 1 for
    u >= 2, stores its part of the halo (one step per store) and arrives on "h_full" (count NP).  Per tap a warpgroup waits
    "b_full", then runs 4 / KG groups: ldmatrix of KG k-steps (the halo reads, issued in one step and complete in the next,
    the mbarrier release orders them before a later arrival), after the slice's last one the four warps arrive on
    "h_free", then the group's wgmma read the weight stage until their wait_group 0; after the tap the warps arrive on
    "b_free".  At each tile start the warpgroups write the bias / scale columns of buffer j & 1, which the finish reads
    after bar.sync 1.

    Checked: no halo is restaged while an ldmatrix read of it is pending or before every consumer warp has released it,
    every ldmatrix reads the halo of the slice it expects, complete; every wgmma reads the weight chunk it expects and no
    stage is refilled while read; no bias / scale buffer is rewritten while a finish reads it; the run terminates.
    `hfree_early` releases each halo after the slice's first tap instead of its last (a broken kernel, for the test)."""

    def __init__(self, tiles, slices, seed, stages=2, kg=4, early=False, nprod=3, hfree_early=False):
        assert 4 % kg == 0
        self.J, self.NS, self.S, self.KG, self.NP = tiles, slices, stages, kg, nprod
        self.hfree_early = hfree_early
        self.rng = random.Random(seed)
        self.nchk = tiles * slices * 9
        self.b_full = [Barrier(1) for _ in range(stages)]
        self.b_free = [Barrier(8) for _ in range(stages)]
        self.h_full = [Barrier(nprod) for _ in range(2)]
        self.h_free = [Barrier(8) for _ in range(2)]
        self.b_content = [None] * stages
        self.b_readers = [set() for _ in range(stages)]
        self.halo = [dict() for _ in range(2)]         # producer thread -> slice whose part it stored
        self.h_readers = [set(), set()]                # pending ldmatrix reads
        self.bs = [None, None]                         # bias / scale columns: tile held by each buffer
        self.bs_readers = [set(), set()]
        self.bar = {"arrived": 0, "gen": 0}            # bar.sync 1, 256 (both consumer warpgroups)
        self.npre = min(stages, self.nchk) if early else 0
        for g in range(self.npre):
            self.issue_b(g)

    def issue_b(self, g):
        s = g % self.S
        assert not self.b_readers[s], f"TMA of chunk {g} overwrites stage {s} while {self.b_readers[s]} read it"
        self.b_content[s] = g
        self.b_full[s].arrive()

    def wait(self, bar, phase):
        while not bar.ready(phase):
            yield False
        assert bar.phases == phase + 1, f"parity wait for phase {phase} passed at {bar.phases} completed phases"

    def weights(self):
        for g in range(self.npre, self.nchk):
            s = g % self.S
            if g >= self.S:
                yield from self.wait(self.b_free[s], g // self.S - 1)
            self.issue_b(g)
            yield True

    def producer(self, t):
        u = 0
        for _ in range(self.J):
            for _ in range(self.NS):
                hb = u & 1
                if u >= 2:
                    yield from self.wait(self.h_free[hb], (u >> 1) - 1)
                yield True                               # the loads (registers only)
                assert not self.h_readers[hb], f"halo {hb} restaged for slice {u} while {self.h_readers[hb]} read it"
                self.halo[hb][t] = u
                yield True
                self.h_full[hb].arrive()
                yield True
                u += 1

    def consumer(self, wg):
        S, KG = self.S, self.KG
        g = u = 0
        for j in range(self.J):
            buf = j & 1
            assert not self.bs_readers[buf], f"bias / scale of tile {j} written while tile {self.bs[buf]} is finished"
            self.bs[buf] = j
            yield True
            for _ in range(self.NS):
                hb = u & 1
                yield from self.wait(self.h_full[hb], u >> 1)
                for tap in range(9):
                    s = g % S
                    yield from self.wait(self.b_full[s], g // S)
                    for k0 in range(0, 4, KG):
                        key = (wg, g, k0)
                        self.h_readers[hb].add(key)      # ldmatrix issued
                        yield True
                        parts = self.halo[hb]
                        assert len(parts) == self.NP and all(v == u for v in parts.values()), \
                            f"warpgroup {wg} reads slice {u} from halo {hb} holding {parts}"
                        self.h_readers[hb].discard(key)  # in registers
                        last = tap == 0 if self.hfree_early else tap == 8
                        if last and k0 + KG == 4:
                            self.h_free[hb].arrive(4)
                        assert self.b_content[s] == g, f"warpgroup {wg} reads chunk {g} from stage {s} holding {self.b_content[s]}"
                        self.b_readers[s].add(key)       # wgmma issued, commit
                        yield True
                        assert self.b_content[s] == g, f"stage {s} changed under chunk {g}"
                        self.b_readers[s].discard(key)   # wait_group 0
                        yield True
                    self.b_free[s].arrive(4)
                    g += 1
                u += 1
            gen = self.bar["gen"]                        # bar.sync 1, 256
            self.bar["arrived"] += 1
            if self.bar["arrived"] == 2:
                self.bar["arrived"], self.bar["gen"] = 0, gen + 1
            while self.bar["gen"] == gen:
                yield False
            self.bs_readers[buf].add(wg)                 # the finish reads the columns of tile j
            yield True
            assert self.bs[buf] == j, f"finish of tile {j} reads the columns of tile {self.bs[buf]}"
            self.bs_readers[buf].discard(wg)
            yield True

    def run(self):
        actors = [self.weights()] + [self.producer(t) for t in range(self.NP)] + [self.consumer(w) for w in range(2)]
        steps = 0
        while actors:
            order = list(range(len(actors)))
            self.rng.shuffle(order)
            progressed = False
            for i in order:
                try:
                    if next(actors[i]):
                        progressed = True
                        break
                except StopIteration:
                    actors.pop(i)
                    progressed = True
                    break
            assert progressed, f"deadlock after {steps} steps"
            steps += 1
        assert all(not r for r in self.b_readers) and all(not r for r in self.h_readers)
        return steps


if __name__ == "__main__":
    for stages in (2, 3, 4, 6, 8):
        for kg in (1, 2, 4):
            for tiles in range(0, 4):
                for slices in (1, 2, 4):
                    for seed in range(4):
                        HaloSim(tiles, slices, seed, stages, kg, early=seed % 2 == 1).run()
    for stages in (2, 3, 4, 8):
        for tiles in range(0, 5):
            for chunks in (1, 2, 3, 5, 9):
                for seed in range(10):
                    for early in (False, True):
                        Sim(tiles, chunks, seed, stages, early).run()
                        if tiles <= 1:
                            Sim(tiles, chunks, seed, stages, early, splitk=True).run()
    print("ok")
