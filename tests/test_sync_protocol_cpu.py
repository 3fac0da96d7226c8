"""Model check of the in-kernel SyncBN exchange protocol (csrc/seg_sync.cuh, DESIGN.md §6) — the cross-GPU part of the path that
a one-GPU box cannot exercise and whose mistakes show up as rare corruption, not as a failing unit test.

The model transcribes the protocol onto W abstract ranks.  Each rank owns a symmetric buffer `data[2][W] | flags[2][W] | seq`
and runs, for every exchange of the step (all ranks issue the same exchanges in the same order), in ONE block
(seg_sync.cuh::sync_exchange_block_*, which the producers' last block and the stand-alone seg_syncbn_exchange both run):
    epoch = seq + 1;  slot = epoch & 1
    push   : store my vector into data[slot][me] of EVERY peer        (one store per peer = one schedulable event)
    publish: store `epoch` into flags[slot][me] of EVERY peer          (after the pushes: fence + release store)
    wait   : spin until flags[slot][p] == epoch for every p in MY buffer
    total  : read data[slot][p] for every p from MY buffer, add in rank order
    advance: seq = epoch
Between exchanges a rank does an arbitrary amount of unrelated work, so ranks drift apart.

Events are interleaved by a seeded random scheduler (sequentially consistent: the memory-ordering side — who fences, release /
acquire at system scope — is argued in the header, the LOGIC is what is checked here).  On every schedule:
  * no deadlock: every rank finishes every exchange;
  * no slot is overwritten while a peer still reads it, and no rank reads a vector of another exchange: every stored vector
    is tagged (exchange index, rank) and `total` asserts the tags;
  * every rank's world total equals the expected sum, bit for bit identical across ranks (same order of addition);
  * a rank never runs more than one exchange ahead of the slowest peer (the invariant the two-slot scheme rests on).
Seeded protocol mistakes (one slot instead of two; flag raised before the data; equality replaced by >= across an epoch
wrap-around) must be caught: the model is not vacuous."""
import random

import pytest


class Rank:
    def __init__(self, world):
        self.data = [[None] * world for _ in range(2)]   # (exchange, rank, payload)
        self.flags = [[0] * world for _ in range(2)]
        self.seq = 0
        self.done = 0        # exchanges completed (model bookkeeping, not protocol state)
        self.reading = None  # slot this rank is currently summing from
        self.totals = []


class Violation(AssertionError):
    pass


def epoch_of(seq):
    e = (seq + 1) & 0xFFFFFFFF
    return 2 if e == 0 else e  # flags start at 0: skip it on wrap-around, keeping the parity alternation (sync_epoch)


def rank_program(me, ranks, n_exchanges, payload, rng, bug):
    """Generator: one yield per externally visible memory event, so the scheduler can interleave ranks between any two."""
    W = len(ranks)
    mine = ranks[me]
    for x in range(n_exchanges):
        for _ in range(rng.randrange(0, 4)):  # unrelated kernels between exchanges: ranks drift
            yield "work"
        epoch = epoch_of(mine.seq)
        slot = 0 if bug == "one_slot" else (epoch & 1)
        order = list(range(W))
        rng.shuffle(order)  # P2P stores to different peers land in any order

        def raise_flags():
            for p in order:
                ranks[p].flags[slot][me] = epoch
                yield "flag"

        if bug == "flag_before_data":
            yield from raise_flags()
        for p in order:
            tgt = ranks[p]
            if tgt.reading == slot and tgt.data[slot][me] is not None and tgt.data[slot][me][0] != x:
                raise Violation(f"rank {me} overwrote slot {slot} of rank {p} (exchange {tgt.data[slot][me][0]} -> {x}) while rank {p} reads it")
            tgt.data[slot][me] = (x, me, payload(x, me))
            yield "push"
        if bug != "flag_before_data":
            yield from raise_flags()

        # ---- wait + total + advance, by the same block
        if bug == "advance_early":
            mine.seq = epoch  # before anyone has read
        spins = 0
        for p in range(W):
            while True:
                f = mine.flags[slot][p]
                ok = (f >= epoch) if bug == "ge_compare" else (f == epoch)
                if ok:
                    break
                spins += 1
                if spins > 200000:
                    raise Violation(f"rank {me} starved waiting for rank {p} at exchange {x} (flag {f}, epoch {epoch})")
                yield "spin"
        mine.reading = slot
        tot = 0.0
        for p in range(W):
            yield "read"
            v = mine.data[slot][p]
            if v is None or v[0] != x or v[1] != p:
                raise Violation(f"rank {me} read {v} from slot {slot} while summing exchange {x}, rank {p}")
            tot += v[2]
        mine.reading = None
        if bug != "advance_early":
            mine.seq = epoch
        yield "advance"
        mine.totals.append(tot)
        mine.done = x + 1
        lead = mine.done - min(r.done for r in ranks)
        if lead > 1 and bug is None:
            raise Violation(f"rank {me} is {lead} exchanges ahead of the slowest peer")


def run(world, n_exchanges, seed, bug=None, seq0=0):
    rng = random.Random(seed)
    ranks = [Rank(world) for _ in range(world)]
    for r in ranks:
        r.seq = seq0

    def payload(x, rank):
        return float((x * 131 + rank * 17) % 1009) + 0.25 * rank

    progs = [rank_program(i, ranks, n_exchanges, payload, random.Random(seed * 977 + i), bug) for i in range(world)]
    alive = list(range(world))
    # a biased scheduler: now and then one rank is held back for a long stretch (a slow data loader, a checkpoint write)
    held, hold_left = None, 0
    steps = 0
    while alive:
        steps += 1
        if steps > 5_000_000:
            raise Violation("no progress: deadlock")
        if hold_left == 0 and rng.random() < 0.01 and len(alive) > 1:
            held, hold_left = rng.choice(alive), rng.randrange(50, 400)
        cands = [i for i in alive if i != held] if hold_left > 0 and len(alive) > 1 else alive
        hold_left = max(0, hold_left - 1)
        i = rng.choice(cands)
        try:
            next(progs[i])
        except StopIteration:
            alive.remove(i)
            if held == i:
                held, hold_left = None, 0
    expect = [sum(payload(x, p) for p in range(world)) for x in range(n_exchanges)]
    for r in ranks:
        assert r.totals == expect, "world totals differ from the expected sums"
        assert r.done == n_exchanges
    return ranks


# seq0: a fresh buffer, and a sequence number whose epoch wraps past 2^32 at the 12th of the 24 exchanges
@pytest.mark.parametrize("seq0", [0, 0xFFFFFFF4], ids=["fresh", "wrap"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_exchange_protocol_is_safe_under_random_interleavings(world, seq0):
    for seed in range(40 if world < 8 else 12):
        run(world, 24, seed, seq0=seq0)


def test_epoch_wraparound_keeps_parity_and_skips_zero():
    # seq close to 2^32: epochs ... fffffffe, ffffffff, (0 skipped ->) 2, 3 ...; the flag value 0 (initial state) is never used
    assert epoch_of(0xFFFFFFFE) == 0xFFFFFFFF and epoch_of(0xFFFFFFFF) == 2 and epoch_of(2) == 3
    for seed in range(10):
        run(2, 6, seed, seq0=0xFFFFFFFC)
        run(3, 6, seed, seq0=0xFFFFFFFD)


@pytest.mark.parametrize("bug", ["one_slot", "flag_before_data", "ge_compare"])
def test_seeded_protocol_mistakes_are_caught(bug):
    caught = 0
    for seed in range(60):
        try:
            run(3, 24, seed, bug=bug, seq0=0xFFFFFFF0 if bug == "ge_compare" else 0)
        except (Violation, AssertionError):
            caught += 1
    assert caught > 0, f"the model did not notice the seeded mistake '{bug}'"


def test_slot_safety_rests_on_the_flag_dependency_not_on_advance_order():
    """Advancing seq BEFORE the totals are read does not break the two-slot scheme: the next-but-one
    exchange — the first that reuses the slot — still needs every peer's flag of the next one, which a peer raises only after
    it has finished reading.  The model documents that it is this dependency, not the advance-after-read order, that protects
    the slot (so the single `__threadfence(); sync(); advance` tail of sync_exchange_block_* is not load-bearing for safety)."""
    for seed in range(20):
        run(3, 16, seed, bug="advance_early")
