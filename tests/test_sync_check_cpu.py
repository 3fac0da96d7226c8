"""Self-test of sync_check.py: a numpy transcription of sync_exchange_block_d / _f over byte images with the real buffer
layout passes the checker at every world size, rank position and across the epoch wrap, and each seeded defect of the
protocol or of its consumers is rejected with a message naming the rank, the slot and the element."""
import numpy as np
import pytest
import torch

import elementwise_check as ec
import sync_check as sc

WORLDS = (1, 2, 3, 8, 64)


def local_vector(n, dtype, seed):
    """A producer's own vector: moderate magnitudes of both signs."""
    rng = np.random.default_rng(seed)
    v = np.ldexp(1.0 + rng.random(n), rng.integers(-8, 9, size=n)) * rng.choice([-1.0, 1.0], size=n)
    return v.astype(np.float64 if dtype == sc.F64 else np.float32)


def exchange(images, world, rank, n_max, local, dtype, defect=None):
    """sync_exchange_block_{d,f} of rank `rank` on host images: push, publish, wait (asserted: staged), rank-order
    total, advance.  Returns the total.  `defect` seeds one mistake."""
    seq = int(sc.seq_word(images[rank], world, n_max)[0])
    e = (seq + 1) & sc.SEQ_MASK
    if e == 0 and defect != "wrap_to_0":
        e = 2
    par = e & 1
    if defect == "parity":
        par ^= 1
    n = local.size
    size = 8 if dtype == sc.F64 else 4
    for p in range(world):  # push
        if defect == "skip_own_push" and p == rank:
            continue
        img = images[p]
        if dtype == sc.F64 and defect == "f64_stride_doubles":
            o = (par * world + rank) * n_max * 8
        else:
            o = sc.slot_byte_offset(world, n_max, par, rank)
        count = n + (1 if defect == "past_end" else 0)
        vals = np.concatenate([local, local[:1]]) if defect == "past_end" else local
        img[o:o + size * count] = vals.astype(local.dtype).view(np.uint8)
    for p in range(world):  # publish
        sc.flags(images[p], world, n_max)[par, rank] = seq if defect == "flag_is_seq" else e
    mine = images[rank]  # wait: the staged flags satisfy it (a defect that waits on other flags would block instead)
    vecs = [sc.slot(mine, world, n_max, par, p, dtype)[:n].copy() for p in range(world)]
    order = list(range(world))
    if defect == "own_first":
        order = [rank] + [p for p in order if p != rank]
    total = sc.world_total([vecs[p] for p in order], dtype)
    if defect != "no_advance":  # advance
        sc.seq_word(images[(rank + 1) % world] if defect == "advance_peer" else mine, world, n_max)[0] = e
    return total


def run_case(world, rank, n_max, n, dtype, seq, seed, defect=None):
    """Stage, exchange with the transcription, check.  Raises what the checker raises."""
    images = sc.fresh_images(world, n_max)
    local = local_vector(n, dtype, seed)
    peers = sc.adversarial(world, rank, n, dtype, seed + 1)
    e = sc.stage(images, world, rank, n_max, seq, peers, dtype)
    before = [img.copy() for img in images]
    total = exchange(images, world, rank, n_max, local, dtype, defect)
    want, e2 = sc.expected_after(before, world, rank, n_max, local, dtype)
    assert e2 == e
    vecs = [peers[p] if p != rank else local for p in range(world)]
    case = f"W={world} rank={rank} e={e} {dtype}"
    sc.check_buffers(case, images, want, world, n_max, dtype)
    sc.check_total(case, total, sc.world_total(vecs, dtype))
    return e


def ranks_of(world):
    return sorted({0, world // 2, world - 1})


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype", [sc.F64, sc.F32])
def test_transcription_passes(world, dtype):
    for rank in ranks_of(world):
        for seq, e in ((0, 1), (1, 2), (0xFFFFFFFE, 0xFFFFFFFF), (0xFFFFFFFF, 2), (2, 3)):
            n = 24
            n_max = 4 * 6 * 2 if dtype == sc.F64 else 2 * 24  # the vector fills the slot exactly
            assert run_case(world, rank, n_max, n, dtype, seq, seed=world * 100 + rank) == e


def test_layout_matches_the_header():
    assert sc.flags_offset(2, 8192) == 2 * 2 * 8192 * 4
    assert sc.flags_offset(3, 10) == 256  # 240 bytes of slots, rounded to 128
    assert sc.seq_offset(3, 10) == 384
    assert sc.buffer_bytes(3, 10) == 512
    assert sc.epoch(0) == 1 and sc.epoch(0xFFFFFFFE) == 0xFFFFFFFF and sc.epoch(0xFFFFFFFF) == 2
    with pytest.raises(AssertionError):
        sc.slot_f64(sc.fresh_images(2, 7)[0], 2, 7, 0, 1)  # odd n_max: rank 1's fp64 slot is misaligned


def test_adversarial_vectors_are_order_sensitive():
    for dtype in (sc.F64, sc.F32):
        for world in (3, 8, 64):
            for rank in [r for r in ranks_of(world) if r >= 2]:
                peers = sc.adversarial(world, rank, 64, dtype, seed=world + rank)
                local = local_vector(64, dtype, seed=7)
                vecs = [peers[p] if p != rank else local for p in range(world)]
                assert sc.order_sensitive(vecs, rank, dtype) >= 16, (dtype, world, rank)


DEFECTS = {
    # defect: (dtype, world, rank, seq, what the message must name)
    "own_first": (sc.F64, 3, 2, 0, "W=3 rank=2 e=1 f8: world total: "),
    "parity": (sc.F32, 3, 2, 0, "buffer of rank 0: data[0][slot 2] element 0"),
    "flag_is_seq": (sc.F64, 3, 1, 4, "buffer of rank 0: flags[1][slot 1]: 0x00000004 expected 0x00000005"),
    "wrap_to_0": (sc.F64, 8, 3, 0xFFFFFFFF, "buffer of rank 0: flags[0][slot 3]: 0x00000000 expected 0x00000002"),
    "no_advance": (sc.F32, 2, 1, 0, "buffer of rank 1: seq"),
    "advance_peer": (sc.F32, 3, 2, 0, "buffer of rank 0: seq"),
    "skip_own_push": (sc.F64, 3, 0, 0, "buffer of rank 0: data[1][slot 0] element 0"),
    "f64_stride_doubles": (sc.F64, 3, 1, 1, "buffer of rank 0: data[0][slot 1] element 0"),
    "past_end": (sc.F32, 2, 0, 0, "buffer of rank 0: data[1][slot 1] element 0"),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_seeded_protocol_defects_are_rejected(defect):
    """Each vector fills its slot exactly (4C == n_max, 2C == n_max), so the guard after a slot is the next one."""
    dtype, world, rank, seq, where = DEFECTS[defect]
    n_max = 48
    n = n_max // 2 if dtype == sc.F64 else n_max
    with pytest.raises(AssertionError) as ei:
        run_case(world, rank, n_max, n, dtype, seq, seed=11, defect=defect)
    msg = str(ei.value)
    assert where in msg, msg


def test_the_wait_needs_every_flag_staged():
    images = sc.fresh_images(3, 16)
    peers = sc.adversarial(3, 1, 8, sc.F32, 3)
    del peers[2]
    with pytest.raises(AssertionError):
        sc.stage(images, 3, 1, 16, 0, peers, sc.F32)


# ------------------------------------------------------------------------------------------------ consumers
def shards(world, rows, C, seed):
    g = torch.Generator().manual_seed(seed)
    cs = ec.channel_scales(C, seed)
    return [ec.bf16_round((torch.randn(rows, C, generator=g, dtype=torch.float64) + 0.3 * (r + 1)) * cs) for r in range(world)]


def test_consumer_with_the_local_count_is_rejected():
    world, rank, rows, C = 4, 2, 64, 16
    xs = shards(world, rows, C, 5)
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.3
    st, pre, acc = sc.concat_apply_ref(xs, rank, gamma, beta, 1e-5)
    # the kernel's result, modelled in float64: BN with the world's sums over the world count passes ...
    ec.check_apply("world count", torch.relu(pre).float(), pre, acc)
    # ... over the local count (the world's sums divided by one rank's rows) it fails
    bad_st = ec.BnStats(ec.exact_stats(torch.cat(xs)), rows, 1e-5, False)
    bad, _ = ec.bn_train_ref(xs[rank], bad_st, gamma, beta)
    with pytest.raises(AssertionError, match=r"local count: bn apply: \d+ element\(s\) over the bound.*\n  \(m=\d+, c=\d+\)"):
        ec.check_apply("local count", torch.relu(bad).float(), pre, acc)
    # the backward: dx of the concatenated batch on rank's rows; the world's sums over the local count fail
    dout = [ec.bf16_round(torch.randn(rows, C, generator=torch.Generator().manual_seed(9 + r), dtype=torch.float64))
            for r in range(world)]
    save = torch.cat([st.mean, st.istd]).float()
    ref = ec.BwdRef(torch.cat(dout), torch.cat(xs), save, gamma, chain=8)
    b = sc.rows_of(ref.dx_bound(), rank * rows, rows)
    ec.check(f"rank {rank}", "dx", b.ref.float(), b)
    A = ref.A
    local = A * (ref.dz - ref.s0 / rows - ref.xhat * ref.s1 / rows)
    with pytest.raises(AssertionError, match=r"dx: \d+ element\(s\) over the bound"):
        ec.check(f"rank {rank}", "dx", local[rank * rows:(rank + 1) * rows].float(), b)


def test_param_grads_from_the_world_sums_are_rejected():
    C = 8
    local = np.arange(1, 2 * C + 1, dtype=np.float32) * np.float32(0.37)
    world = local * np.float32(3)
    sc.check_local_param_grads("local", local[C:], local[:C], local)
    with pytest.raises(AssertionError, match=r"dbeta \(local sum dz\): 8 element\(s\) differ\n  element 0"):
        sc.check_local_param_grads("world", world[C:], world[:C], local)


def test_fused_sync_chain_covers_the_unsynced_grid_minus_one_block_per_sm():
    for M, C in ((4096, 64), (65 * 65 * 2, 256), (33 * 33 * 4, 2064)):
        for sms in (114, 132):
            chain = sc.fused_sync_chain(M, C, sms)
            for bps in range(2, 9):
                gx, _ = ec.fused_grid(M, C, sms, bps - 1)
                assert -(-M // (gx * ec.rows_par(C))) + ec.rows_par(C) + gx + 1 <= chain
