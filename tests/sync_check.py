"""Checker of the SyncBN statistics exchange (csrc/seg_sync.cuh) as the producers run it: the symmetric-buffer layout,
the staged-peer harness that lets ONE rank run the whole protocol on one GPU, and the state every buffer must hold after
that rank's exchange.

The exchange of rank r at epoch e is: push r's vector into data[e&1][r] of every peer's buffer (its own included), raise
flags[e&1][r] = e on every peer, wait for flags[e&1][0..W) == e in its OWN buffer, add data[e&1][0..W) of its own buffer
in rank order starting from 0 (float64 for the forward statistics, float32 for the backward sums), store seq = e in its own
buffer.  With the other ranks' vectors and flags written into r's buffer before the launch, the wait is already
satisfied when the producer reaches it, so every step is checkable bit for bit with no concurrency at all.

Layout and state are modelled on host byte images (numpy uint8, one per rank); the pure functions below need no GPU and
are checked against a numpy transcription of sync_exchange_block_d / _f in test_sync_check_cpu.py.  StagedPeers puts the
images on the device for the GPU conformance file (test_syncbn_conformance_gpu.py).

The concatenated-batch references are elementwise_check's (exact_stats, bn_train_ref, BwdRef, check_apply, ...); only the
fused backward's grid under SyncBN is new here (fused_sync_chain)."""
import ctypes

import numpy as np

import elementwise_check as ec

MAX_WORLD = 64
SENTINEL_BYTE = 0xA5  # float 0xA5A5A5A5 = -2.9e-16, double -6.6e-130, flag 0xA5A5A5A5: no exchange writes any of them
SEQ_MASK = 0xFFFFFFFF
F64, F32 = "f8", "f4"


# ------------------------------------------------------------------------------------------------ layout (seg_sync.cuh)
def flags_offset(world, n_max):
    return (2 * world * n_max * 4 + 127) & ~127


def seq_offset(world, n_max):
    return (flags_offset(world, n_max) + 2 * world * 4 + 127) & ~127


def buffer_bytes(world, n_max):
    """seg_comm_buffer_bytes."""
    return seq_offset(world, n_max) + 128


def epoch(seq):
    """sync_epoch: the epoch of the next exchange after `seq` completed ones; the wrap skips 0 (flags start at 0)."""
    e = (int(seq) + 1) & SEQ_MASK
    return 2 if e == 0 else e


def slot_byte_offset(world, n_max, parity, p):
    return (parity * world + p) * n_max * 4


def slot_f32(img, world, n_max, parity, p):
    o = slot_byte_offset(world, n_max, parity, p)
    return img[o:o + 4 * n_max].view(np.float32)


def slot_f64(img, world, n_max, parity, p):
    """The fp64 view of a slot: its n_max floats as n_max / 2 doubles, starting at the slot's FLOAT offset."""
    o = slot_byte_offset(world, n_max, parity, p)
    assert o % 8 == 0, "an fp64 slot needs an even n_max"
    return img[o:o + 4 * n_max].view(np.float64)


def slot(img, world, n_max, parity, p, dtype):
    return (slot_f64 if dtype == F64 else slot_f32)(img, world, n_max, parity, p)


def flags(img, world, n_max):
    o = flags_offset(world, n_max)
    return img[o:o + 8 * world].view(np.uint32).reshape(2, world)


def seq_word(img, world, n_max):
    o = seq_offset(world, n_max)
    return img[o:o + 4].view(np.uint32)


def fresh_images(world, n_max):
    """One sentinel-filled byte image per rank."""
    return [np.full(buffer_bytes(world, n_max), SENTINEL_BYTE, dtype=np.uint8) for _ in range(world)]


# ------------------------------------------------------------------------------------------------ protocol model
def stage(images, world, rank, n_max, seq, peer_vectors, dtype):
    """Host half of StagedPeers.stage: the other ranks' vectors into data[e&1][p] of rank `rank`'s buffer, their flags
    = e, and rank's seq.  peer_vectors: {p: vector} for every p != rank.  Returns the epoch."""
    e = epoch(seq)
    mine = images[rank]
    assert sorted(peer_vectors) == [p for p in range(world) if p != rank]
    for p, v in peer_vectors.items():
        v = np.asarray(v, dtype=np.float64 if dtype == F64 else np.float32)
        slot(mine, world, n_max, e & 1, p, dtype)[:v.size] = v
        flags(mine, world, n_max)[e & 1, p] = e
    seq_word(mine, world, n_max)[0] = seq
    return e


def world_total(vectors, dtype):
    """The rank-order sequential sum starting from 0 (sync_total_d in float64, sync_total in float32)."""
    t = np.zeros_like(np.asarray(vectors[0], dtype=np.float64 if dtype == F64 else np.float32))
    for v in vectors:
        t = t + np.asarray(v, dtype=t.dtype)
    return t


def expected_after(images, world, rank, n_max, local, dtype):
    """What every buffer must hold after rank `rank`'s exchange at the epoch its seq names: data[e&1][rank] = local in
    every buffer, flags[e&1][rank] = e in every buffer, seq = e in rank's buffer only; every other byte unchanged.
    Returns (images after, epoch)."""
    e = epoch(int(seq_word(images[rank], world, n_max)[0]))
    local = np.asarray(local, dtype=np.float64 if dtype == F64 else np.float32)
    out = [img.copy() for img in images]
    for img in out:
        slot(img, world, n_max, e & 1, rank, dtype)[:local.size] = local
        flags(img, world, n_max)[e & 1, rank] = e
    seq_word(out[rank], world, n_max)[0] = e
    return out, e


def describe(world, n_max, off, dtype):
    """Name of byte `off` of a buffer: data[parity][slot] element (in the exchange's dtype), a flag, seq or padding."""
    fo, so = flags_offset(world, n_max), seq_offset(world, n_max)
    if off < 2 * world * n_max * 4:
        s, within = divmod(off, 4 * n_max)
        parity, p = divmod(s, world)
        size = 8 if dtype == F64 else 4
        return f"data[{parity}][slot {p}] element {within // size}"
    if fo <= off < fo + 8 * world:
        parity, p = divmod((off - fo) // 4, world)
        return f"flags[{parity}][slot {p}]"
    if so <= off < so + 4:
        return "seq"
    return f"padding byte {off}"


def check_buffers(case, got, want, world, n_max, dtype, show=6):
    """Byte-exact comparison of every rank's buffer; raises naming the rank whose buffer differs and the slot, flag,
    seq or padding word with the first differing elements."""
    lines, nbad = [], 0
    for b, (g, w) in enumerate(zip(got, want)):
        diff = np.nonzero(g != w)[0]
        if diff.size == 0:
            continue
        nbad += diff.size
        seen = set()
        for off in diff:
            name = describe(world, n_max, int(off), dtype)
            if name in seen:
                continue
            seen.add(name)
            if len(lines) < show:
                lines.append(f"  buffer of rank {b}: {name}: {_word(g, world, n_max, int(off), dtype)} "
                             f"expected {_word(w, world, n_max, int(off), dtype)}")
    if nbad:
        raise AssertionError(f"{case}: exchange state: {nbad} byte(s) differ\n" + "\n".join(lines))


def _word(img, world, n_max, off, dtype):
    if off < 2 * world * n_max * 4:
        s = (off // (4 * n_max)) * 4 * n_max
        size = 8 if dtype == F64 else 4
        a = s + ((off - s) // size) * size
        v = img[a:a + size].view(np.float64 if size == 8 else np.float32)[0]
        return f"{v!r} ({img[a:a + size].tobytes()[::-1].hex()})"
    a = off // 4 * 4
    return f"0x{int(img[a:a + 4].view(np.uint32)[0]):08x}"


def check_total(case, got, want, what="world total", show=6):
    """Bit-exact comparison of a vector with the host's rank-order total (the element named by its index)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (case, what, got.shape, want.shape)
    bad = np.nonzero(got.view(np.uint64 if got.dtype == np.float64 else np.uint32)
                     != want.astype(got.dtype).view(np.uint64 if got.dtype == np.float64 else np.uint32))[0]
    if bad.size:
        lines = [f"  element {i}: got {got[i]!r} expected {want[i]!r}" for i in bad[:show]]
        raise AssertionError(f"{case}: {what}: {bad.size} element(s) differ\n" + "\n".join(lines))


def adversarial(world, rank, n, dtype, seed):
    """Peer vectors whose rank-order sum depends on the order: in every element, values of widely spread magnitudes of
    both signs, and an exactly cancelling large pair, so that an order other than rank order rounds differently."""
    rng = np.random.default_rng(seed)
    span = 20
    out = {}
    for p in range(world):
        if p == rank:
            continue
        e = rng.integers(-span, span + 1, size=n)
        v = np.ldexp(1.0 + rng.random(n), e) * rng.choice([-1.0, 1.0], size=n)
        out[p] = v.astype(np.float64 if dtype == F64 else np.float32)
    peers = [p for p in range(world) if p != rank]
    if len(peers) >= 2:  # the first two peers carry +-big, exactly cancelling: added after them, the own vector survives
        big = np.ldexp(1.0, 90 if dtype == F64 else 40)  # in full; added first (own + big) it is absorbed
        s = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
        out[peers[0]] = (out[peers[0]].astype(np.float64) + s * big).astype(out[peers[0]].dtype)
        out[peers[1]] = (out[peers[1]].astype(np.float64) - s * big).astype(out[peers[1]].dtype)
    return out


def _bits(v):
    return v.view(np.uint64 if v.dtype == np.float64 else np.uint32)


def order_sensitive(vectors, rank, dtype):
    """Number of elements whose total changes when rank's vector is added first instead of at its position (none can at
    rank < 2: there it is one swap of two operands of the first addition, which commutes)."""
    want = world_total(vectors, dtype)
    alt = world_total([vectors[rank]] + [v for p, v in enumerate(vectors) if p != rank], dtype)
    return int((_bits(want) != _bits(alt)).sum())


# ------------------------------------------------------------------------------------------------ concatenated batch
def concat_apply_ref(shards, rank, gamma, beta, eps, res=None):
    """BatchNorm over the concatenated batch (shards: float64 torch [rows, C] per rank, bf16-exact), restricted to rank's
    rows: (BnStats of the world, pre-activation reference and allowance of rank's rows).  res: rank's residual rows."""
    import torch
    st = ec.BnStats(ec.exact_stats(torch.cat(list(shards))), sum(s.shape[0] for s in shards), eps, False)
    pre, acc = ec.bn_train_ref(shards[rank], st, gamma, beta, res)
    return st, pre, acc


def check_local_param_grads(case, dgamma, dbeta, local_sums):
    """dbeta / dgamma must be this rank's LOCAL sums (s0, s1) bit for bit: the flat gradient all-reduce adds the ranks'
    parameter gradients later, so world sums here would be counted world times."""
    s = np.asarray(local_sums, dtype=np.float32)
    C = s.size // 2
    check_total(case, np.asarray(dbeta, dtype=np.float32), s[:C], "dbeta (local sum dz)", show=4)
    check_total(case, np.asarray(dgamma, dtype=np.float32), s[C:], "dgamma (local sum dz xhat)", show=4)


# ------------------------------------------------------------------------------------------------ grids
def fused_sync_chain(M, C, sms):
    """Summation chain of bn_bwd_fused's local sums under SyncBN: the host leaves one block slot per SM free
    (blocks_per_sm - 1 when it is > 1, seg_elementwise.cu), so the grid is fused_grid(M, C, bps - 1) for the launch's
    occupancy bps, which Python cannot see: the longest thread chain over bps - 1 >= 1 and the widest fold (bps - 1 <= 7)."""
    gx_min, _ = ec.fused_grid(M, C, sms, 1)
    gx_max, _ = ec.fused_grid(M, C, sms, 7)
    return -(-M // (gx_min * ec.rows_par(C))) + ec.rows_par(C) + gx_max + 1


# ------------------------------------------------------------------------------------------------ device harness
def timeout_clocks(seconds):
    """As comm._sync_timeout_clocks: seconds at ~2 GHz."""
    return int(float(seconds) * 2e9)


class _Raw:
    """A device byte range as a zero-copy torch tensor (cudaMalloc'd by seg_comm_alloc)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                         "version": 3}


class StagedPeers:
    """One simulated rank of a W-rank SyncBN world on one GPU: one symmetric buffer per rank (seg_comm_alloc), the
    device peer-pointer array and the lib.SyncDesc of rank `rank`.  Passes as `sync=` to the ops producers and to
    engine.Tape (.desc, .world, .rank, .fused, .force).  The host images (.images) model all W buffers; stage() writes
    the other ranks' vectors / flags and this rank's seq into them and copies them to the device on the current stream,
    expect() returns the state after this rank's exchange and adopts it, read() copies the buffers back."""

    def __init__(self, world, rank, n_max, timeout_s=5.0):
        import torch
        from seg_b200 import lib
        assert 1 <= world <= MAX_WORLD and 0 <= rank < world and n_max % 2 == 0
        self.world, self.rank, self.n_max = world, rank, n_max
        self.fused, self.force = True, True
        self._L = lib.load()
        self.nbytes = buffer_bytes(world, n_max)
        assert self._L.seg_comm_buffer_bytes(world, n_max) == self.nbytes
        self._ptrs = []
        for _ in range(world):
            p = ctypes.c_void_p()
            assert self._L.seg_comm_alloc(self.nbytes, ctypes.byref(p)) == 0, lib.last_error()
            self._ptrs.append(p)
        self.bufs = [torch.as_tensor(_Raw(p.value, self.nbytes), device="cuda") for p in self._ptrs]
        self.peers = torch.tensor([p.value for p in self._ptrs], dtype=torch.int64, device="cuda")
        self.desc = lib.SyncDesc(self.peers.data_ptr(), rank, world, n_max, timeout_clocks(timeout_s))
        self.images = fresh_images(world, n_max)
        self.upload()

    def upload(self):
        import torch
        for b, img in zip(self.bufs, self.images):
            b.copy_(torch.from_numpy(img))

    def stage(self, seq, peer_vectors, dtype):
        e = stage(self.images, self.world, self.rank, self.n_max, seq, peer_vectors, dtype)
        self.upload()
        return e

    def read(self):
        import torch
        torch.cuda.synchronize()
        return [b.cpu().numpy() for b in self.bufs]

    def expect(self, local, dtype):
        want, e = expected_after(self.images, self.world, self.rank, self.n_max, local, dtype)
        self.images = want
        return want, e

    def seq(self):
        import torch
        torch.cuda.synchronize()
        return int(self.bufs[self.rank][seq_offset(self.world, self.n_max):][:4].cpu().numpy().view(np.uint32)[0])

    def close(self):
        import torch
        torch.cuda.synchronize()
        self.bufs = []
        for p in self._ptrs:
            self._L.seg_comm_free(p)
        self._ptrs = []


def rows_of(b, start, rows):
    """The rows [start, start + rows) of an elementwise_check Bound over [M, C] (one rank's shard of the world batch)."""
    sl = slice(start, start + rows)
    return ec.Bound(b.ref[sl], b.rnd[sl], b.acc[sl], b.names)
