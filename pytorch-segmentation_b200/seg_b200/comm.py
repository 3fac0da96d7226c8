"""Multi-GPU plumbing: one process per GPU (torchrun), torch.distributed/NCCL for the gradient all-reduce, and the symmetric
NVLink peer buffers of the SyncBN statistics exchange.

Replaces the reference's single-process nn.DataParallel + threaded SyncBN (base/base_trainer.py:33-38,
utils/sync_batchnorm/batchnorm.py:105-126, comm.py): batch-dim sharding stays, the per-step parameter broadcast and logit gather
disappear, and the two small collectives per BN layer ride inside the kernels that produce the statistics (csrc/seg_sync.cuh;
`SyncBNGroup.desc` is the descriptor those kernels take): the producer's last block performs the whole exchange and leaves the
world's totals in its output, so the kernels that consume them are the single-GPU ones.  The stand-alone exchange
(`allreduce_`, `seg_syncbn_exchange`) is one block running the same protocol code with the same descriptor, for callers outside
the engine.
"""
import ctypes

import torch
import torch.distributed as dist

from . import lib


def _sync_timeout_clocks():
    """Spin-wait bound of the in-kernel exchange in GPU clocks (~2 GHz): SEG_SYNC_TIMEOUT_S seconds, default 120 — rank skew
    from a slow data loader or a checkpoint write on one rank must not kill the job; 0 = wait forever."""
    import os
    return int(float(os.environ.get("SEG_SYNC_TIMEOUT_S", "120")) * 2e9)


def _check_n_max(n_max):
    """The fp64 forward statistics address each rank's slot of n_max floats as doubles: n_max must be even for every
    slot to be 8-byte aligned (the kernels' entry points refuse an odd one too)."""
    if not (isinstance(n_max, int) and n_max > 0 and n_max % 2 == 0):
        raise ValueError(f"SyncBN: n_max must be a positive even number of floats, got {n_max!r}")


def _make_desc(peers, rank, world, n_max):
    return lib.SyncDesc(peers.data_ptr(), rank, world, n_max, _sync_timeout_clocks())


class SyncBNGroup:
    """Symmetric peer buffers for `seg_syncbn_exchange`.  `allreduce_(vec)` sums an fp32 vector
    (<= n_max floats) over all ranks in place, bit-identically on every rank."""

    def __init__(self, n_max=8192, group=None):
        _check_n_max(n_max)
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.n_max = n_max
        L = lib.load()
        nbytes = L.seg_comm_buffer_bytes(self.world, n_max)
        mine = ctypes.c_void_p()
        if L.seg_comm_alloc(nbytes, ctypes.byref(mine)) != 0:
            raise RuntimeError(lib.last_error())
        self._mine = mine
        handle = (ctypes.c_char * 64)()
        if L.seg_comm_ipc_get(mine, handle) != 0:
            raise RuntimeError(lib.last_error())
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle), group=group)
        ptrs = []
        self._opened = []
        for r, h in enumerate(handles):
            if r == self.rank:
                ptrs.append(mine.value)
                continue
            p = ctypes.c_void_p()
            buf = ctypes.create_string_buffer(h, 64)
            if L.seg_comm_ipc_open(buf, ctypes.byref(p)) != 0:
                raise RuntimeError(lib.last_error())
            self._opened.append(p)
            ptrs.append(p.value)
        self.peers = torch.tensor(ptrs, dtype=torch.int64, device="cuda")
        self.desc = _make_desc(self.peers, self.rank, self.world, n_max)
        self.fused = True  # the kernels that produce / consume the statistics carry the exchange (csrc/seg_sync.cuh)
        dist.barrier(group=group)

    def allreduce_(self, vec):
        assert vec.dtype == torch.float32 and vec.is_contiguous() and vec.numel() <= self.n_max
        lib.call("seg_syncbn_exchange", ctypes.addressof(self.desc), vec.data_ptr(), vec.numel())
        return vec

    def close(self):
        L = lib.load()
        torch.cuda.synchronize()
        for p in self._opened:
            L.seg_comm_ipc_close(p)
        L.seg_comm_free(self._mine)
        self._opened = []


class LocalLoopbackGroup:
    """world == 1 stand-in with the same interface (used by single-GPU tests of the exchange kernel)."""

    def __init__(self, n_max=8192):
        _check_n_max(n_max)
        self.rank, self.world, self.n_max = 0, 1, n_max
        L = lib.load()
        mine = ctypes.c_void_p()
        if L.seg_comm_alloc(L.seg_comm_buffer_bytes(1, n_max), ctypes.byref(mine)) != 0:
            raise RuntimeError(lib.last_error())
        self._mine = mine
        self.peers = torch.tensor([mine.value], dtype=torch.int64, device="cuda")
        self.desc = _make_desc(self.peers, 0, 1, n_max)
        self.fused = True
        self.force = False  # True: the engine runs the whole SyncBN protocol (push, flags, wait, sequence number) against
                            # this one-rank buffer — the single-GPU test of the fused exchange

    def allreduce_(self, vec):
        lib.call("seg_syncbn_exchange", ctypes.addressof(self.desc), vec.data_ptr(), vec.numel())
        return vec


def dp_world(group=None):
    """Number of data-parallel replicas (1 without an initialised process group)."""
    return dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1


def dp_rank(group=None):
    return dist.get_rank(group) if (dist.is_available() and dist.is_initialized()) else 0


def allreduce_mean_(flat, world):
    """Gradient exchange of the data-parallel path (what nn.DataParallel's reduce-to-device-0 + next step's broadcast do
    in the reference, base/base_trainer.py:33-38 / trainer.py:70-71): ONE NCCL all-reduce of the flat fp32 gradient
    buffer, then the 1/world scale.  Identical result on every rank, so replicas stay bit-equal."""
    dist.all_reduce(flat)
    flat.mul_(1.0 / world)
    return flat


def init_distributed():
    """Initialise torch.distributed from the torchrun environment (no-op for a single process)."""
    import os
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return 0, 1, 0
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return rank, world, local
