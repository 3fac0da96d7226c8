"""SyncBN exchange: the stand-alone seg_syncbn_exchange (one block running the protocol code of csrc/seg_sync.cuh that the
statistics producers run in their last block) on a single-GPU loopback and on two simulated ranks on one GPU (two streams,
two symmetric buffers); the in-kernel exchange on a one-rank loopback; and — when the box has >= 2 GPUs — a real 2-process
run over CUDA IPC / NVLink peer memory checked against the single-process concatenated batch (the property of
sync_batchnorm/batchnorm.py:160-167)."""
import ctypes
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import comm, lib


def _alloc(world, n_max):
    L = lib.load()
    p = ctypes.c_void_p()
    assert L.seg_comm_alloc(L.seg_comm_buffer_bytes(world, n_max), ctypes.byref(p)) == 0, lib.last_error()
    return p


def test_loopback_world1():
    g = comm.LocalLoopbackGroup(n_max=4096)
    for n in (96, 512, 4096):
        v = torch.randn(n, device="cuda")
        ref = v.clone()
        for _ in range(3):  # repeated exchanges alternate the two slots
            g.allreduce_(v)
        torch.cuda.synchronize()
        assert torch.equal(v, ref)


def test_two_simulated_ranks_exchange_through_the_sync_handle():
    """seg_syncbn_exchange with one seg_sync_desc per rank: the exchange code of the statistics producers, on two streams."""
    L = lib.load()
    n_max = 4096
    bufs = [_alloc(2, n_max), _alloc(2, n_max)]
    peers = torch.tensor([b.value for b in bufs], dtype=torch.int64, device="cuda")
    descs = [comm._make_desc(peers, r, 2, n_max) for r in (0, 1)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    # the handle is read on the host: a device address in its place is refused before anything is launched
    probe = torch.zeros(64, device="cuda")
    assert L.seg_syncbn_exchange(peers.data_ptr(), probe.data_ptr(), 64, None) != 0
    assert "host memory" in lib.last_error()
    for epoch, n in enumerate((128, 2048, 4096, 64), start=1):
        vals = [torch.randn(n, device="cuda"), torch.randn(n, device="cuda")]
        expect = vals[0] + vals[1]
        torch.cuda.synchronize()
        for r in (0, 1):
            with torch.cuda.stream(streams[r]):
                rc = L.seg_syncbn_exchange(ctypes.byref(descs[r]), vals[r].data_ptr(), n, streams[r].cuda_stream)
                assert rc == 0, lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(vals[0], vals[1]), "ranks must end with bit-identical sums"
        assert torch.allclose(vals[0], expect, rtol=0, atol=1e-6)
    for b in bufs:
        L.seg_comm_free(b)


def test_fused_exchange_protocol_on_a_one_rank_loopback():
    """The SyncBN exchange rides inside the kernels that produce the statistics (conv epilogue, BN backward reduction, the
    cooperative BN backward), whose last block runs it from push to advance: run the WHOLE protocol — symmetric-buffer stores, release flags, acquire waits, device-side
    sequence number, slot alternation — against a one-rank buffer.  With one rank the sums are unchanged, so three training
    steps must be bit-identical to the same steps without an exchange, eagerly and replayed from a CUDA graph."""
    import seg_b200
    from seg_b200.train import FusedTrainStep
    from oracle import synth, weights
    sd = weights.deeplab_resnet_state_dict(7, "resnet14", seed=11)
    x, y = synth.make_batch(4, 65, 65, 7, 255, seed=31)
    xd, yd = x.cuda(), y.cuda()
    results = []
    for mode in ("plain", "loopback", "loopback-graph"):
        m = seg_b200.DeepLab(7, backbone="resnet14", pretrained=False)
        m.load_state_dict(sd)
        m.engine_dropout = False
        m = m.cuda().train()
        if mode != "plain":
            m.bn_sync = comm.LocalLoopbackGroup(n_max=8192)
            m.bn_sync.force = True
        st = FusedTrainStep(m, lr=0.01, cuda_graph=(mode == "loopback-graph"))
        losses, after1 = [], None
        for i in range(3):
            losses.append(float(st.step(xd, yd)))
            if i == 0:
                torch.cuda.synchronize()
                after1 = (torch.cat([p.detach().reshape(-1) for p in m.parameters()]).clone(),
                          torch.cat([b.detach().float().reshape(-1) for n, b in m.named_buffers() if "running_" in n]).clone())
        torch.cuda.synchronize()
        results.append((losses, after1))
    l0, (p0, s0) = results[0]
    for losses, (params, stats) in results[1:]:
        # step 1: the forward (exchanged fp64 statistics) is exact -> identical loss and running statistics; the parameters
        # differ only by the fp32 split-K atomics of the weight gradients
        assert losses[0] == l0[0], (losses, l0)
        assert torch.equal(stats, s0)
        assert (params - p0).abs().max().item() <= 1e-5 * p0.abs().max().item()
        # steps 2-3 exercise the slot alternation / sequence number; that last-bit weight noise is amplified by the network
        assert all(abs(a - b) < 2e-2 * abs(b) for a, b in zip(losses[1:], l0[1:])), (losses, l0)


def _worker(rank, world, port, out_path, graph=False, nsteps=1):
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "pytorch-segmentation_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import seg_b200
    from seg_b200 import comm as C
    from seg_b200.train import FusedTrainStep
    from oracle import synth, weights
    sd = weights.deeplab_resnet_state_dict(7, "resnet14", seed=11, randomize_bn=True)
    x, y = synth.make_batch(4, 65, 65, 7, 255, seed=31)
    m = seg_b200.DeepLab(7, backbone="resnet14")
    m.load_state_dict(sd)
    m.engine_dropout = False
    m = m.cuda().train()
    m.bn_sync = C.SyncBNGroup()
    half = slice(rank * 2, rank * 2 + 2)
    st = FusedTrainStep(m, world=world, cuda_graph=graph)
    for _ in range(nsteps):
        loss = st.step(x[half].cuda(), y[half].cuda())
    lt = loss.detach().clone()
    dist.all_reduce(lt)
    # the replicas must stay bit-equal: identical world statistics and one all-reduced gradient on every rank
    mine = torch.cat([p.detach().float().reshape(-1) for p in m.parameters()]
                     + [b.detach().float().reshape(-1) for n, b in m.named_buffers() if "running_" in n])
    every = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(every, mine)
    replicas_equal = all(torch.equal(every[0].view(torch.int32), e.view(torch.int32)) for e in every[1:])
    if rank == 0:
        m1 = seg_b200.DeepLab(7, backbone="resnet14")
        m1.load_state_dict(sd)
        m1.engine_dropout = False
        m1 = m1.cuda().train()
        st1 = FusedTrainStep(m1, world=1)
        for _ in range(nsteps):
            loss1 = st1.step(x.cuda(), y.cuda())
        upd2 = torch.cat([(p.detach().cpu() - sd[n]).reshape(-1) for n, p in m.named_parameters()])
        upd1 = torch.cat([(p.detach().cpu() - sd[n]).reshape(-1) for n, p in m1.named_parameters()])
        rs2 = torch.cat([b.detach().cpu().float().reshape(-1) for n, b in m.named_buffers() if "running_" in n])
        rs1 = torch.cat([b.detach().cpu().float().reshape(-1) for n, b in m1.named_buffers() if "running_" in n])
        torch.save({"loss2": (lt / world).item(), "loss1": loss1.item(), "replicas_equal": replicas_equal,
                    "cos": torch.nn.functional.cosine_similarity(upd2.double(), upd1.double(), dim=0).item(),
                    "stats_rel": ((rs2 - rs1).abs().max() / rs1.abs().max()).item()}, out_path)
    st.release_graph()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_syncbn_train_step_equals_single_gpu_on_concatenated_batch(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r.pt")
    mp.spawn(_worker, args=(2, 29600 + os.getpid() % 1000, out), nprocs=2, join=True)
    r = torch.load(out)
    print(r)
    assert r["replicas_equal"], "rank 1's parameters / running statistics differ from rank 0's"
    assert abs(r["loss2"] - r["loss1"]) < 2e-2 * abs(r["loss1"])
    assert r["stats_rel"] < 2e-2
    assert r["cos"] > 0.95


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_graph_captured_steps_equal_single_gpu_eager_steps(tmp_path):
    """The whole 2-rank step — SyncBN peer exchanges and the NCCL gradient all-reduce included — replayed from a CUDA
    graph three times equals three eager single-GPU steps on the concatenated batch (the capture's warm-up steps are
    rolled back, the device-side exchange sequence number keeps the replays in lockstep)."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "r.pt")
    mp.spawn(_worker, args=(2, 29600 + (os.getpid() + 7) % 1000, out, True, 3), nprocs=2, join=True)
    r = torch.load(out)
    print(r)
    assert r["replicas_equal"], "rank 1's parameters / running statistics differ from rank 0's"
    assert abs(r["loss2"] - r["loss1"]) < 3e-2 * abs(r["loss1"])
    assert r["stats_rel"] < 3e-2
    assert r["cos"] > 0.9
