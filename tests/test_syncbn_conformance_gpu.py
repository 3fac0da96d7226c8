"""SyncBN conformance on one GPU: every statistics producer runs the in-kernel exchange (csrc/seg_sync.cuh) at world > 1
against staged peers (sync_check.StagedPeers), bit for bit.

Before each launch the other ranks' vectors and flags and this rank's seq are written into the symmetric buffers with
ordinary copies, so every wait is already satisfied when the producer reaches it: no rank runs concurrently with another
and no test waits on, or exercises, the timeout.  After each launch:
  - the producer's output holds the host's rank-order world total (float64 statistics / float32 sums) bit for bit;
  - the vector it pushed equals its own output at sync=None on the same input (bn_bwd_fused, whose grid under SyncBN is
    one block per SM smaller, is checked against the float64 sums under the bound of that grid instead);
  - every buffer holds exactly sync_check.expected_after: every other byte, sentinels included, is unchanged;
  - dgamma / dbeta are the local sums.
Every case runs twice on fresh buffers and must be identical.  The concatenated-batch checks run a genuine W-rank batch
through rank r with the float64 references of elementwise_check, the engine checks run Tape(sync=StagedPeers), and the
graph check replays a captured producer.  Each case appends W, rank, epochs, grid and bound usage to
gpu_out_dir/syncbn_conformance.txt."""
import os
import time

import numpy as np
import pytest
import torch

import elementwise_check as ec
import sync_check as sc

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib, ops
    from seg_b200.lib import IMPL_SIMT, IMPL_TC

DEV = "cuda"
EPS, MOM = 1e-5, 0.1
WRAP = (0xFFFFFFFE, 0xFFFFFFFF, 2)  # staged seq values: epochs 0xFFFFFFFF, 2 (the wrap skips 0) and 3
FIRST = (0, 1)                      # epochs 1 and 2: both slot parities


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "syncbn_conformance.txt"), "a")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def rand_bf16(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.randn(shape, generator=g) + offset) * scale).to(DEV, torch.bfloat16)


def host(t):
    return t.detach().cpu().numpy()


def same(case, what, a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    assert a.dtype == b.dtype and a.shape == b.shape, (case, what)
    if a.is_floating_point():
        a, b = a.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]), \
            b.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[b.element_size()])
    assert torch.equal(a, b), f"{case}: {what} differs bit-wise"


# ------------------------------------------------------------------------------------------------ producers
class Producer:
    """One statistics producer on fixed inputs: run(sync) -> dict of outputs, 'vec' the exchanged vector (fp64 [2C]
    statistics or fp32 [2C] sums); local = its 'vec' at sync=None (None for bn_bwd_fused, whose grid changes)."""
    fused = False

    def setup(self):
        self.n = 2 * self.C
        self.need = 2 * self.n if self.dtype == sc.F64 else self.n
        self.plain = self.run(None)
        torch.cuda.synchronize()
        self.local = None if self.fused else host(self.plain["vec"])

    def check_extra(self, case, got, pushed):
        """Outputs other than the exchanged vector equal the unsynced run's (the exchange must not touch them)."""
        for k, v in got.items():
            if k != "vec":
                same(case, k, v, self.plain[k])
        return {}


class ConvFwd(Producer):
    dtype = sc.F64

    def __init__(self, N, H, W, Cin, K, R, impl, seed=1):
        self.C, self.R, self.impl = K, R, impl
        self.x = rand_bf16((N, H, W, Cin), seed)
        w = torch.randn((K, Cin, R, R), generator=torch.Generator().manual_seed(seed + 1)) * (1.0 / (Cin * R * R) ** 0.5)
        self.wp = ops.pack_weight(w.to(DEV))
        self.M = N * H * W
        self.setup()

    def tiles(self):
        return -(-self.M // 128) * -(-self.C // (64 if self.C <= 64 else 128))

    def grid(self):
        if self.impl == IMPL_TC:
            return f"tiles={self.tiles()} grid={min(self.tiles(), sms())}"
        gx, gy, cap = ec.colreduce_grid(self.M, self.C, sms())
        return f"stats_grid={gx}x{gy} cap={cap}"

    def run(self, sync):
        stats = ops.new_stats(self.C, DEV)
        y = ops.conv2d_fwd(self.x, self.wp, self.C, self.R, self.R, 1, self.R // 2, 1, stats=stats, impl=self.impl, sync=sync)
        return {"vec": stats, "y": y}


class DwFwd(Producer):
    dtype = sc.F64

    def __init__(self, N, H, W, C, seed=2):
        self.C, self.M = C, N * H * W
        self.x = rand_bf16((N, H, W, C), seed)
        w = torch.randn((C, 1, 3, 3), generator=torch.Generator().manual_seed(seed + 1)) * 0.3
        self.w9 = ops.dw_pack_weight(w.to(DEV))
        self.setup()

    def grid(self):
        G = self.C // 8
        GB = min(G, 256)
        gy = -(-G // GB)
        gx = max(1, min(-(-self.M // (256 // GB * 2)), -(-sms() * 6 // gy)))
        return f"grid={gx}x{gy}"

    def run(self, sync):
        stats = ops.new_stats(self.C, DEV)
        y = ops.dwconv_fwd(self.x, self.w9, stats=stats, sync=sync)
        return {"vec": stats, "y": y}


class BnStatsP(Producer):
    dtype = sc.F64

    def __init__(self, M, C, seed=3):
        self.C, self.M = C, M
        self.x = rand_bf16((M, C), seed, offset=0.5)
        self.setup()

    def grid(self):
        gx, gy, cap = ec.colreduce_grid(self.M, self.C, sms())
        return f"grid={gx}x{gy} cap={cap}"

    def run(self, sync):
        return {"vec": ops.bn_stats(self.x, sync=sync)}


class BwdInputs:
    """x, dout, gamma, beta and the forward's activation, ReLU bit mask and save (mean, istd) of x."""

    def __init__(self, M, C, seed):
        self.M, self.C = M, C
        self.x = rand_bf16((M, C), seed, offset=0.3)
        self.dout = rand_bf16((M, C), seed + 1)
        g = torch.Generator().manual_seed(seed + 2)
        self.gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
        self.beta = (torch.randn(C, generator=g) * 0.3).to(DEV)
        st = ops.bn_stats(self.x)
        self.mask = ops.relu_mask(self.x)
        self.out, self.save = ops.bn_apply_train(self.x, st, M, self.gamma, self.beta, EPS, MOM, 0, torch.zeros(C, device=DEV),
                                                 torch.ones(C, device=DEV), mask=self.mask)


class BwdReduce(Producer):
    dtype = sc.F32

    def __init__(self, M, C, seed=4):
        self.C, self.M = C, M
        self.b = BwdInputs(M, C, seed)
        self.setup()

    def grid(self):
        gx, gy = ec.reduce2_grid(self.M, self.C, sms())
        return f"grid={gx}x{gy}"

    def run(self, sync):
        b = self.b
        dg, db = torch.empty(self.C, device=DEV), torch.empty(self.C, device=DEV)
        sums = ops.bn_bwd_reduce(b.dout, b.out, b.x, b.save, relu=True, dgamma=dg, dbeta=db, sync=sync)
        return {"vec": sums, "dg": dg, "db": db}

    def check_extra(self, case, got, pushed):
        sc.check_local_param_grads(case, host(got["dg"]), host(got["db"]), pushed)
        return {}


class BwdFused(Producer):
    dtype = sc.F32
    fused = True

    def __init__(self, M, C, mask_src, seed=5):
        self.C, self.M, self.src = C, M, mask_src
        self.b = BwdInputs(M, C, seed)
        self.setup()
        b = self.b
        x2d = b.x.double().cpu()
        save = b.save.cpu()
        amb = None
        if mask_src == "RECOMPUTE":
            mask, amb = ec.remask(x2d, b.gamma.cpu(), b.beta.cpu(), save[:C], save[C:])
        else:
            mask = b.out.double().cpu() > 0
        chain = sc.fused_sync_chain(M, C, sms())
        assert chain <= ec.LONGEST_SUM_CHAIN
        self.ref = ec.BwdRef(b.dout.double().cpu(), x2d, save, b.gamma.cpu(), mask=mask, chain=chain, ambiguous=amb)

    def grid(self):
        f1, f7 = ec.fused_schedule(self.M, self.C, sms(), 1), ec.fused_schedule(self.M, self.C, sms(), 7)
        return f"grid(bps-1 in 1..7)={f1['nb']}..{f7['nb']}x{f1['slabs']}"

    def run(self, sync):
        b = self.b
        dg, db = torch.empty(self.C, device=DEV), torch.empty(self.C, device=DEV)
        kw = {"mask": b.mask} if self.src == "BITS" else {}
        dx, sums = ops.bn_bwd_fused(b.dout, None if self.src == "RECOMPUTE" else b.out, b.x, b.save, b.gamma, self.M * 4,
                                    relu=True, dgamma=dg, dbeta=db, dx=None, beta=b.beta, sync=sync, **kw)
        return {"vec": sums, "dg": dg, "db": db, "dx": dx}

    def check_extra(self, case, got, pushed):
        sc.check_local_param_grads(case, host(got["dg"]), host(got["db"]), pushed)
        u = ec.check(case, "pushed local sums (grid of the synced launch)", torch.from_numpy(pushed.copy()), self.ref.sums_bound())
        return {"sums": u}


def make(kind, size="small"):
    """The producer `kind` at a named size: small, one_block (a one-block grid: its only block is the last), capped (the
    grid cap of the kernel's host function), wide (C = 2064: two channel slabs)."""
    s = sms()
    if kind in ("conv_tc", "conv_simt"):
        impl = IMPL_TC if kind == "conv_tc" else IMPL_SIMT
        if size == "one_block":
            return ConvFwd(1, 8, 16, 64, 64, 1, impl)  # 128 rows: one tile / one stats block
        if size == "capped":  # wgmma: 2 SMs + 1 tiles; CUDA cores: the statistics kernel's grid cap
            return ConvFwd(2 * s + 1 if impl == IMPL_TC else 8 * s + 2, 8, 16, 64, 64, 1, impl)
        return ConvFwd(2, 9, 11, 64, 64, 3, impl)
    if kind == "dwconv":
        if size == "one_block":
            return DwFwd(1, 4, 8, 64)
        if size == "capped":
            return DwFwd(4, 128, 128, 64)
        return DwFwd(2, 9, 11, 48)
    if kind == "bn_stats":
        if size == "one_block":
            return BnStatsP(8, 64)
        if size == "capped":
            return BnStatsP(128 * (s * 8 + 2), 64)
        if size == "wide":
            return BnStatsP(300, 2064)
        return BnStatsP(1000, 48)
    # capped: the cooperative grid is capped at the blocks-per-SM counts the synced launch has (bps - 1 <= 2 under
    # __launch_bounds__(256, 3)) and one more; the map is also over the 24 MB one-launch threshold of the engine
    M, C = {"one_block": (8, 64), "capped": (8 * 16 * (3 * s + 1), 256), "wide": (2000, 2064), "small": (1000, 48)}[size]
    if kind == "bn_bwd_reduce":
        return BwdReduce(M, C)
    return BwdFused(M, C, kind.split(":")[1])


KINDS = ["conv_tc", "conv_simt", "dwconv", "bn_stats", "bn_bwd_reduce", "bn_bwd_fused:ACT", "bn_bwd_fused:RECOMPUTE",
         "bn_bwd_fused:BITS"]


# ------------------------------------------------------------------------------------------------ protocol runner
def run_protocol(log, case, prod, world, rank, seqs, slack=0, seed=0):
    """Stage / launch / check the epochs named by `seqs` (the staged seq of each exchange) on fresh buffers, twice."""
    t0 = time.time()
    n_max = prod.need + slack
    runs, usage = [], {}
    for rep in range(2):
        sp = sc.StagedPeers(world, rank, n_max)
        trace = []
        try:
            for k, seq in enumerate(seqs):
                peers = sc.adversarial(world, rank, prod.n, prod.dtype, seed * 1000 + k)
                e = sp.stage(seq, peers, prod.dtype)
                c = f"{case} W={world} rank={rank} e={e:#x}"
                got = prod.run(sp)
                bufs = sp.read()
                pushed = sc.slot(bufs[rank], world, n_max, e & 1, rank, prod.dtype)[:prod.n].copy()
                if prod.local is not None:
                    sc.check_total(c, pushed, prod.local, "pushed vector vs the sync=None output")
                want, _ = sp.expect(pushed, prod.dtype)
                sc.check_buffers(c, bufs, want, world, n_max, prod.dtype)
                vecs = [peers[p] if p != rank else pushed for p in range(world)]
                sc.check_total(c, host(got["vec"]), sc.world_total(vecs, prod.dtype))
                for k2, u in prod.check_extra(c, got, pushed).items():
                    usage[k2] = max(usage.get(k2, 0.0), u)
                trace.append({k2: v.detach().cpu().clone() for k2, v in got.items()})
                trace[-1]["bufs"] = torch.from_numpy(np.concatenate(bufs))
        finally:
            sp.close()
        runs.append(trace)
    for a, b in zip(*runs):
        for k in a:
            same(case, f"second run: {k}", a[k], b[k])
    epochs = [sc.epoch(s) for s in seqs]
    log(f"protocol {case} W={world} rank={rank} epochs={[hex(e) for e in epochs]} n={prod.n} n_max={n_max} "
        f"{prod.grid()} " + " ".join(f"usage_{k}={v:.4f}" for k, v in usage.items()) + f" wall={time.time() - t0:.1f}s")


@pytest.mark.parametrize("kind", KINDS)
def test_protocol_sweep(log, kind):
    """W in {2, 3, 8, 64} x rank in {0, middle, W - 1} x (epochs 1, 2 | the wrap 0xFFFFFFFF, 2, 3).  n_max is the
    vector's size exactly (4C == n_max, 2C == n_max: the guard after a slot is the next rank's slot) at W = 3 and 64 and
    leaves sentinel slack inside each slot at W = 2 and 8."""
    prod = make(kind)
    for world in (2, 3, 8, 64):
        for rank in sorted({0, world // 2, world - 1}):
            for seqs in (FIRST, WRAP):
                run_protocol(log, kind, prod, world, rank, seqs, slack=0 if world in (3, 64) else 16, seed=world + rank)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", ["one_block", "capped"])
def test_protocol_grids(log, kind, size):
    """The exchanging block at the grid's edges: a one-block grid and the host function's grid cap."""
    prod = make(kind, size)
    if kind.startswith("conv_tc"):
        assert prod.tiles() == (1 if size == "one_block" else 2 * sms() + 1)
    elif kind in ("bn_stats", "conv_simt"):
        gx, _, cap = ec.colreduce_grid(prod.M, prod.C, sms())
        assert gx == (1 if size == "one_block" else cap), prod.grid()
    elif kind.startswith("bn_bwd_fused"):
        for bps1 in (1, 2, 3):
            assert ec.fused_grid(prod.M, prod.C, sms(), bps1)[0] == (1 if size == "one_block" else bps1 * sms())
    elif kind == "bn_bwd_reduce" and size == "one_block":
        assert ec.reduce2_grid(prod.M, prod.C, sms())[0] == 1
    run_protocol(log, f"{kind} {size}", prod, 3, 2, FIRST, seed=7)


@pytest.mark.parametrize("label", ["1", "sms-1", "sms", "sms+1", "2sms+1"])
def test_protocol_conv_tile_counts(log, label):
    """The persistent wgmma grid is min(tiles, SMs): around the SM count one launch mixes CTAs with one tile and with
    two, and each must take exactly one ticket after all its tiles' statistics."""
    s = sms()
    t = {"1": 1, "sms-1": s - 1, "sms": s, "sms+1": s + 1, "2sms+1": 2 * s + 1}[label]
    prod = ConvFwd(t, 8, 16, 64, 64, 1, IMPL_TC)
    assert prod.tiles() == t
    run_protocol(log, f"conv_tc tiles={label}", prod, 8, 7, WRAP, seed=t)


@pytest.mark.parametrize("kind", ["bn_stats", "bn_bwd_reduce", "bn_bwd_fused:ACT", "bn_bwd_fused:BITS"])
def test_protocol_two_slabs(log, kind):
    """C = 2064: gridDim.y = 2 channel slabs; the exchanging block (bn_bwd_fused: block 0) exchanges every slab's totals."""
    prod = make(kind, "wide")
    assert prod.C // 8 > 256
    run_protocol(log, f"{kind} C=2064", prod, 3, 1, FIRST, seed=9)


def test_protocol_forward_then_backward_on_the_same_buffers(log):
    """One step's order: an fp64 forward exchange (conv epilogue), then fp32 backward exchanges (two-launch reduce, fused)
    on the same buffers, epochs 1, 2, 3: each leaves the other parity as the previous one left it."""
    fwd, red, fus = ConvFwd(2, 9, 11, 64, 64, 3, IMPL_TC), BwdReduce(1000, 64), BwdFused(1000, 64, "BITS")
    world, rank = 8, 5
    n_max = fwd.need
    runs = []
    for rep in range(2):
        sp = sc.StagedPeers(world, rank, n_max)
        outs = []
        try:
            for k, prod in enumerate((fwd, red, fus)):
                peers = sc.adversarial(world, rank, prod.n, prod.dtype, 50 + k)
                e = sp.stage(k, peers, prod.dtype)
                assert e == k + 1
                got = prod.run(sp)
                bufs = sp.read()
                pushed = sc.slot(bufs[rank], world, n_max, e & 1, rank, prod.dtype)[:prod.n].copy()
                if prod.local is not None:
                    sc.check_total(f"step e={e}", pushed, prod.local, "pushed vector")
                want, _ = sp.expect(pushed, prod.dtype)
                sc.check_buffers(f"step e={e}", bufs, want, world, n_max, prod.dtype)
                sc.check_total(f"step e={e}", host(got["vec"]),
                               sc.world_total([peers[p] if p != rank else pushed for p in range(world)], prod.dtype))
                prod.check_extra(f"step e={e}", got, pushed)
                outs.append(got["vec"].cpu())
                outs.append(torch.from_numpy(np.concatenate(bufs)))
        finally:
            sp.close()
        runs.append(outs)
    for a, b in zip(*runs):
        same("step", "second run", a, b)
    log(f"step W={world} rank={rank} epochs=1,2,3 n_max={n_max}")


def test_sweep_coverage():
    """The sweep's own coverage from the SM count: tile counts and grids around the SM count, the wrap epoch and both
    n_max boundaries."""
    s = sms()
    assert [sc.epoch(q) for q in WRAP] == [0xFFFFFFFF, 2, 3] and [sc.epoch(q) for q in FIRST] == [1, 2]
    tiles = {1, s - 1, s, s + 1, 2 * s + 1}
    assert all(min(t, s) == (t if t <= s else s) for t in tiles) and any(t > s for t in tiles) and any(t < s for t in tiles)
    gx, _, cap = ec.colreduce_grid(128 * (s * 8 + 2), 64, s)
    assert gx == cap
    assert ec.fused_grid(8 * 16 * (3 * s + 1), 256, s, 3)[0] == 3 * s and 8 * 16 * (3 * s + 1) * 256 * 2 > 24 << 20
    assert ec.fused_grid(2000, 2064, s, 1)[1] == 2


# ------------------------------------------------------------------------------------------------ concatenated batch
def shards(world, rows, C, seed):
    cs = ec.channel_scales(C, seed)
    g = torch.Generator().manual_seed(seed)
    return [ec.bf16_round((torch.randn(rows, C, generator=g, dtype=torch.float64) + 0.4) * cs) for _ in range(world)]


@pytest.mark.parametrize("world", [3, 8])
def test_concatenated_batch_bn(log, world):
    """W shards of one batch: the peers' genuine local totals (bn_stats / bn_bwd_reduce / bn_bwd_fused at sync=None) are
    staged and rank r runs; BatchNorm forward and backward on rank r's rows match the float64 reference of the
    concatenated batch; every rank in turn computes bit-identical world totals."""
    t0 = time.time()
    rows, C = 777, 64
    xs = shards(world, rows, C, 21)
    g = torch.Generator().manual_seed(22)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    douts = [ec.bf16_round(torch.randn(rows, C, generator=g, dtype=torch.float64)) for _ in range(world)]
    xd = [x.to(DEV, torch.bfloat16) for x in xs]
    dd = [d.to(DEV, torch.bfloat16) for d in douts]
    gd, bd = gamma.to(DEV), beta.to(DEV)
    count = world * rows
    local_stats = [host(ops.bn_stats(x)) for x in xd]
    rm0, rv0 = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    usage = {}
    totals = {"stats": [], "two": [], "fused": []}
    for rank in range(world):
        sp = sc.StagedPeers(world, rank, 4 * C)
        try:
            # ---- forward: world statistics, then the single-GPU apply with the world's count
            sp.stage(0, {p: local_stats[p] for p in range(world) if p != rank}, sc.F64)
            stats = ops.bn_stats(xd[rank], sync=sp)
            rm, rv = rm0.to(DEV), rv0.to(DEV)
            mask = ops.relu_mask(xd[rank])
            out, save = ops.bn_apply_train(xd[rank], stats, count, gd, bd, EPS, MOM, 0, rm, rv, mask=mask)
            torch.cuda.synchronize()
            totals["stats"].append(host(stats))
            case = f"concat W={world} rank={rank}"
            st, pre, acc = sc.concat_apply_ref(xs, rank, gamma, beta, EPS)
            usage["apply"] = max(usage.get("apply", 0), ec.check_apply(case, out.reshape(rows, C).double().cpu(), pre, acc))
            usage["save"] = max(usage.get("save", 0), ec.check_save(case, save, st))
            usage["running"] = max(usage.get("running", 0), ec.check_running(case, rm, rv, rm0, rv0, st, MOM))
            # ---- backward: every rank's activation / mask under the world's save, local sums at sync=None
            acts = []
            for p in range(world):
                m_p = ops.relu_mask(xd[p])
                o_p, _ = ops.bn_apply_train(xd[p], stats, count, gd, bd, EPS, MOM, 0, rm0.to(DEV), rv0.to(DEV), mask=m_p)
                acts.append((o_p, m_p))
            same(case, "rank's own activation", acts[rank][0], out)
            mask_h = torch.cat([o.double().cpu() > 0 for o, _ in acts])
            chain = max(ec.bwd_chain_two_launch(rows, C, sms()), sc.fused_sync_chain(rows, C, sms()),
                        ec.bwd_chain_fused(rows, C, sms())) + world
            ref = ec.BwdRef(torch.cat(douts), torch.cat(xs), save.cpu(), gamma, mask=mask_h, chain=chain)
            dxb = sc.rows_of(ref.dx_bound(), rank * rows, rows)
            for path in ("two", "fused"):
                if path == "two":
                    peer = {p: host(ops.bn_bwd_reduce(dd[p], acts[p][0], xd[p], save, mask=acts[p][1]))
                            for p in range(world) if p != rank}
                    e = sp.stage(sp.seq(), peer, sc.F32)
                    sums = ops.bn_bwd_reduce(dd[rank], out, xd[rank], save, mask=mask, sync=sp)
                    dx = ops.bn_bwd_apply(dd[rank], out, xd[rank], save, gd, sums, count, mask=mask)
                else:
                    peer = {p: host(ops.bn_bwd_fused(dd[p], acts[p][0], xd[p], save, gd, count, mask=acts[p][1])[1])
                            for p in range(world) if p != rank}
                    e = sp.stage(sp.seq(), peer, sc.F32)
                    dx, sums = ops.bn_bwd_fused(dd[rank], out, xd[rank], save, gd, count, mask=mask, sync=sp)
                torch.cuda.synchronize()
                totals[path].append(host(sums))
                usage[f"{path}_sums"] = max(usage.get(f"{path}_sums", 0), ec.check(f"{case} {path} e={e}", "world sums", sums, ref.sums_bound()))
                usage[f"{path}_dx"] = max(usage.get(f"{path}_dx", 0),
                                          ec.check(f"{case} {path}", "dx", dx.reshape(rows, C), dxb))
        finally:
            sp.close()
    for k, v in totals.items():
        for r in range(1, world):
            sc.check_total(f"concat W={world} {k}: rank {r} vs rank 0", v[r], v[0])
    log(f"concat W={world} rows={rows} C={C} " + " ".join(f"usage_{k}={u:.4f}" for k, u in usage.items())
        + f" wall={time.time() - t0:.1f}s")


@pytest.mark.parametrize("kind", ["conv_tc", "conv_simt", "dwconv"])
def test_world_totals_identical_on_every_rank(log, kind):
    """Each rank in turn, staged with the others' genuine local statistics (the same producer at sync=None on their
    own shard), computes the same world totals bit for bit."""
    world = 3
    prods = [make(kind) for _ in range(world)]
    if kind.startswith("conv"):
        prods = [ConvFwd(2, 9, 11, 64, 64, 3, IMPL_TC if kind == "conv_tc" else IMPL_SIMT, seed=10 + p) for p in range(world)]
    else:
        prods = [DwFwd(2, 9, 11, 48, seed=10 + p) for p in range(world)]
    got = []
    for rank in range(world):
        sp = sc.StagedPeers(world, rank, prods[0].need)
        try:
            sp.stage(0, {p: prods[p].local for p in range(world) if p != rank}, sc.F64)
            got.append(host(prods[rank].run(sp)["vec"]))
        finally:
            sp.close()
    want = sc.world_total([p.local for p in prods], sc.F64)
    for r in range(world):
        sc.check_total(f"{kind} rank {r}", got[r], want)
    log(f"every-rank {kind} W={world} identical")


# ------------------------------------------------------------------------------------------------ CUDA graph
def test_graph_replay_of_a_producer(log):
    """One conv-fprop producer call captured once and replayed three times, the peers re-staged before each replay by
    copies outside the graph: seq, flags and slots advance exactly as in eager mode and the outputs are bit-identical."""
    prod = ConvFwd(2, 9, 11, 64, 64, 3, IMPL_TC)
    world, rank = 3, 2
    n_max = prod.need
    seqs = (0, 1, 2)
    peers = [sc.adversarial(world, rank, prod.n, sc.F64, 60 + k) for k in range(3)]
    eager = []
    sp = sc.StagedPeers(world, rank, n_max)
    try:
        for k, seq in enumerate(seqs):
            sp.stage(seq, peers[k], sc.F64)
            got = prod.run(sp)
            eager.append((host(got["vec"]), sp.read()))
            sp.expect(prod.local, sc.F64)
    finally:
        sp.close()
    sp = sc.StagedPeers(world, rank, n_max)
    try:
        stats = ops.new_stats(prod.C, DEV)
        tk = torch.zeros(1, dtype=torch.float32, device=DEV)
        y = torch.empty_like(prod.plain["y"])
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                stats.zero_()
                tk.zero_()
                ops.conv2d_fwd(prod.x, prod.wp, prod.C, prod.R, prod.R, 1, prod.R // 2, 1, out=y, stats=stats, impl=IMPL_TC,
                               sync=sp, sync_ticket=tk)
        torch.cuda.synchronize()
        assert sp.seq() == 0xA5A5A5A5, "capture must not run the exchange"
        for k, seq in enumerate(seqs):
            sp.stage(seq, peers[k], sc.F64)
            g.replay()
            bufs = sp.read()
            sc.check_total(f"graph replay {k}", host(stats), eager[k][0])
            same(f"graph replay {k}", "y", y, prod.plain["y"])
            e = k + 1
            pushed = sc.slot(bufs[rank], world, n_max, e & 1, rank, sc.F64)[:prod.n].copy()
            sc.check_total(f"graph replay {k}", pushed, prod.local, "pushed vector")
            want, _ = sp.expect(pushed, sc.F64)
            sc.check_buffers(f"graph replay {k}", bufs, want, world, n_max, sc.F64)
            for b in range(world):
                assert np.array_equal(bufs[b], eager[k][1][b]), f"graph replay {k}: buffer of rank {b} differs from eager"
        del g
    finally:
        sp.close()
    log(f"graph W={world} rank={rank} replays=3 identical to eager")


# ------------------------------------------------------------------------------------------------ descriptor checks
class _Desc:
    """A sync object with a hand-made descriptor (fields of a valid one replaced)."""
    fused, force = True, True

    def __init__(self, base, **fields):
        d = base.desc
        v = dict(peers=d.peers, rank=d.rank, world=d.world, n_max=d.n_max, timeout_clocks=d.timeout_clocks)
        v.update(fields)
        self.desc = lib.SyncDesc(v["peers"], v["rank"], v["world"], v["n_max"], v["timeout_clocks"])
        self.world, self.rank = max(1, v["world"]), v["rank"]


@pytest.mark.parametrize("kind", KINDS)
def test_bad_descriptors_are_refused_before_any_launch(log, kind):
    """Every producer refuses each bad field with an error naming it, before anything is launched: the launch count,
    the ticket, the statistics and every buffer byte stay as they were.  An odd n_max would misalign the fp64 slots."""
    prod = make(kind)
    sp = sc.StagedPeers(3, 1, prod.need)
    try:
        bad = [("peers is NULL", dict(peers=0)), ("world = 0", dict(world=0)), ("world = 65", dict(world=65)),
               ("rank = -1", dict(rank=-1)), ("rank = 3", dict(rank=3)), ("n_max = 0", dict(n_max=0)),
               (f"n_max = {prod.need + 1} must be positive and even", dict(n_max=prod.need + 1)),
               (f"n_max = {prod.need - 2} floats cannot hold", dict(n_max=prod.need - 2))]
        for what, fields in bad:
            n0 = lib.launch_count()
            with pytest.raises(RuntimeError, match=what):
                prod.run(_Desc(sp, **fields))
            assert lib.launch_count() == n0, f"{kind} {what}: launched"
        bufs = sp.read()
        sc.check_buffers(f"{kind} refused descriptors", bufs, sp.images, 3, prod.need, prod.dtype)
        if kind in ("conv_tc", "conv_simt", "dwconv", "bn_stats"):  # the ticket and the statistics stay untouched
            tk = torch.zeros(1, dtype=torch.float32, device=DEV)
            stats = ops.new_stats(prod.C, DEV)
            with pytest.raises(RuntimeError, match="n_max"):
                if kind == "bn_stats":
                    ops.bn_stats(prod.x, stats=stats, sync=_Desc(sp, n_max=prod.need + 1), sync_ticket=tk)
                elif kind == "dwconv":
                    ops.dwconv_fwd(prod.x, prod.w9, stats=stats, sync=_Desc(sp, n_max=prod.need + 1), sync_ticket=tk)
                else:
                    ops.conv2d_fwd(prod.x, prod.wp, prod.C, prod.R, prod.R, 1, prod.R // 2, 1, stats=stats, impl=prod.impl,
                                   sync=_Desc(sp, n_max=prod.need + 1), sync_ticket=tk)
            torch.cuda.synchronize()
            assert int(tk.view(torch.int32).item()) == 0 and not stats.any()
    finally:
        sp.close()
    log(f"refused {kind}: {len(bad)} bad descriptors, no launch")


def test_descriptor_in_device_memory_is_refused():
    L = lib.load()
    sp = sc.StagedPeers(2, 0, 128)
    try:
        x = rand_bf16((64, 32), 1)
        stats = ops.new_stats(32, DEV)
        tk = torch.zeros(1, dtype=torch.float32, device=DEV)
        n0 = lib.launch_count()
        assert L.seg_bn_stats(x.data_ptr(), 64, 32, 32, stats.data_ptr(), sp.peers.data_ptr(), tk.data_ptr(), None) != 0
        assert "host memory" in lib.last_error()
        assert lib.launch_count() == n0
    finally:
        sp.close()


def test_odd_n_max_is_refused_in_python():
    from seg_b200 import comm
    for n_max in (4097, 0, -2):
        with pytest.raises(ValueError, match="n_max"):
            comm.LocalLoopbackGroup(n_max=n_max)


# ------------------------------------------------------------------------------------------------ engine wiring
@pytest.mark.parametrize("case_", ["conv", "conv_res", "conv_two_launch", "dw", "eval", "freeze_bn"])
def test_engine_wiring(log, case_, monkeypatch):
    """Tape(sync=StagedPeers) over conv -> bn_act and depthwise -> bn_act: one in-kernel exchange per producer (the
    statistics are not exchanged a second time), count = count_local * world in both directions, the backward gets the
    descriptor; eval runs no exchange; frozen BN in a training step still has its conv exchange statistics nobody reads
    (nets.py asks for them with want_stats=True) and runs its backward with sync=None."""
    import torch.nn as nn
    from seg_b200.engine import FUSED_BWD_MAX_BYTES, Act, ConvSpec, DwSpec, Tape
    calls = []
    for name in ("bn_apply_train", "bn_bwd_fused", "bn_bwd_reduce", "bn_bwd_apply"):
        def wrap(*a, _f=getattr(ops, name), _n=name, **k):
            calls.append((_n, a, k))
            return _f(*a, **k)
        monkeypatch.setattr(ops, name, wrap)
    world, rank, C = 3, 1, 64
    N, H, W = (2, 330, 330) if case_ == "conv_two_launch" else (2, 17, 17)
    M = N * H * W
    torch.manual_seed(3)
    if case_ == "dw":
        spec = DwSpec("dw", nn.Conv2d(C, C, 3, padding=1, groups=C, bias=False).to(DEV))
    else:
        spec = ConvSpec("c", nn.Conv2d(C, C, 3, padding=1, bias=False).to(DEV))
    bn = nn.BatchNorm2d(C).to(DEV)
    if case_ == "freeze_bn":
        bn.eval()
    x = rand_bf16((N, H, W, C), 5)
    res = Act(rand_bf16((N, H, W, C), 6)) if case_ == "conv_res" else None
    local = host(ops.bn_stats((ops.dwconv_fwd(x, spec.packed()) if case_ == "dw" else
                               ops.conv2d_fwd(x, spec.packed(), C, 3, 3, 1, 1, 1)).reshape(M, C)))
    sp = sc.StagedPeers(world, rank, 4 * C)
    try:
        training = case_ != "eval"
        if training:
            sp.stage(0, {p: local for p in range(world) if p != rank}, sc.F64)
        tape = Tape(training=training, sync=sp)
        xa = Act(x, needs_grad=False)
        ya, stats = (tape.dwconv(xa, spec, want_stats=True) if case_ == "dw" else tape.conv(xa, spec, want_stats=True))
        aa = tape.bn_act(ya, bn, stats=stats, relu=True, res=res)
        torch.cuda.synchronize()
        if not training:
            assert stats is None and sp.seq() == 0xA5A5A5A5, "eval mode must run no exchange"
            assert calls == []
            log(f"engine {case_}: no exchange")
            return
        assert sp.seq() == 1, "one exchange per conv in the forward"
        assert stats.data_ptr() in tape._pushed
        pushed = sc.slot(sp.read()[rank], world, 4 * C, 1, rank, sc.F64)[:2 * C].copy()
        sc.check_total(f"engine {case_}", host(stats), sc.world_total([local if p != rank else pushed for p in range(world)], sc.F64))
        fwd = [c for c in calls if c[0] == "bn_apply_train"]
        if case_ == "freeze_bn":
            assert fwd == []
        else:
            assert len(fwd) == 1 and fwd[0][1][2] == M * world, "forward count must be count_local * world"
        calls.clear()
        if case_ != "freeze_bn":
            g = torch.Generator().manual_seed(8)
            sp.stage(1, {p: (torch.randn(2 * C, generator=g) * 10).numpy() for p in range(world) if p != rank}, sc.F32)
        aa.grad = rand_bf16((N, H, W, C), 7)
        tape.backward()
        torch.cuda.synchronize()
        names = [c[0] for c in calls]
        if case_ == "freeze_bn":
            assert names == ["bn_bwd_fused"] and calls[0][2]["sync"] is None and sp.seq() == 1
        else:
            assert sp.seq() == 2, "one exchange in the backward"
            two = M * C * 2 > FUSED_BWD_MAX_BYTES
            assert names == (["bn_bwd_reduce", "bn_bwd_apply"] if two else ["bn_bwd_fused"]), names
            assert calls[0][2]["sync"] is sp
            count = calls[1][1][6] if two else calls[0][1][5]
            assert count == M * world, "backward count must be count_local * world"
    finally:
        sp.close()
    log(f"engine {case_}: W={world} rank={rank} M={M} exchanges and counts as wired")
