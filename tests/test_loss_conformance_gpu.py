"""Conformance sweep of the loss and metric kernels on NCHW fp32 logits: cross-entropy, class-weighted CE and focal loss
(seg_loss_nchw_fwd / _bwd / seg_loss_finalize), Dice (seg_dice_nchw_fwd / _bwd), Lovász-softmax (seg_lovasz_count /
seg_lovasz_softmax_nchw), eval_metrics (seg_eval_metrics_nchw), and the fused losses of the training step: bilinear
upsample + loss (seg_upsample_loss_fwd / _bwd: loss, arg-max map, counters, fp32 dlo and the padded bf16 dx) and pixel
shuffle + loss (seg_shuffle_loss_fwd / _bwd), called through the C ABI.

Every case is checked element by element against a float64 reference with the bounds of tests/loss_check.py, computed
on the GPU in float64.  The logits sit inside sentinel (NaN) buffers, so a read past them poisons the result; the
gradients are written into sentinel-guarded buffers whose guards must come back bit for bit and whose every element must
have been written; the eval_metrics counters sit between int64 sentinel words.  Every case runs twice: gradients,
counters, the fp32 loss and accum[1] must be bit-identical.  accum[0] (the per-pixel loss sum) is an fp64 atomic sum,
exact only while its addends' exponents span fewer than about 29 bits, which tiny focal terms break; it is checked
against its bound on each run instead.  Each case appends its bound usage, the regime it asserted and its wall time to
gpu_out_dir/loss_conformance.txt.

The schedule cases are sized from the SM count with the host grid mirrors (loss_check.nchw_grid, lovasz_schedule,
upsample_schedule) and assert the regime they name.  Lovász runs with the tie-order check: exactly tied errors take ranks in pixel order."""
import os
import time

import pytest
import torch

import conv_check as cc
import loss_check as lc

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib, ops
    from seg_b200.lib import ptr

DEV = "cuda"
F32, F64, I64, I32, BF16 = torch.float32, torch.float64, torch.int64, torch.int32, torch.bfloat16
KIND = {"ce": 0, "wce": 1, "focal": 2}


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "loss_conformance.txt"), "a")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def place(z):
    """z (fp32) as a dense device tensor inside a sentinel buffer."""
    g = cc.FlatGuarded(tuple(z.shape), F32, device=DEV)
    g.view.copy_(z.to(DEV))
    return g.view


def out_buf(shape, old=None):
    g = cc.FlatGuarded(tuple(shape), F32, device=DEV)
    if old is not None:
        g.view.copy_(old.to(DEV))
    return g


def settle(case, g):
    torch.cuda.synchronize()
    cc.check_guards(case, g.buf, g.guard_mask())
    cc.check_written(case, g.view)


def same_bits(case, what, a, b):
    ia = a.view(I32) if a.dtype == F32 else (a.view(I64) if a.dtype == F64 else a)
    ib = b.view(I32) if b.dtype == F32 else (b.view(I64) if b.dtype == F64 else b)
    assert torch.equal(ia, ib), f"{case}: {what} not bit-reproducible"


def pixels_shape(npix):
    """(N, H, W) with N * H * W = npix and a ragged last image row."""
    W = 97
    if npix < W:
        return 1, 1, npix
    H = npix // W
    if npix % W == 0:
        return 1, H, W
    return 1, 1, npix


# ------------------------------------------------------------------------------------------------ CE / WCE / focal
def run_loss(log, case, z, t, ignore, kind, gamma=0.0, mean=True, weight=None, gscale=1.0, regime=""):
    t0 = time.time()
    N, C, H, W = z.shape
    zd, td = place(z), t.to(DEV)
    wd = None if weight is None else weight.to(DEV, F32).contiguous()
    gs = torch.tensor([gscale], dtype=F32, device=DEV)
    runs = []
    for _ in range(2):
        accum = torch.zeros(2, dtype=F64, device=DEV)
        lib.call("seg_loss_nchw_fwd", ptr(zd), ptr(td), N, C, H, W, int(ignore), ptr(wd), KIND[kind], float(gamma), ptr(accum))
        loss = torch.empty(1, dtype=F32, device=DEV)
        lib.call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
        dl = out_buf((N, C, H, W))
        lib.call("seg_loss_nchw_bwd", ptr(zd), ptr(td), N, C, H, W, int(ignore), ptr(wd), KIND[kind], float(gamma),
                 int(mean), ptr(accum), ptr(gs), ptr(dl.view))
        settle(case, dl)
        runs.append((accum.clone(), loss.clone(), dl.view.clone()))
    (a0, l0, d0), (a1, l1, d1) = runs
    same_bits(case, "dlogits", d0, d1)
    same_bits(case, "loss", l0, l1)
    same_bits(case, "accum[1]", a0[1:], a1[1:])
    r = lc.LossRef(zd.double(), td, ignore, kind, wd, gamma, mean)
    ua = max(r.check_accum(case, a0), r.check_accum(case, a1))
    ul = r.check_loss(case, l0.item())
    ug = lc.check(case, "dlogits", d0, r.grad_bound(gscale))
    log(f"{case}: usage accum0={ua:.4f} loss={ul:.4f} grad={ug:.4f} {regime} time={time.time() - t0:.2f}s")


def nchw_counts():
    s = sms() * 8 * 256
    return [1, 255, 257, s - 1, s, s + 1, 3 * s + 17]


# An unweighted 'sum' is SEG_LOSS_WCE without weights (SEG_LOSS_CE is a mean by contract; test_loss_ce_kind_is_a_mean).
@pytest.mark.parametrize("kind,gamma,mean,weighted", [("ce", 0.0, True, False), ("wce", 0.0, False, False),
                                                      ("wce", 0.0, True, True), ("wce", 0.0, False, True),
                                                      ("focal", 0.0, True, True), ("focal", 0.5, True, True),
                                                      ("focal", 0.5, False, False), ("focal", 2.0, False, True)])
def test_loss_nchw_schedule(log, kind, gamma, mean, weighted):
    for i, npix in enumerate(nchw_counts()):
        C = (150, 21, 2)[i] if npix < 10000 else (19 if i % 2 else 7)
        N, H, W = pixels_shape(npix)
        z = lc.logits(N, C, H, W, 100 + i, sat=npix >= 64)
        t = lc.labels(N, H, W, C, 200 + i)
        w = lc.weights(C, 300 + i) if weighted else None
        blocks, iters, capped = lc.nchw_grid(npix, sms())
        if npix > sms() * 8 * 256:
            assert capped and iters >= 2
        run_loss(log, f"loss {kind} g={gamma} mean={mean} weighted={weighted} npix={npix} C={C}", z, t, 255, kind, gamma,
                 mean, w, 0.375, f"blocks={blocks} iters={iters} capped={capped}")


def test_loss_ce_kind_is_a_mean():
    """SEG_LOSS_CE takes no weight and is a mean; anything else is rejected on the host."""
    z = torch.zeros(1, 3, 4, 4, dtype=F32, device=DEV)
    t = torch.zeros(1, 4, 4, dtype=I64, device=DEV)
    w = torch.ones(3, dtype=F32, device=DEV)
    accum = torch.ones(2, dtype=F64, device=DEV)
    dl = torch.empty_like(z)
    for weight, mean in ((None, 0), (w, 1)):
        with pytest.raises(RuntimeError, match="SEG_LOSS_CE"):
            lib.call("seg_loss_nchw_bwd", ptr(z), ptr(t), 1, 3, 4, 4, 255, ptr(weight), 0, 0.0, mean, ptr(accum), None,
                     ptr(dl))


@pytest.mark.parametrize("ignore", [255, -1, 0])
def test_loss_nchw_ignore_and_edges(log, ignore):
    C = 19
    for kind, gamma in (("ce", 0.0), ("wce", 0.0), ("focal", 0.5), ("focal", 2.0)):
        w = lc.weights(C, 5) if kind != "ce" else None
        z = lc.logits(2, C, 33, 37, 7, sat=True)
        t = lc.labels(2, 33, 37, C, 8, ignore=ignore)
        t[1] = ignore  # a fully ignored image
        run_loss(log, f"loss {kind} g={gamma} ignore={ignore} image ignored", z, t, ignore, kind, gamma, True, w, 1.5)
        run_loss(log, f"loss {kind} g={gamma} ignore={ignore} batch ignored", z, torch.full_like(t, ignore), ignore, kind,
                 gamma, True, w, 1.0)
    w = lc.weights(C, 5)
    # only zero-weight classes (0 and 5) present
    tz = torch.where(torch.rand(2, 33, 37, generator=torch.Generator().manual_seed(10)) < 0.5, 0, 5)
    for kind, gamma in (("wce", 0.0), ("focal", 2.0)):
        run_loss(log, f"loss {kind} ignore={ignore} zero-weight classes only", lc.logits(2, C, 33, 37, 9), tz, 255, kind,
                 gamma, True, w, 1.0)


# ------------------------------------------------------------------------------------------------ Dice
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_dice(log, beta):
    for C, npix in ((7, 33 * 37 * 2), (19, 3 * sms() * 8 * 256 + 17)):
        t0 = time.time()
        N, H, W = pixels_shape(npix)
        z = lc.logits(N, C, H, W, 40 + C, sat=True)
        t = lc.dice_fixup(lc.labels(N, H, W, C, 41 + C), 255)
        zd, td = place(z), t.to(DEV)
        gs = torch.tensor([0.625], dtype=F32, device=DEV)
        old = torch.randn(N, C, H, W) if beta else None
        runs = []
        for _ in range(2):
            accum = torch.zeros(2, dtype=F64, device=DEV)
            loss = torch.empty(1, dtype=F32, device=DEV)
            lib.call("seg_dice_nchw_fwd", ptr(zd), ptr(td), N, C, H, W, 1.0, ptr(accum), ptr(loss))
            dl = out_buf((N, C, H, W), old)
            lib.call("seg_dice_nchw_bwd", ptr(zd), ptr(td), N, C, H, W, ptr(accum), 1.0, ptr(gs), ptr(dl.view), float(beta))
            settle("dice", dl)
            runs.append((accum.clone(), loss.clone(), dl.view.clone()))
        case = f"dice C={C} npix={npix} beta={beta}"
        same_bits(case, "dlogits", runs[0][2], runs[1][2])
        same_bits(case, "loss", runs[0][1], runs[1][1])
        same_bits(case, "accum[1]", runs[0][0][1:], runs[1][0][1:])
        r = lc.DiceRef(zd.double(), td, 1.0)
        uf = max(r.check_fwd(case, runs[0][0], runs[0][1].item()), r.check_fwd(case, runs[1][0], runs[1][1].item()))
        ug = lc.check(case, "dlogits", runs[0][2], r.grad_bound(0.625, beta, old))
        blocks, iters, capped = lc.nchw_grid(npix, sms())
        log(f"{case}: usage fwd={uf:.4f} grad={ug:.4f} blocks={blocks} iters={iters} capped={capped} "
            f"time={time.time() - t0:.2f}s")


# ------------------------------------------------------------------------------------------------ Lovász
def lovasz_call(zd, td, ignore):
    N, C, H, W = zd.shape
    counts = torch.empty(C + 1, dtype=I32, device=DEV)
    lib.call("seg_lovasz_count", ptr(td), N * H * W, C, int(ignore), ptr(counts))
    ch = counts.cpu()
    P, n_present = int(ch[C]), int((ch[:C] > 0).sum())
    nkeys = max(P * n_present, 1)
    keys0 = torch.empty(nkeys, dtype=I64, device=DEV)
    keys1 = torch.empty(nkeys, dtype=I64, device=DEV)
    ws = torch.empty(int(lib.load().seg_lovasz_workspace_bytes(P, n_present, C)), dtype=torch.uint8, device=DEV)
    loss = torch.empty(1, dtype=F32, device=DEV)
    dl = out_buf((N, C, H, W))
    lib.call("seg_lovasz_softmax_nchw", ptr(zd), ptr(td), N, C, H, W, int(ignore), ptr(counts), P, n_present,
             ptr(keys0), ptr(keys1), ptr(ws), ptr(loss), ptr(dl.view))
    settle("lovasz", dl)
    del keys0, keys1, ws
    return loss, dl.view, P, n_present


def run_lovasz(log, case, z, t, ignore=255, regime_check=None):
    t0 = time.time()
    N, C, H, W = z.shape
    zd, td = place(z), t.to(DEV)
    l0, d0, P, n_present = lovasz_call(zd, td, ignore)
    l1, d1, _, _ = lovasz_call(zd, td, ignore)
    same_bits(case, "loss", l0, l1)
    same_bits(case, "dlogits", d0, d1)
    del d1
    s = lc.lovasz_schedule(N * H * W, P, n_present, sms())
    if regime_check is not None:
        regime_check(s)
    r = lc.LovaszRef(zd.double(), td, ignore, tie_order=True)
    assert (P, n_present) == (r.P, len(r.present))
    ul = r.check_loss(case, l0.item())
    ug = lc.check(case, "dlogits", d0, r.grad)
    log(f"{case}: usage loss={ul:.4f} grad={ug:.4f} P={P} n_present={n_present} tied_clusters={r.pure_tie_clusters} "
        + " ".join(f"{k}={v}" for k, v in s.items()) + f" time={time.time() - t0:.2f}s")
    return r


@pytest.mark.parametrize("C", [2, 19, 150])
def test_lovasz_classes(log, C):
    z = lc.logits(2, C, 61, 67, 50 + C, sat=True)
    t = lc.labels(2, 61, 67, C, 51 + C)
    run_lovasz(log, f"lovasz C={C}", z, t)
    run_lovasz(log, f"lovasz C={C} ignore=-1", z, lc.labels(2, 61, 67, C, 52 + C, ignore=-1), ignore=-1)


def test_lovasz_edges(log):
    # LV_MAXC classes, all present (rank 255)
    C = lc.LV_MAXC
    z = lc.logits(1, C, 64, 64, 60)
    t = torch.arange(64 * 64).view(1, 64, 64) % C
    run_lovasz(log, "lovasz C=256 all present", z, t, ignore=-1)
    z = lc.logits(1, 19, 45, 91, 61, sat=True)
    t = lc.labels(1, 45, 91, 19, 62)
    t1 = torch.where(t == 3, 4, t)
    t1[0, 44, 90] = 3  # one foreground pixel in class 3, the last pixel of the batch
    run_lovasz(log, "lovasz one fg pixel", z, t1)
    run_lovasz(log, "lovasz one present class", z, torch.where(t == 255, t, torch.full_like(t, 7)))
    t2 = t.clone()
    t2[0, :5] = 19 + (torch.arange(91) % 3)  # labels >= C, not ignored: valid, background for every class
    run_lovasz(log, "lovasz labels >= C", z, t2)
    run_lovasz(log, "lovasz fg at tile edges", *lovasz_tile_edge_case(), regime_check=lambda s: s["tiles"] == 4)
    # only void pixels: loss 0, gradient 0
    zd = place(z)
    loss, dl, P, _ = lovasz_call(zd, torch.full((1, 45, 91), 255, dtype=I64, device=DEV), 255)
    assert P == 0 and loss.item() == 0.0 and not bool(dl.any())


def lovasz_tile_edge_case(P=3 * lc.LV_JT + 100, seed=63):
    """C = 2 with every error placed on a grid 1 / (P + 2) apart (far above its allowance), so the sorted order of
    class 1 is known: rank k holds error 1 - (k + 1) / (P + 2).  Foreground pixels of class 1 sit at ranks LV_JT - 1,
    LV_JT, LV_JT + 1, 2 LV_JT - 1, 2 LV_JT and 3 LV_JT (the first and last keys of jaccard tiles, so the foreground
    count carried into a tile decides their steps) and at a random quarter of the other ranks."""
    g = torch.Generator().manual_seed(seed)
    J = lc.LV_JT
    fg = torch.rand(P, generator=g, dtype=torch.float64) < 0.25
    fg[[J - 1, J, J + 1, 2 * J - 1, 2 * J, 3 * J]] = True
    err = 1 - (torch.arange(P, dtype=torch.float64) + 1) / (P + 2)
    p1 = torch.where(fg, 1 - err, err)                   # class-1 probability giving that error
    s1 = torch.log(p1) - torch.log1p(-p1)                # logits (0, s1): softmax p_1 = sigmoid(s1)
    perm = torch.randperm(P, generator=g)                 # rank -> pixel
    z = torch.zeros(1, 2, 1, P)
    z[0, 1, 0, perm] = s1.float()
    t = torch.zeros(1, 1, P, dtype=I64)
    t[0, 0, perm] = fg.long()
    return z, t


def test_lovasz_ties(log):
    """Thousands of groups of pixels with bit-identical logit vectors, spread over an image whose emission grid strides
    several times, so that group members fall in different blocks and iterations."""
    z, t = lc.tie_case(N=1, C=19, H=1024, W=2048, seed=70, groups=3000, size=6)

    def regime(s):
        assert s["emit_iters"] >= 2 and s["emit_blocks"] == sms() * 8

    r = run_lovasz(log, "lovasz planted ties", z, t, regime_check=regime)
    assert r.pure_tie_clusters >= 1000


def test_lovasz_largest(log):
    """N*H*W = 2^23 - 1 pixels at C = 8: the radix row scan with more than 1024 blocks per digit (per > 1) and the class
    scan with more than 1024 tiles."""
    n = 2 ** 23 - 1
    z, t = lc.lovasz_case(1, 8, 1, n, seed=80)

    def regime(s):
        assert s["nblocks"] > 1024 and s["radix_per"] > 1 and s["tiles"] > 1024 and s["class_scan_per"] > 1

    run_lovasz(log, "lovasz 2^23-1 pixels", z, t, regime_check=regime)


def test_lovasz_limits():
    """Rejected on the host, before any launch."""
    td = torch.zeros(1, 1, 64, dtype=I64, device=DEV)
    counts = torch.empty(258, dtype=I32, device=DEV)
    with pytest.raises(RuntimeError, match="at most 256 classes"):
        lib.call("seg_lovasz_count", ptr(td), 64, 257, 255, ptr(counts))
    n = 2 ** 23
    zd = torch.zeros(1, 8, 1, n, dtype=F32, device=DEV)
    td = torch.zeros(1, 1, n, dtype=I64, device=DEV)
    with pytest.raises(RuntimeError, match="2\\^23 pixels"):
        lib.call("seg_lovasz_softmax_nchw", ptr(zd), ptr(td), 1, 8, 1, n, 255, ptr(counts), n, 1, None, None, None,
                 ptr(zd), ptr(zd))


# ------------------------------------------------------------------------------------------------ eval_metrics
@pytest.mark.parametrize("K", [7, 19, 150])
def test_eval_metrics(log, K):
    s = sms() * 8 * 256
    for C, npix, ignore in ((K, 2 * 33 * 37, 255), (K + 3, 3 * s + 17, -1), (K, s + 1, 255)):
        t0 = time.time()
        N, H, W = pixels_shape(npix)
        z = lc.logits(N, C, H, W, 90 + K)
        flat = z.permute(0, 2, 3, 1).reshape(-1, C)
        tie = torch.arange(0, N * H * W, 5)
        a, b = 1 % C, (C - 2)
        flat[tie, a] = flat[tie, b] = flat[tie].amax(1) + 1  # planted first-max ties
        z = flat.view(N, H, W, C).permute(0, 3, 1, 2).contiguous()
        t = lc.labels(N, H, W, C, 91 + K, ignore=ignore)
        zd, td = place(z), t.to(DEV)
        outs = []
        for _ in range(2):
            buf = lc.int_sentinel_fill(torch.empty(8 + 2 + 3 * K + 8, dtype=I64, device=DEV))
            lib.call("seg_eval_metrics_nchw", ptr(zd), ptr(td), N, C, H, W, K, ptr(buf[8:]))
            torch.cuda.synchronize()
            lc.check_int_guards("eval_metrics", buf, 8, 2 + 3 * K)
            outs.append(buf[8:8 + 2 + 3 * K].cpu())
        case = f"eval_metrics K={K} C={C} npix={npix} ignore={ignore}"
        assert torch.equal(outs[0], outs[1]), f"{case}: counters not reproducible"
        lc.check_exact(case, "counters", outs[0], lc.metrics_ref(zd, td, K), ("i",))
        blocks, iters, capped = lc.nchw_grid(npix, sms())
        log(f"{case}: exact blocks={blocks} iters={iters} capped={capped} time={time.time() - t0:.2f}s")
    # everything ignored
    zd = place(lc.logits(1, K, 17, 19, 95))
    out = torch.empty(2 + 3 * K, dtype=I64, device=DEV)
    lib.call("seg_eval_metrics_nchw", ptr(zd), ptr(torch.full((1, 17, 19), 255, dtype=I64, device=DEV)), 1, K, 17, 19, K,
             ptr(out))
    assert not bool(out.any())


# ------------------------------------------------------------------------------------------------ fused upsample
def int_buf(n, dtype, zero=False):
    """An int view of n words between int sentinel guards; (buffer, view)."""
    buf = lc.int_sentinel_fill(torch.empty(8 + n + 8, dtype=dtype, device=DEV))
    if zero:
        buf[8:8 + n].zero_()
    return buf, buf[8:8 + n]


def run_upsample(log, case, lo, t, ac, kind="ce", gamma=0.0, mean=True, weight=None, gscale=0.75, ignore=255,
                 regime=None):
    t0 = time.time()
    N, Hi, Wi, C = lo.shape
    Ho, Wo = t.shape[1:]
    lod, td = place(lo), t.to(DEV)
    wd = None if weight is None else weight.to(DEV, F32).contiguous()
    gs = torch.tensor([gscale], dtype=F32, device=DEV)
    s = lc.upsample_schedule(Hi, Wi, Ho, Wo, C, ac)
    assert s["fwd_ok"] and s["bwd_ok"], (case, s)
    if regime is not None:
        regime(s)
    lddx = C + 3
    M = N * Hi * Wi
    runs = []
    for _ in range(2):
        accum = torch.zeros(2, dtype=F64, device=DEV)
        abuf, am = int_buf(N * Ho * Wo, I32)
        cbuf, cnt = int_buf(2 + 3 * C, I64, zero=True)
        lib.call("seg_upsample_loss_fwd", ptr(lod), ptr(td), N, Hi, Wi, Ho, Wo, C, ac, int(ignore), ptr(wd), KIND[kind],
                 float(gamma), ptr(accum), ptr(am), ptr(cnt))
        loss = torch.empty(1, dtype=F32, device=DEV)
        lib.call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
        dlo = out_buf((N, Hi, Wi, C))
        fixed = torch.empty(M * C, dtype=I64, device=DEV)
        dx = cc.FlatGuarded((M, lddx), BF16, device=DEV)
        lib.call("seg_upsample_loss_bwd", ptr(lod), ptr(td), N, Hi, Wi, Ho, Wo, C, ac, int(ignore), ptr(wd), KIND[kind],
                 float(gamma), int(mean), ptr(accum), ptr(gs), ptr(dlo.view), ptr(fixed), ptr(dx.view), lddx)
        settle(case, dlo)
        settle(case, dx)
        lc.check_int_guards(case + " argmax", abuf, 8, N * Ho * Wo)
        lc.check_int_guards(case + " counters", cbuf, 8, 2 + 3 * C)
        assert not bool((am == lc.INT_SENTINEL[I32]).any()), f"{case}: arg-max map not fully written"
        runs.append((accum.clone(), loss.clone(), dlo.view.clone(), dx.view.clone(), am.clone(), cnt.clone()))
    a, b = runs
    for i, what in enumerate(("accum", "loss", "dlo", "dx", "argmax", "counters")):
        if what == "accum":
            same_bits(case, "accum[1]", a[0][1:], b[0][1:])
        elif what == "dx":
            assert torch.equal(a[3].view(torch.int16), b[3].view(torch.int16)), f"{case}: dx not bit-reproducible"
        else:
            same_bits(case, what, a[i], b[i])
    accum, loss, dlo, dx, am, cnt = a
    r = lc.UpsampleRef(lod.double(), td, ac, ignore, kind, wd, gamma, mean)
    ua = max(r.loss.check_accum(case, accum), r.loss.check_accum(case, b[0]))
    ul = r.loss.check_loss(case, loss.item())
    ug = lc.check(case, "dlo", dlo, r.dlo_bound(gscale))
    lc.check_exact(case, "dx = bf16(dlo)", dx[:, :C].float(), dlo.reshape(M, C).bfloat16().float().cpu(), ("row", "c"))
    lc.check_pad(case, dx, C)
    am = am.view(N, Ho, Wo)
    runner_up = lc.check_argmax(case, am, r.x, r.ev)
    lc.check_exact(case, "counters", cnt, lc.counters_from_map(am, td, C), ("i",))
    log(f"{case}: usage accum0={ua:.4f} loss={ul:.4f} dlo={ug:.4f} runner_up_argmax={runner_up} "
        + " ".join(f"{k}={v}" for k, v in s.items()) + f" time={time.time() - t0:.2f}s")


def lo_logits(N, Hi, Wi, C, seed, ties=True):
    """NHWC fp32 low-res logits; ties: classes 1 and C - 2 equal everywhere and the maximum in a block (first-max ties in
    the interpolated logits, the arg-max and the counters)."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(N, Hi, Wi, C, generator=g) * 2.0 ** torch.randint(-4, 3, (N, Hi, Wi, 1), generator=g).float()
    if ties and C >= 4:
        lo[..., C - 2] = lo[..., 1]
        hb, wb = max(1, Hi // 3), max(1, Wi // 3)
        lo[:, :hb, :wb, 1] = lo[:, :hb, :wb].amax(-1) + 1
        lo[:, :hb, :wb, C - 2] = lo[:, :hb, :wb, 1]
    return lo


UPSAMPLE_KINDS = [("ce", 0.0, True, False), ("wce", 0.0, False, True), ("focal", 0.5, True, True), ("focal", 2.0, True, False)]


@pytest.mark.parametrize("ac", [0, 1])
def test_upsample_small(log, ac):
    for C in (2, 19, 150, lc.FUSED_MAXC):
        for kind, gamma, mean, weighted in UPSAMPLE_KINDS:
            lo = lo_logits(2, 17, 19, C, 10 + C)
            t = lc.labels(2, 65, 73, C, 11 + C, ignore=255)
            w = lc.weights(C, 12 + C) if weighted else None
            run_upsample(log, f"upsample 17x19->65x73 ac={ac} C={C} {kind} g={gamma} mean={mean}", lo, t, ac, kind,
                         gamma, mean, w)


def test_upsample_shapes(log):
    def one_row(s):
        assert s["bwd_tile"] == 32 and s["last_tile_rows"] == 1

    run_upsample(log, "upsample 129->513 ac C=19 (C3 size)", lo_logits(4, 129, 129, 19, 20),
                 lc.labels(4, 513, 513, 19, 21), 1, regime=one_row)
    run_upsample(log, "upsample 128->512 C=150 (C5 size)", lo_logits(1, 128, 128, 150, 22),
                 lc.labels(1, 512, 512, 150, 23), 0, "focal", 2.0)
    for ac in (0, 1):
        run_upsample(log, f"upsample 1->33 ac={ac}", lo_logits(2, 1, 1, 7, 24), lc.labels(2, 33, 33, 7, 25), ac)
        run_upsample(log, f"upsample 9x9->1x17 ac={ac} (Ho = 1)", lo_logits(2, 9, 9, 7, 26), lc.labels(2, 1, 17, 7, 27), ac,
                     "wce", 0.0, True, lc.weights(7, 28))

    def tile16(s):
        assert s["bwd_tile"] == 16 and s["fwd_patch"] == 14

    run_upsample(log, "upsample 129->385 ac C=150 (tile 16)", lo_logits(1, 129, 129, 150, 29),
                 lc.labels(1, 385, 385, 150, 30), 1, regime=tile16)


def test_upsample_limits():
    """Rejected on the host, before any launch: C above MAXC, and a forward patch over 200 KB."""
    for C, Hi, Ho in ((lc.FUSED_MAXC + 1, 17, 65), (150, 33, 65)):
        assert not lc.upsample_schedule(Hi, Hi, Ho, Ho, C, 0, metrics=False)["fwd_ok"]
        lo = torch.zeros(1, Hi, Hi, C, dtype=F32, device=DEV)
        t = torch.zeros(1, Ho, Ho, dtype=I64, device=DEV)
        accum = torch.zeros(2, dtype=F64, device=DEV)
        with pytest.raises(RuntimeError, match="upsample_ce"):
            lib.call("seg_upsample_loss_fwd", ptr(lo), ptr(t), 1, Hi, Hi, Ho, Ho, C, 0, 255, None, 0, 0.0, ptr(accum),
                     None, None)


# ------------------------------------------------------------------------------------------------ fused shuffle
def run_shuffle(log, case, lo, r, C, t, kind="ce", gamma=0.0, mean=True, weight=None, gscale=0.75, ignore=255):
    """lo: bf16 [N, h, w, r^2 C] placed as a channel slice (8 sentinel lanes on each side) of a wider pitch."""
    t0 = time.time()
    N, h, w, _ = lo.shape
    rc = r * r * C
    buf = cc.sentinel_fill(torch.empty(N, h, w, 8 + rc + 8, dtype=BF16, device=DEV))
    buf[..., 8:8 + rc] = lo.to(DEV)
    lod, ldlo = buf[..., 8:], 8 + rc + 8
    td = t.to(DEV)
    wd = None if weight is None else weight.to(DEV, F32).contiguous()
    gs = torch.tensor([gscale], dtype=F32, device=DEV)
    lddx = rc + 5
    M = N * h * w
    blocks, iters, capped = lc.nchw_grid(N * h * w * r * r, sms())
    runs = []
    for _ in range(2):
        accum = torch.zeros(2, dtype=F64, device=DEV)
        cbuf, cnt = int_buf(2 + 3 * C, I64, zero=True)
        lib.call("seg_shuffle_loss_fwd", ptr(lod), ldlo, ptr(td), N, h, w, C, r, int(ignore), ptr(wd), KIND[kind],
                 float(gamma), ptr(accum), ptr(cnt))
        loss = torch.empty(1, dtype=F32, device=DEV)
        lib.call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
        dx = cc.FlatGuarded((M, lddx), BF16, device=DEV)
        lib.call("seg_shuffle_loss_bwd", ptr(lod), ldlo, ptr(td), N, h, w, C, r, int(ignore), ptr(wd), KIND[kind],
                 float(gamma), int(mean), ptr(accum), ptr(gs), ptr(dx.view), lddx)
        settle(case, dx)
        lc.check_int_guards(case + " counters", cbuf, 8, 2 + 3 * C)
        runs.append((accum.clone(), loss.clone(), dx.view.clone(), cnt.clone()))
    a, b = runs
    same_bits(case, "accum[1]", a[0][1:], b[0][1:])
    same_bits(case, "loss", a[1], b[1])
    assert torch.equal(a[2].view(torch.int16), b[2].view(torch.int16)), f"{case}: dx not bit-reproducible"
    assert torch.equal(a[3], b[3]), f"{case}: counters not bit-reproducible"
    accum, loss, dx, cnt = a
    r_ = lc.ShuffleRef(lod[..., :rc].double(), r, C, td, ignore, kind, wd, gamma, mean)
    ua = max(r_.loss.check_accum(case, accum), r_.loss.check_accum(case, b[0]))
    ul = r_.loss.check_loss(case, loss.item())
    ug = lc.check(case, "dx", dx[:, :rc].reshape(N, h, w, rc), r_.dx_bound(gscale))
    lc.check_pad(case, dx, rc)
    # the counters against eval_metrics of the materialised logits (the same bf16 values, exactly)
    logits = ops.pixel_shuffle_logits_fwd(lod[..., :rc].contiguous(), r)
    lc.check_exact(case, "counters vs eval_metrics", cnt, ops.eval_metrics_nchw(logits, td, C).cpu(), ("i",))
    lc.check_exact(case, "counters vs first max", cnt.cpu(), lc.metrics_ref(r_.loss.sm.z, td, C), ("i",))
    log(f"{case}: usage accum0={ua:.4f} loss={ul:.4f} dx={ug:.4f} blocks={blocks} iters={iters} capped={capped} "
        f"time={time.time() - t0:.2f}s")


def shuffle_lo(N, h, w, rc, seed, ties_every=0, C=None, r=None):
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(N, h, w, rc, generator=g) * 2.0 ** torch.randint(-3, 3, (N, h, w, 1), generator=g).float()
    if ties_every:  # classes 1 and C - 2 equal and maximal at every sub-pixel of every ties_every-th low-res pixel
        rr = r * r
        sel = lo.view(-1, C, rr)[::ties_every]
        sel[:, 1] = sel.amax(1) + 1
        sel[:, C - 2] = sel[:, 1]
    return lo.bfloat16()


@pytest.mark.parametrize("r", [1, 2, 4, 8])
def test_shuffle(log, r):
    C = 19
    for kind, gamma, mean, weighted in UPSAMPLE_KINDS:
        lo = shuffle_lo(2, 9, 11, r * r * C, 60 + r, ties_every=3, C=C, r=r)
        t = lc.labels(2, 9 * r, 11 * r, C, 61 + r)
        w = lc.weights(C, 62) if weighted else None
        run_shuffle(log, f"shuffle r={r} 2x9x11 C={C} {kind} g={gamma} mean={mean}", lo, r, C, t, kind, gamma, mean, w)
    if r == 4:
        N, h = 2, 129
        assert lc.nchw_grid(N * h * h * r * r, sms())[2]
        run_shuffle(log, "shuffle r=4 2x129x129 C=19 (grid-capped)", shuffle_lo(N, h, h, r * r * C, 63, 7, C, r), r, C,
                    lc.labels(N, h * r, h * r, C, 64))
        run_shuffle(log, "shuffle r=4 C=150 ignore=-1", shuffle_lo(1, 9, 7, r * r * 150, 65, 2, 150, r), r, 150,
                    lc.labels(1, 36, 28, 150, 66, ignore=-1), "focal", 2.0, True, None, 1.0, -1)
