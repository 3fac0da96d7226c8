"""PSPDenseNet on the H100: the dense-block kernels — BatchNorm apply from a block's statistics table, the BN backward that
adds into a gradient buffer (two-launch and cooperative), the floor-mode 2x2 average pool — against gathered-statistics
launches and float64 per-element bounds with guard sentinels around channel slices, and the model against the fp32 oracle
of oracle/pspdensenet.py with bounds set by an ATen bf16 run of the same model, plus FusedTrainStep and graph replay."""
import os

import pytest
import torch
import torch.nn.functional as F

import conv_check as cc
from oracle import losses as ol
from oracle import models as om
from oracle import pspdensenet as opd
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import losses, ops
    from seg_b200.train import FusedTrainStep

DEV = "cuda"
F32, F64, BF16, I16 = torch.float32, torch.float64, torch.bfloat16, torch.int16


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "pspdensenet.txt"), "a")

    def write(line):
        print(line)
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def bits(t):
    return t.view(I16) if t.dtype == BF16 else t


def guarded_slice(N, H, W, C, lead, trail, seed):
    """A bf16 buffer [N,H,W,lead+C+trail] filled with sentinels and the [lead, lead+C) channel slice of it."""
    buf = torch.empty((N, H, W, lead + C + trail), dtype=BF16, device=DEV)
    cc.sentinel_fill(buf)
    return buf, buf[..., lead:lead + C]


def check_guards(case, buf, lead, C):
    g = torch.cat([buf[..., :lead].reshape(-1), buf[..., lead + C:].reshape(-1)]).cpu()
    assert bool(cc.is_sentinel(g).all()), f"{case}: a guard channel outside the slice was overwritten"


def rand_bf16(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + offset).to(BF16).to(DEV)


# ------------------------------------------------------------------------------------------------ BN apply from a table
def make_block(N, H, W, c0, growth, layers, seed, pitch_extra=8):
    """A dense block buffer (pitch c0 + layers*growth + pitch_extra) with per-channel offsets / scales and its statistics
    table: each record the bn_stats of its slice, written into one fp64 allocation."""
    C = c0 + layers * growth
    g = torch.Generator(device="cpu").manual_seed(seed)
    off = torch.randn(C, generator=g) * 2
    sc = torch.rand(C, generator=g) * 2 + 0.25
    buf = torch.empty((N, H, W, C + pitch_extra), dtype=BF16, device=DEV)
    buf[..., :C] = (torch.randn((N, H, W, C), generator=g) * sc + off).to(BF16).to(DEV)
    table = torch.zeros(2 * C + 6, dtype=F64, device=DEV)  # + tail words the kernel must not read
    table[2 * C:] = float("nan")
    ops.bn_stats(buf[..., :c0], stats=table[:2 * c0])
    for k in range(layers):
        c = c0 + k * growth
        ops.bn_stats(buf[..., c:c + growth], stats=table[2 * c:2 * c + 2 * growth])
    return buf, table


def gather(table, c0, growth, C):
    """The contiguous [2C] (sum, sum^2) the table's records hold for channels [0, C)."""
    s = [table[:c0]]
    q = [table[c0:2 * c0]]
    for c in range(c0, C, growth):
        s.append(table[2 * c:2 * c + growth])
        q.append(table[2 * c + growth:2 * c + 2 * growth])
    return torch.cat(s + q).contiguous()


def bn_params(C, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.1).to(DEV)
    rm = (torch.randn(C, generator=g) * 0.1).to(DEV)
    rv = (torch.rand(C, generator=g) + 0.5).to(DEV)
    return gamma, beta, rm, rv


@pytest.mark.parametrize("N,H,W,c0,growth,layers,cin_layers", [
    (2, 7, 9, 64, 32, 6, 0), (2, 7, 9, 64, 32, 6, 1), (2, 7, 9, 64, 32, 6, 6), (1, 1, 1, 128, 32, 3, 2),
    (2, 29, 29, 256, 32, 12, 7), (3, 5, 3, 896, 32, 32, 32), (1, 13, 11, 8, 8, 5, 4)])
def test_bn_apply_from_table_is_bit_identical_to_gathered_stats(log, N, H, W, c0, growth, layers, cin_layers):
    buf, table = make_block(N, H, W, c0, growth, layers, seed=N * 1000 + c0 + cin_layers)
    Cin = c0 + cin_layers * growth
    x = buf[..., :Cin]
    flat = gather(table, c0, growth, Cin)
    gamma, beta, rm, rv = bn_params(Cin, 7)
    count = N * H * W
    outs = []
    for stats, kw in ((flat, {}), (table, {"table": (c0, growth)})):
        rmc, rvc = rm.clone(), rv.clone()
        mask = ops.relu_mask(x)
        ob, out = guarded_slice(N, H, W, Cin, 0, 8, 0)
        a, save = ops.bn_apply_train(x, stats, count, gamma, beta, 1e-5, 0.1, 0, rmc, rvc, out=out, relu=True, mask=mask, **kw)
        check_guards(f"bn_apply table {kw}", ob, 0, Cin)
        outs.append((a.clone(), save, rmc, rvc, mask))
    torch.cuda.synchronize()
    for name, u, v in zip(("out", "save", "running_mean", "running_var", "mask"), outs[0], outs[1]):
        assert torch.equal(bits(u), bits(v)), f"{name} differs between the table and the gathered statistics"
    assert torch.isfinite(outs[1][1]).all()
    log(f"bn_apply_train table {N}x{H}x{W} c0={c0} growth={growth} Cin={Cin}: bit-identical to gathered statistics")


def test_bn_apply_table_rejects_a_bad_tiling():
    buf, table = make_block(1, 3, 3, 64, 32, 2, seed=3)
    gamma, beta, rm, rv = bn_params(80, 1)
    with pytest.raises(AssertionError):
        ops.bn_apply_train(buf[..., :80], table, 9, gamma, beta, 1e-5, 0.1, 0, rm, rv, table=(64, 32))


# ------------------------------------------------------------------------------------------------ accumulating BN backward
def bwd_case(N, H, W, C, seed, fused, mask_kind):
    x = rand_bf16((N, H, W, C), seed, 1.5, 0.3)
    st = ops.bn_stats(x)
    gamma, beta, rm, rv = bn_params(C, seed + 1)
    mask = ops.relu_mask(x) if mask_kind == "bits" else None
    a, save = ops.bn_apply_train(x, st, N * H * W, gamma, beta, 1e-5, 0.1, 0, rm, rv, relu=True, mask=mask)
    da = rand_bf16((N, H, W, C), seed + 2)
    out = None if mask_kind == "recompute" else a
    kw = {"mask": mask} if mask is not None else {}

    def run(dx, **extra):
        if fused:
            return ops.bn_bwd_fused(da, out, x, save, gamma, N * H * W, relu=True, dx=dx, beta=beta,
                                    dgamma=torch.empty(C, device=DEV), dbeta=torch.empty(C, device=DEV), **kw, **extra)[0]
        sums = ops.bn_bwd_reduce(da, out, x, save, relu=True, gamma=gamma, beta=beta, **kw)
        return ops.bn_bwd_apply(da, out, x, save, gamma, sums, N * H * W, relu=True, dx=dx, beta=beta, **kw, **extra)
    return run


@pytest.mark.parametrize("fused", [False, True], ids=["two_launch", "cooperative"])
@pytest.mark.parametrize("mask_kind", ["act", "bits", "recompute"])
@pytest.mark.parametrize("N,H,W,C,lead,trail", [(2, 7, 9, 64, 0, 32), (2, 7, 9, 96, 64, 8), (1, 1, 1, 8, 8, 8),
                                                (2, 29, 31, 352, 128, 40), (4, 58, 58, 128, 0, 64)])
def test_bn_backward_accumulates_into_a_slice(log, fused, mask_kind, N, H, W, C, lead, trail):
    run = bwd_case(N, H, W, C, seed=C + H, fused=fused, mask_kind=mask_kind)
    # beta_dx = 0 is the launch without it, bit for bit
    ref0 = run(None).clone()
    b0, s0 = guarded_slice(N, H, W, C, lead, trail, 0)
    d0 = run(s0, beta_dx=0.0)
    check_guards("beta_dx=0", b0, lead, C)
    assert torch.equal(bits(d0), bits(ref0))
    # beta_dx = 1: old + BN backward, summed in fp32 and rounded once
    old = rand_bf16((N, H, W, C), C + 77, 0.5)
    b1, s1 = guarded_slice(N, H, W, C, lead, trail, 0)
    s1.copy_(old)
    d1 = run(s1, beta_dx=1.0)
    torch.cuda.synchronize()
    check_guards("beta_dx=1", b1, lead, C)
    want = old.double() + ref0.double()
    # |round(a + o) - (round(a) + o)| <= ulp(a + o) / 2 + ulp(a) / 2, with ulp(v) <= 2^-7 |v| for bf16 normals
    bound = (2.0 ** -8) * (want.abs() + ref0.double().abs()) * 1.0001 + 1e-30
    err = (d1.double() - want).abs()
    worst = (err / bound).max().item()
    log(f"bn backward beta_dx=1 [{'fused' if fused else 'two-launch'} {mask_kind}] {N}x{H}x{W}x{C}: worst err / bound {worst:.3f}")
    assert worst <= 1.0
    again = run(s1.copy_(old), beta_dx=1.0)
    assert torch.equal(bits(again), bits(d1)), "rerun differs"


def test_bn_backward_rejects_other_betas():
    run = bwd_case(1, 3, 3, 8, 5, fused=False, mask_kind="act")
    with pytest.raises(RuntimeError, match="beta_dx"):
        run(torch.zeros(1, 3, 3, 8, dtype=BF16, device=DEV), beta_dx=0.5)


# ------------------------------------------------------------------------------------------------ 2x2 average pool
@pytest.mark.parametrize("N,H,W,C", [(1, 2, 2, 8), (2, 15, 17, 128), (2, 16, 16, 64), (1, 3, 2, 8), (3, 117, 115, 128),
                                     (1, 2, 9, 256), (2, 232, 232, 128)])
def test_avgpool2x2_forward_and_backward(log, N, H, W, C):
    # values within 2^8 of each other in magnitude: the fp32 sum of four bf16 values is exact, so the pooled value is the
    # float64 mean rounded to bf16
    x = rand_bf16((N, H, W, C), H * W + C, 1.0, 3.0)
    P, Q = H // 2, W // 2
    lead, trail = 16, 24
    yb, y = guarded_slice(N, P, Q, C, lead, trail, 0)
    ops.avgpool2x2_fwd(x, out=y)
    ref = F.avg_pool2d(x.double().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    check_guards("avgpool2x2_fwd", yb, lead, C)
    assert torch.equal(bits(y.contiguous()), bits(ref.to(BF16)))
    # backward: beta = 0 writes every element (0 for a dropped row / column), beta = 1 adds into a slice
    dy = rand_bf16((N, P, Q, C), C + 5)
    up = torch.zeros((N, H, W, C), dtype=F64, device=DEV)
    up[:, :2 * P, :2 * Q] = dy.double().repeat_interleave(2, 1).repeat_interleave(2, 2) / 4
    xb, dx = guarded_slice(N, H, W, C, lead, trail, 0)
    ops.avgpool2x2_bwd(dy, (N, H, W, C), dx=dx, beta=0.0)
    check_guards("avgpool2x2_bwd beta=0", xb, lead, C)
    assert torch.equal(bits(dx.contiguous()), bits(up.to(BF16)))
    old = rand_bf16((N, H, W, C), C + 6, 0.7)
    dx.copy_(old)
    ops.avgpool2x2_bwd(dy, (N, H, W, C), dx=dx, beta=1.0)
    torch.cuda.synchronize()
    check_guards("avgpool2x2_bwd beta=1", xb, lead, C)
    want = old.double() + up
    assert torch.equal(bits(dx.contiguous()), bits(want.float().to(BF16))) or \
        ((dx.double() - want).abs() <= 2.0 ** -8 * want.abs() * 1.0001 + 1e-30).all()
    log(f"avgpool2x2 {N}x{H}x{W}x{C}: forward exact, backward beta 0 / 1 within bounds")


# ------------------------------------------------------------------------------------------------ model
_SD = {}


def state_dict(nc, backbone, seed):
    key = (nc, backbone, seed)
    if key not in _SD:
        _SD[key] = opd.pspdensenet_state_dict(nc, backbone, seed=seed)
    return _SD[key]


def _model(seed, backbone="densenet121", nc=7, dropout=True):
    m = seg_b200.PSPDenseNet(nc, backbone=backbone, pretrained=False)
    m.load_state_dict(state_dict(nc, backbone, seed), strict=True)
    m.engine_dropout = dropout
    return m.cuda().train()


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def cosine(a, b):
    return F.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


def _loss2(out, aux, y):
    return ol.cross_entropy2d(out, y, 255) + 0.4 * ol.cross_entropy2d(aux, y, 255)


def bf16_control(sd, x, y, backbone):
    """The oracle run by ATen on the GPU in bf16: the error a plain bf16 implementation of the same model makes."""
    moved = {}  # one device copy per tensor: block0.6 / block0.7 stay the same tensors as block0.3 / block0.4
    for v in sd.values():
        if id(v) not in moved:
            moved[id(v)] = v.to(DEV, BF16) if v.is_floating_point() else v.to(DEV)
    bsd = om.clone_sd({k: moved[id(v)] for k, v in sd.items()}, requires_grad=True)
    out, aux = opd.pspdensenet_forward(bsd, x.to(DEV, BF16), backbone)
    loss = _loss2(out.float(), aux.float(), y.to(DEV))
    loss.backward()
    return (out.detach().float().cpu(), {k: v.grad.float().cpu() for k, v in bsd.items() if v.grad is not None}, loss.item(),
            {k: v.float().cpu() for k, v in bsd.items() if k.endswith(("running_mean", "running_var"))})


BOUND_FACTOR = 4.0  # the engine may be this many times further from the fp32 oracle than the ATen bf16 run is


# At initialisation these deep batch-statistics networks amplify bf16 storage rounding (DESIGN.md §4): a plain ATen bf16
# run of the oracle lands 15-25 % from the fp32 logits here.  Every bound is therefore a multiple of that run's error.
@pytest.mark.parametrize("backbone,hw", [("densenet121", (64, 64)), ("densenet121", (70, 78)), ("densenet201", (70, 78))],
                         ids=["121-64x64", "121-70x78", "201-70x78"])
def test_train_step_parity(log, backbone, hw):
    nc = 21
    sd = state_dict(nc, backbone, 11)
    m = _model(11, backbone, nc, dropout=False)
    x, y = synth.make_batch(2, hw[0], hw[1], nc, 255, seed=9161)
    osd = om.clone_sd(sd, requires_grad=True)
    ref, ref_aux = opd.pspdensenet_forward(osd, x, backbone)
    ref_loss = _loss2(ref, ref_aux, y)
    ref_loss.backward()
    ctrl_out, ctrl_grads, ctrl_loss, ctrl_rs = bf16_control(sd, x, y, backbone)
    nbt = m.block0[4].num_batches_tracked.item()
    out, aux = m(x.cuda())
    crit = seg_b200.CrossEntropyLoss2d(ignore_index=255)
    loss = crit(out, y.cuda()) + 0.4 * crit(aux, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[pspdensenet {backbone} {hw[0]}x{hw[1]}]"
    e, ec = relerr(out, ref), relerr(ctrl_out, ref)
    log(f"{tag} logits rel_err vs fp32 oracle {e:.3e} (ATen bf16 {ec:.3e}); loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert out.shape == ref.shape == (2, nc) + hw and e <= BOUND_FACTOR * ec
    assert abs(loss.item() - ref_loss.item()) <= BOUND_FACTOR * abs(ctrl_loss - ref_loss.item()) + 1e-3 * abs(ref_loss.item())
    assert m.block0[4].num_batches_tracked.item() == nbt + 2
    cos, ccos = {}, {}
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        cos[name] = cosine(p.grad, osd[name].grad)
        ccos[name] = cosine(ctrl_grads[name], osd[name].grad)
    worst, cworst = min(cos, key=cos.get), min(ccos, key=ccos.get)
    log(f"{tag} grads vs fp32 oracle: min cosine {cos[worst]:.5f} at {worst} (ATen bf16 {ccos[cworst]:.5f} at {cworst}); "
        f"block0.3 {cos['block0.3.weight']:.5f}, block0.4 {cos['block0.4.weight']:.5f}")
    assert 1 - cos[worst] <= BOUND_FACTOR * (1 - ccos[cworst]) + 1e-4, (cos[worst], worst, ccos[cworst], cworst)
    # running statistics (the shared block0.4 updated twice, every norm1 from its block's table)
    worst_rs = max(relerr(b, osd[n]) for n, b in m.state_dict().items() if n.endswith(("running_mean", "running_var")))
    cworst_rs = max(relerr(ctrl_rs[n], osd[n]) for n in ctrl_rs)
    log(f"{tag} running statistics: worst rel_err {worst_rs:.3e} (ATen bf16 {cworst_rs:.3e})")
    assert worst_rs <= BOUND_FACTOR * cworst_rs
    m.eval()  # the eval forward, then the step on the same weights
    with torch.no_grad():
        ev = m(x.cuda())
    assert relerr(ev, opd.pspdensenet_forward(osd, x, backbone, train=False)) <= BOUND_FACTOR * max(ec, 1e-3)
    # one SGD step (lr 0.01): the post-step weights, each tensor's distance from the oracle's against the ATen bf16 run's
    # gradients applied the same way
    lr = 0.01
    torch.optim.SGD(m.parameters(), lr=lr).step()
    worst_w, cworst_w = 0.0, 0.0
    with torch.no_grad():
        for n, p in m.named_parameters():
            want = osd[n] - lr * osd[n].grad
            wn = want.double().norm().item() + 1e-30
            worst_w = max(worst_w, (p.detach().double().cpu() - want.double()).norm().item() / wn)
            cworst_w = max(cworst_w, (lr * (ctrl_grads[n].double() - osd[n].grad.double())).norm().item() / wn)
    log(f"{tag} post-step weights: worst per-tensor rel distance {worst_w:.3e} (ATen bf16 gradients {cworst_w:.3e})")
    assert worst_w <= BOUND_FACTOR * cworst_w + 1e-6


def test_fused_step_first_loss_and_counters_equal_plugin(log):
    x, y = synth.make_batch(2, 70, 78, 7, 255, seed=9163)
    xd, yd = x.cuda(), y.cuda()
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    m = _model(41, dropout=False)
    with torch.no_grad():
        o, a = m(xd)
        ref = float(crit(o, yd) + 0.4 * crit(a, yd))
        want = ops.eval_metrics_nchw(o, yd, 7)
    s = FusedTrainStep(_model(41, dropout=False), lr=0.005, loss=crit, metrics=True)
    got = float(s.step(xd, yd))
    log(f"fused step [pspdensenet121 70x78] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-5 * abs(ref)
    assert torch.equal(s.seg_counters, want)
    assert s.model.block0[4].num_batches_tracked.item() == 2


def test_fused_step_graph_replay_is_bit_identical():
    x, y = synth.make_batch(2, 70, 78, 7, 255, seed=9164)
    xd, yd = x.cuda(), y.cuda()
    se = FusedTrainStep(_model(42, dropout=False), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model(42, dropout=False), lr=0.005, metrics=True, cuda_graph=True)
    for i in range(4):
        le, lg = float(se.step(xd, yd)), float(sg.step(xd, yd))
        assert le == le and le == lg, (i, le, lg)
        assert torch.equal(se.seg_counters, sg.seg_counters)
    assert torch.equal(se.flat_grad, sg.flat_grad)
    for (n, a), (_, b) in zip(se.model.state_dict().items(), sg.model.state_dict().items()):
        assert torch.equal(a, b), n
    assert sg.model.block0[4].num_batches_tracked.item() == 8
    sg.release_graph()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_evaluate_changes_no_training_state(graph):
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9165)
    xd, yd = x.cuda(), y.cuda()
    s = FusedTrainStep(_model(43), lr=0.005, metrics=True, cuda_graph=graph)
    s.step(xd, yd)
    m = s.model
    before = ([t.clone() for t in m.state_dict().values()], s.flat_mom.clone(), m._step_ctr.clone(), s.steps, m.training)
    s.reset_metrics()
    loss = float(s.evaluate(xd, yd))
    after = ([t.clone() for t in m.state_dict().values()], s.flat_mom.clone(), m._step_ctr.clone(), s.steps, m.training)
    assert all(torch.equal(a, b) for a, b in zip(before[0], after[0]))
    assert torch.equal(before[1], after[1]) and torch.equal(before[2], after[2]) and before[3:] == after[3:]
    m.eval()
    with torch.no_grad():
        out = m(xd)
    m.train()
    assert torch.equal(s.seg_counters, ops.eval_metrics_nchw(out, yd, 7))
    ref = float(losses.CrossEntropyLoss2d(ignore_index=255)(out, yd))
    assert abs(loss - ref) <= 1e-5 * abs(ref)
    if graph:
        s.release_graph()


def test_full_size_densenet201_graph_step(log):
    """Graph-replayed 8 x 3 x 473^2 fused steps of densenet201 at 21 classes have finite losses."""
    x, y = synth.make_batch(8, 473, 473, 21, 255, seed=9168)
    s = FusedTrainStep(_model(48, "densenet201", nc=21), lr=0.01, cuda_graph=True)
    losses_ = [float(s.step(x.cuda(), y.cuda())) for _ in range(3)]
    torch.cuda.synchronize()
    log(f"[pspdensenet201 21 classes 8x3x473x473 graph step] losses " + " ".join(f"{v:.6f}" for v in losses_)
        + f"; peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert all(v == v and abs(v) < 1e3 for v in losses_)
    s.release_graph()
