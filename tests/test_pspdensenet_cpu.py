"""PSPDenseNet (models/pspnet.py:117-205) on the CPU box: the engine model's constructor (names, order, counts, the shared
block0 conv / BN, parameter groups, options) against the reference's, the oracle against the unmodified reference, and the
engine's host logic (dense-block buffers written in place, the statistics table, norm1 backwards adding into the block's
gradient, the shared block0 modules, the PSP concat as block4's buffer) under the ATen emulation of tests/cpu_emulation.py
with fp32 storage against the oracle's train step, at world 1 and over a two-rank gloo group.  The kernels are checked on
the GPU by tests/test_pspdensenet_gpu.py."""
import logging
import os
import socket
import subprocess
import sys
import zipfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import cpu_emulation as emu
from oracle import losses as ol
from oracle import models as om
from oracle import pspdensenet as opd
from oracle import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
COUNTS = {"densenet121": 13941802, "densenet169": 30158058, "densenet201": 42290282}


GOLD = os.path.join(ROOT, "tests", "golden", "pspdensenet.npz")
# (prefix, H, W, weight seed, batch seed) of oracle/make_golden_pspdensenet.py
GOLDEN_STEPS = [("s64/", 64, 64, 41, 9041), ("s70x78/", 70, 78, 42, 9042)]


def close(a, b, rtol):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    err = np.abs(a - b).max() / (np.abs(b).max() + 1e-12)
    assert err <= rtol, f"rel err {err:.3e} > {rtol:.1e}"


@pytest.mark.parametrize("prefix,h,w,seed,xseed", GOLDEN_STEPS, ids=[c[0] for c in GOLDEN_STEPS])
def test_oracle_train_step_matches_reference_golden(prefix, h, w, seed, xseed):
    """The fp32 oracle against the unmodified reference's recorded train step and eval forward (densenet121, 21 classes).
    Gradient tolerances: batch statistics over block4's small maps make some norm1 gradients ill-conditioned (fp32 summation
    order alone moves them by several per cent), so per-parameter norms get 5e-2 and the recorded gradients, which are
    well-conditioned, 2e-3."""
    g = np.load(GOLD)
    sd = om.clone_sd(opd.pspdensenet_state_dict(21, "densenet121", seed=seed), requires_grad=True)
    x, y = synth.make_batch(2, h, w, 21, 255, seed=xseed)
    out, aux = opd.pspdensenet_forward(sd, x, "densenet121")
    loss = ol.cross_entropy2d(out, y, 255) + 0.4 * ol.cross_entropy2d(aux, y, 255)
    loss.backward()
    assert tuple(out.shape) == tuple(g[prefix + "out_shape"]) == (2, 21, h, w)
    close(out.detach()[:, :, ::4, ::4].numpy(), g[prefix + "logits_sub"], 2e-4)
    close(out.detach().double().sum((2, 3)).numpy(), g[prefix + "logits_sum"], 2e-4)
    close(aux.detach().double().sum((2, 3)).numpy(), g[prefix + "aux_sum"], 2e-4)
    assert (out.detach().argmax(1).numpy() == g[prefix + "argmax"]).mean() > 0.9995
    close(loss.item(), g[prefix + "loss"], 1e-5)
    names = [str(n) for n in g[prefix + "param_names"]]
    assert names == om.param_names({k: v for k, v in sd.items() if not k.startswith(("block0.6.", "block0.7."))})
    norms = np.array([sd[n].grad.double().norm().item() for n in names])
    np.testing.assert_allclose(norms, g[prefix + "grad_norms"], rtol=5e-2)
    for k in g.files:
        if k.startswith(prefix + "grad/"):
            close(sd[k[len(prefix) + 5:]].grad.numpy(), g[k], 2e-3)
        elif k.startswith(prefix + "grad_head/"):
            v = g[k]
            close(sd[k[len(prefix) + 10:]].grad[:v.shape[0]].numpy(), v, 2e-3)
        elif k.startswith(prefix + "buf/"):
            t = sd[k[len(prefix) + 4:]]
            if t.is_floating_point():
                close(t.numpy(), g[k], 1e-5)
            else:
                assert g[k] == 2  # the reference's block0.4 counts both of its applications (F.batch_norm counts nothing)
    with torch.no_grad():
        ev = opd.pspdensenet_forward(sd, x, "densenet121", train=False)
    close(ev.double().sum((2, 3)).numpy(), g[prefix + "eval_logits_sum"], 2e-4)


def _nets():
    from seg_b200 import nets
    return nets


@pytest.mark.parametrize("backbone", list(COUNTS))
def test_state_dict_counts_and_shared_block0(backbone):
    nets = _nets()
    m = nets.PSPDenseNet(21, backbone=backbone, pretrained=False)
    assert list(m.state_dict()) == list(opd.pspdensenet_state_dict(21, backbone))
    assert m._n_trainable() == COUNTS[backbone]
    assert m.block0[3] is m.block0[6] and m.block0[4] is m.block0[7]
    sd = m.state_dict()
    for k in ("weight",):
        assert sd["block0.3." + k].data_ptr() == sd["block0.6." + k].data_ptr()
    assert sd["block0.4.running_mean"].data_ptr() == sd["block0.7.running_mean"].data_ptr()
    names = [s.name for s in m.all_conv_specs()]
    assert "block0.3" in names and "block0.6" not in names and len(names) == len(set(names))


def test_options():
    nets = _nets()
    with pytest.raises(NotImplementedError, match="96"):
        nets.PSPDenseNet(21, backbone="densenet161", pretrained=False)
    with pytest.raises(RuntimeError, match="network"):
        nets.PSPDenseNet(21, backbone="densenet121", pretrained=True)
    log = logging.getLogger("PSPDenseNet")
    records = []
    h = logging.Handler()
    h.emit = records.append
    log.addHandler(h)
    try:
        nets.PSPDenseNet(21, backbone="densenet121")
    finally:
        log.removeHandler(h)
    assert any("pretrained" in r.getMessage() for r in records)
    m = nets.PSPDenseNet(21, backbone="densenet121", pretrained=False, freeze_backbone=True)
    assert all(p.requires_grad for p in m.parameters())
    m = nets.PSPDenseNet(21, backbone="densenet121", pretrained=False, in_channels=4)
    assert m.block0[0].weight.shape == (64, 4, 3, 3) and m._spec("block0.0", m.block0[0]).explicit
    m = nets.PSPDenseNet(21, backbone="densenet121", pretrained=False, freeze_bn=True)
    assert not any(b.training for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))


def test_parameter_groups():
    """As the reference's: block0-3 and the transitions in the backbone group, the heads in the decoder group; block4 in
    neither."""
    nets = _nets()
    m = nets.PSPDenseNet(21, backbone="densenet121", pretrained=False)
    names = {id(p): n for n, p in m.named_parameters()}
    bb = [names[id(p)] for p in m.get_backbone_params()]
    dec = [names[id(p)] for p in m.get_decoder_params()]
    assert not set(bb) & set(dec)
    rest = set(names.values()) - set(bb) - set(dec)
    assert rest and all(n.startswith("block4.") for n in rest)
    assert all(n.startswith(("block0.", "block1.", "block2.", "block3.", "transition")) for n in bb)
    assert all(n.startswith(("master_branch.", "auxiliary_branch.")) for n in dec)


# ------------------------------------------------------------------------------------------------ emulated host logic
_ORIG = {}


def _gather(table, c0, growth, C):
    s, q = [table[:c0]], [table[c0:2 * c0]]
    for c in range(c0, C, growth):
        s.append(table[2 * c:2 * c + growth])
        q.append(table[2 * c + growth:2 * c + 2 * growth])
    return torch.cat(s + q)


def _bn_apply_train(x, stats, *a, table=None, **k):
    if table is not None:
        stats = _gather(stats, table[0], table[1], x.shape[-1])
    return _ORIG["bn_apply_train"](x, stats, *a, **k)


def _acc(dx, g, beta_dx):
    if dx is None:
        return g
    dx.copy_((dx.float() + g.float()).to(dx.dtype) if beta_dx else g)
    return dx


def _bn_bwd_apply(*a, dx=None, beta_dx=0.0, **k):
    return _acc(dx, _ORIG["bn_bwd_apply"](*a, dx=None, **k), beta_dx)


def _bn_bwd_fused(*a, dx=None, beta_dx=0.0, **k):
    g, sums = _ORIG["bn_bwd_fused"](*a, dx=None, **k)
    return _acc(dx, g, beta_dx), sums


def _avgpool2x2_fwd(x, out=None):
    y = F.avg_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    if out is None:
        return y.to(emu.ACT_DTYPE).contiguous()
    out.copy_(y)
    return out


def _avgpool2x2_bwd(dy, x_shape, dx=None, beta=0.0):
    N, H, W, C = x_shape
    g = torch.zeros(x_shape)
    g[:, :H // 2 * 2, :W // 2 * 2] = dy.float().repeat_interleave(2, 1).repeat_interleave(2, 2) / 4
    if dx is None:
        return g.to(emu.ACT_DTYPE)
    dx.copy_(dx.float() * beta + g if beta else g)
    return dx


def _nhwc_to_nchw(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


EMU_EXTRA = (("bn_apply_train", _bn_apply_train), ("bn_bwd_apply", _bn_bwd_apply), ("bn_bwd_fused", _bn_bwd_fused),
             ("avgpool2x2_fwd", _avgpool2x2_fwd), ("avgpool2x2_bwd", _avgpool2x2_bwd), ("nhwc_to_nchw_f32", _nhwc_to_nchw))


def _install(setattr_):
    for name in ("bn_apply_train", "bn_bwd_apply", "bn_bwd_fused"):
        _ORIG.setdefault(name, getattr(emu, name))
    from seg_b200 import engine, nets
    from seg_b200 import losses as plosses
    for name, fn in EMU_EXTRA:
        setattr_(emu, name, fn)
    for mod in (engine, nets, plosses):
        setattr_(mod, "ops", emu)
    setattr_(engine, "ACT_DTYPE", torch.float32)
    setattr_(emu, "ACT_DTYPE", torch.float32)
    setattr_(nets._EngineModel, "_check_input", lambda self, x: None)
    return nets


@pytest.fixture()
def emulated(monkeypatch):
    return _install(lambda o, n, v: monkeypatch.setattr(o, n, v, raising=False))


def relerr(a, b):
    return ((a.detach().double() - b.detach().double()).abs().max() / (b.detach().double().abs().max() + 1e-12)).item()


def _step(nets, plosses, sd, x, y, dp_reduce=True, nc=5):
    m = nets.PSPDenseNet(nc, backbone="densenet121", pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m.dp_reduce = dp_reduce
    m.train()
    out, aux = m(x)
    # per-rank mean losses (no cross-rank loss reduction inside the loss)
    loss = plosses._CEFn.apply(out, y, 255, False) + 0.4 * plosses._CEFn.apply(aux, y, 255, False)
    loss.backward()
    return m, out, loss


@pytest.mark.parametrize("hw", [(64, 64), (70, 78)], ids=["64x64", "70x78"])
def test_train_step_host_logic(emulated, hw):
    """Logits, loss, every parameter gradient (the shared block0 conv's summed over its two uses) and the running
    statistics (block0.4 updated twice, num_batches_tracked + 2) of one emulated train step against the oracle's.  At 70x78
    the unpadded stride-2 stem and the floor-mode average pool both drop a trailing row and column."""
    from seg_b200 import losses as plosses
    nc = 5
    sd = opd.pspdensenet_state_dict(nc, "densenet121", seed=5)
    x, y = synth.make_batch(2, hw[0], hw[1], nc, 255, seed=78)
    osd = om.clone_sd(sd, requires_grad=True)
    ref, ref_aux = opd.pspdensenet_forward(osd, x, "densenet121")
    ref_loss = ol.cross_entropy2d(ref, y, 255) + 0.4 * ol.cross_entropy2d(ref_aux, y, 255)
    ref_loss.backward()
    m, out, loss = _step(emulated, plosses, sd, x, y, nc=nc)
    assert out.shape == ref.shape == (2, nc) + hw
    assert relerr(out, ref) < 2e-3
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item())
    # per-parameter max-norm errors are not a fair bound here: small-count batch statistics in block4 make some norm1 bias
    # gradients ill-conditioned (the fp32 oracle itself is ~0.1 from a float64 run there); the whole gradient is not
    g = torch.cat([p.grad.reshape(-1).double() for p in m.parameters()])
    go = torch.cat([osd[n].grad.reshape(-1).double() for n, _ in m.named_parameters()])
    assert ((g - go).norm() / go.norm()).item() < 2e-2
    msd = m.state_dict()
    for n, v in msd.items():
        if n.endswith("running_mean") or n.endswith("running_var"):
            assert relerr(v, osd[n]) < 1e-3, n
    assert msd["block0.4.num_batches_tracked"].item() == 2 and msd["block0.1.num_batches_tracked"].item() == 1


def test_eval_forward_host_logic(emulated):
    nc = 5
    sd = opd.pspdensenet_state_dict(nc, "densenet121", seed=6)
    x, _ = synth.make_batch(2, 70, 78, nc, 255, seed=79)
    m = emulated.PSPDenseNet(nc, backbone="densenet121", pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.eval()
    with torch.no_grad():
        out = m(x)
    assert relerr(out, opd.pspdensenet_forward(sd, x, "densenet121", train=False)) < 2e-3


# ------------------------------------------------------------------------------------------------ data parallel, gloo world 2
class _GlooSync:
    """The exchange object without the in-kernel protocol: sums a statistics vector over the ranks."""
    fused = False

    def __init__(self, world):
        self.world = world

    def allreduce_(self, v):
        w = v.double()
        dist.all_reduce(w)
        v.copy_(w)


def _dp_worker(rank, world, port, result_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import test_pspdensenet_cpu as t
    from seg_b200 import losses as plosses
    nets = t._install(setattr)
    sd = opd.pspdensenet_state_dict(5, "densenet121", seed=11)
    x, y = synth.make_batch(4, 64, 64, 5, 255, seed=31)
    y[:, :2] = 255  # the same count of ignored pixels in every image: per-rank means average to the global mean
    half = slice(rank * 2, rank * 2 + 2)
    m = nets.PSPDenseNet(5, backbone="densenet121", pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m.bn_sync = _GlooSync(world)
    m.dp_reduce = False  # gradients averaged by hand below, as tests/test_distributed_cpu.py does
    m.train()
    xh, yh = x[half].contiguous(), y[half].contiguous()
    out, aux = m(xh)
    loss = plosses._CEFn.apply(out, yh, 255, False) + 0.4 * plosses._CEFn.apply(aux, yh, 255, False)
    loss.backward()
    grads = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    dist.all_reduce(grads)
    grads /= world
    rs = torch.cat([v.reshape(-1).double() for n, v in m.state_dict().items() if n.endswith(("running_mean", "running_var"))])
    dist.all_reduce(loss)
    loss /= world
    if rank == 0:
        m1, _, loss1 = t._step(nets, plosses, sd, x, y, dp_reduce=False)
        g1 = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
        rs1 = torch.cat([v.reshape(-1).double() for n, v in m1.state_dict().items() if n.endswith(("running_mean", "running_var"))])
        torch.save({"loss2": loss, "loss1": loss1.detach(), "grad_rel": (grads.double() - g1.double()).norm() / g1.double().norm(),
                    "rs_rel": (rs - rs1).abs().max() / rs1.abs().max()}, result_path)
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_rank_step_equals_single_rank_on_concatenated_batch(tmp_path):
    """Two ranks on half batches, with the statistics exchanged over gloo and the gradients averaged, give the
    loss, gradients and running statistics of one rank on the concatenated batch.  A table record exchanged more than once
    (a consumer all-reducing its prefix) would double those channels' statistics."""
    result = str(tmp_path / "r.pt")
    mp.spawn(_dp_worker, args=(2, _free_port(), result), nprocs=2, join=True)
    r = torch.load(result)
    assert abs(r["loss2"].item() - r["loss1"].item()) < 1e-4 * abs(r["loss1"].item()), r
    # the whole gradient, loosely: at this initialisation it is ill-conditioned (test_train_step_host_logic); a record
    # exchanged twice shows in the loss and the running statistics, which are tight
    assert r["grad_rel"].item() < 5e-2, r
    assert r["rs_rel"].item() < 1e-4, r


# ------------------------------------------------------------------------------------------------ against the reference
CODE = r"""
import sys
import torch
import torch.nn.functional as F
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
sys.path.insert(0, sys.argv[2])
import models, seg_b200
assert models.PSPDenseNet is seg_b200.PSPDenseNet, models.PSPDenseNet
assert 'PSPDenseNet' in (models.__doc__ or '')
import importlib
from oracle import pspdensenet as opd, models as om, losses as ol, synth
Pm = importlib.import_module('models.pspnet')
counts = []
for bb in ('densenet121', 'densenet169', 'densenet201'):
    ref = Pm.PSPDenseNet(21, backbone=bb, pretrained=False)
    eng = seg_b200.PSPDenseNet(21, backbone=bb, pretrained=False)
    rs, es = ref.state_dict(), eng.state_dict()
    assert [(k, tuple(v.shape)) for k, v in rs.items()] == [(k, tuple(v.shape)) for k, v in es.items()], bb
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in eng.named_parameters()], bb
    rn = {id(p): n for n, p in ref.named_parameters()}
    en = {id(p): n for n, p in eng.named_parameters()}
    assert [rn[id(p)] for p in ref.get_backbone_params()] == [en[id(p)] for p in eng.get_backbone_params()], bb
    assert [rn[id(p)] for p in ref.get_decoder_params()] == [en[id(p)] for p in eng.get_decoder_params()], bb
    counts.append(sum(p.numel() for p in ref.parameters() if p.requires_grad))
    assert counts[-1] == eng._n_trainable()
    assert ref.block0[3] is ref.block0[6]
try:
    Pm.PSPDenseNet(21, backbone='densenet161', pretrained=False).train()(torch.zeros(2, 3, 64, 64))
    raise SystemExit('densenet161 trained')
except RuntimeError as e:
    assert '96' in str(e), e
# the oracle against the unmodified reference: one train step (loss, gradients, running statistics) and an eval forward
for h, w in ((64, 64), (70, 78)):
    sd = opd.pspdensenet_state_dict(21, 'densenet121', seed=21)
    ref = Pm.PSPDenseNet(21, backbone='densenet121', pretrained=False)
    ref.load_state_dict(sd)
    for m in ref.modules():
        if isinstance(m, torch.nn.Dropout2d):
            m.p = 0.0
    ref.train()
    x, y = synth.make_batch(2, h, w, 21, 255, seed=5)
    out, aux = ref(x)
    loss = ol.cross_entropy2d(out, y, 255) + 0.4 * ol.cross_entropy2d(aux, y, 255)
    loss.backward()
    osd = om.clone_sd(sd, requires_grad=True)
    o2, a2 = opd.pspdensenet_forward(osd, x, 'densenet121')
    l2 = ol.cross_entropy2d(o2, y, 255) + 0.4 * ol.cross_entropy2d(a2, y, 255)
    l2.backward()
    assert abs(loss.item() - l2.item()) <= 1e-5 * abs(loss.item()), (loss.item(), l2.item())
    assert (out - o2).abs().max() <= 1e-4 * out.abs().max()
    for n, p in ref.named_parameters():
        g = osd[n].grad
        assert (p.grad - g).abs().max() <= 2e-4 * g.abs().max() + 1e-12, n
    for n, v in ref.state_dict().items():
        if n.endswith(('running_mean', 'running_var')):
            assert (v - osd[n]).abs().max() <= 1e-5 * (osd[n].abs().max() + 1), n
    assert ref.state_dict()['block0.4.num_batches_tracked'].item() == 2
    ref.eval()
    with torch.no_grad():
        e1 = ref(x)
    e2 = opd.pspdensenet_forward(osd, x, 'densenet121', train=False)
    assert (e1 - e2).abs().max() <= 1e-4 * e1.abs().max()
print('PSPDENSENET_OK', *counts)
"""


@pytest.mark.skipif(not os.path.isfile(REF_ZIP), reason="oracle/_ref/reference.zip not built (build() found no reference checkout)")
def test_overlay_reference_constructor_and_oracle(tmp_path):
    ref = tmp_path / "reference"
    with zipfile.ZipFile(REF_ZIP) as z:
        z.extractall(ref)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "pytorch-segmentation_b200")
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", CODE, str(ref), ROOT], env=env, cwd=str(ref), capture_output=True,
                       text=True, timeout=900)
    assert "PSPDENSENET_OK 13941802 30158058 42290282" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
