"""SegNet (models/segnet.py:13-132) on the CPU box: the oracle against the reference's golden outputs, the engine model's
constructor (names, shapes, parameter order, parameter groups, init quirks) against the reference's, and the engine's host
logic (2x2 max-pool codes, unpooling to the encoder maps' sizes with odd rows / columns dropped, the full-resolution head)
under the ATen emulation of tests/cpu_emulation.py with fp32 storage against the oracle's train step.  The kernels are
checked on the GPU by tests/test_segnet_gpu.py."""
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
import torch.nn as nn
import torch.nn.functional as F

import cpu_emulation as emu
from oracle import losses as ol
from oracle import models as om
from oracle import segnet as osn
from oracle import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden", "segnet.npz")
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
RTOL = 2e-4  # as tests/test_oracle_golden.py


def close(a, b, rtol=RTOL):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    err = np.abs(a - b).max() / (np.abs(b).max() + 1e-12)
    assert err <= rtol, f"rel err {err:.3e} > {rtol:.1e}"


# (prefix, H, W, weight seed, batch seed) of oracle/make_golden_segnet.py
GOLDEN_STEPS = [("s64/", 64, 64, 21, 9021), ("s50x75/", 50, 75, 22, 9022)]


@pytest.mark.parametrize("prefix,h,w,seed,xseed", GOLDEN_STEPS, ids=[c[0] for c in GOLDEN_STEPS])
def test_oracle_train_step_matches_reference_golden(prefix, h, w, seed, xseed):
    g = np.load(GOLD)
    sd = om.clone_sd(osn.segnet_state_dict(19, seed=seed, randomize_bn=True), requires_grad=True)
    x, y = synth.make_batch(2, h, w, 19, 255, seed=xseed)
    out = osn.segnet_forward(sd, x, train=True)
    loss = ol.cross_entropy2d(out, y, 255)
    loss.backward()
    assert tuple(out.shape) == tuple(g[prefix + "out_shape"]) == (2, 19, h, w)
    close(out.detach()[:, :, ::4, ::4].numpy(), g[prefix + "logits_sub"])
    close(out.detach().double().sum((2, 3)).numpy(), g[prefix + "logits_sum"])
    assert (out.detach().argmax(1).numpy() == g[prefix + "argmax"]).mean() > 0.9995
    close(loss.item(), g[prefix + "loss"], 1e-5)
    names = [str(n) for n in g[prefix + "param_names"]]
    assert names == om.param_names(sd), "oracle parameter order/names differ from the reference's named_parameters()"
    close(np.array([sd[n].grad.double().norm().item() for n in names]), g[prefix + "grad_norms"], 2e-3)
    for k in g.files:
        if not k.startswith(prefix):
            continue
        k2 = k[len(prefix):]
        if k2.startswith("grad/"):
            close(sd[k2[5:]].grad.numpy(), g[k], 2e-3)
        elif k2.startswith("rm/"):
            close(sd[k2[3:] + ".running_mean"].numpy(), g[k])
        elif k2.startswith("rv/"):
            close(sd[k2[3:] + ".running_var"].numpy(), g[k])
    with torch.no_grad():
        ev = osn.segnet_forward(sd, x, train=False)
    close(ev.double().sum((2, 3)).numpy(), g[prefix + "eval_logits_sum"])


# ------------------------------------------------------------------------------------------------ constructor
def test_state_dict_and_parameter_order():
    import seg_b200
    m = seg_b200.SegNet(19, pretrained=False)
    sd = osn.segnet_state_dict(19)
    esd = m.state_dict()
    assert len(esd) == len(sd) == 184
    assert [(k, tuple(v.shape)) for k, v in esd.items()] == [(k, tuple(v.shape)) for k, v in sd.items()]
    assert [n for n, _ in m.named_parameters()] == om.param_names(sd) and len(om.param_names(sd)) == 106
    assert sum(p.numel() for p in m.parameters()) == 29491027
    m.load_state_dict(sd, strict=True)
    assert [str(n) for n in np.load(GOLD)["s64/param_names"]] == [n for n, _ in m.named_parameters()]
    assert tuple(m.stage5_decoder[6].weight.shape) == (19, 64, 3, 3) and len(m.stage4_decoder) == 6


def test_init_quirks():
    """Encoder: torchvision's VGG init (kaiming-normal fan_out, bias 0, BN 1 / 0).  Decoder: kaiming-normal fan_in, bias 0,
    BN 1 / 0.  in_channels != 3: stage1_encoder.0 is a default-initialised Conv2d."""
    import seg_b200
    torch.manual_seed(0)
    m = seg_b200.SegNet(19, pretrained=False)
    bns = [b for b in m.modules() if isinstance(b, nn.BatchNorm2d)]
    assert len(bns) == 26 and all((b.weight == 1).all() and (b.bias == 0).all() for b in bns)
    convs = [(n, c) for n, c in m.named_modules() if isinstance(c, nn.Conv2d)]
    assert len(convs) == 27 and all((c.bias == 0).all() for _, c in convs)
    for n, c in convs:
        fan = c.out_channels * 9 if "encoder" in n else c.in_channels * 9
        sd = (2.0 / fan) ** 0.5
        tol = 0.1 if c.weight.numel() < 5000 else 0.05
        assert abs(c.weight.std().item() - sd) < tol * sd, (n, c.weight.std().item(), sd)
    m4 = seg_b200.SegNet(7, in_channels=4, pretrained=False)
    c0 = m4.stage1_encoder[0]
    bound = (4 * 9) ** -0.5
    assert tuple(c0.weight.shape) == (64, 4, 3, 3) and c0.bias.abs().max() <= bound and c0.bias.std() > 0.3 * bound
    assert c0.weight.abs().max() <= bound
    assert tuple(m4.stage5_decoder[6].weight.shape) == (7, 64, 3, 3)


def test_parameter_groups_and_options():
    import seg_b200
    m = seg_b200.SegNet(19, pretrained=False)
    assert list(m.get_backbone_params()) == []
    assert [id(p) for p in m.get_decoder_params()] == [id(p) for p in m.parameters()]
    m = seg_b200.SegNet(19, pretrained=False, freeze_bn=True, freeze_backbone=True)
    assert all(not b.training for b in m.modules() if isinstance(b, nn.BatchNorm2d))
    for n, p in m.named_parameters():
        assert p.requires_grad == ("decoder" in n), n
    with pytest.raises(RuntimeError, match="network"):
        seg_b200.SegNet(7, pretrained=True)
    specs = {s.name: s for s in m.all_conv_specs()}
    assert len(specs) == 27 and specs["stage1_encoder.0"].explicit
    assert not any(s.explicit for n, s in specs.items() if n != "stage1_encoder.0")
    assert seg_b200.SegNet(7, in_channels=8, pretrained=False).all_conv_specs()[0].explicit


@pytest.mark.parametrize("hw", [(31, 64), (64, 31), (16, 16)])
def test_small_inputs_raise(hw):
    import seg_b200
    m = seg_b200.SegNet(7, pretrained=False)
    with pytest.raises(ValueError, match=f"{hw[0]}x{hw[1]}"):
        m(torch.zeros(1, 3, *hw))


# ------------------------------------------------------------------------------------------------ host logic, emulated
def _nhwc_to_nchw(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


def _logits_bwd(dy, r, ldx):
    assert r == 1
    out = torch.zeros(dy.shape[0], dy.shape[2], dy.shape[3], ldx, dtype=emu.ACT_DTYPE)
    out[..., : dy.shape[1]] = dy.permute(0, 2, 3, 1).to(emu.ACT_DTYPE)
    return out


def _code_to_index(code, W):
    """NHWC uint8 codes 2r + s of a [N,P,Q,C] pool -> ATen's NCHW flat indices h * W + w."""
    c = code.permute(0, 3, 1, 2).long()
    P, Q = c.shape[2:]
    p = torch.arange(P).view(1, 1, P, 1)
    q = torch.arange(Q).view(1, 1, 1, Q)
    return (2 * p + c // 2) * W + 2 * q + c % 2


def _maxpool2x2_fwd(x):
    N, H, W, C = x.shape
    y, idx = F.max_pool2d(_nhwc_to_nchw(x), 2, 2, return_indices=True)
    P, Q = y.shape[2:]
    h, w = idx // W, idx % W
    code = 2 * (h - 2 * torch.arange(P).view(1, 1, P, 1)) + (w - 2 * torch.arange(Q).view(1, 1, 1, Q))
    assert code.min() >= 0 and code.max() <= 3
    return y.permute(0, 2, 3, 1).to(emu.ACT_DTYPE).contiguous(), code.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _maxunpool2x2_fwd(x, code, out_hw):
    H, W = out_hw
    y = F.max_unpool2d(_nhwc_to_nchw(x), _code_to_index(code, W), 2, 2, output_size=(H, W))
    return y.permute(0, 2, 3, 1).to(emu.ACT_DTYPE).contiguous()


def _maxpool2x2_bwd(dy, code, x_shape):
    return _maxunpool2x2_fwd(dy, code, x_shape[1:3])


def _maxunpool2x2_bwd(dy, code):
    N, H, W, C = dy.shape
    idx = _code_to_index(code, W)
    g = _nhwc_to_nchw(dy).flatten(2).gather(2, idx.flatten(2)).view(idx.shape)
    return g.permute(0, 2, 3, 1).to(emu.ACT_DTYPE).contiguous()


EMU_EXTRA = (("nhwc_to_nchw_f32", _nhwc_to_nchw), ("pixel_shuffle_logits_bwd", _logits_bwd), ("maxpool2x2_fwd", _maxpool2x2_fwd),
             ("maxpool2x2_bwd", _maxpool2x2_bwd), ("maxunpool2x2_fwd", _maxunpool2x2_fwd), ("maxunpool2x2_bwd", _maxunpool2x2_bwd))


@pytest.fixture()
def emulated(monkeypatch):
    from seg_b200 import engine, nets
    from seg_b200 import losses as plosses
    for name, fn in EMU_EXTRA:
        monkeypatch.setattr(emu, name, fn, raising=False)
    for mod in (engine, nets, plosses):
        monkeypatch.setattr(mod, "ops", emu)
    monkeypatch.setattr(engine, "ACT_DTYPE", torch.float32)
    monkeypatch.setattr(emu, "ACT_DTYPE", torch.float32)
    monkeypatch.setattr(nets._EngineModel, "_check_input", lambda self, x: None)
    return nets


def relerr(a, b):
    return ((a.detach().double() - b.detach().double()).abs().max() / (b.detach().double().abs().max() + 1e-12)).item()


def _emulated_step(nets, hw, frozen_bn, nc=7):
    """(engine model, oracle state_dict with gradients, input, engine logits, oracle logits, engine loss, oracle loss)."""
    from seg_b200.losses import _CEFn
    sd = osn.segnet_state_dict(nc, seed=5, randomize_bn=True)
    m = nets.SegNet(nc, pretrained=False, freeze_bn=frozen_bn)
    m.load_state_dict(sd, strict=True)
    m.train()
    if frozen_bn:
        m.freeze_bn()
    x, y = synth.make_batch(2, hw[0], hw[1], nc, 255, seed=78)
    osd = om.clone_sd(sd, requires_grad=True)
    ref = osn.segnet_forward(osd, x, train=not frozen_bn)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    out = m(x)
    loss = _CEFn.apply(out, y, 255)
    loss.backward()
    return m, osd, x, out, ref, loss, ref_loss


def _grad_errors(m, osd):
    """(worst elementwise relative error, parameter name), smallest cosine over the parameters."""
    cos_min, worst = 1.0, (0.0, None)
    for n, p in m.named_parameters():
        assert p.grad is not None, n
        g, r = p.grad.double().flatten(), osd[n].grad.double().flatten()
        if r.abs().max() > 1e-6 * max(1.0, g.abs().max().item()):  # conv biases before a batch-statistics BN: ~0
            cos_min = min(cos_min, F.cosine_similarity(g, r, dim=0).item())
        worst = max(worst, (relerr(p.grad, osd[n].grad), n))
    return worst, cos_min


@pytest.mark.parametrize("hw", [(64, 64), (50, 75)], ids=["64x64", "50x75"])
@pytest.mark.parametrize("frozen_bn", [False, True], ids=["batchstats", "frozen_bn"])
def test_train_step_host_logic(emulated, hw, frozen_bn):
    """Logits, loss, every parameter gradient and the running statistics of one emulated train step against the oracle's.
    50x75 drops odd rows / columns at several pools on each axis.  With frozen BatchNorm gradients are compared
    elementwise; with batch statistics by direction (the conv biases in front of a batch-statistics BN have a gradient that
    is zero up to rounding, so they are left out of the direction check)."""
    m, osd, x, out, ref, loss, ref_loss = _emulated_step(emulated, hw, frozen_bn)
    assert out.shape == ref.shape == (2, 7) + hw
    assert relerr(out, ref) < (1e-5 if frozen_bn else 2e-3)
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item())
    worst, cos_min = _grad_errors(m, osd)
    if frozen_bn:
        assert worst[0] < 2e-2, worst
    else:
        assert cos_min > 0.99, cos_min
    esd = m.state_dict()
    for k in esd:
        if k.endswith("running_mean") or k.endswith("running_var"):
            assert relerr(esd[k], osd[k]) < 2e-3, k
    m.eval()
    with torch.no_grad():
        ev = m(x)
        ev_ref = osn.segnet_forward(osd, x, train=False)
    assert relerr(ev, ev_ref) < 2e-3


def test_unpool_to_the_wrong_position_is_caught(emulated, monkeypatch):
    """Planted fault: the unpool writes each value to the horizontally mirrored position of its window (code ^ 1).  The
    check of test_train_step_host_logic must fail on the logits."""
    monkeypatch.setattr(emu, "maxunpool2x2_fwd", lambda x, code, hw: _maxunpool2x2_fwd(x, code ^ 1, hw))
    m, osd, x, out, ref, *_ = _emulated_step(emulated, (64, 64), True)
    assert relerr(out, ref) > 1e-2


# ------------------------------------------------------------------------------------------------ SyncBN, gloo world 2
class GlooSync:
    def __init__(self):
        self.rank, self.world = dist.get_rank(), dist.get_world_size()

    def allreduce_(self, vec):
        dist.all_reduce(vec)
        return vec


def _syncbn_step(nets, plosses, sd, x, y, sync):
    m = nets.SegNet(7, pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.bn_sync = sync
    m.dp_reduce = False
    m.train()
    out = m(x)
    loss = plosses._CEFn.apply(out, y, 255, False)
    loss.backward()
    return m, loss.detach()


def _syncbn_worker(rank, world, port, result_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import cpu_emulation as emu_
    from seg_b200 import engine, nets
    from seg_b200 import losses as plosses
    for name, fn in EMU_EXTRA:
        setattr(emu_, name, fn)
    for mod in (engine, nets, plosses):
        mod.ops = emu_
    engine.ACT_DTYPE = torch.float32
    emu_.ACT_DTYPE = torch.float32
    nets._EngineModel._check_input = lambda self, x: None
    sd = osn.segnet_state_dict(7, seed=11, randomize_bn=True)
    x, y = synth.make_batch(4, 48, 40, 7, 255, seed=31)
    half = slice(rank * 2, rank * 2 + 2)
    m, loss = _syncbn_step(nets, plosses, sd, x[half].contiguous(), y[half].contiguous(), GlooSync())
    grads = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    dist.all_reduce(grads)
    grads /= world
    dist.all_reduce(loss)
    loss /= world
    stats = torch.cat([b.reshape(-1).float() for n, b in m.named_buffers() if "running_" in n])
    if rank == 0:
        m1, loss1 = _syncbn_step(nets, plosses, sd, x, y, None)  # single process, concatenated batch
        g1 = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
        s1 = torch.cat([b.reshape(-1).float() for n, b in m1.named_buffers() if "running_" in n])
        torch.save({"loss2": loss, "loss1": loss1,
                    "cos": F.cosine_similarity(grads.double(), g1.double(), dim=0),
                    "grad_rel": (grads - g1).abs().max() / g1.abs().max(),
                    "stats_rel": (stats - s1).abs().max() / s1.abs().max()}, result_path)
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_rank_syncbn_step_equals_single_rank_on_concatenated_batch(tmp_path):
    """A 2-rank SyncBN step on half batches equals the 1-rank step on the concatenated batch (sync_batchnorm/batchnorm.py:
    160-167): loss, rank-averaged gradients and running statistics, through the pool / unpool routing."""
    result = str(tmp_path / "r.pt")
    mp.spawn(_syncbn_worker, args=(2, _free_port(), result), nprocs=2, join=True)
    r = torch.load(result)
    assert abs(r["loss2"].item() - r["loss1"].item()) < 1e-4 * abs(r["loss1"].item()), r
    assert r["stats_rel"].item() < 1e-4, r
    assert r["cos"].item() > 0.999 and r["grad_rel"].item() < 5e-2, r


# ------------------------------------------------------------------------------------------------ against the reference
CODE = r"""
import sys
import torch
import torchvision
_vgg16_bn = torchvision.models.vgg16_bn
def _no_download(*a, **k):  # segnet.py:16 always asks for ImageNet weights: build the network with weights=None instead
    k['weights'] = None
    return _vgg16_bn(*a, **k)
torchvision.models.vgg16_bn = _no_download
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
import models, seg_b200
assert models.SegNet is seg_b200.SegNet, models.SegNet
for name in ('SegResNet', 'UNet'):
    cls = getattr(models, name)
    assert 'reference' in cls.__init__.__code__.co_filename and not cls.__module__.startswith('seg_b200'), (name, cls)
assert 'SegNet' in (models.__doc__ or '')
import importlib
S = importlib.import_module('models.segnet')
for cin in (3, 4):
    ref = S.SegNet(19, in_channels=cin, pretrained=False)
    eng = seg_b200.SegNet(19, in_channels=cin, pretrained=False)
    rs, es = ref.state_dict(), eng.state_dict()
    assert [(k, tuple(v.shape)) for k, v in rs.items()] == [(k, tuple(v.shape)) for k, v in es.items()]
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in eng.named_parameters()]
    eng.load_state_dict(rs, strict=True)
    ref.load_state_dict(es, strict=True)
    assert list(ref.get_backbone_params()) == list(eng.get_backbone_params()) == []
    rn = {id(p): n for n, p in ref.named_parameters()}
    en = {id(p): n for n, p in eng.named_parameters()}
    assert [rn[id(p)] for p in ref.get_decoder_params()] == [en[id(p)] for p in eng.get_decoder_params()]
    for m in (S.SegNet(19, in_channels=cin, pretrained=False, freeze_bn=True, freeze_backbone=True),
              seg_b200.SegNet(19, in_channels=cin, pretrained=False, freeze_bn=True, freeze_backbone=True)):
        assert [n for n, p in m.named_parameters() if p.requires_grad] == [n for n in en.values() if 'decoder' in n]
        assert all(not b.training for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))
    print('SEGNET_OK', cin, sum(p.numel() for p in ref.parameters()), len(rs), len(list(ref.parameters())))
"""


@pytest.mark.skipif(not os.path.isfile(REF_ZIP), reason="oracle/_ref/reference.zip not built (build() found no reference checkout)")
def test_overlay_and_reference_constructor(tmp_path):
    ref = tmp_path / "reference"
    with zipfile.ZipFile(REF_ZIP) as z:
        z.extractall(ref)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "pytorch-segmentation_b200")
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", CODE, str(ref)], env=env, cwd=str(ref), capture_output=True, text=True,
                       timeout=600)
    assert "SEGNET_OK 3 29491027 184 106" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    assert "SEGNET_OK 4 " in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
