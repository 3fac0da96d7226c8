"""UNetResnet (models/unet.py:126-209) on the CPU box: the oracle against the reference's golden outputs, the engine model's
constructor (names, shapes, parameter order, parameter groups, init quirks) against the reference's, and the engine's host
logic (transposed convs as dgrad / fprop / wgrad of the mirrored conv, skips written into concat slices by the trunk, the
accumulation of their two gradients, the resample paths, the full-resolution head) under the ATen emulation of
tests/cpu_emulation.py with fp32 storage against the oracle's train step.  The kernels are checked on the GPU by
tests/test_unet_resnet_gpu.py."""
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
from oracle import synth
from oracle import unet_resnet as ou

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden", "unet_resnet.npz")
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
RTOL = 2e-4  # as tests/test_oracle_golden.py


def close(a, b, rtol=RTOL):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    err = np.abs(a - b).max() / (np.abs(b).max() + 1e-12)
    assert err <= rtol, f"rel err {err:.3e} > {rtol:.1e}"


# (prefix, input size, weight seed, batch seed) of oracle/make_golden_unet_resnet.py
GOLDEN_STEPS = [("s64/", 64, 11, 9011), ("s65/", 65, 12, 9012)]


@pytest.mark.parametrize("prefix,size,seed,xseed", GOLDEN_STEPS, ids=[c[0] for c in GOLDEN_STEPS])
def test_oracle_train_step_matches_reference_golden(prefix, size, seed, xseed):
    g = np.load(GOLD)
    sd = om.clone_sd(ou.unet_resnet_state_dict(19, seed=seed, randomize_bn=True), requires_grad=True)
    x, y = synth.make_batch(2, size, size, 19, 255, seed=xseed)
    out = ou.unet_resnet_forward(sd, x, train=True)
    loss = ol.cross_entropy2d(out, y, 255)
    loss.backward()
    assert tuple(out.shape) == tuple(g[prefix + "out_shape"]) == (2, 19, size, size)
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
        ev = ou.unet_resnet_forward(sd, x, train=False)
    close(ev.double().sum((2, 3)).numpy(), g[prefix + "eval_logits_sum"])


# ------------------------------------------------------------------------------------------------ constructor
@pytest.mark.parametrize("backbone,n_keys,n_params,n_numel", [("resnet50", 348, 183, 30000464), ("resnet101", 654, 336, 48992592)])
def test_state_dict_and_parameter_order(backbone, n_keys, n_params, n_numel):
    import seg_b200
    m = seg_b200.UNetResnet(19, backbone=backbone, pretrained=False)
    sd = ou.unet_resnet_state_dict(19, backbone=backbone)
    esd = m.state_dict()
    assert len(esd) == len(sd) == n_keys
    assert [(k, tuple(v.shape)) for k, v in esd.items()] == [(k, tuple(v.shape)) for k, v in sd.items()]
    assert [n for n, _ in m.named_parameters()] == om.param_names(sd) and len(om.param_names(sd)) == n_params
    assert sum(p.numel() for p in m.parameters()) == n_numel
    m.load_state_dict(sd, strict=True)
    if backbone == "resnet50":
        assert [str(n) for n in np.load(GOLD)["s64/param_names"]] == [n for n, _ in m.named_parameters()]


def test_init_quirks():
    """initialize_weights over the whole model: kaiming-normal Conv2d weights and BN gamma 1 / beta 1e-4, trunk included;
    conv biases and ConvTranspose2d weights keep PyTorch's default uniform initialisation."""
    import seg_b200
    torch.manual_seed(0)
    m = seg_b200.UNetResnet(19, pretrained=False)
    bns = [b for b in m.modules() if isinstance(b, nn.BatchNorm2d)]
    assert len(bns) == 55 and all((b.weight == 1).all() and (b.bias == 1e-4).all() for b in bns)
    for name in ("upconv1", "upconv3", "upconv5"):
        w = getattr(m, name).weight  # [in, out, 4, 4]: PyTorch's fan_in is out * 16, kaiming_uniform_(a=sqrt(5))
        bound = 1.0 / (w.shape[1] * 16) ** 0.5
        assert w.abs().max() <= bound and abs(w.std().item() - bound / 3 ** 0.5) < 0.05 * bound, name
    for name in ("conv1", "conv4", "conv6"):
        c = getattr(m, name)
        fan_in = c.in_channels * 9
        assert c.bias.abs().max() <= fan_in ** -0.5 and c.bias.std() > 0.3 * fan_in ** -0.5, name
        assert abs(c.weight.std().item() - (2.0 / fan_in) ** 0.5) < 0.05 * (2.0 / fan_in) ** 0.5, name
    w = m.layer3[2].conv2.weight  # the trunk is re-initialised with kaiming-normal (fan_in), not resnet.py's fan-out normal
    assert abs(w.std().item() - (2.0 / (256 * 9)) ** 0.5) < 0.03 * (2.0 / (256 * 9)) ** 0.5
    assert m.conv7.bias is None and all(getattr(m, f"upconv{i}").bias is None for i in range(1, 6))


def test_parameter_groups_and_options():
    import seg_b200
    m = seg_b200.UNetResnet(19, pretrained=False)
    bb = {id(p) for p in m.get_backbone_params()}
    dec = {id(p) for p in m.get_decoder_params()}
    assert bb == {id(p) for n, p in m.named_parameters() if n.startswith(("initial.", "layer"))}
    assert not (bb & dec) and len(bb | dec) == len(list(m.parameters()))
    m = seg_b200.UNetResnet(19, pretrained=False, freeze_bn=True, freeze_backbone=True)
    assert all(not b.training for b in m.modules() if isinstance(b, nn.BatchNorm2d))
    assert all(not p.requires_grad for p in m.get_backbone_params()) and all(p.requires_grad for p in m.get_decoder_params())
    with pytest.raises(NotImplementedError, match="in_channels"):
        seg_b200.UNetResnet(7, in_channels=4, pretrained=False)
    for bb_name in ("resnet18", "resnet34"):
        with pytest.raises(NotImplementedError, match="backbone"):
            seg_b200.UNetResnet(7, backbone=bb_name, pretrained=False)
    with pytest.raises(RuntimeError, match="network"):
        seg_b200.UNetResnet(7, pretrained=True)


def test_conv_specs_cover_the_transposed_convs():
    """FusedTrainStep's batched weight pack and packed weight-gradient accumulators are built from all_conv_specs()."""
    import seg_b200
    m = seg_b200.UNetResnet(19, pretrained=False)
    specs = {s.name: s for s in m.all_conv_specs()}
    assert len(specs) == sum(1 for x in m.modules() if isinstance(x, (nn.Conv2d, nn.ConvTranspose2d)))
    for i, (cin, cout) in enumerate(((192, 128), (128, 96), (96, 64), (64, 48), (48, 32)), 1):
        s = specs[f"upconv{i}"]
        assert s.transposed and not s.explicit and (s.K, s.C, s.R, s.S, s.stride, s.pad) == (cin, cout, 4, 4, 2, 1)
        assert s.packed_shape() == (16, cin, cout)
    assert not any(s.transposed for s in seg_b200.DeepLab(19, backbone="resnet50", pretrained=False).all_conv_specs())


@pytest.mark.parametrize("mod", [nn.ConvTranspose2d(16, 16, 4, 2, 1, output_padding=1), nn.ConvTranspose2d(16, 16, 4, 2, 1, bias=True),
                                 nn.ConvTranspose2d(16, 16, 4, 2, 1, groups=2, bias=False),
                                 nn.ConvTranspose2d(16, 16, 3, 2, 1, dilation=2, bias=False),
                                 nn.ConvTranspose2d(16, 12, 4, 2, 1, bias=False)],
                         ids=["output_padding", "bias", "groups", "dilation", "cout12"])
def test_unsupported_transposed_convs_raise(mod):
    from seg_b200.engine import ConvSpec
    with pytest.raises(NotImplementedError):
        ConvSpec("t", mod)


# ------------------------------------------------------------------------------------------------ host logic, emulated
def _nhwc_to_nchw(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


def _logits_bwd(dy, r, ldx):
    assert r == 1
    out = torch.zeros(dy.shape[0], dy.shape[2], dy.shape[3], ldx, dtype=emu.ACT_DTYPE)
    out[..., : dy.shape[1]] = dy.permute(0, 2, 3, 1).to(emu.ACT_DTYPE)
    return out


EMU_EXTRA = (("nhwc_to_nchw_f32", _nhwc_to_nchw), ("pixel_shuffle_logits_bwd", _logits_bwd))


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


def _emulated_step(nets, size, frozen_bn, nc=7):
    """(engine model, oracle state_dict with gradients, engine logits, oracle logits, engine loss, oracle loss)."""
    from seg_b200.losses import _CEFn
    sd = ou.unet_resnet_state_dict(nc, seed=5, randomize_bn=True)
    m = nets.UNetResnet(nc, pretrained=False, freeze_bn=frozen_bn)
    m.load_state_dict(sd, strict=True)
    m.train()
    if frozen_bn:
        m.freeze_bn()
    x, y = synth.make_batch(2, size, size, nc, 255, seed=78)
    osd = om.clone_sd(sd, requires_grad=True)
    ref = ou.unet_resnet_forward(osd, x, train=not frozen_bn)
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
        cos_min = min(cos_min, F.cosine_similarity(p.grad.double().flatten(), osd[n].grad.double().flatten(), dim=0).item())
        worst = max(worst, (relerr(p.grad, osd[n].grad), n))
    return worst, cos_min


@pytest.mark.parametrize("size", [64, 65])
@pytest.mark.parametrize("frozen_bn", [False, True], ids=["batchstats", "frozen_bn"])
def test_train_step_host_logic(emulated, size, frozen_bn):
    """Logits, loss, every parameter gradient and the running statistics of one emulated train step against the oracle's.
    64x64 writes upconv3 straight into the x1 concat and needs no final resample; 65x65 takes every resample path.  With
    batch statistics a 50-layer trunk at initialisation amplifies summation-order differences, so gradients are compared by
    direction there; with frozen BatchNorm they are compared elementwise."""
    m, osd, x, out, ref, loss, ref_loss = _emulated_step(emulated, size, frozen_bn)
    assert out.shape == ref.shape == (2, 7, size, size)
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
        ev_ref = ou.unet_resnet_forward(osd, x, train=False)
    assert relerr(ev, ev_ref) < 2e-3


def test_overwritten_skip_gradient_is_caught(emulated, monkeypatch):
    """Planted wiring fault: without Tape.shared_slice the trunk's dgrad into x1 / x2 / x3 overwrites (beta = 0) the slice
    the decoder's concat consumer wrote, instead of adding to it.  The check of test_train_step_host_logic must fail."""
    from seg_b200 import engine
    monkeypatch.setattr(engine.Tape, "shared_slice", lambda self, act: None)
    m, osd, *_ = _emulated_step(emulated, 64, True)
    worst, _ = _grad_errors(m, osd)
    assert worst[0] > 0.1, worst
    assert worst[1].startswith(("initial.", "layer")), worst


# ------------------------------------------------------------------------------------------------ SyncBN, gloo world 2
class GlooSync:
    def __init__(self):
        self.rank, self.world = dist.get_rank(), dist.get_world_size()

    def allreduce_(self, vec):
        dist.all_reduce(vec)
        return vec


def _syncbn_step(nets, plosses, sd, x, y, sync):
    m = nets.UNetResnet(7, backbone="resnet14", pretrained=False)
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
    sd = ou.unet_resnet_state_dict(7, backbone="resnet14", seed=11, randomize_bn=True)
    x, y = synth.make_batch(4, 49, 49, 7, 255, seed=31)
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
    160-167): loss, rank-averaged gradients and running statistics.  Every BatchNorm is in the trunk, so this is the
    trunk's exchange with the decoder's gradients flowing back through the skips."""
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
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
import models, seg_b200
assert models.UNetResnet is seg_b200.UNetResnet, models.UNetResnet
assert models.UNet.__module__.endswith('unet') and 'reference' in models.UNet.__init__.__code__.co_filename
import importlib
U = importlib.import_module('models.unet')
for backbone in ('resnet50', 'resnet101'):
    ref = U.UNetResnet(19, backbone=backbone, pretrained=False)
    eng = seg_b200.UNetResnet(19, backbone=backbone, pretrained=False)
    rs, es = ref.state_dict(), eng.state_dict()
    assert [(k, tuple(v.shape)) for k, v in rs.items()] == [(k, tuple(v.shape)) for k, v in es.items()]
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in eng.named_parameters()]
    eng.load_state_dict(rs, strict=True)
    ref.load_state_dict(es, strict=True)
    for m in (U.UNetResnet(19, backbone=backbone, pretrained=False), seg_b200.UNetResnet(19, backbone=backbone, pretrained=False)):
        names = {id(p): n for n, p in m.named_parameters()}
        groups = ([names[id(p)] for p in m.get_backbone_params()], [names[id(p)] for p in m.get_decoder_params()])
        if m.__class__ is U.UNetResnet:
            ref_groups = groups
        else:
            assert groups == ref_groups
        bns = [b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]
        assert all((b.weight == 1).all() and (b.bias == 1e-4).all() for b in bns)
        w = m.upconv2.weight
        assert w.abs().max() <= (96 * 16) ** -0.5 and w.std() > 0.5 * (96 * 16) ** -0.5 / 3 ** 0.5
        assert m.conv2.bias.abs().max() <= (1152 * 9) ** -0.5 and m.conv2.bias.std() > 0
    print('UNET_OK', backbone, sum(p.numel() for p in ref.parameters()), len(rs), len(list(ref.parameters())))
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
    assert "UNET_OK resnet50 30000464 348 183" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    assert "UNET_OK resnet101 48992592 654 336" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
