"""DeepLab_DUC_HDC (models/duc_hdc.py) on the CPU box: the oracle against the reference's golden outputs, the engine model's
constructor (names, shapes, parameter order, HDC plan, ICNR init, parameter groups) against the reference's, and the engine's
host logic (tape order, pixel-shuffle slices, the data gradient of DUC_out's im2col conv, the shuffle head) under the ATen
emulation of tests/cpu_emulation.py with fp32 storage against the oracle's train step.  The kernels are checked on the GPU by
tests/test_duc_hdc_gpu.py."""
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cpu_emulation as emu
from oracle import duc_hdc as od
from oracle import losses as ol
from oracle import models as om
from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "duc_hdc.npz")
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
RTOL = 2e-4  # as tests/test_oracle_golden.py


def close(a, b, rtol=RTOL):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    err = np.abs(a - b).max() / (np.abs(b).max() + 1e-12)
    assert err <= rtol, f"rel err {err:.3e} > {rtol:.1e}"


# (prefix, output_stride, weight seed, input size, batch seed) of oracle/make_golden_duc_hdc.py
GOLDEN_STEPS = [("os8/", 8, 7, 64, 9005), ("os4/", 4, 8, 32, 9007)]


def golden_batch(os_, size, seed):
    x, y = synth.make_batch(2, size, size, 19, 255, seed=seed)
    if os_ == 4:
        y = F.interpolate(y[:, None].float(), size=(2 * size, 2 * size), mode="nearest")[:, 0].long()
    return x, y


@pytest.mark.parametrize("prefix,os_,seed,size,xseed", GOLDEN_STEPS, ids=[c[0] for c in GOLDEN_STEPS])
def test_oracle_train_step_matches_reference_golden(prefix, os_, seed, size, xseed):
    g = np.load(GOLD)
    sd = om.clone_sd(od.duc_hdc_state_dict(19, seed=seed, randomize_bn=True), requires_grad=True)
    x, y = golden_batch(os_, size, xseed)
    out = od.duc_hdc_forward(sd, x, output_stride=os_, train=True)
    loss = ol.cross_entropy2d(out, y, 255)
    loss.backward()
    assert tuple(out.shape) == tuple(g[prefix + "out_shape"])
    close(out.detach()[:, :, ::3, ::3].numpy(), g[prefix + "logits_sub"])
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
        ev = od.duc_hdc_forward(sd, x, output_stride=os_, train=False)
    close(ev.double().sum((2, 3)).numpy(), g[prefix + "eval_logits_sum"])


def test_oracle_odd_input_is_not_cropped():
    """A 65x65 input gives a 68x68 output (4 x the 17x17 layer1 map), as the reference does."""
    g = np.load(GOLD)
    sd = od.duc_hdc_state_dict(19, seed=7, randomize_bn=True)
    x, _ = synth.make_batch(2, 65, 65, 19, 255, seed=9006)
    with torch.no_grad():
        out = od.duc_hdc_forward(sd, x, train=False)
    assert tuple(out.shape) == tuple(g["odd65/out_shape"]) == (2, 19, 68, 68)
    close(out[:, :, ::3, ::3].numpy(), g["odd65/logits_sub"])
    close(out.double().sum((2, 3)).numpy(), g["odd65/logits_sum"])


# ------------------------------------------------------------------------------------------------ constructor
def test_state_dict_and_parameter_order_match_the_reference():
    import seg_b200
    m = seg_b200.DeepLab_DUC_HDC(19, pretrained=False)
    sd = od.duc_hdc_state_dict(19)
    esd = m.state_dict()
    assert len(esd) == len(sd) == 704
    assert [(k, tuple(v.shape)) for k, v in esd.items()] == [(k, tuple(v.shape)) for k, v in sd.items()]
    names = [str(n) for n in np.load(GOLD)["os8/param_names"]]  # the reference's named_parameters()
    assert [n for n, _ in m.named_parameters()] == names
    assert sum(p.numel() for p in m.parameters()) == 69183651
    m.load_state_dict(sd, strict=True)
    assert [c for c, _ in m.named_children()] == ["backbone", "ASSP", "decoder", "DUC_out"]


def test_hdc_dilation_plan():
    import seg_b200
    for os_ in (8, 4):
        m = seg_b200.DeepLab_DUC_HDC(5, pretrained=False, output_stride=os_)
        bb = m.backbone
        assert bb.layer0[0].stride == ((2, 2) if os_ == 8 else (1, 1))
        want = {1: [1] * 3, 2: [1] * 4, 3: [1, 2, 3] * 7 + [2, 2], 4: [3, 4, 5]}
        for li, dils in want.items():
            layer = getattr(bb, f"layer{li}")
            assert [b.conv2.dilation[0] for b in layer] == dils, li
            assert [b.conv2.padding[0] for b in layer] == dils, li
            assert [b.conv2.stride[0] for b in layer] == [2 if li == 2 else 1] + [1] * (len(dils) - 1), li
            assert layer[0].downsample[0].stride[0] == (2 if li == 2 else 1)
        assert [getattr(m.ASSP, f"aspp{i}")[0].dilation[0] for i in range(1, 7)] == [1, 6, 12, 18, 24, 36]
        assert [getattr(m.ASSP, f"aspp{i}")[0].padding[0] for i in range(1, 7)] == [0, 6, 12, 18, 24, 36]
    with pytest.raises(AssertionError):
        seg_b200.DeepLab_DUC_HDC(5, pretrained=False, output_stride=16)


def test_existing_plans_build_the_same_layers():
    """The per-block dilation form of _res_layers and the (stride, first, other) form describe the same modules."""
    from seg_b200.nets import _res_layers
    a = _res_layers((3, 4, 6, 3), 64, [(1, 1, 1), (2, 1, 1), (1, 1, 2), (1, 2, 4)])
    b = _res_layers((3, 4, 6, 3), 64, [(1, [1] * 3), (2, [1] * 4), (1, [1] + [2] * 5), (1, [2, 4, 4])])
    assert [repr(x) for x in a] == [repr(x) for x in b]


def test_init_quirks():
    """ICNR on DUC_out.conv only (Decoder's initialize_weights overwrites decoder.DUC.conv); BN gamma 1 / beta 1e-4 where
    initialize_weights reaches, torchvision's 1 / 0 in layers 1-4."""
    import seg_b200
    m = seg_b200.DeepLab_DUC_HDC(19, pretrained=False)
    assert od.is_icnr(m.DUC_out.conv.weight, 4)
    assert not od.is_icnr(m.decoder.DUC.conv.weight, 2)
    for bn in (m.DUC_out.bn, m.decoder.DUC.bn, m.ASSP.bn1, m.backbone.layer0[1], m.decoder.output[4]):
        assert (bn.weight == 1).all() and (bn.bias == 1e-4).all()
    assert (m.backbone.layer3[5].bn2.bias == 0).all()
    w = m.DUC_out.conv.weight
    assert abs(w[::16].std().item() - (2.0 / 19) ** 0.5) < 0.1  # kaiming-normal, fan_in = 19


def test_parameter_groups_and_options():
    import seg_b200
    m = seg_b200.DeepLab_DUC_HDC(19, pretrained=False)
    bb = {id(p) for p in m.get_backbone_params()}
    dec = {id(p) for p in m.get_decoder_params()}
    assert bb == {id(p) for n, p in m.named_parameters() if n.startswith("backbone.")}
    assert not (bb & dec) and len(bb | dec) == len(list(m.parameters()))
    m = seg_b200.DeepLab_DUC_HDC(19, pretrained=False, freeze_bn=True, freeze_backbone=True)
    assert all(not b.training for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))
    assert all(not p.requires_grad for p in m.get_backbone_params()) and all(p.requires_grad for p in m.get_decoder_params())
    assert seg_b200.DeepLab_DUC_HDC(7, in_channels=4, pretrained=False).backbone.layer0[0].weight.shape == (64, 4, 7, 7)
    with pytest.raises(RuntimeError, match="network"):
        seg_b200.DeepLab_DUC_HDC(7, pretrained=True)


# ------------------------------------------------------------------------------------------------ host logic, emulated
def _ps_fwd(x, r, Ho, Wo, out=None):
    y = F.pixel_shuffle(emu._nchw(x), r)[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    if out is None:
        out = torch.empty(y.shape, dtype=emu.ACT_DTYPE)
    return emu._store(out, y)


def _ps_bwd(dy, r, H, W, dx=None, beta=0.0):
    N, Ho, Wo, C = dy.shape
    full = torch.zeros(N, C, H * r, W * r)
    full[:, :, :Ho, :Wo] = emu._nchw(dy)
    g = F.pixel_unshuffle(full, r).permute(0, 2, 3, 1)
    if dx is None:
        dx, beta = torch.empty(g.shape, dtype=emu.ACT_DTYPE), 0.0
    return emu._store(dx, g, beta)


def _psl_fwd(x, r):
    return F.pixel_shuffle(emu._nchw(x), r).contiguous()


def _psl_bwd(dy, r, ldx):
    g = F.pixel_unshuffle(dy, r).permute(0, 2, 3, 1)
    out = torch.zeros(g.shape[:3] + (ldx,), dtype=emu.ACT_DTYPE)
    out[..., : g.shape[-1]] = g.to(emu.ACT_DTYPE)
    return out


@pytest.fixture()
def emulated(monkeypatch):
    from seg_b200 import engine, nets
    from seg_b200 import losses as plosses
    for name, fn in (("pixel_shuffle_fwd", _ps_fwd), ("pixel_shuffle_bwd", _ps_bwd), ("pixel_shuffle_logits_fwd", _psl_fwd),
                     ("pixel_shuffle_logits_bwd", _psl_bwd)):
        monkeypatch.setattr(emu, name, fn, raising=False)
    for mod in (engine, nets, plosses):
        monkeypatch.setattr(mod, "ops", emu)
    monkeypatch.setattr(engine, "ACT_DTYPE", torch.float32)
    monkeypatch.setattr(emu, "ACT_DTYPE", torch.float32)
    monkeypatch.setattr(nets._EngineModel, "_check_input", lambda self, x: None)
    return nets


def relerr(a, b):
    return ((a.detach().double() - b.detach().double()).abs().max() / (b.detach().double().abs().max() + 1e-12)).item()


@pytest.mark.parametrize("os_,size", [(8, 64), (4, 32)])
@pytest.mark.parametrize("frozen_bn", [False, True], ids=["batchstats", "frozen_bn"])
def test_train_step_host_logic(emulated, os_, size, frozen_bn):
    """Logits, loss, every parameter gradient and the running statistics of one emulated train step against the oracle's.
    Without the data gradient of DUC_out's im2col conv, nothing upstream of it would get a gradient.  With batch statistics a
    101-layer trunk at initialisation amplifies summation-order differences (as for DeepLab in test_engine_cpu_emulated.py),
    so gradients are compared by direction there; with frozen BatchNorm the step is smooth and they are compared elementwise."""
    from seg_b200.losses import _CEFn
    nc = 7
    sd = od.duc_hdc_state_dict(nc, seed=5, randomize_bn=True)
    m = emulated.DeepLab_DUC_HDC(nc, pretrained=False, output_stride=os_, freeze_bn=frozen_bn)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m.train()
    if frozen_bn:
        m.freeze_bn()
    x, y = synth.make_batch(4, size, size, nc, 255, seed=78)  # 4 images: the image-pooling BN sees 4 samples
    if os_ == 4:
        y = F.interpolate(y[:, None].float(), size=(2 * size, 2 * size), mode="nearest")[:, 0].long()
    osd = om.clone_sd(sd, requires_grad=True)
    ref = od.duc_hdc_forward(osd, x, output_stride=os_, train=not frozen_bn)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    out = m(x)
    loss = _CEFn.apply(out, y, 255)
    loss.backward()
    assert out.shape == ref.shape
    assert relerr(out, ref) < (1e-5 if frozen_bn else 2e-3)
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item())
    norms = torch.tensor([osd[n].grad.double().norm().item() for n, _ in m.named_parameters()])
    floor = 1e-4 * norms.median().item()
    cos_min, worst = 1.0, (0.0, None)
    for n, p in m.named_parameters():
        assert p.grad is not None, n
        if osd[n].grad.double().norm().item() < floor:
            # analytically zero: decoder.output.7's bias shifts every input channel of the 1x1 DUC_out conv by a constant,
            # which the batch-statistics BatchNorm after it removes; both sides hold rounding noise only
            assert p.grad.double().norm().item() < 100 * floor, n
            continue
        cos_min = min(cos_min, F.cosine_similarity(p.grad.double().flatten(), osd[n].grad.double().flatten(), dim=0).item())
        worst = max(worst, (relerr(p.grad, osd[n].grad), n))
    if frozen_bn:
        assert worst[0] < 2e-2, worst  # ReLU-mask flips on near-zero pre-activations deep in the trunk
    else:
        assert cos_min > 0.99, cos_min
    for n in ("backbone.layer0.0.weight", "backbone.layer3.22.conv2.weight", "ASSP.conv1.weight", "decoder.DUC.conv.weight",
              "decoder.output.7.weight"):
        assert dict(m.named_parameters())[n].grad.norm() > 0, n
    esd = m.state_dict()
    for k in esd:
        if k.endswith("running_mean") or k.endswith("running_var"):
            assert relerr(esd[k], osd[k]) < 2e-3, k
    m.eval()
    with torch.no_grad():
        ev = m(x)
        ev_ref = od.duc_hdc_forward(osd, x, output_stride=os_, train=False)
    assert relerr(ev, ev_ref) < 2e-3


# ------------------------------------------------------------------------------------------------ against the reference
CODE = r"""
import sys
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
import models, seg_b200
assert models.DeepLab_DUC_HDC is seg_b200.DeepLab_DUC_HDC, models.DeepLab_DUC_HDC
assert models.UNet.__module__.endswith('unet') and 'reference' in models.UNet.__init__.__code__.co_filename
import importlib
D = importlib.import_module('models.duc_hdc')
from utils import helpers
D.freeze_backbone, D.set_trainable = False, helpers.set_trainable   # duc_hdc.py:225 reads both, defines neither
ref = D.DeepLab_DUC_HDC(19, pretrained=False)
eng = seg_b200.DeepLab_DUC_HDC(19, pretrained=False)
rs, es = ref.state_dict(), eng.state_dict()
assert [(k, tuple(v.shape)) for k, v in rs.items()] == [(k, tuple(v.shape)) for k, v in es.items()]
assert [n for n, _ in ref.named_parameters()] == [n for n, _ in eng.named_parameters()]
eng.load_state_dict(rs, strict=True)
ref.load_state_dict(es, strict=True)
assert [id(p) for p in ref.get_backbone_params()] and len(list(ref.get_decoder_params())) == len(list(eng.get_decoder_params()))
w = D.DeepLab_DUC_HDC(19, pretrained=False)
for m in (w, seg_b200.DeepLab_DUC_HDC(19, pretrained=False)):
    v = m.DUC_out.conv.weight.detach().reshape(19, 16, 19)
    assert (v == v[:, :1]).all()
    v = m.decoder.DUC.conv.weight.detach().reshape(256, 4, 256)
    assert not (v == v[:, :1]).all()
print('DUC_HDC_OK', sum(p.numel() for p in ref.parameters()))
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
    assert "DUC_HDC_OK 69183651" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
