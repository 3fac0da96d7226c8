"""FCN8 (models/fcn.py:9-103) on the CPU box: the oracle against the reference's golden outputs, the engine model's
constructor (names, shapes, parameter order, parameter groups, init quirks) against the reference's, and the engine's host
logic (ceil-mode ReLU + pool codes, the windowed score upsamplers with their skip crops, scales and biases, the
full-resolution head) under the ATen emulation of tests/cpu_emulation.py with fp32 storage against the oracle's train step.
The kernels are checked on the GPU by tests/test_fcn_gpu.py."""
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
from oracle import fcn as ofc
from oracle import losses as ol
from oracle import models as om
from oracle import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden", "fcn.npz")
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
RTOL = 2e-4  # as tests/test_oracle_golden.py
NC = 21


def close(a, b, rtol=RTOL):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    err = np.abs(a - b).max() / (np.abs(b).max() + 1e-12)
    assert err <= rtol, f"rel err {err:.3e} > {rtol:.1e}"


# (prefix, H, W, weight seed, batch seed) of oracle/make_golden_fcn.py
GOLDEN_STEPS = [("s64/", 64, 64, 31, 9031), ("s50x75/", 50, 75, 32, 9032)]


@pytest.fixture(scope="module")
def golden_sds():
    return {c[0]: ofc.fcn8_state_dict(NC, seed=c[3]) for c in GOLDEN_STEPS}


@pytest.mark.parametrize("prefix,h,w,seed,xseed", GOLDEN_STEPS, ids=[c[0] for c in GOLDEN_STEPS])
def test_oracle_train_step_matches_reference_golden(golden_sds, prefix, h, w, seed, xseed):
    g = np.load(GOLD)
    sd = om.clone_sd(golden_sds[prefix], requires_grad=True)
    for name, _ in ofc.UPSAMPLERS:
        sd[name + ".weight"].requires_grad_(False)
    x, y = synth.make_batch(2, h, w, NC, 255, seed=xseed)
    out = ofc.fcn8_forward(sd, x)
    loss = ol.cross_entropy2d(out, y, 255)
    loss.backward()
    assert tuple(out.shape) == tuple(g[prefix + "out_shape"]) == (2, NC, h, w)
    close(out.detach()[:, :, ::4, ::4].numpy(), g[prefix + "logits_sub"])
    close(out.detach().double().sum((2, 3)).numpy(), g[prefix + "logits_sum"])
    assert (out.detach().argmax(1).numpy() == g[prefix + "argmax"]).mean() > 0.9995
    close(loss.item(), g[prefix + "loss"], 1e-5)
    names = [str(n) for n in g[prefix + "param_names"]]
    assert names == om.param_names(sd), "oracle parameter order/names differ from the reference's named_parameters()"
    norms = np.array([0.0 if sd[n].grad is None else sd[n].grad.double().norm().item() for n in names])
    close(norms, g[prefix + "grad_norms"], 2e-3)
    for k in g.files:
        if k.startswith(prefix + "grad/"):
            close(sd[k[len(prefix) + 5:]].grad.numpy(), g[k], 2e-3)
    with torch.no_grad():
        ev = ofc.fcn8_forward(sd, x)
    close(ev.double().sum((2, 3)).numpy(), g[prefix + "eval_logits_sum"])


# ------------------------------------------------------------------------------------------------ constructor
@pytest.fixture(scope="module")
def model21():
    import seg_b200
    torch.manual_seed(0)
    return seg_b200.FCN8(NC, pretrained=False)


def test_state_dict_and_parameter_order(model21, golden_sds):
    m = model21
    sd = golden_sds["s64/"]
    esd = m.state_dict()
    assert len(esd) == len(sd) == 39
    assert [(k, tuple(v.shape)) for k, v in esd.items()] == [(k, tuple(v.shape)) for k, v in sd.items()]
    assert [n for n, _ in m.named_parameters()] == om.param_names(sd)
    assert sum(p.numel() for p in m.parameters()) == 134489759
    assert sum(p.numel() for p in m.parameters() if p.requires_grad) == 134362751
    assert [str(n) for n in np.load(GOLD)["s64/param_names"]] == [n for n, _ in m.named_parameters()]


def test_init_quirks(model21):
    """Features: torchvision's VGG init (kaiming-normal fan_out, bias 0) and the first conv padded by 100.  conv6 / conv7:
    N(0, 0.01) Linear weights, bias 0.  Upsamplers: get_upsampling_weight, frozen.  Every pool in ceil mode."""
    m = model21
    assert m.pool3[0].padding == (100, 100) and all(c.padding == (1, 1) for c in m.modules()
                                                    if isinstance(c, nn.Conv2d) and c.kernel_size == (3, 3) and c is not m.pool3[0])
    pools = [p for p in m.modules() if isinstance(p, nn.MaxPool2d)]
    assert len(pools) == 5 and all(p.ceil_mode for p in pools)
    for n, c in m.named_modules():
        if isinstance(c, nn.Conv2d) and n.startswith("pool"):
            sd = (2.0 / (c.out_channels * 9)) ** 0.5
            assert (c.bias == 0).all() and abs(c.weight.std().item() - sd) < 0.1 * sd, n
    for c in (m.output[0], m.output[3]):
        assert (c.bias == 0).all() and abs(c.weight.std().item() - 0.01) < 1e-4 and abs(c.weight.mean().item()) < 1e-4
    for c in (m.adj_pool3, m.adj_pool4, m.output[6]):  # default init: U(-1/sqrt(fan_in), 1/sqrt(fan_in))
        bound = c.in_channels ** -0.5
        assert c.weight.abs().max() <= bound and c.bias.abs().max() <= bound and c.weight.std() > 0.5 * bound
    for up, k in ((m.up_output, 4), (m.up_pool4_out, 4), (m.up_final, 16)):
        assert up.bias is None and not up.weight.requires_grad and up.stride == (k // 2, k // 2)
        assert torch.equal(up.weight, ofc.upsampling_weight(NC, k))
    assert isinstance(m.output[2], nn.Dropout) and m.output[2].p == 0.5 and m.output[5].p == 0.5


def test_parameter_groups_and_options(model21):
    import seg_b200
    m = model21
    names = {id(p): n for n, p in m.named_parameters()}
    back = [names[id(p)] for p in m.get_backbone_params()]
    dec = [names[id(p)] for p in m.get_decoder_params()]
    assert back == [n for n in names.values() if n.split(".")[0] in ("pool3", "pool4", "pool5", "output")]
    assert dec == ["up_output.weight", "adj_pool4.weight", "adj_pool4.bias", "up_pool4_out.weight", "adj_pool3.weight",
                   "adj_pool3.bias", "up_final.weight"]
    specs = {s.name: s for s in m.all_conv_specs()}
    assert sorted(specs) == sorted(n for n, c in m.named_modules() if isinstance(c, nn.Conv2d)) and len(specs) == 18
    assert specs["pool3.0"].explicit and not any(s.explicit for n, s in specs.items() if n != "pool3.0")
    with pytest.raises(RuntimeError, match="network"):
        seg_b200.FCN8(7, pretrained=True)


def test_freeze_backbone_freezes_the_trunk():
    import seg_b200
    m = seg_b200.FCN8(5, pretrained=False, freeze_backbone=True, freeze_bn=True)
    for n, p in m.named_parameters():
        assert p.requires_grad == (n.split(".")[0] in ("output", "adj_pool3", "adj_pool4")), n


@pytest.mark.parametrize("shape", [(1, 4, 64, 64), (1, 1, 64, 64), (3, 64, 64)])
def test_input_without_three_channels_raises(model21, shape):
    with pytest.raises(ValueError, match="3-channel"):
        model21(torch.zeros(*shape))


# ------------------------------------------------------------------------------------------------ host logic, emulated
def _nhwc_to_nchw(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


def _nhwc(t):
    return t.permute(0, 2, 3, 1).to(emu.ACT_DTYPE).contiguous()


def _logits_bwd(dy, r, ldx):
    assert r == 1
    out = torch.zeros(dy.shape[0], dy.shape[2], dy.shape[3], ldx, dtype=emu.ACT_DTYPE)
    out[..., : dy.shape[1]] = dy.permute(0, 2, 3, 1).to(emu.ACT_DTYPE)
    return out


def _relu_maxpool_fwd(x, ceil=True):
    N, H, W, C = x.shape
    y, idx = F.max_pool2d(F.relu(_nhwc_to_nchw(x)), 2, 2, ceil_mode=ceil, return_indices=True)
    P, Q = y.shape[2:]
    code = 2 * (idx // W - 2 * torch.arange(P).view(1, 1, P, 1)) + (idx % W - 2 * torch.arange(Q).view(1, 1, 1, Q))
    assert code.min() >= 0 and code.max() <= 3
    code = torch.where(y > 0, code, code + 4)
    return _nhwc(y), code.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _relu_maxpool_bwd(dy, code, x_shape):
    N, H, W, C = x_shape
    c = code.permute(0, 3, 1, 2).long()
    P, Q = c.shape[2:]
    live = c < 4
    c = c & 3
    idx = (2 * torch.arange(P).view(1, 1, P, 1) + c // 2) * W + 2 * torch.arange(Q).view(1, 1, 1, Q) + c % 2
    return _nhwc(F.max_unpool2d(_nhwc_to_nchw(dy) * live, idx, 2, 2, output_size=(H, W)))


def _relu_dropout_fwd(x, drop_p, seed=0, step_ctr=None):
    assert drop_p == 0.0, "the emulated steps run with the engine's dropout off"
    return F.relu(x)


def _relu_dropout_bwd(dy, y, drop_p, dx, beta):
    g = torch.where(y > 0, dy / (1.0 - drop_p), torch.zeros_like(dy))
    if beta:
        dx += g
    else:
        dx.copy_(g)
    return dx


def _score_pack(w, bwd):
    return w.detach().float().clone()


def _score_upsample_fwd(x, packed, k, window, skip=None, skip_off=(0, 0), alpha=0.0, bias=None, out_dtype=None):
    y0, x0, Ho, Wo = window
    y = F.conv_transpose2d(_nhwc_to_nchw(x), packed, stride=k // 2)[:, :, y0:y0 + Ho, x0:x0 + Wo]
    if skip is not None:
        sy, sx = skip_off
        t = alpha * _nhwc_to_nchw(skip)[:, :, sy:sy + Ho, sx:sx + Wo]
        y = (t + bias.view(1, -1, 1, 1) if bias is not None else t) + y
    return y.permute(0, 2, 3, 1).to(out_dtype or emu.ACT_DTYPE).contiguous()


def _score_upsample_bwd(dy, packed_bwd, x_shape, k, window):
    N, h, w, C = x_shape
    y0, x0, Ho, Wo = window
    s = k // 2
    g = torch.zeros(N, C, (h + 1) * s, (w + 1) * s)
    g[:, :, y0:y0 + Ho, x0:x0 + Wo] = _nhwc_to_nchw(dy)
    return _nhwc(F.conv2d(g, packed_bwd, stride=s))


def _score_skip_bwd(dy, skip_shape, skip_off, alpha, out=None):
    N, Hs, Ws, C = skip_shape
    g = torch.zeros(N, Hs, Ws, C, dtype=emu.ACT_DTYPE)
    g[:, skip_off[0]:skip_off[0] + dy.shape[1], skip_off[1]:skip_off[1] + dy.shape[2]] = alpha * dy.float()
    return g


EMU_EXTRA = (("nhwc_to_nchw_f32", _nhwc_to_nchw), ("pixel_shuffle_logits_bwd", _logits_bwd),
             ("relu_maxpool2x2_ceil_fwd", _relu_maxpool_fwd), ("relu_maxpool2x2_ceil_bwd", _relu_maxpool_bwd),
             ("relu_dropout_fwd", _relu_dropout_fwd), ("relu_dropout_bwd", _relu_dropout_bwd), ("score_pack", _score_pack),
             ("score_upsample_fwd", _score_upsample_fwd), ("score_upsample_bwd", _score_upsample_bwd),
             ("score_skip_bwd", _score_skip_bwd))


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


_SD_CACHE = {}


def _emulated_step(nets, hw, nc=7, dense_up=False):
    """(engine model, oracle state_dict with gradients, input, engine logits, oracle logits, engine loss, oracle loss)."""
    from seg_b200.losses import _CEFn
    key = (nc, dense_up)
    if key not in _SD_CACHE:
        _SD_CACHE[key] = ofc.fcn8_state_dict(nc, seed=5, dense_up=dense_up)
    sd = _SD_CACHE[key]
    m = nets.FCN8(nc, pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m.train()
    x, y = synth.make_batch(2, hw[0], hw[1], nc, 255, seed=78)
    osd = om.clone_sd(sd, requires_grad=True)
    for name, _ in ofc.UPSAMPLERS:
        osd[name + ".weight"].requires_grad_(False)
    ref = ofc.fcn8_forward(osd, x)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    out = m(x)
    loss = _CEFn.apply(out, y, 255)
    loss.backward()
    return m, osd, x, out, ref, loss, ref_loss


def _worst_grad(m, osd):
    worst = (0.0, None)
    for n, p in m.named_parameters():
        if not p.requires_grad:
            assert p.grad is None, n
            continue
        assert p.grad is not None, n
        worst = max(worst, (relerr(p.grad, osd[n].grad), n))
    return worst


@pytest.mark.parametrize("dense_up", [False, True], ids=["bilinear_up", "dense_up"])
@pytest.mark.parametrize("hw", [(64, 64), (50, 75)], ids=["64x64", "50x75"])
def test_train_step_host_logic(emulated, hw, dense_up):
    """Logits, loss and every parameter gradient of one emulated train step (dropout off) against the oracle's, with the
    reference's bilinear upsamplers and with dense random ones.  50x75 has partial ceil windows at four pools."""
    m, osd, x, out, ref, loss, ref_loss = _emulated_step(emulated, hw, dense_up=dense_up)
    assert out.shape == ref.shape == (2, 7) + hw
    assert relerr(out, ref) < 2e-3
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item())
    worst = _worst_grad(m, osd)
    assert worst[0] < 2e-2, worst
    m.eval()
    with torch.no_grad():
        ev = m(x)
    assert relerr(ev, ofc.fcn8_forward(osd, x)) < 2e-3


def test_skip_window_offset_by_one_is_caught(emulated, monkeypatch):
    """Planted fault: every skip crop starts one row and one column late.  The check of test_train_step_host_logic fails."""
    monkeypatch.setattr(emu, "score_upsample_fwd", lambda x, p, k, win, skip=None, skip_off=(0, 0), **kw:
                        _score_upsample_fwd(x, p, k, win, skip, (skip_off[0] + 1, skip_off[1] + 1), **kw))
    m, osd, x, out, ref, *_ = _emulated_step(emulated, (64, 64))
    assert relerr(out, ref) > 2e-3


def test_floor_mode_pools_are_caught(emulated, monkeypatch):
    """Planted fault: the pools in floor mode (smaller maps, different crops).  The check of test_train_step_host_logic
    fails."""
    monkeypatch.setattr(emu, "relu_maxpool2x2_ceil_fwd", lambda x: _relu_maxpool_fwd(x, ceil=False))
    monkeypatch.setattr(emu, "relu_maxpool2x2_ceil_bwd", lambda dy, code, s: _relu_maxpool_bwd(dy, code, s))
    m, osd, x, out, ref, *_ = _emulated_step(emulated, (64, 64))
    assert relerr(out, ref) > 2e-3


def test_trainable_upsampler_raises(emulated):
    m = emulated.FCN8(5, pretrained=False)
    m.up_final.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="upsampling weight"):
        m(torch.zeros(1, 3, 40, 40))


# ------------------------------------------------------------------------------------------------ data parallel, gloo world 2
def _dp_step(nets, plosses, sd, x, y, dp_reduce):
    m = nets.FCN8(5, pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m.dp_reduce = dp_reduce
    m.train()
    out = m(x)
    loss = plosses._CEFn.apply(out, y, 255, False)
    loss.backward()
    return m, loss.detach()


def _dp_worker(rank, world, port, result_path):
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
    sd = ofc.fcn8_state_dict(5, seed=11)
    x, y = synth.make_batch(4, 48, 40, 5, 255, seed=31)
    y[:, :2] = 255  # the same count of ignored pixels in every image: per-rank means average to the global mean
    half = slice(rank * 2, rank * 2 + 2)
    m, loss = _dp_step(nets, plosses, sd, x[half].contiguous(), y[half].contiguous(), True)  # the engine's own exchange
    grads = torch.cat([p.grad.reshape(-1) for p in m.parameters() if p.requires_grad])
    dist.all_reduce(loss)
    loss /= world
    if rank == 0:
        m1, loss1 = _dp_step(nets, plosses, sd, x, y, False)  # single process, concatenated batch
        g1 = torch.cat([p.grad.reshape(-1) for p in m1.parameters() if p.requires_grad])
        torch.save({"loss2": loss, "loss1": loss1, "grad_rel": (grads - g1).abs().max() / g1.abs().max()}, result_path)
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_rank_step_equals_single_rank_on_concatenated_batch(tmp_path):
    """Two ranks on half batches, with the model's own gradient all-reduce, give the loss and gradients of one rank on the
    concatenated batch (FCN8 has no BatchNorm: no statistics exchange)."""
    result = str(tmp_path / "r.pt")
    mp.spawn(_dp_worker, args=(2, _free_port(), result), nprocs=2, join=True)
    r = torch.load(result)
    assert abs(r["loss2"].item() - r["loss1"].item()) < 1e-5 * abs(r["loss1"].item()), r
    assert r["grad_rel"].item() < 1e-4, r


# ------------------------------------------------------------------------------------------------ against the reference
CODE = r"""
import sys
import torch
import torchvision
_vgg16 = torchvision.models.vgg16
def _no_download(*a, **k):  # fcn.py:12 asks for ImageNet weights: build the network with weights=None instead
    k.pop('pretrained', None)
    k['weights'] = None
    return _vgg16(**k)
torchvision.models.vgg16 = _no_download
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
import models, seg_b200
assert models.FCN8 is seg_b200.FCN8, models.FCN8
for name in ('SegResNet', 'UNet'):
    cls = getattr(models, name)
    assert 'reference' in cls.__init__.__code__.co_filename and not cls.__module__.startswith('seg_b200'), (name, cls)
assert 'FCN8' in (models.__doc__ or '')
import importlib
Fm = importlib.import_module('models.fcn')
try:
    Fm.FCN8(21, pretrained=False)
    raise SystemExit('the reference FCN8 constructed without the shim')
except NameError:
    pass
from utils.helpers import set_trainable
Fm.freeze_backbone = False
Fm.set_trainable = set_trainable
ref = Fm.FCN8(21, pretrained=False)
eng = seg_b200.FCN8(21, pretrained=False)
rs, es = ref.state_dict(), eng.state_dict()
assert [(k, tuple(v.shape)) for k, v in rs.items()] == [(k, tuple(v.shape)) for k, v in es.items()]
assert [n for n, _ in ref.named_parameters()] == [n for n, _ in eng.named_parameters()]
eng.load_state_dict(rs, strict=True)
ref.load_state_dict(es, strict=True)
rn = {id(p): n for n, p in ref.named_parameters()}
en = {id(p): n for n, p in eng.named_parameters()}
assert [rn[id(p)] for p in ref.get_backbone_params()] == [en[id(p)] for p in eng.get_backbone_params()]
assert [rn[id(p)] for p in ref.get_decoder_params()] == [en[id(p)] for p in eng.get_decoder_params()]
assert [n for n, p in ref.named_parameters() if p.requires_grad] == [n for n, p in eng.named_parameters() if p.requires_grad]
for a, b in ((ref.up_output, eng.up_output), (ref.up_pool4_out, eng.up_pool4_out), (ref.up_final, eng.up_final)):
    assert torch.equal(a.weight, b.weight) and not a.weight.requires_grad and not b.weight.requires_grad
for a, b in ((ref.output[0], eng.output[0]), (ref.output[3], eng.output[3])):
    assert abs(a.weight.std().item() - b.weight.std().item()) < 1e-4 and (a.bias == 0).all() and (b.bias == 0).all()
# freeze_backbone as the reference intends it (set_trainable over pool3 / pool4 / pool5)
Fm.freeze_backbone = True
rf = Fm.FCN8(21, pretrained=False)
ef = seg_b200.FCN8(21, pretrained=False, freeze_backbone=True)
assert [n for n, p in rf.named_parameters() if p.requires_grad] == [n for n, p in ef.named_parameters() if p.requires_grad]
print('FCN8_OK', sum(p.numel() for p in ref.parameters()), sum(p.numel() for p in ref.parameters() if p.requires_grad), len(rs))
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
    assert "FCN8_OK 134489759 134362751 39" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
