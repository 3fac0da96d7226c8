"""Conformance of the parameter path: the batched weight packing and weight-gradient unpacking of `train.WeightTables`,
the single-tensor `seg_pack_weight` / `seg_unpack_wgrad`, the multi-tensor SGD kernel (`seg_sgd_step`,
`seg_sgd_step_dev`), and `FusedTrainStep`'s gradients and updates, all against the float64 references and bounds of
tests/param_check.py.

Kernel-level cases read from and write into sentinel-guarded buffers (NaN pad columns in packed gradients, NaN-prefilled
destinations, sentinel words between rows), run twice and must be bit-identical.  The FusedTrainStep cases take small
models of every engine architecture eagerly and graph-replayed, and check after every step that each packed weight is
the exact bf16 image of the weight the step started from, that each conv weight's gradient is the exact unpacking of its
packed gradient, and that every parameter and momentum buffer satisfies the SGD bound with learning rates derived
independently from the model's parameter groups.  Every case appends its bound usage, the schedule regime it reached and
its wall time to gpu_out_dir/param_conformance.txt."""
import copy
import functools
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import conv_check as cc
import param_check as pc

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib
    from seg_b200.train import FusedTrainStep

from oracle import duc_hdc as od
from oracle import synth, weights
from oracle import unet_resnet as ou

DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32
GAP = 8  # sentinel words before every row and after the last one


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "param_conformance.txt"), "a")
    f.write(f"# {torch.cuda.get_device_name(0)} sms={sms()}\n")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def fmt(u):
    return f"{u:.4f}"


def ibits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


class Arena:
    """n rows of `count` elements in one flat sentinel-filled buffer, GAP sentinel words before every row and after the
    last: each row is a guarded buffer of its own."""

    def __init__(self, n, count, dtype):
        self.n, self.count, self.stride = n, count, count + GAP
        self.buf = cc.sentinel_fill(torch.empty(GAP + n * self.stride, dtype=dtype, device=DEV))

    def rows(self):
        return self.buf[GAP:].view(self.n, self.stride)[:, :self.count]

    def ptr(self, i):
        return self.buf.data_ptr() + (GAP + i * self.stride) * self.buf.element_size()

    def guard_mask(self):
        m = torch.ones(self.buf.shape, dtype=torch.bool)
        m[GAP:].view(self.n, self.stride)[:, :self.count] = False
        return m

    def reset(self):
        cc.sentinel_fill(self.buf)


def make_weights(shape, seed):
    """fp32 weights ~ N(0, 0.05^2), with every 5th element moved exactly onto a bf16 tie, every 7th one ulp below a tie
    and every 11th into the subnormal range: the packing's rounding is exercised where truncation or a flush differs."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(shape, generator=g, device=DEV) * 0.05
    b = w.view(torch.int32).view(-1)
    i = torch.arange(b.numel(), device=DEV)
    b[i % 5 == 0] = (b[i % 5 == 0] & ~0xFFFF) | 0x8000
    b[i % 7 == 0] = (b[i % 7 == 0] & ~0xFFFF) | 0x7FFF
    b[i % 11 == 0] = b[i % 11 == 0] & ~0x7F800000
    return w


def randn(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale


# ------------------------------------------------------------------------------------------------ 1. batched pack / unpack
# (K, C, R, S, explicit)
BIG_ROW = (2048, 512, 3, 3, False)          # 9.4 M elements: hundreds of grid-stride passes per thread
ROW_MIX = [
    (64, 64, 1, 1, False), (64, 64, 3, 3, False), (16, 8, 7, 7, False),
    (64, 3, 7, 7, True),                     # the explicit stem: R*S*C = 147 -> Kpad 152
    (21, 16, 3, 3, True),                    # explicit with R*S*C = 144 already a multiple of 8
    (64, 32, 4, 4, False),                   # ConvTranspose2d(64 -> 32, 4) weight [64, 32, 4, 4] read as OIHW
    (19, 64, 1, 1, False), (21, 256, 1, 1, False), (150, 512, 3, 3, False),
    (1, 8, 1, 1, False),                     # an 8-element row
    (1535, 8, 1, 1, False), (96, 128, 1, 1, False), (1537, 8, 1, 1, False),   # 12288 - 8, 12288, 12288 + 8 elements
    (1117, 11, 1, 1, True), (12289, 1, 1, 1, True),                            # 12287 and 12289 OIHW elements
]
SMALL_ROWS = [(1, 8, 1, 1, False), (3, 8, 1, 1, False), (2, 3, 3, 3, True)]


def geometry(key):
    K, C, R, S, ex = key
    cpad = pc.kpad_for(R, S, C) if ex else C
    pshape = pc.packed_shape(K, C, R, S, ex, cpad)
    return cpad, pshape, int(np.prod(pshape)), K * C * R * S


def upload(tab):
    return torch.from_numpy(tab.view(np.uint8).copy()).to(DEV)


def run_batched(log, case, rows, seed=0):
    """Pack and unpack (beta 0 and 0.5) one table whose row i has shape rows[i]; rows of one shape share an Arena."""
    t0 = time.perf_counter()
    groups = {}
    for i, key in enumerate(rows):
        groups.setdefault(key, []).append(i)
    data, slot = {}, {}
    for gi, (key, idx) in enumerate(groups.items()):
        K, C, R, S, ex = key
        cpad, pshape, pcount, ocount = geometry(key)
        n = len(idx)
        w, pk, gs, ud = Arena(n, ocount, F32), Arena(n, pcount, BF16), Arena(n, pcount, F32), Arena(n, ocount, F32)
        w.rows().copy_(make_weights((n, ocount), seed + 10 * gi))
        ncols = R * S * C if ex else C
        gs.rows().view(n, *pshape)[..., :ncols] = randn((n, *pshape[:-1], ncols), seed + 10 * gi + 1)
        old = randn((n, ocount), seed + 10 * gi + 2)
        data[key] = (w, pk, gs, ud, old)
        for j, i in enumerate(idx):
            slot[i] = j
    prow, urow = [], []
    for i, key in enumerate(rows):
        K, C, R, S, ex = key
        cpad = geometry(key)[0]
        w, pk, gs, ud, _ = data[key]
        prow.append((w.ptr(slot[i]), pk.ptr(slot[i]), K, C, R, S, cpad, ex))
        urow.append((ud.ptr(slot[i]), gs.ptr(slot[i]), K, C, R, S, cpad, ex))
    ptab, ptotal = pc.build_table(prow, "pack")
    utab, utotal = pc.build_table(urow, "unpack")
    ptab_d, utab_d = upload(ptab), upload(utab)
    n = len(rows)

    runs = []
    for _ in range(2):
        for key in groups:
            data[key][1].reset()
        lib.call("seg_pack_weights_batched", ptab_d.data_ptr(), n, ptotal)
        torch.cuda.synchronize()
        runs.append({key: ibits(data[key][1].rows()).clone() for key in groups})
    for key in groups:
        K, C, R, S, ex = key
        _, pshape, _, _ = geometry(key)
        w, pk, _, _, _ = data[key]
        name = f"{case} pack {K}x{C}x{R}x{S}{' explicit' if ex else ''}"
        assert torch.equal(runs[0][key], runs[1][key]), f"{name}: not bit-reproducible"
        cc.check_guards(name, pk.buf, pk.guard_mask())
        pc.check_pack(name, runs[0][key].view(-1, *pshape), pc.pack_ref(w.rows().view(-1, K, C, R, S), ex))
    usage = 0.0
    for beta in (0.0, 0.5):
        runs = []
        for _ in range(2):
            for key in groups:
                ud, old = data[key][3], data[key][4]
                ud.reset()
                if beta != 0.0:
                    ud.rows().copy_(old)
            lib.call("seg_unpack_wgrads_batched", utab_d.data_ptr(), n, utotal, beta)
            torch.cuda.synchronize()
            runs.append({key: data[key][3].rows().clone() for key in groups})
        for key in groups:
            K, C, R, S, ex = key
            cpad, pshape, _, _ = geometry(key)
            _, _, gs, ud, old = data[key]
            name = f"{case} unpack beta={beta} {K}x{C}x{R}x{S}{' explicit' if ex else ''}"
            assert torch.equal(ibits(runs[0][key]), ibits(runs[1][key])), f"{name}: not bit-reproducible"
            cc.check_guards(name, ud.buf, ud.guard_mask())
            cc.check_written(name, runs[0][key])
            ref, bound = pc.unpack_ref(gs.rows().view(-1, *pshape), K, C, R, S, cpad, ex, beta, old.view(-1, K, C, R, S))
            usage = max(usage, pc.check_bounded(name, "unpack", runs[0][key].view(-1, K, C, R, S), ref, bound))
    passes = max(pc.batched_passes(geometry(k)[2]) for k in groups), max(pc.batched_passes(geometry(k)[3]) for k in groups)
    log(f"batched {case}: rows={n} shapes={len(groups)} pack_total={ptotal} unpack_total={utotal} "
        f"unpack_usage(beta=0.5)={fmt(usage)} max_passes_per_thread(pack,unpack)={passes} "
        f"time={time.perf_counter() - t0:.2f}s")


def test_batched_single_big_row(log):
    run_batched(log, "1 row 2048x512x3x3", [BIG_ROW], seed=1)


def test_batched_mixed_rows(log):
    run_batched(log, "mixed", ROW_MIX, seed=2)


def test_batched_resnet101_sized_table(log):
    """~300 rows (a ResNet-101 model's parameters) cycling through the mixed shapes."""
    rows = [ROW_MIX[i % len(ROW_MIX)] for i in range(300) if ROW_MIX[i % len(ROW_MIX)] != (150, 512, 3, 3, False)]
    run_batched(log, f"{len(rows)} rows", rows, seed=3)


def test_batched_largest_table(log):
    rows = [SMALL_ROWS[i % len(SMALL_ROWS)] for i in range(pc.MAX_ROWS)]
    run_batched(log, "65535 rows", rows, seed=4)


# ------------------------------------------------------------------------------------------------ 2. refusals
def refused(name, *args):
    """The call must fail with the library's own refusal, before any launch."""
    before = lib.launch_count()
    with pytest.raises(RuntimeError, match="65535|too many"):
        lib.call(name, *args)
    assert lib.launch_count() == before, f"{name}: a launch was attempted"


def test_tables_and_tensor_lists_over_65535_rows_are_refused():
    n = pc.MAX_ROWS + 1
    tab = upload(pc.build_table([(0, 0, 0, 0, 0, 0, 0, False)] * n, "pack")[0])  # zero-work rows
    refused("seg_pack_weights_batched", tab.data_ptr(), n, 0)
    refused("seg_unpack_wgrads_batched", tab.data_ptr(), n, 0, 0.0)
    ptrs = torch.zeros(n, dtype=torch.int64, device=DEV)
    sizes = torch.zeros(n, dtype=torch.int64, device=DEV)
    lrs = torch.zeros(n, dtype=F32, device=DEV)
    hyper = torch.zeros(2, dtype=F32, device=DEV)
    refused("seg_sgd_step", ptrs.data_ptr(), ptrs.data_ptr(), ptrs.data_ptr(), sizes.data_ptr(), lrs.data_ptr(), n, 0.9, 0.0, 0, 1.0)
    refused("seg_sgd_step_dev", ptrs.data_ptr(), ptrs.data_ptr(), ptrs.data_ptr(), sizes.data_ptr(), lrs.data_ptr(), n,
            hyper.data_ptr(), 0, 1.0)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 3. single pack / unpack
def single_shapes():
    """ROW_MIX as the single kernels see it (an explicit row is packed as the engine does: the [K][R*S*C] matrix as a 1x1
    weight over Kpad channels), one padded Cpad, and 1x1 weights of SMs*8*256 -+ 8 elements, just under and over the
    grid cap (one pass vs two)."""
    out = []
    for K, C, R, S, ex in ROW_MIX:
        out.append((K, C, R, S, ex, pc.kpad_for(R, S, C) if ex else C))
    out.append((19, 64, 1, 1, False, 72))
    k = sms() * 256
    out += [(k - 1, 8, 1, 1, False, 8), (k + 1, 8, 1, 1, False, 8)]
    return out


def test_single_pack_and_unpack(log):
    t0 = time.perf_counter()
    worst, regimes = 0.0, set()
    for i, (K, C, R, S, ex, cpad) in enumerate(single_shapes()):
        name = f"single {K}x{C}x{R}x{S}{' explicit' if ex else ''} Cpad={cpad}"
        w = make_weights((K, C, R, S), 100 + i)
        if ex:  # the engine's explicit packing: OIHW -> [K][(r, s, c)] as a 1x1 weight
            kw, kc, kr, ks = K, R * S * C, 1, 1
            wk = w.permute(0, 2, 3, 1).reshape(K, R * S * C, 1, 1).contiguous()
        else:
            kw, kc, kr, ks, wk = K, C, R, S, w
        pshape = (kr * ks, kw, cpad)
        total = int(np.prod(pshape))
        regimes.add((pc.single_grid(total, sms()), pc.single_passes(total, sms())))
        runs = []
        for _ in range(2):
            dst = cc.FlatGuarded(pshape, BF16, device=DEV)
            lib.call("seg_pack_weight", wk.data_ptr(), dst.view.data_ptr(), kw, kc, kr, ks, cpad)
            torch.cuda.synchronize()
            cc.check_guards(name, dst.buf, dst.guard_mask())
            runs.append(ibits(dst.view).clone())
        assert torch.equal(runs[0], runs[1]), f"{name}: pack not bit-reproducible"
        pc.check_pack(name, runs[0], pc.pack_ref(w, ex, cpad))
        src = cc.sentinel_fill(torch.empty(pshape, dtype=F32, device=DEV))
        src[..., :kc] = randn((*pshape[:-1], kc), 200 + i)
        old = randn((kw, kc, kr, ks), 300 + i)
        for beta in (0.0, 0.5):
            runs = []
            for _ in range(2):
                dst = cc.FlatGuarded((kw, kc, kr, ks), F32, device=DEV)
                if beta != 0.0:
                    dst.view.copy_(old)
                lib.call("seg_unpack_wgrad", src.data_ptr(), dst.view.data_ptr(), kw, kc, kr, ks, cpad, beta)
                torch.cuda.synchronize()
                cc.check_guards(name, dst.buf, dst.guard_mask())
                cc.check_written(name, dst.view)
                runs.append(dst.view.clone())
            assert torch.equal(ibits(runs[0]), ibits(runs[1])), f"{name}: unpack not bit-reproducible"
            ref, bound = pc.unpack_ref(src, kw, kc, kr, ks, cpad, False, beta, old)
            worst = max(worst, pc.check_bounded(f"{name} beta={beta}", "unpack", runs[0], ref, bound))
    assert {p for _, p in regimes} >= {1, 2}
    log(f"single pack/unpack: {len(single_shapes())} shapes unpack_usage(beta=0.5)={fmt(worst)} "
        f"(grid, passes) reached={sorted(regimes)} cap={pc.single_cap(sms())} time={time.perf_counter() - t0:.2f}s")


# ------------------------------------------------------------------------------------------------ 4. SGD kernel
SGD_SIZES = [1, 255, 256, 257, 16383, 16384, 16385]
BIG_N = 2048 * 512 * 9


class SgdSet:
    """n tensors whose params, grads and momentum buffers are slices of three sentinel-guarded fp32 buffers, with pointer
    tables, sizes and a distinct lr per tensor (one of them 0 when n > 1)."""

    def __init__(self, sizes, seed):
        self.sizes, n = sizes, len(sizes)
        self.offs = [GAP + sum(sizes[:i]) + i * GAP for i in range(n)]
        total = self.offs[-1] + sizes[-1] + GAP
        self.p, self.g, self.b = (cc.sentinel_fill(torch.empty(total, dtype=F32, device=DEV)) for _ in range(3))
        self.mask = torch.ones(total, dtype=torch.bool)
        for i, (o, s) in enumerate(zip(self.offs, sizes)):
            self.mask[o:o + s] = False
            self.p[o:o + s] = randn(s, seed + 3 * i)
            self.g[o:o + s] = randn(s, seed + 3 * i + 1, 1e-2)
            self.b[o:o + s] = randn(s, seed + 3 * i + 2, 1e-2)
        lrs = [0.01 * (1 + i % 7) / 4 for i in range(n)]
        if n > 1:
            lrs[n // 2] = 0.0
        self.lrs_host = [pc.f32(v) for v in lrs]
        self.lrs = torch.tensor(lrs, dtype=F32, device=DEV)
        i64 = dict(dtype=torch.int64, device=DEV)
        self.ptrs = [torch.tensor([t.data_ptr() + 4 * o for o in self.offs], **i64) for t in (self.p, self.g, self.b)]
        self.n_t = torch.tensor(sizes, **i64)

    def view(self, t, i):
        return t[self.offs[i]:self.offs[i] + self.sizes[i]]

    def launch(self, entry, mom, wd, first, gs, hyper=None):
        pp, gp, bp = (t.data_ptr() for t in self.ptrs)
        n = len(self.sizes)
        if entry == "seg_sgd_step":
            lib.call(entry, pp, gp, bp, self.n_t.data_ptr(), self.lrs.data_ptr(), n, mom, wd, first, gs)
        else:
            if hyper is None:
                hyper = torch.tensor([mom, wd], dtype=F32, device=DEV)
            lib.call(entry, pp, gp, bp, self.n_t.data_ptr(), self.lrs.data_ptr(), n, hyper.data_ptr(), first, gs)


def run_sgd(case, st, entry, mom, wd, first, gs, hyper=None, nan_buf=False):
    """One launch from the set's current state, checked per tensor; then the same launch again from the same state must
    give the same bits.  Leaves the set in the updated state; returns the largest bound usage."""
    if nan_buf:
        for i in range(len(st.sizes)):
            cc.sentinel_fill(st.view(st.b, i))
    p0, g0, b0 = st.p.clone(), st.g.clone(), st.b.clone()
    outs = []
    for _ in range(2):
        st.p.copy_(p0)
        st.b.copy_(b0)
        st.launch(entry, mom, wd, first, gs, hyper)
        torch.cuda.synchronize()
        outs.append((st.p.clone(), st.b.clone()))
    assert torch.equal(ibits(outs[0][0]), ibits(outs[1][0])) and torch.equal(ibits(outs[0][1]), ibits(outs[1][1])), \
        f"{case}: not bit-reproducible"
    assert torch.equal(ibits(st.g), ibits(g0)), f"{case}: gradients changed"
    cc.check_guards(case + " params", st.p, st.mask)
    cc.check_guards(case + " momentum", st.b, st.mask)
    usage = 0.0
    for i in range(len(st.sizes)):
        r = pc.sgd_ref(st.view(p0, i), st.view(g0, i), st.view(b0, i), st.lrs_host[i], mom, wd, gs, first)
        usage = max(usage, pc.check_sgd(f"{case} tensor {i} (n={st.sizes[i]})", r, st.view(st.p, i), st.view(st.b, i),
                                        st.view(p0, i), st.view(b0, i)))
    return usage


HYPER = [(mom, wd, first, gs) for mom in (0.0, 0.9) for wd in (0.0, 0.1) for first in (0, 1) for gs in (1.0, 0.5, 1 / 3)]
ENTRIES = ["seg_sgd_step", "seg_sgd_step_dev"]


@pytest.mark.parametrize("entry", ENTRIES)
def test_sgd_three_tensors_every_hyperparameter_set(log, entry):
    t0 = time.perf_counter()
    worst = 0.0
    for k, (m, w, f, g) in enumerate(HYPER):  # a fresh set each time: a first step leaves a NaN buffer behind at mu = 0
        st = SgdSet([257, 16385, 1], 500 + 10 * k)
        worst = max(worst, run_sgd(f"{entry} mom={m} wd={w} first={f} gs={g:.4g}", st, entry, m, w, f, g, nan_buf=bool(f)))
    log(f"sgd {entry} n=3 sizes={st.sizes} {len(HYPER)} hyperparameter sets usage={fmt(worst)} "
        f"passes={[pc.sgd_passes(s) for s in st.sizes]} time={time.perf_counter() - t0:.2f}s")


@pytest.mark.parametrize("entry", ENTRIES)
def test_sgd_sizes_at_the_grid_stride_edges(log, entry):
    t0 = time.perf_counter()
    worst = 0.0
    for k, size in enumerate(SGD_SIZES + [BIG_N]):
        st = SgdSet([size], 600 + k)
        for m, w, f, g in [(0.9, 0.1, 0, 1 / 3), (0.9, 0.0, 1, 0.5), (0.0, 0.1, 0, 1.0)]:
            worst = max(worst, run_sgd(f"{entry} size={size} mom={m} wd={w} first={f}", st, entry, m, w, f, g, nan_buf=bool(f)))
    log(f"sgd {entry} single tensors sizes={SGD_SIZES + [BIG_N]} usage={fmt(worst)} "
        f"max_passes={pc.sgd_passes(BIG_N)} time={time.perf_counter() - t0:.2f}s")


@pytest.mark.parametrize("entry", ENTRIES)
def test_sgd_three_hundred_tensors(log, entry):
    t0 = time.perf_counter()
    st = SgdSet([SGD_SIZES[i % len(SGD_SIZES)] for i in range(300)], 700)
    worst = max(run_sgd(f"{entry} n=300 mom={m} wd={w} first={f}", st, entry, m, w, f, g, nan_buf=bool(f))
                for m, w, f, g in [(0.9, 0.1, 0, 1 / 3), (0.0, 0.1, 1, 1.0)])
    log(f"sgd {entry} n=300 usage={fmt(worst)} time={time.perf_counter() - t0:.2f}s")


def test_sgd_dev_reads_hyperparameters_changed_on_the_device(log):
    st = SgdSet([257, 16385, 1], 800)
    hyper = torch.tensor([0.9, 0.1], dtype=F32, device=DEV)
    u1 = run_sgd("dev hyper (0.9, 0.1)", st, "seg_sgd_step_dev", 0.9, 0.1, 0, 1.0, hyper=hyper)
    hyper.copy_(torch.tensor([0.5, 0.0], dtype=F32, device=DEV))  # a device-side write, as a graph replay would see
    u2 = run_sgd("dev hyper (0.5, 0.0)", st, "seg_sgd_step_dev", 0.5, 0.0, 0, 1.0, hyper=hyper)
    hyper.copy_(torch.tensor([0.0, 0.1], dtype=F32, device=DEV))
    u3 = run_sgd("dev hyper (0.0, 0.1)", st, "seg_sgd_step_dev", 0.0, 0.1, 0, 1.0, hyper=hyper)
    log(f"sgd dev hyper changes: usage={fmt(max(u1, u2, u3))}")


# ------------------------------------------------------------------------------------------------ 5. FusedTrainStep
NC, SIZE = 7, 64
MODELS = ["deeplab_r14_os16", "pspnet_r14", "unet_r14", "duc_hdc", "deeplab_xception_os16"]


@functools.lru_cache(maxsize=None)
def base_model(name):
    """The CPU model of `name` with reference-style random weights (built once; tests take deep copies)."""
    if name == "deeplab_r14_os16":
        m, sd = seg_b200.DeepLab(NC, backbone="resnet14", pretrained=False, output_stride=16), \
            weights.deeplab_resnet_state_dict(NC, "resnet14", seed=31, randomize_bn=True)
    elif name == "pspnet_r14":
        m, sd = seg_b200.PSPNet(NC, backbone="resnet14", pretrained=False), \
            weights.pspnet_state_dict(NC, "resnet14", seed=32, randomize_bn=True)
    elif name == "unet_r14":
        m, sd = seg_b200.UNetResnet(NC, backbone="resnet14", pretrained=False), \
            ou.unet_resnet_state_dict(NC, backbone="resnet14", seed=33, randomize_bn=True)
    elif name == "duc_hdc":
        m, sd = seg_b200.DeepLab_DUC_HDC(NC, pretrained=False), od.duc_hdc_state_dict(NC, seed=34, randomize_bn=True)
    else:
        m, sd = seg_b200.DeepLab(NC, backbone="xception", pretrained=False, output_stride=16), \
            weights.deeplab_xception_state_dict(NC, seed=35, randomize_bn=True)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    return m


def fresh(name):
    return copy.deepcopy(base_model(name)).cuda().train()


def batch(seed):
    x, y = synth.make_batch(2, SIZE, SIZE, NC, 255, seed=seed)
    return x.cuda(), y.cuda()


def expected_lrs(m, params, lr):
    """base_trainer.py's parameter groups: lr for get_decoder_params(), lr / 10 for get_backbone_params()."""
    dec = {id(p) for p in m.get_decoder_params()}
    bb = {id(p) for p in m.get_backbone_params()}
    assert not dec & bb
    out = []
    for p in params:
        assert (id(p) in dec) != (id(p) in bb), "a trainable parameter in neither or both groups"
        out.append(lr if id(p) in dec else lr / 10)
    return torch.tensor(out, dtype=F32)


class Snapshot:
    def __init__(self, st):
        self.p = {id(p): p.detach().clone() for p in st.model.parameters()}
        self.mom = st.flat_mom.clone()
        self.mom_views, off = [], 0
        for p in st.params:
            self.mom_views.append(self.mom[off:off + p.numel()].view(p.shape))
            off += p.numel()


def check_tables(case, st, snap):
    """Check 1: every packed weight is the bf16 image of the weight the step started from, and every trainable conv
    weight's gradient view is the exact unpacking of its packed weight gradient."""
    wt = st.wt
    for s in wt.specs:
        name = f"{case} {s.name}"
        pc.check_pack(name, ibits(wt.packed_bufs[s]), pc.pack_ref(snap.p[id(s.m.weight)], s.explicit, s.kpad))
        if s in wt.dw_bufs:
            ref, bound = pc.unpack_ref(wt.dw_bufs[s], s.K, s.C, s.R, s.S, wt.dw_bufs[s].shape[-1], s.explicit)
            pc.check_bounded(name, "weight gradient", st.grad_views[s.m.weight], ref, bound)


def check_update(case, st, snap, lrs, mom, wd):
    """Check 2: every trainable parameter and its momentum against sgd_ref from the step's own gradient."""
    usage = 0.0
    for i, p in enumerate(st.params):
        r = pc.sgd_ref(snap.p[id(p)], st.grad_views[p], snap.mom_views[i], float(lrs[i]), mom, wd, 1.0 / st.world, 0)
        usage = max(usage, pc.check_sgd(f"{case} param {i} {tuple(p.shape)}", r, p.detach(), st.mom_views[i],
                                        snap.p[id(p)], snap.mom_views[i]))
    return usage


def swapped_rows_selftest(case, st, snap):
    """The table check must see two same-shape rows of the unpack table exchanged (snap: the step's snapshot)."""
    tab = st.wt.unpack_table.cpu().numpy().view(pc.PACK_DTYPE).copy()
    seen, pair = {}, None
    for i, e in enumerate(tab):
        key = tuple(int(e[f]) for f in ("K", "C", "R", "S", "Cpad", "explicit"))
        if key in seen:
            pair = (seen[key], i)
            break
        seen[key] = i
    assert pair is not None, f"{case}: no two same-shape rows"
    a, b = pair
    tab[a]["oihw"], tab[b]["oihw"] = int(tab[b]["oihw"]), int(tab[a]["oihw"])
    bad = upload(tab)
    lib.call("seg_unpack_wgrads_batched", bad.data_ptr(), st.wt.unpack_n, st.wt.unpack_total, 0.0)
    torch.cuda.synchronize()
    with pytest.raises(AssertionError, match="weight gradient"):
        check_tables(case + " (rows swapped)", st, snap)
    st.wt.unpack()
    torch.cuda.synchronize()


def check_subtables(case, st):
    """Check 6: unpack_subtables at world 1, a bucket every three parameters and one bucket with no conv weight: after
    the conv-weight gradient views are overwritten with the sentinel, running every subtable must restore flat_grad bit
    for bit, and leave the other views alone."""
    conv_w = {id(s.m.weight) for s in st.wt.specs if s.m.weight.requires_grad}
    bucket_of = {p: (i // 3 if id(p) in conv_w else 10 ** 6) for i, p in enumerate(st.params)}
    subs = st.wt.unpack_subtables(bucket_of)
    assert 10 ** 6 not in subs and len(subs) > 1
    want = st.flat_grad.clone()
    for p in st.params:
        if id(p) in conv_w:
            cc.sentinel_fill(st.grad_views[p])
    for b in sorted(subs):
        tab, n, total = subs[b]
        lib.call("seg_unpack_wgrads_batched", tab.data_ptr(), n, total, 0.0)
    torch.cuda.synchronize()
    assert torch.equal(ibits(st.flat_grad), ibits(want)), f"{case}: bucket subtables differ from the full unpack"
    return len(subs)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", MODELS)
def test_fused_step_tables_and_updates(log, name, graph):
    """Checks 1-3 (and 6, eager) on three steps; between the second and the third, set_lr_scale(0.5) and momentum 0.85
    (a replayed graph must read both)."""
    t0 = time.perf_counter()
    m = fresh(name)
    lr, wd = 0.01, 1e-4
    st = FusedTrainStep(m, lr=lr, momentum=0.9, weight_decay=wd, cuda_graph=graph)
    lrs = expected_lrs(m, st.params, lr)
    assert torch.equal(st.lrs.cpu(), lrs), f"{name}: FusedTrainStep.lrs differ from base_trainer's groups"
    x, y = batch(9400)
    usage, mom = 0.0, 0.9
    for step in range(3):
        if step == 2:
            st.set_lr_scale(0.5)
            st.momentum = 0.85
            lrs, mom = lrs * 0.5, 0.85
            assert torch.equal(st.lrs.cpu(), lrs)
        snap = Snapshot(st)
        st.step(x, y)
        torch.cuda.synchronize()
        case = f"{name} {'graph' if graph else 'eager'} step {step}"
        check_tables(case, st, snap)
        usage = max(usage, check_update(case, st, snap, lrs, mom, wd))
        if step == 0 and not graph:
            swapped_rows_selftest(case, st, snap)
    nsub = check_subtables(name, st) if not graph else 0
    log(f"fused {name} {'graph' if graph else 'eager'}: {len(st.params)} params, {len(st.specs)} packed convs, "
        f"{st.wt.unpack_n} unpack rows, 3 steps update_usage={fmt(usage)} subtables={nsub} "
        f"sgd_passes_max={max(pc.sgd_passes(p.numel()) for p in st.params)} "
        f"pack_passes_max={max(pc.batched_passes(int(np.prod(s.packed_shape()))) for s in st.specs)} "
        f"time={time.perf_counter() - t0:.2f}s")


# Fused and plugin gradients come from the same kernels and differ only in how the loss gradient reaches the logits.
# Measured on an H100 80GB HBM3: 1 - cosine <= 4.4e-16 for every parameter of the five models (the float64 rounding of
# the cosine itself: the two gradients agree to the last bit or nearly so).  The floor leaves a factor of 10^6.
COSINE_FLOOR = 1 - 1e-9


@pytest.mark.parametrize("name", MODELS)
def test_fused_gradients_cover_the_plugin_gradients(log, name):
    """Check 4: frozen BN, one fused step against model(x) -> CrossEntropyLoss2d -> backward on an identical copy: the
    same parameters get a non-zero gradient, and each gradient points the same way."""
    t0 = time.perf_counter()
    mf, mp = fresh(name), fresh(name)
    mf.freeze_bn()
    mp.freeze_bn()
    x, y = batch(9401)
    st = FusedTrainStep(mf, lr=0.01)
    st.step(x, y)
    crit = seg_b200.CrossEntropyLoss2d(ignore_index=255)
    out = mp(x)
    if isinstance(out, tuple):  # PSPNet in training: trainer.py adds 0.4 x the aux head's loss
        loss = crit(out[0], y) + 0.4 * crit(out[1], y)
    else:
        loss = crit(out, y)
    loss.backward()
    torch.cuda.synchronize()
    fused = {n: st.grad_views[p] for n, p in mf.named_parameters() if p.requires_grad}
    plug = dict(mp.named_parameters())
    nz_f = {n for n, g in fused.items() if bool(g.abs().max() > 0)}
    nz_p = {n for n, p in plug.items() if p.grad is not None and bool(p.grad.abs().max() > 0)}
    assert nz_f == nz_p, f"{name}: non-zero gradients only fused {sorted(nz_f - nz_p)[:5]}, only plugin {sorted(nz_p - nz_f)[:5]}"
    cmin, cname = 1.0, None
    for n in nz_f:
        c = torch.nn.functional.cosine_similarity(fused[n].double().flatten(), plug[n].grad.double().flatten(), dim=0).item()
        if c < cmin:
            cmin, cname = c, n
    log(f"coverage {name}: {len(nz_f)} params with a gradient, min cosine fused vs plugin {cmin:.9f} (1 - cos = {1 - cmin:.2e}) at {cname} "
        f"time={time.perf_counter() - t0:.2f}s")
    assert cmin > COSINE_FLOOR, (name, cname, cmin)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_fused_step_with_frozen_backbone(log, graph):
    """Check 5: freeze_backbone=True gives pack rows without unpack rows; the frozen weights stay bit-identical over two
    steps and are still packed correctly, and every other parameter passes the update check."""
    t0 = time.perf_counter()
    sd = base_model("deeplab_r14_os16").state_dict()
    m = seg_b200.DeepLab(NC, backbone="resnet14", pretrained=False, output_stride=16, freeze_backbone=True)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m = m.cuda().train()
    frozen = [p for p in m.parameters() if not p.requires_grad]
    assert frozen and len(frozen) == len(list(m.get_backbone_params()))
    init = [p.detach().clone() for p in frozen]
    st = FusedTrainStep(m, lr=0.01, cuda_graph=graph)
    assert st.wt.unpack_n < len(st.specs)
    lrs = expected_lrs(m, st.params, 0.01)
    assert torch.equal(st.lrs.cpu(), lrs)
    x, y = batch(9402)
    usage = 0.0
    for step in range(2):
        snap = Snapshot(st)
        st.step(x, y)
        torch.cuda.synchronize()
        case = f"frozen backbone {'graph' if graph else 'eager'} step {step}"
        check_tables(case, st, snap)
        usage = max(usage, check_update(case, st, snap, lrs, 0.9, 1e-4))
    for p, q in zip(frozen, init):
        assert torch.equal(ibits(p.detach()), ibits(q)), "a frozen parameter changed"
    log(f"frozen backbone {'graph' if graph else 'eager'}: {len(frozen)} frozen, {len(st.params)} trained, "
        f"{len(st.specs)} pack rows, {st.wt.unpack_n} unpack rows, update_usage={fmt(usage)} "
        f"time={time.perf_counter() - t0:.2f}s")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_bucketed_backward_equals_single_exchange(log, tmp_path):
    """Check 7: see tests/param_dp_worker.py."""
    out = tmp_path / "param_dp.txt"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29619", os.path.join(root, "tests", "param_dp_worker.py"), str(out)],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    text = out.read_text().strip()
    log("two-GPU bucketed vs single exchange: " + text.replace("\n", "; "))
    assert text.endswith("ok"), text
