"""Self-tests of tests/param_check.py (no GPU): the references and bounds accept fp32 emulations of the parameter-path
kernels, with and without FMA contraction, and reject the seeded mistakes a packing table, a packing kernel or the SGD
kernel could make.  The last tests build `train.WeightTables` for small models on the CPU and compare its device tables,
byte for byte, with the checker's independent builder."""
import os
import sys

import numpy as np
import pytest
import torch

import param_check as pc
from conv_check import check_guards, check_written, sentinel_fill

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pytorch-segmentation_b200", "libseg_b200.so")
F32 = torch.float32


def rand(n, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g, dtype=torch.float64) * scale).float()


def rejects(fn, *args, match=None, **kw):
    with pytest.raises(AssertionError, match=match):
        fn(*args, **kw)


# ------------------------------------------------------------------------------------------------ SGD
SGD_SETS = [(lr, mom, wd, gs, first) for lr in (0.1, 0.0) for mom in (0.0, 0.9) for wd in (0.0, 0.1)
            for gs in (1.0, 0.5, 1 / 3) for first in (0, 1)]


def sgd_inputs(n=4096, seed=0, nan_buf=False):
    p, g = rand(n, seed), rand(n, seed + 1, 1e-2)
    buf = sentinel_fill(torch.empty(n, dtype=F32)) if nan_buf else rand(n, seed + 2, 1e-2)
    return p, g, buf


@pytest.mark.parametrize("fma", [False, True], ids=["no-fma", "fma"])
@pytest.mark.parametrize("lr,mom,wd,gs,first", SGD_SETS)
def test_sgd_bounds_accept_fp32_emulation(lr, mom, wd, gs, first, fma):
    p, g, buf = sgd_inputs(nan_buf=bool(first))
    r = pc.sgd_ref(p, g, buf, lr, mom, wd, gs, first)
    pn, bn = pc.sgd_emulate(p, g, buf, lr, mom, wd, gs, first, fma)
    pc.check_sgd("emulated", r, pn, bn, p, buf)


def test_sgd_fma_and_plain_emulations_differ():
    """The two emulations are different arithmetic (otherwise accepting both shows nothing)."""
    p, g, buf = sgd_inputs(1 << 14)
    a = pc.sgd_emulate(p, g, buf, 0.1, 0.9, 0.1, 1 / 3, 0, False)
    b = pc.sgd_emulate(p, g, buf, 0.1, 0.9, 0.1, 1 / 3, 0, True)
    assert not torch.equal(a[0], b[0]) and not torch.equal(a[1], b[1])


def test_sgd_ref_uses_the_fp32_scalars():
    """grad_scale 1/3 reaches the kernel as float32(1/3): a float64 1/3 reference is off by more than the bound allows
    for large gradients."""
    p, g = torch.zeros(1, dtype=F32), torch.full((1,), 3.0 * 2 ** 20, dtype=F32)
    r = pc.sgd_ref(p, g, torch.zeros(1), 1.0, 0.9, 0.0, 1 / 3, 1)
    assert r.m.item() == float(np.float32(1 / 3)) * 3.0 * 2 ** 20 != 2.0 ** 20


def _sgd_mistake(kind, p, g, buf, lr, mom, wd, gs, first):
    """(p', buf') of an fp32 SGD with one seeded mistake."""
    f = lambda v: torch.tensor(pc.f32(v), dtype=F32)  # noqa: E731
    lr_t, mom_t, wd_t, gs_t = f(lr), f(mom), f(wd), f(gs)
    if kind == "no_weight_decay":
        wd_t = f(0.0)
    if kind == "grad_scale_ignored":
        gs_t = f(1.0)
    if kind == "neighbour_lr":
        lr_t = f(lr * 0.1)
    b = buf.clone()
    if kind == "momentum_before_weight_decay":
        m = mom_t * buf + g * gs_t if not first else g * gs_t
        b = m
        return p - lr_t * (m + wd_t * p), b
    d = g * gs_t + wd_t * p
    if float(mom_t) != 0.0:
        if kind == "dampening":
            m = mom_t * buf + (1 - mom_t) * d
        elif kind == "first_step_ignored" or not first:
            m = mom_t * buf + d
        else:
            m = d
        b, d = m, m
    elif kind == "buffer_written_at_zero_momentum":
        b = d
    return p - lr_t * d, b


SGD_MISTAKES = {  # kind: (lr, mom, wd, gs, first, NaN-filled old buffer)
    "no_weight_decay": (0.1, 0.9, 0.1, 1.0, 0, False),
    "grad_scale_ignored": (0.1, 0.9, 0.0, 0.5, 0, False),
    "neighbour_lr": (0.1, 0.9, 0.1, 1.0, 0, False),
    "dampening": (0.1, 0.9, 0.1, 1.0, 0, False),
    "momentum_before_weight_decay": (0.1, 0.9, 0.1, 1.0, 0, False),
    "first_step_ignored": (0.1, 0.9, 0.1, 1.0, 1, True),
    "buffer_written_at_zero_momentum": (0.1, 0.0, 0.1, 1.0, 0, False),
}


@pytest.mark.parametrize("kind", list(SGD_MISTAKES))
def test_sgd_check_rejects_seeded_mistake(kind):
    lr, mom, wd, gs, first, nan_buf = SGD_MISTAKES[kind]
    p, g, buf = sgd_inputs(nan_buf=nan_buf)
    r = pc.sgd_ref(p, g, buf, lr, mom, wd, gs, first)
    pn, bn = _sgd_mistake(kind, p, g, buf, lr, mom, wd, gs, first)
    rejects(pc.check_sgd, kind, r, pn, bn, p, buf)


def test_sgd_zero_lr_must_return_the_parameter_bit_for_bit():
    p, g, buf = sgd_inputs()
    r = pc.sgd_ref(p, g, buf, 0.0, 0.9, 0.1, 1.0, 0)
    pn, bn = pc.sgd_emulate(p, g, buf, 0.0, 0.9, 0.1, 1.0, 0, False)
    pc.check_sgd("lr 0", r, pn, bn, p, buf)
    pn2 = pn.clone()
    pn2[7] = torch.nextafter(pn2[7], torch.tensor(np.inf, dtype=F32))
    rejects(pc.check_sgd, "lr 0, one ulp", r, pn2, bn, p, buf, match="lr = 0")


# ------------------------------------------------------------------------------------------------ pack
def tie_inputs():
    """fp32 values exactly on bf16 ties and one ulp either side, with even and odd kept bits, in the normal and the
    subnormal range and with both signs."""
    vals = []
    for hi in (0x3F80, 0x3F81, 0x4049, 0x0000, 0x0001, 0x007F, 0x0080, 0x7F7E, 0x4B7F):
        for lo in (0x7FFF, 0x8000, 0x8001, 0x0000, 0xFFFF):
            for sign in (0, 0x80000000):
                vals.append(sign | (hi << 16) | lo)
    return torch.tensor(np.array(vals, dtype=np.uint32).view(np.int32)).view(F32)


def test_bf16_bits_is_round_to_nearest_even():
    x = tie_inputs()
    want = x.to(torch.bfloat16).view(torch.int16)
    assert torch.equal(pc.bf16_bits(x), want)
    assert torch.equal(pc.bf16_bits(rand(1 << 16, 3)), rand(1 << 16, 3).to(torch.bfloat16).view(torch.int16))


def test_pack_check_rejects_truncation_at_ties():
    x = tie_inputs()
    trunc = (x.view(torch.int32) >> 16).to(torch.int16)
    w = x[:40].reshape(5, 8, 1, 1)  # K=5, C=8
    want = pc.pack_ref(w, False)
    got_trunc = pc.pack_ref(w, False).clone()
    got_trunc.view(-1)[:] = trunc[:40].reshape(5, 8).view(-1)
    rejects(pc.check_pack, "truncation", got_trunc, want)
    sub = x[(x.view(torch.int32) & 0x7F800000) == 0]  # subnormal inputs alone
    assert sub.numel() >= 20
    rejects(pc.check_pack, "truncation, subnormals", (sub.view(torch.int32) >> 16).to(torch.int16), pc.bf16_bits(sub))


def test_pack_ref_layouts():
    w = torch.arange(2 * 3 * 2 * 2, dtype=F32).reshape(2, 3, 2, 2)  # K=2, C=3, R=S=2: small integers are bf16-exact
    normal = pc.pack_ref(w, False, 8).view(torch.bfloat16).float()
    assert normal.shape == (4, 2, 8)
    assert normal[1 * 2 + 0, 1, 2].item() == w[1, 2, 1, 0].item() and normal[..., 3:].abs().sum() == 0
    ex = pc.pack_ref(w, True).view(torch.bfloat16).float()
    assert ex.shape == (1, 2, 16)  # R*S*C = 12 -> Kpad 16
    assert ex[0, 1, (1 * 2 + 0) * 3 + 2].item() == w[1, 2, 1, 0].item()
    assert torch.equal(pc.pack_ref(w, True)[..., 12:], torch.zeros(1, 2, 4, dtype=torch.int16))


def test_pack_check_rejects_crs_column_order():
    w = rand(8 * 3 * 7 * 7, 5).reshape(8, 3, 7, 7)
    want = pc.pack_ref(w, True)
    crs = w.reshape(8, 3 * 7 * 7)
    got = torch.cat([pc.bf16_bits(crs), torch.zeros(8, 152 - 147, dtype=torch.int16)], 1).view(1, 8, 152)
    assert want.shape == got.shape == (1, 8, 152)
    rejects(pc.check_pack, "(c, r, s) columns", got, want)


def test_pack_check_rejects_transposed_conv_read_with_k_and_c_swapped():
    """A ConvTranspose2d(64 -> 32) weight is [64, 32, 4, 4], read as OIHW with K = 64, C = 32; a packer that takes the
    memory for [32][64][4][4] and transposes packs the same shape with the wrong values."""
    w = rand(64 * 32 * 16, 6).reshape(64, 32, 4, 4)
    want = pc.pack_ref(w, False)
    assert want.shape == (16, 64, 32)
    got = pc.pack_ref(w.reshape(32, 64, 4, 4).transpose(0, 1), False)
    rejects(pc.check_pack, "K/C swapped", got, want)


@pytest.mark.parametrize("bits", [0x8000, 0x3F80], ids=["minus_zero", "one"])
def test_pack_check_rejects_dirty_pad_column(bits):
    w = rand(4 * 3 * 7 * 7, 7).reshape(4, 3, 7, 7)
    want = pc.pack_ref(w, True, 152)
    got = want.clone()
    got[0, 2, 150] = bits - 0x10000 if bits >= 0x8000 else bits
    rejects(pc.check_pack, "pad", got, want)


# ------------------------------------------------------------------------------------------------ unpack
def packed_src(K, C, R, S, explicit, seed, nan_pad=True):
    cpad = pc.kpad_for(R, S, C) if explicit else C
    shape = pc.packed_shape(K, C, R, S, explicit, cpad)
    t = sentinel_fill(torch.empty(shape, dtype=F32))
    n = R * S * C if explicit else C
    t[..., :n] = rand(int(np.prod(shape[:-1])) * n, seed).reshape(*shape[:-1], n)
    return t, cpad


@pytest.mark.parametrize("fma", [False, True], ids=["no-fma", "fma"])
@pytest.mark.parametrize("explicit", [False, True], ids=["normal", "explicit"])
@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
def test_unpack_bounds_accept_fp32_emulation(beta, explicit, fma):
    K, C, R, S = (19, 3, 7, 7) if explicit else (19, 64, 3, 3)
    src, cpad = packed_src(K, C, R, S, explicit, 11)
    old = rand(K * C * R * S, 12).reshape(K, C, R, S)
    ref, bound = pc.unpack_ref(src, K, C, R, S, cpad, explicit, beta, old)
    got = pc.unpack_emulate(src, K, C, R, S, explicit, beta, old, fma)
    assert not torch.isnan(got).any()  # the NaN pad columns were not read
    pc.check_bounded("emulated", "unpack", got, ref, bound)


def test_unpack_beta0_overwrites_nan_destination_exactly():
    src, cpad = packed_src(8, 16, 3, 3, False, 13)
    ref, bound = pc.unpack_ref(src, 8, 16, 3, 3, cpad, False)
    assert bound.abs().sum() == 0
    dst = sentinel_fill(torch.empty(8, 16, 3, 3, dtype=F32))
    rejects(pc.check_bounded, "NaN left", "unpack", dst, ref, bound)
    got = pc.unpack_emulate(src, 8, 16, 3, 3, False, 0.0, dst, False)
    pc.check_bounded("ok", "unpack", got, ref, bound)
    got.view(-1)[5] = torch.nextafter(got.view(-1)[5], torch.tensor(np.inf, dtype=F32))
    rejects(pc.check_bounded, "one ulp", "unpack", got, ref, bound)


def test_unpack_check_rejects_ignored_beta():
    src, cpad = packed_src(19, 64, 3, 3, False, 14)
    old = rand(19 * 64 * 9, 15).reshape(19, 64, 3, 3)
    ref, bound = pc.unpack_ref(src, 19, 64, 3, 3, cpad, False, 0.5, old)
    rejects(pc.check_bounded, "beta ignored", "unpack", pc.unpack_emulate(src, 19, 64, 3, 3, False, 0.0, old, False), ref, bound)


def test_unpack_check_rejects_k_and_cpad_swapped_in_the_source_index():
    """src[((r S + s) Cpad + k) K + c] instead of src[((r S + s) K + k) Cpad + c]: stays inside the tap's block for K < Cpad."""
    K, C, R, S = 19, 64, 3, 3
    src, cpad = packed_src(K, C, R, S, False, 16)
    ref, bound = pc.unpack_ref(src, K, C, R, S, cpad, False)
    k, c, r, s = torch.meshgrid(*(torch.arange(n) for n in (K, C, R, S)), indexing="ij")
    idx = ((r * S + s) * cpad + k) * K + c
    got = src.reshape(-1)[idx]
    rejects(pc.check_bounded, "K/Cpad swapped", "unpack", got, ref, bound)


# ---- the batched unpack over a table, emulated on flat CPU arenas (offsets stand in for pointers)
def emulate_batched_unpack(tab, total, src, dst):
    """unpack_wgrads_batched_kernel with beta = 0: row i covers work items [start_i, start_{i+1}) (the last up to
    total), reading the packed gradient at src[packed] and writing OIHW dst[oihw + j]."""
    n = len(tab)
    for i in range(n):
        e = tab[i]
        count = (int(tab[i + 1]["start"]) if i + 1 < n else total) - int(e["start"])
        K, C, R, S, cpad, ex = (int(e[f]) for f in ("K", "C", "R", "S", "Cpad", "explicit"))
        j = torch.arange(count)
        s_, t = j % S, j // S
        r_, t = t % R, t // R
        c_, k_ = t % C, t // C
        si = k_ * cpad + (r_ * S + s_) * C + c_ if ex else ((r_ * S + s_) * K + k_) * cpad + c_
        dst[int(e["oihw"]) + j] = src[int(e["packed"]) + si]


UNPACK_ROWS = [(96, 128, 1, 1, False), (19, 64, 3, 3, False), (64, 3, 7, 7, True), (8, 8, 1, 1, False)]


def unpack_arena(rows, gap=8):
    """Sources (NaN pad columns) and sentinel destinations of `rows` on flat arenas with `gap` sentinel words around
    every row; returns (table rows with offsets, src arena, dst arena, [(dst offset, OIHW shape, packed source, cpad)])."""
    src_parts, trows, views = [], [], []
    s_off, d_off = gap, gap
    for i, (K, C, R, S, ex) in enumerate(rows):
        p, cpad = packed_src(K, C, R, S, ex, 20 + i)
        src_parts.append((s_off, p))
        trows.append((d_off, s_off, K, C, R, S, cpad, ex))
        views.append((d_off, (K, C, R, S), p, cpad, ex))
        s_off += p.numel() + gap
        d_off += K * C * R * S + gap
    src = sentinel_fill(torch.empty(s_off, dtype=F32))
    for o, p in src_parts:
        src[o:o + p.numel()] = p.reshape(-1)
    dst = sentinel_fill(torch.empty(d_off, dtype=F32))
    return trows, src, dst, views


def check_unpack_arena(case, dst, views):
    mask = torch.ones(dst.shape, dtype=torch.bool)
    for d_off, shape, p, cpad, ex in views:
        n = int(np.prod(shape))
        mask[d_off:d_off + n] = False
        v = dst[d_off:d_off + n].view(shape)
        check_written(case, v)
        ref, bound = pc.unpack_ref(p, *shape, cpad, ex)
        pc.check_bounded(case, "unpack", v, ref, bound)
    check_guards(case, dst, mask)


def test_batched_unpack_emulation_passes_the_arena_checks():
    trows, src, dst, views = unpack_arena(UNPACK_ROWS)
    tab, total = pc.build_table(trows, "unpack")
    assert int(tab[1]["start"]) == pc.BATCHED_STRIDE  # the first row is exactly one grid-stride pass
    emulate_batched_unpack(tab, total, src, dst)
    check_unpack_arena("emulated", dst, views)


@pytest.mark.parametrize("delta", [1, -1])
def test_batched_unpack_check_rejects_start_off_by_one_at_the_stride_boundary(delta):
    trows, src, dst, views = unpack_arena(UNPACK_ROWS)
    tab, total = pc.build_table(trows, "unpack")
    tab[1]["start"] += delta  # 12288 +- 1: row 0 writes one element past its end, or leaves its last one unwritten
    emulate_batched_unpack(tab, total, src, dst)
    rejects(check_unpack_arena, f"start {delta:+d}", dst, views)


def test_batched_unpack_check_rejects_a_missing_last_element():
    trows, src, dst, views = unpack_arena(UNPACK_ROWS)
    tab, total = pc.build_table(trows, "unpack")
    emulate_batched_unpack(tab, total - 1, src, dst)
    rejects(check_unpack_arena, "total - 1", dst, views, match="never written")


def test_batched_unpack_check_rejects_two_same_shape_rows_swapped():
    trows, src, dst, views = unpack_arena([(16, 16, 3, 3, False), (8, 8, 1, 1, False), (16, 16, 3, 3, False)])
    trows[0], trows[2] = trows[2][:1] + trows[0][1:], trows[0][:1] + trows[2][1:]  # destinations exchanged
    tab, total = pc.build_table(trows, "unpack")
    emulate_batched_unpack(tab, total, src, dst)
    rejects(check_unpack_arena, "rows swapped", dst, views)


# ------------------------------------------------------------------------------------------------ schedule mirrors
def test_schedule_mirrors():
    assert pc.BATCHED_STRIDE == 12288 and pc.SGD_STRIDE == 16384
    assert [pc.batched_passes(n) for n in (1, 12287, 12288, 12289)] == [1, 1, 1, 2]
    assert [pc.sgd_passes(n) for n in (1, 16383, 16384, 16385)] == [1, 1, 1, 2]
    cap = pc.single_cap(132)
    assert cap == 132 * 8 * 256
    assert pc.single_grid(cap - 256, 132) == 132 * 8 - 1 and pc.single_passes(cap - 256, 132) == 1
    assert pc.single_grid(cap + 1, 132) == 132 * 8 and pc.single_passes(cap + 1, 132) == 2


# ------------------------------------------------------------------------------------------------ tables vs WeightTables
@pytest.fixture(scope="module")
def lib_built():
    for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    if not os.path.exists(LIB):
        import __graft_entry__
        __graft_entry__.build()
    from seg_b200 import lib
    assert pc.PACK_DTYPE.itemsize == lib.load().seg_pack_entry_bytes()
    return lib


def small_models():
    import seg_b200
    torch.manual_seed(0)
    yield "deeplab_r14", seg_b200.DeepLab(7, backbone="resnet14", pretrained=False, output_stride=16)
    yield "deeplab_r14_frozen_backbone", seg_b200.DeepLab(7, backbone="resnet14", pretrained=False, output_stride=16,
                                                          freeze_backbone=True)
    yield "unet_r14", seg_b200.UNetResnet(7, backbone="resnet14", pretrained=False)


def test_weight_tables_match_the_independent_builder(lib_built):
    """WeightTables on CPU tensors (raw pointers are just numbers here): its pack and unpack tables, and the bucket
    subtables, must be the bytes the checker's builder makes from the weights' shapes."""
    from seg_b200.train import WeightTables
    for name, m in small_models():
        params = [p for p in m.parameters() if p.requires_grad]
        gv = {p: torch.zeros_like(p) for p in params}
        wt = WeightTables(m, gv, "cpu")
        prow, urow = pc.spec_rows(wt.specs, wt.packed_bufs, wt.dw_bufs, gv)
        kinds = {(r[7], r[2] != r[3]) for r in prow}
        if name.startswith("unet"):
            assert any(s.transposed and s.K != s.C for s in wt.specs), name
        assert (True, True) in kinds, name  # the explicit stem
        ptab, ptotal = pc.build_table(prow, "pack")
        assert ptotal == wt.pack_total and bytes(wt.pack_table.numpy()) == ptab.tobytes(), name
        utab, utotal = pc.build_table(urow, "unpack")
        assert utotal == wt.unpack_total and wt.unpack_n == len(urow), name
        if "frozen" in name:
            assert len(urow) < len(prow)
        assert bytes(wt.unpack_table.numpy()) == utab.tobytes(), name
        # buckets of every third trainable conv weight, and one bucket holding only non-conv parameters
        conv_w = [s.m.weight for s in wt.specs if s.m.weight.requires_grad]
        bucket_of = {p: (i // 3) for i, p in enumerate(conv_w)}
        other = [p for p in params if all(p is not w for w in conv_w)]
        for p in other:
            bucket_of[p] = 10 ** 6
        subs = wt.unpack_subtables(bucket_of)
        assert 10 ** 6 not in subs
        for b, (tab, n, total) in subs.items():
            rows = [r for r, w in zip(urow, conv_w) if bucket_of[w] == b]
            want, wtotal = pc.build_table(rows, "unpack")
            assert (n, total) == (len(rows), wtotal) and bytes(tab.numpy()) == want.tobytes(), (name, b)
