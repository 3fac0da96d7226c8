"""GPU parity tests of every C-ABI entry point against the ATen CPU ops the reference dispatches to
(nn.Conv2d / BatchNorm2d / MaxPool2d / AdaptiveAvgPool2d / F.interpolate / CrossEntropyLoss — SURVEY.md §2.3).
Inputs are bf16-rounded first so the comparison isolates kernel arithmetic (fp32 accumulate) from quantisation.
Tolerances: fp32 outputs 2e-3 of the output scale, bf16 outputs 1e-2 (north_star: 1e-3 fp32 / 1e-2 bf16)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib, ops
    from seg_b200.lib import IMPL_SIMT, IMPL_TC
else:  # keep collection working on the CPU box
    IMPL_SIMT, IMPL_TC = 1, 2

DEV = "cuda"


def bf(t):
    return t.to(torch.bfloat16).to(torch.float32)


def rel_err(got, ref):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    scale = ref.abs().max().item() + 1e-12
    return (got - ref).abs().max().item() / scale


def check(name, got, ref, tol, gpu_out_dir=None):
    e = rel_err(got, ref)
    msg = f"{name}: rel_err={e:.3e} tol={tol:.1e}"
    print(msg)
    if gpu_out_dir:
        with open(os.path.join(gpu_out_dir, "op_parity.txt"), "a") as f:
            f.write(msg + "\n")
    if not (e <= tol):
        g = got.detach().float().cpu()
        r = ref.detach().float().cpu()
        diff = (g - r).abs()
        bad = (diff > tol * (r.abs().max() + 1e-12)).nonzero()
        detail = f"{msg}; shape={tuple(g.shape)} nbad={bad.shape[0]} first_bad={bad[:8].tolist()} got_absmax={g.abs().max():.4g} ref_absmax={r.abs().max():.4g} nan={torch.isnan(g).sum().item()}"
        if gpu_out_dir:
            with open(os.path.join(gpu_out_dir, "op_parity.txt"), "a") as f:
                f.write("FAIL " + detail + "\n")
        pytest.fail(detail)


# (N, H, W, C, K, ksize, stride, pad, dil)
CONV_SHAPES = [
    (2, 33, 33, 64, 64, 1, 1, 0, 1),      # plain 1x1 GEMM, M tail
    (2, 33, 33, 256, 48, 1, 1, 0, 1),     # decoder.conv1: K=48 (N tile tail)
    (1, 17, 19, 64, 64, 3, 1, 1, 1),      # 3x3, non-square odd map
    (2, 33, 33, 128, 256, 3, 1, 2, 2),    # layer4-style dilation 2
    (2, 33, 33, 512, 256, 3, 1, 6, 6),    # ASPP d=6
    (2, 33, 33, 256, 256, 3, 1, 12, 12),  # ASPP d=12
    (2, 33, 33, 128, 64, 3, 1, 18, 18),   # ASPP d=18 (most taps in padding)
    (1, 33, 33, 304, 256, 3, 1, 1, 1),    # decoder concat: C=304 (K-chunk tail)
    (2, 33, 33, 128, 128, 3, 2, 1, 1),    # stride-2 3x3 (layer2.0.conv2)
    (2, 33, 33, 256, 512, 1, 2, 0, 1),    # stride-2 1x1 downsample
    (3, 9, 9, 2048, 512, 1, 1, 0, 1),     # deep K
    (2, 34, 30, 64, 128, 3, 2, 1, 1),     # stride 2 on even maps (parity classes of unequal size)
    (1, 129, 129, 64, 256, 1, 1, 0, 1),   # many M tiles, short K: epilogue-bound shape
    (4, 65, 65, 128, 1024, 1, 1, 0, 1),   # persistent kernel: 8 column blocks, several tiles per CTA
    (2, 65, 65, 192, 320, 3, 1, 1, 1),    # persistent kernel: column-block tail (320 = 2.5 x 128), C tail
    (1, 129, 129, 64, 64, 3, 1, 1, 1),    # one-tile kernel with 131 row tiles: two-level statistics fold (layer1 conv2 shape)
]


def conv_inputs(shape, seed=0):
    N, H, W, C, K, ks, stride, pad, dil = shape
    g = torch.Generator().manual_seed(seed)
    x = bf(torch.randn(N, C, H, W, generator=g))
    w = bf(torch.randn(K, C, ks, ks, generator=g) / (C * ks * ks) ** 0.5)
    return x, w


def to_nhwc_dev(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(DEV, torch.bfloat16)


@pytest.mark.parametrize("impl", [IMPL_SIMT, IMPL_TC], ids=["simt", "tc"])
@pytest.mark.parametrize("shape", CONV_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_fwd(shape, impl, gpu_out_dir):
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = conv_inputs(shape)
    ref = F.conv2d(x, w, None, stride, pad, dil)
    wp = ops.pack_weight(w.to(DEV))
    # fp32 output + statistics: wgmma path only (the CUDA-core path reduces the stored bf16 output)
    stats = ops.new_stats(K, DEV) if impl == IMPL_TC else None  # zeroed fp64 accumulators
    y = ops.conv2d_fwd(to_nhwc_dev(x), wp, K, ks, ks, stride, pad, dil, out_dtype=torch.float32, stats=stats, impl=impl)
    torch.cuda.synchronize()
    check(f"conv_fwd[{impl}] {shape}", y.permute(0, 3, 1, 2), ref, 2e-3, gpu_out_dir)
    ref_s = torch.cat([ref.sum((0, 2, 3)), (ref * ref).sum((0, 2, 3))])
    if stats is not None:
        check(f"conv_fwd_stats[{impl}] {shape}", stats, ref_s, 2e-3, gpu_out_dir)
    stats_b = ops.new_stats(K, DEV)
    yb = ops.conv2d_fwd(to_nhwc_dev(x), wp, K, ks, ks, stride, pad, dil, stats=stats_b, impl=impl)
    torch.cuda.synchronize()
    check(f"conv_fwd_bf16[{impl}] {shape}", yb.permute(0, 3, 1, 2), ref, 1e-2, gpu_out_dir)
    check(f"conv_fwd_bf16_stats[{impl}] {shape}", stats_b, ref_s, 2e-3, gpu_out_dir)
    # the statistics are the sums of the output AS STORED, accumulated exactly in fp64: equal to a float64 sum of the stored
    # bf16 values up to the fp32 rounding of the per-CTA partial sums, and bit-identical from run to run
    yd = yb.double().reshape(-1, K)
    exact = torch.cat([yd.sum(0), (yd * yd).sum(0)])
    check(f"conv_fwd_bf16_stats_vs_stored[{impl}] {shape}", stats_b, exact, 2e-5, gpu_out_dir)
    for _ in range(3):
        again = ops.new_stats(K, DEV)
        ops.conv2d_fwd(to_nhwc_dev(x), wp, K, ks, ks, stride, pad, dil, stats=again, impl=impl)
        assert torch.equal(again, stats_b), "BatchNorm statistics are not bit-reproducible"


@pytest.mark.parametrize("impl", [IMPL_SIMT, IMPL_TC], ids=["simt", "tc"])
@pytest.mark.parametrize("shape", CONV_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_dgrad(shape, impl, gpu_out_dir):
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = conv_inputs(shape)
    x.requires_grad_(True)
    y = F.conv2d(x, w, None, stride, pad, dil)
    g = torch.Generator().manual_seed(1)
    dy = bf(torch.randn(y.shape, generator=g))
    y.backward(dy)
    wp = ops.pack_weight(w.to(DEV))
    dx = ops.conv2d_dgrad(to_nhwc_dev(dy), wp, (N, H, W, C), ks, ks, stride, pad, dil, impl=impl)
    torch.cuda.synchronize()
    check(f"conv_dgrad[{impl}] {shape}", dx.permute(0, 3, 1, 2), x.grad, 1e-2, gpu_out_dir)
    # beta = 1 accumulation
    dx2 = ops.conv2d_dgrad(to_nhwc_dev(dy), wp, (N, H, W, C), ks, ks, stride, pad, dil, out=dx.clone(), beta=1.0, impl=impl)
    check(f"conv_dgrad_beta1[{impl}] {shape}", dx2.permute(0, 3, 1, 2), 2 * x.grad, 1.5e-2, gpu_out_dir)


@pytest.mark.parametrize("impl", [IMPL_SIMT, IMPL_TC], ids=["simt", "tc"])
@pytest.mark.parametrize("shape", CONV_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_wgrad(shape, impl, gpu_out_dir):
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = conv_inputs(shape)
    w.requires_grad_(True)
    y = F.conv2d(x, w, None, stride, pad, dil)
    g = torch.Generator().manual_seed(1)
    dy = bf(torch.randn(y.shape, generator=g))
    y.backward(dy)
    dwp = ops.conv2d_wgrad(to_nhwc_dev(dy), to_nhwc_dev(x), ks, ks, stride, pad, dil, impl=impl)
    dw = ops.unpack_wgrad(dwp, (K, C, ks, ks))
    torch.cuda.synchronize()
    check(f"conv_wgrad[{impl}] {shape}", dw, w.grad, 2e-3, gpu_out_dir)


def test_conv_bias_k19_and_slices(gpu_out_dir):
    """decoder.output.7: 256 -> 19 with bias, fp32 logits; input read from / output written to channel slices."""
    g = torch.Generator().manual_seed(3)
    x = bf(torch.randn(2, 256, 17, 17, generator=g))
    w = bf(torch.randn(19, 256, 1, 1, generator=g) / 16)
    b = torch.randn(19, generator=g)
    ref = F.conv2d(x, w, b)
    big = torch.zeros(2, 17, 17, 320, device=DEV, dtype=torch.bfloat16)
    big[..., 48:304] = to_nhwc_dev(x)
    for impl in (IMPL_SIMT, IMPL_TC):
        y = ops.conv2d_fwd(big[..., 48:304], ops.pack_weight(w.to(DEV)), 19, 1, 1, out_dtype=torch.float32, bias=b.to(DEV), impl=impl)
        check(f"conv_k19_bias[{impl}]", y.permute(0, 3, 1, 2), ref, 2e-3, gpu_out_dir)
    # 3x3 conv writing into a slice of a wider buffer
    w3 = bf(torch.randn(64, 256, 3, 3, generator=g) / 48)
    ref3 = F.conv2d(x, w3, None, 1, 1, 1)
    for impl in (IMPL_SIMT, IMPL_TC):
        outbuf = torch.zeros(2, 17, 17, 128, device=DEV, dtype=torch.bfloat16)
        ops.conv2d_fwd(big[..., 48:304], ops.pack_weight(w3.to(DEV)), 64, 3, 3, 1, 1, 1, out=outbuf[..., 64:128], impl=impl)
        check(f"conv_slice_out[{impl}]", outbuf[..., 64:128].permute(0, 3, 1, 2), ref3, 1e-2, gpu_out_dir)
        assert outbuf[..., :64].abs().max().item() == 0


def test_stem_im2col(gpu_out_dir):
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 65, 65, generator=g)
    w = bf(torch.randn(64, 3, 7, 7, generator=g) / 12)
    ref = F.conv2d(bf(x), w, None, 2, 3, 1)
    col = ops.im2col(x.to(DEV), 7, 7, 2, 3, 1, 152, nchw_f32=True)
    wp = ops.pack_weight(w.permute(0, 2, 3, 1).reshape(64, 147, 1, 1).contiguous().to(DEV), cpad=152)
    for impl in (IMPL_SIMT, IMPL_TC):
        y = ops.conv2d_fwd(col, wp, 64, 1, 1, out_dtype=torch.float32, impl=impl)
        check(f"stem_im2col[{impl}]", y.permute(0, 3, 1, 2), ref, 2e-3, gpu_out_dir)


@pytest.mark.parametrize("C,M_shape", [(64, (2, 33, 33)), (48, (1, 17, 9)), (2048, (2, 5, 5)), (256, (4, 1, 1))])
def test_bn_train_fwd_bwd(C, M_shape, gpu_out_dir):
    g = torch.Generator().manual_seed(5)
    N, H, W = M_shape
    x = bf(torch.randn(N, C, H, W, generator=g) * 1.5 + 0.3).requires_grad_(True)
    res = bf(torch.randn(N, C, H, W, generator=g))
    gamma = (torch.rand(C, generator=g) + 0.5).requires_grad_(True)
    beta = (torch.randn(C, generator=g) * 0.1).requires_grad_(True)
    rm, rv = torch.zeros(C), torch.ones(C)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    y = F.relu(F.batch_norm(x, rm_ref, rv_ref, gamma, beta, True, 0.1, 1e-5) + res)
    dy = bf(torch.randn(y.shape, generator=g))
    res_g = res.clone().requires_grad_(True)
    y2 = F.relu(F.batch_norm(x, rm.clone(), rv.clone(), gamma, beta, True, 0.1, 1e-5) + res_g)
    y2.backward(dy)
    xd, resd, dyd = to_nhwc_dev(x.detach()), to_nhwc_dev(res), to_nhwc_dev(dy)
    gd, bd, rmd, rvd = gamma.detach().to(DEV), beta.detach().to(DEV), rm.to(DEV), rv.to(DEV)
    stats = ops.bn_stats(xd)
    count = N * H * W
    ss, save = ops.bn_finalize(stats, count, gd, bd, 1e-5, 0.1, 0, rmd, rvd)
    out = ops.bn_apply(xd, ss, res=resd, relu=True)
    check(f"bn_fwd C={C}", out.permute(0, 3, 1, 2), y, 1e-2, gpu_out_dir)
    check(f"bn_running_mean C={C}", rmd, rm_ref, 1e-3, gpu_out_dir)
    check(f"bn_running_var C={C}", rvd, rv_ref, 1e-3, gpu_out_dir)
    sums = ops.bn_bwd_reduce(dyd, out, xd, save, relu=True)
    dres = torch.empty_like(xd)
    dx = ops.bn_bwd_apply(dyd, out, xd, save, gd, sums, count, relu=True, dres=dres)
    dgamma, dbeta = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    ops.bn_param_grad(sums, dgamma, dbeta)
    # the GPU path masks with its own bf16-rounded output; compare where the mask agrees (exclude |y| tiny)
    check(f"bn_dx C={C}", dx.permute(0, 3, 1, 2), x.grad, 3e-2, gpu_out_dir)
    check(f"bn_dres C={C}", dres.permute(0, 3, 1, 2), res_g.grad, 1e-2, gpu_out_dir)
    check(f"bn_dgamma C={C}", dgamma, gamma.grad, 2e-2, gpu_out_dir)
    check(f"bn_dbeta C={C}", dbeta, beta.grad, 2e-2, gpu_out_dir)
    # single-launch forms used by the engine: finalize inside apply; the last block of the reduction folds the slots
    rm2, rv2 = rm.to(DEV), rv.to(DEV)
    out2, save2 = ops.bn_apply_train(xd, stats, count, gd, bd, 1e-5, 0.1, 0, rm2, rv2, res=resd, relu=True)
    check(f"bn_apply_train out C={C}", out2.float(), out.float(), 1e-2, gpu_out_dir)
    check(f"bn_apply_train save C={C}", save2, save, 1e-5, gpu_out_dir)
    assert torch.allclose(rm2, rmd, rtol=1e-6, atol=1e-7) and torch.allclose(rv2, rvd, rtol=1e-6, atol=1e-7)
    dg2, db2 = torch.ones(C, device=DEV), torch.ones(C, device=DEV)
    zs = torch.zeros(ops.bn_bwd_reduce_acc_words(C), dtype=torch.float64, device=DEV)  # accumulators + ticket from a zeroed arena
    sums2 = ops.bn_bwd_reduce(dyd, out, xd, save, relu=True, dgamma=dg2, dbeta=db2, accumulate=True, acc=zs)
    assert torch.equal(sums2, sums), "the exact fp64 accumulation must be bit-reproducible"
    check(f"bn_dgamma accumulate C={C}", dg2 - 1.0, dgamma, 1e-4, gpu_out_dir)
    check(f"bn_dbeta accumulate C={C}", db2 - 1.0, dbeta, 1e-4, gpu_out_dir)
    # no residual: the ReLU mask recomputed from x (out=None) gives the same sums / dx as the mask read from the activation
    out3, save3 = ops.bn_apply_train(xd, stats, count, gd, bd, 1e-5, 0.1, 0, None, None, relu=True)
    s_read = ops.bn_bwd_reduce(dyd, out3, xd, save3, relu=True)
    s_re = ops.bn_bwd_reduce(dyd, None, xd, save3, relu=True, gamma=gd, beta=bd)
    check(f"bn_bwd_reduce remask C={C}", s_re, s_read, 1e-5, gpu_out_dir)
    dx_read = ops.bn_bwd_apply(dyd, out3, xd, save3, gd, s_read, count, relu=True)
    dx_re = ops.bn_bwd_apply(dyd, None, xd, save3, gd, s_read, count, relu=True, beta=bd)
    assert torch.equal(dx_re, dx_read)
    # ONE cooperative launch (reduce -> grid barrier -> distributed fixed-order sum -> apply) == the two-launch path
    dg3, db3, dres3 = torch.ones(C, device=DEV), torch.ones(C, device=DEV), torch.empty_like(xd)
    dx3, sums3 = ops.bn_bwd_fused(dyd, out, xd, save, gd, count, relu=True, dgamma=dg3, dbeta=db3, accumulate=True, dres=dres3)
    check(f"bn_bwd_fused sums C={C}", sums3, sums, 1e-6, gpu_out_dir)
    check(f"bn_bwd_fused dx C={C}", dx3.float(), dx.float(), 1e-2, gpu_out_dir)
    assert torch.equal(dres3, dres)
    check(f"bn_bwd_fused dgamma C={C}", dg3 - 1.0, dgamma, 1e-4, gpu_out_dir)
    check(f"bn_bwd_fused dbeta C={C}", db3 - 1.0, dbeta, 1e-4, gpu_out_dir)
    dx4, sums4 = ops.bn_bwd_fused(dyd, out, xd, save, gd, count, relu=True)
    assert torch.equal(sums4, sums3) and torch.equal(dx4, dx3), "the cooperative BN backward must be bit-reproducible"
    dx5, s5 = ops.bn_bwd_fused(dyd, None, xd, save3, gd, count, relu=True, beta=bd)  # mask recomputed from x
    check(f"bn_bwd_fused remask sums C={C}", s5, s_read, 1e-6, gpu_out_dir)
    check(f"bn_bwd_fused remask dx C={C}", dx5.float(), dx_read.float(), 1e-2, gpu_out_dir)
    dx6, _ = ops.bn_bwd_fused(dyd, out, xd, save, gd, count, relu=True, zero_sums=True)  # frozen BN: dx = gamma*istd*dz
    z = torch.zeros_like(sums)
    check(f"bn_bwd_fused frozen dx C={C}", dx6.float(), ops.bn_bwd_apply(dyd, out, xd, save, gd, z, count, relu=True).float(), 1e-2, gpu_out_dir)


def test_dropout2d_is_channelwise():
    """nn.Dropout2d (models/pspnet.py:22,68, upernet.py:22) zeroes WHOLE channels per image; nn.Dropout draws per element
    (deeplabv3_plus.py:282,318).  bn_apply's dropout epilogue does both (drop_hw = H*W selects the channel-wise draw)."""
    N, H, W, C, p = 4, 9, 7, 256, 0.3
    x = torch.ones(N, H, W, C, device=DEV, dtype=torch.bfloat16)
    ss = torch.cat([torch.ones(C), torch.zeros(C)]).to(DEV)  # identity BatchNorm
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    y2 = ops.bn_apply(x, ss, relu=True, drop_p=p, seed=123, step_ctr=ctr, drop_hw=H * W).float().reshape(N, H * W, C)
    kept = y2[:, 0, :] > 0
    assert torch.equal(y2 > 0, kept[:, None, :].expand_as(y2)), "Dropout2d mask must be constant over a channel's pixels"
    assert abs(kept.float().mean().item() - (1 - p)) < 0.06
    vals = y2[y2 > 0]
    assert torch.allclose(vals, torch.full_like(vals, 1 / (1 - p)), rtol=1e-2)
    assert not torch.equal(kept[0], kept[1]), "different images draw different channels"
    y1 = ops.bn_apply(x, ss, relu=True, drop_p=p, seed=123, step_ctr=ctr, drop_hw=0).float().reshape(N, H * W, C)
    per_pixel = (y1 > 0)
    assert not torch.equal(per_pixel, per_pixel[:, :1, :].expand_as(per_pixel)), "nn.Dropout draws per element"
    assert abs(per_pixel.float().mean().item() - (1 - p)) < 0.02


def test_bn_clamp_eps_and_eval(gpu_out_dir):
    C = 64
    g = torch.Generator().manual_seed(6)
    x = bf(torch.randn(2, C, 9, 9, generator=g) * 1e-3)  # tiny variance: clamp(var, eps) != var + eps
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    xd = to_nhwc_dev(x)
    stats = ops.bn_stats(xd)
    ss, save = ops.bn_finalize(stats, 2 * 81, gamma.to(DEV), beta.to(DEV), 1e-5, 0.1, 1, None, None)
    mean = x.mean((0, 2, 3))
    var = x.var((0, 2, 3), unbiased=False)
    istd = var.clamp(min=1e-5) ** -0.5  # sync_batchnorm/batchnorm.py:145
    check("bn_clamp_istd", save[C:], istd, 1e-3, gpu_out_dir)
    check("bn_clamp_mean", save[:C], mean, 1e-3, gpu_out_dir)
    rm, rv = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    ss = ops.bn_eval_scale_shift(gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV), 1e-5)
    out = ops.bn_apply(xd, ss, relu=False)
    ref = F.batch_norm(x, rm, rv, gamma, beta, False, 0.1, 1e-5)
    check("bn_eval", out.permute(0, 3, 1, 2), ref, 1e-2, gpu_out_dir)


def test_dropout_statistics():
    x = torch.ones(4, 32, 32, 256, device=DEV, dtype=torch.bfloat16)
    ss = torch.cat([torch.ones(256), torch.zeros(256)]).to(DEV)
    out = ops.bn_apply(x, ss, relu=True, drop_p=0.5, seed=123).float()
    keep = (out > 0).float().mean().item()
    assert abs(keep - 0.5) < 0.01
    assert abs(out.max().item() - 2.0) < 1e-6
    out2 = ops.bn_apply(x, ss, relu=True, drop_p=0.5, seed=123).float()
    assert torch.equal(out, out2)
    out3 = ops.bn_apply(x, ss, relu=True, drop_p=0.5, seed=124).float()
    assert not torch.equal(out, out3)


@pytest.mark.parametrize("C,ignore", [(19, 255), (21, 255), (150, -1)])
def test_cross_entropy(C, ignore, gpu_out_dir):
    g = torch.Generator().manual_seed(10)
    N, H, W = 2, 33, 37
    logits = (torch.randn(N, C, H, W, generator=g) * 3).requires_grad_(True)
    target = torch.randint(0, C, (N, H, W), generator=g)
    target[:, :3, :] = ignore
    target[:, :, -2:] = ignore
    loss = F.cross_entropy(logits, target, ignore_index=ignore)
    loss.backward()
    ld, td = logits.detach().to(DEV), target.to(DEV)
    l, accum = ops.loss_nchw_fwd(ld, td, ignore)
    check(f"ce_fwd C={C}", l, loss, 1e-5, gpu_out_dir)
    dl = ops.loss_nchw_bwd(ld, td, ignore, accum)
    check(f"ce_bwd C={C}", dl, logits.grad, 1e-4, gpu_out_dir)


@pytest.mark.parametrize("ac", [True, False])
@pytest.mark.parametrize("C,ignore", [(19, 255), (150, -1)])
def test_fused_upsample_ce(C, ignore, ac, gpu_out_dir):
    g = torch.Generator().manual_seed(11)
    N, Hi, Wi, Ho, Wo = 2, 17, 19, 65, 73
    lo = (torch.randn(N, C, Hi, Wi, generator=g) * 3).requires_grad_(True)
    target = torch.randint(0, C, (N, Ho, Wo), generator=g)
    target[:, :4, :] = ignore
    full = F.interpolate(lo, size=(Ho, Wo), mode="bilinear", align_corners=ac)
    loss = F.cross_entropy(full, target, ignore_index=ignore)
    loss.backward()
    lod = lo.detach().permute(0, 2, 3, 1).contiguous().to(DEV)
    l, accum, am = ops.upsample_loss_fwd(lod, target.to(DEV), ac, ignore, want_argmax=True)
    check(f"fused_ce_fwd C={C} ac={ac}", l, loss, 1e-5, gpu_out_dir)
    ref_am = full.detach().argmax(1)
    mism = (am.cpu().long() != ref_am).float().mean().item()
    assert mism < 1e-4, f"argmax mismatch fraction {mism}"
    ldx = (C + 7) // 8 * 8
    dx, dlo = ops.upsample_loss_bwd(lod, target.to(DEV), ac, ignore, accum, ldx)
    check(f"fused_ce_bwd C={C} ac={ac}", dlo.permute(0, 3, 1, 2), lo.grad, 1e-4, gpu_out_dir)
    check(f"fused_ce_bwd_bf16 C={C} ac={ac}", dx[..., :C].permute(0, 3, 1, 2), lo.grad, 1e-2, gpu_out_dir)


def test_dice_and_ce_dice_match_oracle_and_golden(gpu_out_dir):
    """DiceLoss / CE_DiceLoss (utils/losses.py:33-50,67-77) incl. the in-place target fix-up, against the oracle and the
    values captured from the reference itself (tests/golden/losses_syncbn.npz)."""
    import numpy as np
    import seg_b200
    from oracle import losses as ol
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "losses_syncbn.npz"))
    logits = torch.from_numpy(g["c7/logits"])
    target = torch.from_numpy(g["c7/target"])
    # Dice with ignored pixels present: the reference overwrites them with target.min() in place
    lg = logits.clone().cuda().requires_grad_(True)
    tg = target.clone().cuda()
    loss = seg_b200.DiceLoss(ignore_index=255)(lg, tg)
    loss.backward()
    check("dice_loss vs reference golden", loss.detach().cpu(), torch.tensor(float(g["c7/dice/loss"])), 1e-5, gpu_out_dir)
    check("dice_grad vs reference golden", lg.grad.cpu(), torch.from_numpy(g["c7/dice/grad"]), 1e-4, gpu_out_dir)
    assert (tg.cpu().numpy() == g["c7/dice/target_after"]).all(), "target mutation (losses.py:40-42) not reproduced"
    # CE + Dice on a target without ignored pixels (the only combination the reference can run on torch >= 1.5)
    t_in = torch.from_numpy(g["c7/ce_dice/target_in"])
    lg = logits.clone().cuda().requires_grad_(True)
    loss = seg_b200.CE_DiceLoss(ignore_index=255)(lg, t_in.clone().cuda())
    loss.backward()
    check("ce_dice_loss vs reference golden", loss.detach().cpu(), torch.tensor(float(g["c7/ce_dice/loss"])), 1e-5, gpu_out_dir)
    check("ce_dice_grad vs reference golden", lg.grad.cpu(), torch.from_numpy(g["c7/ce_dice/grad"]), 1e-4, gpu_out_dir)
    # a larger random case against the oracle
    gen = torch.Generator().manual_seed(12)
    lo = (torch.randn(2, 21, 37, 41, generator=gen) * 2)
    tt = torch.randint(0, 21, (2, 37, 41), generator=gen)
    tt[:, :3] = 255
    ref_l = lo.clone().requires_grad_(True)
    rl = ol.dice_loss(ref_l, tt.clone(), 1.0, 255)
    rl.backward()
    lg = lo.clone().cuda().requires_grad_(True)
    l2 = seg_b200.DiceLoss(ignore_index=255)(lg, tt.clone().cuda())
    l2.backward()
    check("dice_loss vs oracle", l2.detach().cpu(), rl.detach(), 1e-5, gpu_out_dir)
    check("dice_grad vs oracle", lg.grad.cpu(), ref_l.grad, 1e-4, gpu_out_dir)


@pytest.mark.parametrize("shape", [(2, 33, 35, 64, 1, 1), (2, 33, 33, 728, 1, 2), (1, 34, 30, 128, 2, 1), (2, 17, 17, 1536, 1, 4)],
                         ids=lambda s: "x".join(map(str, s)))
def test_depthwise_conv(shape, gpu_out_dir):
    """SeparableConv2d.conv1 (deeplabv3_plus.py:77-78): groups == channels, 3x3, 'same' padding = dilation."""
    N, H, W, C, stride, dil = shape
    g = torch.Generator().manual_seed(13)
    x = bf(torch.randn(N, C, H, W, generator=g)).requires_grad_(True)
    w = (torch.randn(C, 1, 3, 3, generator=g) * 0.4).requires_grad_(True)
    y = F.conv2d(x, w, None, stride, dil, dil, groups=C)
    dy = bf(torch.randn(y.shape, generator=g))
    y.backward(dy)
    w9 = ops.dw_pack_weight(w.detach().to(DEV))
    stats = ops.new_stats(C, DEV)
    yd = ops.dwconv_fwd(to_nhwc_dev(x.detach()), w9, stride, dil, dil, stats=stats)
    torch.cuda.synchronize()
    check(f"dwconv_fwd {shape}", yd.permute(0, 3, 1, 2), y, 1e-2, gpu_out_dir)
    yr = y.detach()
    check(f"dwconv_stats {shape}", stats, torch.cat([yr.sum((0, 2, 3)), (yr * yr).sum((0, 2, 3))]), 2e-3, gpu_out_dir)
    dx = ops.dwconv_bwd_data(to_nhwc_dev(dy), w9, (N, H, W, C), stride, dil, dil)
    check(f"dwconv_bwd_data {shape}", dx.permute(0, 3, 1, 2), x.grad, 1e-2, gpu_out_dir)
    dx2 = ops.dwconv_bwd_data(to_nhwc_dev(dy), w9, (N, H, W, C), stride, dil, dil, out=dx.clone(), beta=1.0)
    check(f"dwconv_bwd_data_beta1 {shape}", dx2.permute(0, 3, 1, 2), 2 * x.grad, 1.5e-2, gpu_out_dir)
    g9 = ops.dwconv_bwd_weight(to_nhwc_dev(dy), to_nhwc_dev(x.detach()), stride, dil, dil)
    gw = torch.empty(C, 1, 3, 3, device=DEV)
    ops.dw_unpack_wgrad(g9, gw)
    check(f"dwconv_bwd_weight {shape}", gw, w.grad, 2e-3, gpu_out_dir)


def test_lovasz_softmax_matches_reference_golden_and_oracle(gpu_out_dir):
    """LovaszSoftmax (utils/losses.py:79-89) — device radix-sort implementation against the values captured from the
    reference itself (C=7 ignore 255; C=150 ignore -1) and against the oracle on a larger random case."""
    import numpy as np
    import seg_b200
    from oracle import losses as ol
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "losses_syncbn.npz"))
    for tag, ignore in (("c7", 255), ("c150", -1)):
        lg = torch.from_numpy(g[f"{tag}/logits"]).cuda().requires_grad_(True)
        tg = torch.from_numpy(g[f"{tag}/target"]).cuda()
        loss = seg_b200.LovaszSoftmax(ignore_index=ignore)(lg, tg)
        loss.backward()
        check(f"lovasz_loss {tag} vs reference golden", loss.detach().cpu(), torch.tensor(float(g[f"{tag}/lovasz/loss"])), 1e-5, gpu_out_dir)
        check(f"lovasz_grad {tag} vs reference golden", lg.grad.cpu(), torch.from_numpy(g[f"{tag}/lovasz/grad"]), 1e-4, gpu_out_dir)
    gen = torch.Generator().manual_seed(15)
    lo = torch.randn(3, 21, 61, 67, generator=gen) * 2
    tt = torch.randint(0, 19, (3, 61, 67), generator=gen)  # classes 19, 20 absent
    tt[:, :5] = 255
    ref_l = lo.clone().requires_grad_(True)
    rl = ol.lovasz_softmax(ref_l, tt, 255)
    rl.backward()
    lg = lo.clone().cuda().requires_grad_(True)
    l2 = seg_b200.LovaszSoftmax(ignore_index=255)(lg, tt.cuda()) * 2.0
    l2.backward()
    check("lovasz_loss vs oracle", l2.detach().cpu() / 2, rl.detach(), 1e-5, gpu_out_dir)
    check("lovasz_grad vs oracle (x2 upstream)", lg.grad.cpu() / 2, ref_l.grad, 1e-4, gpu_out_dir)
    # only void pixels: zero loss, zero gradient (lovasz_losses.py:178-180)
    lg = lo.clone().cuda().requires_grad_(True)
    l3 = seg_b200.LovaszSoftmax(ignore_index=255)(lg, torch.full((3, 61, 67), 255, dtype=torch.long, device="cuda"))
    l3.backward()
    assert float(l3) == 0.0 and float(lg.grad.abs().max()) == 0.0


def test_eval_metrics_bit_exact_vs_reference_golden_and_oracle(gpu_out_dir):
    """seg_b200.eval_metrics (one device pass, utils/metrics.py:59-67) — integer counters, bit-exact."""
    import numpy as np
    import seg_b200
    from oracle import metrics as om
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz"))
    for tag, K in (("c7", 7), ("c19", 19), ("c150", 150)):
        out = seg_b200.eval_metrics(torch.from_numpy(g[f"{tag}/logits"]).cuda(), torch.from_numpy(g[f"{tag}/target"]).cuda(), K)
        assert int(out[0]) == int(g[f"{tag}/correct"]) and int(out[1]) == int(g[f"{tag}/labeled"]), tag
        assert np.array_equal(out[2], g[f"{tag}/inter"]) and np.array_equal(out[3], g[f"{tag}/union"]), tag
    gen = torch.Generator().manual_seed(77)
    lo = torch.randn(4, 21, 129, 131, generator=gen)
    tt = torch.randint(0, 21, (4, 129, 131), generator=gen)
    tt[:, :7] = 255
    lo.scatter_add_(1, tt.clamp(0, 20).unsqueeze(1), (torch.rand(4, 1, 129, 131, generator=gen) < 0.5).float() * 5)
    ref = om.eval_metrics(lo.numpy(), tt.numpy(), 21)
    out = seg_b200.eval_metrics(lo.cuda(), tt.cuda(), 21)
    for a, b in zip(out, ref):
        assert np.array_equal(np.asarray(a), np.asarray(b))
