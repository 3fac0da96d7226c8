"""The ReLU bit mask of the BatchNorm training path: bn_apply_train(mask=) writes one byte per (row, 8-channel group),
bit j = (stored bf16 activation > 0), and the three backward entry points given that mask must reproduce, bit for bit,
what they compute when they read the activation itself (sums, dgamma / dbeta, dx, dres).  Cases cover channel counts
whose groups do not divide the block's 256 threads, the activation as a channel slice of a wider buffer, row counts
that are not a multiple of a block's row lanes, residual inputs with beta_res 0 and 1, nn.Dropout and nn.Dropout2d,
frozen BN, accumulating parameter gradients, and maps on both sides of the engine's one-launch backward threshold."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import ops
    from seg_b200.engine import FUSED_BWD_MAX_BYTES

DEV = "cuda"
GUARD = 64     # sentinel bytes on each side of the mask
SENTINEL = 0xA5


def _bf(shape, g, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=g) * scale + shift).to(torch.bfloat16).to(DEV)


def _guarded_mask(M, C):
    buf = torch.full((M * (C // 8) + 2 * GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
    return buf, buf[GUARD:GUARD + M * (C // 8)].view(M, C // 8)


def _packed(a):
    """(a > 0) packed as the kernel does: uint8 [M][C/8], bit j = channel 8g + j."""
    C = a.shape[-1]
    bits = (a.float() > 0).reshape(-1, C // 8, 8).to(torch.int32)
    return (bits << torch.arange(8, dtype=torch.int32, device=a.device)).sum(-1).to(torch.uint8)


def _forward(N, H, W, C, g, sliced, res, drop_p, drop2d):
    """x, the activation A (a channel slice of a wider buffer when sliced), save, the guarded mask."""
    x = _bf((N, H, W, C), g, 1.5, 0.2)
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.5).to(DEV)
    r = _bf((N, H, W, C), g) if res else None
    stats = ops.bn_stats(x)
    M = N * H * W
    if sliced:
        wide = torch.zeros((N, H, W, C + 24), dtype=torch.bfloat16, device=DEV)
        out = wide[..., 8:8 + C]
    else:
        out = torch.empty((N, H, W, C), dtype=torch.bfloat16, device=DEV)
    buf, mask = _guarded_mask(M, C)
    kw = dict(res=r, relu=True, drop_p=drop_p, seed=1234, drop_hw=H * W if drop2d else 0)
    a, save = ops.bn_apply_train(x, stats, M, gamma, beta, 1e-5, 0.1, 0, None, None, out=out, mask=mask, **kw)
    a_ref, save_ref = ops.bn_apply_train(x, stats, M, gamma, beta, 1e-5, 0.1, 0, None, None, **kw)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), a_ref.view(torch.int16)), "writing the mask changed the activation"
    assert torch.equal(save, save_ref)
    assert torch.equal(mask, _packed(a)), "mask bytes differ from (A > 0) packed"
    assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all(), "bytes outside the mask were written"
    return x, a, save, gamma, beta, mask, buf


def _same(name, got, ref):
    if got.dtype == torch.bfloat16:
        got, ref = got.view(torch.int16), ref.view(torch.int16)
    assert torch.equal(got, ref), f"{name}: the mask path is not bit-identical to the activation path"


# (C, sliced, res, drop_p, drop2d, beta_res, accumulate)
CASES = [
    (48, False, False, 0.0, False, 0.0, False),
    (48, True, True, 0.0, False, 1.0, True),
    (304, True, True, 0.0, False, 0.0, False),
    (304, False, False, 0.1, False, 0.0, True),
    (1024, True, True, 0.0, False, 1.0, False),
    (1024, False, False, 0.2, True, 0.0, False),
    (2048, False, True, 0.0, False, 1.0, True),
    (2048, True, False, 0.1, True, 0.0, False),
]


@pytest.mark.parametrize("C,sliced,res,drop_p,drop2d,beta_res,accumulate", CASES)
def test_mask_matches_activation(C, sliced, res, drop_p, drop2d, beta_res, accumulate):
    N, H, W = 3, 13, 11  # M = 429: not a multiple of the 42 / 6 / 2 row lanes of C = 48 / 304 / 1024
    g = torch.Generator().manual_seed(C * 7 + int(sliced) * 3 + int(res))
    x, a, save, gamma, beta, mask, buf = _forward(N, H, W, C, g, sliced, res, drop_p, drop2d)
    M = N * H * W
    dout = _bf((N, H, W, C), g)
    dres0 = _bf((N, H, W, C), g) if res else None
    pg0 = torch.randn(2, C, generator=g).to(DEV)

    def run(kind, use_mask, zero_sums=False):
        src = dict(mask=mask) if use_mask else {}
        out = None if use_mask else a
        pg = pg0.clone()
        dres = dres0.clone() if res else None
        if kind == "two":
            sums = ops.bn_bwd_reduce(dout, out, x, save, relu=True, drop_p=drop_p, dgamma=pg[1], dbeta=pg[0],
                                     accumulate=accumulate, **src)
            dx = ops.bn_bwd_apply(dout, out, x, save, gamma, sums, M, relu=True, drop_p=drop_p, dres=dres,
                                  beta_res=beta_res, **src)
        else:
            dx, sums = ops.bn_bwd_fused(dout, out, x, save, gamma, M, relu=True, drop_p=drop_p, dgamma=pg[1], dbeta=pg[0],
                                        accumulate=accumulate, dres=dres, beta_res=beta_res, zero_sums=zero_sums, **src)
        torch.cuda.synchronize()
        return sums, pg, dx, dres

    for kind, zero_sums in (("two", False), ("fused", False), ("fused", True)):
        ref, got = run(kind, False, zero_sums), run(kind, True, zero_sums)
        for name, r, o in zip(("sums", "dgamma/dbeta", "dx", "dres"), ref, got):
            if r is not None:
                _same(f"{kind} zero_sums={zero_sums} {name} C={C}", o, r)
    assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all()


@pytest.mark.parametrize("N,H,W,C,res", [(16, 33, 33, 1024, True), (16, 33, 33, 256, False)])
def test_mask_on_both_sides_of_the_one_launch_threshold(N, H, W, C, res):
    """A 35.7 MB residual map (the engine's two-launch backward) and an 8.9 MB one (its one-launch backward)."""
    M = N * H * W
    assert (M * C * 2 > FUSED_BWD_MAX_BYTES) == res
    g = torch.Generator().manual_seed(C)
    x, a, save, gamma, beta, mask, _ = _forward(N, H, W, C, g, False, res, 0.0, False)
    dout = _bf((N, H, W, C), g)
    if res:
        s_ref = ops.bn_bwd_reduce(dout, a, x, save, relu=True)
        s_got = ops.bn_bwd_reduce(dout, None, x, save, relu=True, mask=mask)
        _same("sums", s_got, s_ref)
        dres_ref, dres_got = torch.empty_like(x), torch.empty_like(x)
        _same("dx", ops.bn_bwd_apply(dout, None, x, save, gamma, s_ref, M, relu=True, dres=dres_got, mask=mask),
              ops.bn_bwd_apply(dout, a, x, save, gamma, s_ref, M, relu=True, dres=dres_ref))
        _same("dres", dres_got, dres_ref)
    else:
        dx_ref, s_ref = ops.bn_bwd_fused(dout, a, x, save, gamma, M, relu=True)
        dx_got, s_got = ops.bn_bwd_fused(dout, None, x, save, gamma, M, relu=True, mask=mask)
        _same("sums", s_got, s_ref)
        _same("dx", dx_got, dx_ref)
