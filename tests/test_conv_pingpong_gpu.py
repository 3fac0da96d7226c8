"""The persistent ping-pong convolution kernel (fprop / dgrad) on the large C3 shapes, where a CTA runs several tiles and the
two consumer warpgroups alternate: parity against ATen on the CPU, bit-reproducible statistics, and the SyncBN exchange
counting one ticket per CTA of the persistent grid."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import comm, ops
    from seg_b200.lib import IMPL_TC

DEV = "cuda"

# (N, H, W, C, K, ksize, stride, pad, dil)
SHAPES = [
    (16, 33, 33, 256, 256, 3, 1, 1, 1),   # 137 row tiles x 2 column blocks = 274 tiles: some CTAs run three
    (16, 33, 33, 1024, 256, 1, 1, 0, 1),  # l3.conv1: short k loop (16 k-blocks), 1x1 through the 2-D map
]


def bf(t):
    return t.to(torch.bfloat16).to(torch.float32)


def rel_err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)


def inputs(shape, seed=0):
    N, H, W, C, K, ks, stride, pad, dil = shape
    g = torch.Generator().manual_seed(seed)
    x = bf(torch.randn(N, C, H, W, generator=g))
    w = bf(torch.randn(K, C, ks, ks, generator=g) / (C * ks * ks) ** 0.5)
    return x, w


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().to(DEV, torch.bfloat16)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_fprop_large(shape):
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = inputs(shape)
    ref = F.conv2d(x, w, None, stride, pad, dil)
    ref_s = torch.cat([ref.sum((0, 2, 3)), (ref * ref).sum((0, 2, 3))])
    wp = ops.pack_weight(w.to(DEV))
    xd = nhwc(x)
    stats = ops.new_stats(K, DEV)
    y = ops.conv2d_fwd(xd, wp, K, ks, ks, stride, pad, dil, out_dtype=torch.float32, stats=stats, impl=IMPL_TC)
    torch.cuda.synchronize()
    assert rel_err(y.permute(0, 3, 1, 2), ref) <= 2e-3
    assert rel_err(stats, ref_s) <= 2e-3
    bias = torch.randn(K, device=DEV)
    stats_b = ops.new_stats(K, DEV)
    yb = ops.conv2d_fwd(xd, wp, K, ks, ks, stride, pad, dil, bias=bias, stats=stats_b, impl=IMPL_TC)
    torch.cuda.synchronize()
    assert rel_err(yb.permute(0, 3, 1, 2), ref + bias.cpu().view(1, K, 1, 1)) <= 1e-2
    yd = yb.double().reshape(-1, K)
    exact = torch.cat([yd.sum(0), (yd * yd).sum(0)])
    assert rel_err(stats_b, exact) <= 2e-5
    for _ in range(3):
        again = ops.new_stats(K, DEV)
        y2 = ops.conv2d_fwd(xd, wp, K, ks, ks, stride, pad, dil, bias=bias, stats=again, impl=IMPL_TC)
        assert torch.equal(again, stats_b), "BatchNorm statistics are not bit-reproducible"
        assert torch.equal(y2, yb)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_dgrad_large(shape):
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = inputs(shape)
    x.requires_grad_(True)
    y = F.conv2d(x, w, None, stride, pad, dil)
    dy = bf(torch.randn(y.shape, generator=torch.Generator().manual_seed(1)))
    y.backward(dy)
    wp = ops.pack_weight(w.to(DEV))
    dx = ops.conv2d_dgrad(nhwc(dy), wp, (N, H, W, C), ks, ks, stride, pad, dil, impl=IMPL_TC)
    torch.cuda.synchronize()
    assert rel_err(dx.permute(0, 3, 1, 2), x.grad) <= 1e-2
    dx2 = ops.conv2d_dgrad(nhwc(dy), wp, (N, H, W, C), ks, ks, stride, pad, dil, out=dx.clone(), beta=1.0, impl=IMPL_TC)
    torch.cuda.synchronize()
    assert rel_err(dx2.permute(0, 3, 1, 2), 2 * x.grad) <= 1.5e-2


def test_syncbn_statistics_on_the_persistent_grid():
    """fprop with statistics and the SyncBN exchange on a one-rank loopback buffer, 274 tiles on a grid of one CTA per SM:
    the ticket counts exactly one arrival per CTA, the last one pushes the finished totals, and with one rank they are the
    plain statistics bit for bit — twice in a row, so the exchange's slot alternation and sequence number are exercised."""
    shape = SHAPES[0]
    N, H, W, C, K, ks, stride, pad, dil = shape
    x, w = inputs(shape)
    wp = ops.pack_weight(w.to(DEV))
    xd = nhwc(x)
    plain = ops.new_stats(K, DEV)
    y0 = ops.conv2d_fwd(xd, wp, K, ks, ks, stride, pad, dil, stats=plain, impl=IMPL_TC)
    g = comm.LocalLoopbackGroup(n_max=8192)
    tiles = -(-N * H * W // 128) * (K // 128)
    grid = min(tiles, torch.cuda.get_device_properties(0).multi_processor_count)
    for _ in range(2):
        ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
        stats = ops.new_stats(K, DEV)
        y = ops.conv2d_fwd(xd, wp, K, ks, ks, stride, pad, dil, stats=stats, impl=IMPL_TC, sync=g, sync_ticket=ticket)
        torch.cuda.synchronize()
        assert ticket.item() == grid, (ticket.item(), grid, tiles)
        assert torch.equal(stats, plain)
        assert torch.equal(y, y0)
