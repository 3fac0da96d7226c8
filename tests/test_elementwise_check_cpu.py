"""Self-tests of the streaming-kernel conformance checker (tests/elementwise_check.py), CPU only.

Acceptance: the checker passes correct results computed differently — its own float64 reference rounded to the output
type, and ATen's float32 CPU results (F.batch_norm and its autograd, max / adaptive-average pooling, F.interpolate and
their gradients) — at every shape class of the GPU sweep, scaled down where float64 time requires.  Sensitivity: it
rejects each planted defect a broken kernel would produce, and names its coordinates.  The planted defects stand in for
broken kernels, which are never run."""
import pytest
import torch
import torch.nn.functional as F

import elementwise_check as ec

SMS = 132  # H100 SXM; the grid mirrors only change the chain lengths the sums are charged
EPS, MOM = 1e-5, 0.1


def to_bf16(t):
    return t.to(torch.bfloat16).double()


def bn_operands(M, C, seed, res=True, scale=1.0):
    """x with per-channel magnitudes and offsets, residual, gamma, beta, dout (all bf16 / fp32 exact)."""
    g = torch.Generator().manual_seed(seed)
    cs = ec.channel_scales(C, seed + 1)
    x = to_bf16((torch.randn(M, C, generator=g, dtype=torch.float64) + 0.5) * cs * scale)
    r = to_bf16(torch.randn(M, C, generator=g, dtype=torch.float64)) if res else None
    gamma = (torch.rand(C, generator=g) + 0.5)
    beta = torch.randn(C, generator=g) * 0.3
    dout = to_bf16(torch.randn(M, C, generator=g, dtype=torch.float64))
    return x, r, gamma, beta, dout


def aten_bn_fwd(x, r, gamma, beta):
    """ATen float32 F.batch_norm (+res) on [M, C] and its running statistics from (0, 1)."""
    C = x.shape[1]
    rm, rv = torch.zeros(C), torch.ones(C)
    xf = x.float().t().reshape(1, C, -1, 1).requires_grad_(True)
    y = F.batch_norm(xf, rm, rv, gamma, beta, True, MOM, EPS)
    pre = y.reshape(C, -1).t()
    if r is not None:
        pre = pre + r.float()
    return pre, rm, rv


# (M, C): the channel classes of the sweep (idle row lanes at 304 / 728 / 1536, two slabs at 2064 / 4096) and the row
# classes (M = 1, M < rows_par, M = 8 image-pool BN), scaled down
BN_SHAPES = [(1, 64), (5, 64), (100, 8), (162, 48), (198, 256), (8, 256), (99, 304), (40, 728), (33, 1536), (15, 2048),
             (9, 2064), (7, 4096), (8450, 8)]


@pytest.mark.parametrize("M,C", BN_SHAPES, ids=[f"{m}x{c}" for m, c in BN_SHAPES])
def test_accepts_bn_forward(M, C):
    x, r, gamma, beta, _ = bn_operands(M, C, 1)
    stats = ec.exact_stats(x)
    st = ec.BnStats(stats, M, EPS, 0)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    assert ec.check_apply("ref", to_bf16(pre.clamp_min(0)), pre, acc) <= 1
    assert ec.check_apply("ref no relu", to_bf16(pre), pre, acc, relu=False) <= 1
    if M > 1:  # ATen refuses one value per channel in training mode
        a_pre, rm, rv = aten_bn_fwd(x, r, gamma, beta)
        assert ec.check_apply("aten", to_bf16(a_pre.double().clamp_min(0)), pre, acc) <= 1
        assert ec.check_running("aten", rm, rv, torch.zeros(C), torch.ones(C), st, MOM) <= 1
    assert ec.check_save("fp32 ref", torch.cat([st.mean, st.istd]).float(), st) <= 1
    ss = torch.cat([gamma.double() * st.istd, beta.double() - st.mean * gamma.double() * st.istd]).float()
    assert ec.check_scale_shift("fp32 ref", ss, gamma, beta, st.mean, st.istd) <= 1
    # bn_apply with given scale / shift (eval mode)
    pre2, acc2 = ec.bn_ss_ref(x, ss, r)
    aten2 = (x.float() * ss[:C] + ss[C:] + r.float()).double()
    assert ec.check_apply("ss aten", to_bf16(aten2.clamp_min(0)), pre2, acc2) <= 1


def test_accepts_bn_clamp_eps_and_stats():
    M, C = 162, 64
    x, r, gamma, beta, _ = bn_operands(M, C, 2, scale=1e-3)  # var < eps: clamp(var, eps) != var + eps
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 1)
    assert (st.var < EPS).any()
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    var_f = x.float().var(0, unbiased=False)
    aten = ((x.float() - x.float().mean(0)) * var_f.clamp_min(EPS).rsqrt() * gamma + beta + r.float()).double()
    assert ec.check_apply("clamp aten", to_bf16(aten.clamp_min(0)), pre, acc) <= 1
    # bn_stats: fp32 sums over the chain of the sweep's largest bn_stats case
    f32 = torch.cat([x.float().sum(0), (x.float() ** 2).sum(0)]).double()
    assert ec.check_stats("f32 sum", f32, x, ec.stat_chain_simt(M, C, SMS)) <= 1


@pytest.mark.parametrize("p,units", [(0.1, False), (0.5, False), (0.5, True)], ids=["p0.1", "p0.5", "p0.5_2d"])
def test_accepts_dropout(p, units):
    N, HW, C = 4, 63, 256
    M = N * HW
    x, r, gamma, beta, _ = bn_operands(M, C, 3)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 0)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    g = torch.Generator().manual_seed(4)
    if units:
        uid = (torch.arange(M).view(M, 1) // HW) * C + torch.arange(C).view(1, C)
        keepm = (torch.rand(N * C, generator=g) >= p)[uid]
    else:
        uid = None
        keepm = torch.rand(M, C, generator=g) >= p
    got = to_bf16(torch.where(keepm, pre.float().clamp_min(0) * ec.fp32_keep(p), torch.zeros(M, C)))
    usage, frac, n = ec.check_dropout("emulated", got, pre, acc, p, units=uid)
    assert usage <= 1 and n > 0


def bwd_case(M, C, seed, keep_p=0.0, res=True):
    """Operands of a backward case: the stored activation is the forward reference (+ dropout from a torch RNG)."""
    x, r, gamma, beta, dout = bn_operands(M, C, seed, res)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 0)
    save = torch.cat([st.mean, st.istd]).float()
    pre, _ = ec.bn_train_ref(x, st, gamma, beta, r)
    out = to_bf16(pre.clamp_min(0))
    if keep_p:
        out = out * (torch.rand(M, C, generator=torch.Generator().manual_seed(seed + 9)) >= keep_p)
    return x, r, gamma, beta, dout, save, out


@pytest.mark.parametrize("M,C", BN_SHAPES, ids=[f"{m}x{c}" for m, c in BN_SHAPES])
def test_accepts_bn_backward(M, C):
    x, r, gamma, beta, dout, save, out = bwd_case(M, C, 5)
    mask = out > 0
    for chain, name in ((ec.bwd_chain_two_launch(M, C, SMS), "two-launch"), (ec.bwd_chain_fused(M, C, SMS), "fused")):
        ref = ec.BwdRef(dout, x, save, gamma, mask=mask, chain=chain)
        sb = ref.sums_bound()
        assert ec.check(name, "sums", sb.ref.float(), sb) <= 1
        assert ec.check(name, "dx", to_bf16(ref.dx_bound().ref), ref.dx_bound()) <= 1
        assert ec.check(name, "dx frozen", to_bf16(ref.dx_bound(True).ref), ref.dx_bound(True)) <= 1
        old = to_bf16(torch.randn(M, C, generator=torch.Generator().manual_seed(6), dtype=torch.float64))
        db = ref.dres_bound(1.0, old)
        assert ec.check(name, "dres", to_bf16(db.ref), db) <= 1
        pb = ref.param_bound(1, old=torch.ones(C))
        assert ec.check(name, "dgamma", pb.ref.float(), pb) <= 1
    # ATen's float32 autograd through F.batch_norm (its own istd and summation order); the mask is the stored output's
    ref = ec.BwdRef(dout, x, save, gamma, mask=mask, chain=ec.bwd_chain_two_launch(M, C, SMS))
    if M > 1:
        xf = x.float().t().reshape(1, C, M, 1).requires_grad_(True)
        gf, bf_ = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        y = F.batch_norm(xf, None, None, gf, bf_, True, MOM, EPS)
        dz = (dout * mask).float().t().reshape(1, C, M, 1)
        y.backward(dz)
        dx_aten = xf.grad.reshape(C, M).t().double()
        assert ec.check("aten", "dx", to_bf16(dx_aten), ref.dx_bound()) <= 1
        assert ec.check("aten", "dbeta", bf_.grad, ref.param_bound(0)) <= 1
        assert ec.check("aten", "dgamma", gf.grad, ref.param_bound(1)) <= 1


def test_accepts_bn_backward_dropout_and_remask():
    M, C, p = 198, 256, 0.1
    x, r, gamma, beta, dout, save, out = bwd_case(M, C, 7, keep_p=p)
    keep = ec.fp32_keep(p)
    ref = ec.BwdRef(dout, x, save, gamma, mask=out > 0, keep=keep, chain=ec.bwd_chain_fused(M, C, SMS))
    dz = (dout.float() * (out > 0).float() * keep).double()  # the kernel's fp32 dz'
    xhat = ((x.float() - save[:C]) * save[C:]).double()
    s0, s1 = dz.sum(0), (dz * xhat).sum(0)
    A = gamma.double() * save[C:].double()
    dx = A * (dz - s0 / M - xhat * s1 / M)
    assert ec.check("emulated", "sums", torch.cat([s0, s1]).float(), ref.sums_bound()) <= 1
    assert ec.check("emulated", "dx", to_bf16(dx), ref.dx_bound()) <= 1
    # remask: no residual, the mask is the sign of x sc + sh with the kernels' fp32 coefficients
    x, _, gamma, beta, dout, save, out = bwd_case(M, C, 8, res=False)
    mask, amb = ec.remask(x, gamma, beta, save[:C], save[C:])
    assert int(amb.sum()) <= 8
    ref = ec.BwdRef(dout, x, save, gamma, mask=mask, chain=ec.bwd_chain_fused(M, C, SMS), ambiguous=amb)
    assert ec.check("remask", "dx", to_bf16(ref.dx_bound().ref), ref.dx_bound(), alt=ref.dx_alt()) <= 1
    # the stored activation's mask agrees with the recomputed one away from zero
    assert bool(((out > 0) == mask)[~amb].all())


MAXPOOL_SHAPES = [(2, 33, 35, 64), (1, 1, 1, 8), (1, 2, 2, 16), (2, 1, 6, 8), (1, 8, 7, 24), (1, 65, 64, 8)]


@pytest.mark.parametrize("shape", MAXPOOL_SHAPES, ids=["x".join(map(str, s)) for s in MAXPOOL_SHAPES])
def test_accepts_maxpool(shape):
    N, H, W, C = shape
    x = to_bf16(torch.randn(N, H, W, C, generator=torch.Generator().manual_seed(9), dtype=torch.float64)).clamp_min(0)
    xf = ec.nchw(x).float().requires_grad_(True)
    y, ind = F.max_pool2d(xf, 3, 2, 1, return_indices=True)
    ry, rtap = ec.maxpool_ref(x)
    ind = ec.nhwc(ind)  # ATen's flat h * W + w of the first maximum -> the kernel's tap code r * 3 + s
    tap = (ind // W - (2 * torch.arange(y.shape[2]).view(1, -1, 1, 1) - 1)) * 3 + \
        (ind % W - (2 * torch.arange(y.shape[3]).view(1, 1, -1, 1) - 1))
    ec.check_maxpool_fwd("aten f32", ec.nhwc(y), tap, x)
    dy = to_bf16(torch.randn(y.shape, generator=torch.Generator().manual_seed(10), dtype=torch.float64))
    y.backward(dy.float())
    b = ec.maxpool_bwd_bound(ec.nhwc(dy), rtap, x.shape)
    assert ec.check("aten f32", "maxpool dx", to_bf16(ec.nhwc(xf.grad).double()), b) <= 1
    assert ec.check("ref", "maxpool dx", to_bf16(b.ref), b) <= 1


AVG_CASES = [(65, 1), (65, 6), (60, 2), (60, 3), (33, 6), (17, 3), (7, 6), (1, 1), (15, 6)]


@pytest.mark.parametrize("H,bins", AVG_CASES, ids=[f"{h}b{b}" for h, b in AVG_CASES])
def test_accepts_adaptive_avgpool(H, bins):
    N, W, C = 2, H + 2 if H > 1 else 1, 16
    x = to_bf16(torch.randn(N, H, W, C, generator=torch.Generator().manual_seed(11), dtype=torch.float64))
    xf = ec.nchw(x).float().requires_grad_(True)
    y = F.adaptive_avg_pool2d(xf, bins)
    b = ec.avgpool_fwd_bound(x, bins)
    assert ec.check("aten f32", "avgpool y", to_bf16(ec.nhwc(y).double()), b) <= 1
    assert ec.check("ref", "avgpool y", to_bf16(b.ref), b) <= 1
    dy = to_bf16(torch.randn(y.shape, generator=torch.Generator().manual_seed(12), dtype=torch.float64))
    y.backward(dy.float())
    old = to_bf16(torch.randn(x.shape, generator=torch.Generator().manual_seed(13), dtype=torch.float64))
    bb = ec.avgpool_bwd_bound(ec.nhwc(dy), x.shape, bins, beta=1.0, old=old)
    assert ec.check("aten f32", "avgpool dx", to_bf16(ec.nhwc(xf.grad).double() + old), bb) <= 1
    assert ec.check("ref", "avgpool dx", to_bf16(bb.ref), bb) <= 1


# (Hi, Wi, Ho, Wo, align_corners): the engine's pairs, the MAXN boundary, non-integer ratios, downsampling, identity
BIL_CASES = [(1, 1, 33, 33, True), (1, 1, 65, 65, True), (2, 2, 60, 60, True), (3, 3, 60, 60, True),
             (6, 6, 60, 60, True), (33, 33, 129, 129, True), (33, 33, 129, 129, False), (9, 7, 31, 29, False),
             (65, 65, 33, 33, True), (65, 65, 33, 33, False), (13, 13, 13, 13, False), (3, 5, 26, 27, True)]


@pytest.mark.parametrize("case", BIL_CASES, ids=[f"{a}x{b}to{c}x{d}{'ac' if e else ''}" for a, b, c, d, e in BIL_CASES])
def test_accepts_bilinear(case):
    Hi, Wi, Ho, Wo, ac = case
    N, C = 1, 8
    x = to_bf16(torch.randn(N, Hi, Wi, C, generator=torch.Generator().manual_seed(14), dtype=torch.float64))
    xf = ec.nchw(x).float().requires_grad_(True)
    y = F.interpolate(xf, size=(Ho, Wo), mode="bilinear", align_corners=ac)
    b = ec.bilinear_fwd_bound(x, Ho, Wo, ac)
    bf32 = ec.bilinear_fwd_bound(x, Ho, Wo, ac, out_bf16=False)
    # the float32-index matrix reproduces F.interpolate on float32 inputs
    assert ec.check("aten f32", "bilinear y fp32", ec.nhwc(y).double(), bf32) <= 1
    assert ec.check("aten f32", "bilinear y", to_bf16(ec.nhwc(y).double()), b) <= 1
    dy = to_bf16(torch.randn(y.shape, generator=torch.Generator().manual_seed(15), dtype=torch.float64))
    y.backward(dy.float())
    old = to_bf16(torch.randn(x.shape, generator=torch.Generator().manual_seed(16), dtype=torch.float64))
    for beta in (0.0, 1.0):
        bb = ec.bilinear_bwd_bound(ec.nhwc(dy), Hi, Wi, ac, beta=beta, old=old)
        assert ec.check("aten f32", "bilinear dx", to_bf16(ec.nhwc(xf.grad).double() + beta * old), bb) <= 1
        assert ec.check("ref", "bilinear dx", to_bf16(bb.ref), bb) <= 1


def test_outputs_per_input_matches_the_engine_pairs():
    assert ec.outputs_per_input(1, 33, True) == 33 > ec.MAXN   # ASPP image pool: fallback loop
    assert ec.outputs_per_input(2, 60, True) > ec.MAXN           # PSP bins 2 and 3: fallback loop
    assert ec.outputs_per_input(3, 60, True) > ec.MAXN
    assert ec.outputs_per_input(6, 60, True) <= ec.MAXN          # PSP bin 6: just under
    assert ec.outputs_per_input(33, 129, False) <= ec.MAXN


def test_accepts_relu_and_axpby():
    g = torch.Generator().manual_seed(17)
    v = to_bf16(torch.randn(50, 24, generator=g, dtype=torch.float64))
    y = to_bf16(torch.randn(50, 24, generator=g, dtype=torch.float64)).clamp_min(0)
    old = to_bf16(torch.randn(50, 24, generator=g, dtype=torch.float64))
    for beta in (0.0, 1.0, 0.5):
        b = ec.relu_bwd_bound(v, y, beta, old)
        got = to_bf16(torch.where(y > 0, v, torch.zeros_like(v)).float() + beta * old.float())
        assert ec.check("f32", "relu dx", got, b) <= 1
        b = ec.axpby_bound(v, beta, old)
        assert ec.check("f32", "axpby", to_bf16(v.float() + beta * old.float()), b) <= 1


# ------------------------------------------------------------------------------------------------ sensitivity
def rejects(fn, *coords):
    with pytest.raises(AssertionError) as ei:
        fn()
    msg = str(ei.value)
    for c in coords:
        assert c in msg, f"{c!r} not in the failure message:\n{msg}"
    return msg


def test_rejects_dropped_row_in_bn_sums_at_the_longest_chain():
    """bn_stats and the backward sums at the longest chain of the GPU sweep (which asserts it stays within it)."""
    M, C, c = 4 * 129 * 129, 8, 5
    x = to_bf16(torch.randn(M, C, generator=torch.Generator().manual_seed(18), dtype=torch.float64))
    s = ec.exact_stats(x)
    row = x[:, c].abs().argmax()
    bad = s.clone()
    bad[c] -= x[row, c]
    rejects(lambda: ec.check_stats("stats row", bad, x, ec.LONGEST_SUM_CHAIN), f"(sum, c={c})")
    bad = s.clone()
    bad[C + c] -= x[row, c] ** 2
    rejects(lambda: ec.check_stats("stats row", bad, x, ec.LONGEST_SUM_CHAIN), f"(sum of squares, c={c})")
    save = torch.cat([x.mean(0), x.var(0, unbiased=False).add(EPS).rsqrt()]).float()
    dout = to_bf16(torch.randn(M, C, generator=torch.Generator().manual_seed(19), dtype=torch.float64))
    ref = ec.BwdRef(dout, x, save, torch.ones(C), chain=ec.LONGEST_SUM_CHAIN)
    got = torch.cat([ref.s0, ref.s1])
    got[c] -= dout[dout[:, c].abs().argmax(), c]
    rejects(lambda: ec.check("s0 row", "sums", got.float(), ref.sums_bound()), f"(i={c})")


def test_rejects_unbiased_variance():
    M, C = 8, 256  # the image-pool BN at batch 8
    x, r, gamma, beta, _ = bn_operands(M, C, 20)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 0)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    wrong = gamma.double() * (x - st.mean) / torch.sqrt(st.unbiased + EPS) + beta.double() + r
    rejects(lambda: ec.check_apply("unbiased", to_bf16(wrong.clamp_min(0)), pre, acc), "m=")


def test_rejects_var_plus_eps_instead_of_clamp():
    M, C = 162, 64
    x, r, gamma, beta, _ = bn_operands(M, C, 21, scale=1e-3)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 1)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    wrong = gamma.double() * (x - st.mean) / torch.sqrt(st.var + EPS) + beta.double() + r
    rejects(lambda: ec.check_apply("var + eps", to_bf16(wrong.clamp_min(0)), pre, acc), "m=")


def test_rejects_residual_missing_at_one_element():
    M, C = 99, 304
    x, r, gamma, beta, _ = bn_operands(M, C, 22)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 0)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    got = to_bf16(pre)
    m, c = 57, 301
    assert abs(r[m, c]) > 0.1
    got[m, c] = to_bf16(pre[m, c] - r[m, c])
    rejects(lambda: ec.check_apply("no res", got, pre, acc, relu=False), f"(m={m}, c={c})", "1 element(s)")


def test_rejects_missing_keep_scale_in_backward():
    M, C, p = 198, 64, 0.1
    x, r, gamma, beta, dout, save, out = bwd_case(M, C, 23, keep_p=p)
    keep = ec.fp32_keep(p)
    ref = ec.BwdRef(dout, x, save, gamma, mask=out > 0, keep=keep, chain=ec.bwd_chain_fused(M, C, SMS))
    wrong = ec.BwdRef(dout, x, save, gamma, mask=out > 0, keep=1.0)
    rejects(lambda: ec.check("no keep", "sums", torch.cat([wrong.s0, wrong.s1]).float(), ref.sums_bound()), "(i=")
    rejects(lambda: ec.check("no keep", "dx", to_bf16(wrong.dx_bound().ref), ref.dx_bound()), "(m=")
    rejects(lambda: ec.check("no keep", "dres", to_bf16(wrong.dz), ref.dres_bound()), "(m=")


def test_rejects_mask_from_pre_activation():
    M, C = 198, 256
    x, r, gamma, beta, dout, save, out = bwd_case(M, C, 24)
    st = ec.BnStats(ec.exact_stats(x), M, EPS, 0)
    pre_bn, _ = ec.bn_train_ref(x, st, gamma, beta)  # before the residual add
    ref = ec.BwdRef(dout, x, save, gamma, mask=out > 0, chain=ec.bwd_chain_two_launch(M, C, SMS))
    wrong = ec.BwdRef(dout, x, save, gamma, mask=pre_bn > 0)
    rejects(lambda: ec.check("pre-activation mask", "dx", to_bf16(wrong.dx_bound().ref), ref.dx_bound()), "(m=")


def test_rejects_off_by_one_bin_edge():
    N, H, W, C, bins = 1, 17, 17, 8, 3
    x = to_bf16(torch.randn(N, H, W, C, generator=torch.Generator().manual_seed(25), dtype=torch.float64))
    b = ec.avgpool_fwd_bound(x, bins)
    got = b.ref.clone()
    (h0, h1), (w0, w1) = ec.bin_edges(H, bins)[1], ec.bin_edges(W, bins)[2]
    got[:, 1, 2] = x[:, h0:h1 + 1, w0:w1].mean((1, 2))  # one row too many in bin (1, 2)
    rejects(lambda: ec.check("bin edge", "avgpool y", to_bf16(got), b), "h=1, w=2")


def test_rejects_last_maximum_on_a_tie():
    x = torch.zeros(1, 5, 5, 8, dtype=torch.float64)  # ReLU zeros: every window is a tie
    x[0, 4, 4, 3] = 1.0
    y, tap = ec.maxpool_ref(x)
    assert int(tap[0, 0, 0, 0]) == 4  # window (0, 0) starts at (-1, -1): its first in-bounds tap is (1, 1)
    wrong = tap.clone()
    wrong[0, 1, 1, 0] = 8  # the last tap of window (1, 1)
    rejects(lambda: ec.check_maxpool_fwd("last max", y, wrong, x), "n=0, h=1, w=1, c=0")


def test_rejects_wrong_lambda_in_one_output_row():
    Hi, Wi, Ho, Wo, ac = 9, 9, 33, 33, False
    x = to_bf16(torch.randn(1, Hi, Wi, 16, generator=torch.Generator().manual_seed(26), dtype=torch.float64))
    b = ec.bilinear_fwd_bound(x, Ho, Wo, ac)
    Ay, Ax = ec.lerp_matrix(Hi, Ho, ac), ec.lerp_matrix(Wi, Wo, ac)
    oy = 14
    i0, i1, l1, l0 = ec.lerp_axis(Hi, Ho, ac)
    Ay[oy] = 0
    Ay[oy, i0[oy]] += float(l0[oy + 1])  # the next row's lambda
    Ay[oy, i1[oy]] += float(l1[oy + 1])
    got = torch.einsum("oh,nhwc,pw->nopc", Ay, x, Ax)
    msg = rejects(lambda: ec.check("wrong lambda", "bilinear y", to_bf16(got), b), f"h={oy}")
    assert "h=13," not in msg and "h=15," not in msg


def test_rejects_align_corners_swapped():
    for Hi, Ho in ((9, 33), (6, 60), (33, 129)):
        x = to_bf16(torch.randn(1, Hi, Hi, 8, generator=torch.Generator().manual_seed(27), dtype=torch.float64))
        for ac in (True, False):
            b = ec.bilinear_fwd_bound(x, Ho, Ho, ac)
            got = ec.bilinear_fwd_bound(x, Ho, Ho, not ac).ref
            rejects(lambda: ec.check("ac swapped", "bilinear y", to_bf16(got), b), "n=0")
            dy = to_bf16(torch.randn(1, Ho, Ho, 8, generator=torch.Generator().manual_seed(28), dtype=torch.float64))
            bb = ec.bilinear_bwd_bound(dy, Hi, Hi, ac)
            got = ec.bilinear_bwd_bound(dy, Hi, Hi, not ac).ref
            rejects(lambda: ec.check("ac swapped", "bilinear dx", to_bf16(got), bb), "n=0")


def test_rejects_missing_tap_in_backward_fallback():
    """1 x 2 -> 33 x 60 with align_corners: every input pixel feeds > MAXN outputs per axis (the fallback loop)."""
    Hi, Wi, Ho, Wo = 1, 2, 33, 60
    assert ec.outputs_per_input(Hi, Ho, True) > ec.MAXN and ec.outputs_per_input(Wi, Wo, True) > ec.MAXN
    dy = to_bf16(torch.randn(1, Ho, Wo, 8, generator=torch.Generator().manual_seed(29), dtype=torch.float64))
    bb = ec.bilinear_bwd_bound(dy, Hi, Wi, True)
    Ay, Ax = ec.lerp_matrix(Hi, Ho, True), ec.lerp_matrix(Wi, Wo, True)
    c, oy, ox = 6, 17, 21
    got = bb.ref.clone()
    got[0, :, :, c] -= Ay[oy].view(Hi, 1) * Ax[ox].view(1, Wi) * dy[0, oy, ox, c]  # tap (17, 21) left out
    assert abs(dy[0, oy, ox, c]) > 0.5
    rejects(lambda: ec.check("missing tap", "bilinear dx", to_bf16(got), bb), f"c={c}")


def test_rejects_beta_ignored():
    x_shape = (1, 17, 17, 8)
    g = torch.Generator().manual_seed(30)
    dy = to_bf16(torch.randn(1, 6, 6, 8, generator=g, dtype=torch.float64))
    old = to_bf16(torch.randn(x_shape, generator=g, dtype=torch.float64))
    bb = ec.bilinear_bwd_bound(dy, 17, 17, True, beta=1.0, old=old)
    got = ec.bilinear_bwd_bound(dy, 17, 17, True).ref
    rejects(lambda: ec.check("beta ignored", "bilinear dx", to_bf16(got), bb), "n=0, h=0, w=0")
    ab = ec.avgpool_bwd_bound(dy, x_shape, 6, beta=1.0, old=old)
    got = ec.avgpool_bwd_bound(dy, x_shape, 6).ref
    rejects(lambda: ec.check("beta ignored", "avgpool dx", to_bf16(got), ab), "n=0, h=0, w=0")
    v = dy.reshape(-1, 8)
    o = old[0, :6, :6].reshape(-1, 8)
    rejects(lambda: ec.check("beta ignored", "axpby", v, ec.axpby_bound(v, 1.0, o)), "m=0")


def test_rejects_element_one_channel_to_the_right():
    N, H, W, C = 1, 3, 5, 24
    ref = to_bf16(torch.randn(N, H, W, C, generator=torch.Generator().manual_seed(31), dtype=torch.float64))
    b = ec.bound(ref, torch.zeros_like(ref), True, ec.NAMES_NHWC)
    # interior channel: the value lands on its neighbour, and the element itself keeps the sentinel
    g = ec.Guarded(N, H, W, C, torch.bfloat16)
    g.view.copy_(ref)
    g.view[0, 1, 2, 10] = g.view[0, 1, 2, 9]
    g.view[0, 1, 2, 9] = float("nan")
    ec.sentinel_fill(g.view[0, 1, 2, 9:10])
    rejects(lambda: ec.check("shift", "y", g.view, b), "n=0, h=1, w=2, c=10")
    rejects(lambda: ec.check_written("shift", g.view), "(0, 1, 2, 9)")
    # last channel: the write lands in the right guard
    g = ec.Guarded(N, H, W, C, torch.bfloat16)
    g.view.copy_(ref)
    g.buf[0, 2, 4, ec.GUARD + C] = g.view[0, 2, 4, C - 1]
    rejects(lambda: ec.check_guards("shift", g.buf, g.guard_mask()), f"(0, 2, 4, {ec.GUARD + C})")
