"""Conformance sweep of the streaming kernels of seg_elementwise.cu: BatchNorm statistics / finalize / apply
(+residual, ReLU, dropout) / backward (two-launch and cooperative), max pool, adaptive average pool, bilinear resize
(bf16 NHWC and fp32 logits), ReLU and axpby.

Every case is checked element by element against a float64 reference with the bounds of tests/elementwise_check.py.
Outputs are written into guarded buffers (conv_check.Guarded: sentinel guard channels on both sides of the slice and a
trailing guard image; conv_check.FlatGuarded for outputs that are dense by API), which must come back bit for bit, and
the logical region starts as the sentinel whenever the kernel does not read it, so an element never written is caught.
Inputs are slices of sentinel-filled (NaN) buffers: a read outside the slice produces NaN and fails.  Every case runs
twice and must be bit-identical between the runs (fixed-order fp32 folds and exact fp64 atomics).  Each case appends its
bound usage, the schedule regime it asserted and its wall time to gpu_out_dir/elementwise_conformance.txt.

The schedule cases are sized from the SM count at run time with mirrors of the host grid functions
(elementwise_check.colreduce_grid / rowmap_grid / fused_grid), and each asserts that it reaches the regime it names."""
import math
import os
import time

import pytest
import torch

import conv_check as cc
import elementwise_check as ec

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib, ops

DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32
EPS, MOM = 1e-5, 0.1


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "elementwise_conformance.txt"), "a")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def place(t, lead=cc.GUARD):
    """A bf16 NHWC device tensor holding t (float64, bf16-exact) as a channel slice at offset `lead` of a sentinel
    buffer whose pitch is a multiple of 8, with a trailing guard image."""
    N, H, W, C = t.shape
    trail = cc.GUARD + (-(lead + C + cc.GUARD)) % 8
    buf = cc.sentinel_fill(torch.empty(N + 1, H, W, lead + C + trail, dtype=BF16, device=DEV))
    buf[:N, ..., lead:lead + C] = t.to(DEV, BF16)
    return buf[:N, ..., lead:lead + C]


def place_flat(t, dtype=BF16):
    """A dense device tensor holding t inside a FlatGuarded sentinel buffer (dense-by-API inputs)."""
    g = cc.FlatGuarded(tuple(t.shape), dtype, device=DEV)
    g.view.copy_(t.to(DEV, dtype))
    return g.view


def guarded(shape, old=None, dtype=BF16):
    N, H, W, C = shape
    g = cc.Guarded(N, H, W, C, dtype, device=DEV)
    if old is not None:
        g.view.copy_(old.to(DEV, dtype))
    return g


def settle(case, gs, written=True):
    torch.cuda.synchronize()
    for g in gs:
        cc.check_guards(case, g.buf, g.guard_mask())
        if written:
            cc.check_written(case, g.view)


def same_bits(case, what, a, b):
    ia = a.view(torch.int16) if a.dtype == BF16 else (a.view(torch.int32) if a.dtype == F32 else a)
    ib = b.view(torch.int16) if b.dtype == BF16 else (b.view(torch.int32) if b.dtype == F32 else b)
    assert torch.equal(ia, ib), f"{case}: {what} not bit-reproducible"


def fmt(u):
    return f"{u:.4f}"


def rand_bf16(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ec.bf16_round(torch.randn(shape, generator=g, dtype=torch.float64) * scale)


# ------------------------------------------------------------------------------------------------ BatchNorm
def bn_operands(N, H, W, C, seed, clamp_eps=False):
    """x with per-channel magnitudes 2^0 .. 2^-9 and offsets, residual, gamma, beta, dout (bf16 / fp32 exact)."""
    M = N * H * W
    g = torch.Generator().manual_seed(seed)
    cs = ec.channel_scales(C, seed + 1) * (1e-3 if clamp_eps else 1.0)
    x = ec.bf16_round((torch.randn(M, C, generator=g, dtype=torch.float64) + 0.5) * cs)
    r = ec.bf16_round(torch.randn(M, C, generator=g, dtype=torch.float64))
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.3
    dout = ec.bf16_round(torch.randn(M, C, generator=g, dtype=torch.float64))
    return x, r, gamma, beta, dout


def regimes(M, C):
    """The schedule facts a case reaches, from the host grid mirrors."""
    s = sms()
    sx, sy, cap = ec.colreduce_grid(M, C, s)
    f1, f8 = ec.fused_schedule(M, C, s, 1), ec.fused_schedule(M, C, s, 8)
    G = C // 8
    return {"stats_gx": sx, "stats_cap": cap, "stats_cap_hit": -(-M // (ec.rows_par(C) * 4)) > cap,
            "rows_par": ec.rows_par(C), "idle_row_lanes": ec.rows_par(C) * min(G, 256) < 256,
            "apply_gx": ec.rowmap_grid(M, C, s)[0], "reduce_gx": ec.reduce2_grid(M, C, s)[0],
            "slabs": f1["slabs"], "last_slab_groups": G - (f1["slabs"] - 1) * 256,
            "fused_nb": (f1["nb"], f8["nb"]), "cpb": (f1["cpb"], f8["cpb"]),
            "cpb_gt_256": f1["cpb"] > 256 and f8["cpb"] > 256,
            "idle_fold": f1["idle_fold_blocks"] > 0 and f8["idle_fold_blocks"] > 0}


def fmt_reg(rg, keys):
    return " ".join(f"{k}={rg[k]}" for k in keys)


def run_bn(log, case, shape, res=True, relu=True, drop_p=0.0, drop_hw=False, remask=False, beta_res=0.0,
           accumulate=False, clamp_eps=False, zero_sums=False, paths=("two", "fused"), seed=0, show=()):
    t0 = time.time()
    N, H, W, C = shape
    M = N * H * W
    s = sms()
    assert not (remask and (res or drop_p or not relu))
    x, r, gamma, beta, dout = bn_operands(N, H, W, C, seed, clamp_eps)
    if not res:
        r = None
    xd = place(x.view(shape))
    rd = place(r.view(shape)) if res else None
    dd = place(dout.view(shape))
    gd, bd = gamma.to(DEV), beta.to(DEV)
    usage = {}
    # ---- bn_stats (sums read back against the exact sums of the input)
    st1, st2 = ops.bn_stats(xd), ops.bn_stats(xd)
    torch.cuda.synchronize()
    same_bits(case, "bn_stats", st1.view(torch.int64), st2.view(torch.int64))
    chain = cc.stat_chain_simt(M, C, s)
    assert chain <= ec.LONGEST_SUM_CHAIN
    usage["stats"] = cc.check_stats(case, st1, x, chain)
    # ---- bn_apply_train from exact host sums: the apply kernel in isolation
    stats = ec.exact_stats(x)
    st = ec.BnStats(stats, M, EPS, clamp_eps)
    pre, acc = ec.bn_train_ref(x, st, gamma, beta, r)
    g = torch.Generator().manual_seed(seed + 7)
    rm0, rv0 = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    runs = []
    for _ in range(2):
        go = guarded(shape)
        rm, rv = rm0.to(DEV), rv0.to(DEV)
        ctr = torch.zeros(1, dtype=torch.int64, device=DEV) if drop_p else None
        _, save = ops.bn_apply_train(xd, stats.to(DEV), M, gd, bd, EPS, MOM, int(clamp_eps), rm, rv, res=rd, out=go.view,
                                     relu=relu, drop_p=drop_p, seed=1234 + seed, step_ctr=ctr,
                                     drop_hw=H * W if drop_hw else 0)
        settle(case, [go])
        runs.append((go, save.clone(), rm.clone(), rv.clone()))
    for i, what in enumerate(("out", "save", "running mean", "running var")):
        a, b = (runs[0][i].view if i == 0 else runs[0][i]), (runs[1][i].view if i == 0 else runs[1][i])
        same_bits(case, what, a, b)
    go, save, rm, rv = runs[0]
    out2d = go.view.reshape(M, C).cpu().double()
    note = ""
    if drop_p:
        units = ((torch.arange(M).view(M, 1) // (H * W)) * C + torch.arange(C).view(1, C)) if drop_hw else None
        usage["out"], frac, n = ec.check_dropout(case, out2d, pre, acc, drop_p, units=units)
        note += f" dropped={frac:.4f}/{n}"
    else:
        usage["out"] = ec.check_apply(case, out2d, pre, acc, relu)
    usage["save"] = ec.check_save(case, save, st)
    usage["running"] = ec.check_running(case, rm, rv, rm0, rv0, st, MOM)
    # ---- backward: the stored activation is the kernel's own output (as in the engine)
    save_h = save.cpu()
    keep = ec.fp32_keep(drop_p) if drop_p else 1.0
    amb = None
    if not relu:
        mask = None
    elif remask:
        mask, amb = ec.remask(x, gamma, beta, save_h[:C], save_h[C:])
        n_amb = int(amb.sum())
        assert n_amb <= 8 + M * C // 10000, f"{case}: {n_amb} mask values within rounding of zero"
        note += f" remask_ambiguous={n_amb}"
    else:
        mask = out2d > 0
    outd = None if remask else go.view
    old = rand_bf16((M, C), seed + 11) if beta_res else None
    old_pg = torch.randn(2, C, generator=torch.Generator().manual_seed(seed + 12)) if accumulate else None
    for path in paths:
        chain = ec.bwd_chain_two_launch(M, C, s) if path == "two" else ec.bwd_chain_fused(M, C, s)
        assert chain <= ec.LONGEST_SUM_CHAIN
        ref = ec.BwdRef(dout, x, save_h, gamma, mask=mask, keep=keep, chain=chain, ambiguous=amb)
        outs = []
        for _ in range(2):
            pg = [cc.FlatGuarded((C,), F32, device=DEV) for _ in range(2)]  # dbeta, dgamma
            if accumulate:
                pg[0].view.copy_(old_pg[0])
                pg[1].view.copy_(old_pg[1])
            gx = guarded(shape)
            gr = guarded(shape, old.view(shape) if beta_res else None)
            if path == "two":
                assert not zero_sums
                sums = ops.bn_bwd_reduce(dd, outd, xd, save, relu=relu, drop_p=drop_p, dgamma=pg[1].view, dbeta=pg[0].view,
                                         accumulate=accumulate, gamma=gd, beta=bd)
                ops.bn_bwd_apply(dd, outd, xd, save, gd, sums, M, relu=relu, drop_p=drop_p, dx=gx.view, dres=gr.view,
                                 beta_res=beta_res, beta=bd)
            else:
                _, sums = ops.bn_bwd_fused(dd, outd, xd, save, gd, M, relu=relu, drop_p=drop_p, dgamma=pg[1].view,
                                           dbeta=pg[0].view, accumulate=accumulate, dx=gx.view, dres=gr.view,
                                           beta_res=beta_res, beta=bd, zero_sums=zero_sums)
            settle(case, [gx, gr])
            for p in pg:
                cc.check_guards(case, p.buf, p.guard_mask())
            outs.append((gx.view.clone(), gr.view.clone(), sums.clone(), pg[0].view.clone(), pg[1].view.clone()))
        for i, what in enumerate(("dx", "dres", "sums", "dbeta", "dgamma")):
            same_bits(f"{case} {path}", what, outs[0][i], outs[1][i])
        dx, dres, sums, dbeta, dgamma = outs[0]
        c2 = f"{case} {path}"
        usage[f"{path}_sums"] = ec.check(c2, "sums", sums, ref.sums_bound())
        usage[f"{path}_dx"] = ec.check(c2, "dx", dx.reshape(M, C), ref.dx_bound(zero_sums), alt=ref.dx_alt(zero_sums))
        usage[f"{path}_dres"] = ec.check(c2, "dres", dres.reshape(M, C), ref.dres_bound(beta_res, old))
        usage[f"{path}_dbeta"] = ec.check(c2, "dbeta", dbeta, ref.param_bound(0, old_pg[0] if accumulate else None))
        usage[f"{path}_dgamma"] = ec.check(c2, "dgamma", dgamma, ref.param_bound(1, old_pg[1] if accumulate else None))
        if path == "fused":  # the host's workspace sizing mirrors fused_grid at the larger occupancy
            nr, _ = ops.bn_bwd_fused_workspace(M, C)
            W_ = min(C // 8, 256) * 8
            gy = -(-(C // 8) // 256)
            nb = nr // (gy * 2 * W_)
            assert any(ec.fused_grid(M, C, s, b)[0] == nb for b in range(1, 9)), (case, nb)
            note += f" fused_nb_ws={nb}"
    rg = regimes(M, C)
    worst = max(usage.values())
    log(f"bn {case} M={M} C={C} usage={fmt(worst)} " + " ".join(f"{k}={fmt(v)}" for k, v in usage.items())
        + " " + fmt_reg(rg, ("stats_gx", "stats_cap") + tuple(show)) + note + f" wall={time.time() - t0:.1f}s")
    return rg


CHANNELS = [8, 48, 64, 256, 304, 728, 1536, 2048, 2064, 4096]


@pytest.mark.parametrize("C", CHANNELS)
def test_bn_channels(log, C):
    rg = run_bn(log, f"channels C={C}", (2, 9, 11, C), seed=C, beta_res=1.0 if C % 16 else 0.0,
                accumulate=C % 3 == 0, show=("idle_row_lanes", "slabs", "last_slab_groups", "cpb"))
    if C in (304, 728, 1536):
        assert rg["idle_row_lanes"]
    if C == 2064:
        assert rg["slabs"] == 2 and rg["last_slab_groups"] == 2
    if C == 4096:
        assert rg["slabs"] == 2 and rg["last_slab_groups"] == 256


def cap_rows(C, over):
    """Rows at which bn_stats's grid reaches its cap exactly (over=False) or would pass it by one block (True)."""
    _, _, cap = ec.colreduce_grid(1, C, sms())
    return cap * ec.rows_par(C) * 4 + (1 if over else 0)


ROW_CASES = {
    "m1_c64": lambda: ((1, 1, 1, 64), None),
    "m1_c2064": lambda: ((1, 1, 1, 2064), None),
    "m5_under_rows_par_c64": lambda: ((1, 1, 5, 64), "m_lt_rows_par"),
    "m100_under_rows_par_c8": lambda: ((1, 10, 10, 8), "m_lt_rows_par"),
    "stats_cap_c2048": lambda: ((1, 1, cap_rows(2048, False), 2048), "at_cap"),
    "stats_cap_plus1_c2048": lambda: ((1, 1, cap_rows(2048, True), 2048), "over_cap"),
    "stats_cap_plus1_c64": lambda: ((1, 1, cap_rows(64, True), 64), "over_cap"),
    "engine_layer1_4x129x129_c256": lambda: ((4, 129, 129, 256), "over_cap"),
}


@pytest.mark.parametrize("name", list(ROW_CASES))
def test_bn_rows(log, name):
    shape, regime = ROW_CASES[name]()
    N, H, W, C = shape
    M = N * H * W
    rg = regimes(M, C)
    if regime == "m_lt_rows_par":
        assert M < rg["rows_par"]
    elif regime == "at_cap":
        assert not rg["stats_cap_hit"] and rg["stats_gx"] == rg["stats_cap"]
    elif regime == "over_cap":
        assert rg["stats_cap_hit"] and rg["stats_gx"] == rg["stats_cap"]
    run_bn(log, f"rows {name}", shape, seed=len(name), beta_res=1.0, show=("stats_cap_hit", "apply_gx", "reduce_gx",
                                                                            "fused_nb"))


FUSED_CASES = {
    "cpb_gt_256_c2048_m15": ((1, 3, 5, 2048), "cpb_gt_256"),
    "cpb_gt_256_c2048_m8": ((8, 1, 1, 2048), "cpb_gt_256"),
    "idle_fold_c8": ((2, 65, 65, 8), "idle_fold"),
    "idle_fold_c64": ((2, 65, 65, 64), "idle_fold"),
    "image_pool_c256_m8": ((8, 1, 1, 256), None),
    "psp_bin1_c512_m8": ((8, 1, 1, 512), None),
}


@pytest.mark.parametrize("name", list(FUSED_CASES))
def test_bn_fused_schedules(log, name):
    shape, regime = FUSED_CASES[name]
    N, H, W, C = shape
    rg = regimes(N * H * W, C)
    if regime:
        assert rg[regime], (name, rg)
    run_bn(log, f"fused {name}", shape, seed=len(name), accumulate=True, show=("fused_nb", "cpb", "cpb_gt_256", "idle_fold"))


VARIANTS = {
    "relu_off": dict(relu=False),
    "remask": dict(res=False, remask=True),
    "remask_c2064": dict(res=False, remask=True, C=2064),
    "dropout_p0.1": dict(drop_p=0.1),
    "dropout_p0.5": dict(drop_p=0.5, beta_res=1.0),
    "dropout2d_p0.5": dict(drop_p=0.5, drop_hw=True),
    "dropout2d_p0.1_no_res": dict(drop_p=0.1, drop_hw=True, res=False),
    "zero_sums": dict(zero_sums=True, paths=("fused",)),
    "accumulate_beta_res1": dict(accumulate=True, beta_res=1.0),
    "beta_res0_no_res": dict(res=False, beta_res=0.0),
    "clamp_eps": dict(clamp_eps=True),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_bn_variants(log, name):
    kw = dict(VARIANTS[name])
    C = kw.pop("C", 304)
    run_bn(log, f"variant {name}", (2, 17, 19, C), seed=len(name) * 7, **kw)


@pytest.mark.parametrize("C,clamp", [(64, 0), (304, 1), (2064, 0)])
def test_bn_finalize_eval_and_apply(log, C, clamp):
    """bn_finalize (fp64 sqrt) and bn_eval_scale_shift (rsqrtf) coefficients; bn_apply with given scale / shift."""
    N, H, W = 2, 9, 11
    M = N * H * W
    x, r, gamma, beta, _ = bn_operands(N, H, W, C, C + clamp, clamp_eps=bool(clamp))
    stats = ec.exact_stats(x)
    st = ec.BnStats(stats, M, EPS, clamp)
    g = torch.Generator().manual_seed(5)
    rm0, rv0 = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    rm, rv = rm0.to(DEV), rv0.to(DEV)
    ss, save = ops.bn_finalize(stats.to(DEV), M, gamma.to(DEV), beta.to(DEV), EPS, MOM, clamp, rm, rv)
    case = f"finalize C={C} clamp={clamp}"
    u = [ec.check_scale_shift(case, ss, gamma, beta, st.mean, st.istd), ec.check_save(case, save, st),
         ec.check_running(case, rm, rv, rm0, rv0, st, MOM)]
    shape = (N, H, W, C)
    xd, rd = place(x.view(shape)), place(r.view(shape))
    for relu in (True, False):
        outs = []
        for _ in range(2):
            go = guarded(shape)
            ops.bn_apply(xd, ss, res=rd, out=go.view, relu=relu)
            settle(case, [go])
            outs.append(go.view.clone())
        same_bits(case, "bn_apply", outs[0], outs[1])
        pre, acc = ec.bn_ss_ref(x, ss.cpu(), r)
        u.append(ec.check_apply(case, outs[0].reshape(M, C), pre, acc, relu))
    ss_e, save_e = ops.bn_eval_scale_shift(gamma.to(DEV), beta.to(DEV), rm0.to(DEV), rv0.to(DEV), EPS, want_save=True)
    istd_e = 1.0 / torch.sqrt(rv0.double() + float(torch.tensor(EPS, dtype=F32)))
    u.append(ec.check_scale_shift(case + " eval", ss_e, gamma, beta, rm0.double(), istd_e))
    u.append(ec.check(case + " eval", "save", save_e, ec.bound(torch.cat([rm0.double(), istd_e]),
                                                                ec.K_COEF * ec.U32 * torch.cat([rm0.double(), istd_e]).abs(),
                                                                False, ("i",))))
    log(f"bn {case} usage={fmt(max(u))}")


@pytest.mark.parametrize("kernel", ["reduce", "apply", "fused"])
def test_bn_backward_dropout_without_relu_is_rejected(kernel):
    """The backward reads the keep mask from the stored activation (out > 0), which without the ReLU does not tell a
    dropped element from a negative one: relu = 0 with drop_p > 0 must be refused, not silently run without dropout."""
    N, H, W, C = 1, 3, 5, 64
    t = torch.zeros(N, H, W, C, dtype=BF16, device=DEV)
    save = torch.cat([torch.zeros(C), torch.ones(C)]).to(DEV)
    gamma, beta = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
    sums = torch.zeros(2 * C, device=DEV)
    with pytest.raises(RuntimeError, match="needs relu"):
        if kernel == "reduce":
            ops.bn_bwd_reduce(t, t, t, save, relu=False, drop_p=0.1)
        elif kernel == "apply":
            ops.bn_bwd_apply(t, t, t, save, gamma, sums, N * H * W, relu=False, drop_p=0.1)
        else:
            ops.bn_bwd_fused(t, t, t, save, gamma, N * H * W, relu=False, drop_p=0.1, beta=beta)


# ------------------------------------------------------------------------------------------------ bilinear
def maxn_boundary_pair(target):
    """(in, out) with align_corners whose widest input row feeds exactly `target` outputs."""
    for inp in range(3, 12):
        for out in range(inp, 400):
            if ec.outputs_per_input(inp, out, True) == target:
                return inp, out
    raise AssertionError(target)


BIL_PAIRS = {  # name: (Hi, Wi, Ho, Wo, align_corners)
    "aspp_pool_1to33": (1, 1, 33, 33, True),
    "aspp_pool_1to65": (1, 1, 65, 65, True),
    "psp_2to60": (2, 2, 60, 60, True),
    "psp_3to60": (3, 3, 60, 60, True),
    "psp_6to60": (6, 6, 60, 60, True),
    "decoder_33to129": (33, 33, 129, 129, True),
    "maxn_24": None,
    "maxn_25": None,
    "ratio_9x7to31x29": (9, 7, 31, 29, True),
    "ratio_9x7to31x29_half_pixel": (9, 7, 31, 29, False),
    "down_65to33": (65, 65, 33, 33, True),
    "down_65to33_half_pixel": (65, 65, 33, 33, False),
    "identity_13": (13, 13, 13, 13, False),
    "up_1to33_half_pixel": (1, 1, 33, 33, False),
    "up_17to65_half_pixel": (17, 17, 65, 65, False),
    "up_9to33": (9, 9, 33, 33, True),
    "up_9to33_half_pixel": (9, 9, 33, 33, False),
    "up_1to9": (1, 1, 9, 9, True),
    "up_1to9_half_pixel": (1, 1, 9, 9, False),
    "up_6to15": (6, 6, 15, 15, True),
    "up_6to15_half_pixel": (6, 6, 15, 15, False),
    "up_8to31x29": (8, 8, 31, 29, True),
    "up_8to31x29_half_pixel": (8, 8, 31, 29, False),
}
BIL_CHANNELS = {"aspp_pool_1to33": (8, 256, 304), "psp_2to60": (8, 304), "psp_6to60": (8, 256), "decoder_33to129": (8, 256)}


def bil_case(name):
    if name.startswith("maxn_"):
        inp, out = maxn_boundary_pair(int(name[5:]))
        return inp, inp, out, out, True
    return BIL_PAIRS[name]


BIL_IDS = [(n, c) for n in BIL_PAIRS for c in BIL_CHANNELS.get(n, (8,))]


@pytest.mark.parametrize("name,C", BIL_IDS, ids=[f"{n}-C{c}" for n, c in BIL_IDS])
def test_bilinear(log, name, C):
    t0 = time.time()
    Hi, Wi, Ho, Wo, ac = bil_case(name)
    N = 2
    per = max(ec.outputs_per_input(Hi, Ho, ac), ec.outputs_per_input(Wi, Wo, ac))
    fallback = per > ec.MAXN
    if name.startswith("aspp_pool_1to33") or name.startswith("psp_2") or name.startswith("psp_3"):
        assert fallback, (name, per)
    if name == "psp_6to60":
        assert not fallback and per >= ec.MAXN - 1, per
    if name.startswith("maxn_"):
        assert per == int(name[5:])
    case = f"{name} C={C} ac={ac}"
    x = rand_bf16((N, Hi, Wi, C), 1) * ec.channel_scales(C, 2)
    xd = place(x)
    outs = []
    for _ in range(2):
        go = guarded((N, Ho, Wo, C))
        ops.bilinear_fwd(xd, Ho, Wo, ac, out=go.view)
        settle(case, [go])
        outs.append(go.view.clone())
    same_bits(case, "bilinear y", outs[0], outs[1])
    u = [ec.check(case, "bilinear y", outs[0], ec.bilinear_fwd_bound(x, Ho, Wo, ac))]
    dy = rand_bf16((N, Ho, Wo, C), 3) * ec.channel_scales(C, 4)
    dyd = place(dy)
    old = rand_bf16((N, Hi, Wi, C), 5)
    for beta in (0.0, 1.0):
        outs = []
        for _ in range(2):
            gd = guarded((N, Hi, Wi, C), old if beta else None)
            ops.bilinear_bwd(dyd, Hi, Wi, ac, dx=gd.view, beta=beta)
            settle(case, [gd])
            outs.append(gd.view.clone())
        same_bits(case, "bilinear dx", outs[0], outs[1])
        u.append(ec.check(f"{case} beta={beta}", "bilinear dx", outs[0], ec.bilinear_bwd_bound(dy, Hi, Wi, ac, beta, old)))
    log(f"bilinear {case} {Hi}x{Wi}->{Ho}x{Wo} usage={fmt(max(u))} outputs_per_input={per} fallback={fallback}"
        f" wall={time.time() - t0:.1f}s")


LOGIT_CASES = [(33, 33, 129, 129, True, 21), (33, 33, 129, 129, False, 19), (9, 7, 31, 29, False, 8), (1, 1, 33, 33, True, 3),
               (9, 9, 33, 33, True, 16), (1, 1, 9, 9, False, 16), (6, 6, 15, 15, True, 16), (8, 8, 31, 29, False, 16)]


@pytest.mark.parametrize("case_", LOGIT_CASES, ids=[f"{a}x{b}to{c}x{d}{'ac' if e else ''}_C{f}" for a, b, c, d, e, f in LOGIT_CASES])
def test_bilinear_logits(log, case_):
    Hi, Wi, Ho, Wo, ac, C = case_
    N, ldx = 2, -(-C // 8) * 8 + 8
    case = f"logits {Hi}x{Wi}->{Ho}x{Wo} ac={ac} C={C}"
    x = torch.randn(N, Hi, Wi, C, generator=torch.Generator().manual_seed(1)).double()  # fp32 logits
    xd = place_flat(x, F32)
    outs = []
    for _ in range(2):
        gy = cc.FlatGuarded((N, C, Ho, Wo), F32, device=DEV)
        lib.call("seg_bilinear_logits_fwd", lib.ptr(xd), lib.ptr(gy.view), N, Hi, Wi, Ho, Wo, C, int(ac))
        torch.cuda.synchronize()
        cc.check_guards(case, gy.buf, gy.guard_mask())
        cc.check_written(case, gy.view)
        outs.append(gy.view.clone())
    same_bits(case, "logits y", outs[0], outs[1])
    same_bits(case, "logits y (ops wrapper)", outs[0], ops.bilinear_logits_fwd(xd, Ho, Wo, ac))
    b = ec.bilinear_fwd_bound(x, Ho, Wo, ac, out_bf16=False)
    u = [ec.check(case, "logits y", cc.nhwc(outs[0]), b)]
    dy = torch.randn(N, C, Ho, Wo, generator=torch.Generator().manual_seed(2)).double()
    dyd = place_flat(dy, F32)
    outs = []
    for _ in range(2):
        gx = cc.FlatGuarded((N, Hi, Wi, ldx), BF16, device=DEV)
        lib.call("seg_bilinear_logits_bwd", lib.ptr(dyd), lib.ptr(gx.view), ldx, N, Hi, Wi, Ho, Wo, C, int(ac))
        torch.cuda.synchronize()
        cc.check_guards(case, gx.buf, gx.guard_mask())
        cc.check_written(case, gx.view)
        outs.append(gx.view.clone())
    same_bits(case, "logits dx", outs[0], outs[1])
    same_bits(case, "logits dx (ops wrapper)", outs[0], ops.bilinear_logits_bwd(dyd, Hi, Wi, ac, ldx))
    assert outs[0][..., C:].float().abs().max().item() == 0, f"{case}: pad channels C..ldx-1 not zero"
    u.append(ec.check(case, "logits dx", outs[0][..., :C], ec.bilinear_bwd_bound(cc.nhwc(dy), Hi, Wi, ac)))
    log(f"bilinear_logits {case} usage={fmt(max(u))}")


# ------------------------------------------------------------------------------------------------ pooling
MAXPOOL_SHAPES = [(2, 33, 35, 64), (1, 1, 1, 8), (1, 2, 2, 16), (2, 1, 6, 8), (1, 8, 7, 24), (2, 2, 9, 8),
                  (2, 65, 64, 8), (2, 129, 129, 64)]


class U8Guarded:
    """uint8 tensor inside a flat buffer of 0xA5 words (not a tap code)."""

    def __init__(self, shape):
        n = math.prod(shape)
        self.buf = torch.full((n + 2 * cc.GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
        self.view = self.buf[cc.GUARD:cc.GUARD + n].view(shape)

    def check(self, case):
        b = self.buf.cpu()
        assert bool((b[:cc.GUARD] == 0xA5).all() and (b[-cc.GUARD:] == 0xA5).all()), f"{case}: idx guard overwritten"
        assert int(self.view.max()) <= 8, f"{case}: idx holds a code > 8 (never written?)"


@pytest.mark.parametrize("shape", MAXPOOL_SHAPES, ids=["x".join(map(str, s)) for s in MAXPOOL_SHAPES])
def test_maxpool(log, shape):
    N, H, W, C = shape
    P, Q = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    case = f"maxpool {'x'.join(map(str, shape))}"
    x = rand_bf16(shape, 1).clamp_min(0)  # ReLU zeros: ties
    xd = place_flat(x)
    outs = []
    for _ in range(2):
        gy, gi = cc.FlatGuarded((N, P, Q, C), BF16, device=DEV), U8Guarded((N, P, Q, C))
        lib.call("seg_maxpool3x3s2_fwd", lib.ptr(xd), lib.ptr(gy.view), lib.ptr(gi.view), N, H, W, C, P, Q)
        torch.cuda.synchronize()
        cc.check_guards(case, gy.buf, gy.guard_mask())
        cc.check_written(case, gy.view)
        gi.check(case)
        outs.append((gy.view.clone(), gi.view.clone()))
    same_bits(case, "y", outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])
    y, idx = outs[0]
    yw, iw = ops.maxpool3x3s2_fwd(xd)
    same_bits(case, "y (ops wrapper)", y, yw)
    assert torch.equal(idx, iw), f"{case}: idx differs through the ops wrapper"
    ec.check_maxpool_fwd(case, y, idx.cpu(), x)
    dy = rand_bf16((N, P, Q, C), 2)
    dyd = place_flat(dy)
    outs = []
    for _ in range(2):
        gx = cc.FlatGuarded(shape, BF16, device=DEV)
        lib.call("seg_maxpool3x3s2_bwd", lib.ptr(dyd), lib.ptr(idx), lib.ptr(gx.view), N, H, W, C, P, Q)
        torch.cuda.synchronize()
        cc.check_guards(case, gx.buf, gx.guard_mask())
        cc.check_written(case, gx.view)
        outs.append(gx.view.clone())
    same_bits(case, "dx", outs[0], outs[1])
    same_bits(case, "dx (ops wrapper)", outs[0], ops.maxpool3x3s2_bwd(dyd, idx, shape))
    u = ec.check(case, "maxpool dx", outs[0], ec.maxpool_bwd_bound(dy, idx.cpu().to(torch.int64), shape))
    log(f"{case} usage={fmt(u)} ties={int((x == 0).sum())}")


AVG_SIZES = [(65, 68), (60, 63), (33, 36), (17, 20), (15, 17), (7, 10), (1, 1)]


@pytest.mark.parametrize("bins", [1, 2, 3, 6])
@pytest.mark.parametrize("H,W", AVG_SIZES, ids=[f"{h}x{w}" for h, w in AVG_SIZES])
def test_adaptive_avgpool(log, H, W, bins):
    N, C = 2, 64
    shape = (N, H, W, C)
    case = f"avgpool {H}x{W} bins={bins}"
    overlap = any(e[i][1] > e[i + 1][0] for e in (ec.bin_edges(H, bins), ec.bin_edges(W, bins)) for i in range(bins - 1))
    x = rand_bf16(shape, 1) * ec.channel_scales(C, 2)
    xd = place(x)  # pitched input
    outs = []
    for _ in range(2):
        gy = cc.FlatGuarded((N, bins, bins, C), BF16, device=DEV)
        lib.call("seg_adaptive_avgpool_fwd", lib.ptr(xd), ops.ld(xd), lib.ptr(gy.view), N, H, W, C, bins)
        torch.cuda.synchronize()
        cc.check_guards(case, gy.buf, gy.guard_mask())
        cc.check_written(case, gy.view)
        outs.append(gy.view.clone())
    same_bits(case, "y", outs[0], outs[1])
    same_bits(case, "y (ops wrapper)", outs[0], ops.adaptive_avgpool_fwd(xd, bins))
    u = [ec.check(case, "avgpool y", outs[0], ec.avgpool_fwd_bound(x, bins))]
    dy = rand_bf16((N, bins, bins, C), 3)
    dyd = place_flat(dy)
    old = rand_bf16(shape, 4)
    for beta in (0.0, 1.0):
        outs = []
        for _ in range(2):
            gx = guarded(shape, old if beta else None)
            ops.adaptive_avgpool_bwd(dyd, shape, bins, dx=gx.view, beta=beta)
            settle(case, [gx])
            outs.append(gx.view.clone())
        same_bits(case, "dx", outs[0], outs[1])
        u.append(ec.check(f"{case} beta={beta}", "avgpool dx", outs[0], ec.avgpool_bwd_bound(dy, shape, bins, beta, old)))
    log(f"{case} usage={fmt(max(u))} overlapping_bins={overlap}")


# ------------------------------------------------------------------------------------------------ ReLU, axpby
@pytest.mark.parametrize("C", [8, 304])
def test_relu_and_axpby(log, C):
    shape = (2, 9, 11, C)
    M = 2 * 9 * 11
    case = f"relu/axpby C={C}"
    x, dy, old = rand_bf16(shape, 1), rand_bf16(shape, 2), rand_bf16(shape, 3)
    xd, dyd = place(x), place(dy)
    gy = guarded(shape)
    lib.call("seg_relu_fwd", lib.ptr(xd), ops.ld(xd), lib.ptr(gy.view), ops.ld(gy.view), M, C)
    settle(case, [gy])
    ec.check_exact(case, "relu y", gy.view, ec.relu_fwd_ref(x), ec.NAMES_NHWC)
    same_bits(case, "relu y (ops wrapper)", gy.view.contiguous(), ops.relu_fwd(xd))
    y = gy.view
    u = [0.0]
    for beta in (0.0, 1.0, 0.5):
        outs = []
        for _ in range(2):
            gx = guarded(shape, old if beta else None)
            ops.relu_bwd(dyd, y, gx.view, beta)
            settle(case, [gx])
            outs.append(gx.view.clone())
        same_bits(case, "relu dx", outs[0], outs[1])
        u.append(ec.check(f"{case} beta={beta}", "relu dx", outs[0], ec.relu_bwd_bound(dy, x.clamp_min(0), beta, old)))
        ga = guarded(shape, old)
        ops.axpby(xd, ga.view, beta)
        settle(case, [ga])
        u.append(ec.check(f"{case} beta={beta}", "axpby", ga.view, ec.axpby_bound(x, beta, old)))
    log(f"{case} usage={fmt(max(u))}")
