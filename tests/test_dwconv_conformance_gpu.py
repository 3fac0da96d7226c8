"""Conformance sweep of the depthwise 3x3 kernels (seg_dwconv.cu: forward with BatchNorm statistics, data gradient,
weight gradient, and the weight packing).

Every case is checked element by element against a float64 reference with the bounds of tests/dwconv_check.py, reads
its inputs from channel slices whose neighbouring channels hold NaN sentinels, writes into guarded buffers (sentinel
guard channels on both sides of the slice, a multiple of 8 before it, and a trailing guard image, which must come back
bit for bit; the output starts as the sentinel whenever beta = 0, so an element the kernel never wrote is caught), and
runs twice: outputs, statistics and weight gradients must be bit-identical between the runs (the cross-block sums are
exact fp64).  Each case appends its bound usage to gpu_out_dir/dwconv_conformance.txt.

The schedule cases are sized from the SM count at run time: dw_grid caps the grid at SMs * 6 blocks (forward, data
gradient) or SMs * 4 (weight gradient), two rows per thread until then; the cases put M just below, at and just above
the point where the cap is reached, and one case makes every thread stride many rows."""
import math
import os

import pytest
import torch

import dwconv_check as dc

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import ops

DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32
BETAS = (0.0, 0.5, 1.0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "dwconv_conformance.txt"), "a")
    f.write(f"# {torch.cuda.get_device_name(0)} sms={sms()}\n")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def place(t, lead=dc.GUARD):
    """A bf16 NHWC device tensor holding t in a channel slice at offset `lead` (a multiple of 8) of a wider buffer whose
    other channels hold the sentinel (a kernel reading outside the slice produces NaNs)."""
    N, H, W, C = t.shape
    buf = dc.sentinel_fill(torch.empty(N, H, W, lead + C + dc.GUARD, dtype=BF16, device=DEV))
    buf[..., lead:lead + C] = t.to(DEV, BF16)
    return buf[..., lead:lead + C]


def fmt(u):
    return f"{u:.4f}"


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def grid_note(M, C, blocks_per_sm):
    gx, gy, rp = dc.dw_grid(M, C, sms(), blocks_per_sm)
    return f" grid={gx}x{gy} rows_par={rp} rows_per_thread={-(-M // (gx * rp))}"


# ------------------------------------------------------------------------------------------------ runners
def run_fwd(log, case, x, w9, stride, pad, dil, lead=dc.GUARD):
    N, H, W, C = x.shape
    P, Q = dc.outsz(H, stride, pad, dil), dc.outsz(W, stride, pad, dil)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    xin, w9d = place(x), w9.float().to(DEV)
    runs = []
    for _ in range(2):
        g = dc.Guarded(N, P, Q, C, BF16, lead=lead, device=DEV)
        st = ops.new_stats(C, DEV)
        ops.dwconv_fwd(xin, w9d, stride, pad, dil, out=g.view, stats=st)
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        dc.check_written(case, g.view)
        runs.append((g.view.clone(), st.clone()))
    (y, st), (y2, st2) = runs
    assert torch.equal(bits(y), bits(y2)), f"{case}: output not bit-reproducible"
    assert torch.equal(st, st2), f"{case}: statistics not bit-reproducible"
    usage = dc.check_fprop(case, y, b)
    M = N * P * Q
    su = dc.check_stats(case, st, y.reshape(M, C), dc.stat_chain_dw(M, C, sms()))
    log(f"fwd {case} usage={fmt(usage)} stats_usage={fmt(su)}" + grid_note(M, C, dc.DW_BLOCKS_PER_SM))
    return max(usage, su)


def run_dgrad(log, case, dy, w9, x_shape, stride, pad, dil, beta=0.0, seed=0, lead=dc.GUARD):
    N, H, W, C = x_shape
    old = dc.make_x(N, H, W, C, seed + 200) if beta != 0.0 else None
    b = dc.dgrad_ref(dy, w9, x_shape, stride, pad, dil, beta=beta, old=old)
    dyin, w9d = place(dy), w9.float().to(DEV)
    runs = []
    for _ in range(2):
        g = dc.Guarded(N, H, W, C, BF16, lead=lead, device=DEV)
        if old is not None:
            g.view.copy_(old.to(DEV, BF16))
        ops.dwconv_bwd_data(dyin, w9d, x_shape, stride, pad, dil, out=g.view, beta=beta)
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        dc.check_written(case, g.view)
        runs.append(g.view.clone())
    assert torch.equal(bits(runs[0]), bits(runs[1])), f"{case}: dx not bit-reproducible"
    usage = dc.check_dgrad(case, runs[0], b)
    log(f"bwd_data {case} beta={beta} usage={fmt(usage)}" + grid_note(N * H * W, C, dc.DW_BLOCKS_PER_SM))
    return usage


def run_wgrad(log, case, dy, x, stride, pad, dil, beta=0.0, seed=0):
    """dw9 starts as random fp32 values (beta != 0) or as the sentinel (beta = 0: it must be overwritten, not read)."""
    N, H, W, C = x.shape
    M = dy.shape[0] * dy.shape[1] * dy.shape[2]
    chain = dc.wgrad_chain(M, C, sms())
    assert chain <= dc.LARGEST_DW_WGRAD_CHAIN and M <= dc.LARGEST_DW_WGRAD_PIXELS, (case, chain, M)
    old = dc.make_w9(C, seed + 300) if beta != 0.0 else None
    b = dc.wgrad_ref(dy, x, stride, pad, dil, chain, beta=beta, old=old)
    dyin, xin = place(dy), place(x)
    runs = []
    for _ in range(2):
        f = dc.FlatGuarded((9, C), F32, device=DEV)
        if old is not None:
            f.view.copy_(old.float())
        ops.dwconv_bwd_weight(dyin, xin, stride, pad, dil, out=f.view, beta=beta)
        torch.cuda.synchronize()
        dc.check_guards(case, f.buf, f.guard_mask())
        dc.check_written(case, f.view)
        runs.append(f.view.clone())
    assert torch.equal(bits(runs[0]), bits(runs[1])), f"{case}: dw9 not bit-reproducible"
    usage = dc.check_wgrad(case, runs[0], b)
    log(f"bwd_weight {case} beta={beta} chain={chain} usage={fmt(usage)}" + grid_note(M, C, dc.DW_WGRAD_BLOCKS_PER_SM))
    return usage


def run_all(log, case, shape, beta_d=0.0, beta_w=0.0, seed=0):
    N, H, W, C, stride, pad, dil = shape
    P, Q = dc.outsz(H, stride, pad, dil), dc.outsz(W, stride, pad, dil)
    x, w9, dy = dc.make_x(N, H, W, C, seed), dc.make_w9(C, seed + 10), dc.make_x(N, P, Q, C, seed + 20)
    run_fwd(log, case, x, w9, stride, pad, dil)
    run_dgrad(log, case, dy, w9, x.shape, stride, pad, dil, beta=beta_d, seed=seed)
    run_wgrad(log, case, dy, x, stride, pad, dil, beta=beta_w, seed=seed)


# ------------------------------------------------------------------------------------------------ 1. Xception layers
@pytest.mark.parametrize("i", range(len(dc.XCEPTION_CASES)), ids=["x".join(map(str, c)) for c in dc.XCEPTION_CASES])
def test_xception_layer(log, i):
    shape = dc.xception_shape(*dc.XCEPTION_CASES[i])
    N, H, W, C, stride, pad, dil = shape
    run_all(log, f"xception {N}x{H}x{W}x{C} s{stride} p{pad} d{dil}", shape, beta_d=BETAS[i % 3],
            beta_w=BETAS[(i + 1) % 3], seed=i)


# ------------------------------------------------------------------------------------------------ 2. lane layouts
# C: (rows_par, idle lanes of a block, gridDim.y)
LANES = {8: (256, 0, 1), 24: (85, 1, 1), 728: (2, 74, 1), 2048: (1, 0, 1), 2056: (1, 0, 2), 4104: (1, 0, 3)}


@pytest.mark.parametrize("C", list(LANES))
def test_lane_layout(log, C):
    """One channel group with the longest block reduction (C = 8), idle lanes (24, 728), GB = 256 exactly (2048), and
    gridDim.y = 2 and 3 with a ragged last column of blocks (2056, 4104)."""
    rows_par, idle, gy = LANES[C]
    G = C // 8
    GB = min(G, 256)
    assert dc.dw_grid(1000, C, sms())[1:] == (gy, rows_par)
    assert 256 - GB * rows_par == idle
    for k, shape in enumerate([(2, 9, 11, C, 1, 1, 1), (1, 10, 9, C, 2, 2, 2)]):
        run_all(log, f"lanes C={C} idle={idle} gy={gy} " + "x".join(map(str, shape)), shape,
                beta_d=BETAS[k + 1], beta_w=BETAS[2 - k], seed=40 + k)


# ------------------------------------------------------------------------------------------------ 3. geometry edges
# name: (N, H, W, C, stride, pad, dil)
EDGES = {
    "3x5_dil4": (1, 3, 5, 16, 1, 4, 4),        # map smaller than the dilation: only the centre row of taps in range
    "3x5_dil4_s2": (1, 3, 5, 16, 2, 4, 4),
    "1x1_dil1": (2, 1, 1, 24, 1, 1, 1),        # only the centre tap in range
    "1x1_dil2_s2": (1, 1, 1, 16, 2, 2, 2),
    "odd_s2": (2, 9, 11, 16, 2, 1, 1),
    "even_s2": (2, 10, 8, 16, 2, 1, 1),
    "odd_even_s2_dil2": (1, 9, 10, 32, 2, 2, 2),
    "pad0_s2": (1, 10, 9, 16, 2, 0, 1),        # the last row and column are reached by no tap
    "pad0_s1": (1, 7, 8, 16, 1, 0, 1),
    "pad0_dil2": (1, 9, 9, 16, 1, 0, 2),
    "pad2_dil1": (1, 7, 7, 16, 1, 2, 1),
    "pad1_dil2_s2": (1, 12, 12, 16, 2, 1, 2),
    "pad3_dil4": (1, 11, 10, 16, 1, 3, 4),
}


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("name", list(EDGES))
def test_geometry_edge(log, name, beta):
    """Input pixels that no tap reaches must still be written: beta * old, or 0."""
    run_all(log, f"edge {name}", EDGES[name], beta_d=beta, beta_w=beta, seed=60)


# ------------------------------------------------------------------------------------------------ 4. packing
@pytest.mark.parametrize("C", [8, 728, 2056])
def test_pack_and_unpack(log, C):
    g = torch.Generator().manual_seed(C)
    w = torch.randn(C, 1, 3, 3, generator=g)
    w9 = ops.dw_pack_weight(w.to(DEV))
    torch.cuda.synchronize()
    assert torch.equal(w9.cpu().view(torch.int32), dc.oihw_to_w9(w).contiguous().view(torch.int32)), f"C={C}: pack"
    g9 = dc.make_w9(C, C + 1)
    for beta in BETAS:
        case = f"unpack C={C} beta={beta}"
        old = dc.make_w9(C, C + 2).t().reshape(C, 1, 3, 3) if beta != 0.0 else None
        b = dc.unpack_ref(g9, beta, old)
        f = dc.FlatGuarded((C, 1, 3, 3), F32, device=DEV)
        if old is not None:
            f.view.copy_(old.float())
        ops.dw_unpack_wgrad(g9.float().to(DEV), f.view, beta)
        torch.cuda.synchronize()
        dc.check_guards(case, f.buf, f.guard_mask())
        dc.check_written(case, f.view)
        usage = dc.check_unpack(case, f.view, b)
        if beta == 0.0:
            dc.check_pack(case, dc.oihw_to_w9(f.view.cpu()), dc.w9_to_oihw(g9))
        log(f"{case} usage={fmt(usage)}")


# ------------------------------------------------------------------------------------------------ 5. schedules
def map_for_rows(lo, hi):
    """(1, H, W) with lo <= H W <= hi and H as close to W as the range allows (a single row if the range holds only
    primes)."""
    for H in range(math.isqrt(hi), 2, -1):
        W = -(-lo // H)
        if H * W <= hi:
            return 1, H, W
    return 1, 1, lo


def cap_point_rows(C, blocks_per_sm, point):
    """Row-count range where the uncapped gx = ceil(M / (2 rows_par)) is cap - 1 ("below"), cap ("at") or cap + 1
    ("above", the first capped grid: some threads take a third row)."""
    gx1, gy, rp = dc.dw_grid(1 << 40, C, sms(), blocks_per_sm)  # the cap
    want = {"below": gx1 - 1, "at": gx1, "above": gx1 + 1}[point]
    return 2 * rp * (want - 1) + 1, 2 * rp * want, gx1


@pytest.mark.parametrize("C", [64, 2056])
@pytest.mark.parametrize("point", ["below", "at", "above"])
def test_schedule_fwd_dgrad_cap(log, point, C):
    lo, hi, cap = cap_point_rows(C, dc.DW_BLOCKS_PER_SM, point)
    N, H, W = map_for_rows(lo, hi)
    M = N * H * W
    gx, _, rp = dc.dw_grid(M, C, sms())
    assert gx == (cap - 1 if point == "below" else cap)
    assert -(-M // (gx * rp)) == (3 if point == "above" else 2)
    shape = (N, H, W, C, 1, 1, 1)  # stride 1, "same" padding: the forward's and the data gradient's M are both H W
    x, w9, dy = dc.make_x(N, H, W, C, 70), dc.make_w9(C, 71), dc.make_x(N, H, W, C, 72)
    case = f"sched 6/SM {point} cap={cap} {N}x{H}x{W}x{C}"
    run_fwd(log, case, x, w9, 1, 1, 1)
    run_dgrad(log, case, dy, w9, shape[:4], 1, 1, 1, beta=1.0, seed=73)


@pytest.mark.parametrize("C", [64, 2056])
@pytest.mark.parametrize("point", ["below", "at", "above"])
def test_schedule_wgrad_cap(log, point, C):
    lo, hi, cap = cap_point_rows(C, dc.DW_WGRAD_BLOCKS_PER_SM, point)
    N, H, W = map_for_rows(lo, hi)
    M = N * H * W
    gx, _, rp = dc.dw_grid(M, C, sms(), dc.DW_WGRAD_BLOCKS_PER_SM)
    assert gx == (cap - 1 if point == "below" else cap)
    x, dy = dc.make_x(N, H, W, C, 80), dc.make_x(N, H, W, C, 81)
    run_wgrad(log, f"sched 4/SM {point} cap={cap} {N}x{H}x{W}x{C}", dy, x, 1, 1, 1, beta=0.5, seed=82)


def test_schedule_many_rows_per_thread(log):
    """The largest map the weight-gradient bound allows at C = 64 (32 row lanes): every thread of the capped grids
    strides over a dozen rows or more, in all three kernels."""
    C = 64
    gx, _, rp = dc.dw_grid(1 << 40, C, sms(), dc.DW_WGRAD_BLOCKS_PER_SM)
    rows = dc.LARGEST_DW_WGRAD_PIXELS // (gx * rp)
    N, H, W = map_for_rows(gx * rp * (rows - 1) + 1, gx * rp * rows)
    M = N * H * W
    assert dc.rows_per_thread(M, C, sms(), dc.DW_WGRAD_BLOCKS_PER_SM) == rows >= 12
    assert dc.rows_per_thread(M, C, sms(), dc.DW_BLOCKS_PER_SM) >= 8
    x, w9, dy = dc.make_x(N, H, W, C, 90), dc.make_w9(C, 91), dc.make_x(N, H, W, C, 92)
    case = f"sched many rows {N}x{H}x{W}x{C}"
    run_fwd(log, case, x, w9, 1, 1, 1)
    run_dgrad(log, case, dy, w9, (N, H, W, C), 1, 1, 1, beta=0.5, seed=93)
    run_wgrad(log, case, dy, x, 1, 1, 1, beta=1.0, seed=94)
