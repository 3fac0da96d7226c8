#!/usr/bin/env python
"""Every forward and data-gradient convolution of the C3 training step (DeepLabV3+ / ResNet-101, 513 x 513 crops, batch
16, output stride 16), with the tiles each kernel plan launches for it.

    python tools/conv_shapes.py --count                 # the table for both plans, no GPU needed
    python tools/conv_shapes.py --time --iters 50       # also time every shape on the GPU (CUDA events)

Plans:
  onetile  : one 128 x BN tile per CTA, BN in {64, 128, 256}; the launch runs in ceil(CTAs / SMs) waves.
  pingpong : persistent grid of min(tiles, SMs) CTAs, 128 x BN tiles with BN in {64, 128}; a CTA runs ceil(tiles / grid)
             tiles one after the other (`rounds`).
`eff` = tiles / (rounds x SMs): the share of the SMs' tile slots that hold a tile.  `T128` = rounds x BN / 128, the
launch's length in units of one 128 x 128 tile's main loop, assuming a tile's time scales with its width.  `share` is the
launch's part of all fprop + dgrad FLOPs of the step.  Stride-2 data gradients are split into the four parity classes of
the input pixels, one launch each (a class that no tap reaches is a launch that writes zeros).
Timing (--time) runs each launch through the C ABI with rotating input buffers and prints TFLOP/s next to the card's name,
power limit and SM clock."""
import argparse
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-segmentation_b200"))

BATCH = 16
BM = 128


def c3_convs():
    """(name, count, H_in, C, K, ksize, stride, dil) of every conv with C % 8 == 0 (the stem's C = 3 runs elsewhere)."""
    L = []

    def add(name, h_in, c, k, ks, s=1, d=1, cnt=1):
        L.append((name, cnt, h_in, c, k, ks, s, d))
    add("l1.0.conv1", 129, 64, 64, 1)
    add("l1.conv1", 129, 256, 64, 1, cnt=2)
    add("l1.conv2", 129, 64, 64, 3, cnt=3)
    add("l1.conv3", 129, 64, 256, 1, cnt=3)
    add("l1.ds", 129, 64, 256, 1)
    add("l2.0.conv1", 129, 256, 128, 1)
    add("l2.0.conv2", 129, 128, 128, 3, s=2)
    add("l2.conv1", 65, 512, 128, 1, cnt=3)
    add("l2.conv2", 65, 128, 128, 3, cnt=3)
    add("l2.conv3", 65, 128, 512, 1, cnt=4)
    add("l2.ds", 129, 256, 512, 1, s=2)
    add("l3.0.conv1", 65, 512, 256, 1)
    add("l3.0.conv2", 65, 256, 256, 3, s=2)
    add("l3.conv1", 33, 1024, 256, 1, cnt=22)
    add("l3.conv2", 33, 256, 256, 3, cnt=22)
    add("l3.conv3", 33, 256, 1024, 1, cnt=23)
    add("l3.ds", 65, 512, 1024, 1, s=2)
    add("l4.0.conv1", 33, 1024, 512, 1)
    add("l4.conv1", 33, 2048, 512, 1, cnt=2)
    add("l4.conv2", 33, 512, 512, 3, d=2, cnt=3)
    add("l4.conv3", 33, 512, 2048, 1, cnt=3)
    add("l4.ds", 33, 1024, 2048, 1)
    add("aspp.1x1", 33, 2048, 256, 1)
    add("aspp.3x3", 33, 2048, 256, 3, d=6)   # d = 6, 12, 18: same work
    add("aspp.3x3", 33, 2048, 256, 3, d=12)
    add("aspp.3x3", 33, 2048, 256, 3, d=18)
    add("aspp.cat", 33, 1280, 256, 1)
    add("dec.conv1", 129, 256, 48, 1)
    add("dec.conv2", 129, 304, 256, 3)
    add("dec.conv3", 129, 256, 256, 3)
    add("dec.cls", 129, 256, 19, 1)
    return L


def pick_bn(plan, ncols):
    if ncols <= 64:
        return 64
    if plan == "pingpong" or ncols < 256:
        return 128
    return 256 if math.ceil(ncols / 256) * 256 - ncols < 128 else 128


def launches(sms):
    """One row per kernel launch: dict(name, kind, count, conv geometry, M, ncols, taps, kdepth, flops)."""
    rows = []
    for name, cnt, h, c, k, ks, s, d in c3_convs():
        pad = d * (ks - 1) // 2
        p = (h + 2 * pad - d * (ks - 1) - 1) // s + 1
        flops = 2.0 * BATCH * p * p * k * c * ks * ks
        geo = dict(name=name, count=cnt, H=h, C=c, K=k, ks=ks, stride=s, dil=d, pad=pad, P=p)
        rows.append(dict(geo, kind="fprop", M=BATCH * p * p, ncols=k, taps=ks * ks, kch=math.ceil(c / 64), flops=flops))
        # data gradient: one launch per parity class (py, px) of the input pixels
        for py in range(s):
            for px in range(s):
                hs, ws = (h - py + s - 1) // s, (h - px + s - 1) // s
                th = sum(1 for r in range(ks) if (py + pad - r * d) % s == 0)
                tw = sum(1 for q in range(ks) if (px + pad - q * d) % s == 0)
                taps = th * tw
                m = BATCH * hs * ws
                rows.append(dict(geo, kind="dgrad" if s == 1 else f"dgrad{py}{px}", M=m, ncols=c, taps=taps,
                                 kch=math.ceil(k / 64), flops=2.0 * m * c * k * taps))
    return rows


def plan_row(r, plan, sms):
    bn = pick_bn(plan, r["ncols"])
    mt = math.ceil(r["M"] / BM)
    tiles = mt * math.ceil(r["ncols"] / bn)
    ctas = tiles if plan == "onetile" else min(tiles, sms)
    rounds = math.ceil(tiles / ctas) if plan == "pingpong" else math.ceil(tiles / sms)
    return dict(bn=bn, mtiles=mt, tiles=tiles, ctas=ctas, rounds=rounds, eff=tiles / (rounds * sms),
                t128=rounds * bn / 128, kblocks=r["taps"] * r["kch"])


def count(sms):
    rows = launches(sms)
    total = sum(r["flops"] * r["count"] for r in rows)
    print(f"C3 fprop + dgrad: {len(rows)} distinct launches, {total / 1e12:.2f} TFLOP per step, {sms} SMs")
    print(f"{'layer':11s} {'kind':7s} {'cnt':>3s} {'M':>7s} {'cols':>5s} {'kblk':>4s} {'rowT':>5s} | "
          f"{'BN':>3s} {'CTAs':>5s} {'wav':>3s} {'eff':>4s} {'T128':>4s} | {'BN':>3s} {'tiles':>5s} {'grid':>4s} {'rnd':>3s} "
          f"{'eff':>4s} {'T128':>4s} | share")
    weff = {"onetile": 0.0, "pingpong": 0.0}
    for r in sorted(rows, key=lambda r: -r["flops"] * r["count"]):
        a, b = plan_row(r, "onetile", sms), plan_row(r, "pingpong", sms)
        share = r["flops"] * r["count"] / total
        weff["onetile"] += a["eff"] * share
        weff["pingpong"] += b["eff"] * share
        print(f"{r['name']:11s} {r['kind']:7s} {r['count']:3d} {r['M']:7d} {r['ncols']:5d} {a['kblocks']:4d} {a['mtiles']:5d} | "
              f"{a['bn']:3d} {a['ctas']:5d} {a['rounds']:3d} {a['eff']:.2f} {a['t128']:4.1f} | "
              f"{b['bn']:3d} {b['tiles']:5d} {b['ctas']:4d} {b['rounds']:3d} {b['eff']:.2f} {b['t128']:4.1f} | {share:.3f}")
    for plan in ("onetile", "pingpong"):
        print(f"{plan}: FLOP-weighted tile-slot efficiency {weff[plan]:.2f}")
    sel = [r for r in rows if plan_row(r, "onetile", sms)["mtiles"] > sms and plan_row(r, "onetile", sms)["ctas"] % sms
           and plan_row(r, "onetile", sms)["eff"] < 0.6]
    print(f"launches at < 0.6 one-tile wave efficiency with more row tiles than SMs: "
          f"{sum(r['flops'] * r['count'] for r in sel) / total:.2f} of the FLOPs")
    return rows


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def time_all(rows, iters, only):
    import torch
    from seg_b200 import lib, ops
    lib.require_device()
    print(f"GPU: {gpu_info()}  (name, power limit, max SM clock, SM clock)")
    seen = set()
    tot_ms = {}
    for r in rows:
        key = (r["H"], r["C"], r["K"], r["ks"], r["stride"], r["dil"], r["kind"][:5])
        if key in seen or (only and only not in r["name"]):
            continue
        seen.add(key)
        h, c, k, ks, s, d, pad, p = r["H"], r["C"], r["K"], r["ks"], r["stride"], r["dil"], r["pad"], r["P"]
        nbuf = 3
        g = torch.Generator(device="cuda").manual_seed(0)
        w = torch.randn(k, c, ks, ks, device="cuda", generator=g) / (c * ks * ks) ** 0.5
        wp = ops.pack_weight(w)
        if r["kind"] == "fprop":
            xs = [torch.randn(BATCH, h, h, c, device="cuda", generator=g).to(torch.bfloat16) for _ in range(nbuf)]
            ys = [torch.empty(BATCH, p, p, k, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]
            st = torch.zeros(2 * k, dtype=torch.float64, device="cuda")

            def one(i):
                st.zero_()
                ops.conv2d_fwd(xs[i % nbuf], wp, k, ks, ks, s, pad, d, out=ys[i % nbuf], stats=st)
            flops = r["flops"]
        else:  # the whole data gradient (every parity class of a strided conv)
            dys = [torch.randn(BATCH, p, p, k, device="cuda", generator=g).to(torch.bfloat16) for _ in range(nbuf)]
            dxs = [torch.empty(BATCH, h, h, c, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]

            def one(i):
                ops.conv2d_dgrad(dys[i % nbuf], wp, (BATCH, h, h, c), ks, ks, s, pad, d, out=dxs[i % nbuf])
            flops = sum(x["flops"] for x in rows if x["name"] == r["name"] and x["H"] == h and x["dil"] == d
                        and x["kind"].startswith("dgrad"))
        for i in range(5):
            one(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            one(i)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        kind = r["kind"][:5]
        tot_ms[kind] = tot_ms.get(kind, 0.0) + us * r["count"] / 1e3
        print(f"time {r['name']:11s} {kind:5s} N={BATCH} H={h} C={c} K={k} k={ks} s={s} d={d}: {us:9.2f} us/launch "
              f"{flops / us / 1e6:7.1f} TFLOP/s", flush=True)
    print("per step (count-weighted, fprop includes zeroing its statistics):",
          ", ".join(f"{k} {v:.2f} ms" for k, v in tot_ms.items()))
    print(f"GPU after timing: {gpu_info()}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--count", action="store_true", help="print the tile table (no GPU needed)")
    ap.add_argument("--time", action="store_true", help="time every distinct launch on the GPU")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--only", default=None, help="time only layers whose name contains this")
    a = ap.parse_args()
    rows = count(a.sms) if (a.count or not a.time) else launches(a.sms)
    if a.time:
        time_all(rows, a.iters, a.only)
