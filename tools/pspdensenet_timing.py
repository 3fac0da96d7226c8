"""Times one PSPDenseNet training step on the GPU with CUDA events, at the C2 shape: N x 3 x 473^2, 21 classes, densenet121
and densenet201 (--backbones), cross-entropy with ignore_index 255 on the main head plus 0.4 x the aux head's (trainer.py:
57-60), SGD (lr 0.01, momentum 0.9, weight decay 1e-4, the backbone group at lr / 10; base/base_trainer.py:46-57).

  fused      FusedTrainStep(model, cuda_graph=True).step(x, y)
  plugin     model.cuda_graphs(True); (CE(out) + 0.4 CE(aux)).backward(); torch.optim.SGD.step()  (trainer.py:55-71)
  reference  the unmodified models/pspnet.py PSPDenseNet (pretrained=False) from oracle/_ref/reference.zip, fp32 NCHW, cuDNN
             with cudnn.benchmark, utils.losses.CrossEntropyLoss2d, torch.optim.SGD
  kernels    (--kernels) the dense-block kernels per launch at the model's shapes, as GB/s of the bytes each must move: the
             table-reading BN apply (+ ReLU + bit mask) of the largest norm1 prefixes, the accumulating BN backward apply
             (beta_dx = 1, against the same launch at beta_dx = 0) and the 2x2 average pool forward / backward of transition1

    python tools/pspdensenet_timing.py [--batch 16] [--iters 3] [--rounds 3] [--legs fused,plugin,reference]
                                       [--backbones densenet121,densenet201] [--kernels] [--out FILE]

Each leg is built, warmed up and timed on its own (round medians), then freed, so that torch.cuda.max_memory_allocated
after its warm-up is the leg's own peak.  A leg that runs out of memory at the batch is reported as such.  Prints the
device name, power limit and max SM clock with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from loss_timing import device_info, timed  # noqa: E402

S, C = 473, 21


def sgd(model, lr=0.01):
    groups = [{"params": model.get_decoder_params()}, {"params": model.get_backbone_params(), "lr": lr * 0.1}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9, weight_decay=1e-4)


def fused_leg(backbone):
    import seg_b200
    from seg_b200.train import FusedTrainStep
    stepper = FusedTrainStep(seg_b200.PSPDenseNet(C, backbone=backbone, pretrained=False).cuda().train(), ignore_index=255,
                             cuda_graph=True)
    return lambda x, y: stepper.step(x, y)


def _plain_step(model, crit, opt):
    def step(x, y):
        opt.zero_grad()
        out, aux = model(x)
        (crit(out, y) + 0.4 * crit(aux, y)).backward()
        opt.step()
    return step


def plugin_leg(backbone):
    import seg_b200
    model = seg_b200.PSPDenseNet(C, backbone=backbone, pretrained=False).cuda().train().cuda_graphs(True, warmup=2)
    return _plain_step(model, seg_b200.CrossEntropyLoss2d(ignore_index=255), sgd(model))


def reference_leg(backbone):
    from bench import _import_reference_tree
    if _import_reference_tree() is None:
        raise SystemExit("pspdensenet_timing: oracle/_ref/reference.zip not built (build() packs it from a reference checkout)")
    import importlib
    from utils import losses
    Pm = importlib.import_module("models.pspnet")
    torch.backends.cudnn.benchmark = True
    model = Pm.PSPDenseNet(C, backbone=backbone, pretrained=False).cuda().train()
    return _plain_step(model, losses.CrossEntropyLoss2d(ignore_index=255), sgd(model))


def block_shapes(backbone, N):
    """(H, c0, width) of each dense block at an S x S input: stem 3x3 s2 unpadded, two unpadded 3x3, max-pool(3, 2, 1),
    transition1's 2x2 pool."""
    from seg_b200.nets import DENSENET_BLOCKS, GROWTH
    h = ((S - 3) // 2 + 1) - 4
    h = (h - 1) // 2 + 1
    out, c = [], 64
    for bi, n in enumerate(DENSENET_BLOCKS[backbone]):
        out.append((h, c, c + n * GROWTH))
        c = (c + n * GROWTH) // 2
        if bi == 0:
            h //= 2
    return out


def kernel_rows(backbone, N, iters):
    from seg_b200 import ops
    from seg_b200.nets import GROWTH
    rows = []

    def add(op, shape, fn, nbytes):
        ms = statistics.median(timed(fn, iters) for _ in range(5))
        r = {"op": op, "backbone": backbone, "shape": shape, "ms": round(ms, 4), "GB_per_s": round(nbytes / ms / 1e6, 1),
             "share_of_3350": round(nbytes / ms / 1e6 / 3350.0, 3)}
        rows.append(r)
        print(json.dumps(r))

    dev = "cuda"
    for bi, (H, c0, width) in enumerate(block_shapes(backbone, N)):
        M = N * H * H
        buf = torch.randn(N, H, H, width, device=dev).bfloat16()
        table = torch.zeros(2 * width, dtype=torch.float64, device=dev)
        ops.bn_stats(buf[..., :c0], stats=table[:2 * c0])
        for c in range(c0, width, GROWTH):
            ops.bn_stats(buf[..., c:c + GROWTH], stats=table[2 * c:2 * c + 2 * GROWTH])
        cin = width - GROWTH  # the block's last (widest) norm1
        x = buf[..., :cin]
        gamma, beta = torch.ones(cin, device=dev), torch.zeros(cin, device=dev)
        rm, rv = torch.zeros(cin, device=dev), torch.ones(cin, device=dev)
        mask = ops.relu_mask(x)
        out = torch.empty(N, H, H, cin, device=dev, dtype=torch.bfloat16)
        shape = f"block{bi + 1} last norm1 {N}x{H}x{H}x{cin} (pitch {width})"
        add("bn_apply_train table", shape,
            lambda: ops.bn_apply_train(x, table, M, gamma, beta, 1e-5, 0.1, 0, rm, rv, out=out, relu=True, mask=mask,
                                       table=(c0, GROWTH)),
            nbytes=4 * M * cin + M * cin / 8)
        a, save = ops.bn_apply_train(x, table, M, gamma, beta, 1e-5, 0.1, 0, rm, rv, out=out, relu=True, mask=mask,
                                     table=(c0, GROWTH))
        da = torch.randn_like(out)
        sums = ops.bn_bwd_reduce(da, a, x, save, relu=True, mask=mask)
        gbuf = torch.zeros(N, H, H, width, device=dev, dtype=torch.bfloat16)
        dx = gbuf[..., :cin]
        for beta_dx in (0.0, 1.0):
            add(f"bn_bwd_apply beta_dx={beta_dx:g}", shape,
                lambda: ops.bn_bwd_apply(da, a, x, save, gamma, sums, M, relu=True, dx=dx, mask=mask, beta_dx=beta_dx),
                nbytes=(6 if beta_dx else 4) * M * cin + M * cin / 8)
        if bi == 0:
            # transition1's pool: its conv output [N,H,H,c_next] -> slice 0 of block2's buffer
            cn = width // 2
            y = torch.randn(N, H, H, cn, device=dev).bfloat16()
            nxt = torch.empty(N, H // 2, H // 2, 2 * cn, device=dev, dtype=torch.bfloat16)
            add("avgpool2x2_fwd", f"{N}x{H}x{H}x{cn} -> slice", lambda: ops.avgpool2x2_fwd(y, out=nxt[..., :cn]),
                nbytes=2 * N * H * H * cn + 2 * N * (H // 2) ** 2 * cn)
            dy = nxt[..., :cn]
            gy = torch.empty_like(y)
            add("avgpool2x2_bwd", f"{N}x{H}x{H}x{cn}", lambda: ops.avgpool2x2_bwd(dy, tuple(y.shape), dx=gy),
                nbytes=2 * N * H * H * cn + 2 * N * (H // 2) ** 2 * cn)
        del buf, out, a, da, gbuf, mask
        torch.cuda.empty_cache()
    return rows


def run_leg(make, backbone, x, y, iters, rounds):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    fn = None
    try:
        torch.manual_seed(0)
        fn = make(backbone)
        for _ in range(3):  # graph capture (fused / plugin), cudnn.benchmark's algorithm search (reference)
            fn(x, y)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        ts = [timed(lambda: fn(x, y), iters) for _ in range(rounds)]
    except torch.OutOfMemoryError:
        return {"oom": True}
    finally:
        fn = None
        import gc
        gc.collect()
        torch.cuda.empty_cache()
    ms = statistics.median(ts)
    return {"ms_per_step": round(ms, 2), "min_ms": round(min(ts), 2), "max_ms": round(max(ts), 2),
            "img_per_s": round(x.shape[0] * 1000.0 / ms, 1), "peak_GiB": round(peak / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--legs", default="fused,plugin,reference")
    ap.add_argument("--backbones", default="densenet121,densenet201")
    ap.add_argument("--kernels", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pspdensenet_timing: needs a CUDA device")
    from seg_b200 import lib
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    N = a.batch
    results = {"device": name, "power_limit_max_sm_clock": power, "batch": N, "size": S, "classes": C, "iters": a.iters,
               "rounds": a.rounds, "runs": []}
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, 3, S, S, device="cuda", generator=g)
    y = torch.randint(0, C, (N, S, S), device="cuda", generator=g)
    y[:, :16] = 255
    makers = {"fused": fused_leg, "plugin": plugin_leg, "reference": reference_leg}
    for bb in a.backbones.split(","):
        kernels = kernel_rows(bb, N, 10) if a.kernels else []
        rows = []
        for leg in filter(None, a.legs.split(",")):
            r = {"leg": leg, "backbone": bb, **run_leg(makers[leg], bb, x, y, a.iters, a.rounds)}
            rows.append(r)
            if r.get("oom"):
                print(f"{bb} {leg:10s} {N}x3x{S}x{S}: out of memory")
            else:
                print(f"{bb} {leg:10s} {N}x3x{S}x{S} median {r['ms_per_step']:9.2f} ms/step (range {r['min_ms']:.2f}-"
                      f"{r['max_ms']:.2f}), {r['img_per_s']:7.1f} img/s, peak {r['peak_GiB']:.2f} GiB")
        results["runs"].append({"backbone": bb, "rows": rows, "kernels": kernels})
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
