"""Worker of tests/test_losses_focal_weighted_gpu.py::test_two_gpu_global_batch_losses, launched as
`python -m torch.distributed.run --nproc-per-node 2 tests/losses_dp_worker.py OUT`: each rank takes half of a batch whose
halves have different valid-pixel counts, and the class-weighted and focal losses (the global-batch value, and the
gradient the engine's rank-averaged exchange expects) must equal one process computing the whole batch."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    out_path = sys.argv[1]
    from seg_b200 import launch
    rank, world = launch.init_data_parallel()
    import torch
    from seg_b200 import losses
    g = torch.Generator().manual_seed(77)
    C, ign = 19, 255
    z = torch.randn(4, C, 33, 37, generator=g) * 3
    t = torch.randint(0, C, (4, 33, 37), generator=g)
    t[0, :20] = ign  # unequal valid-pixel counts on the two ranks
    w = (torch.rand(C, generator=g) * 2).tolist()
    w[3] = 0.0
    crits = {"ce_w_mean": losses.CrossEntropyLoss2d(weight=w, ignore_index=ign),
             "ce_w_sum": losses.CrossEntropyLoss2d(weight=w, ignore_index=ign, reduction="sum"),
             "focal_mean": losses.FocalLoss(ignore_index=ign),
             "focal_alpha_sum": losses.FocalLoss(gamma=0.5, alpha=w, ignore_index=ign, size_average=False)}
    n = 4 // world
    half = slice(rank * n, rank * n + n)
    lines = []
    for name, crit in crits.items():
        x = z[half].clone().cuda().requires_grad_(True)
        loss = crit(x, t[half].clone().cuda())
        loss.backward()
        xf = z.clone().cuda().requires_grad_(True)
        ref = losses._CEFn.apply(xf, t.clone().cuda(), ign, False, crit.spec)  # one process, whole batch
        ref.backward()
        el = abs(float(loss) - float(ref)) / abs(float(ref))
        # the engine averages gradients over ranks, so a rank's gradient is world x its share of the global one
        ge = float((x.grad / world - xf.grad[half]).abs().max()) / float(xf.grad.abs().max())
        lines.append(f"rank {rank} {name}: loss {float(loss):.6f} one-GPU {float(ref):.6f} (rel {el:.1e}), grad {ge:.1e}")
        assert el <= 1e-5 and ge <= 1e-4, lines[-1]
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(lines) + "\nok\n")
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
