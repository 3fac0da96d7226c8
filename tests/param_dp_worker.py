"""Worker of tests/test_param_conformance_gpu.py::test_two_gpu_bucketed_backward_equals_single_exchange, launched as
`python -m torch.distributed.run --nproc-per-node 2 tests/param_dp_worker.py OUT`.

Two FusedTrainStep(world=2) trainers start from the same state and take two steps on the same batch halves: one
exchanges its gradients in ~0.5 MB buckets launched during the backward (bucket_mb=0.5, many buckets), the other in one
all-reduce after it (bucket_mb=0).  With two ranks every element is reduced by one commutative fp32 addition, so how the
buckets are cut cannot change the result: flat_grad, the parameters and the momentum must be bit-identical.  A bucket
whose all-reduce or unpack started before its last weight gradient was written would differ."""
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
    import torch.distributed as dist
    import seg_b200
    from oracle import synth, weights
    from seg_b200.train import FusedTrainStep

    sd = weights.deeplab_resnet_state_dict(7, "resnet14", seed=21, randomize_bn=True)
    x, y = synth.make_batch(4, 65, 65, 7, 255, seed=9301)
    half = slice(rank * 2, rank * 2 + 2)
    xd, yd = x[half].cuda(), y[half].cuda()
    steppers = []
    for bucket_mb in (0.5, 0.0):
        m = seg_b200.DeepLab(7, backbone="resnet14", pretrained=False, output_stride=16)
        m.load_state_dict(sd, strict=True)
        m.engine_dropout = False
        m = m.cuda().train()
        m.freeze_bn()
        st = FusedTrainStep(m, lr=0.01, world=world, bucket_mb=bucket_mb)
        for _ in range(2):
            st.step(xd, yd)
        steppers.append(st)
    torch.cuda.synchronize()
    a, b = steppers
    msgs = []
    if len(a.buckets) < 8:
        msgs.append(f"only {len(a.buckets)} buckets")
    if b.buckets:
        msgs.append("bucket_mb=0 made buckets")
    if not torch.equal(a.flat_grad, b.flat_grad):
        msgs.append(f"flat_grad differs in {int((a.flat_grad != b.flat_grad).sum())} elements")
    if not torch.equal(a.flat_mom, b.flat_mom):
        msgs.append("momentum differs")
    for i, (p, q) in enumerate(zip(a.params, b.params)):
        if not torch.equal(p, q):
            msgs.append(f"parameter {i} differs")
            break
    flag = torch.tensor([len(msgs)], device="cuda")
    dist.all_reduce(flag)
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(msgs) + f"\nbuckets={len(a.buckets)}\n" + ("ok" if int(flag) == 0 else "FAIL"))
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
