"""Worker of tests/test_fused_metrics_gpu.py::test_two_gpu_metrics_and_validation_loss, launched as
`python -m torch.distributed.run --nproc-per-node 2 tests/fused_metrics_dp_worker.py OUT`: each rank takes half of a batch
whose halves have different labeled-pixel counts.  FusedTrainStep(world=2, metrics=True) must give the validation loss
and seg_metrics() (training and validation) of one process running FusedTrainStep on the whole batch.

BatchNorm is frozen (running statistics, as in freeze_bn configs) and dropout is off, so an image's logits do not depend
on which rank computes it; the training metrics are those of the first step, before the ranks' updates could differ in
their last bits from the one-process update."""
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
    import seg_b200
    from oracle import synth, weights
    from seg_b200.train import FusedTrainStep

    C = 7
    x, y = synth.make_batch(4, 65, 65, C, 255, seed=9201)
    y[0, :20] = 255  # unequal labeled-pixel counts on the two ranks
    x, y = x.cuda(), y.cuda()
    n = 4 // world
    half = slice(rank * n, rank * n + n)

    def model():
        m = seg_b200.DeepLab(C, backbone="resnet14", pretrained=False, output_stride=16)
        m.load_state_dict(weights.deeplab_resnet_state_dict(C, "resnet14", seed=41, randomize_bn=True), strict=True)
        m.engine_dropout = False
        m = m.cuda().train()
        m.freeze_bn()
        return m

    dp = FusedTrainStep(model(), lr=0.005, world=world, metrics=True)
    one = FusedTrainStep(model(), lr=0.005, world=1, metrics=True)
    lines = []
    v_dp, v_one = float(dp.evaluate(x[half], y[half])), float(one.evaluate(x, y))
    lines.append(f"rank {rank} validation loss {v_dp:.7f} one-GPU {v_one:.7f}")
    assert abs(v_dp - v_one) <= 1e-6 * abs(v_one), lines[-1]
    for phase in ("validation", "training"):
        if phase == "training":
            dp.reset_metrics()
            one.reset_metrics()
            dp.step(x[half], y[half])
            one.step(x, y)
        got, want = dp.seg_metrics(), one.seg_metrics()
        lines.append(f"rank {rank} {phase}: pixel accuracy {got['Pixel_Accuracy']} one-GPU {want['Pixel_Accuracy']}, "
                     f"mIoU {got['Mean_IoU']} one-GPU {want['Mean_IoU']}")
        assert got == want, lines[-1]
    torch.distributed.barrier()
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(lines) + "\nok\n")
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
