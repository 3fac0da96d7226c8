"""Device implementation of the reference's test-time augmentation (seg_b200.inference: multi-scale + flip, sliding
window, label map) against the CPU oracle (oracle/inference.py, pinned to the reference by tests/golden/inference.npz)
and against the golden vectors themselves.  The stand-in network runs on the GPU on both sides, so the comparison
isolates what seg_data.cu computes: the image pyramid, flips, up-sampling, accumulation and the arg-max."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import data_check as dc
from oracle import inference as oi
from oracle import synth, weights

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import inference as di
    from seg_b200 import ops

if torch.cuda.is_available():  # the fp32 stand-in network must not run its convolutions in TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference.npz")
TOL = 2e-5  # fp32 accumulation over scales / windows against the reference's float64 numpy accumulation


def rel(a, b):
    return float(np.abs(a - b).max() / max(1e-12, np.abs(b).max()))


@pytest.mark.parametrize("tag", ["a", "b"])
def test_device_tta_matches_reference_golden(tag, gpu_out_dir):
    g = np.load(GOLD)
    C = int(g["num_classes"])
    model = oi.toy_model(C, seed=3)
    img = torch.from_numpy(g[f"{tag}/image"]).cuda()
    scales = [float(s) for s in g[f"{tag}/scales"]]
    got = {"ms": di.multi_scale_predict(model, img, scales, C, flip=False),
           "ms_flip": di.multi_scale_predict(model, img, scales, C, flip=True),
           "slide": di.sliding_predict(model, img, C, flip=False),
           "slide_flip": di.sliding_predict(model, img, C, flip=True)}
    for k, v in got.items():
        ref = g[f"{tag}/{k}"]
        e = rel(v.cpu().double().numpy(), ref)
        lab = di.predict_labels(v)
        # every score is within TOL max|ref| of the reference (asserted below), so a label may differ from the
        # reference's (inference.py:156) only where the top-two margin is within twice that
        acc = torch.full(ref.shape, TOL * float(np.abs(ref).max()), dtype=torch.float64)
        free = dc.check_tta_labels(f"inference {tag}/{k}", lab, torch.from_numpy(ref), acc)
        msg = f"[inference {tag}/{k}] scores relerr {e:.2e}  pixels without a clear label margin {free}"
        print(msg)
        with open(os.path.join(gpu_out_dir, "model_parity.txt"), "a") as f:
            f.write(msg + "\n")
        assert e < TOL, msg


def test_engine_model_multi_scale_shapes_and_agreement(gpu_out_dir):
    """The real engine model under test-time augmentation: variable input sizes (scales 0.75 .. 1.5 of 97 x 129) run through
    the same kernels, and the device TTA agrees with the oracle TTA wrapped around the SAME model (bf16 noise only)."""
    nc = 7
    sd = weights.deeplab_resnet_state_dict(nc, "resnet14", seed=4, randomize_bn=True)
    m = seg_b200.DeepLab(nc, backbone="resnet14", output_stride=16)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    x, _ = synth.make_batch(1, 97, 129, nc, 255, seed=9400)
    scales = [0.75, 1.0, 1.5]
    dev = di.multi_scale_predict(m, x.cuda(), scales, nc, flip=True)
    assert dev.shape == (nc, 97, 129) and torch.isfinite(dev).all()
    with torch.no_grad():
        ref = oi.multi_scale_predict(lambda t: m(t.cuda()), x, scales, nc, torch.device("cuda"), flip=True)
    e = rel(dev.cpu().double().numpy(), ref)
    agree = float((di.predict_labels(dev).cpu().numpy() == ref.argmax(0)).mean())
    msg = f"[inference engine-model] multi-scale+flip scores relerr {e:.2e} label agreement {agree:.4f}"
    print(msg)
    with open(os.path.join(gpu_out_dir, "model_parity.txt"), "a") as f:
        f.write(msg + "\n")
    assert e < 5e-2 and agree > 0.9, msg  # random-init logits have small margins; the scores are the sharp check
    sl = di.sliding_predict(m, x.cuda(), nc, flip=True)
    assert sl.shape == (nc, 97, 129) and torch.isfinite(sl).all()
