"""Counters -> metrics (seg_b200.metrics.counters_to_values / seg_metrics, used by seg_b200.eval_metrics and
FusedTrainStep.seg_metrics) against the reference's rules, without a GPU.

Counters are built on the CPU by oracle/metrics.py's restatement of utils/metrics.py from the inputs of
tests/golden/metrics.npz (whose outputs the reference produced) and accumulated per image, as a training or validation
loop accumulates them per batch."""
import os

import numpy as np
import pytest

from oracle import metrics as om
from seg_b200 import metrics

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")
CASES = (("c7", 7), ("c19", 19), ("c150", 150))


def counters(logits, target, K):
    """int64 [2 + 3K]: correct, labeled, inter[K], pred[K], lab[K] (the layout of seg_eval_metrics_nchw)."""
    predict = logits.argmax(1).astype(np.int64)
    t = target.astype(np.int64)
    lab = (t >= 0) & (t < K)
    p, tt = predict[lab], t[lab]
    inter = np.bincount(tt[p == tt], minlength=K)
    return np.concatenate([[int((p == tt).sum()), int(lab.sum())], inter, np.bincount(p, minlength=K)[:K],
                           np.bincount(tt, minlength=K)]).astype(np.int64)


def reference_seg_metrics(batches, K):
    """Trainer._reset_metrics / _update_seg_metrics / _get_seg_metrics (trainer.py:173-194) restated in float64 over the
    per-batch outputs of utils/metrics.py's eval_metrics."""
    tc = tl = 0.0
    ti, tu = np.zeros(K), np.zeros(K)
    for correct, labeled, inter, union in batches:
        tc, tl = tc + float(correct), tl + float(labeled)
        ti, tu = ti + inter.astype(np.float64), tu + union.astype(np.float64)
    pix = 1.0 * tc / (np.spacing(1) + tl)
    iou = 1.0 * ti / (np.spacing(1) + tu)
    return {"Pixel_Accuracy": np.round(pix, 3), "Mean_IoU": np.round(iou.mean(), 3),
            "Class_IoU": dict(zip(range(K), np.round(iou, 3)))}


@pytest.mark.parametrize("tag,K", CASES)
def test_counters_to_values_match_reference_golden(tag, K):
    g = np.load(GOLD)
    c, lab, inter, union = metrics.counters_to_values(counters(g[f"{tag}/logits"], g[f"{tag}/target"], K), K)
    assert c == int(g[f"{tag}/correct"]) and lab == int(g[f"{tag}/labeled"])
    assert np.array_equal(inter.astype(np.float32), g[f"{tag}/inter"])
    assert np.array_equal(union.astype(np.float32), g[f"{tag}/union"])


@pytest.mark.parametrize("tag,K", CASES)
def test_seg_metrics_equal_trainer_restatement(tag, K):
    g = np.load(GOLD)
    logits, target = g[f"{tag}/logits"], g[f"{tag}/target"]
    total = np.zeros(2 + 3 * K, dtype=np.int64)
    batches = []
    for n in range(logits.shape[0]):  # one image per batch: the counters are summed, as the device vector is
        total += counters(logits[n:n + 1], target[n:n + 1], K)
        batches.append(om.eval_metrics(logits[n:n + 1], target[n:n + 1], K))
    got, want = metrics.seg_metrics(total, K), reference_seg_metrics(batches, K)
    assert got["Pixel_Accuracy"] == want["Pixel_Accuracy"] and got["Mean_IoU"] == want["Mean_IoU"]
    assert got["Class_IoU"] == want["Class_IoU"]
    assert list(got) == ["Pixel_Accuracy", "Mean_IoU", "Class_IoU"]


def test_empty_counters_give_zero_metrics():
    got = metrics.seg_metrics(np.zeros(2 + 3 * 4, dtype=np.int64), 4)
    assert got["Pixel_Accuracy"] == 0.0 and got["Mean_IoU"] == 0.0 and list(got["Class_IoU"].values()) == [0.0] * 4


def test_exact_totals_past_float32_precision():
    """The reference sums each batch's float32 inter / union into float32 running totals (trainer.py:180-184); past 2**24
    pixels of a class they round.  The counters are exact int64.  Class 0: one batch of 2**24 correctly predicted pixels,
    then 2**20 batches with one correct and one wrong pixel each (inter + 1, union + 2 per batch)."""
    nb = 1 << 20
    inter_b = np.concatenate([[2.0 ** 24], np.ones(nb)]).astype(np.float32)
    union_b = np.concatenate([[2.0 ** 24], np.full(nb, 2.0)]).astype(np.float32)
    ref_inter = np.add.accumulate(inter_b, dtype=np.float32)[-1]  # sequential float32 sums, as the trainer's loop does
    ref_union = np.add.accumulate(union_b, dtype=np.float32)[-1]
    assert ref_inter == 2.0 ** 24  # every +1 after 2**24 rounds away
    ref_iou = np.round(ref_inter / (np.spacing(1) + ref_union), 3)
    K = 2
    inter, lab = (1 << 24) + nb, (1 << 24) + 2 * nb
    c = np.zeros(2 + 3 * K, dtype=np.int64)
    c[0], c[1] = inter, lab
    c[2], c[2 + K], c[2 + 2 * K] = inter, inter, lab  # inter, pred, lab of class 0: union = lab
    got = metrics.seg_metrics(c, K)
    assert got["Class_IoU"][0] == np.round(17 / 18, 3) == 0.944
    assert ref_iou == 0.889
