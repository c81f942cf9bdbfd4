"""The mAP protocol (oracle/ap_ref.py) on hand-computed cases, the annotation conversion the product shares with it, and
the evaluator's C-ABI symbols.  CPU only."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import ap_ref

C, K = 3, 12


def block(images, C=C, K=K):
    """images: per image a list of (class, score, (ymin, xmin, ymax, xmax)) in record order -> (dets, counts)."""
    rec = np.zeros((len(images), C, K), ap_ref.DET_DTYPE)
    counts = np.zeros((len(images), C), np.int32)
    for b, dets in enumerate(images):
        for cls, score, box in dets:
            k = counts[b, cls]
            rec[b, cls, k] = tuple(np.float32(v) for v in box) + (np.float32(score), k)
            counts[b, cls] += 1
    return rec.view(np.int32).reshape(len(images), C, K, 6), counts


def label(cls, box, hw):
    """A relative (class, x, y, w, h) row whose pixel box in an image of size hw is box = (ymin, xmin, ymax, xmax)."""
    H, W = hw
    y0, x0, y1, x1 = box
    return [cls, (x0 + x1) / 2 / W, (y0 + y1) / 2 / H, (x1 - x0) / W, (y1 - y0) / H]


def run(images, gts, thresholds=(0.5,), C=C):
    ev = ap_ref.ApRef(C, K, thresholds)
    d, c = block(images, C)
    ev.update(d, c, gts)
    return ev, ev.result()


HW = (100, 100)
GT0 = (10, 10, 50, 50)
FAR = (60, 60, 90, 90)


def test_fp_then_tp_gives_half():
    ev, r = run([[(0, 0.9, FAR), (0, 0.8, GT0)]], [([label(0, GT0, HW)], HW)])
    assert ev.tp_flags[0][0, :2].tolist() == [0, 1]
    assert r["ap"][0, 0] == 0.5
    assert r["npos"].tolist() == [1, 0, 0]


def test_duplicate_on_taken_gt_is_fp():
    ev, r = run([[(0, 0.9, GT0), (0, 0.8, (11, 10, 50, 50))]], [([label(0, GT0, HW)], HW)])
    assert ev.tp_flags[0][0, :2].tolist() == [1, 0]
    assert r["ap"][0, 0] == 1.0


def test_best_gt_taken_means_fp_even_if_another_gt_overlaps():
    g1, g2 = (0, 0, 10, 10), (0, 6, 10, 16)
    d = (0, 1, 10, 11)      # IoU 0.8182 with g1, 0.4286 with g2: the best box is g1 both times
    ev, r = run([[(0, 0.9, d), (0, 0.8, d)]], [([label(0, g1, (20, 20)), label(0, g2, (20, 20))], (20, 20))], (0.4,))
    assert ev.tp_flags[0][0, :2].tolist() == [1, 0]


def test_iou_exactly_threshold_matches_and_one_ulp_less_does_not():
    gt = (0, 0, 10, 10)
    on = (0, 0, 10, 5)
    below = (0, 0, 10, float(np.nextafter(np.float32(5), np.float32(0))))
    assert ap_ref.iou(np.float32(on), np.float32([gt]))[0] == np.float32(0.5)
    assert ap_ref.iou(np.float32(below), np.float32([gt]))[0] < np.float32(0.5)
    g = [([label(0, gt, (10, 10))], (10, 10))]
    assert run([[(0, 0.9, on)]], g)[0].tp_flags[0][0, 0] == 1
    assert run([[(0, 0.9, below)]], g)[0].tp_flags[0][0, 0] == 0


def test_iou_has_no_plus_one_and_normalises_corners():
    a = np.float32([0, 0, 4, 4])
    assert ap_ref.iou(a, np.float32([[2, 2, 6, 6]]))[0] == np.float32(4 / 28)
    assert ap_ref.iou(a, np.float32([[6, 6, 2, 2]]))[0] == np.float32(4 / 28)
    assert ap_ref.iou(a, np.float32([[4, 0, 8, 4]]))[0] == 0          # touching boxes
    assert ap_ref.iou(np.float32([1, 1, 1, 1]), np.float32([[1, 1, 1, 1]]))[0] == 0   # empty union


def test_detection_on_other_class_gt_is_fp():
    ev, r = run([[(1, 0.9, GT0)]], [([label(0, GT0, HW)], HW)])
    assert ev.tp_flags[0][1, 0] == 0
    assert r["ap"][0, 0] == 0.0          # class 0: ground truth, no detections
    assert r["ap"][0, 1] != r["ap"][0, 1]  # class 1: no ground truth -> NaN


def test_class_without_gt_is_nan_and_left_out_of_map():
    ev, r = run([[(0, 0.9, GT0), (2, 0.7, FAR)], [(0, 0.8, FAR)]], [([label(0, GT0, HW)], HW), (np.zeros((0, 5)), HW)])
    assert r["npos"].tolist() == [1, 0, 0]
    assert math.isnan(r["ap"][0, 1]) and math.isnan(r["ap"][0, 2]) and math.isnan(r["ap07"][2])
    assert ev.tp_flags[1][0, 0] == 0     # the image without ground truth: an FP
    assert r["ap"][0, 0] == 1.0          # TP ranked first, then the FP
    assert r["map"][0] == 1.0 and r["map07"] == 1.0


def test_equal_scores_across_images_rank_in_stream_order():
    g = ([label(0, GT0, HW)], HW)
    none = (np.zeros((0,)), HW)
    _, r = run([[(0, 0.5, FAR)], [(0, 0.5, GT0)]], [none, g])
    assert r["ap"][0, 0] == 0.5
    _, r = run([[(0, 0.5, GT0)], [(0, 0.5, FAR)]], [g, none])
    assert r["ap"][0, 0] == 1.0


def test_eleven_point_uses_the_arange_values():
    assert ap_ref.RECALL_POINTS[3] == 0.30000000000000004
    assert ap_ref.RECALL_POINTS[6] == 0.6000000000000001 and ap_ref.RECALL_POINTS[7] == 0.7000000000000001
    hw = (200, 200)
    gts = [(i * 15, 0, i * 15 + 10, 10) for i in range(10)]
    dets = [(0, 0.99 - 0.01 * i, gts[i]) for i in range(3)] + [(0, 0.9 - 0.01 * i, (150, 150, 160, 160 + i)) for i in range(5)]
    dets.append((0, 0.5, gts[3]))
    _, r = run([dets], [([label(0, g, hw) for g in gts], hw)])
    # rec = 3/10 (= 0.3 < 0.30000000000000004) does not reach t_3: max precision there is 4/9, not 1
    assert r["npos"][0] == 10
    assert r["ap07"][0] == pytest.approx((1 + 1 + 1 + 4 / 9 + 4 / 9) / 11, abs=1e-15)
    assert r["ap"][0, 0] == pytest.approx((3 + 4 / 9) / 10, abs=1e-15)


def test_all_point_equals_devkit_area():
    rng = np.random.default_rng(0)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        tp = rng.random(n) < rng.random()
        npos = int(tp.sum() + rng.integers(0, 5)) or 1
        assert ap_ref.average_precision(tp, npos)[0] == pytest.approx(ap_ref.voc_devkit_ap(tp, npos), abs=1e-12)


def test_thresholds_are_independent():
    d = (10, 10, 50, 40)        # IoU 0.75 with GT0
    ev, r = run([[(0, 0.9, d)]], [([label(0, GT0, HW)], HW)], (0.5, 0.75, 0.8))
    assert ev.tp_flags[0][0, 0] == 0b011
    assert r["ap"][:, 0].tolist() == [1.0, 1.0, 0.0]


def test_bad_records_raise():
    ev = ap_ref.ApRef(C, K)
    d, c = block([[(0, 0.9, GT0)]])
    c2 = c.copy()
    c2[0, 1] = K + 1
    with pytest.raises(ValueError):
        ev.update(d, c2, [(np.zeros((0, 5)), HW)])
    d2 = d.copy()
    d2[0, 0, 0, 4] = np.float32(np.nan).view(np.int32)
    with pytest.raises(ValueError):
        ev.update(d2, c, [(np.zeros((0, 5)), HW)])


def test_annotation_conversion():
    cls, box = ap_ref.gt_boxes([[1, 0.5, 0.25, 0.5, 0.5]], (100, 200), 20)
    assert cls.tolist() == [1] and box.dtype == np.float32
    assert box.tolist() == [[0.0, 50.0, 50.0, 150.0]]
    rng = np.random.default_rng(1)
    lab = np.concatenate([rng.integers(0, 20, (50, 1)), rng.random((50, 4))], 1)
    hw = (375, 500)
    _, b = ap_ref.gt_boxes(lab, hw, 20)
    x, y, w, h = lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4]
    want = np.float32(np.stack([(y - h / 2) * 375, (x - w / 2) * 500, (y + h / 2) * 375, (x + w / 2) * 500], 1))
    assert np.array_equal(b, want)
    from k210_yolo_framework_b200.evaluate import voc_gt_boxes
    packed = voc_gt_boxes(lab, hw, 20)
    assert np.array_equal(packed[:, 1:], b) and np.array_equal(packed[:, 0], lab[:, 0].astype(np.float32))
    assert voc_gt_boxes(np.zeros((0,)), hw, 20).shape == (0, 5)
    assert ap_ref.gt_boxes(np.zeros((0, 5)), hw, 20)[1].shape == (0, 4)


@pytest.mark.parametrize("labels", [[[20, 0.5, 0.5, 0.1, 0.1]], [[-1, 0.5, 0.5, 0.1, 0.1]], [[1.5, 0.5, 0.5, 0.1, 0.1]],
                                    [[float("nan"), 0.5, 0.5, 0.1, 0.1]], [[1, 0.5, 0.5, 0.1]], [1, 0.5, 0.5, 0.1, 0.1],
                                    np.zeros((0, 4)), np.zeros((1, 0)), np.zeros((2, 5, 1))])
def test_malformed_annotation_rows_raise(labels):
    from k210_yolo_framework_b200.evaluate import voc_gt_boxes
    with pytest.raises(ValueError):
        ap_ref.gt_boxes(labels, (10, 10), 20)
    with pytest.raises(ValueError):
        voc_gt_boxes(labels, (10, 10), 20)


def test_load_voc_annotations(tmp_path):
    from k210_yolo_framework_b200.evaluate import load_voc_annotations
    rows = np.empty((2, 3), object)
    rows[0] = ["a.jpg", np.array([[3.0, 0.5, 0.5, 0.2, 0.4]]), np.array([375, 500])]
    rows[1] = ["b.jpg", np.zeros((0, 5)), np.array([10, 20])]
    p = str(tmp_path / "ann.npy")
    np.save(p, rows)
    paths, labels, hw = load_voc_annotations(p)
    assert paths == ["a.jpg", "b.jpg"] and hw == [(375, 500), (10, 20)]
    assert labels[0].tolist() == [[3.0, 0.5, 0.5, 0.2, 0.4]] and labels[1].shape == (0, 5)


def test_ap_abi_symbols():
    from k210_yolo_framework_b200 import _lib
    src = open(os.path.join(ROOT, "include", "k210_yolo_b200.h")).read()
    names = ["k2y_ap_create", "k2y_ap_destroy", "k2y_ap_match", "k2y_ap_result", "k2y_ap_reset", "k2y_ap_tp_flags"]
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert re.search(rf"\b{n}\s*\(", src), n
        assert hasattr(lib, n) and n in _lib._SIGNATURES, n
