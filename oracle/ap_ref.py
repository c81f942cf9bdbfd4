"""Detection mAP on an annotated image list, restated in numpy — TEST INFRASTRUCTURE ONLY.

This module defines the evaluation protocol that ``k210_yolo_framework_b200.evaluate.DetectionAP`` (csrc/evaluate.cu)
implements on the GPU; tests/test_ap_oracle.py pins it on hand-computed cases and tests/test_gpu_ap.py compares the
kernels against it.

Ground truth: the rows ``make_voc_list.py`` writes, ``(path, labels [n, 5] = (class, x, y, w, h) relative to the image,
(H, W))``.  Each label becomes the pixel box ``(ymin, xmin, ymax, xmax) = ((y - h/2) H, (x - w/2) W, (y + h/2) H,
(x + w/2) W)``, computed in float64 and rounded once to float32: the corner order and frame of the detection records.
The labels ``voc_label.py`` writes carry no "difficult" flag, so every object counts; that is the one difference from
the VOC devkit, which ignores difficult objects.

IoU of two corner boxes, float32, every operation rounded to nearest: each box is normalised to (min, max) per axis
(fmin / fmax, as the NMS does), ``ih = max(0, min(ymax) - max(ymin))``, ``iw`` likewise, ``inter = ih * iw``,
``union = area_a + area_b - inter``, ``iou = inter / union`` if ``union > 0`` else 0.  There is no "+1 pixel" term.
A NaN IoU never matches.

Matching at threshold t (VOC rule): the detections of one (image, class) are walked in record order (score descending,
ties by index, as the NMS emits them).  Each takes the ground-truth box of its class in its image with the largest IoU
(ties: lowest index); if that IoU >= float32(t) and the box is not yet taken, the detection is a TP and the box is
taken, otherwise (including a taken best box) it is an FP.

Ranking: all detections of a class, over the whole evaluation, by score descending; ties keep stream order (image
order of ``update`` calls, then record order), i.e. ``np.argsort(-score, kind="stable")``.

AP per class, npos = ground-truth boxes of the class, float64: ``prec_r = cumTP_r / (r + 1)``, ``rec_r = cumTP_r / npos``,
``env_r = max_{r' >= r} prec_r'``.  All-point: ``AP = sum_{r TP} env_r / npos`` (the devkit's mrec / mpre area).
11-point (VOC 2007): the mean over ``t_k in np.arange(0.0, 1.1, 0.1)`` (exactly those float64 values) of
``max(prec_r : rec_r >= t_k)``, 0 where no rank qualifies.  ``npos == 0`` gives NaN, and the mAP averages the classes
with ``npos > 0``; a class with ground truth but no detections has AP 0.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

DET_DTYPE = np.dtype([("ymin", "<f4"), ("xmin", "<f4"), ("ymax", "<f4"), ("xmax", "<f4"), ("score", "<f4"),
                      ("index", "<i4")])
RECALL_POINTS = np.arange(0.0, 1.1, 0.1)


def gt_boxes(labels, hw, class_num: int) -> Tuple[np.ndarray, np.ndarray]:
    """(classes int64 [n], boxes float32 [n, 4] pixel (ymin, xmin, ymax, xmax)) of one annotation row."""
    lab = np.asarray(labels, dtype=np.float64)
    if lab.size == 0:
        if lab.shape not in ((0, 5), (0,)):
            raise ValueError(f"an empty label array must have shape (0, 5) or (0,), not {lab.shape}")
        return np.zeros(0, np.int64), np.zeros((0, 4), np.float32)
    if lab.ndim != 2 or lab.shape[1] != 5:
        raise ValueError(f"labels must be [n, 5] (class, x, y, w, h), not {lab.shape}")
    cls = lab[:, 0]
    if not np.all((cls == np.floor(cls)) & (cls >= 0) & (cls < class_num)):
        raise ValueError(f"class ids must be integers in [0, {class_num}); got {cls.tolist()}")
    H, W = (float(v) for v in np.asarray(hw, np.float64).reshape(2))
    x, y, w, h = lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4]
    boxes = np.stack([(y - h / 2) * H, (x - w / 2) * W, (y + h / 2) * H, (x + w / 2) * W], 1).astype(np.float32)
    return cls.astype(np.int64), boxes


def _norm(b: np.ndarray):
    b = np.asarray(b, np.float32)
    y0, x0, y1, x1 = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.fmin(y0, y1), np.fmin(x0, x1), np.fmax(y0, y1), np.fmax(x0, x1)


def iou(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """float32 IoU of box a [4] against boxes b [g, 4], in the kernel's operation order."""
    ay0, ax0, ay1, ax1 = _norm(a)
    by0, bx0, by1, bx1 = _norm(b)
    z = np.float32(0)
    area_a = (ay1 - ay0) * (ax1 - ax0)
    area_b = (by1 - by0) * (bx1 - bx0)
    ih = np.fmax(np.fmin(ay1, by1) - np.fmax(ay0, by0), z)
    iw = np.fmax(np.fmin(ax1, bx1) - np.fmax(ax0, bx0), z)
    inter = ih * iw
    union = (area_a + area_b) - inter
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(union > z, inter / np.where(union > z, union, np.float32(1)), z)
    return out.astype(np.float32)


def match(det_boxes: np.ndarray, gt: np.ndarray, thresholds: Sequence[float]) -> np.ndarray:
    """TP flags [k, T] of one (image, class): det_boxes [k, 4] in record order, gt [g, 4] of that class."""
    thr = np.asarray(thresholds, np.float32)
    tp = np.zeros((len(det_boxes), len(thr)), bool)
    if len(gt) == 0 or len(det_boxes) == 0:
        return tp
    ious = iou(np.asarray(det_boxes, np.float32)[:, None, :], np.asarray(gt, np.float32)[None, :, :])   # [k, g]
    ious = np.where(np.isnan(ious), np.float32(-1), ious)
    j = np.argmax(ious, 1)                       # the best box does not depend on which boxes are taken
    best = ious[np.arange(len(j)), j]
    for t in range(len(thr)):
        # walking the records in order, a box is taken by the first detection that reaches t on it; the later ones are FPs
        cand = np.nonzero(best >= thr[t])[0]
        _, first = np.unique(j[cand], return_index=True)
        tp[cand[first], t] = True
    return tp


def average_precision(tp: np.ndarray, npos: int) -> Tuple[float, float]:
    """(all-point AP, 11-point AP) of one class from its ranked TP flags."""
    if npos == 0:
        return float("nan"), float("nan")
    tp = np.asarray(tp, bool)
    if tp.size == 0:
        return 0.0, 0.0
    cum = np.cumsum(tp, dtype=np.int64)
    prec = cum / np.arange(1, len(tp) + 1, dtype=np.float64)
    rec = cum / np.float64(npos)
    env = np.maximum.accumulate(prec[::-1])[::-1]
    ap = float(env[tp].sum() / npos)
    pts = [float(prec[rec >= t].max()) if np.any(rec >= t) else 0.0 for t in RECALL_POINTS]
    return ap, sum(pts) / 11.0


def voc_devkit_ap(tp: np.ndarray, npos: int) -> float:
    """The VOC devkit's all-point formula (mrec / mpre envelope area), for checking ``average_precision``."""
    tp = np.asarray(tp, bool)
    cum = np.cumsum(tp)
    rec = cum / float(npos)
    prec = cum / np.arange(1, len(tp) + 1, dtype=np.float64)
    mrec = np.concatenate(([0.0], rec, [1.0]))
    mpre = np.concatenate(([0.0], prec, [0.0]))
    for i in range(len(mpre) - 1, 0, -1):
        mpre[i - 1] = max(mpre[i - 1], mpre[i])
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return float(np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1]))


class ApRef:
    """The evaluator, on the host: ``update`` with the record blocks the pipeline returns, ``result`` at the end."""

    def __init__(self, class_num: int, max_per_class: int, iou_thresholds: Sequence[float] = (0.5,)):
        self.C, self.K = int(class_num), int(max_per_class)
        self.thr = [float(t) for t in iou_thresholds]
        self.reset()

    def reset(self) -> None:
        self.npos = np.zeros(self.C, np.int64)
        self.scores: List[List[np.ndarray]] = [[] for _ in range(self.C)]
        self.tps: List[List[np.ndarray]] = [[] for _ in range(self.C)]
        self.tp_flags: List[np.ndarray] = []      # per image: uint16 [C, K], bit t = TP at threshold t

    def update(self, dets, counts, gt) -> None:
        """dets int32 [N, C, K, 6] (k2y_det records), counts int32 [N, C], gt: N (labels, (h, w)) pairs."""
        d = np.ascontiguousarray(np.asarray(dets, np.int32)).view(DET_DTYPE)[..., 0]
        cnt = np.asarray(counts, np.int64)
        if np.any(cnt < 0) or np.any(cnt > self.K):
            raise ValueError("a record count is outside [0, max_per_class]")
        bits = np.arange(len(self.thr), dtype=np.uint16)
        for b, (labels, hw) in enumerate(gt):
            gcls, gbox = gt_boxes(labels, hw, self.C)
            self.npos += np.bincount(gcls, minlength=self.C)
            flags = np.zeros((self.C, self.K), np.uint16)
            for c in range(self.C):
                n = int(cnt[b, c])
                if n == 0:
                    continue
                rec = d[b, c, :n]
                score = rec["score"]
                if np.any(np.isnan(score)) or np.any(np.signbit(score)):
                    raise ValueError("a record has a negative or NaN score")
                box = np.stack([rec["ymin"], rec["xmin"], rec["ymax"], rec["xmax"]], 1)
                tp = match(box, gbox[gcls == c], self.thr)
                flags[c, :n] = (tp.astype(np.uint16) << bits).sum(1)
                self.scores[c].append(score.copy())
                self.tps[c].append(tp)
            self.tp_flags.append(flags)

    def result(self) -> dict:
        T = len(self.thr)
        ap = np.zeros((T, self.C))
        ap07 = np.zeros(self.C)
        for c in range(self.C):
            s = np.concatenate(self.scores[c]) if self.scores[c] else np.zeros(0, np.float32)
            tp = np.concatenate(self.tps[c]) if self.tps[c] else np.zeros((0, T), bool)
            order = np.argsort(-s, kind="stable")
            for t in range(T):
                a, a07 = average_precision(tp[order, t], int(self.npos[c]))
                ap[t, c] = a
                if t == 0:
                    ap07[c] = a07
        valid = self.npos > 0
        mean = (lambda v: float(np.mean(v[valid])) if valid.any() else float("nan"))
        return {"ap": ap, "ap07": ap07, "npos": self.npos.copy(), "map": np.array([mean(ap[t]) for t in range(T)]),
                "map07": mean(ap07)}
