"""COCO detection evaluation (pycocotools ``COCOeval(gt, dt, "bbox")``), restated in Python — TEST INFRASTRUCTURE ONLY.

This module defines the protocol that ``k210_yolo_framework_b200.evaluate.CocoEval`` (csrc/evaluate.cu) implements on the
GPU; tests/test_coco_oracle.py pins it on hand-computed cases and tests/test_gpu_coco.py compares the kernels against it.
It restates COCOeval's bbox path as plain loops: ``_prepare``, ``computeIoU`` (maskApi.c ``bbIou``), ``evaluateImg``,
``accumulate`` and ``summarize``, with COCOeval's default parameters and no other mode.

Ground truth: a COCO instances dict.  Image ids and category ids are sorted; every listed image counts.  Within one
(image, category) the annotations keep their file order.  An annotation's ``ignore`` flag is its ``iscrowd``; in area
range [lo, hi] it is also ignored when ``area < lo`` or ``area > hi`` (the ``area`` field, not w * h).

Detections: a results list as ``COCO.loadRes`` reads it: ``id`` = position + 1, ``area`` = w * h, never crowd.  The
pipeline's records (ymin, xmin, ymax, xmax) float32 become ``x = xmin``, ``y = ymin``, ``w = xmax - xmin``,
``h = ymax - ymin``, the subtractions in float64 on the float32 values (``records_to_results``).

IoU (bbIou, float64): ``iw = min(xd + wd, xg + wg) - max(xd, xg)``, 0 if ``iw <= 0``; ``ih`` likewise;
``i = iw * ih``; ``u = area_d`` for a crowd box, else ``area_d + wg * hg - i``; IoU ``i / u``.

Matching, per (image, category, area range, threshold t): the ground truth stably sorted non-ignored first; each of
the first 100 detections (score descending, stable) walks it from ``best = min(t, 1 - 1e-10)``: skip a taken box unless
crowd, stop at the first ignored box once a non-ignored one matched, skip IoU < best, else the box becomes the match and
best its IoU (so the later of equal IoUs wins).  A matched detection takes the box's ignore flag; an unmatched one outside
the area range is ignored.

Accumulate, per (category, area range, maxDet): the detections with per-image rank < maxDet over all images, ranked by
score with a stable mergesort of their concatenation in sorted image-id order.  ``npig`` = non-ignored ground truth;
-1 stays when it is 0.  ``tp`` / ``fp`` cumulative sums of (matched, not ignored) / (unmatched, not ignored);
``rc = tp / npig``; ``pr = tp / (fp + tp + spacing(1))`` then its suffix maximum; recall ``rc[-1]`` (0 without
detections); precision at recall point r: ``pr[searchsorted(rc, r, "left")]``, 0 past the end.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, List, Sequence

import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
DET_DTYPE = np.dtype([("ymin", "<f4"), ("xmin", "<f4"), ("ymax", "<f4"), ("xmax", "<f4"), ("score", "<f4"),
                      ("index", "<i4")])


def _fmin(a, b):
    return float(np.fmin(a, b))


def _fmax(a, b):
    return float(np.fmax(a, b))


def bb_iou(d: Sequence, g: Sequence, iscrowd: Sequence) -> np.ndarray:
    """maskApi.c bbIou: IoU [len(d), len(g)] of (x, y, w, h) boxes, float64, crowd boxes against the detection's area."""
    out = np.zeros((len(d), len(g)))
    with np.errstate(divide="ignore", invalid="ignore"):
        for gi, G in enumerate(g):
            ga = G[2] * G[3]
            for di, D in enumerate(d):
                da = D[2] * D[3]
                w = _fmin(D[2] + D[0], G[2] + G[0]) - _fmax(D[0], G[0])
                if w <= 0:
                    continue
                h = _fmin(D[3] + D[1], G[3] + G[1]) - _fmax(D[1], G[1])
                if h <= 0:
                    continue
                i = w * h
                u = da if iscrowd[gi] else da + ga - i
                out[di, gi] = np.float64(i) / np.float64(u)
    return out


def match_literal(ious: np.ndarray, gt_ignore: Sequence, iscrowd: Sequence, t: float) -> List[int]:
    """evaluateImg's loop at one threshold: the matched ground-truth index (in the given, ignore-sorted order) of each
    detection, -1 for none.  ious [D, G]."""
    G = len(gt_ignore)
    gtm = np.zeros(G)
    out = []
    for dind in range(ious.shape[0]):
        iou = min([t, 1 - 1e-10])
        m = -1
        for gind in range(G):
            if gtm[gind] > 0 and not iscrowd[gind]:
                continue
            if m > -1 and gt_ignore[m] == 0 and gt_ignore[gind] == 1:
                break
            if ious[dind, gind] < iou:
                continue
            iou = ious[dind, gind]
            m = gind
        if m > -1:
            gtm[m] = dind + 1
        out.append(m)
    return out


def match_two_tier(ious: np.ndarray, gt_ignore: Sequence, iscrowd: Sequence, t: float) -> List[int]:
    """The same matches as ``match_literal``, as a two-tier arg-max: the last index of the highest IoU >= min(t, 1 - 1e-10)
    among the available non-ignored boxes, else the same among the available ignored boxes."""
    G = len(gt_ignore)
    taken = np.zeros(G, bool)
    out = []
    for dind in range(ious.shape[0]):
        m = -1
        for tier in (0, 1):
            best = min(t, 1 - 1e-10)
            for g in range(G):
                if gt_ignore[g] != tier or (taken[g] and not iscrowd[g]) or ious[dind, g] < best:
                    continue
                best, m = ious[dind, g], g
            if m > -1:
                break
        if m > -1:
            taken[m] = True
        out.append(m)
    return out


def records_to_results(dets, counts, image_ids: Sequence[int], category_ids: Sequence[int]) -> List[dict]:
    """The COCO results list of record blocks dets int32 [N, C, K, 6] / counts [N, C]: per image, class and record."""
    d = np.ascontiguousarray(np.asarray(dets, np.int32)).view(DET_DTYPE)[..., 0]
    out = []
    for b, img in enumerate(image_ids):
        for c, cat in enumerate(category_ids):
            for r in d[b, c, :int(counts[b, c])]:
                x, y = float(r["xmin"]), float(r["ymin"])
                out.append({"image_id": int(img), "category_id": int(cat),
                            "bbox": [x, y, float(r["xmax"]) - x, float(r["ymax"]) - y], "score": float(r["score"])})
    return out


class CocoRef:
    """COCOeval over one instances dict; ``evaluate(results)`` returns ``{"precision", "recall", "stats"}``."""

    def __init__(self, dataset: dict):
        self.img_ids = sorted(np.unique([im["id"] for im in dataset["images"]]).tolist())
        self.cat_ids = sorted(np.unique([c["id"] for c in dataset["categories"]]).tolist())
        self.gts: Dict[tuple, List[dict]] = defaultdict(list)
        for ann in dataset["annotations"]:
            g = dict(ann)
            g["ignore"] = "iscrowd" in g and g["iscrowd"]
            self.gts[g["image_id"], g["category_id"]].append(g)

    def _load_res(self, results: Sequence[dict]) -> Dict[tuple, List[dict]]:
        known = set(self.img_ids)
        dts: Dict[tuple, List[dict]] = defaultdict(list)
        for i, ann in enumerate(results):
            if ann["image_id"] not in known:
                raise ValueError("Results do not correspond to current coco set")
            d = dict(ann)
            bb = d["bbox"]
            d["area"] = bb[2] * bb[3]
            d["id"] = i + 1
            d["iscrowd"] = 0
            dts[d["image_id"], d["category_id"]].append(d)
        return dts

    def _evaluate_img(self, gt, dt, ious, a_rng, max_det):
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g["_ignore"] = 1 if (g["ignore"] or (g["area"] < a_rng[0] or g["area"] > a_rng[1])) else 0
        gtind = np.argsort([g["_ignore"] for g in gt], kind="mergesort")
        gt = [gt[i] for i in gtind]
        dt = dt[:max_det]               # already score-sorted by computeIoU
        iscrowd = [int(o["iscrowd"]) for o in gt]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        dtm = np.zeros((T, D))
        gt_ig = np.array([g["_ignore"] for g in gt])
        dt_ig = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, m in enumerate(match_literal(ious, gt_ig, iscrowd, t)):
                    if m == -1:
                        continue
                    dt_ig[tind, dind] = gt_ig[m]
                    dtm[tind, dind] = gt[m]["id"]
        a = np.array([d["area"] < a_rng[0] or d["area"] > a_rng[1] for d in dt]).reshape((1, len(dt)))
        dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"dtMatches": dtm, "dtScores": [d["score"] for d in dt], "gtIgnore": gt_ig, "dtIgnore": dt_ig}

    def evaluate(self, results: Sequence[dict]) -> dict:
        dts = self._load_res(results)
        max_det = MAX_DETS[-1]
        evals = {}
        for c in self.cat_ids:
            for i in self.img_ids:
                gt, dt = self.gts.get((i, c), []), dts.get((i, c), [])
                if not gt and not dt:
                    continue
                inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
                dt = [dt[j] for j in inds][:max_det]
                ious = bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gt], [int(o["iscrowd"]) for o in gt]) \
                    if dt and gt else []
                for a, rng in enumerate(AREA_RNG):
                    evals[c, a, i] = self._evaluate_img(gt, dt, ious, rng, max_det)
        return self._accumulate(evals)

    def _accumulate(self, evals) -> dict:
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.cat_ids), len(AREA_RNG), len(MAX_DETS)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        for k, c in enumerate(self.cat_ids):
            for a in range(A):
                E = [evals.get((c, a, i)) for i in self.img_ids]
                E = [e for e in E if e is not None]
                if len(E) == 0:
                    continue
                for m, max_det in enumerate(MAX_DETS):
                    scores = np.concatenate([np.asarray(e["dtScores"][0:max_det], np.float64) for e in E])
                    inds = np.argsort(-scores, kind="mergesort")
                    dtm = np.concatenate([e["dtMatches"][:, 0:max_det] for e in E], axis=1)[:, inds]
                    dt_ig = np.concatenate([e["dtIgnore"][:, 0:max_det] for e in E], axis=1)[:, inds]
                    gt_ig = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gt_ig == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dt_ig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        for ri, pi in enumerate(np.searchsorted(rc, REC_THRS, side="left")):
                            if pi >= nd:
                                break
                            q[ri] = pr[pi]
                        precision[t, :, k, a, m] = np.array(q)
        stats, lines = summarize(precision, recall)
        return {"precision": precision, "recall": recall, "stats": stats, "lines": lines,
                "ap_per_class": ap_per_class(precision)}


def summarize(precision: np.ndarray, recall: np.ndarray):
    """COCOeval.summarize: (stats [12], the 12 printed lines)."""
    lines = []

    def _summarize(ap=1, iou_thr=None, area_rng="all", max_dets=100):
        i_str = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
        title = "Average Precision" if ap == 1 else "Average Recall"
        type_str = "(AP)" if ap == 1 else "(AR)"
        iou_str = "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1]) if iou_thr is None else "{:0.2f}".format(iou_thr)
        aind = [i for i, a in enumerate(AREA_LBL) if a == area_rng]
        mind = [i for i, m in enumerate(MAX_DETS) if m == max_dets]
        if ap == 1:
            s = precision
            if iou_thr is not None:
                s = s[np.where(iou_thr == IOU_THRS)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = recall
            if iou_thr is not None:
                s = s[np.where(iou_thr == IOU_THRS)[0]]
            s = s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        lines.append(i_str.format(title, type_str, iou_str, area_rng, max_dets, mean_s))
        return mean_s

    stats = np.zeros((12,))
    stats[0] = _summarize(1)
    stats[1] = _summarize(1, iou_thr=.5, max_dets=MAX_DETS[2])
    stats[2] = _summarize(1, iou_thr=.75, max_dets=MAX_DETS[2])
    stats[3] = _summarize(1, area_rng="small", max_dets=MAX_DETS[2])
    stats[4] = _summarize(1, area_rng="medium", max_dets=MAX_DETS[2])
    stats[5] = _summarize(1, area_rng="large", max_dets=MAX_DETS[2])
    stats[6] = _summarize(0, max_dets=MAX_DETS[0])
    stats[7] = _summarize(0, max_dets=MAX_DETS[1])
    stats[8] = _summarize(0, max_dets=MAX_DETS[2])
    stats[9] = _summarize(0, area_rng="small", max_dets=MAX_DETS[2])
    stats[10] = _summarize(0, area_rng="medium", max_dets=MAX_DETS[2])
    stats[11] = _summarize(0, area_rng="large", max_dets=MAX_DETS[2])
    return stats, lines


def ap_per_class(precision: np.ndarray) -> np.ndarray:
    """Per category: the mean of precision[:, :, c, all, 100] over the entries > -1 (NaN without any)."""
    out = np.full(precision.shape[2], np.nan)
    for c in range(precision.shape[2]):
        s = precision[:, :, c, 0, 2]
        if np.any(s > -1):
            out[c] = np.mean(s[s > -1])
    return out
