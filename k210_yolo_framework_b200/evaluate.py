"""Evaluation on the GPU.

``PrecisionRecall``: precision / recall of the confidence channel, as the reference's Keras metrics define them
(/root/reference/tools/custom.py:13-75 ``Yolo_Precision`` / ``Yolo_Recall``), counted by k2y_pr_counts.

``DetectionAP``: per-class AP and mAP of the detection records against annotated boxes (VOC matching rule, all-point and
VOC 2007 11-point AP, any set of IoU thresholds), matched, ranked and reduced by the k2y_ap_* kernels.  The protocol is
that of oracle/ap_ref.py: IoU without a "+1 pixel" term, and every object counts (the annotation lists carry no
"difficult" flag).  ``load_voc_annotations`` reads the lists make_voc_list.py writes.

``CocoEval``: what pycocotools' ``COCOeval(gt, dt, "bbox")`` computes with its default parameters (precision / recall
arrays and the 12 summary stats), matched, ranked and reduced by the k2y_coco_* kernels; the protocol is that of
oracle/coco_ref.py.  ``load_coco_annotations`` reads a COCO instances JSON file, ``coco_results`` writes the records as
a COCO results list and ``coco_summary`` prints the stats as COCOeval does.
"""
from __future__ import annotations

import ctypes
import json
from typing import List, NamedTuple, Sequence, Tuple

import numpy as np
import torch

from ._lib import check, lib, require_cuda

AP_STATUS = {1: "a record has a negative or NaN score", 2: "a record count is outside [0, max_per_class]",
             4: "an image has more ground-truth boxes than the match kernel was told"}


class PrecisionRecall:
    """Accumulates tp / fp / fn over batches of (label, prediction) head tensors ``[..., A, 5+C]`` or ``[..., A*(5+C)]``."""

    def __init__(self, class_num: int, threshold: float = 0.5, apply_sigmoid: bool = False, device=None):
        require_cuda()
        self.entry = 5 + int(class_num)
        self.threshold, self.apply_sigmoid = float(threshold), bool(apply_sigmoid)
        self.counts = torch.zeros(3, dtype=torch.int64, device=device or "cuda")

    def update(self, y_true: Sequence[torch.Tensor], y_pred: Sequence[torch.Tensor]) -> None:
        for t, p in zip(y_true, y_pred):
            if not (t.is_cuda and p.is_cuda and t.dtype == p.dtype == torch.float32 and t.is_contiguous() and p.is_contiguous()
                    and t.numel() == p.numel() and t.numel() % self.entry == 0):
                raise ValueError("expected contiguous CUDA float32 tensors of equal size, a multiple of 5 + class_num floats")
            st = torch.cuda.current_stream(t.device.index)
            check(lib.k2y_pr_counts(t.data_ptr(), p.data_ptr(), t.numel() // self.entry, self.entry, self.threshold,
                                    int(self.apply_sigmoid), self.counts.data_ptr(), ctypes.c_void_p(st.cuda_stream)))

    def result(self) -> Tuple[float, float]:
        tp, fp, fn = (int(v) for v in self.counts.cpu())
        return (tp / (tp + fp) if tp + fp else 0.0), (tp / (tp + fn) if tp + fn else 0.0)

    def reset(self) -> None:
        self.counts.zero_()


def load_voc_annotations(npy_path: str) -> Tuple[List[str], List[np.ndarray], List[Tuple[int, int]]]:
    """A make_voc_list.py list (rows ``(path, labels [n, 5] = (class, x, y, w, h) relative, (h, w))``) as
    ``(paths, labels, hw)``."""
    rows = np.load(npy_path, allow_pickle=True)
    paths, labels, hw = [], [], []
    for row in rows:
        if len(row) != 3:
            raise ValueError(f"{npy_path}: rows must be (path, labels, (h, w)), got {len(row)} fields")
        paths.append(str(row[0]))
        labels.append(np.asarray(row[1], np.float64))
        h, w = (int(v) for v in np.asarray(row[2]).reshape(2))
        hw.append((h, w))
    return paths, labels, hw


def voc_gt_boxes(labels, hw, class_num: int) -> np.ndarray:
    """One annotation row's labels ``[n, 5] (class, x, y, w, h)`` relative to an image of size ``hw = (H, W)`` as
    ``[n, 5]`` float32 ``(class, ymin, xmin, ymax, xmax)`` in image pixels: the corner order and frame of the detection
    records, computed in float64 and rounded once.  ``ValueError`` for a malformed array or a class outside [0, C)."""
    lab = np.asarray(labels, dtype=np.float64)
    if lab.size == 0:
        if lab.shape not in ((0, 5), (0,)):
            raise ValueError(f"an empty label array must have shape (0, 5) or (0,), not {lab.shape}")
        return np.zeros((0, 5), np.float32)
    if lab.ndim != 2 or lab.shape[1] != 5:
        raise ValueError(f"labels must be [n, 5] (class, x, y, w, h), not {lab.shape}")
    cls = lab[:, 0]
    if not np.all((cls == np.floor(cls)) & (cls >= 0) & (cls < class_num)):
        raise ValueError(f"class ids must be integers in [0, {class_num}); got {cls.tolist()}")
    H, W = (float(v) for v in np.asarray(hw, np.float64).reshape(2))
    x, y, w, h = lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4]
    return np.stack([cls, (y - h / 2) * H, (x - w / 2) * W, (y + h / 2) * H, (x + w / 2) * W], 1).astype(np.float32)


class DetectionAP:
    """Accumulates detection records and ground truth over ``update`` calls; ``result`` ranks and reduces on the GPU.

    ``iou_thresholds``: 1 to 16 matching thresholds in (0, 1]; the 11-point AP is reported at the first.  Every call runs on
    the current CUDA stream."""

    def __init__(self, class_num: int, max_per_class: int, iou_thresholds: Sequence[float] = (0.5,), device=None):
        require_cuda()
        self.C, self.K = int(class_num), int(max_per_class)
        self.thresholds = [float(t) for t in iou_thresholds]
        if not 1 <= len(self.thresholds) <= 16 or not all(0.0 < t <= 1.0 for t in self.thresholds):
            raise ValueError(f"1 to 16 IoU thresholds in (0, 1] are needed, got {self.thresholds}")
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device or "cuda")
        self.device = torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)
        thr = (ctypes.c_float * len(self.thresholds))(*self.thresholds)
        h = ctypes.c_void_p()
        check(lib.k2y_ap_create(self.C, self.K, thr, len(self.thresholds), self.device.index, ctypes.byref(h)))
        self._h = h

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def update(self, dets: torch.Tensor, counts: torch.Tensor, gt: Sequence) -> None:
        """dets int32 ``[N, C, K, 6]`` (dense per image) and counts int32 ``[N, C]`` as ``DetectionPipeline`` returns them:
        the device views of ``step_device`` or the pinned host views of ``collect``, strided per image.  gt: one
        ``(labels, (h, w))`` pair per image, the last two fields of an annotation row (``load_voc_annotations``).  Device
        records are read asynchronously on the current stream; host records have been copied when this returns."""
        n = len(gt)
        if (dets.dtype != torch.int32 or counts.dtype != torch.int32 or dets.dim() != 4 or counts.dim() != 2
                or tuple(dets.shape) != (n, self.C, self.K, 6) or tuple(counts.shape) != (n, self.C)
                or tuple(dets.stride()[1:]) != (self.K * 6, 6, 1) or counts.stride(1) != 1 or dets.is_cuda != counts.is_cuda):
            raise ValueError(f"expected int32 dets [{n}, {self.C}, {self.K}, 6] (dense per image) and counts [{n}, {self.C}] "
                             f"on one side of the bus, one per ground-truth entry; got {tuple(dets.shape)} / {tuple(counts.shape)}")
        if n == 0:
            return
        boxes = [voc_gt_boxes(labels, hw, self.C) for labels, hw in gt]
        sizes = np.array([len(b) for b in boxes], np.int64)
        off = np.zeros(n + 1, np.int64)
        np.cumsum(sizes, out=off[1:])
        with torch.cuda.device(self.device):
            if dets.is_cuda:
                if dets.device != self.device or counts.device != self.device:
                    raise ValueError(f"records on {dets.device}, evaluator on {self.device}")
            else:   # a blocking copy: the host views may be overwritten as soon as this returns
                dets, counts = dets.to(self.device), counts.to(self.device)
            packed = torch.from_numpy(np.concatenate(boxes + [np.zeros((1, 5), np.float32)])).to(self.device)
            offsets = torch.from_numpy(off).to(self.device)
            check(lib.k2y_ap_match(self._h, dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0), n,
                                   packed.data_ptr(), offsets.data_ptr(), int(sizes.max()), self._stream()))

    def result(self) -> dict:
        """``{"ap": [T, C], "ap07": [C], "npos": [C], "map": [T], "map07": float}``: all-point AP per threshold and class, the
        VOC 2007 11-point AP at the first threshold, ground-truth counts, and the means over the classes with ground
        truth (AP is NaN for the others).  ``ValueError`` if an update held an invalid record."""
        T, C = len(self.thresholds), self.C
        ap, ap07, npos = np.zeros((T, C)), np.zeros(C), np.zeros(C, np.int64)
        status = ctypes.c_uint()
        with torch.cuda.device(self.device):
            check(lib.k2y_ap_result(self._h, ap.ctypes.data, ap07.ctypes.data, npos.ctypes.data, ctypes.byref(status),
                                    self._stream()))
        if status.value:
            raise ValueError("DetectionAP: " + "; ".join(m for bit, m in AP_STATUS.items() if status.value & bit))
        valid = npos > 0
        mean = (lambda v: float(np.mean(v[valid])) if valid.any() else float("nan"))
        return {"ap": ap, "ap07": ap07, "npos": npos, "map": np.array([mean(ap[t]) for t in range(T)]), "map07": mean(ap07)}

    def tp_flags(self) -> np.ndarray:
        """uint16 ``[images, C, K]``: bit t of entry (image, class, k) is set when record k was a TP at threshold t."""
        n = ctypes.c_longlong()
        check(lib.k2y_ap_tp_flags(self._h, None, 0, ctypes.byref(n), self._stream()))
        out = np.zeros((n.value, self.C, self.K), np.uint16)
        with torch.cuda.device(self.device):
            check(lib.k2y_ap_tp_flags(self._h, out.ctypes.data, out.size, ctypes.byref(n), self._stream()))
        return out

    def reset(self) -> None:
        with torch.cuda.device(self.device):
            check(lib.k2y_ap_reset(self._h, self._stream()))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.k2y_ap_destroy(h)
            self._h = None


COCO_STATUS = {1: "a record has a negative or NaN score", 2: "a record count is outside [0, max_per_class]",
               4: "an image position is outside [0, images)", 8: "an image was given twice since the last reset"}
# COCOeval's default parameters, exactly its np.linspace values
COCO_IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
COCO_REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
COCO_MAX_DETS = (1, 10, 100)
COCO_AREA_LBL = ("all", "small", "medium", "large")


class CocoGroundTruth(NamedTuple):
    """The annotations of a COCO instances file, packed for ``CocoEval``: rows float64 [n, 7] (class index, x, y, w, h,
    area, iscrowd), image i's (in sorted image-id order, file order within) at rows [offsets[i], offsets[i + 1])."""
    rows: np.ndarray
    offsets: np.ndarray
    category_ids: Tuple[int, ...]


def load_coco_annotations(json_path: str):
    """``(images, category_ids, gt)`` of a COCO instances JSON file: images as ``(id, file_name, (h, w))`` sorted by id
    (all of them, with annotations or not), the sorted category ids (class index c is ``category_ids[c]``) and the
    ``CocoGroundTruth``.  ``ValueError`` on a malformed file: a duplicate image id, an annotation of an unknown category or
    an unlisted image, an annotation id of 0 (COCOeval reads id 0 as "unmatched") or repeated, a bbox that is not 4
    numbers, or an iscrowd other than 0 / 1."""
    with open(json_path) as fh:
        data = json.load(fh)
    try:
        images = sorted((int(im["id"]), str(im.get("file_name", "")), (int(im["height"]), int(im["width"])))
                        for im in data["images"])
        cats = sorted(int(c["id"]) for c in data["categories"])
        anns = data["annotations"]
    except (KeyError, TypeError, ValueError) as e:
        raise ValueError(f"{json_path}: not a COCO instances file ({e!r})") from None
    if len({im[0] for im in images}) != len(images) or len(set(cats)) != len(cats):
        raise ValueError(f"{json_path}: image or category ids repeat")
    pos = {im[0]: i for i, im in enumerate(images)}
    cls = {c: i for i, c in enumerate(cats)}
    per_image: List[list] = [[] for _ in images]
    seen = set()
    for a in anns:
        aid, img, cat = a.get("id"), a.get("image_id"), a.get("category_id")
        if not isinstance(aid, int) or aid == 0 or aid in seen:
            raise ValueError(f"{json_path}: annotation id {aid!r} is 0, repeated or not an integer")
        seen.add(aid)
        if img not in pos:
            raise ValueError(f"{json_path}: annotation {aid} is on image {img!r}, which is not listed")
        if cat not in cls:
            raise ValueError(f"{json_path}: annotation {aid} has unknown category {cat!r}")
        bbox, crowd = a.get("bbox"), a.get("iscrowd")
        if not (isinstance(bbox, list) and len(bbox) == 4) or crowd not in (0, 1) or "area" not in a:
            raise ValueError(f"{json_path}: annotation {aid} needs bbox [x, y, w, h], area and iscrowd 0 / 1")
        per_image[pos[img]].append([cls[cat]] + [float(v) for v in bbox] + [float(a["area"]), float(crowd)])
    offsets = np.zeros(len(images) + 1, np.int64)
    np.cumsum([len(r) for r in per_image], out=offsets[1:])
    rows = np.array([r for rs in per_image for r in rs], np.float64).reshape(-1, 7)
    return images, cats, CocoGroundTruth(rows, offsets, tuple(cats))


def coco_results(dets, counts, image_ids: Sequence[int], category_ids: Sequence[int]) -> List[dict]:
    """The COCO results list of record blocks (dets int32 [N, C, K, 6], counts [N, C], host or device; image_ids [N]):
    one entry per record within its count, per image, class and record.  A record (ymin, xmin, ymax, xmax) becomes
    ``bbox = [xmin, ymin, xmax - xmin, ymax - ymin]``, computed in float64 from the float32 values, and its float32 score
    as float64: what ``CocoEval`` evaluates."""
    d = dets.cpu().numpy() if hasattr(dets, "cpu") else np.asarray(dets)
    n = counts.cpu().numpy() if hasattr(counts, "cpu") else np.asarray(counts)
    rec = np.ascontiguousarray(d, np.int32).view(np.float32)
    out = []
    for b, img in enumerate(image_ids):
        for c, cat in enumerate(category_ids):
            for y0, x0, y1, x1, score in rec[b, c, :int(n[b, c]), :5].astype(np.float64).tolist():
                out.append({"image_id": int(img), "category_id": int(cat), "bbox": [x0, y0, x1 - x0, y1 - y0], "score": score})
    return out


def coco_stats(precision: np.ndarray, recall: np.ndarray) -> np.ndarray:
    """COCOeval.summarize's 12 stats of precision [10, 101, C, 4, 3] and recall [10, C, 4, 3]: each the mean of the
    selected entries > -1 (-1 without any)."""
    def mean(ap, iou_thr=None, area="all", max_dets=100):
        s = precision if ap else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == COCO_IOU_THRS)[0]]
        a, m = COCO_AREA_LBL.index(area), COCO_MAX_DETS.index(max_dets)
        s = s[:, :, :, [a], [m]] if ap else s[:, :, [a], [m]]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
    return np.array([mean(1), mean(1, iou_thr=.5), mean(1, iou_thr=.75), mean(1, area="small"), mean(1, area="medium"),
                     mean(1, area="large"), mean(0, max_dets=1), mean(0, max_dets=10), mean(0), mean(0, area="small"),
                     mean(0, area="medium"), mean(0, area="large")], np.float64)


def coco_summary(stats: Sequence[float]) -> List[str]:
    """The 12 lines COCOeval.summarize prints for ``stats``."""
    spec = [(1, None, "all", 100), (1, .5, "all", 100), (1, .75, "all", 100), (1, None, "small", 100),
            (1, None, "medium", 100), (1, None, "large", 100), (0, None, "all", 1), (0, None, "all", 10),
            (0, None, "all", 100), (0, None, "small", 100), (0, None, "medium", 100), (0, None, "large", 100)]
    lines = []
    for (ap, thr, area, md), v in zip(spec, stats):
        iou = "{:0.2f}:{:0.2f}".format(COCO_IOU_THRS[0], COCO_IOU_THRS[-1]) if thr is None else "{:0.2f}".format(thr)
        lines.append(" {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}".format(
            "Average Precision" if ap else "Average Recall", "(AP)" if ap else "(AR)", iou, area, md, v))
    return lines


class CocoEval:
    """COCOeval (bbox, default parameters) on the GPU.  The ground truth (``load_coco_annotations``) is uploaded once;
    ``update`` matches a batch of record blocks, ``result`` ranks and reduces.  Every call runs on the current CUDA
    stream."""

    def __init__(self, gt: CocoGroundTruth, class_num: int, max_per_class: int, device=None):
        require_cuda()
        self.C, self.K = int(class_num), int(max_per_class)
        if len(gt.category_ids) != self.C:
            raise ValueError(f"the annotations have {len(gt.category_ids)} categories, the network {self.C} classes")
        rows = np.ascontiguousarray(gt.rows, np.float64).reshape(-1, 7)
        offsets = np.ascontiguousarray(gt.offsets, np.int64)
        if len(offsets) < 1 or offsets[-1] != len(rows):
            raise ValueError("ground-truth offsets do not cover the rows")
        self.n_images = len(offsets) - 1
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device or "cuda")
        self.device = torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)
        h = ctypes.c_void_p()
        check(lib.k2y_coco_create(rows.ctypes.data, offsets.ctypes.data, self.n_images, self.C, self.K,
                                  COCO_IOU_THRS.ctypes.data, COCO_REC_THRS.ctypes.data, self.device.index,
                                  ctypes.byref(h)))
        self._h = h

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def update(self, dets: torch.Tensor, counts: torch.Tensor, image_positions) -> None:
        """dets int32 ``[N, C, K, 6]`` (dense per image) and counts int32 ``[N, C]`` as ``DetectionPipeline`` returns
        them (device views of ``step_device`` or pinned host views of ``collect``, strided per image); image_positions:
        each image's index in the sorted image list of ``load_coco_annotations``.  Device records are read
        asynchronously on the current stream; host records have been copied when this returns."""
        pos = np.asarray(image_positions.cpu() if hasattr(image_positions, "cpu") else image_positions, np.int64).reshape(-1)
        n = len(pos)
        if (dets.dtype != torch.int32 or counts.dtype != torch.int32 or dets.dim() != 4 or counts.dim() != 2
                or tuple(dets.shape) != (n, self.C, self.K, 6) or tuple(counts.shape) != (n, self.C)
                or tuple(dets.stride()[1:]) != (self.K * 6, 6, 1) or counts.stride(1) != 1 or dets.is_cuda != counts.is_cuda):
            raise ValueError(f"expected int32 dets [{n}, {self.C}, {self.K}, 6] (dense per image) and counts [{n}, {self.C}] "
                             f"on one side of the bus, one per image position; got {tuple(dets.shape)} / {tuple(counts.shape)}")
        if n == 0:
            return
        with torch.cuda.device(self.device):
            if dets.is_cuda:
                if dets.device != self.device or counts.device != self.device:
                    raise ValueError(f"records on {dets.device}, evaluator on {self.device}")
            else:   # a blocking copy: the host views may be overwritten as soon as this returns
                dets, counts = dets.to(self.device), counts.to(self.device)
            positions = torch.from_numpy(pos).to(self.device)
            check(lib.k2y_coco_match(self._h, dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0), n,
                                     positions.data_ptr(), self._stream()))

    def result(self) -> dict:
        """``{"precision": [10, 101, C, 4, 3], "recall": [10, C, 4, 3], "stats": [12], "ap_per_class": [C]}``: COCOeval's
        eval arrays and summary stats, and per class the mean of precision[:, :, c, all, 100] over its entries > -1 (NaN
        for a class without ground truth).  ``ValueError`` if an update held an invalid record or image position."""
        precision = np.zeros((len(COCO_IOU_THRS), len(COCO_REC_THRS), self.C, 4, 3))
        recall = np.zeros((len(COCO_IOU_THRS), self.C, 4, 3))
        status = ctypes.c_uint()
        with torch.cuda.device(self.device):
            check(lib.k2y_coco_result(self._h, precision.ctypes.data, recall.ctypes.data, ctypes.byref(status),
                                      self._stream()))
        if status.value:
            raise ValueError("CocoEval: " + "; ".join(m for bit, m in COCO_STATUS.items() if status.value & bit))
        per_class = np.full(self.C, np.nan)
        for c in range(self.C):
            s = precision[:, :, c, 0, 2]
            if np.any(s > -1):
                per_class[c] = np.mean(s[s > -1])
        return {"precision": precision, "recall": recall, "stats": coco_stats(precision, recall), "ap_per_class": per_class}

    def reset(self) -> None:
        with torch.cuda.device(self.device):
            check(lib.k2y_coco_reset(self._h, self._stream()))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.k2y_coco_destroy(h)
            self._h = None
