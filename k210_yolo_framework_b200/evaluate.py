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

``MotEval``: CLEAR MOT and the identity metrics of tracks on MOTChallenge sequences (TrackEval's MotChallenge2DBox
preprocessing, CLEAR and Identity, as oracle/mot_ref.py restates them), matched and counted by the k2y_mot_* kernels.
``read_seqinfo`` and ``load_mot_gt`` read a sequence directory's seqinfo.ini and gt/gt.txt.
"""
from __future__ import annotations

import configparser
import ctypes
import json
import os
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


MOT_BENCHMARKS = {"MOT15": 15, "MOT16": 16, "MOT17": 17, "MOT20": 20}
MOT_STATUS = {1: "a frame has more than 512 tracker rows", 2: "a track id is >= 2^22",
              4: "a track id appears twice in one frame", 8: "a track box is not finite",
              16: "a record count is outside [0, max_per_class]",
              32: "a sequence's gt ids x tracker ids exceed 2^28"}
MOT_MAX_ROWS = 512
MOT_FIELDS = ("TP", "FP", "FN", "IDSW", "Frag", "MT", "PT", "ML", "IDTP", "gt_rows", "tracker_rows")


def read_seqinfo(seq_dir: str) -> dict:
    """The [Sequence] section of ``seq_dir/seqinfo.ini``: name, imDir, imExt (str), frameRate, seqLength, imWidth, imHeight
    (int).  ValueError when the file or a key is missing."""
    path = os.path.join(seq_dir, "seqinfo.ini")
    cp = configparser.ConfigParser()
    cp.optionxform = str
    if not cp.read(path) or "Sequence" not in cp:
        raise ValueError(f"{path}: no [Sequence] section")
    sec = cp["Sequence"]
    try:
        info = {k: sec[k] for k in ("name", "imDir", "imExt")}
        info.update({k: int(sec[k]) for k in ("frameRate", "seqLength", "imWidth", "imHeight")})
    except (KeyError, ValueError) as e:
        raise ValueError(f"{path}: {e!r}") from None
    return info


def load_mot_gt(path: str, benchmark: str = "MOT17") -> np.ndarray:
    """float64 rows [n, 8] (frame, id, left, top, w, h, conf, class) of a gt.txt: MOT16/17/20 rows (frame, id, left, top, w,
    h, conf, class, visibility), MOT15 rows (frame, id, left, top, w, h, conf, x, y, z) read as class 1."""
    if benchmark not in MOT_BENCHMARKS:
        raise ValueError(f"benchmark {benchmark!r} is not one of {tuple(MOT_BENCHMARKS)}")
    rows = np.loadtxt(path, delimiter=",", dtype=np.float64, ndmin=2)
    if rows.size == 0:
        return np.zeros((0, 8))
    want = 10 if benchmark == "MOT15" else 9
    if rows.shape[1] != want:
        raise ValueError(f"{path}: {benchmark} gt rows have {want} values, not {rows.shape[1]}")
    if benchmark == "MOT15":
        return np.concatenate([rows[:, :7], np.ones((len(rows), 1))], 1)
    return np.ascontiguousarray(rows[:, :8])


def check_mot_gt(name: str, gt: np.ndarray, seq_length: int, benchmark: str) -> None:
    """ValueError naming the sequence and frame for a frame outside 1..seq_length, an id twice in one frame, a class outside
    1..13 (MOT16/17/20) or more than MOT_MAX_ROWS rows in one frame."""
    if not np.all(np.isfinite(gt)):
        raise ValueError(f"{name}: the gt has a value that is not finite")
    f = gt[:, 0]
    bad = np.flatnonzero((f != np.floor(f)) | (f < 1) | (f > seq_length))
    if len(bad):
        raise ValueError(f"{name}: gt frame {f[bad[0]]:g} is outside 1..{seq_length}")
    if benchmark != "MOT15":
        c = gt[:, 7]
        bad = np.flatnonzero((c != np.floor(c)) | (c < 1) | (c > 13))
        if len(bad):
            raise ValueError(f"{name}: gt class {c[bad[0]]:g} in frame {int(f[bad[0]])} is outside 1..13")
    pairs = gt[:, :2]
    uniq, n = np.unique(pairs, axis=0, return_counts=True)
    if np.any(n > 1):
        fr, i = uniq[np.argmax(n > 1)]
        raise ValueError(f"{name}: gt id {i:g} appears twice in frame {int(fr)}")
    per = np.bincount(f.astype(np.int64), minlength=seq_length + 1)
    if per.max(initial=0) > MOT_MAX_ROWS:
        raise ValueError(f"{name}: frame {int(np.argmax(per))} has {per.max()} gt rows, more than {MOT_MAX_ROWS}")


HOTA_ALPHAS = 19
HOTA_ARRAY_FIELDS = ("HOTA", "DetA", "AssA", "DetRe", "DetPr", "AssRe", "AssPr", "LocA", "OWTA", "HOTA_TP", "HOTA_FN",
                     "HOTA_FP")
HOTA_SCALAR_FIELDS = ("HOTA(0)", "LocA(0)", "HOTALocA(0)")


def hota_final(TP, FN, FP, ass_a, ass_re, ass_pr, loc_a) -> dict:
    """TrackEval's final HOTA fields from arrays of 19: lists per alpha (counts as ints) and the three (0) scalars."""
    TP, FN, FP = (np.asarray(x, np.float64) for x in (TP, FN, FP))
    d = dict(AssA=np.asarray(ass_a, np.float64), AssRe=np.asarray(ass_re, np.float64), AssPr=np.asarray(ass_pr, np.float64),
             LocA=np.asarray(loc_a, np.float64))
    d["DetRe"] = TP / np.maximum(1, TP + FN)
    d["DetPr"] = TP / np.maximum(1, TP + FP)
    d["DetA"] = TP / np.maximum(1, TP + FN + FP)
    d["HOTA"] = np.sqrt(d["DetA"] * d["AssA"])
    d["OWTA"] = np.sqrt(d["DetRe"] * d["AssA"])
    out = {k: [float(v) for v in d[k]] for k in HOTA_ARRAY_FIELDS if k in d}
    for k, x in (("HOTA_TP", TP), ("HOTA_FN", FN), ("HOTA_FP", FP)):
        out[k] = [int(v) for v in x]
    out["HOTA(0)"] = float(d["HOTA"][0])
    out["LocA(0)"] = float(d["LocA"][0])
    out["HOTALocA(0)"] = float(d["HOTA"][0] * d["LocA"][0])
    return {k: out[k] for k in HOTA_ARRAY_FIELDS + HOTA_SCALAR_FIELDS}


def hota_sequence(counts, sums) -> dict:
    """One sequence's HOTA fields from the device's counts [3][19] (TP, FN, FP) and sums [4][19] (LocA, AssA, AssRe,
    AssPr): AssX = AssX_sum / max(1, TP), LocA = max(1e-10, LocA_sum) / max(1e-10, TP)."""
    TP = np.asarray(counts[0], np.float64)
    ass = [np.asarray(sums[k], np.float64) / np.maximum(1, TP) for k in (1, 2, 3)]
    loc_a = np.maximum(1e-10, np.asarray(sums[0], np.float64)) / np.maximum(1e-10, TP)
    return hota_final(counts[0], counts[1], counts[2], ass[0], ass[1], ass[2], loc_a)


def hota_combine(results) -> dict:
    """TrackEval's combine_sequences: counts summed, AssA / AssRe / AssPr and LocA weighted by each sequence's TP, summed in
    sequence order."""
    if not results:
        z = np.zeros(HOTA_ALPHAS)
        return hota_final(z, z, z, z, z, z, np.ones(HOTA_ALPHAS))
    TP, FN, FP = (sum(np.asarray(r[k], np.int64) for r in results) for k in ("HOTA_TP", "HOTA_FN", "HOTA_FP"))
    w = {}
    for k in ("AssRe", "AssPr", "AssA"):
        w[k] = sum(np.asarray(r[k], np.float64) * np.asarray(r["HOTA_TP"], np.float64) for r in results) / np.maximum(1.0, TP)
    loc = sum(np.asarray(r["LocA"], np.float64) * np.asarray(r["HOTA_TP"], np.float64) for r in results)
    return hota_final(TP, FN, FP, w["AssA"], w["AssRe"], w["AssPr"], np.maximum(1e-10, loc) / np.maximum(1e-10, TP))


def mot_ratios(d: dict) -> dict:
    """Adds MOTA, MOTP, Rcll, Prcn, IDR, IDP and IDF1 to a dict of the counts and MOTP_sum."""
    TP, FP, FN, IDSW, IDTP, IDFP, IDFN = (d[k] for k in ("TP", "FP", "FN", "IDSW", "IDTP", "IDFP", "IDFN"))
    d = dict(d)
    d["MOTA"] = (TP - FP - IDSW) / max(1, TP + FN)
    d["MOTP"] = d["MOTP_sum"] / max(1, TP)
    d["Rcll"] = TP / max(1, TP + FN)
    d["Prcn"] = TP / max(1, TP + FP)
    d["IDR"] = IDTP / max(1, IDTP + IDFN)
    d["IDP"] = IDTP / max(1, IDTP + IDFP)
    d["IDF1"] = IDTP / max(1, IDTP + 0.5 * IDFP + 0.5 * IDFN)
    return d


class MotEval:
    """MOTChallenge CLEAR MOT, identity metrics and HOTA on the GPU.  ``add_sequence`` uploads a sequence's gt once; ``update``
    takes the tracked record blocks of a batch of its frames; ``result`` evaluates every sequence.  Every call runs on the
    current CUDA stream, and is ordered after the evaluator's previous call whatever stream that used.

    Caps: 512 gt rows and 512 tracker rows per frame, track ids below 2^22, and gt ids x tracker ids of a sequence up to
    2^28; past them ``add_sequence`` or ``result`` raises ValueError."""

    def __init__(self, benchmark: str = "MOT17", device=None):
        require_cuda()
        if benchmark not in MOT_BENCHMARKS:
            raise ValueError(f"benchmark {benchmark!r} is not one of {tuple(MOT_BENCHMARKS)}")
        self.benchmark = benchmark
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device or "cuda")
        self.device = torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)
        self._seqs = {}         # name -> (index, seq_length, positions given)
        h = ctypes.c_void_p()
        check(lib.k2y_mot_create(MOT_BENCHMARKS[benchmark], self.device.index, ctypes.byref(h)))
        self._h = h

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def add_sequence(self, name: str, gt_rows, seq_length: int) -> None:
        """gt_rows float64 [n, 8] (frame, id, left, top, w, h, conf, class) as ``load_mot_gt`` reads them."""
        if name in self._seqs:
            raise ValueError(f"sequence {name!r} was added already")
        gt = np.ascontiguousarray(np.asarray(gt_rows, np.float64).reshape(-1, 8))
        seq_length = int(seq_length)
        if seq_length < 1:
            raise ValueError(f"{name}: seqLength {seq_length} < 1")
        check_mot_gt(name, gt, seq_length, self.benchmark)
        order = np.argsort(gt[:, 0], kind="stable")
        gt = np.ascontiguousarray(gt[order])
        idx = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib.k2y_mot_add_sequence(self._h, gt.ctypes.data, len(gt), seq_length, ctypes.byref(idx)))
        self._seqs[name] = (idx.value, seq_length, set())

    def update(self, name: str, positions, ids: torch.Tensor, boxes: torch.Tensor, dets: torch.Tensor, counts: torch.Tensor,
               person_class: int) -> None:
        """One batch of frames of sequence `name`: positions (host ints, 0..seqLength-1, each once), ids int32 [N, C, K] and
        boxes float32 [N, C, K, 4] as ``DetectionPipeline.tracks`` returns them, dets int32 [N, C, K, 6] and counts int32
        [N, C] as ``collect`` does: pinned host views or device tensors, all on one side of the bus.  The records of
        `person_class` with a track id >= 0 are the frame's tracker rows."""
        if name not in self._seqs:
            raise ValueError(f"unknown sequence {name!r}: add_sequence first")
        idx, L, given = self._seqs[name]
        pos = [int(p) for p in positions]
        n = len(pos)
        if ids.dim() != 3 or n != ids.shape[0]:
            raise ValueError(f"expected ids [{n}, C, K], got {tuple(ids.shape)}")
        C, K = int(ids.shape[1]), int(ids.shape[2])
        if (ids.dtype != torch.int32 or boxes.dtype != torch.float32 or dets.dtype != torch.int32 or counts.dtype != torch.int32
                or tuple(boxes.shape) != (n, C, K, 4) or tuple(dets.shape) != (n, C, K, 6) or tuple(counts.shape) != (n, C)
                or tuple(ids.stride()[1:]) != (K, 1) or tuple(boxes.stride()[1:]) != (K * 4, 4, 1) or counts.stride(1) != 1
                or len({t.is_cuda for t in (ids, boxes, dets, counts)}) != 1):
            raise ValueError(f"expected int32 ids [{n}, {C}, {K}], float32 boxes [{n}, {C}, {K}, 4], int32 dets [{n}, {C}, {K}, 6] "
                             f"and counts [{n}, {C}], dense per frame, on one side of the bus")
        if not 0 <= int(person_class) < C:
            raise ValueError(f"person_class {person_class} is outside [0, {C})")
        for p in pos:
            if not 0 <= p < L:
                raise ValueError(f"{name}: frame position {p} is outside 0..{L - 1} (frame {p + 1} outside 1..{L})")
            if p in given:
                raise ValueError(f"{name}: frame {p + 1} was given twice")
            given.add(p)
        if n == 0:
            return
        with torch.cuda.device(self.device):
            if ids.is_cuda:
                if any(t.device != self.device for t in (ids, boxes, counts)):
                    raise ValueError(f"blocks on {ids.device}, evaluator on {self.device}")
            else:   # a blocking copy: the host views may be overwritten as soon as this returns
                ids, boxes, counts = ids.to(self.device), boxes.to(self.device), counts.to(self.device)
            p = torch.tensor(pos, dtype=torch.int64).to(self.device)
            check(lib.k2y_mot_update(self._h, idx, counts.data_ptr(), ids.data_ptr(), boxes.data_ptr(), counts.stride(0),
                                     ids.stride(0), boxes.stride(0), n, p.data_ptr(), C, K, int(person_class), self._stream()))

    def result(self) -> dict:
        """``{"sequences": {name: fields}, "combined": fields, "rounds": {name: CLEAR rounds}, "solved": {name: frame solves
        that needed an assignment}}``; fields: TP, FP, FN, IDSW, Frag, MT, PT, ML, IDTP, IDFP, IDFN, gt_rows, tracker_rows
        (int), MOTP_sum, MOTA, MOTP, Rcll, Prcn, IDR, IDP, IDF1 (float).  Integer fields and MOTP_sum (in sequence order)
        are summed over the sequences and the ratios recomputed.  ``"hota"``: ``{"sequences": {name: fields}, "combined":
        fields}`` with HOTA, DetA, AssA, DetRe, DetPr, AssRe, AssPr, LocA, OWTA (lists of 19 floats, one per alpha 0.05 ..
        0.95), HOTA_TP, HOTA_FN, HOTA_FP (lists of 19 ints) and HOTA(0), LocA(0), HOTALocA(0), as TrackEval's HOTA gives
        them (oracle/mot_hota_ref.py).  ``ValueError`` if an update held invalid input."""
        S = len(self._seqs)
        counts = np.zeros((max(S, 1), 12), np.int64)
        motp = np.zeros(max(S, 1))
        rounds = np.zeros(max(S, 1), np.int32)
        solved = np.zeros(max(S, 1), np.int64)
        hcounts = np.zeros((max(S, 1), 3, HOTA_ALPHAS), np.int64)
        hsums = np.zeros((max(S, 1), 4, HOTA_ALPHAS))
        status = ctypes.c_uint()
        with torch.cuda.device(self.device):
            check(lib.k2y_mot_result_ex(self._h, counts.ctypes.data, motp.ctypes.data, rounds.ctypes.data, solved.ctypes.data,
                                        hcounts.ctypes.data, hsums.ctypes.data, ctypes.byref(status), self._stream()))
        if status.value:
            raise ValueError("MotEval: " + "; ".join(m for bit, m in MOT_STATUS.items() if status.value & bit))
        seqs, out_rounds, out_solved, hota = {}, {}, {}, {}
        for name, (i, _, _) in self._seqs.items():
            hota[name] = hota_sequence(hcounts[i], hsums[i])
            d = {k: int(v) for k, v in zip(MOT_FIELDS, counts[i, :11])}
            d.update(IDFN=d["gt_rows"] - d["IDTP"], IDFP=d["tracker_rows"] - d["IDTP"], MOTP_sum=float(motp[i]))
            seqs[name] = mot_ratios(d)
            out_rounds[name], out_solved[name] = int(rounds[i]), int(solved[i])
        comb = {k: sum(d[k] for d in seqs.values()) for k in MOT_FIELDS + ("IDFN", "IDFP")}
        s = 0.0
        for d in seqs.values():
            s += d["MOTP_sum"]
        comb["MOTP_sum"] = s
        return {"sequences": seqs, "combined": mot_ratios(comb), "rounds": out_rounds, "solved": out_solved,
                "hota": {"sequences": hota, "combined": hota_combine(list(hota.values()))}}

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.k2y_mot_destroy(h)
            self._h = None
