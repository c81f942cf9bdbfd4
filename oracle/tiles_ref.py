"""TEST INFRASTRUCTURE — numpy restatement of tiled detection: the tile windows and the merge of the views' records.

Only tests/ and scripts/ may import this module; the product path is k210_yolo_framework_b200/tiles.py (windows) and
``k2y_merge_views`` in k210_yolo_framework_b200/csrc/detect.cu (merge).

Windows.  View 0 is the whole image, views 1 .. rows*cols the tiles, row-major, each (y0, x0, th, tw).  One axis of length L
cut into k tiles with overlap fraction f = p/q:  t = min(L, ceil(L / (k - (k-1) f))),  start_i = round_half_even(i (L - t) / (k-1)).
Everything below is integer arithmetic on p, q (``float.as_integer_ratio`` — the float IS that rational).

Merge, per image and class: the records of every view v are shifted by the view's origin (float32 adds), renumbered
index = v * nbox + index, ordered by (score descending, view ascending, index ascending) and passed through the greedy NMS of
oracle/decode_ref.py's dialect: a candidate is dropped iff its IoU with a record kept earlier is > iou_thresh, IoU in float32 in
tf.image.non_max_suppression's operation order, a zero-area box has IoU 0; stop at max_per_class.
"""
from __future__ import annotations

import numpy as np

F = np.float32


def axis_tiles(L, k, f):
    if k < 1 or not (0 <= f < 1) or L < k:
        raise ValueError((L, k, f))
    p, q = (f.as_integer_ratio() if isinstance(f, float) else (f.numerator, f.denominator)) if not isinstance(f, int) else (f, 1)
    den = k * q - (k - 1) * p                    # (k - (k-1) f) * q  > 0
    t = min(L, -((-L * q) // den))               # ceil(L q / den)
    out = []
    for i in range(k):
        if k == 1:
            out.append((0, t))
            continue
        a, r = divmod(i * (L - t), k - 1)
        if 2 * r > k - 1 or (2 * r == k - 1 and a % 2 == 1):
            a += 1
        out.append((a, t))
    return out


def tile_windows(h, w, rows, cols, overlap):
    ys, xs = axis_tiles(h, rows, overlap), axis_tiles(w, cols, overlap)
    win = [(0, 0, h, w)]
    for y0, th in ys:
        for x0, tw in xs:
            win.append((y0, x0, th, tw))
    return np.array(win, np.int32)


def _iou(box, kept):
    """float32 IoU of one (ymin, xmin, ymax, xmax) box with each row of `kept` [m, 4], corners in any order; 0 where either
    box has no area."""
    def norm(b):
        b = np.asarray(b, F).reshape(-1, 4)
        lo_y, hi_y = np.minimum(b[:, 0], b[:, 2]), np.maximum(b[:, 0], b[:, 2])
        lo_x, hi_x = np.minimum(b[:, 1], b[:, 3]), np.maximum(b[:, 1], b[:, 3])
        return lo_y, lo_x, hi_y, hi_x, (hi_y - lo_y) * (hi_x - lo_x)
    ay0, ax0, ay1, ax1, area_a = norm(box)
    by0, bx0, by1, bx1, area_b = norm(kept)
    ih = np.maximum(np.minimum(ay1, by1) - np.maximum(ay0, by0), F(0))
    iw = np.maximum(np.minimum(ax1, bx1) - np.maximum(ax0, bx0), F(0))
    inter = ih * iw
    iou = inter / ((area_a + area_b) - inter)
    return np.where((area_a <= 0) | (area_b <= 0), F(0), iou).astype(F)


def merge_class(view_records, origins, nbox, iou_thresh, max_per_class):
    """view_records[v]: list of (ymin, xmin, ymax, xmax, score, index) of view v for ONE class, any order; origins[v] = (y0, x0).
    Returns the merged list of (ymin, xmin, ymax, xmax, score, index) in output order (float32 / int values)."""
    cand = []
    for v, recs in enumerate(view_records):
        y0, x0 = F(origins[v][0]), F(origins[v][1])
        for r in recs:
            box = (F(F(r[0]) + y0), F(F(r[1]) + x0), F(F(r[2]) + y0), F(F(r[3]) + x0))
            cand.append((box, F(r[4]), v, int(r[5])))
    cand.sort(key=lambda c: (-float(c[1]), c[2], c[3]))
    kept = []
    thr = F(iou_thresh)
    with np.errstate(all="ignore"):
        for box, score, v, idx in cand:
            if len(kept) >= max_per_class:
                break
            if kept and bool((_iou(box, [k[0] for k in kept]) > thr).any()):
                continue
            kept.append((box, score, v * nbox + idx))
    return [(b[0], b[1], b[2], b[3], s, i) for b, s, i in kept]


DET = np.dtype([("ymin", "<f4"), ("xmin", "<f4"), ("ymax", "<f4"), ("xmax", "<f4"), ("score", "<f4"), ("index", "<i4")])


def merge_views(view_dets, view_counts, origins, n_images, nbox, iou_thresh):
    """Block form.  view_dets: [n_images * V, C, K] array of dtype DET (or int32 [..., 6] words), view_counts [n_images * V, C],
    origins [n_images * V, 2] (y0, x0).  Returns (dets [n_images, C, K] DET, zero past each count, counts [n_images, C])."""
    view_dets = np.ascontiguousarray(view_dets)
    if view_dets.dtype != DET:
        view_dets = view_dets.view(DET)[..., 0]
    nv, C, K = view_dets.shape
    V = nv // n_images
    dets = np.zeros((n_images, C, K), DET)
    counts = np.zeros((n_images, C), np.int32)
    for b in range(n_images):
        for c in range(C):
            lists = [[tuple(view_dets[b * V + v, c, k]) for k in range(int(view_counts[b * V + v, c]))] for v in range(V)]
            out = merge_class(lists, origins[b * V:(b + 1) * V], nbox, iou_thresh, K)
            counts[b, c] = len(out)
            for k, r in enumerate(out):
                dets[b, c, k] = r
    return dets, counts
