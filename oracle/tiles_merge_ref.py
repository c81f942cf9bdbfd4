"""TEST INFRASTRUCTURE — numpy restatement of size-driven tile grids and of the merge of views with its options.

Only tests/ and scripts/ may import this module; the product path is k210_yolo_framework_b200/tiles.py (``plan_grid``,
``plan_windows``, ``view_sides``) and ``k2y_merge_views_ex`` in k210_yolo_framework_b200/csrc/detect.cu (merge).  The windows
of one grid and the default merge are oracle/tiles_ref.py's, which this module leaves as they are.

Grid.  An axis of L pixels with a target tile length T and overlap f = p/q gets k tiles: 1 when L <= T, else the least k in
1..L whose tile length t(k) (tiles_ref.axis_tiles) is <= T, else L.  Found here by walking k upwards in integer arithmetic.
An image cut rows x cols has 1 view when rows * cols == 1, else 1 + rows * cols (the whole image, then the tiles row-major).
While that exceeds max_views, one tile comes off the axis with more tiles (the rows on a tie).

Merge, per image and class.  Image b owns views [off[b], off[b+1]); view numbers stay per image (0 is the whole image).
 1. Border drop (border m >= 0; None is off).  A record of view v is dropped before anything else if, in the window's own
    coordinates and float32 compares, with lo/hi the IEEE minNum / maxNum (fminf / fmaxf: a NaN gives way to the other value)
    of its two y (or x) fields:  side bit 1 set and lo_y < m;  bit 2 and lo_x < m;  bit 4 and hi_y > fl(th - m);  bit 8 and
    hi_x > fl(tw - m).  The bits are the window's interior sides (tiles.view_sides); the whole image has none.  A comparison
    with NaN is false, so a NaN bound never drops a record.
 2. Shift (one float32 add of the origin per field; a NaN sum is the GPU's canonical NaN 0x7fffffff, not the payload x86
    keeps), index = v * nbox + index, order by (score descending, view ascending, index ascending).
 3. Rounds: the first live candidate is kept; every live candidate whose metric with the kept candidate's own shifted box is
    > thr dies (the kept one dies with them).  Stop when nothing is live or max_per_class are kept.
    Both metrics normalise the boxes with fminf / fmaxf and compute, in float32, inter = max(min(hi) - max(lo), 0) per axis
    multiplied; a box of area <= 0 has metric 0.
      iou  inter / ((area_a + area_b) - inter)   (the default; what tiles_ref.merge_class computes for NaN-free boxes)
      ios  inter / fminf(area_a, area_b)
 4. Action.  suppress: the kept record as it is.  union: its box becomes the field-wise union of every record that died in its
    round (itself included): ymin, xmin the minimum, ymax, xmax the maximum of the raw shifted fields, -0.0 ordered below
    +0.0.  NaN fields take no part; a field that is NaN in every record of the group stays the kept record's.  Score and index
    stay the kept record's, so a kept record that matched nothing is bit for bit its suppress form.
"""
from __future__ import annotations

import numpy as np

from oracle.tiles_ref import DET, F, tile_windows


def _ratio(f):
    if isinstance(f, int):
        return f, 1
    if isinstance(f, float):
        return f.as_integer_ratio()
    return f.numerator, f.denominator


def tile_length(L, k, f):
    """t(k) of tiles_ref.axis_tiles: min(L, ceil(L q / (k q - (k-1) p)))."""
    p, q = _ratio(f)
    return min(L, -((-L * q) // (k * q - (k - 1) * p)))


def axis_count(L, T, f):
    if L <= T:
        return 1
    for k in range(1, L + 1):
        if tile_length(L, k, f) <= T:
            return k
    return L


def plan_grid(h, w, tile_hw, overlap, max_views):
    if tile_hw[0] < 1 or tile_hw[1] < 1 or max_views < 1:
        raise ValueError((tile_hw, max_views))
    p, q = _ratio(overlap)
    if not (0 <= p < q):
        raise ValueError(overlap)
    rows, cols = axis_count(h, tile_hw[0], overlap), axis_count(w, tile_hw[1], overlap)
    while (1 if rows * cols == 1 else 1 + rows * cols) > max_views:
        if rows >= cols:
            rows -= 1
        else:
            cols -= 1
    return rows, cols


def plan_windows(h, w, tile_hw, overlap, max_views):
    rows, cols = plan_grid(h, w, tile_hw, overlap, max_views)
    if rows * cols == 1:
        return np.array([(0, 0, h, w)], np.int32)
    return tile_windows(h, w, rows, cols, overlap)


def view_sides(windows, h, w):
    out = []
    for y0, x0, th, tw in np.asarray(windows).tolist():
        out.append((1 if y0 > 0 else 0) | (2 if x0 > 0 else 0) | (4 if y0 + th < h else 0) | (8 if x0 + tw < w else 0))
    return np.array(out, np.int32)


def _fmin(a, b):
    return np.fmin(F(a), F(b))


def _fmax(a, b):
    return np.fmax(F(a), F(b))


def border_drops(rec, sides, th, tw, m):
    """True iff record `rec` (ymin, xmin, ymax, xmax, ...) of a view with interior-side bits `sides` and size th x tw is dropped
    by a border of m pixels."""
    if m is None:
        return False
    m = F(m)
    lo_y, hi_y = _fmin(rec[0], rec[2]), _fmax(rec[0], rec[2])
    lo_x, hi_x = _fmin(rec[1], rec[3]), _fmax(rec[1], rec[3])
    return bool((sides & 1 and lo_y < m) or (sides & 2 and lo_x < m) or (sides & 4 and hi_y > F(F(th) - m))
                or (sides & 8 and hi_x > F(F(tw) - m)))


def _norm(b):
    b = np.asarray(b, F).reshape(-1, 4)
    ly, hy = np.fmin(b[:, 0], b[:, 2]), np.fmax(b[:, 0], b[:, 2])
    lx, hx = np.fmin(b[:, 1], b[:, 3]), np.fmax(b[:, 1], b[:, 3])
    return ly, lx, hy, hx, (hy - ly) * (hx - lx)


def metric_gt_many(a, boxes, thr, match="iou"):
    """metric(a, b) > thr in float32 for one box `a` and every row b of `boxes` [m, 4] (module docstring, step 3)."""
    ay0, ax0, ay1, ax1, area_a = _norm(a)
    by0, bx0, by1, bx1, area_b = _norm(boxes)
    thr = F(thr)
    with np.errstate(all="ignore"):
        ih = np.fmax(np.fmin(ay1, by1) - np.fmax(ay0, by0), F(0))
        iw = np.fmax(np.fmin(ax1, bx1) - np.fmax(ax0, bx0), F(0))
        inter = ih * iw
        den = ((area_a + area_b) - inter) if match == "iou" else np.fmin(area_a, area_b)
        gt = (inter / den) > thr
    return np.where((area_a <= 0) | (area_b <= 0), F(0) > thr, gt)


def metric_gt(a, b, thr, match="iou"):
    return bool(metric_gt_many(a, [b], thr, match)[0])


def _key(v):
    """Total order of non-NaN float32 values with -0.0 below +0.0."""
    u = int(np.array(v, F).view(np.uint32))
    return (~u & 0xffffffff) if u & 0x80000000 else (u | 0x80000000)


def _union(boxes, kept):
    out = list(kept)
    for f, take_min in ((0, True), (1, True), (2, False), (3, False)):
        vals = [b[f] for b in boxes if not np.isnan(b[f])]
        if vals:
            out[f] = (min if take_min else max)(vals, key=_key)
    return tuple(out)


CANONICAL_NAN = np.array(0x7fffffff, np.uint32).view(F)


def _add(a, b):
    r = F(F(a) + F(b))
    return CANONICAL_NAN if np.isnan(r) else r


def merge_class(view_records, origins, sides, view_hw, nbox, thr, max_per_class, match="iou", merge="suppress", border=None):
    """view_records[v]: list of (ymin, xmin, ymax, xmax, score, index) of view v of ONE image for ONE class; origins[v] = (y0,
    x0), sides[v] its interior-side bits, view_hw[v] = (th, tw).  Returns the merged list in output order."""
    cand = []
    with np.errstate(all="ignore"):
        for v, recs in enumerate(view_records):
            y0, x0 = F(origins[v][0]), F(origins[v][1])
            for r in recs:
                if border_drops(r, int(sides[v]), view_hw[v][0], view_hw[v][1], border):
                    continue
                box = (_add(r[0], y0), _add(r[1], x0), _add(r[2], y0), _add(r[3], x0))
                cand.append((box, F(r[4]), v, int(r[5])))
        cand.sort(key=lambda c: (-float(c[1]), c[2], c[3]))
        boxes = np.array([c[0] for c in cand], F).reshape(-1, 4)
        live = np.ones(len(cand), bool)
        out = []
        for i, (box, score, v, idx) in enumerate(cand):
            if len(out) >= max_per_class:
                break
            if not live[i]:
                continue
            live[i] = False
            rest = np.nonzero(live)[0]
            dies = rest[metric_gt_many(box, boxes[rest], thr, match)]
            live[dies] = False
            kept = _union([box] + [tuple(boxes[j]) for j in dies], box) if merge == "union" else box
            out.append((kept[0], kept[1], kept[2], kept[3], score, v * nbox + idx))
    return out


def merge_views(view_dets, view_counts, origins, offsets, nbox, thr, match="iou", merge="suppress", border=None, sides=None,
                view_hw=None):
    """Block form.  view_dets [N, C, K] DET (or int32 [..., 6] words), view_counts [N, C], origins [N, 2] (y0, x0), offsets
    [n + 1] (image b owns views offsets[b] .. offsets[b+1] - 1), sides [N] and view_hw [N, 2] (needed with a border).
    Returns (dets [n, C, K] DET, zero past each count, counts [n, C])."""
    view_dets = np.ascontiguousarray(view_dets)
    if view_dets.dtype != DET:
        view_dets = view_dets.view(DET)[..., 0]
    _, C, K = view_dets.shape
    n = len(offsets) - 1
    N = int(offsets[-1])
    sides = np.zeros(N, np.int32) if sides is None else sides
    view_hw = np.zeros((N, 2), np.int64) if view_hw is None else view_hw
    dets = np.zeros((n, C, K), DET)
    counts = np.zeros((n, C), np.int32)
    for b in range(n):
        a, e = int(offsets[b]), int(offsets[b + 1])
        for c in range(C):
            lists = [[tuple(view_dets[g, c, k]) for k in range(int(view_counts[g, c]))] for g in range(a, e)]
            out = merge_class(lists, origins[a:e], sides[a:e], view_hw[a:e], nbox, thr, K, match, merge, border)
            counts[b, c] = len(out)
            for k, r in enumerate(out):
                dets[b, c, k] = r
    return dets, counts
