"""TEST INFRASTRUCTURE — numpy restatement of the merge of views when some views are mirrored (test-time flip).

Only tests/ and scripts/ may import this module; the product path is ``k2y_merge_views_mirror`` in
k210_yolo_framework_b200/csrc/detect.cu.  Every rule of oracle/tiles_merge_ref.py holds as it is stated there; this module
adds what a mirrored view changes and leaves that module untouched.

A view flagged `mirrored` is its window (y0, x0, th, tw) flipped left to right, and its records are in mirrored window
coordinates: what np.fliplr(crop) gives when submitted as an image of its own.
 1. Border drop.  A mirrored view's record is tested as it comes, in the mirrored coordinates, against the window's side bits
    with 2 (left) and 8 (right) exchanged (``swap_sides``): the window's left edge is the mirrored view's right edge.  Bits 1
    and 4 stay.  A plain view's record is tested against its window's bits, as in tiles_merge_ref.
 2. Un-mirror and shift, in float32 with tw the window's width:  xmin = fl(fl(tw - xmax_m) + x0),
    xmax = fl(fl(tw - xmin_m) + x0);  the y fields are shifted as for any view.  tw - tw is +0.0 and tw - (-0.0) is tw.  A NaN
    result is the canonical NaN 0x7fffffff, whatever payload the subtraction left (tiles_merge_ref's shift rule).
 3. The index is v * nbox + index like any view's, v being the view's own number within its image (W + v for window v of an
    image of W windows with flip).  Ordering, matching, the action and max_per_class are tiles_merge_ref's.

``merge_class`` applies steps 1 and the subtraction of step 2 itself, then hands the records to
``tiles_merge_ref.merge_class`` without a border, which shifts them by (y0, x0) with its own float32 add and merges them.  So
the composition is exactly the rules above, and with no view mirrored it is tiles_merge_ref's merge.
"""
from __future__ import annotations

import numpy as np

from oracle import tiles_merge_ref as ref
from oracle.tiles_ref import DET, F


def swap_sides(sides) -> int:
    """Side bits of a mirrored view: the window's left (2) and right (8) bits exchanged."""
    sides = int(sides)
    return (sides & 5) | (8 if sides & 2 else 0) | (2 if sides & 8 else 0)


def merge_class(view_records, origins, sides, view_hw, nbox, thr, max_per_class, match="iou", merge="suppress", border=None,
                mirrored=None):
    """tiles_merge_ref.merge_class with `mirrored` [V] (true for a mirrored view; None: none is).  view_records[v]: list of
    (ymin, xmin, ymax, xmax, score, index) of view v of ONE image for ONE class in its own coordinates; origins[v] = (y0, x0),
    sides[v] its window's interior-side bits, view_hw[v] = (th, tw).  Returns the merged list in output order."""
    kept = []
    with np.errstate(all="ignore"):
        for v, recs in enumerate(view_records):
            mir = mirrored is not None and bool(mirrored[v])
            side = swap_sides(sides[v]) if mir else int(sides[v])
            th, tw = view_hw[v][0], view_hw[v][1]
            out = []
            for r in recs:
                if ref.border_drops(r, side, th, tw, border):
                    continue
                if mir:
                    r = (r[0], F(F(tw) - F(r[3])), r[2], F(F(tw) - F(r[1]))) + tuple(r[4:])
                out.append(r)
            kept.append(out)
    return ref.merge_class(kept, origins, [0] * len(kept), view_hw, nbox, thr, max_per_class, match, merge, None)


def merge_views(view_dets, view_counts, origins, offsets, nbox, thr, match="iou", merge="suppress", border=None, sides=None,
                view_hw=None, mirrored=None):
    """Block form, as tiles_merge_ref.merge_views, with `mirrored` [N] (None: no view is mirrored).  view_hw [N, 2] is needed
    with a border or a mirrored view.  Returns (dets [n, C, K] DET, zero past each count, counts [n, C])."""
    view_dets = np.ascontiguousarray(view_dets)
    if view_dets.dtype != DET:
        view_dets = view_dets.view(DET)[..., 0]
    _, C, K = view_dets.shape
    n = len(offsets) - 1
    N = int(offsets[-1])
    sides = np.zeros(N, np.int32) if sides is None else sides
    view_hw = np.zeros((N, 2), np.int64) if view_hw is None else view_hw
    mirrored = np.zeros(N, np.int32) if mirrored is None else mirrored
    dets = np.zeros((n, C, K), DET)
    counts = np.zeros((n, C), np.int32)
    for b in range(n):
        a, e = int(offsets[b]), int(offsets[b + 1])
        for c in range(C):
            lists = [[tuple(view_dets[g, c, k]) for k in range(int(view_counts[g, c]))] for g in range(a, e)]
            out = merge_class(lists, origins[a:e], sides[a:e], view_hw[a:e], nbox, thr, K, match, merge, border, mirrored[a:e])
            counts[b, c] = len(out)
            for k, r in enumerate(out):
                dets[b, c, k] = r
    return dets, counts
