"""Tiled ("sliced") detection: the windows of an image that are detected as views of their own beside the whole image.

A view is a window ``(y0, x0, th, tw)`` in integer pixels.  View 0 is the whole image, views ``1 .. rows * cols`` are the tiles
in row-major order.  One axis of length ``L`` cut into ``k`` tiles with overlap fraction ``f`` has tiles of length
``t = min(L, ceil(L / (k - (k - 1) * f)))``; tile ``i`` starts at ``round_half_even(i * (L - t) / (k - 1))`` (0 when k == 1), so the
first tile starts at 0 and the last ends at ``L``.  The arithmetic is exact (``fractions.Fraction``; a float ``f`` is the rational
it stores), so no rounding depends on the platform.  ``DetectionPipeline.enable_tiling`` runs the views through the network and
``k2y_merge_views`` merges their records.

``plan_grid`` / ``plan_windows`` choose an image's grid from a tile size instead (``enable_tiling(tile_size=...)``), and
``view_sides`` tells which edges of each window lie inside the image, for the border drop of ``k2y_merge_views_ex``.

With flip (``DetectionPipeline.enable_flip``) an image of W windows has 2W views: view ``v < W`` is window v, view ``W + v`` is
window v mirrored left to right (``mirror_views``).  ``plan_views`` derives the views of every image, the images one batch
holds and what the merge needs from the grid and the flip, in one place.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np


def axis_tiles(length: int, k: int, overlap) -> list:
    """[(start, size)] of the k tiles of one axis."""
    length, k = int(length), int(k)
    if k < 1:
        raise ValueError(f"{k} tiles: at least one per axis")
    f = Fraction(overlap)
    if not 0 <= f < 1:
        raise ValueError(f"tile overlap {overlap} is outside [0, 1)")
    if length < k:
        raise ValueError(f"an axis of {length} pixels cannot be cut into {k} tiles")
    t = min(length, math.ceil(length / (k - (k - 1) * f)))
    return [(round(Fraction(i * (length - t), k - 1)) if k > 1 else 0, t) for i in range(k)]


def tile_windows(h: int, w: int, rows: int, cols: int, overlap=0.2) -> np.ndarray:
    """int32 [1 + rows * cols, 4] windows (y0, x0, th, tw) of an h x w image: the whole image, then the tiles row-major.
    ``ValueError`` for rows or cols below 1, an overlap outside [0, 1) or an image with fewer rows / columns than tiles."""
    ys, xs = axis_tiles(h, rows, overlap), axis_tiles(w, cols, overlap)
    return np.array([(0, 0, int(h), int(w))] + [(y0, x0, th, tw) for y0, th in ys for x0, tw in xs], dtype=np.int32)


def view_count(rows: int, cols: int) -> int:
    """Views of an image cut rows x cols: one (the whole image) for 1x1, else the whole image and its rows * cols tiles."""
    return 1 if rows * cols == 1 else 1 + rows * cols


def axis_count(length: int, tile: int, overlap) -> int:
    """Tiles of one axis of `length` pixels for a target tile length `tile`: the least k in 1..length whose tiles
    (``axis_tiles``) are at most `tile` long, or `length` if there is none.  ``t(k) = ceil(L / (k (1 - f) + f))`` falls with k,
    so k is the least one with ``k (1 - f) + f >= L / T``."""
    length, tile = int(length), int(tile)
    f = Fraction(overlap)
    if length <= tile:
        return 1
    return min(length, max(1, math.ceil((Fraction(length, tile) - f) / (1 - f))))


def plan_grid(h: int, w: int, tile_hw, overlap, max_views: int) -> tuple:
    """(rows, cols) of an h x w image cut into tiles of at most tile_hw = (th, tw) pixels (``axis_count`` per axis), then,
    while the image has more than `max_views` views (``view_count``), one tile fewer on the axis with more tiles (on a tie, the
    rows).  1x1 is one view, so the loop ends there at the latest.  ``ValueError`` for a tile side below 1, an overlap
    outside [0, 1) or `max_views` below 1."""
    th, tw, max_views = int(tile_hw[0]), int(tile_hw[1]), int(max_views)
    if th < 1 or tw < 1:
        raise ValueError(f"tile size {th}x{tw}: at least one pixel per side")
    if not 0 <= Fraction(overlap) < 1:
        raise ValueError(f"tile overlap {overlap} is outside [0, 1)")
    if max_views < 1:
        raise ValueError(f"at most {max_views} views per image: at least one is needed")
    rows, cols = axis_count(h, th, overlap), axis_count(w, tw, overlap)
    while view_count(rows, cols) > max_views:
        if rows >= cols:
            rows -= 1
        else:
            cols -= 1
    return rows, cols


def plan_windows(h: int, w: int, tile_hw, overlap, max_views: int) -> np.ndarray:
    """int32 [V, 4] windows of an h x w image under ``plan_grid``: the whole image alone for a 1x1 grid, else
    ``tile_windows``."""
    rows, cols = plan_grid(h, w, tile_hw, overlap, max_views)
    if rows * cols == 1:
        return np.array([(0, 0, int(h), int(w))], dtype=np.int32)
    return tile_windows(h, w, rows, cols, overlap)


def view_sides(windows: np.ndarray, h: int, w: int) -> np.ndarray:
    """int32 [V] interior-side bits of an h x w image's windows: 1 top (y0 > 0), 2 left (x0 > 0), 4 bottom (y0 + th < h),
    8 right (x0 + tw < w).  The merge's border drop tests a record only against the sides whose bit is set; the whole image
    has none."""
    win = np.asarray(windows, np.int64).reshape(-1, 4)
    y0, x0, th, tw = win[:, 0], win[:, 1], win[:, 2], win[:, 3]
    return ((y0 > 0) * 1 + (x0 > 0) * 2 + (y0 + th < h) * 4 + (x0 + tw < w) * 8).astype(np.int32)


def mirror_views(windows: np.ndarray):
    """(int32 [2W, 4] windows, int32 [2W] mirror flags) of an image's W windows with flip: the windows as they are, then each
    one again, mirrored."""
    win = np.asarray(windows, np.int32).reshape(-1, 4)
    return np.concatenate([win, win]), np.repeat(np.array([0, 1], np.int32), len(win))


MATCHES = ("iou", "ios")
MERGES = ("suppress", "union")


class SizedTiling:
    """A per-image grid: every image is cut into tiles of at most `tile_hw` pixels (``plan_windows``), with at most
    `max_views` views.  ``BatchLayout`` takes it where it takes (rows, cols, overlap)."""

    def __init__(self, tile_hw, overlap, max_views: int):
        plan_grid(1, 1, tile_hw, overlap, max_views)        # validates the arguments
        self.tile_hw, self.overlap, self.max_views = (int(tile_hw[0]), int(tile_hw[1])), overlap, int(max_views)

    def windows(self, h: int, w: int) -> np.ndarray:
        return plan_windows(h, w, self.tile_hw, self.overlap, self.max_views)


def plan_views(batch: int, max_per_class: int, max_records: int, grid=None, flip: bool = False):
    """The views a pipeline of `batch` inputs detects each image as: (tiling, views, images_per_batch), where `tiling` is what
    ``BatchLayout`` takes (None, (rows, cols, overlap) or a ``SizedTiling``), `views` the most views of one image (the merge's
    max_views) and `images_per_batch` the images one batch holds.  `grid` is None (the whole image only), ("grid", rows, cols,
    overlap) or ("size", (th, tw), overlap, images_per_batch); with `flip` every window is detected mirrored as well.
      fixed grid (or none): V = (1 + rows * cols, or 1) * (2 with flip), images_per_batch = batch // V;
      sized grid: max_views = min(batch // images_per_batch, max_records // max_per_class), windows planned under max_views
                  (max_views // 2 with flip), views = that cap (doubled with flip).
    ``ValueError`` when V exceeds the batch or V * max_per_class exceeds `max_records` (the records one merge holds), or when no
    window fits a sized grid's cap."""
    batch, K, limit, mult = int(batch), int(max_per_class), int(max_records), 2 if flip else 1
    if grid is None or grid[0] == "grid":
        rows, cols, overlap = (1, 1, 0) if grid is None else grid[1:]
        V = (1 if grid is None else 1 + rows * cols) * mult
        if V > batch:
            raise ValueError(f"{V} views per image do not fit a batch of {batch}")
        if V * K > limit:
            raise ValueError(f"{V} views x {K} records per class exceed the {limit} records one merge holds")
        return (None if grid is None else (rows, cols, overlap)), V, batch // V
    _, tile_hw, overlap, ipb = grid
    cap = min(batch // ipb, limit // K)
    if cap // mult < 1:
        raise ValueError(f"no view fits: {K} records per class exceed the {limit} records one merge holds" if cap < 1 else
                         f"a flipped window takes 2 views and an image may have {cap}")
    return SizedTiling(tile_hw, overlap, cap // mult), cap // mult * mult, ipb
