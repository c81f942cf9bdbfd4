"""Tiled ("sliced") detection: the windows of an image that are detected as views of their own beside the whole image.

A view is a window ``(y0, x0, th, tw)`` in integer pixels.  View 0 is the whole image, views ``1 .. rows * cols`` are the tiles
in row-major order.  One axis of length ``L`` cut into ``k`` tiles with overlap fraction ``f`` has tiles of length
``t = min(L, ceil(L / (k - (k - 1) * f)))``; tile ``i`` starts at ``round_half_even(i * (L - t) / (k - 1))`` (0 when k == 1), so the
first tile starts at 0 and the last ends at ``L``.  The arithmetic is exact (``fractions.Fraction``; a float ``f`` is the rational
it stores), so no rounding depends on the platform.  ``DetectionPipeline.enable_tiling`` runs the views through the network and
``k2y_merge_views`` merges their records.
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
