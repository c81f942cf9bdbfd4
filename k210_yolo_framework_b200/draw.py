"""Result rendering of keras_inference.py:137-174: one rectangle per detection in the class colour of ``Helper.colormap``,
``(h + w) // 300`` pixels thick, and a filled ``'{class:2d} {score:.2f}'`` label box at the rectangle's top-left corner.

``box_geometry`` is the integer geometry the reference derives (``floor(v + 0.5)`` rounding, clipping to the image, the label
origin rule) — separated from the PIL calls so that it can be tested without a font file."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def box_geometry(image_shape: Sequence[int], box: Sequence[float], label_size: Sequence[int]):
    """(top, left, bottom, right, text_origin) as keras_inference.py:155-165 computes them."""
    top, left, bottom, right = box
    top = max(0, int(np.floor(top + 0.5)))
    left = max(0, int(np.floor(left + 0.5)))
    bottom = min(int(image_shape[0]), int(np.floor(bottom + 0.5)))
    right = min(int(image_shape[1]), int(np.floor(right + 0.5)))
    # the reference tests `top - image_shape[0] >= 0` (never true for a box inside the image): the label sits INSIDE the box
    origin = (left, top - int(label_size[1])) if top - int(image_shape[0]) >= 0 else (left, top + 1)
    return top, left, bottom, right, origin


def label_font(image_h: int, font_path: str = "asset/FiraMono-Medium.otf"):
    """The label font keras_inference.py picks for an image `image_h` rows high: the TrueType file at ``floor(0.03 h + 0.5)``
    points, or PIL's default font when the file cannot be opened."""
    from PIL import ImageFont
    try:
        return ImageFont.truetype(font=font_path, size=label_font_size(image_h))
    except OSError:
        return ImageFont.load_default()


def label_font_size(image_h: int) -> int:
    return int(np.floor(3e-2 * image_h + 0.5))


def _draw_labelled(orig_img: np.ndarray, items, font_path: str):
    """Draws (box, label, colour) items onto a copy of `orig_img` as keras_inference.py:150-172 draws one detection, a later
    item over an earlier one.  Returns the PIL image."""
    from PIL import Image, ImageDraw
    image_shape = orig_img.shape[0:2]
    pil_img = Image.fromarray(orig_img)
    font = label_font(image_shape[0], font_path)
    thickness = (image_shape[0] + image_shape[1]) // 300
    for box, label, colour in items:
        draw = ImageDraw.Draw(pil_img)
        tb = draw.textbbox((0, 0), label, font=font)
        label_size = (tb[2] - tb[0], tb[3] - tb[1])
        top, left, bottom, right, origin = box_geometry(image_shape, box, label_size)
        colour = tuple(int(v) for v in colour)
        for j in range(thickness):
            draw.rectangle([left + j, top + j, right - j, bottom - j], outline=colour)
        draw.rectangle([origin, (origin[0] + label_size[0], origin[1] + label_size[1])], fill=colour)
        draw.text(origin, label, fill=(0, 0, 0), font=font)
        del draw
    return pil_img


def draw_detections(orig_img: np.ndarray, found: List[Tuple], colormap, font_path: str = "asset/FiraMono-Medium.otf"):
    """found: (class, flat_index, score, top, left, bottom, right) tuples.  Returns the annotated PIL image."""
    return _draw_labelled(orig_img, (((top, left, bottom, right), "{:2d} {:.2f}".format(int(c), score), colormap[int(c)])
                                     for c, _idx, score, top, left, bottom, right in found), font_path)


def track_label(cls: int, track_id: int) -> str:
    """The label of a drawn track: ``"{class:2d} #{track_id}"``."""
    return "{:2d} #{}".format(int(cls), int(track_id))


def draw_tracks(orig_img: np.ndarray, tracks: List[Tuple], colormap, font_path: str = "asset/FiraMono-Medium.otf"):
    """tracks: (class, track_id, top, left, bottom, right) tuples, the track boxes of one frame in the order
    ``DetectionPipeline.tracks`` lays them out (class ascending, then record order).  Draws each as ``draw_detections`` draws
    a record (font, ring thickness, geometry, label origin, a later track over an earlier one), with three differences: the
    box is the track's, the colour is ``colormap[track_id % len(colormap)]``, so it follows the track and an id switch shows as
    a colour change, and the label is ``"{class:2d} #{track_id}"``.  Tracks with id -1 (none) are not drawn.  Returns the
    annotated PIL image."""
    return _draw_labelled(orig_img, (((top, left, bottom, right), track_label(c, tid), colormap[int(tid) % len(colormap)])
                                     for c, tid, top, left, bottom, right in tracks if int(tid) >= 0), font_path)
