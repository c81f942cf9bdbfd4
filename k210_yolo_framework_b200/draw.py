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


def draw_detections(orig_img: np.ndarray, found: List[Tuple], colormap, font_path: str = "asset/FiraMono-Medium.otf"):
    """found: (class, flat_index, score, top, left, bottom, right) tuples.  Returns the annotated PIL image."""
    from PIL import Image, ImageDraw
    image_shape = orig_img.shape[0:2]
    pil_img = Image.fromarray(orig_img)
    font = label_font(image_shape[0], font_path)
    thickness = (image_shape[0] + image_shape[1]) // 300
    for c, _idx, score, top, left, bottom, right in found:
        label = "{:2d} {:.2f}".format(int(c), score)
        draw = ImageDraw.Draw(pil_img)
        tb = draw.textbbox((0, 0), label, font=font)
        label_size = (tb[2] - tb[0], tb[3] - tb[1])
        top, left, bottom, right, origin = box_geometry(image_shape, (top, left, bottom, right), label_size)
        colour = tuple(int(v) for v in colormap[int(c)])
        for j in range(thickness):
            draw.rectangle([left + j, top + j, right - j, bottom - j], outline=colour)
        draw.rectangle([origin, (origin[0] + label_size[0], origin[1] + label_size[1])], fill=colour)
        draw.text(origin, label, fill=(0, 0, 0), font=font)
        del draw
    return pil_img
