"""numpy statement of what csrc/render.cu draws for one image: draw.draw_detections' geometry, the label atlas's glyphs and
Pillow's fill_mask_L blend, with rings stopping at the first crossing ring where PIL raises.  Records PIL cannot format or
draw get the kernel's documented clamps: a coordinate rounds to floor(v + 0.5) clamped to +-2^30 (NaN to -2^30), and the
label's hundredths rint(score * 100) are clamped to 0..100 (NaN to 0)."""
import math

import numpy as np

from k210_yolo_framework_b200.draw import box_geometry
from k210_yolo_framework_b200.render import ENTRY_WORDS, HEADER_WORDS, LABELS_PER_CLASS

COORD_LIMIT = 1 << 30


def clamped_coord(v: float) -> int:
    """round_coord: floor(double(v) + 0.5), NaN -> -2^30, clamped to +-2^30."""
    d = float(np.float32(v))
    if math.isnan(d):
        return -COORD_LIMIT
    d = math.floor(d + 0.5) if math.isfinite(d) else d
    return int(min(max(d, -COORD_LIMIT), COORD_LIMIT))


def clamped_hundredths(score: float) -> int:
    """rint(double(score) * 100) clamped to 0..100 (NaN -> 0): ties to even, as "{:.2f}" rounds a float32 in range."""
    d = float(np.float32(score)) * 100.0
    if math.isnan(d):
        return 0
    return int(min(max(np.rint(d), 0.0), 100.0))


def atlas_entry(atlas: np.ndarray, cls: int, hundredths: int):
    classes = int(atlas[0])
    e = atlas[HEADER_WORDS + (cls * LABELS_PER_CLASS + hundredths) * ENTRY_WORDS:][:ENTRY_WORDS]
    masks = atlas[HEADER_WORDS + classes * LABELS_PER_CLASS * ENTRY_WORDS:].view(np.uint8)
    off, mw, mh, mx, my, lw, lh, _ = (int(v) for v in e)
    return masks[off:off + mw * mh].reshape(mh, mw), (mx, my), (lw, lh)


def render_ref(img: np.ndarray, found, colormap, atlas: np.ndarray) -> np.ndarray:
    out = img.copy()
    h, w = out.shape[:2]
    thickness = (h + w) // 300

    def put(x0, y0, x1, y1, colour):     # inclusive box, clipped
        x0, y0, x1, y1 = max(x0, 0), max(y0, 0), min(x1, w - 1), min(y1, h - 1)
        if x0 <= x1 and y0 <= y1:
            out[y0:y1 + 1, x0:x1 + 1] = colour

    for c, _idx, score, *box in found:
        hund = clamped_hundredths(score)
        mask, (mx, my), size = atlas_entry(atlas, int(c), hund)
        top, left, bottom, right, (ox, oy) = box_geometry((h, w), [float(clamped_coord(v)) for v in box], size)
        colour = np.array(colormap[int(c)], np.uint8)
        for j in range(thickness):
            L, T, R, B = left + j, top + j, right - j, bottom - j
            if L > R or T > B:
                break
            put(L, T, R, T, colour)
            put(L, B, R, B, colour)
            put(L, T + 1, L, max(B - 1, T + 1), colour)
            put(R, T + 1, R, max(B - 1, T + 1), colour)
        put(ox, oy, ox + size[0], oy + size[1], colour)
        x0, y0 = ox + mx, oy + my
        ys, xs = np.mgrid[0:mask.shape[0], 0:mask.shape[1]]
        ok = (ys + y0 >= 0) & (ys + y0 < h) & (xs + x0 >= 0) & (xs + x0 < w)
        ty, tx, m = ys[ok] + y0, xs[ok] + x0, mask[ok].astype(np.int32)[:, None]
        t = out[ty, tx].astype(np.int32) * (255 - m) + 128
        out[ty, tx] = (((t >> 8) + t) >> 8).astype(np.uint8)
    return out
