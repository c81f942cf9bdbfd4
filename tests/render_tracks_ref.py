"""numpy statement of what k2y_render_tracks (csrc/render.cu) draws for one image, built only from a track atlas
(render.TrackLabelAtlas): draw.draw_tracks' geometry and colours, the label composed from per-glyph masks, and Pillow's
fill_mask_L blend, with rings stopping at the first crossing ring where PIL raises and coordinates clamped as render_ref
states.

The label "{class:2d} #{id}" is composed as FreeType renders a string into one bitmap: glyph i starts at the integer pen
position sum(advance[c_j] for j < i) (the atlas builder refuses fonts where advances are fractional or kern), its mask lies at
pen + its own mask offset, and each glyph in string order goes over the mask so far as t = s + DIV255(t * (255 - s)).  The
label box is the union of the glyphs' textbboxes placed at their pens."""
import numpy as np

from render_ref import clamped_coord
from k210_yolo_framework_b200.draw import box_geometry, track_label
from k210_yolo_framework_b200.render import HEADER_WORDS, TRACK_ENTRY_WORDS, TRACK_GLYPHS


def div255(a):
    t = a + 128
    return ((t >> 8) + t) >> 8


def glyph_table(atlas: np.ndarray):
    n = int(atlas[0])
    entries = atlas[HEADER_WORDS:HEADER_WORDS + n * TRACK_ENTRY_WORDS].reshape(n, TRACK_ENTRY_WORDS)
    masks = atlas[HEADER_WORDS + n * TRACK_ENTRY_WORDS:].view(np.uint8)
    out = []
    for off, mw, mh, mx, my, bl, bt, br, bb, adv in entries.tolist():
        out.append((masks[off:off + mw * mh].reshape(mh, mw), (mx, my), (bl, bt, br, bb), adv))
    return out


def compose_label(atlas: np.ndarray, label: str, blend: str = "over"):
    """(mask uint8 [mh, mw], (mask x, mask y), (label w, label h)) of `label` composed from the atlas's glyphs.  `blend`
    "max" combines overlapping glyphs by maximum instead (what Pillow does not do; for the tests that tell them apart)."""
    table = glyph_table(atlas)
    pen, placed = 0, []
    l = t = 1 << 30
    r = b = -(1 << 30)
    for ch in label:
        mask, (mx, my), (bl, bt, br, bb), adv = table[TRACK_GLYPHS.index(ch)]
        l, t, r, b = min(l, pen + bl), min(t, bt), max(r, pen + br), max(b, bb)
        if mask.size:
            placed.append((pen + mx, my, mask))
        pen += adv
    size = (r - l, b - t)
    if not placed:
        return np.zeros((0, 0), np.uint8), (0, 0), size
    x0, y0 = min(p[0] for p in placed), min(p[1] for p in placed)
    x1, y1 = max(p[0] + p[2].shape[1] for p in placed), max(p[1] + p[2].shape[0] for p in placed)
    acc = np.zeros((y1 - y0, x1 - x0), np.int64)
    for gx, gy, mask in placed:
        sub = acc[gy - y0:gy - y0 + mask.shape[0], gx - x0:gx - x0 + mask.shape[1]]
        s = mask.astype(np.int64)
        sub[...] = np.maximum(sub, s) if blend == "max" else s + div255(sub * (255 - s))
    return acc.astype(np.uint8), (x0, y0), size


def render_tracks_ref(img: np.ndarray, tracks, colormap, atlas: np.ndarray, blend: str = "over") -> np.ndarray:
    """tracks: (class, id, top, left, bottom, right) in draw order; ids < 0 are skipped."""
    out = img.copy()
    h, w = out.shape[:2]
    thickness = (h + w) // 300

    def put(x0, y0, x1, y1, colour):     # inclusive box, clipped
        x0, y0, x1, y1 = max(x0, 0), max(y0, 0), min(x1, w - 1), min(y1, h - 1)
        if x0 <= x1 and y0 <= y1:
            out[y0:y1 + 1, x0:x1 + 1] = colour

    for c, tid, *box in tracks:
        if int(tid) < 0:
            continue
        mask, (mx, my), size = compose_label(atlas, track_label(c, tid), blend)
        top, left, bottom, right, (ox, oy) = box_geometry((h, w), [float(clamped_coord(v)) for v in box], size)
        colour = np.array(colormap[int(tid) % len(colormap)], np.uint8)
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
        out[ty, tx] = div255(out[ty, tx].astype(np.int32) * (255 - m)).astype(np.uint8)
    return out
