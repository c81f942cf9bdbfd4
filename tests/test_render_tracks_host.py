"""Host side of GPU track drawing (no GPU): the track atlas's glyphs composed as k2y_render_tracks composes them
(tests/render_tracks_ref.py) against draw.draw_tracks and PIL's whole-string masks, for PIL's default font and its TrueType
bytes at several sizes, every id up to 2000 and the decades up to 2^31 - 1, every class; the atlas's refusal of fonts whose
advances are fractional or kern; and serve.py's --draw_tracks argument rules."""
import os

import numpy as np
import pytest
from PIL import Image, ImageDraw, ImageFont

from render_tracks_ref import compose_label, render_tracks_ref
from k210_yolo_framework_b200.draw import box_geometry, draw_tracks, label_font, track_label
from k210_yolo_framework_b200.helper import _COLORMAP
from k210_yolo_framework_b200.render import TRACK_GLYPHS, TrackLabelAtlas, build_track_atlas, glyphs

INT32_MAX = 2 ** 31 - 1
DECADES = [v for k in range(1, 10) for v in (10 ** k - 1, 10 ** k)] + [INT32_MAX]


@pytest.fixture(scope="module")
def default_ttf(tmp_path_factory):
    p = tmp_path_factory.mktemp("font") / "default.ttf"
    p.write_bytes(ImageFont.load_default().font_bytes)
    return str(p)


def on_canvas(mask, offset, x0, y0, w, h):
    c = np.zeros((h, w), np.int32)
    mh, mw = mask.shape
    c[offset[1] - y0:offset[1] - y0 + mh, offset[0] - x0:offset[0] - x0 + mw] = mask
    return c


def same_label(font, atlas, label):
    """The composed mask equals PIL's whole-string mask pixel for pixel (wherever either lies), and the label sizes agree."""
    pm, po, psize = glyphs(font, label)
    cm, co, csize = compose_label(atlas, label)
    if psize != csize:
        return False
    x0, y0 = min(po[0], co[0]), min(po[1], co[1])
    x1 = max(po[0] + pm.shape[1], co[0] + cm.shape[1])
    y1 = max(po[1] + pm.shape[0], co[1] + cm.shape[0])
    return np.array_equal(on_canvas(pm, po, x0, y0, x1 - x0, y1 - y0), on_canvas(cm, co, x0, y0, x1 - x0, y1 - y0))


def seeded_tracks(h, w, n, class_num, seed, ids=None):
    """(class, id, top, left, bottom, right) in tracks() order: boxes clipped at every edge, overlapping, of every size down to
    two pixels; ids -1, small, large and 2^31 - 1."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        c = int(rng.integers(0, class_num))
        t, l = rng.uniform(-0.2 * h, 1.0 * h), rng.uniform(-0.2 * w, 1.0 * w)
        bh, bw = rng.uniform(2, 0.8 * h), rng.uniform(2, 0.8 * w)
        tid = ids[k % len(ids)] if ids is not None else [-1, 1, 7, 42, INT32_MAX, int(rng.integers(0, 100000))][k % 6]
        out.append((c, tid, *(float(np.float32(v)) for v in (t, l, t + bh, l + bw))))
    out.sort(key=lambda r: r[0])
    return [r for r in out if no_crossing(r, h, w)]


def no_crossing(rec, h, w):
    """draw_tracks raises on a box whose outline rings cross; keep the tracks it can draw."""
    t, l, b, r, _ = box_geometry((h, w), rec[2:], (0, 0))
    th = (h + w) // 300
    return th == 0 or (l + th - 1 <= r - th + 1 and t + th - 1 <= b - th + 1)


def check_image(img, tracks, font_path, atlas):
    ref = np.array(draw_tracks(img, tracks, _COLORMAP, font_path=font_path))
    got = render_tracks_ref(img, tracks, _COLORMAP, atlas.host(img.shape[0]))
    assert np.array_equal(got, ref), (font_path, img.shape, int((got != ref).any(-1).sum()))


@pytest.mark.parametrize("h", [17, 224, 375, 700, 1080])
@pytest.mark.parametrize("which", ["missing", "ttf"])
def test_restatement_reproduces_draw_tracks(which, h, default_ttf):
    font_path = "missing.otf" if which == "missing" else default_ttf
    atlas = TrackLabelAtlas(font_path)
    w = int(h * 1.4) + 3
    img = np.random.default_rng(h).integers(0, 256, (h, w, 3), dtype=np.uint8)
    check_image(img, seeded_tracks(h, w, 30, 80, h), font_path, atlas)


@pytest.mark.parametrize("h", [224, 700])
def test_every_id_up_to_2000_and_every_decade(h, default_ttf):
    font = label_font(h, default_ttf)
    atlas = build_track_atlas(font)
    bad = [i for i in list(range(2001)) + DECADES if not same_label(font, atlas, track_label(i % 80, i))]
    assert not bad, bad[:20]


def test_every_id_up_to_2000_default_font():
    font = label_font(375, "missing.otf")
    atlas = TrackLabelAtlas("missing.otf").host(375)
    bad = [i for i in list(range(2001)) + DECADES if not same_label(font, atlas, track_label(i % 80, i))]
    assert not bad, bad[:20]


def test_every_class(default_ttf):
    for font_path in ["missing.otf", default_ttf]:
        font = label_font(375, font_path)
        atlas = TrackLabelAtlas(font_path).host(375)
        assert all(same_label(font, atlas, track_label(c, tid)) for c in range(80) for tid in (0, 5, 1234, INT32_MAX))
    img = np.full((375, 1400, 3), 200, np.uint8)
    tracks = [(c, 3 * c + 1, 10.0 + 3 * (c % 4), 5.0 + 17 * c, 300.0, 40.0 + 17 * c) for c in range(80)]
    check_image(img, tracks, default_ttf, TrackLabelAtlas(default_ttf))


def test_overlapping_glyphs_blend_over_not_max(default_ttf):
    """Glyphs whose masks overlap combine as t = s + DIV255(t * (255 - s)), which PIL's string masks show, and at least one
    label exists where that differs from max."""
    differ = []
    for font_path in ["missing.otf", default_ttf]:
        for h in [224, 375, 700]:
            font = label_font(h, font_path)
            atlas = build_track_atlas(font)
            for label in ["0 #4444", "11 #4747", "7 #1111111111", "44 #44444", "40 #2147483647", "79 #7777777"]:
                assert same_label(font, atlas, label), (font_path, h, label)
                if not np.array_equal(compose_label(atlas, label)[0], compose_label(atlas, label, "max")[0]):
                    differ.append((font_path, h, label))
    assert differ


def test_labels_off_the_right_and_bottom_edges_and_top_past_the_image(default_ttf):
    atlas = TrackLabelAtlas(default_ttf)
    for h, w in [(224, 320), (200, 390)]:      # one ring: PIL draws a box whose top is clipped to h only then
        img = np.random.default_rng(w).integers(0, 256, (h, w, 3), dtype=np.uint8)
        tracks = [(3, INT32_MAX, 10.0, w - 12.0, 60.0, w + 40.0),           # label runs off the right edge
                  (12, 999999, h - 4.0, 30.0, h + 50.0, 90.0),              # off the bottom edge
                  (40, 77, float(h), 100.0, h + 20.0, 160.0),               # top >= h: the label sits above the box's top
                  (41, 123456, h + 0.4, w - 5.0, h + 60.0, w + 30.0),       # both
                  (79, 0, -50.0, -50.0, 3.0, 3.0)]
        check_image(img, tracks, default_ttf, atlas)


class StubFont:
    def __init__(self, length):
        self.length = length

    def getlength(self, text):
        return self.length(text)


def test_atlas_refuses_fractional_or_kerned_advances():
    with pytest.raises(ValueError, match="whole number"):
        build_track_atlas(StubFont(lambda t: 6.5 * len(t)))
    with pytest.raises(ValueError, match="kerning"):
        build_track_atlas(StubFont(lambda t: 6 * len(t) - (1 if t == "#1" else 0)))
    with pytest.raises(ValueError, match="kerning"):
        build_track_atlas(StubFont(lambda t: 6 * len(t) + (len(t) > 1)))
    assert TRACK_GLYPHS == "0123456789 #"


def test_atlas_accepts_the_default_font_at_every_size(default_ttf):
    for size in range(1, 60):
        build_track_atlas(ImageFont.truetype(default_ttf, size))


def test_serve_draw_tracks_arguments(tmp_path):
    import serve
    clip, imgs = str(tmp_path / "clip.avi"), str(tmp_path / "imgs")
    with open(clip, "wb") as fh:        # what serve.is_video sniffs: a RIFF AVI header
        fh.write(b"RIFF\0\0\0\0AVI LIST")
    os.makedirs(imgs)
    ap = serve.build_parser()
    a = ap.parse_args(["ck.npz", clip, "--track", "--draw", "out", "--draw_tracks"])
    assert a.draw_tracks and a.track and a.draw == "out"
    assert not ap.parse_args(["ck.npz", clip, "--track", "--draw", "out"]).draw_tracks
    for bad in ([clip, "--draw", "out", "--draw_tracks"], [clip, "--track", "--draw_tracks"], [clip, "--draw_tracks"],
                [imgs, "--draw", "out", "--draw_tracks"]):
        with pytest.raises(SystemExit):
            ap.parse_args(["ck.npz"] + bad)
