"""Host side of GPU rendering and JPEG encoding (no GPU): the encoder's marker segments against PIL's, the label atlas
composited with the documented blend against draw_detections for PIL's default font and a TrueType font, and serve.py's
--draw argument handling."""
import io
import os

import numpy as np
import pytest
from PIL import Image, ImageFont

from render_ref import render_ref
from k210_yolo_framework_b200.draw import draw_detections
from k210_yolo_framework_b200.helper import _COLORMAP
from k210_yolo_framework_b200.render import LabelAtlas, jpeg_header, label_hundredths, label_text


def pil_jpeg(img, quality):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=quality)
    return b.getvalue()


@pytest.mark.parametrize("quality", [1, 50, 75, 95, 100])
@pytest.mark.parametrize("hw", [(1, 1), (7, 9), (16, 16), (224, 320), (1080, 1920), (65500, 3)])  # libjpeg-turbo writes up to 65500
def test_headers_equal_pil_up_to_sos(hw, quality):
    h, w = hw
    img = np.random.default_rng(h + w).integers(0, 256, (min(h, 64), w, 3), dtype=np.uint8)
    if h > 64:     # PIL needs the whole image; only the header matters here
        img = np.resize(img, (h, w, 3))
    ref = pil_jpeg(img, quality)
    hdr = jpeg_header(h, w, quality)
    assert hdr[-14:-12] == b"\xff\xda" and ref[:len(hdr)] == hdr


def test_header_refuses_bad_sizes_and_qualities():
    for h, w, q in [(0, 5, 75), (5, 65501, 75), (65501, 5, 75), (5, 65536, 75), (5, 5, 0), (5, 5, 101)]:
        with pytest.raises(ValueError):
            jpeg_header(h, w, q)


def test_label_text_matches_python_formatting():
    for s in [0.005, 0.125, 0.995, 1.0, 0.7, 0.715, 0.33333334, 0.0, 0.5049999]:
        f = float(np.float32(s))
        assert label_text(7, label_hundredths(f)) == "{:2d} {:.2f}".format(7, f)
    rng = np.random.default_rng(0)
    for f in rng.uniform(0, 1, 2000).astype(np.float32):
        assert label_text(12, label_hundredths(float(f))) == "{:2d} {:.2f}".format(12, float(f))


def seeded_records(h, w, n, class_num, seed):
    """(class, index, score, top, left, bottom, right) in to_host order: boxes clipped at every edge, overlapping, of every
    size down to two pixels, with the edge scores."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        c = int(rng.integers(0, class_num))
        t, l = rng.uniform(-0.2 * h, 1.0 * h), rng.uniform(-0.2 * w, 1.0 * w)
        bh, bw = rng.uniform(2, 0.8 * h), rng.uniform(2, 0.8 * w)
        score = [0.005, 0.125, 0.995, 1.0][k % 4] if k < 8 else float(rng.uniform(0.3, 1))
        out.append((c, k, float(np.float32(score)), float(np.float32(t)), float(np.float32(l)), float(np.float32(t + bh)),
                    float(np.float32(l + bw))))
    out.sort(key=lambda r: r[0])
    return [r for r in out if no_crossing(r, h, w)]


def no_crossing(rec, h, w):
    """draw_detections raises on a box whose outline rings cross; keep the records it can draw."""
    from k210_yolo_framework_b200.draw import box_geometry
    t, l, b, r, _ = box_geometry((h, w), rec[3:], (0, 0))
    th = (h + w) // 300
    return th == 0 or (l + th - 1 <= r - th + 1 and t + th - 1 <= b - th + 1)


def font_cases(tmp_path):
    ttf = tmp_path / "default.ttf"
    ttf.write_bytes(ImageFont.load_default().font_bytes)
    return [("missing.otf", [224, 375]), (str(ttf), [17, 224, 375, 700])]


def test_atlas_composite_reproduces_draw_detections(tmp_path):
    for font_path, heights in font_cases(tmp_path):
        atlas = LabelAtlas(20, font_path)
        for h in heights:
            w = int(h * 1.4) + 3
            img = np.random.default_rng(h).integers(0, 256, (h, w, 3), dtype=np.uint8)
            found = seeded_records(h, w, 24, 20, h)
            ref = np.array(draw_detections(img, found, _COLORMAP, font_path=font_path))
            got = render_ref(img, found, _COLORMAP, atlas.host(h))
            assert np.array_equal(got, ref), (font_path, h, int((got != ref).any(-1).sum()))


def test_atlas_covers_every_class_and_hundredth(tmp_path):
    atlas = LabelAtlas(80, "missing.otf")
    img = np.full((120, 400, 3), 200, np.uint8)
    found = [(c, 0, float(np.float32(((c * 37) % 101) / 100)), 10.0, 5.0 + 4 * c, 100.0, 40.0 + 4 * c) for c in range(80)]
    ref = np.array(draw_detections(img, found, _COLORMAP, font_path="missing.otf"))
    assert np.array_equal(render_ref(img, found, _COLORMAP, atlas.host(120)), ref)


def test_atlas_refuses_more_classes_than_colours():
    with pytest.raises(ValueError):
        LabelAtlas(81)


def test_serve_draw_arguments():
    import serve
    ap = serve.build_parser()
    a = ap.parse_args(["ck.npz", "imgs"])
    assert a.draw is None and a.draw_quality == 75
    a = ap.parse_args(["ck.npz", "imgs", "--draw", "out", "--draw_quality", "90"])
    assert a.draw == "out" and a.draw_quality == 90
    for bad in ["0", "101", "x"]:
        with pytest.raises(SystemExit):
            ap.parse_args(["ck.npz", "imgs", "--draw", "out", "--draw_quality", bad])


def test_serve_refuses_duplicate_stems(tmp_path):
    import serve
    assert serve.draw_paths(["a/x.png", "b/y.jpg"], "o") == [os.path.join("o", "x.jpg"), os.path.join("o", "y.jpg")]
    with pytest.raises(ValueError, match="x.jpg"):
        serve.draw_paths(["a/x.png", "b/x.jpg"], "o")


def test_serve_refuses_duplicate_stems_before_any_work(tmp_path, monkeypatch):
    import serve
    d = tmp_path / "imgs"
    (d / "a").mkdir(parents=True)
    for name in ["x.png", "x.jpg"]:
        Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(d / name)
    called = []
    monkeypatch.setattr(serve, "open_pipeline", lambda *a, **k: called.append(1))
    args = serve.build_parser().parse_args(["ck.npz", str(d), "--draw", str(tmp_path / "out")])
    with pytest.raises(ValueError, match="x.jpg"):
        serve.serve(args)
    assert not called and not (tmp_path / "out").exists()
