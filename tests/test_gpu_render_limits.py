"""GPU rendering (csrc/render.cu) past its one-pass limits, pixel for pixel against draw.draw_detections (or, where PIL raises,
against tests/render_ref.py): more records than one pass of the CTA, more images than one launch with gather-block strides,
a TrueType atlas per image in one launch, non-finite and huge records, and images one pixel high or wide."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from PIL import ImageFont

from render_ref import render_ref
from test_gpu_render import FONT, f32, render_gpu
from test_render_host import no_crossing, seeded_records
from k210_yolo_framework_b200.detect import DET_DTYPE
from k210_yolo_framework_b200.dist import DetectionGather
from k210_yolo_framework_b200.draw import box_geometry, draw_detections
from k210_yolo_framework_b200.helper import _COLORMAP
from k210_yolo_framework_b200.render import LabelAtlas, render_detections_device

RENDER_THREADS = 256                       # csrc/render.cu: records per pass (test_image_limits checks it)
RECORD_COUNTS = [255, 256, 257, 512, 513]
MANY = (8000, 80, 100)                     # records, C, K: evaluate_coco.py's defaults fill every class
IMAGE_COUNTS = [130, 257]
FONT_HEIGHTS = [17, 50, 224, 375, 700, 1080, 2000]   # TrueType sizes 1, 2, 7, 11, 21, 32, 60
NON_FINITE = [float("inf"), float("-inf"), float("nan"), 1e30, -1e30]
BAD_SCORES = [float("nan"), -0.5, 1.5, float("inf"), float("-inf")]


def boxes(h, w, n, seed):
    """n (score, top, left, bottom, right) float32 boxes draw_detections can draw on an h x w image: clipped at every edge,
    overlapping, of many sizes."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        t, l = rng.uniform(-0.1 * h, 0.95 * h), rng.uniform(-0.1 * w, 0.95 * w)
        bh, bw = rng.uniform(2, 0.6 * h), rng.uniform(2, 0.6 * w)
        rec = (0, 0) + tuple(float(np.float32(v)) for v in (rng.uniform(0, 1), t, l, t + bh, l + bw))
        if no_crossing(rec, h, w):
            out.append(rec[2:])
    return out


def by_position(bxs, per_class):
    """Records in to_host order whose class is position // per_class, so that position p's class changes at the boundaries."""
    return [(p // per_class, p) + b for p, b in enumerate(bxs)]


def assert_pil(imgs, found_per_image, C, K, font=FONT, atlas=None):
    got = render_gpu(imgs, found_per_image, C, K, atlas=atlas or LabelAtlas(C, font))
    for i, (g, x, f) in enumerate(zip(got, imgs, found_per_image)):
        ref = np.array(draw_detections(x, f, _COLORMAP, font_path=font))
        assert np.array_equal(g, ref), (i, x.shape, len(f), int((g != ref).any(-1).sum()))


def test_record_passes_and_paint_order_across_them():
    """255..513 records: records 255 / 256 and 511 / 512 are the same box in two classes, so a later pass painting before
    an earlier one (or a pass skipped) changes pixels."""
    h, w = 300, 400
    imgs, found = [], []
    for i, n in enumerate(RECORD_COUNTS):
        bxs = boxes(h, w, n, 50 + i)
        for a in (RENDER_THREADS - 1, 2 * RENDER_THREADS - 1):
            if a + 1 < n:
                bxs[a + 1] = (bxs[a + 1][0],) + bxs[a][1:]       # the same box, another score (and class)
        found.append(by_position(bxs, RENDER_THREADS))
        imgs.append(np.random.default_rng(i).integers(0, 256, (h, w, 3), dtype=np.uint8))
    assert found[2][255][3:] == found[2][256][3:] and found[2][255][0] != found[2][256][0]
    assert_pil(imgs, found, C=20, K=RENDER_THREADS)


def test_eight_thousand_records():
    n, C, K = MANY
    h, w = 600, 800
    found = by_position(boxes(h, w, n, 7), K)
    assert found[-1][0] == C - 1
    assert_pil([np.full((h, w, 3), 128, np.uint8)], [found], C=C, K=K)


def gather_block(found_per_image, C, K):
    """Records in a DetectionGather buffer: per image C*K*6 record words, then its C counts (stride C*(K*6+1))."""
    n = len(found_per_image)
    rec = np.zeros((n, C, K), DET_DTYPE)
    counts = np.zeros((n, C), np.int32)
    for i, found in enumerate(found_per_image):
        for c, idx, s, t, l, b, r in found:
            rec[i, c, counts[i, c]] = (t, l, b, r, s, idx)
            counts[i, c] += 1
    buf = np.zeros((n, C * (K * 6 + 1)), np.int32)
    buf[:, :C * K * 6] = rec.view(np.int32).reshape(n, -1)
    buf[:, C * K * 6:] = counts
    return DetectionGather.split(torch.from_numpy(buf).cuda(), C, K)


@pytest.mark.parametrize("n", IMAGE_COUNTS)
def test_launch_groups_with_gather_block_strides(n):
    C, K = 20, 4
    shapes = [(17 + (i * 5) % 41, 30 + (i * 11) % 67) for i in range(n)]
    imgs = [np.random.default_rng(i).integers(0, 256, s + (3,), dtype=np.uint8) for i, s in enumerate(shapes)]
    assert all((h + w) // 300 == 0 for h, w in shapes)      # no rings: every seeded record is kept
    found = [seeded_records(h, w, 1 + i % K, C, 1000 + i) for i, (h, w) in enumerate(shapes)]
    dets, counts = gather_block(found, C, K)
    assert dets.stride(0) == counts.stride(0) > C * K * 6
    views = [torch.from_numpy(x).cuda() for x in imgs]
    render_detections_device(views, dets, counts, LabelAtlas(C, FONT))
    torch.cuda.synchronize()
    for i, (v, x, f) in enumerate(zip(views, imgs, found)):
        ref = np.array(draw_detections(x, f, _COLORMAP, font_path=FONT))
        assert np.array_equal(v.cpu().numpy(), ref), (i, x.shape)
    assert all(len(f) for f in found[128:])


def edge_records(h, w, seed):
    """Records whose labels cross every edge the label can reach (right, bottom, above the bottom for top >= h) and the
    32x8 tile boundaries, plus seeded ones; all drawable by PIL."""
    th = (h + w) // 300
    cand = []
    for k in range(1, 6):
        x, y = 32 * k * max(1, w // 200) - 3, 8 * k * max(1, h // 100) - 2
        cand.append((float(y), float(x) + 0.25, float(y + 3 * th + 20), float(x + 4 * th + 30)))
    cand += [(h * 0.3, w - 2.0 * th - 3.0, h * 0.6, w + 50.0),        # label runs off the right edge
             (h - 2.0 * th - 1.0, w * 0.2, h + 40.0, w * 0.7),        # label runs off the bottom edge
             (h + 0.3, w * 0.4, h + 9.0, w * 0.9),                    # top >= h: label above the bottom edge
             (-7.0, -9.0, h * 0.5, w * 0.5)]                          # clipped at the top-left
    rng = np.random.default_rng(seed)
    found = [(int(rng.integers(0, 20)), k, float(np.float32(rng.uniform(0, 1))), *map(float, np.float32(c))) for k, c in enumerate(cand)]
    found = [r for r in found if no_crossing(r, h, w)]
    found += [(c, 100 + k, *rest) for k, (c, _i, *rest) in enumerate(seeded_records(h, w, 12, 20, seed))]
    found.sort(key=lambda r: r[0])
    return found


def test_truetype_atlas_per_image_in_one_launch(tmp_path):
    ttf = tmp_path / "default.ttf"
    ttf.write_bytes(ImageFont.load_default().font_bytes)
    atlas = LabelAtlas(20, str(ttf))
    imgs, found = [], []
    for i, h in enumerate(FONT_HEIGHTS):
        w = int(1.3 * h) + 5
        imgs.append(np.random.default_rng(h).integers(0, 256, (h, w, 3), dtype=np.uint8))
        f = edge_records(h, w, h)
        off_right = off_bottom = False
        for c, _i, s, *box in f:
            _m, _o, (lw, lh) = atlas_glyphs(atlas, h, c, s)
            *_, (ox, oy) = box_geometry((h, w), box, (lw, lh))
            off_right |= ox + lw >= w
            off_bottom |= oy + lh >= h
        assert off_right and off_bottom, h
        found.append(f)
    assert_pil(imgs, found, C=20, K=40, font=str(ttf), atlas=atlas)
    dev = torch.device("cuda", torch.cuda.current_device())
    assert len({atlas.device(h, dev).data_ptr() for h in FONT_HEIGHTS}) >= 4


def atlas_glyphs(atlas, h, cls, score):
    from render_ref import atlas_entry, clamped_hundredths
    return atlas_entry(atlas.host(h), cls, clamped_hundredths(score))


def non_finite_records(h, w):
    out, k = [], 0
    for j in range(4):
        for v in NON_FINITE:
            box = [0.2 * h, 0.2 * w, 0.7 * h, 0.8 * w]
            box[j] = v
            out.append((k % 20, k, BAD_SCORES[k % len(BAD_SCORES)], *box))
            k += 1
    for s in BAD_SCORES:
        out.append((k % 20, k, s, 0.1 * h + k, 0.1 * w + k, 0.5 * h, 0.6 * w))
        k += 1
    out.sort(key=lambda r: r[0])
    return out


def test_non_finite_and_huge_records_follow_the_documented_clamps():
    shapes = [(200, 300), (700, 900)]
    imgs = [np.full(s + (3,), 100 + 50 * i, np.uint8) for i, s in enumerate(shapes)]
    found = [non_finite_records(h, w) for h, w in shapes]
    atlas = LabelAtlas(20, FONT)
    got = render_gpu(imgs, found, C=20, K=40, atlas=atlas)
    for g, x, f in zip(got, imgs, found):
        ref = render_ref(x, f, _COLORMAP, atlas.host(x.shape[0]))
        assert np.array_equal(g, ref), (x.shape, int((g != ref).any(-1).sum()))
        assert (ref != x).any()


def test_one_pixel_high_or_wide_images():
    shapes = [(1, 1), (1, 300), (300, 1)]
    imgs = [np.random.default_rng(i).integers(0, 256, s + (3,), dtype=np.uint8) for i, s in enumerate(shapes)]
    found = [f32([(0, 0, 0.5, 0.0, 0.0, 1.0, 1.0), (3, 1, 0.25, -5.0, -5.0, 10.0, 10.0), (3, 2, 0.75, 0.4, 0.6, 0.4, 0.6)]),
             f32([(1, 0, 0.9, 0.0, 10.0, 1.0, 200.0), (2, 1, 0.1, -3.0, 150.0, 4.0, 400.0), (5, 2, 1.0, 0.0, 290.0, 0.0, 299.0)]),
             f32([(1, 0, 0.9, 10.0, 0.0, 200.0, 1.0), (2, 1, 0.1, 150.0, -3.0, 400.0, 4.0), (5, 2, 1.0, 299.0, 0.0, 310.0, 0.0)])]
    atlas = LabelAtlas(20, FONT)
    got = render_gpu(imgs, found, atlas=atlas)
    for g, x, f in zip(got, imgs, found):
        assert np.array_equal(g, render_ref(x, f, _COLORMAP, atlas.host(x.shape[0]))), x.shape
    # 300 rows: PIL's label font exists (below 17 rows draw_detections raises for the font size), so compare with PIL too
    assert np.array_equal(got[2], np.array(draw_detections(imgs[2], found[2], _COLORMAP, font_path=FONT)))
