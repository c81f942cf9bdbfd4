"""Tiling by tile size on the GPU: k2y_merge_views_ex against oracle/tiles_merge_ref.py for every metric, action and border
setting, and DetectionPipeline.enable_tiling(tile_size=...) / serve.py --tile_size against the composed reference: each
image's planned windows sent as crops through an untiled pipeline, then the oracle merge."""
import ctypes
import io
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import GOLDEN
from k210_yolo_framework_b200 import tiles
from k210_yolo_framework_b200._lib import check, lib
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline
from oracle import tiles_merge_ref as ref
from oracle import tiles_ref

IN_HW = (224, 320)
NBOX = 1050          # (7 * 10 + 14 * 20) * 3 boxes per network input
K2Y_ERR_INVALID = -1
FONT = "missing.otf"
MATCH = {"iou": 0, "ios": 1}
MERGE = {"suppress": 0, "union": 1}


# ---- the merge entry ----------------------------------------------------------------------------------------------------
def _blocks(rng, views, C, K, fill, kinds):
    """Seeded per-view record blocks for images with `views` views each: (dets [N, C, K] DET, counts [N, C], origins [N, 2],
    offsets [n + 1], sides [N], view_hw [N, 2]).  Records of a (view, class) in (score descending, index ascending) order, as
    the detector writes them; `kinds` adds score ties, one box per class seen by every view at the same place (and so at
    identical image coordinates for origins that shift it exactly), zero-area boxes and boxes at the tiles' borders."""
    offsets = np.concatenate([[0], np.cumsum(views)]).astype(np.int32)
    N = int(offsets[-1])
    dets = np.zeros((N, C, K), tiles_ref.DET)
    counts = np.zeros((N, C), np.int32)
    origins = np.zeros((N, 2), np.float32)
    sides = np.zeros(N, np.int32)
    view_hw = np.zeros((N, 2), np.float32)
    for b, V in enumerate(views):
        for v in range(V):
            g = offsets[b] + v
            if v:
                origins[g] = rng.integers(0, 400, 2)
                sides[g] = rng.integers(1, 16)
            view_hw[g] = rng.integers(150, 420, 2) if v else (600, 800)
    levels = np.float32(np.linspace(0.05, 0.99, 12))
    shared = rng.uniform(100, 400, (C, 4)).astype(np.float32)
    for g in range(N):
        for c in range(C):
            m = K if fill == "full" else 0 if fill == "empty" else int(rng.integers(0, K + 1)) if rng.random() < 0.7 else 0
            score = rng.choice(levels, m) if "ties" in kinds else rng.uniform(0.01, 1.0, m).astype(np.float32)
            index = rng.choice(NBOX, m, replace=False)
            order = np.lexsort((index, -score.astype(np.float64)))
            y, x = rng.uniform(-5, 300, m), rng.uniform(-5, 300, m)
            h, w = rng.uniform(5, 150, m), rng.uniform(5, 150, m)
            box = np.stack([y, x, y + h, x + w], 1).astype(np.float32)
            if "zero" in kinds:
                z = rng.random(m) < 0.2
                box[z, 2] = box[z, 0]
            if "edge" in kinds and m:
                e = rng.random(m) < 0.3
                box[e, 0] = rng.uniform(0, 6, int(e.sum()))
                box[e, 3] = view_hw[g, 1] - rng.uniform(-2, 6, int(e.sum()))
            if "same" in kinds and m:
                box[0] = np.round(shared[c]) - np.tile(origins[g], 2)
            rec = dets[g, c]
            for k, j in enumerate(order):
                rec[k] = (box[j, 0], box[j, 1], box[j, 2], box[j, 3], score[j], index[j])
            counts[g, c] = m
    return dets, counts, origins, offsets, sides, view_hw


def _gpu(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def _merge_ex(dets, counts, origins, offsets, sides, view_hw, max_views, thr, match, merge, border, rows=None, uniform=False):
    N, C, K = dets.shape
    n = len(offsets) - 1
    rows = n + 2 if rows is None else rows
    vd = _gpu(dets.view(np.int32).reshape(N, C, K, 6))
    vc, yx, off, sd, hw = _gpu(counts), _gpu(origins, np.float32), _gpu(offsets, np.int32), _gpu(sides, np.int32), _gpu(view_hw, np.float32)
    words = C * (K * 6 + 1)
    buf = torch.full((rows, words), -7, dtype=torch.int32, device="cuda")
    out_d = buf.as_strided((rows, C, K, 6), (words, K * 6, 6, 1))
    out_c = buf.as_strided((rows, C), (words, 1), C * K * 6)
    bordered = border is not None
    rc = lib.k2y_merge_views_ex(vd.data_ptr(), vc.data_ptr(), yx.data_ptr(), None if uniform else off.data_ptr(),
                                sd.data_ptr() if bordered else None, hw.data_ptr() if bordered else None,
                                border if bordered else -1.0, MATCH[match], MERGE[merge], n, rows, max_views, NBOX, C, K, thr,
                                out_d.data_ptr(), out_c.data_ptr(), out_d.stride(0), out_c.stride(0),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out_d.cpu().numpy(), out_c.cpu().numpy()


def _assert_equal_to_oracle(blocks, max_views, thr, match, merge, border):
    dets, counts, origins, offsets, sides, view_hw = blocks
    rc, got_d, got_c = _merge_ex(dets, counts, origins, offsets, sides, view_hw, max_views, thr, match, merge, border)
    check(rc)
    want_d, want_c = ref.merge_views(dets, counts, origins, offsets, NBOX, thr, match, merge, border, sides, view_hw)
    n = len(offsets) - 1
    np.testing.assert_array_equal(got_c[:n], want_c)
    assert (got_c[n:] == 0).all()
    got = np.ascontiguousarray(got_d[:n]).view(tiles_ref.DET)[..., 0]
    for b in range(n):
        for c in range(want_c.shape[1]):
            m = want_c[b, c]
            assert got[b, c, :m].tobytes() == want_d[b, c, :m].tobytes(), (b, c)
    return want_c


MODES = [(m, a, bd) for m in ("iou", "ios") for a in ("suppress", "union") for bd in (None, 4.0)]


@pytest.mark.parametrize("match,merge,border", MODES)
@pytest.mark.parametrize("C,K,views,thr,fill,kinds", [
    (20, 30, (1, 8, 3, 8, 1), 0.5, "random", ("edge",)), (20, 30, (8, 1, 5), 0.3, "random", ("ties", "same", "edge")),
    (1, 30, (34, 1), 0.5, "full", ("zero", "same")), (80, 100, (10, 1, 4), 0.5, "random", ("ties", "edge")),
    (1, 100, (10, 10), 0.3, "full", ("ties", "same", "edge")), (20, 30, (5, 5), 0.5, "empty", ()),
    (1, 32, (32, 1, 32), 0.0, "full", ("ties", "edge"))])
def test_merge_ex_equals_the_oracle(match, merge, border, C, K, views, thr, fill, kinds):
    """Images of one view beside images at the cap, C = 1 / 20 / 80, K = 30 / 100, and 1024 records in one merge (32 views
    x 32 records, 34 x 30)."""
    rng = np.random.default_rng(C * 1000 + K * 10 + len(views) + sum(views))
    want_c = _assert_equal_to_oracle(_blocks(rng, list(views), C, K, fill, kinds), max(views), thr, match, merge, border)
    if fill == "empty":
        assert (want_c == 0).all()
    else:
        assert want_c.sum() > 0


@pytest.mark.parametrize("match,merge", [(m, a) for m in ("iou", "ios") for a in ("suppress", "union")])
def test_merge_ex_identical_boxes(match, merge):
    """Every view holds the same boxes at the same image place: each image keeps one per place, the first view's."""
    V, C, K = 6, 3, 30
    rng = np.random.default_rng(11)
    base = rng.uniform(0, 200, (K, 4)).astype(np.float32)
    base[:, 2:] = base[:, :2] + 50
    views = [V, 1, V]
    dets, counts, origins, offsets, sides, view_hw = _blocks(rng, views, C, K, "empty", ())
    for g in range(len(dets)):
        origins[g] = (32 * (g % 3), 16 * (g % 2))
        for c in range(C):
            for k in range(K):
                b = base[k] - np.tile(origins[g], 2)
                dets[g, c, k] = (b[0], b[1], b[2], b[3], np.float32(0.9 - 0.01 * k), k)
            counts[g, c] = K
    _assert_equal_to_oracle((dets, counts, origins, offsets, sides, view_hw), V, 0.5, match, merge, None)


def test_merge_ex_with_uniform_ranges_equals_merge_views():
    rng = np.random.default_rng(4)
    V, C, K, n = 5, 20, 30, 3
    dets, counts, origins, offsets, sides, view_hw = _blocks(rng, [V] * n, C, K, "random", ("ties", "same", "zero"))
    nv = n * V
    vd = _gpu(dets.view(np.int32).reshape(nv, C, K, 6))
    vc, yx = _gpu(counts), _gpu(origins)
    old = torch.full((n + 1, C, K, 6), -7, dtype=torch.int32, device="cuda")
    old_c = torch.full((n + 1, C), -7, dtype=torch.int32, device="cuda")
    check(lib.k2y_merge_views(vd.data_ptr(), vc.data_ptr(), yx.data_ptr(), n, n + 1, V, NBOX, C, K, 0.5, old.data_ptr(), old_c.data_ptr(),
                              old.stride(0), old_c.stride(0), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for uniform in (True, False):
        rc, got_d, got_c = _merge_ex(dets, counts, origins, offsets, sides, view_hw, V, 0.5, "iou", "suppress", None, rows=n + 1,
                                     uniform=uniform)
        check(rc)
        assert (got_c == old_c.cpu().numpy()).all()
        oc = old_c.cpu().numpy()
        od = old.cpu().numpy()
        for b in range(n):
            for c in range(C):
                assert (got_d[b, c, :oc[b, c]] == od[b, c, :oc[b, c]]).all()


def test_merge_ex_minus_zero_and_nan():
    """-0.0 below +0.0 in the union (an origin of -0.0 keeps a -0.0 field through the shift), NaN fields skipped."""
    nan = np.float32("nan")
    dets = np.zeros((1, 2, 4), tiles_ref.DET)
    dets[0, 0, 0] = (0.0, 0.0, -0.0, -0.0, 0.9, 0)
    dets[0, 0, 1] = (-0.0, -0.0, 0.0, 0.0, 0.8, 1)
    dets[0, 1, 0] = (nan, 0.0, 10.0, 10.0, 0.9, 0)
    dets[0, 1, 1] = (2.0, -1.0, nan, 12.0, 0.8, 1)
    dets[0, 1, 2] = (nan, 1.0, nan, 5.0, 0.7, 2)
    counts = np.array([[2, 3]], np.int32)
    origins = np.array([[-0.0, -0.0]], np.float32)
    for match in ("iou", "ios"):
        for merge in ("suppress", "union"):
            _assert_equal_to_oracle((dets, counts, origins, np.array([0, 1]), np.zeros(1, np.int32), np.zeros((1, 2))), 1, -1.0,
                                    match, merge, None)
    rc, got_d, got_c = _merge_ex(dets, counts, origins, np.array([0, 1]), np.zeros(1, np.int32), np.zeros((1, 2)), 1, -1.0, "iou",
                                 "union", None)
    got = np.ascontiguousarray(got_d[:1]).view(tiles_ref.DET)[..., 0]
    assert got_c[0].tolist() == [1, 1]
    assert [bool(np.signbit(got[0, 0, 0][f])) for f in ("ymin", "xmin", "ymax", "xmax")] == [True, True, False, False]
    assert [float(got[0, 1, 0][f]) for f in ("ymin", "xmin", "ymax", "xmax")] == [2.0, -1.0, 10.0, 12.0]


def test_merge_ex_refuses_bad_arguments():
    dets = np.zeros((2, 2, 30), tiles_ref.DET)
    z = np.zeros((2, 2), np.int32)
    args = (dets, z, np.zeros((2, 2), np.float32), np.array([0, 2]), np.zeros(2, np.int32), np.zeros((2, 2)))
    rc, _, got_c = _merge_ex(*args, 35, 0.5, "iou", "suppress", None)          # 35 views x 30 records > 1024
    assert rc == K2Y_ERR_INVALID and (got_c == -7).all()
    rc, _, got_c = _merge_ex(*args, 2, 0.5, "iou", "suppress", float("nan"))   # a NaN border
    assert rc == K2Y_ERR_INVALID and (got_c == -7).all()
    vd = _gpu(dets.view(np.int32).reshape(2, 2, 30, 6))
    out = torch.full((1, 2, 30, 6), -7, dtype=torch.int32, device="cuda")
    for match, merge in ((2, 0), (0, 2), (-1, 0)):
        rc = lib.k2y_merge_views_ex(vd.data_ptr(), vd.data_ptr(), vd.data_ptr(), None, None, None, -1.0, match, merge, 1, 1, 2, NBOX, 2,
                                    30, 0.5, out.data_ptr(), out.data_ptr(), 2 * 30 * 6 + 2, 2 * 30 * 6 + 2, None)
        assert rc == K2Y_ERR_INVALID
    assert (out == -7).all()


# ---- end to end --------------------------------------------------------------------------------------------------------
def _pipeline(golden_weights, voc_anchors, batch, lanes=None, obj=0.3, iou=0.5):
    if lanes is None:
        p = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=obj, iou_thresh=iou)
        p.engine.set_weights(golden_weights)
    else:
        p = LanedPipeline(lanes, "yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=obj, iou_thresh=iou, sm_split=False)
        p.set_weights(golden_weights)
    return p


def _jpeg(img, quality=90):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img)).save(f, "JPEG", quality=quality)
    return f.getvalue()


def _pixels(item):
    from k210_yolo_framework_b200.helper import read_image
    return item if isinstance(item, np.ndarray) else read_image(io.BytesIO(bytes(item)))


@pytest.fixture(scope="module")
def mixed(dog_u8, people_u8):
    """224x320 (one view at 224x320 tiles), 374x499 (2x2), 748x998 (4x4, capped), 187x640 (1x2) and 300x333."""
    big = np.ascontiguousarray(np.repeat(np.repeat(people_u8, 2, 0), 2, 1))
    wide = np.ascontiguousarray(np.concatenate([people_u8[100:287, :320], dog_u8[:187]], 1))
    return [dog_u8, people_u8, big, wide, np.ascontiguousarray(people_u8[40:340, 100:433][:, ::-1])]


def _composed(plain, images, tile_hw, cap, thr=0.5, overlap=0.2, **opts):
    """What tiling by size is defined to give: every image's planned windows (oracle) as crops through the untiled pipeline
    `plain` in one batch, then the oracle merge with the options.  Per image the records as DetectionPipeline.records lists
    them."""
    pixels = [_pixels(im) for im in images]
    per = [ref.plan_windows(p.shape[0], p.shape[1], tile_hw, overlap, cap) for p in pixels]
    windows = np.concatenate(per)
    offsets = np.concatenate([[0], np.cumsum([len(w) for w in per])])
    sides = np.concatenate([ref.view_sides(w, p.shape[0], p.shape[1]) for w, p in zip(per, pixels)])
    crops = [np.ascontiguousarray(pixels[b][y0:y0 + th, x0:x0 + tw]) for b, w in enumerate(per) for y0, x0, th, tw in w.tolist()]
    d, c = plain.collect(plain.submit_images(crops))
    dets, counts = ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], offsets, NBOX, thr, sides=sides, view_hw=windows[:, 2:],
                                   **opts)
    return [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
             for cls in range(dets.shape[1]) for r in dets[b, cls, :counts[b, cls]]] for b in range(len(images))]


OPTIONS = [dict(), dict(match="ios", merge="union"), dict(match="ios", merge="suppress", border=3.0),
           dict(match="iou", merge="union", border=0.0)]


@pytest.mark.parametrize("opts", OPTIONS)
def test_sized_tiling_equals_the_composed_reference(golden_weights, voc_anchors, mixed, opts):
    """Mixed photo sizes as arrays and as JPEG bytes, batch 24 with 3 images per batch: at most 8 views an image."""
    plain = _pipeline(golden_weights, voc_anchors, 24)
    tiled = _pipeline(golden_weights, voc_anchors, 24)
    tiled.enable_tiling(tile_size=IN_HW, images_per_batch=3, **opts)
    assert tiled.images_per_batch == 3
    total, views_seen = 0, set()
    for images in ([mixed[0], mixed[1], mixed[2]], [_jpeg(mixed[2]), _jpeg(mixed[3]), mixed[4]], [_jpeg(mixed[0])]):
        d, c = tiled.collect(tiled.submit_images(images))
        got = DetectionPipeline.records(d, c)
        assert len(got) == len(images)
        assert got == _composed(plain, images, IN_HW, 8, **opts)
        total += sum(len(r) for r in got)
        views_seen |= {r[1] // NBOX for recs in got for r in recs}
    assert total > 10 and len(views_seen) > 2 and 0 in views_seen


@pytest.mark.parametrize("lanes", [None, 2])
def test_sized_tiling_in_flight_with_rendering(golden_weights, voc_anchors, mixed, lanes):
    from k210_yolo_framework_b200.draw import draw_detections
    from k210_yolo_framework_b200.helper import _COLORMAP
    batches = [[mixed[(2 * b + i) % 5] for i in range(2)] for b in range(5)]
    batches[1] = [_jpeg(batches[1][0]), batches[1][1]]
    opts = dict(match="ios", merge="union", border=2.0)
    plain = _pipeline(golden_weights, voc_anchors, 16)
    want = [_composed(plain, imgs, IN_HW, 8, **opts) for imgs in batches]
    pipe = _pipeline(golden_weights, voc_anchors, 16, lanes)
    pipe.enable_tiling(tile_size=IN_HW, images_per_batch=2, **opts)
    pipe.enable_rendering(quality=85, font_path=FONT)
    limit = 2 if lanes is None else pipe.in_flight_limit()
    tickets, got, files = [], [], []
    for i, imgs in enumerate(batches):
        tickets.append(pipe.submit_images(imgs))
        if i + 1 >= limit:
            t = tickets[i + 1 - limit]
            got.append(DetectionPipeline.records(*pipe.collect(t)))
            files.append(pipe.rendered(t))
    for t in tickets[len(got):]:
        got.append(DetectionPipeline.records(*pipe.collect(t)))
        files.append(pipe.rendered(t))
    assert got == want
    for imgs, recs, fs in zip(batches, got, files):
        for item, rec, f in zip(imgs, recs, fs):
            out = io.BytesIO()
            draw_detections(_pixels(item), rec, _COLORMAP, font_path=FONT).save(out, "JPEG", quality=85)
            assert f == out.getvalue()


def test_enable_tiling_refuses_bad_values(golden_weights, voc_anchors, mixed):
    pipe = _pipeline(golden_weights, voc_anchors, 10)
    bad = [dict(tile_size=(0, 320), images_per_batch=2), dict(tile_size=IN_HW), dict(tile_size=IN_HW, images_per_batch=0),
           dict(tile_size=IN_HW, images_per_batch=11), dict(rows=2, cols=2, images_per_batch=2), dict(rows=2, cols=2, tile_size=IN_HW,
                                                                                                      images_per_batch=2),
           dict(rows=2, cols=2, match="giou"), dict(tile_size=IN_HW, images_per_batch=2, merge="wbf"),
           dict(rows=2, cols=2, border=-1.0), dict(tile_size=IN_HW, images_per_batch=2, border=float("nan")), dict(),
           dict(tile_size=IN_HW, images_per_batch=2, overlap=1.0)]
    for kw in bad:
        with pytest.raises(ValueError):
            pipe.enable_tiling(**kw)
    assert pipe.images_per_batch == 10 and pipe._tiling is None
    pipe.enable_tiling(tile_size=IN_HW, images_per_batch=10)                 # one view per image: every image whole
    images = [mixed[0], mixed[1]]
    plain = _pipeline(golden_weights, voc_anchors, 10)
    assert DetectionPipeline.records(*pipe.collect(pipe.submit_images(images))) == _composed(plain, images, IN_HW, 1)
    with pytest.raises(ValueError):
        pipe.submit_images([mixed[0]] * 11)


def _serve_args(tmp_path, golden_weights, files_dir, batch):
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    import serve
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    return serve.build_parser().parse_args([str(ckpt), str(files_dir), "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch",
                                            str(batch), "--tile_size", "224", "320", "--tile_images", "2", "--tile_match", "ios",
                                            "--tile_merge", "union", "--tile_border", "2", "--decode_threads", "2"])


def test_serve_with_tile_size(tmp_path, golden_weights, voc_anchors, mixed):
    """serve.py --tile_size 224 320 --tile_images 2, batch 12 (at most 6 views an image, a short final batch): the JSON lines
    of the composed reference."""
    import serve
    from PIL import Image
    from k210_yolo_framework_b200.helper import read_image
    d = tmp_path / "imgs"
    d.mkdir()
    files = []
    for i, im in enumerate(mixed):
        path = d / (f"{i:02d}.png" if i % 2 else f"{i:02d}.jpg")
        Image.fromarray(im).save(path, **({} if i % 2 else {"quality": 90}))
        files.append(str(path))
    a = _serve_args(tmp_path, golden_weights, d, 12)
    out = tmp_path / "dets.jsonl"
    with open(out, "w") as fh:
        assert serve.serve(a, fh) == 5
    text = open(out).read().splitlines(keepends=True)
    plain = _pipeline(golden_weights, voc_anchors, 12, obj=0.7)
    filler = np.full(IN_HW + (3,), 128, np.uint8)
    lines = []
    for g0 in range(0, len(files), 2):
        chunk = files[g0:g0 + 2]
        imgs = [read_image(p) for p in chunk]
        recs = _composed(plain, imgs + [filler] * (2 - len(imgs)), IN_HW, 6, match="ios", merge="union", border=2.0)
        for path, rec in zip(chunk, recs):
            lines.append(json.dumps({"image": path, "detections": [
                {"class": int(c), "score": round(float(s), 6), "box_tlbr": [float(t), float(l), float(b), float(r)], "index": int(i)}
                for c, i, s, t, l, b, r in rec]}) + "\n")
    assert text == lines
    assert any(det["index"] >= NBOX for line in text for det in json.loads(line)["detections"])
