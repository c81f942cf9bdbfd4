"""Test-time flip on the GPU, bit for bit: the mirrored letterbox (k2y_letterbox_u8_views_mirror) against
oracle/preprocess_ref.py on np.fliplr of each window, k2y_merge_views_mirror against oracle/flip_ref.py, and
DetectionPipeline.enable_flip / serve.py --flip against the composed reference: every crop and every mirrored crop through an
unflipped, untiled pipeline, then the oracle merge."""
import ctypes
import io
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import preprocess, tiles
from k210_yolo_framework_b200._lib import check, lib
from k210_yolo_framework_b200.pipeline import DetectionPipeline
from oracle import flip_ref, preprocess_ref
from oracle import tiles_merge_ref as ref
from oracle import tiles_ref
from test_gpu_tiles_sized import (FONT, IN_HW, MATCH, MERGE, NBOX, _blocks, _gpu, _jpeg, _pipeline, _pixels, _serve_args,
                                  mixed)  # noqa: F401  (mixed is a fixture)

K2Y_ERR_INVALID = -1


def _synthetic(hw, lo, seed):
    return np.random.default_rng(seed).integers(lo, 256, (hw[0], hw[1], 3), dtype=np.uint8)


# ---- the mirrored letterbox -----------------------------------------------------------------------------------------------
def _letterbox_views(images, windows, mirror, per_image):
    """k2y_letterbox_u8_views_mirror on `images` packed as BatchLayout packs them; `per_image[i]` is the image of view i."""
    layout = preprocess.BatchLayout(images, IN_HW)
    packed = np.zeros(layout.nbytes, np.uint8)
    layout.pack(images, packed)
    src = torch.from_numpy(packed).cuda()
    nv = len(windows)
    windows = np.ascontiguousarray(windows, np.int32)
    mirror = None if mirror is None else np.ascontiguousarray(mirror, np.int32)
    offsets = np.ascontiguousarray(layout.offsets[per_image])
    hw = np.ascontiguousarray(layout.hw[per_image])
    mats = np.array([preprocess.letterbox_params((t[2], t[3]), IN_HW)[2][:2].reshape(-1) for t in windows.tolist()], np.float64)
    out = torch.full((nv + 1,) + IN_HW + (3,), 77, dtype=torch.uint8, device="cuda")
    view_hw = torch.full((nv + 1, 2), -1.0, device="cuda")
    view_yx = torch.full((nv + 1, 2), -1.0, device="cuda")
    minmax = torch.empty((nv, 2), dtype=torch.int32, device="cuda")
    rc = lib.k2y_letterbox_u8_views_mirror(src.data_ptr(), nv, offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                           hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                           windows.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                           None if mirror is None else mirror.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                           mats.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), out.data_ptr(), IN_HW[0], IN_HW[1],
                                           view_hw.data_ptr(), view_yx.data_ptr(), minmax.data_ptr(),
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out, view_hw, view_yx


def _assert_equal_to_the_flipped_crops(images, windows, mirror, per_image):
    rc, out, view_hw, view_yx = _letterbox_views(images, windows, mirror, per_image)
    check(rc)
    got = out.cpu().numpy()
    for i, ((y0, x0, th, tw), m) in enumerate(zip(windows.tolist(), mirror)):
        crop = images[per_image[i]][y0:y0 + th, x0:x0 + tw]
        want = preprocess_ref.letterbox(np.ascontiguousarray(np.fliplr(crop) if m else crop), IN_HW)
        assert np.array_equal(got[i], want), (i, (y0, x0, th, tw), m)
    assert view_hw[:len(windows)].cpu().numpy().tolist() == windows[:, 2:].tolist()
    assert view_yx[:len(windows)].cpu().numpy().tolist() == windows[:, :2].tolist()
    assert (got[len(windows)] == 77).all()


def test_mirrored_letterbox_hand_made_windows():
    """Odd and even widths, 1-pixel-wide windows, windows on each edge of the image, a bright image (minimum 30) and a window
    row longer than one block's chunk; each window plain and mirrored."""
    img = _synthetic((97, 131), 30, 1)
    even = _synthetic((64, 90), 0, 3)
    big = _synthetic((60, 6000), 0, 2)
    windows = [(0, [0, 0, 97, 131]), (0, [0, 0, 97, 1]), (0, [0, 130, 97, 1]), (0, [0, 0, 1, 131]), (0, [96, 0, 1, 131]),
               (0, [50, 77, 1, 1]), (0, [13, 17, 40, 51]), (0, [0, 0, 40, 60]), (0, [0, 71, 40, 60]), (0, [57, 0, 40, 60]),
               (0, [57, 71, 40, 60]), (1, [0, 0, 64, 90]), (1, [5, 3, 50, 44]), (1, [0, 1, 64, 2]), (2, [0, 0, 60, 6000]),
               (2, [3, 1, 50, 5999])]
    per_image = np.array([i for i, _ in windows] * 2)
    win = np.array([w for _, w in windows] * 2, np.int32)
    mirror = np.array([0] * len(windows) + [1] * len(windows), np.int32)
    _assert_equal_to_the_flipped_crops([img, even, big], win, mirror, per_image)


def test_mirrored_letterbox_more_than_one_launch_group(dog_u8, people_u8):
    """2x2 tiles of 6 images, plain then mirrored: 60 views, so a second group of 48 runs, with flags on both sides of it."""
    images = [dog_u8, people_u8, _synthetic((375, 500), 0, 4), _synthetic((33, 61), 25, 5), _synthetic((480, 641), 40, 6),
              np.ascontiguousarray(people_u8[40:, 31:450])]
    per, per_image, mirror = [], [], []
    for b, im in enumerate(images):
        w, m = tiles.mirror_views(tiles.tile_windows(im.shape[0], im.shape[1], 2, 2, 0.2))
        per.append(w)
        per_image += [b] * len(w)
        mirror.append(m)
    windows, mirror = np.concatenate(per), np.concatenate(mirror)
    assert len(windows) == 60
    _assert_equal_to_the_flipped_crops(images, windows, mirror, np.array(per_image))


def test_mirrored_letterbox_with_no_flags_is_the_plain_letterbox():
    img = _synthetic((97, 131), 0, 7)
    windows = np.array([[0, 0, 97, 131], [10, 20, 50, 61]], np.int32)
    rc, a, _, _ = _letterbox_views([img], windows, None, np.zeros(2, int))
    check(rc)
    rc, b, _, _ = _letterbox_views([img], windows, np.zeros(2, np.int32), np.zeros(2, int))
    check(rc)
    assert torch.equal(a, b)
    _assert_equal_to_the_flipped_crops([img], windows, np.zeros(2, np.int32), np.zeros(2, int))


# ---- the merge entry ------------------------------------------------------------------------------------------------------
def _merge_mirror(blocks, mirror, max_views, thr, match, merge, border, uniform=False):
    dets, counts, origins, offsets, sides, view_hw = blocks
    N, C, K = dets.shape
    n = len(offsets) - 1
    rows = n + 2
    vd = _gpu(dets.view(np.int32).reshape(N, C, K, 6))
    vc, yx, off, sd, hw = _gpu(counts), _gpu(origins, np.float32), _gpu(offsets, np.int32), _gpu(sides, np.int32), _gpu(view_hw, np.float32)
    mr = _gpu(mirror, np.int32)
    words = C * (K * 6 + 1)
    buf = torch.full((rows, words), -7, dtype=torch.int32, device="cuda")
    out_d = buf.as_strided((rows, C, K, 6), (words, K * 6, 6, 1))
    out_c = buf.as_strided((rows, C), (words, 1), C * K * 6)
    bordered = border is not None
    rc = lib.k2y_merge_views_mirror(vd.data_ptr(), vc.data_ptr(), yx.data_ptr(), None if uniform else off.data_ptr(),
                                    sd.data_ptr() if bordered else None, mr.data_ptr(), hw.data_ptr(),
                                    border if bordered else -1.0, MATCH[match], MERGE[merge], n, rows, max_views, NBOX, C, K, thr,
                                    out_d.data_ptr(), out_c.data_ptr(), out_d.stride(0), out_c.stride(0),
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out_d.cpu().numpy(), out_c.cpu().numpy()


def _assert_merge_equal_to_oracle(blocks, mirror, max_views, thr, match, merge, border, uniform=False):
    dets, counts, origins, offsets, sides, view_hw = blocks
    rc, got_d, got_c = _merge_mirror(blocks, mirror, max_views, thr, match, merge, border, uniform)
    check(rc)
    want_d, want_c = flip_ref.merge_views(dets, counts, origins, offsets, NBOX, thr, match, merge, border, sides, view_hw, mirror)
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
@pytest.mark.parametrize("C,K,views,thr,kinds,uniform", [
    (20, 30, (2, 10, 6, 10, 2), 0.5, ("edge",), False), (20, 30, (10, 2, 6), 0.3, ("ties", "same", "edge"), False),
    (80, 100, (10, 2, 4), 0.5, ("ties", "edge", "zero"), False), (1, 32, (32, 2, 32), 0.0, ("ties", "edge"), False),
    (20, 30, (10, 10, 10), 0.5, ("ties", "edge"), True), (1, 100, (10, 10), 0.3, ("ties", "same", "edge"), True)])
def test_merge_mirror_equals_the_oracle(match, merge, border, C, K, views, thr, kinds, uniform):
    """Per-image and uniform view ranges; each image's second half of views mirrored, and a few plain views flagged at random
    too, so mirrored and plain views mix in one image."""
    rng = np.random.default_rng(C * 1000 + K * 10 + len(views) + sum(views) + uniform)
    blocks = _blocks(rng, list(views), C, K, "random", kinds)
    mirror = np.zeros(int(sum(views)), np.int32)
    offsets = blocks[3]
    for b, V in enumerate(views):
        mirror[offsets[b] + V // 2:offsets[b + 1]] = 1
    mirror[rng.random(len(mirror)) < 0.1] ^= 1
    want_c = _assert_merge_equal_to_oracle(blocks, mirror, max(views), thr, match, merge, border, uniform)
    assert want_c.sum() > 0


@pytest.mark.parametrize("match,merge", [(m, a) for m in ("iou", "ios") for a in ("suppress", "union")])
def test_merge_mirror_minus_zero_and_nan(match, merge):
    """-0.0 and tw in x (tw - tw = +0.0, tw - -0.0 = tw), NaN fields of every kind in mirrored and plain views."""
    nan = np.float32("nan")
    neg_nan = np.array(0xffc00123, np.uint32).view(np.float32)
    dets = np.zeros((2, 2, 4), tiles_ref.DET)
    dets[0, 0, 0] = (0.0, -0.0, 10.0, 64.0, 0.9, 0)
    dets[1, 0, 0] = (-0.0, 0.0, 0.0, -0.0, 0.8, 1)
    dets[1, 0, 1] = (1.0, 64.0, 5.0, 64.0, 0.7, 2)
    dets[0, 1, 0] = (nan, 0.0, 10.0, 10.0, 0.9, 0)
    dets[1, 1, 0] = (2.0, neg_nan, nan, 12.0, 0.8, 1)
    dets[1, 1, 1] = (nan, 1.0, neg_nan, nan, 0.7, 2)
    counts = np.array([[1, 1], [2, 2]], np.int32)
    blocks = (dets, counts, np.array([[-0.0, -0.0], [0.0, 0.0]], np.float32), np.array([0, 2]), np.array([0, 0], np.int32),
              np.array([[10, 64], [10, 64]], np.float32))
    for mirror in ([0, 1], [1, 1], [1, 0]):
        _assert_merge_equal_to_oracle(blocks, np.array(mirror, np.int32), 2, -1.0, match, merge, None)
        _assert_merge_equal_to_oracle(blocks, np.array(mirror, np.int32), 2, 2.0, match, merge, None)


def test_merge_mirror_refuses_flags_without_view_sizes():
    dets = np.zeros((2, 2, 30), tiles_ref.DET)
    vd = _gpu(dets.view(np.int32).reshape(2, 2, 30, 6))
    mr = _gpu(np.ones(2, np.int32))
    out = torch.full((1, 2, 30, 6), -7, dtype=torch.int32, device="cuda")
    rc = lib.k2y_merge_views_mirror(vd.data_ptr(), vd.data_ptr(), vd.data_ptr(), None, None, mr.data_ptr(), None, -1.0, 0, 0, 1, 1, 2,
                                    NBOX, 2, 30, 0.5, out.data_ptr(), out.data_ptr(), 2 * 30 * 6 + 2, 2 * 30 * 6 + 2, None)
    assert rc == K2Y_ERR_INVALID and bool((out == -7).all())


# ---- end to end -----------------------------------------------------------------------------------------------------------
def _windows(pixels, grid):
    h, w = pixels.shape[:2]
    if grid is None:
        return np.array([(0, 0, h, w)], np.int32)
    if grid[0] == "grid":
        return tiles_ref.tile_windows(h, w, grid[1], grid[2], 0.2)
    return ref.plan_windows(h, w, grid[1], 0.2, grid[2])


def _composed(plain, images, grid, thr=0.5, **opts):
    """What flip is defined to give: every image's windows, then the same windows mirrored, as crops (np.fliplr for the
    mirrored ones) through the plain pipeline in one batch, then the oracle merge with the flags."""
    pixels = [_pixels(im) for im in images]
    per = [_windows(p, grid) for p in pixels]
    crops, windows, sides, mirror, counts = [], [], [], [], []
    for p, w in zip(pixels, per):
        cut = [np.ascontiguousarray(p[y0:y0 + th, x0:x0 + tw]) for y0, x0, th, tw in w.tolist()]
        crops += cut + [np.ascontiguousarray(np.fliplr(c)) for c in cut]
        windows += [w, w]
        s = ref.view_sides(w, p.shape[0], p.shape[1])
        sides += [s, s]
        mirror += [np.zeros(len(w), np.int32), np.ones(len(w), np.int32)]
        counts.append(2 * len(w))
    windows, sides, mirror = np.concatenate(windows), np.concatenate(sides), np.concatenate(mirror)
    offsets = np.concatenate([[0], np.cumsum(counts)])
    d, c = plain.collect(plain.submit_images(crops))
    dets, cnt = flip_ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], offsets, NBOX, thr, sides=sides, view_hw=windows[:, 2:],
                                mirrored=mirror, **opts)
    return [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
             for cls in range(dets.shape[1]) for r in dets[b, cls, :cnt[b, cls]]] for b in range(len(images))]


@pytest.mark.parametrize("grid,flip_first,opts", [
    (None, True, dict()), (None, True, dict(match="ios", merge="union")), (("grid", 2, 2), False, dict()),
    (("grid", 2, 2), True, dict(match="ios", merge="union", border=3.0)), (("size", IN_HW, 4), False, dict(match="ios", border=2.0)),
    (("size", IN_HW, 4), True, dict())])
def test_flip_equals_the_composed_reference(golden_weights, voc_anchors, mixed, grid, flip_first, opts):
    """Arrays and JPEG bytes, two batches in flight; a 2x2 grid of 10 views an image, or a sized grid capped at 8 // 2 = 4
    windows."""
    batch = 20 if grid is not None and grid[0] == "grid" else 16
    plain = _pipeline(golden_weights, voc_anchors, batch)
    pipe = _pipeline(golden_weights, voc_anchors, batch)

    def tile():
        if grid is not None and grid[0] == "grid":
            pipe.enable_tiling(grid[1], grid[2], 0.2, **opts)
        elif grid is not None:
            pipe.enable_tiling(tile_size=grid[1], images_per_batch=2, **opts)
    if flip_first:
        pipe.enable_flip(**({} if grid is not None else opts))
        tile()
    else:
        tile()
        pipe.enable_flip()
    assert pipe.images_per_batch == (2 if grid is not None else 8)
    batches = [[mixed[0], _jpeg(mixed[1])], [mixed[2], mixed[3]], [_jpeg(mixed[4])]]
    tickets = [pipe.submit_images(batches[0]), pipe.submit_images(batches[1])]
    got = [DetectionPipeline.records(*pipe.collect(tickets[0]))]
    tickets.append(pipe.submit_images(batches[2]))
    got += [DetectionPipeline.records(*pipe.collect(t)) for t in tickets[1:]]
    want = [_composed(plain, imgs, grid, **opts) for imgs in batches]
    assert got == want
    assert sum(len(recs) for b in got for recs in b) > 5


def test_flip_on_lanes_with_rendering(golden_weights, voc_anchors, mixed):
    from k210_yolo_framework_b200.draw import draw_detections
    from k210_yolo_framework_b200.helper import _COLORMAP
    batches = [[mixed[(2 * b + i) % 5] for i in range(2)] for b in range(4)]
    batches[1] = [_jpeg(batches[1][0]), batches[1][1]]
    plain = _pipeline(golden_weights, voc_anchors, 20)
    want = [_composed(plain, imgs, ("grid", 2, 2), match="ios", merge="union") for imgs in batches]
    pipe = _pipeline(golden_weights, voc_anchors, 20, lanes=2)
    pipe.enable_flip(match="ios", merge="union")
    pipe.enable_tiling(2, 2, 0.2, match="ios", merge="union")
    pipe.enable_rendering(quality=85, font_path=FONT)
    limit = pipe.in_flight_limit()
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


def test_enable_flip_refusals_leave_the_pipeline_as_it_was(golden_weights, voc_anchors, mixed):
    pipe = _pipeline(golden_weights, voc_anchors, 9)
    pipe.enable_tiling(2, 2, 0.2)
    with pytest.raises(ValueError):
        pipe.enable_flip()                                   # 10 views, batch 9
    assert pipe.images_per_batch == 1 and pipe._views == 5 and not pipe._flip
    unflipped = _pipeline(golden_weights, voc_anchors, 9)
    unflipped.enable_tiling(2, 2, 0.2)
    got = DetectionPipeline.records(*pipe.collect(pipe.submit_images([mixed[1]])))
    assert got == DetectionPipeline.records(*unflipped.collect(unflipped.submit_images([mixed[1]])))
    small = _pipeline(golden_weights, voc_anchors, 3)
    small.enable_tiling(tile_size=IN_HW, images_per_batch=3)
    with pytest.raises(ValueError):
        small.enable_flip()                                  # max_views 1
    assert small.images_per_batch == 3 and small._views == 1 and not small._flip


def test_serve_with_flip(tmp_path, golden_weights, voc_anchors, mixed):
    """serve.py --flip and --flip --tiles 2 2, batch 20: the JSON lines of the composed reference."""
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
    base = _serve_args(tmp_path, golden_weights, d, 20)
    plain = _pipeline(golden_weights, voc_anchors, 20, obj=0.7)
    filler = np.full(IN_HW + (3,), 128, np.uint8)       # serve.py fills a short last batch up to images_per_batch
    for grid, ipb in ((None, 10), (("grid", 2, 2), 2)):
        a = serve.build_parser().parse_args([base.ckpt, str(d), "--anchors", base.anchors, "--batch", "20", "--flip",
                                             "--decode_threads", "2"] + ([] if grid is None else ["--tiles", "2", "2"]))
        out = tmp_path / "dets.jsonl"
        with open(out, "w") as fh:
            assert serve.serve(a, fh) == 5
        text = open(out).read().splitlines(keepends=True)
        lines = []
        for g0 in range(0, len(files), ipb):
            chunk = files[g0:g0 + ipb]
            imgs = [read_image(p) for p in chunk]
            recs = _composed(plain, imgs + [filler] * (ipb - len(imgs)), grid)
            for path, rec in zip(chunk, recs):
                lines.append(json.dumps({"image": path, "detections": [
                    {"class": int(c), "score": round(float(s), 6), "box_tlbr": [float(t), float(l), float(b), float(r)], "index": int(i)}
                    for c, i, s, t, l, b, r in rec]}) + "\n")
        assert text == lines, grid
        assert any(det["index"] >= NBOX * (1 if grid is None else 5) for line in text for det in json.loads(line)["detections"])
