"""Tiled detection on the GPU: the letterbox of views (k2y_letterbox_u8_views) against the letterbox of the numpy crops, the
merge of views (k2y_merge_views) against oracle/tiles_ref.py, and DetectionPipeline.enable_tiling / serve.py --tiles against
the composed reference: an untiled pipeline fed the crops, then the oracle merge."""
import ctypes
import io
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import GOLDEN
from k210_yolo_framework_b200 import preprocess, tiles
from k210_yolo_framework_b200._lib import check, lib
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline
from oracle import tiles_ref

IN_HW = (224, 320)
K2Y_ERR_INVALID = -1
NBOX = 1050          # (7 * 10 + 14 * 20) * 3 boxes per network input
FONT = "missing.otf"  # PIL's default font, as draw_detections falls back to it


def _synthetic(hw, lo, seed):
    return np.random.default_rng(seed).integers(lo, 256, (hw[0], hw[1], 3), dtype=np.uint8)


@pytest.fixture(scope="module")
def photos(dog_u8, people_u8):
    return [dog_u8, people_u8, dog_u8[:, ::-1], people_u8[:, ::-1], people_u8[40:, 30:450], dog_u8[10:200, 20:],
            np.ascontiguousarray(people_u8[::-1])]


def _jpeg(img, quality=90):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img)).save(f, "JPEG", quality=quality)
    return f.getvalue()


def _crops(images, windows):
    """The numpy crops of `windows` [n * V, 4], image-major."""
    V = len(windows) // len(images)
    return [np.ascontiguousarray(images[i // V][y0:y0 + th, x0:x0 + tw]) for i, (y0, x0, th, tw) in enumerate(windows.tolist())]


# ---- the letterbox of views ---------------------------------------------------------------------------------------------
def _letterbox_views(images, windows, in_hw=IN_HW):
    """k2y_letterbox_u8_views on `images` packed as BatchLayout packs them, windows [n * V, 4] image-major."""
    layout = preprocess.BatchLayout(images, in_hw)
    V = len(windows) // len(images)
    packed = np.zeros(layout.nbytes, np.uint8)
    layout.pack(images, packed)
    src = torch.from_numpy(packed).cuda()
    nv = len(windows)
    windows = np.ascontiguousarray(windows, np.int32)
    offsets = np.repeat(layout.offsets, V)
    hw = np.ascontiguousarray(np.repeat(layout.hw, V, axis=0))
    mats = np.array([preprocess.letterbox_params((max(t[2], 1), max(t[3], 1)), in_hw)[2][:2].reshape(-1) for t in windows.tolist()], np.float64)
    out = torch.full((nv + 1,) + tuple(in_hw) + (3,), 77, dtype=torch.uint8, device="cuda")
    view_hw = torch.full((nv + 1, 2), -1.0, device="cuda")
    view_yx = torch.full((nv + 1, 2), -1.0, device="cuda")
    minmax = torch.empty((nv, 2), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream()
    rc = lib.k2y_letterbox_u8_views(src.data_ptr(), nv, offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                    hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), windows.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                    mats.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), out.data_ptr(), in_hw[0], in_hw[1],
                                    view_hw.data_ptr(), view_yx.data_ptr(), minmax.data_ptr(), ctypes.c_void_p(st.cuda_stream))
    torch.cuda.synchronize()
    return rc, out, view_hw, view_yx


def _assert_views_equal_crops(images, windows, in_hw=IN_HW):
    rc, out, view_hw, view_yx = _letterbox_views(images, windows, in_hw)
    check(rc)
    nv = len(windows)
    want = preprocess.letterbox_batch_device(_crops(images, windows), in_hw)
    assert torch.equal(out[:nv], want)
    assert view_hw[:nv].cpu().numpy().tolist() == windows[:, 2:].tolist()
    assert view_yx[:nv].cpu().numpy().tolist() == windows[:, :2].tolist()
    assert bool((out[nv] == 77).all()) and bool((view_hw[nv] == -1).all()) and bool((view_yx[nv] == -1).all())
    return out[:nv]


MIXED = [((375, 500), 0), ((100, 37), 0), ((224, 320), 0), ((480, 640), 40), ((33, 61), 25), ((720, 1280), 1), ((500, 333), 90)]


@pytest.mark.parametrize("rows,cols,overlap", [(1, 1, 0.2), (2, 2, 0.0), (2, 2, 0.5), (3, 3, 0.0), (3, 3, 0.5), (1, 4, 0.5), (4, 1, 0.0)])
def test_views_letterbox_equals_the_crops(photos, rows, cols, overlap):
    """Mixed photo sizes and synthetic images whose minimum is above 0 (so a tile's fill pixels must stay zero although its
    neighbours in the image are not): every view is, byte for byte, the letterbox of its numpy crop.  3x3 over ten images is
    100 views: more than the 48 one launch carries."""
    images = [np.ascontiguousarray(p) for p in photos[:3]] + [_synthetic(hw, lo, hw[0] + hw[1]) for hw, lo in MIXED]
    windows = np.concatenate([tiles.tile_windows(im.shape[0], im.shape[1], rows, cols, overlap) for im in images])
    out = _assert_views_equal_crops(images, windows)
    if (rows, cols) == (3, 3):
        assert len(windows) == 100
    # a tall tile of a bright image is letterboxed with fill on both sides, and the fill is zero
    if (rows, cols, overlap) == (1, 4, 0.5):
        V = 5
        tile = out[(3 + 3) * V + 2].cpu().numpy()          # MIXED[3]: minimum 40
        assert (tile[:, 0] == 0).all() and (tile[:, -1] == 0).all() and tile.max() > 40


def test_views_letterbox_hand_made_windows():
    """Windows touching every edge, one pixel wide, one pixel high, a single pixel, an interior window of a bright image, and
    odd origins (rows that start at any byte alignment)."""
    img = _synthetic((97, 131), 30, 1)
    big = _synthetic((300, 6000), 0, 2)                    # a window row longer than one block's chunk of pass 1
    windows = np.array([[0, 0, 97, 131], [0, 0, 97, 1], [0, 130, 97, 1], [0, 0, 1, 131], [96, 0, 1, 131], [50, 77, 1, 1],
                        [13, 17, 40, 51], [1, 1, 95, 129], [0, 5, 97, 126], [7, 0, 90, 131],
                        [0, 0, 300, 6000], [3, 1, 290, 5990], [100, 2999, 7, 3001], [299, 0, 1, 6000], [0, 5999, 300, 1]], np.int32)
    rc, out, view_hw, _ = _letterbox_views([img] * 10 + [big] * 5, np.ascontiguousarray(windows))
    check(rc)
    imgs = [img] * 10 + [big] * 5
    want = preprocess.letterbox_batch_device([np.ascontiguousarray(im[y0:y0 + th, x0:x0 + tw]) for im, (y0, x0, th, tw) in zip(imgs, windows.tolist())], IN_HW)
    assert torch.equal(out[:15], want)
    assert view_hw[:15].cpu().numpy().tolist() == windows[:, 2:].tolist()


@pytest.mark.parametrize("window", [(0, 0, 98, 131), (0, 0, 97, 132), (-1, 0, 10, 10), (0, -1, 10, 10), (90, 0, 8, 10), (0, 0, 0, 5),
                                    (0, 130, 5, 2)])
def test_views_letterbox_refuses_windows_outside_the_image(window):
    img = _synthetic((97, 131), 0, 1)
    rc, out, _, _ = _letterbox_views([img], np.array([window], np.int32))
    assert rc == K2Y_ERR_INVALID and bool((out == 77).all())


def test_layout_with_tiling_through_letterbox_packed(photos):
    images = [np.ascontiguousarray(photos[4]), _jpeg(photos[0]), _synthetic((200, 300), 9, 3)]
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.Stream(device=dev)
    staging = preprocess.Staging(dev, stream)
    layout = preprocess.BatchLayout(images, IN_HW, tiling=(2, 2, 0.2))
    out = torch.empty((15,) + IN_HW + (3,), dtype=torch.uint8, device=dev)
    hw = torch.empty((15, 2), device=dev)
    yx = torch.empty((15, 2), device=dev)
    preprocess.letterbox_packed(layout, images, staging, out, hw, yx)
    stream.synchronize()
    from k210_yolo_framework_b200.helper import read_image
    pixels = [images[0], read_image(io.BytesIO(images[1])), images[2]]
    assert torch.equal(out, preprocess.letterbox_batch_device(_crops(pixels, layout.windows), IN_HW))
    assert hw.cpu().numpy().tolist() == layout.windows[:, 2:].tolist() and yx.cpu().numpy().tolist() == layout.windows[:, :2].tolist()


# ---- the merge ---------------------------------------------------------------------------------------------------------
def _view_blocks(rng, n, V, C, K, fill, kinds):
    """Seeded per-view record blocks as the detector writes them: per (view, class) `count` records in (score descending, index
    ascending) order.  `kinds` adds score ties across views, boxes identical across views and zero-area boxes."""
    dets = np.zeros((n * V, C, K), tiles_ref.DET)
    counts = np.zeros((n * V, C), np.int32)
    origins = np.zeros((n * V, 2), np.float32)
    levels = np.float32(np.linspace(0.05, 0.99, 12))
    for b in range(n):
        for v in range(V):
            origins[b * V + v] = (0, 0) if v == 0 else rng.integers(0, 400, 2)
    shared = rng.uniform(0, 500, (C, 4)).astype(np.float32)          # one box per class, seen by every view at the same place
    for i in range(n * V):
        for c in range(C):
            m = K if fill == "full" else 0 if fill == "empty" else int(rng.integers(0, K + 1)) if rng.random() < 0.7 else 0
            score = rng.choice(levels, m) if "ties" in kinds else rng.uniform(0.01, 1.0, m).astype(np.float32)
            index = rng.choice(NBOX, m, replace=False)
            order = np.lexsort((index, -score.astype(np.float64)))
            y, x = rng.uniform(0, 300, m), rng.uniform(0, 300, m)
            h, w = rng.uniform(5, 200, m), rng.uniform(5, 200, m)
            box = np.stack([y, x, y + h, x + w], 1).astype(np.float32)
            if "zero" in kinds:
                z = rng.random(m) < 0.2
                box[z, 2] = box[z, 0]
            if "same" in kinds and m:
                box[0] = shared[c] - np.tile(origins[i], 2)              # lands on `shared[c]` after the shift (up to a rounding)
            rec = dets[i, c]
            for k, j in enumerate(order):
                rec[k] = (box[j, 0], box[j, 1], box[j, 2], box[j, 3], score[j], index[j])
            counts[i, c] = m
    return dets, counts, origins


def _merge_gpu(dets, counts, origins, n, rows, V, iou, nbox=NBOX, strided=True):
    nv, C, K = dets.shape
    vd = torch.from_numpy(dets.view(np.int32).reshape(nv, C, K, 6).copy()).cuda()
    vc = torch.from_numpy(counts).cuda()
    yx = torch.from_numpy(np.ascontiguousarray(origins, np.float32)).cuda()
    words = C * (K * 6 + 1)
    buf = torch.full((rows, words), -7, dtype=torch.int32, device="cuda")        # records and counts of an image adjacent, as in a gather slot
    out_d = buf.as_strided((rows, C, K, 6), (words, K * 6, 6, 1))
    out_c = buf.as_strided((rows, C), (words, 1), C * K * 6)
    rc = lib.k2y_merge_views(vd.data_ptr(), vc.data_ptr(), yx.data_ptr(), n, rows, V, nbox, C, K, iou, out_d.data_ptr(), out_c.data_ptr(),
                             out_d.stride(0), out_c.stride(0), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out_d.cpu().numpy(), out_c.cpu().numpy()


def _assert_merge_equals_oracle(dets, counts, origins, n, rows, V, iou):
    rc, got_d, got_c = _merge_gpu(dets, counts, origins, n, rows, V, iou)
    check(rc)
    want_d, want_c = tiles_ref.merge_views(dets, counts, origins, n, NBOX, iou)
    np.testing.assert_array_equal(got_c[:n], want_c)
    assert (got_c[n:] == 0).all()
    got = np.ascontiguousarray(got_d[:n]).view(tiles_ref.DET)[..., 0]
    C, K = want_c.shape[1], want_d.shape[2]
    for b in range(n):
        for c in range(C):
            m = want_c[b, c]
            assert got[b, c, :m].tobytes() == want_d[b, c, :m].tobytes(), (b, c)
    return want_c


@pytest.mark.parametrize("C,K,V,iou,fill,kinds", [
    (20, 30, 5, 0.5, "random", ()), (20, 30, 10, 0.3, "random", ("ties", "same")), (20, 30, 17, 0.5, "random", ("zero",)),
    (20, 30, 2, 0.0, "random", ("ties", "same", "zero")), (20, 30, 10, 0.999, "random", ("same",)),
    (80, 100, 10, 0.5, "random", ("ties",)), (80, 100, 5, 0.5, "full", ()), (1, 100, 10, 0.3, "full", ("ties", "same")),
    (1, 30, 17, 0.5, "full", ("zero", "same")), (20, 30, 17, 0.999, "full", ()), (20, 30, 5, 0.5, "empty", ())])
def test_merge_equals_the_oracle(C, K, V, iou, fill, kinds):
    rng = np.random.default_rng(C * 1000 + K * 10 + V)
    n = 3 if C < 80 else 2
    dets, counts, origins = _view_blocks(rng, n, V, C, K, fill, kinds)
    want_c = _assert_merge_equals_oracle(dets, counts, origins, n, n + 2, V, iou)     # n < rows: the rows past n get count 0
    if fill == "empty":
        assert (want_c == 0).all()
    if fill == "full":
        assert want_c.max() == K or iou < 0.999
    if fill == "full" and iou == 0.999:
        assert (want_c == K).all()                           # the cap binds everywhere: V * K candidates, almost none suppressed


def test_merge_of_one_view_is_the_identity():
    rng = np.random.default_rng(5)
    dets, counts, origins = _view_blocks(rng, 2, 1, 20, 30, "random", ("ties",))
    rc, got_d, got_c = _merge_gpu(dets, counts, origins, 2, 2, 1, 1.5)      # nothing overlaps by more than 1.5: every record survives
    check(rc)
    np.testing.assert_array_equal(got_c, counts)
    got = np.ascontiguousarray(got_d).view(tiles_ref.DET)[..., 0]
    for b in range(2):
        for c in range(20):
            assert got[b, c, :counts[b, c]].tobytes() == dets[b, c, :counts[b, c]].tobytes()


def test_merge_refuses_more_records_than_it_holds():
    limit = lib.k2y_merge_views_max_records()
    assert limit >= 17 * 30 and limit >= 10 * 100            # VOC at 4x4 and COCO at 3x3 fit
    V, K = limit // 100 + 1, 100
    dets = np.zeros((V, 2, K), tiles_ref.DET)
    rc, got_d, got_c = _merge_gpu(dets, np.zeros((V, 2), np.int32), np.zeros((V, 2), np.float32), 1, 1, V, 0.5)
    assert rc == K2Y_ERR_INVALID
    assert (got_c == -7).all() and (got_d == -7).all()       # nothing was launched
    rc, _, got_c = _merge_gpu(dets[:1], np.zeros((1, 2), np.int32), np.zeros((1, 2), np.float32), 1, 1, 0, 0.5)
    assert rc == K2Y_ERR_INVALID and (got_c == -7).all()     # V >= 1


# ---- end to end --------------------------------------------------------------------------------------------------------
def _pipeline(golden_weights, voc_anchors, batch, lanes=None, obj=0.7, iou=0.5):
    if lanes is None:
        p = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=obj, iou_thresh=iou)
        p.engine.set_weights(golden_weights)
    else:
        p = LanedPipeline(lanes, "yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=obj, iou_thresh=iou, sm_split=False)
        p.set_weights(golden_weights)
    return p


def _pixels(item):
    from k210_yolo_framework_b200.helper import read_image
    return item if isinstance(item, np.ndarray) else read_image(io.BytesIO(bytes(item)))


def _composed(plain, images, rows, cols, overlap, iou=0.5):
    """What tiling is defined to give: every view's crop through the untiled pipeline `plain` as one batch, image-major, then
    the oracle merge.  Returns per image the records as DetectionPipeline.records lists them."""
    pixels = [_pixels(im) for im in images]
    windows = np.concatenate([tiles_ref.tile_windows(p.shape[0], p.shape[1], rows, cols, overlap) for p in pixels])
    d, c = plain.collect(plain.submit_images(_crops(pixels, windows)))
    dets, counts = tiles_ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], len(images), NBOX, iou)
    return [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
             for cls in range(dets.shape[1]) for r in dets[b, cls, :counts[b, cls]]] for b in range(len(images))]


@pytest.mark.parametrize("rows,cols,batch,n", [(2, 2, 20, 4), (3, 3, 30, 3)])
def test_tiled_pipeline_equals_the_composed_reference(golden_weights, voc_anchors, photos, rows, cols, batch, n):
    """Arrays and JPEG bytes, a full batch (n * V == batch) and a short one; the same batch size on both sides, and the same
    element count, because the tensor-core plans depend on them."""
    plain = _pipeline(golden_weights, voc_anchors, batch, obj=0.3)
    tiled = _pipeline(golden_weights, voc_anchors, batch, obj=0.3)
    tiled.enable_tiling(rows, cols)
    assert tiled.images_per_batch == n and plain.images_per_batch == batch
    total, views_seen = 0, set()
    for images in ([np.ascontiguousarray(p) for p in photos[:n]], [_jpeg(p) for p in photos[3:3 + n]],
                   [np.ascontiguousarray(photos[5]), _jpeg(photos[6])]):
        d, c = tiled.collect(tiled.submit_images(images))
        assert d.shape[0] == len(images)
        got = DetectionPipeline.records(d, c)
        assert got == _composed(plain, images, rows, cols, 0.2)
        total += sum(len(r) for r in got)
        views_seen |= {r[1] // NBOX for recs in got for r in recs}
    assert total > 20 and len(views_seen) > 2 and 0 in views_seen     # the whole image and several tiles contribute


def test_one_tile_returns_the_untiled_records(golden_weights, voc_anchors, photos):
    """1x1: the tile duplicates view 0 and loses every tie, so the records (view-0 indices included) are the untiled ones."""
    images = [np.ascontiguousarray(p) for p in photos[:4]]
    plain = _pipeline(golden_weights, voc_anchors, 8)
    tiled = _pipeline(golden_weights, voc_anchors, 8)
    tiled.enable_tiling(1, 1)
    # the untiled side runs the same eight inputs, so both sides plan their convolutions for the same element count
    want = DetectionPipeline.records(*plain.collect(plain.submit_images([im for im in images for _ in range(2)])))[::2]
    got = DetectionPipeline.records(*tiled.collect(tiled.submit_images(images)))
    assert got == want and sum(len(r) for r in got) > 5


@pytest.mark.parametrize("lanes", [None, 2])
def test_batches_in_flight_keep_their_own_windows(golden_weights, voc_anchors, photos, lanes):
    k = len(photos)
    batches = [[np.ascontiguousarray(photos[(2 * b + i) % k]) for i in range(2)] for b in range(5)]
    batches[2][1] = _synthetic((1080, 1920), 0, 3)          # the staging buffer of one slot grows mid-stream
    plain = _pipeline(golden_weights, voc_anchors, 10)
    ref = [_composed(plain, imgs, 2, 2, 0.2) for imgs in batches]
    pipe = _pipeline(golden_weights, voc_anchors, 10, lanes)
    pipe.enable_tiling(2, 2)
    assert pipe.images_per_batch == 2
    limit = 2 if lanes is None else pipe.in_flight_limit()
    tickets, got = [], []
    for i, imgs in enumerate(batches):
        tickets.append(pipe.submit_images(imgs))
        if i + 1 >= limit:
            got.append(DetectionPipeline.records(*pipe.collect(tickets[i + 1 - limit])))
    for t in tickets[len(got):]:
        got.append(DetectionPipeline.records(*pipe.collect(t)))
    assert got == ref


def test_rendering_draws_the_merged_records(golden_weights, voc_anchors, photos):
    from k210_yolo_framework_b200.draw import draw_detections
    from k210_yolo_framework_b200.helper import _COLORMAP
    from PIL import Image
    images = [np.ascontiguousarray(photos[0]), _jpeg(photos[1])]
    pipe = _pipeline(golden_weights, voc_anchors, 10)
    pipe.enable_tiling(2, 2)
    pipe.enable_rendering(quality=85, font_path=FONT)
    t = pipe.submit_images(images)
    recs = DetectionPipeline.records(*pipe.collect(t))
    files = pipe.rendered(t)
    assert len(files) == 2 and any(r[1] >= NBOX for rec in recs for r in rec)
    for item, rec, f in zip(images, recs, files):
        ref = io.BytesIO()
        draw_detections(_pixels(item), rec, _COLORMAP, font_path=FONT).save(ref, "JPEG", quality=85)
        assert f == ref.getvalue()


def test_bad_input_raises_and_leaves_the_pipeline_usable(golden_weights, voc_anchors, photos):
    pipe = _pipeline(golden_weights, voc_anchors, 10)
    with pytest.raises(ValueError):
        pipe.enable_tiling(3, 4)                             # 13 views > batch
    with pytest.raises(ValueError):
        pipe.enable_tiling(0, 2)
    with pytest.raises(ValueError):
        pipe.enable_tiling(2, 2, overlap=1.0)
    assert pipe.images_per_batch == 10
    coco = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 32, max_per_class=100)
    with pytest.raises(ValueError, match="records"):
        coco.enable_tiling(2, 5)                             # 11 views x 100 records
    coco.enable_tiling(3, 3)
    images = [np.ascontiguousarray(p) for p in photos[:2]]
    untiled = DetectionPipeline.records(*pipe.collect(pipe.submit_images(images)))
    pipe.enable_tiling(3, 1)
    before = pipe._submitted
    for bad in ([images[0]] * 3, [images[0], np.zeros((2, 50, 3), np.uint8)], []):
        with pytest.raises(ValueError):
            pipe.submit_images(bad)
    assert pipe._submitted == before
    plain = _pipeline(golden_weights, voc_anchors, 10)
    got = DetectionPipeline.records(*pipe.collect(pipe.submit_images(images)))
    assert got == _composed(plain, images, 3, 1, 0.2) and len(untiled) == 2


def _serve_args(tmp_path, golden_weights, files_dir, batch, tiles_arg):
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    if not ckpt.exists():
        save_keras_weights(str(ckpt), golden_weights)

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(files_dir), "yolo_mobilev1", 0.75, IN_HW, 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), batch, 0.7, 0.5, 2
    a.tiles, a.tile_overlap = tiles_arg, 0.2
    return a


def _write_files(tmp_path, dog_u8, people_u8):
    from PIL import Image
    d = tmp_path / "imgs"
    d.mkdir()
    kinds = [dog_u8, people_u8, np.ascontiguousarray(people_u8[60:, 40:420][:, ::-1])]
    files = []
    for i in range(5):
        path = d / (f"{i:02d}.png" if i % 2 else f"{i:02d}.jpg")
        Image.fromarray(kinds[i % 3]).save(path, **({} if i % 2 else {"quality": 90}))
        files.append(str(path))
    return d, files


def _composed_lines(golden_weights, voc_anchors, files, batch):
    from k210_yolo_framework_b200.helper import read_image
    plain = _pipeline(golden_weights, voc_anchors, batch)
    filler = np.full(IN_HW + (3,), 128, np.uint8)
    lines = []
    for g0 in range(0, len(files), 2):
        chunk = files[g0:g0 + 2]
        imgs = [read_image(p) for p in chunk]
        recs = _composed(plain, imgs + [filler] * (2 - len(imgs)), 2, 2, 0.2)
        for path, rec in zip(chunk, recs):
            lines.append(json.dumps({"image": path, "detections": [
                {"class": int(c), "score": round(float(s), 6), "box_tlbr": [float(t), float(l), float(b), float(r)], "index": int(i)}
                for c, i, s, t, l, b, r in rec]}) + "\n")
    return lines


def test_serve_with_tiles(tmp_path, golden_weights, voc_anchors, dog_u8, people_u8):
    """serve.py --tiles 2 2, batch 10 (two images per batch, a short final batch): the JSON lines of the composed reference."""
    import serve
    files_dir, files = _write_files(tmp_path, dog_u8, people_u8)
    a = _serve_args(tmp_path, golden_weights, files_dir, 10, (2, 2))
    ns = serve.build_parser().parse_args([a.ckpt, a.images, "--tiles", "2", "2"])
    assert ns.tiles == [2, 2] and ns.tile_overlap == 0.2
    out = tmp_path / "dets.jsonl"
    with open(out, "w") as fh:
        assert serve.serve(a, fh) == 5
    text = open(out).read().splitlines(keepends=True)
    assert text == _composed_lines(golden_weights, voc_anchors, files, 10)
    assert any(d["index"] >= NBOX for line in text for d in json.loads(line)["detections"])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_serve_with_tiles_on_two_gpus(tmp_path, golden_weights, voc_anchors, dog_u8, people_u8):
    import subprocess
    import sys
    from conftest import ROOT
    files_dir, files = _write_files(tmp_path, dog_u8, people_u8)
    a = _serve_args(tmp_path, golden_weights, files_dir, 10, (2, 2))
    out = tmp_path / "dets2.jsonl"
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", os.path.join(ROOT, "serve.py"), a.ckpt, a.images,
                    "--anchors", a.anchors, "--batch", "10", "--tiles", "2", "2", "--out", str(out)], check=True, cwd=ROOT, timeout=600)
    assert open(out).read().splitlines(keepends=True) == _composed_lines(golden_weights, voc_anchors, files, 10)
