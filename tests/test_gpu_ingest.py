"""Batched ragged letterbox (k2y_letterbox_u8_batch) and the raw-image streaming API (submit_images / collect, serve.py)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import GOLDEN
from k210_yolo_framework_b200 import KerasDetector, preprocess, yolonet
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline
from oracle import preprocess_ref

IN_HW = (224, 320)
# every (size, lowest pixel value) of test_gpu_preprocess.test_letterbox_bit_exact: 1x1, identity, up- and downscaling,
# width- and height-limited images, and min > 0 (the clip branch that keeps the zero fill)
SIZES = [((375, 500), 0), ((100, 37), 0), ((224, 320), 0), ((480, 640), 0), ((33, 61), 25), ((1, 1), 7), ((720, 1280), 1),
         ((500, 333), 0)]


def _synthetic(hw, lo, seed):
    return np.random.default_rng(seed).integers(lo, 256, (hw[0], hw[1], 3), dtype=np.uint8)


@pytest.fixture(scope="module")
def mixed():
    return [_synthetic(hw, lo, hw[0] * 1000 + hw[1]) for hw, lo in SIZES]


@pytest.fixture(scope="module")
def photos(dog_u8, people_u8):
    """Real images of different sizes (crops keep objects in view, so the original sizes change the boxes)."""
    return [dog_u8, people_u8, dog_u8[:, ::-1], people_u8[:, ::-1], people_u8[40:, 30:450], dog_u8[10:200, 20:],
            np.ascontiguousarray(people_u8[::-1])]


@pytest.mark.parametrize("in_hw", [(224, 320), (416, 416), (608, 608)])
def test_batch_letterbox_bit_exact(mixed, in_hw):
    out = preprocess.letterbox_batch_device(mixed, in_hw).cpu().numpy()
    assert out.shape == (len(mixed),) + in_hw + (3,) and out.dtype == np.uint8
    for got, img in zip(out, mixed):
        np.testing.assert_array_equal(got, preprocess_ref.letterbox(img, in_hw))


def test_staging_grows_for_a_large_image_and_stays_exact(mixed):
    """A 1080x1920 image among small ones: the staging buffers grow once, geometrically, and every image stays bit-exact."""
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.Stream(device=dev)
    staging = preprocess.Staging(dev, stream)
    big = _synthetic((1080, 1920), 0, 1080)
    batches = [mixed[:3], [mixed[4], big, mixed[5], mixed[1]], mixed[5:]]
    sizes = []
    for imgs in batches:
        layout = preprocess.BatchLayout(imgs, IN_HW)
        out = torch.empty((len(imgs),) + IN_HW + (3,), dtype=torch.uint8, device=dev)
        hw = torch.empty((len(imgs), 2), dtype=torch.float32, device=dev)
        preprocess.letterbox_packed(layout, imgs, staging, out, hw)
        stream.synchronize()
        sizes.append(staging.host.numel())
        assert staging.host.is_pinned() and staging.dev.numel() == staging.host.numel() >= layout.nbytes
        for got, img in zip(out.cpu().numpy(), imgs):
            np.testing.assert_array_equal(got, preprocess_ref.letterbox(img, IN_HW))
        assert hw.cpu().numpy().tolist() == [list(im.shape[:2]) for im in imgs]
    assert sizes[0] < sizes[1] == sizes[2] and sizes[1] >= 1080 * 1920 * 3


def test_batch_equals_single_image_kernel(mixed):
    """Every image of a batch equals the single-image letterbox_device, and the kernel writes each source's (h, w)."""
    n = len(mixed)
    out = torch.full((n + 2,) + IN_HW + (3,), 77, dtype=torch.uint8, device="cuda")
    hw = torch.full((n + 2, 2), -1.0, dtype=torch.float32, device="cuda")
    preprocess.letterbox_batch_device(mixed, IN_HW, out=out, image_hw_out=hw)
    for i, img in enumerate(mixed):
        single = preprocess.letterbox_device(torch.from_numpy(img).cuda(), IN_HW)
        assert torch.equal(out[i], single), i
    assert hw[:n].cpu().numpy().tolist() == [list(hw_) for hw_, _ in SIZES]
    assert bool((out[n:] == 77).all()) and bool((hw[n:] == -1).all())       # rows past n untouched


def _reference(golden_weights, voc_anchors, batches, batch):
    """Per-image route on one engine of the same batch size: letterbox_device per image, predict_device_u8, then the
    decode with each image's own shape."""
    model, wrapper = yolonet.yolo_mobilev1([IN_HW[0], IN_HW[1], 3], 3, 20, alpha=0.75, max_batch=batch)
    wrapper.set_weights_dict(golden_weights)
    det = KerasDetector(voc_anchors, list(IN_HW), [(7, 10), (14, 20)], 20, 0.7, 0.5, max_per_class=30, max_batch=batch)
    out = []
    for imgs in batches:
        x = torch.stack([preprocess.letterbox_device(torch.from_numpy(np.ascontiguousarray(im)).cuda(), IN_HW) for im in imgs])
        heads = wrapper.predict_device_u8(x)
        shapes = np.array([im.shape[:2] for im in imgs], np.float32)
        out.append(KerasDetector.to_host(*det.run([t.contiguous() for t in heads], shapes)))
    return out


def _pipeline(golden_weights, voc_anchors, batch, lanes=None):
    if lanes is None:
        p = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=0.7, iou_thresh=0.5)
        p.engine.set_weights(golden_weights)
    else:
        # no SM split: the lanes then plan their convolutions as the single-lane reference engine does (same bits)
        p = LanedPipeline(lanes, "yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=0.7, iou_thresh=0.5, sm_split=False)
        p.set_weights(golden_weights)
    return p


def test_real_images_end_to_end(golden_weights, voc_anchors, photos):
    imgs = photos[:4] + [_synthetic((300, 200), 0, 5), _synthetic((150, 600), 3, 6)]
    pipe = _pipeline(golden_weights, voc_anchors, len(imgs))
    d, c = pipe.collect(pipe.submit_images(imgs))
    got = DetectionPipeline.records(d, c)
    ref = _reference(golden_weights, voc_anchors, [imgs], len(imgs))[0]
    assert got == ref
    assert [(r[0], r[1]) for r in got[0]] == [(6, 53), (11, 765)]
    assert [r[1] for r in got[1]] == [637, 778, 745, 676, 590] and all(r[0] == 14 for r in got[1])


@pytest.mark.parametrize("lanes", [None, 2])
def test_streaming_carries_each_batch_sizes(golden_weights, voc_anchors, photos, lanes):
    """Six batches of 4 with different size mixes, two in flight per lane (one pipeline, or two lanes): every ticket returns
    its own batch's records, so each batch's original sizes reach its own decode."""
    k = len(photos)
    batches = [[photos[(3 * b + i) % k] for i in range(4)] for b in range(6)]
    batches[3][2] = _synthetic((1080, 1920), 0, 3)         # the staging buffer of one slot grows mid-stream
    ref = _reference(golden_weights, voc_anchors, batches, 4)
    pipe = _pipeline(golden_weights, voc_anchors, 4, lanes)
    limit = 2 if lanes is None else pipe.in_flight_limit()
    tickets, got = [], []
    for i, imgs in enumerate(batches):
        tickets.append(pipe.submit_images(imgs))
        if i + 1 >= limit:
            got.append(DetectionPipeline.records(*pipe.collect(tickets[i + 1 - limit])))
    for t in tickets[len(got):]:
        got.append(DetectionPipeline.records(*pipe.collect(t)))
    assert got == ref
    assert sum(len(r) for recs in ref for r in recs) > 20


def test_partial_batch_and_bad_inputs(golden_weights, voc_anchors, photos):
    pipe = _pipeline(golden_weights, voc_anchors, 4)
    imgs = photos[1:4]
    d, c = pipe.collect(pipe.submit_images(imgs))
    assert d.shape[0] == 3 and c.shape[0] == 3
    assert DetectionPipeline.records(d, c) == _reference(golden_weights, voc_anchors, [imgs], 4)[0]
    bad = [[], [photos[0].astype(np.float32)], [photos[0][..., 0]], [np.zeros((8, 8, 4), np.uint8)], [photos[0]] * 5,
           [torch.from_numpy(photos[0])], [np.zeros((0, 8, 3), np.uint8)]]
    before = pipe._submitted
    for b in bad:
        with pytest.raises(ValueError):
            pipe.submit_images(b)
    assert pipe._submitted == before
    out = torch.full((2,) + IN_HW + (3,), 9, dtype=torch.uint8, device="cuda")
    for b in bad[:4] + [photos[:3]]:
        with pytest.raises(ValueError):
            preprocess.letterbox_batch_device(b, IN_HW, out=out)
    with pytest.raises(ValueError):
        preprocess.letterbox_batch_device(photos[:2], IN_HW, image_hw_out=torch.zeros((1, 2), device="cuda"))
    torch.cuda.synchronize()
    assert bool((out == 9).all())
    # the pipeline is still in step after the refusals
    d, c = pipe.collect(pipe.submit_images(imgs))
    assert DetectionPipeline.records(d, c) == _reference(golden_weights, voc_anchors, [imgs], 4)[0]


def _old_serve_lines(args, files):
    """The serving loop before submit_images: per-image letterbox_device into one buffer, shared image shapes, step_device
    on the full batch, a synchronise per batch."""
    from k210_yolo_framework_b200 import Helper
    anchors = np.load(args.anchors)
    H, W = args.image_size
    h = Helper(None, args.class_num, anchors, [[H, W]], [[H // 32, W // 32], [H // 16, W // 16]])
    pipe = DetectionPipeline(args.model_def, (H, W), anchors, args.class_num, args.depth_multiplier, args.batch, args.obj_thresh,
                             args.iou_thresh, 30)
    pipe.engine.load_weights(args.ckpt)
    buf = torch.zeros((args.batch, H, W, 3), dtype=torch.uint8, device="cuda")
    shapes = np.tile(np.array([[H, W]], np.float32), (args.batch, 1))
    lines = []
    for g0 in range(0, len(files), args.batch):
        chunk = files[g0:g0 + args.batch]
        for j, path in enumerate(chunk):
            img = h._read_img(path)
            shapes[j] = img.shape[:2]
            buf[j].copy_(h.letterbox_device(img))
        pipe.set_image_shapes(shapes)
        pipe.engine.bind_input(buf)
        dets, counts = pipe.step_device(args.batch)
        pipe.wait_gathered()
        torch.cuda.synchronize()
        recs = DetectionPipeline.records(dets[:len(chunk)].clone(), counts.clone())
        for j, path in enumerate(chunk):
            lines.append(json.dumps({"image": path, "detections": [
                {"class": int(c), "score": round(float(s), 6), "box_tlbr": [float(t), float(l), float(b), float(r)], "index": int(i)}
                for c, i, s, t, l, b, r in recs[j]]}) + "\n")
    return lines


def test_serve_streams_raw_images(tmp_path, monkeypatch, golden_weights, dog_u8, people_u8):
    """serve.py over three image sizes, batch 4 with a short final batch, 1 and 2 decode threads: the same JSON lines as the
    per-image serving loop, byte for byte, and the detections of per-image keras_inference.detect."""
    from PIL import Image
    import keras_inference
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    imgs_dir = tmp_path / "imgs"
    imgs_dir.mkdir()
    kinds = [dog_u8, people_u8, np.ascontiguousarray(people_u8[60:, 40:420][:, ::-1])]
    files = []
    for i in range(10):
        path = imgs_dir / f"{i:02d}.png"
        Image.fromarray(kinds[i % 3]).save(path)
        files.append(str(path))

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(imgs_dir), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.7, 0.5
    old = _old_serve_lines(a, files)
    monkeypatch.chdir(tmp_path)                     # keras_inference.detect reads data/voc_anchor.npy
    (tmp_path / "data").mkdir()
    np.save(tmp_path / "data" / "voc_anchor.npy", np.load(a.anchors))
    per_image = [keras_inference.detect(str(ckpt), (224, 320), (7, 10, 14, 20), "yolo_mobilev1", 20, 0.75, 0.7, 0.5, "voc",
                                        files[i])[2] for i in range(3)]
    for threads in (1, 2):
        a.decode_threads = threads
        out = tmp_path / f"dets{threads}.jsonl"
        with open(out, "w") as fh:
            assert serve.serve(a, fh) == 10
        text = open(out).read().splitlines(keepends=True)
        assert text == old
        for i, line in enumerate(text):
            rec = json.loads(line)
            assert rec["image"] == files[i]
            ref = per_image[i % 3]
            assert [(d["class"], d["index"]) for d in rec["detections"]] == [(r[0], r[1]) for r in ref]
            for d, r in zip(rec["detections"], ref):
                assert abs(d["score"] - r[2]) < 1e-3
                assert np.abs(np.array(d["box_tlbr"]) - np.array(r[3:])).max() < 0.05
    assert [d["class"] for d in json.loads(text[1])["detections"]] == [14] * 5
