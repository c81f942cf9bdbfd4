"""GPU baseline-JPEG decode (csrc/jpeg.cu): bit-exact with Helper._read_img (PIL / libjpeg-turbo) over sizes, sampling layouts,
qualities, Huffman tables, restart intervals and content; the reference's own files; synchronisation stress; mixed batches
through submit_images; corrupt input; serve.py."""
import io
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import GOLDEN
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200.helper import read_image
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline

IN_HW = (224, 320)
SIZES = [(1, 1), (1, 17), (2, 3), (3, 5), (7, 7), (8, 8), (9, 9), (15, 17), (16, 16), (17, 31), (33, 61), (224, 320), (375, 500),
         (500, 333), (720, 1280), (1080, 1920)]
CV2_SAMPLING = {"440": "IMWRITE_JPEG_SAMPLING_FACTOR_440", "411": "IMWRITE_JPEG_SAMPLING_FACTOR_411"}


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    f = rng.uniform(0.005, 0.05, 3)
    base = np.stack([127.5 + 127.5 * np.sin(f[c] * (xx + rng.uniform(0, 1) * yy) + rng.uniform(0, 6)) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)


def noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def flat(h, w, seed):
    return np.broadcast_to(np.array([seed % 256, 90, 200], np.uint8), (h, w, 3)).copy()


def detail(h, w, seed):
    """Flat field with isolated bright dots: blocks of long zero runs (ZRL) and a few large AC coefficients."""
    img = flat(h, w, 40)
    rng = np.random.default_rng(seed)
    k = max(1, h * w // 97)
    img[rng.integers(0, h, k), rng.integers(0, w, k)] = 255
    return img


def encode(img, layout="420", **kw):
    """JPEG bytes: PIL for 4:4:4 / 4:2:2 / 4:2:0 / grey, cv2 (libjpeg-turbo) for 4:4:0 and 4:1:1."""
    if layout in CV2_SAMPLING:
        import cv2
        params = [cv2.IMWRITE_JPEG_QUALITY, kw.get("quality", 90), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, CV2_SAMPLING[layout])]
        ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(img[..., ::-1]), params)
        assert ok
        return buf.tobytes()
    from PIL import Image
    b = io.BytesIO()
    if layout == "gray":
        Image.fromarray(img).convert("L").save(b, "JPEG", **kw)
    else:
        Image.fromarray(img).save(b, "JPEG", subsampling={"444": 0, "422": 1, "420": 2}[layout], **kw)
    return b.getvalue()


def pil(data):
    return read_image(io.BytesIO(data))


def assert_exact(files):
    got = preprocess.decode_jpeg_batch(files)
    torch.cuda.synchronize()
    for i, (g, f) in enumerate(zip(got, files)):
        ref = pil(f)
        g = g.cpu().numpy()
        assert g.shape == ref.shape, (i, g.shape, ref.shape)
        if not np.array_equal(g, ref):
            bad = np.argwhere(g != ref)
            raise AssertionError(f"file {i} {ref.shape}: {len(bad)} bytes differ, first at {bad[0].tolist()}: "
                                 f"{g[tuple(bad[0])]} vs {ref[tuple(bad[0])]}")


@pytest.mark.parametrize("layout", ["444", "422", "420", "440", "411", "gray"])
def test_sizes_and_sampling_bit_exact(layout):
    files = [encode(photo(h, w, h * 7 + w), layout) for h, w in SIZES]
    for f in files:
        assert preprocess.inspect_jpeg(f)[2]
    assert_exact(files)


@pytest.mark.parametrize("quality", [10, 50, 75, 90, 95, 100])
def test_qualities_bit_exact(quality):
    files = [encode(photo(h, w, quality + h), lay, quality=quality) for (h, w), lay in
             zip([(375, 500), (33, 61), (224, 320), (17, 31), (500, 333), (9, 9)], ["420", "444", "422", "440", "411", "gray"])]
    assert_exact(files)


@pytest.mark.parametrize("content", [photo, noise, flat, detail])
def test_content_and_custom_tables_bit_exact(content):
    files = []
    for lay in ("420", "444", "gray"):
        files.append(encode(content(240, 352, 1), lay, quality=100))
        files.append(encode(content(97, 131, 2), lay, quality=75, optimize=True))   # optimised (custom) Huffman tables
    assert_exact(files)


@pytest.mark.parametrize("restart", [{"restart_marker_blocks": 1}, {"restart_marker_blocks": 4}, {"restart_marker_rows": 1}])
def test_restart_intervals_bit_exact(restart):
    files = [encode(photo(h, w, 3), lay, **restart) for (h, w), lay in
             zip([(375, 500), (33, 61), (8, 8), (101, 203)], ["420", "422", "444", "gray"])]
    for f in files:
        assert b"\xff\xdd" in f      # a DRI marker
    files.append(encode(noise(131, 97, 4), "420", quality=100, **restart))
    assert_exact(files)


def test_many_tiny_images_one_batch():
    """100 JPEGs in one call: more than the letterbox's 48 descriptors per launch; the decode has no per-launch cap."""
    rng = np.random.default_rng(5)
    lays = ["444", "422", "420", "gray", "440", "411"]
    files = [encode(photo(int(rng.integers(1, 40)), int(rng.integers(1, 40)), i), lays[i % 6]) for i in range(100)]
    assert_exact(files)


def test_reference_files_equal_golden_pixels(dog_u8, people_u8):
    files = [open(os.path.join(GOLDEN, n), "rb").read() for n in ("dog.jpg", "people.jpg")]
    got = [g.cpu().numpy() for g in preprocess.decode_jpeg_batch(files)]
    np.testing.assert_array_equal(got[0], dog_u8)
    np.testing.assert_array_equal(got[1], people_u8)


def _pipeline(golden_weights, voc_anchors, batch, lanes=None):
    if lanes is None:
        p = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=0.7, iou_thresh=0.5)
        p.engine.set_weights(golden_weights)
    else:
        p = LanedPipeline(lanes, "yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, batch, obj_thresh=0.7, iou_thresh=0.5, sm_split=False)
        p.set_weights(golden_weights)
    return p


def test_dog_file_reproduces_golden_records(golden_weights, voc_anchors, dog_golden):
    pipe = _pipeline(golden_weights, voc_anchors, 1)
    dog = open(os.path.join(GOLDEN, "dog.jpg"), "rb").read()
    found = DetectionPipeline.records(*pipe.collect(pipe.submit_images([dog])))[0]
    gold = dog_golden["keras"]["detections"]
    assert [(d[0], d[1]) for d in found] == [(g[0], g[1]) for g in gold]
    np.testing.assert_allclose([d[2] for d in found], [g[2] for g in gold], atol=1e-5)
    np.testing.assert_allclose([d[3:] for d in found], [g[3:] for g in gold], atol=1e-3)


def test_sync_stress():
    """A 1080x1920 quality-100 noise image (one segment of many windows of subsequences), the same with a restart every MCU,
    and images smaller than one subsequence."""
    big = noise(1080, 1920, 9)
    files = [encode(big, "420", quality=100), encode(big, "420", quality=100, restart_marker_blocks=1),
             encode(flat(8, 8, 1), "444"), encode(flat(16, 16, 2), "420"), encode(noise(3, 5, 3), "gray")]
    assert len(files[0]) > 256 * 512 // 8 * 4     # spans several windows of 256 subsequences of 512 bits
    got, status = preprocess.decode_jpeg_batch(files, with_status=True)
    assert (status[:, 0] == 0).all(), status
    assert status[0, 3] > 1 and status[1, 3] >= 1
    for g, f in zip(got, files):
        np.testing.assert_array_equal(g.cpu().numpy(), pil(f))


def _mixed_files(tmp=None):
    """Supported JPEGs, progressive JPEGs, PNG bytes (and their _read_img pixels)."""
    from PIL import Image
    imgs = [photo(375, 500, 1), photo(240, 180, 2), photo(500, 333, 3), photo(100, 400, 4), photo(300, 300, 5)]
    out = [encode(imgs[0], "420"), encode(imgs[1], "444", quality=95, restart_marker_blocks=2), encode(imgs[2], "420", progressive=True)]
    b = io.BytesIO()
    Image.fromarray(imgs[3]).save(b, "PNG")
    out.append(b.getvalue())
    out.append(encode(imgs[4], "gray"))
    return out


@pytest.mark.parametrize("lanes", [None, 2])
def test_mixed_batches_through_submit_images(golden_weights, voc_anchors, dog_u8, lanes):
    files = _mixed_files()
    assert [preprocess.gpu_decodable(f) for f in files] == [True, True, False, False, True]
    arrays = [pil(f) for f in files]
    big = encode(noise(1080, 1920, 11), "420", quality=100)      # grows a slot's staging mid-stream
    batches = [[files[0], dog_u8, bytearray(files[2]), memoryview(files[3])],
               [files[4], files[1], dog_u8[:, ::-1], files[0]],
               [big, files[3], files[1], dog_u8],
               [files[2], files[4], files[0], files[1]]]
    ref_batches = [[pil(bytes(e)) if isinstance(e, (bytes, bytearray, memoryview)) else e for e in b] for b in batches]
    assert len(arrays) == 5
    ref_pipe = _pipeline(golden_weights, voc_anchors, 4, lanes)
    pipe = _pipeline(golden_weights, voc_anchors, 4, lanes)
    limit = 2 if lanes is None else pipe.in_flight_limit()

    def run(p, bs):
        tickets, got = [], []
        for i, imgs in enumerate(bs):
            tickets.append(p.submit_images(imgs))
            if i + 1 >= limit:
                got.append(DetectionPipeline.records(*p.collect(tickets[i + 1 - limit])))
        for t in tickets[len(got):]:
            got.append(DetectionPipeline.records(*p.collect(t)))
        return got

    assert run(pipe, batches) == run(ref_pipe, ref_batches)
    # inputs the pipeline rejects still raise before anything is enqueued
    p1 = pipe.lanes[0] if lanes else pipe
    before = p1._submitted
    for bad in (["dog.jpg"], [b""], [torch.zeros(4, 4, 3, dtype=torch.uint8)], [b"not an image"]):
        with pytest.raises(ValueError):
            p1.submit_images(bad)
    assert p1._submitted == before


def test_letterbox_batch_device_takes_files(dog_u8):
    from oracle import preprocess_ref
    files = _mixed_files()
    out = preprocess.letterbox_batch_device(files + [dog_u8], IN_HW).cpu().numpy()
    for got, f in zip(out, files):
        np.testing.assert_array_equal(got, preprocess_ref.letterbox(pil(f), IN_HW))
    np.testing.assert_array_equal(out[-1], preprocess_ref.letterbox(dog_u8, IN_HW))


def test_corrupt_entropy_data_sets_status_and_spares_the_others():
    good = [encode(photo(200, 300, 1), "420"), encode(photo(64, 80, 2), "444", restart_marker_blocks=2)]
    victim = encode(photo(240, 320, 3), "420")
    sos = victim.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(victim[sos + 2:sos + 4], "big")
    truncated = victim[:start + (len(victim) - start) // 3]
    garbled = bytearray(victim)
    garbled[start + 200:start + 216] = b"\xff\x00" * 8   # 64 one bits: no Huffman code is all ones
    files = [good[0], truncated, good[1], bytes(garbled)]
    got, status = preprocess.decode_jpeg_batch(files, with_status=True)
    assert status[0, 0] == 0 and status[2, 0] == 0
    assert status[1, 0] & 2, status          # premature end
    assert status[3, 0] != 0, status         # invalid code (or the blocks after it run short)
    np.testing.assert_array_equal(got[0].cpu().numpy(), pil(good[0]))
    np.testing.assert_array_equal(got[2].cpu().numpy(), pil(good[1]))
    with pytest.raises(Exception, match="corrupt"):
        preprocess.decode_jpeg_batch(files)


def test_serve_routes_files_and_keeps_its_lines(tmp_path, golden_weights, monkeypatch):
    """serve.py on JPEG, progressive JPEG and PNG files: the same JSON lines as decoding every file with PIL."""
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    files = _mixed_files()
    names = ["a.jpg", "b.jpg", "c.jpg", "d.png", "e.jpg", "f.jpg", "g.png"]
    for i, n in enumerate(names):
        (d / n).write_bytes(files[i % len(files)] if i < 5 else (open(os.path.join(GOLDEN, "dog.jpg"), "rb").read() if i == 5 else files[3]))

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(d), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.7, 0.5, 2
    with open(tmp_path / "gpu.jsonl", "w") as fh:
        assert serve.serve(a, fh) == len(names)
    monkeypatch.setattr(serve, "load_image", lambda p: read_image(p))     # every file through PIL
    with open(tmp_path / "pil.jsonl", "w") as fh:
        assert serve.serve(a, fh) == len(names)
    lines = open(tmp_path / "gpu.jsonl").read()
    assert lines == open(tmp_path / "pil.jsonl").read()
    assert [json.loads(l)["image"] for l in lines.splitlines()] == [str(d / n) for n in sorted(names)]


def _victims():
    victim = encode(photo(240, 320, 3), "420")
    sos = victim.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(victim[sos + 2:sos + 4], "big")
    garbled = bytearray(victim)
    garbled[start + 200:start + 216] = b"\xff\x00" * 8   # complete file (ends with EOI), invalid code inside
    return victim[:start + (len(victim) - start) // 3], bytes(garbled)


@pytest.mark.parametrize("lanes", [None, 2])
def test_submit_images_reports_corrupt_jpegs(golden_weights, voc_anchors, lanes):
    """A truncated JPEG is refused before anything is enqueued (the host decoder raises, as PIL does); a complete file with
    corrupt entropy data makes collect raise, naming the image; the pipeline stays in step for the next batch."""
    truncated, garbled = _victims()
    good = _mixed_files()
    pipe = _pipeline(golden_weights, voc_anchors, 4, lanes)
    ref = _pipeline(golden_weights, voc_anchors, 4, lanes)
    with pytest.raises(ValueError, match="image 1: cannot decode"):
        pipe.submit_images([good[0], truncated])
    t = pipe.submit_images([good[0], good[4], garbled])
    t2 = pipe.submit_images([good[1], good[0]])
    with pytest.raises(Exception, match="corrupt JPEG data: image 2: "):
        pipe.collect(t)
    got = DetectionPipeline.records(*pipe.collect(t2))
    ref.collect(ref.submit_images([good[0], good[4], good[1]]))
    assert got == DetectionPipeline.records(*ref.collect(ref.submit_images([good[1], good[0]])))
    with pytest.raises(Exception, match="corrupt JPEG data: image 0"):
        preprocess.letterbox_batch_device([garbled, good[0]], IN_HW)


def test_serve_stops_on_a_truncated_jpeg_as_pil_does(tmp_path, golden_weights):
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    truncated, _ = _victims()
    (d / "a.jpg").write_bytes(_mixed_files()[0])
    (d / "b.jpg").write_bytes(truncated)
    with pytest.raises(OSError, match="truncated"):
        read_image(str(d / "b.jpg"))

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(d), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.7, 0.5, 2
    with open(tmp_path / "out.jsonl", "w") as fh:
        with pytest.raises(OSError, match="truncated"):
            serve.serve(a, fh)
    assert open(tmp_path / "out.jsonl").read() == ""
