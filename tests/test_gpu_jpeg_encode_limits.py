"""GPU JPEG encoding (csrc/jpeg_encode.cu) past its one-pass limits, byte for byte against PIL's save: every quality, a file
whose stuffing scan runs more than one pass, strips at libjpeg's 65500-pixel limit (and their GPU decode), hundreds of tiny
images, views at odd offsets; and the refusals above that limit on every route that writes or reads a JPEG."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from PIL import Image

from test_gpu_jpeg_encode import CONTENT, assert_same, photo, pil_jpeg
from test_image_limits import OVERSIZE, entropy_bytes, oversize_jpeg
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200.helper import read_image
from k210_yolo_framework_b200.render import JPEG_MAX_DIMENSION, JpegEncoder, encode_jpeg_batch

BIG_HW, BIG_QUALITY = (3000, 4000), 100
STRIPS = [(1, JPEG_MAX_DIMENSION), (JPEG_MAX_DIMENSION, 1), (2, JPEG_MAX_DIMENSION)]
TINY = [(h, w) for h in range(1, 18) for w in range(1, 18)] + [(1 + k, 17 - k) for k in range(11)]


def big_noise():
    return np.random.default_rng(3000).integers(0, 256, BIG_HW + (3,), dtype=np.uint8)


def test_every_quality_on_a_mixed_batch():
    sizes = [(13, 29), (37, 53), (75, 41)]              # off the 16x16 MCU grid
    for q in range(1, 101):
        imgs = [CONTENT[kind](h, w, q + 7 * k) for k, kind in enumerate(["noise", "photo", "gradient"]) for h, w in sizes]
        assert_same(imgs, q)


def test_stuffing_scan_runs_more_than_one_pass():
    """A 3000x4000 noise image at quality 100 among small ones: its entropy-coded data is longer than one pass of the
    stuffing scan (SCAN_THREADS chunks of CHUNK_BYTES), so the pass carry adds real 0xFF counts."""
    imgs = [photo(37, 53, 1), big_noise(), photo(16, 16, 2)]
    files = assert_same(imgs, BIG_QUALITY)
    data = entropy_bytes(files[1])
    assert len(data) > 1024 * 8192 and data[:1024 * 8192].count(b"\xff") > 0


def test_strips_at_the_size_limit_encode_and_decode_as_pil_does():
    imgs = [photo(h, w, h + w) for h, w in STRIPS]
    files = assert_same(imgs, 90)
    dec = preprocess.decode_jpeg_batch(files)
    for d, f in zip(dec, files):
        assert np.array_equal(d.cpu().numpy(), read_image(io.BytesIO(f)))


def test_three_hundred_tiny_images_in_one_batch():
    assert len(TINY) == 300
    imgs = [CONTENT["noise"](h, w, 17 * h + w) for h, w in TINY]
    assert_same(imgs, 85)


def test_views_at_odd_byte_offsets_of_one_buffer():
    shapes = [(9, 13), (16, 16), (33, 7), (1, 5)]
    imgs = [photo(h, w, k) for k, (h, w) in enumerate(shapes)]
    buf = torch.zeros(sum(im.size for im in imgs) + 64, dtype=torch.uint8, device="cuda")
    views, off = [], 1
    for im in imgs:
        v = buf[off:off + im.size].view(im.shape)
        v.copy_(torch.from_numpy(im))
        views.append(v)
        off = (off + im.size) | 1     # the next odd offset
    assert all(v.data_ptr() % 2 for v in views)
    assert encode_jpeg_batch(views, quality=80) == [pil_jpeg(im, 80) for im in imgs]


@pytest.mark.parametrize("hw", OVERSIZE)
def test_encoder_refuses_what_pil_cannot_write(hw):
    h, w = hw
    with pytest.raises(OSError):      # libjpeg's "Maximum supported image dimension is 65500 pixels"
        Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(io.BytesIO(), "JPEG")
    img = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="65500"):
        encode_jpeg_batch([torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"), img])
    enc = JpegEncoder(img.device)
    with pytest.raises(ValueError, match="65500"):
        enc.enqueue(img.data_ptr(), np.zeros(1, np.int64), np.array([[h, w]], np.int32), 75, torch.cuda.current_stream())


@pytest.mark.parametrize("hw", OVERSIZE)
def test_oversize_files_take_the_pil_route_and_raise_as_pil_does(hw):
    f = oversize_jpeg(*hw)
    with pytest.raises(OSError):      # libjpeg reports "Maximum supported image dimension is 65500 pixels" on stderr
        read_image(io.BytesIO(f))
    assert not preprocess.gpu_decodable(f)
    ok = pil_jpeg(photo(20, 30, 0), 90)
    with pytest.raises(ValueError, match="65500"):
        preprocess.decode_jpeg_batch([ok, f])
    with pytest.raises(ValueError, match="image 1: cannot decode"):
        preprocess.letterbox_batch_device([photo(20, 30, 1), f], (224, 320))


@pytest.mark.parametrize("laned", [False, True])
def test_rendering_pipeline_refuses_oversize_images_and_stays_in_step(voc_anchors, golden_weights, dog_u8, laned):
    from test_gpu_render import FONT, make_pipe
    from k210_yolo_framework_b200.draw import draw_detections
    from k210_yolo_framework_b200.helper import _COLORMAP
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    pipe = make_pipe(voc_anchors, golden_weights, laned)
    pipe.enable_rendering(quality=85, font_path=FONT)
    counter = (lambda: pipe._next_host) if laned else (lambda: pipe._submitted)
    before = counter()
    for h, w in OVERSIZE:
        with pytest.raises(ValueError, match="image 1 .*65500"):
            pipe.submit_images([dog_u8, np.zeros((h, w, 3), np.uint8)])
        with pytest.raises(ValueError, match="image 0: cannot decode"):
            pipe.submit_images([oversize_jpeg(h, w), dog_u8])
    assert counter() == before
    strip = photo(JPEG_MAX_DIMENSION, 3, 5)          # the largest size a JPEG file holds is drawn and encoded
    imgs = [dog_u8, strip, dog_u8[:, ::-1].copy()]
    t = pipe.submit_images(imgs)
    recs = DetectionPipeline.records(*pipe.collect(t))
    files = pipe.rendered(t)
    assert any(recs)
    for img, rec, f in zip(imgs, recs, files):
        ref = io.BytesIO()
        draw_detections(img, rec, _COLORMAP, font_path=FONT).save(ref, "JPEG", quality=85)
        assert f == ref.getvalue(), img.shape
