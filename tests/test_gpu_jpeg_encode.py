"""GPU baseline-JPEG encoding (csrc/jpeg_encode.cu): byte-identical with PIL's save over sizes, qualities and content, in
mixed-size batches; the files decode on the GPU decoder to what PIL decodes."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from PIL import Image

from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200.helper import read_image
from k210_yolo_framework_b200.render import encode_jpeg_batch

SIZES = [(1, 1), (1, 600), (600, 1), (7, 9), (8, 8), (15, 17), (16, 16), (37, 53), (224, 320), (375, 500), (1080, 1920)]
QUALITIES = [1, 10, 50, 75, 90, 95, 100]


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    f = rng.uniform(0.005, 0.05, 3)
    base = np.stack([127.5 + 127.5 * np.sin(f[c] * (xx + rng.uniform(0, 1) * yy) + rng.uniform(0, 6)) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)


CONTENT = {
    "noise": lambda h, w, s: np.random.default_rng(s).integers(0, 256, (h, w, 3), dtype=np.uint8),
    "flat": lambda h, w, s: np.full((h, w, 3), (s * 37) % 256, np.uint8),
    "gradient": lambda h, w, s: np.stack(np.broadcast_arrays(np.arange(w)[None] * 255 // max(w - 1, 1),
                                                             np.arange(h)[:, None] * 255 // max(h - 1, 1), np.full((h, w), s % 256)),
                                         -1).astype(np.uint8),
    "saturated": lambda h, w, s: (np.random.default_rng(s).integers(0, 2, (h, w, 3)) * 255).astype(np.uint8),
    "photo": photo,
}


def pil_jpeg(img, quality):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=quality)
    return b.getvalue()


def assert_same(imgs, quality):
    got = encode_jpeg_batch([torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in imgs], quality=quality)
    for i, (g, x) in enumerate(zip(got, imgs)):
        ref = pil_jpeg(x, quality)
        if g != ref:
            k = next((j for j in range(min(len(g), len(ref))) if g[j] != ref[j]), min(len(g), len(ref)))
            raise AssertionError(f"image {i} {x.shape} q{quality}: {len(g)} vs {len(ref)} bytes, first difference at {k}")
    return got


@pytest.mark.parametrize("content", sorted(CONTENT))
@pytest.mark.parametrize("quality", QUALITIES)
def test_encode_matches_pil_mixed_sizes(content, quality):
    imgs = [CONTENT[content](h, w, 11 * h + w + quality) for h, w in SIZES]
    assert_same(imgs, quality)


@pytest.mark.parametrize("quality", QUALITIES)
def test_encode_photos(dog_u8, people_u8, quality):
    assert_same([dog_u8, people_u8, dog_u8[:101, 3:250]], quality)


def test_gpu_encoded_files_decode_as_pil_decodes_them(dog_u8):
    imgs = [dog_u8, photo(375, 500, 1), photo(17, 33, 2)]
    files = assert_same(imgs, 90)
    dec = preprocess.decode_jpeg_batch(files)
    for d, f in zip(dec, files):
        assert np.array_equal(d.cpu().numpy(), read_image(io.BytesIO(f)))


def test_encode_views_of_one_buffer_and_refusals():
    files = [pil_jpeg(photo(40, 60, s), 90) for s in range(3)]
    views = preprocess.decode_jpeg_batch(files)
    got = encode_jpeg_batch(views, quality=75)
    assert got == [pil_jpeg(v.cpu().numpy(), 75) for v in views]
    with pytest.raises(ValueError):
        encode_jpeg_batch(views, quality=0)
    with pytest.raises(ValueError):
        encode_jpeg_batch([torch.zeros((4, 4, 3), dtype=torch.float32, device="cuda")])
    with pytest.raises(ValueError):
        encode_jpeg_batch([torch.zeros((4, 4, 3), dtype=torch.uint8)])
