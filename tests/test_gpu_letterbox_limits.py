"""The batched letterbox (csrc/preprocess.cu) past its one-pass limits, exactly against oracle/preprocess_ref.letterbox: the
per-image min/max reduction with its extremes planted at the chunk, vector and tail edges (aligned and unaligned), more
images than one launch takes, and extreme source geometry."""
import ctypes
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from PIL import Image

from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import check, lib
from k210_yolo_framework_b200.pipeline import DetectionPipeline
from oracle import preprocess_ref

LB_CHUNK = 256 * 64           # csrc/preprocess.cu: source bytes per block of the min/max pass (test_image_limits checks it)
PLANT_HW = (61, 97)           # 17751 bytes: two min/max chunks, the second ending in a 7-byte scalar tail
GROUP_BATCH = 97              # 48 + 48 + 1: three letterbox launches
PIPE_BATCH = 64
GEOMETRY_SOURCES = [(1, 4000), (4000, 1), (2, 3), (3000, 4000)]
GEOMETRY_TARGETS = [(224, 320), (608, 608), (97, 131)]
LO, HI = 3, 250               # the planted extremes; every other value lies in [40, 200]


def plant_positions(nbytes):
    """Byte offsets of the planted extremes: the first byte, the last byte (scalar tail), the last byte of the first chunk
    and the first of the second, the first byte of the final partial 16-byte vector and one inside it."""
    tail = nbytes // 16 * 16
    return [0, nbytes - 1, LB_CHUNK - 1, LB_CHUNK, tail, tail + 3]


def planted(hw, lo_at, hi_at, seed):
    img = np.random.default_rng(seed).integers(40, 201, hw + (3,), dtype=np.uint8)
    flat = img.reshape(-1)
    flat[lo_at], flat[hi_at] = LO, HI
    return img


def planted_cases():
    nbytes = PLANT_HW[0] * PLANT_HW[1] * 3
    pos = plant_positions(nbytes)
    assert nbytes % 16 and pos[4] > LB_CHUNK and len(set(pos)) == len(pos)
    return [(planted(PLANT_HW, p, q, i), p, q) for i, (p, q) in enumerate(zip(pos, pos[1:] + pos[:1]))]


def assert_sensitive(img, at, in_hw):
    """The oracle's output changes when the planted byte takes its neighbour's value: a min/max that missed it shows."""
    other = img.copy()
    flat = other.reshape(-1)
    flat[at] = flat[at + 3] if at + 3 < flat.size else flat[at - 3]
    assert not np.array_equal(preprocess_ref.letterbox(other, in_hw), preprocess_ref.letterbox(img, in_hw)), at


@pytest.mark.parametrize("in_hw", [PLANT_HW, (224, 320)], ids=["identity", "upscale"])
def test_planted_extremes_at_chunk_vector_and_tail_edges(in_hw):
    cases = planted_cases()
    for img, p, q in cases:
        assert_sensitive(img, p, in_hw)
        assert_sensitive(img, q, in_hw)
    out = preprocess.letterbox_batch_device([c[0] for c in cases], in_hw).cpu().numpy()
    for got, (img, p, q) in zip(out, cases):
        np.testing.assert_array_equal(got, preprocess_ref.letterbox(img, in_hw), err_msg=f"min at {p}, max at {q}")


def test_unaligned_offsets_take_the_scalar_path():
    """One k2y_letterbox_u8_batch call over images packed at offsets that are not multiples of 16 (the Python API always
    aligns them), planted extremes included."""
    cases = planted_cases()
    imgs = [c[0] for c in cases] + [np.random.default_rng(9).integers(1, 256, (5, 7, 3), dtype=np.uint8)]
    offsets, pos = [], 3
    for im in imgs:
        offsets.append(pos)
        pos += im.size + 5 + 2 * len(offsets)          # odd gaps: offsets 3, 17759, ...
    assert any(o % 16 for o in offsets) and all(o % 16 for o in offsets[:2])
    host = np.zeros(pos + 16, np.uint8)
    for im, o in zip(imgs, offsets):
        host[o:o + im.size] = im.reshape(-1)
    src = torch.from_numpy(host).cuda()
    in_hw = (224, 320)
    n = len(imgs)
    out = torch.empty((n,) + in_hw + (3,), dtype=torch.uint8, device="cuda")
    minmax = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    offs = np.array(offsets, np.int64)
    hw = np.array([im.shape[:2] for im in imgs], np.int32)
    mats = np.array([preprocess.letterbox_params(im.shape[:2], in_hw)[2][:2].reshape(-1) for im in imgs], np.float64)
    st = torch.cuda.current_stream()
    check(lib.k2y_letterbox_u8_batch(src.data_ptr(), n, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                     hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), mats.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                     out.data_ptr(), in_hw[0], in_hw[1], None, minmax.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
    got = out.cpu().numpy()
    assert minmax.cpu().numpy().tolist() == [[255 - int(im.min()), int(im.max())] for im in imgs]
    for i, im in enumerate(imgs):
        np.testing.assert_array_equal(got[i], preprocess_ref.letterbox(im, in_hw), err_msg=f"image {i} at offset {offsets[i]}")


def group_images():
    """GROUP_BATCH upscaled images of distinct sizes whose minimum grows with the index (and whose maximum falls), so an image
    that took another launch group's min/max would be clipped differently at its fill border."""
    imgs = []
    for i in range(GROUP_BATCH):
        h, w = 20 + (i * 7) % 90, 30 + (i * 13) % 120
        lo, hi = 1 + i, 254 - i
        img = np.random.default_rng(100 + i).integers(lo, hi + 1, (h, w, 3), dtype=np.uint8)
        img.reshape(-1)[[i % img.size, -1 - (i % 5)]] = lo, hi
        imgs.append(img)
    assert len({im.shape for im in imgs}) == GROUP_BATCH
    return imgs


def test_three_launch_groups_in_one_call():
    imgs = group_images()
    in_hw = (224, 320)
    n, extra = len(imgs), 3
    out = torch.full((n + extra,) + in_hw + (3,), 77, dtype=torch.uint8, device="cuda")
    hw = torch.full((n + extra, 2), -1.0, dtype=torch.float32, device="cuda")
    preprocess.letterbox_batch_device(imgs, in_hw, out=out, image_hw_out=hw)
    got = out.cpu().numpy()
    for i, im in enumerate(imgs):
        np.testing.assert_array_equal(got[i], preprocess_ref.letterbox(im, in_hw), err_msg=f"image {i}")
    assert hw[:n].cpu().numpy().tolist() == [list(im.shape[:2]) for im in imgs]
    assert bool((out[n:] == 77).all()) and bool((hw[n:] == -1).all())       # rows past n untouched


def _jpeg(img, q=90):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=q)
    return b.getvalue()


def test_pipeline_batch_over_one_launch_group(golden_weights, voc_anchors, photos_for_limits):
    """submit_images with 64 mixed images (arrays and GPU-decoded JPEGs): two letterbox launches, the per-image route's
    records."""
    from test_gpu_ingest import _pipeline, _reference
    from k210_yolo_framework_b200.helper import read_image
    items, pixels = [], []
    for i in range(PIPE_BATCH):
        img = photos_for_limits[i % len(photos_for_limits)]
        if i % 3 == 1:
            f = _jpeg(img, 70 + i % 30)
            assert preprocess.gpu_decodable(f)
            items.append(f)
            pixels.append(read_image(io.BytesIO(f)))
        else:
            items.append(img)
            pixels.append(img)
    pipe = _pipeline(golden_weights, voc_anchors, PIPE_BATCH)
    got = DetectionPipeline.records(*pipe.collect(pipe.submit_images(items)))
    ref = _reference(golden_weights, voc_anchors, [pixels], PIPE_BATCH)[0]
    assert got == ref
    assert sum(len(r) for r in got[48:]) > 0


@pytest.fixture(scope="module")
def photos_for_limits(dog_u8, people_u8):
    """Photo crops of 16 different sizes."""
    out = []
    for k in range(16):
        src = dog_u8 if k % 2 else people_u8
        out.append(np.ascontiguousarray(src[(5 * k) % 40:, (11 * k) % 90:][:, ::(-1 if k % 4 == 3 else 1)]))
    return out


def test_extreme_geometry():
    imgs = []
    for i, (h, w) in enumerate(GEOMETRY_SOURCES):
        img = np.random.default_rng(i).integers(20, 231, (h, w, 3), dtype=np.uint8)
        img.reshape(-1)[-1] = 7 + i                      # the minimum sits in the last byte of the last chunk
        imgs.append(img)
    for in_hw in GEOMETRY_TARGETS:
        out = preprocess.letterbox_batch_device(imgs, in_hw).cpu().numpy()
        for got, img in zip(out, imgs):
            np.testing.assert_array_equal(got, preprocess_ref.letterbox(img, in_hw), err_msg=f"{img.shape[:2]} -> {in_hw}")
