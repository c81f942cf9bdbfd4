"""GPU progressive-JPEG decode (csrc/jpeg_progressive.cu): byte for byte Helper._read_img (PIL / libjpeg-turbo) over sizes,
sampling layouts, qualities, restart intervals, content and unusual scan scripts written by tests/progressive_writer.py;
mixed batches through submit_images, lanes and tiling; serve.py --gpu_progressive; corrupt input."""
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
from k210_yolo_framework_b200.pipeline import DetectionPipeline
from oracle import jpeg_ref as J
import progressive_writer as W
from test_gpu_jpeg import IN_HW, SIZES, _pipeline, detail, encode, flat, noise, photo

Q = [J.quality_table(J.STD_Q_LUMA, 90), J.quality_table(J.STD_Q_CHROMA, 90)]


def pil(data):
    return read_image(io.BytesIO(data))


def prog(img, layout="420", **kw):
    return encode(img, layout, progressive=True, **kw)


def assert_exact(files):
    for f in files:
        assert preprocess.progressive_gpu_decodable(f), preprocess.inspect_jpeg_progressive(f)
    got, status = preprocess.decode_progressive_jpeg_batch(files, with_status=True)
    torch.cuda.synchronize()
    assert (status[:, 0] == 0).all(), status
    for i, (g, f) in enumerate(zip(got, files)):
        ref = pil(f)
        g = g.cpu().numpy()
        assert g.shape == ref.shape, (i, g.shape, ref.shape)
        if not np.array_equal(g, ref):
            bad = np.argwhere(g != ref)
            raise AssertionError(f"file {i} {ref.shape}: {len(bad)} bytes differ, first at {bad[0].tolist()}: "
                                 f"{g[tuple(bad[0])]} vs {ref[tuple(bad[0])]}")


@pytest.mark.parametrize("layout", ["444", "422", "420", "gray"])
def test_sizes_and_sampling_bit_exact(layout):
    assert_exact([prog(photo(h, w, h * 7 + w), layout) for h, w in SIZES])


@pytest.mark.parametrize("layout", ["440", "411"])
def test_cv2_progressive_layouts_bit_exact(layout):
    import cv2
    files = []
    for h, w in [(1, 1), (9, 9), (33, 61), (375, 500), (720, 1280)]:
        params = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                  getattr(cv2, {"440": "IMWRITE_JPEG_SAMPLING_FACTOR_440", "411": "IMWRITE_JPEG_SAMPLING_FACTOR_411"}[layout])]
        ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(photo(h, w, h + w)[..., ::-1]), params)
        assert ok and buf.tobytes()[:4] == b"\xff\xd8\xff\xe0"
        files.append(buf.tobytes())
    assert_exact(files)


@pytest.mark.parametrize("quality", [10, 50, 75, 90, 95, 100])
def test_qualities_bit_exact(quality):
    assert_exact([prog(photo(h, w, quality + h), lay, quality=quality) for (h, w), lay in
                  zip([(375, 500), (33, 61), (224, 320), (17, 31), (9, 9)], ["420", "444", "422", "gray", "420"])])


@pytest.mark.parametrize("restart", [{"restart_marker_blocks": 1}, {"restart_marker_blocks": 4}, {"restart_marker_rows": 1}])
def test_restart_intervals_bit_exact(restart):
    files = [prog(photo(h, w, 3), lay, **restart) for (h, w), lay in
             zip([(375, 500), (33, 61), (8, 8), (101, 203)], ["420", "422", "444", "gray"])]
    for f in files:
        assert b"\xff\xdd" in f
    files.append(prog(noise(131, 97, 4), "420", quality=100, **restart))
    assert_exact(files)


@pytest.mark.parametrize("content", [photo, noise, flat, detail])
def test_content_bit_exact(content):
    # PIL cannot write a progressive 4:4:4 noise image this large (its encoder suspends mid-scan): the writer makes that one
    files = [prog(content(240, 352, 1), lay, quality=q) for lay in ("420", "444", "gray") for q in (75, 95)
             if not (content is noise and lay == "444")]
    if content is noise:
        files.append(_written(noise(240, 352, 1), "444", Y))
    assert_exact(files)


def _written(img, layout, script, **kw):
    coefs, samp = J.pixels_to_coefs(img, layout, Q)
    return W.write_progressive(coefs, {0: Q[0], 1: Q[1]}, height=img.shape[0], width=img.shape[1], sampling=samp, script=script,
                               **kw)


Y = W.DEFAULT_SCRIPT_YCC
FULL_DC = [((0, 1, 2), 0, 0, 0, 0)]
AC_FULL = [((c,), 1, 63, 0, 0) for c in (0, 1, 2)]
SCRIPTS = {
    "dc_without_approximation": FULL_DC + AC_FULL,
    "one_coefficient_bands": [((0, 1, 2), 0, 0, 0, 1)] + [((0,), k, k, 0, 0) for k in range(1, 33)]
                             + [((0,), 33, 63, 0, 0), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0), ((0, 1, 2), 0, 0, 1, 0)],
    "three_refinement_levels": [((0, 1, 2), 0, 0, 0, 3)] + [((c,), 1, 63, 0, 3) for c in (0, 1, 2)]
                               + [((0, 1, 2), 0, 0, a + 1, a) for a in (2, 1, 0)] + [((c,), 1, 63, a + 1, a) for a in (2, 1, 0)
                                                                                       for c in (0, 1, 2)],
    "high_band_partly_refined": FULL_DC + [((c,), 1, 9, 0, 0) for c in (0, 1, 2)] + [((c,), 10, 63, 0, 2) for c in (0, 1, 2)]
                                + [((0,), 10, 63, 2, 1)],
    "high_band_never_sent": FULL_DC + [((c,), 1, 9, 0, 0) for c in (0, 1, 2)] + [((0,), 10, 40, 0, 0)],
    "chroma_dc_separately": [((0,), 0, 0, 0, 0), ((1, 2), 0, 0, 0, 1), ((1, 2), 0, 0, 1, 0)] + AC_FULL,
    "same_level_disjoint_bands": [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 5, 0, 1), ((0,), 6, 63, 0, 1), ((0,), 1, 5, 1, 0),
                                  ((0,), 6, 63, 1, 0), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)],
}


@pytest.mark.parametrize("name", sorted(SCRIPTS))
@pytest.mark.parametrize("restart", [0, 3])
def test_unusual_scripts_bit_exact(name, restart):
    script = SCRIPTS[name]
    files = [_written(photo(h, w, len(name) + h), lay, script, restart=restart) for (h, w), lay in
             zip([(37, 53), (64, 80), (131, 97)], ["420", "444", "422"])]
    files.append(_written(noise(48, 40, 2), "420", script, restart=restart, huffman="flat"))
    assert_exact(files)


def test_grey_scripts_and_dri_changing_between_scans():
    grey = [((0,), 0, 0, 0, 2), ((0,), 1, 63, 0, 1), ((0,), 0, 0, 2, 1), ((0,), 0, 0, 1, 0), ((0,), 1, 63, 1, 0)]
    files = [_written(photo(61, 77, 1), "gray", grey, restart=[0, 5, 5, 1, 2]),
             _written(photo(61, 77, 2), "gray", W.DEFAULT_SCRIPT_GREY, restart=[3, 0, 7, 1, 0, 2]),
             _written(photo(100, 64, 3), "420", Y, restart=[2, 0, 1, 4, 4, 3, 0, 9, 1, 5])]
    assert_exact(files)


def test_long_eob_runs():
    """A flat image: AC first scans are one EOB run per restart interval, across thousands of blocks (EOB14 runs of up to
    32767 blocks), and runs that must end at each restart marker."""
    files = [_written(flat(720, 1280, 7), lay, script, restart=r) for lay, script in (("420", Y), ("gray", W.DEFAULT_SCRIPT_GREY))
             for r in (0, 7)]
    files.append(prog(flat(1080, 1920, 3), "444"))
    assert_exact(files)


@pytest.mark.parametrize("kind", ["dc", "full"])
def test_extreme_coefficients(kind):
    """Coefficients far outside what an 8-bit encoder writes (DC anywhere in +-32767, AC up to +-32767), sent with up to four
    successive-approximation levels."""
    rng = np.random.default_rng(3 if kind == "dc" else 4)
    blocks = J.extreme_blocks(rng, 12 * 16, kind)
    coefs = [blocks.reshape(12, 16, 8, 8)]
    q = np.ones(64, np.int64) * (1 if kind == "dc" else 2)
    files = [W.write_progressive(coefs, {0: q}, height=96, width=128, sampling=[(1, 1)], script=s, huffman=h)
             for s, h in ((W.DEFAULT_SCRIPT_GREY, "optimal"), ([((0,), 0, 0, 0, 4), ((0,), 1, 63, 0, 3), ((0,), 0, 0, 4, 3),
                                                               ((0,), 0, 0, 3, 2), ((0,), 0, 0, 2, 1), ((0,), 0, 0, 1, 0),
                                                               ((0,), 1, 63, 3, 2), ((0,), 1, 63, 2, 1), ((0,), 1, 63, 1, 0)],
                                                              "flat"))]
    assert_exact(files)


def test_more_than_48_images_one_call():
    rng = np.random.default_rng(5)
    lays = ["444", "422", "420", "gray"]
    assert_exact([prog(photo(int(rng.integers(1, 60)), int(rng.integers(1, 60)), i), lays[i % 4]) for i in range(100)])


def _mixed():
    """Baseline JPEG, progressive JPEGs, PNG, a progressive file the GPU leaves to PIL (block smoothing), a grey progressive."""
    from PIL import Image
    imgs = [photo(375, 500, 1), photo(240, 180, 2), photo(500, 333, 3), photo(100, 400, 4), photo(300, 300, 5)]
    b = io.BytesIO()
    Image.fromarray(imgs[3]).save(b, "PNG")
    smoothed = _written(imgs[4], "420", Y[:5])      # coefficients 1..5 of luma known to bit 2 only
    assert not preprocess.inspect_jpeg_progressive(smoothed)[2]
    return [encode(imgs[0], "420"), prog(imgs[1], "444", quality=95, restart_marker_blocks=2), prog(imgs[2], "420"), b.getvalue(),
            smoothed, prog(imgs[4], "gray")]


@pytest.mark.parametrize("lanes", [None, 2])
def test_mixed_batches_through_submit_images(golden_weights, voc_anchors, dog_u8, lanes):
    files = _mixed()
    assert [preprocess.progressive_gpu_decodable(f) for f in files] == [False, True, True, False, False, True]
    batches = [[files[0], dog_u8, bytearray(files[2]), memoryview(files[3])],
               [files[4], files[1], dog_u8[:, ::-1], files[5]],
               [prog(photo(1080, 1920, 11), "420", quality=95), files[3], files[1], dog_u8],
               [files[2], files[5], files[0], files[1]]]
    ref_batches = [[pil(bytes(e)) if isinstance(e, (bytes, bytearray, memoryview)) else e for e in b] for b in batches]

    def run(p, bs):
        limit = 2 if lanes is None else p.in_flight_limit()
        tickets, got = [], []
        for i, imgs in enumerate(bs):
            tickets.append(p.submit_images(imgs))
            if i + 1 >= limit:
                got.append(DetectionPipeline.records(*p.collect(tickets[i + 1 - limit])))
        for t in tickets[len(got):]:
            got.append(DetectionPipeline.records(*p.collect(t)))
        return got

    ref = run(_pipeline(golden_weights, voc_anchors, 4, lanes), ref_batches)
    on = _pipeline(golden_weights, voc_anchors, 4, lanes)
    on.enable_progressive_jpeg_decode()
    on.enable_png_decode()
    assert run(on, batches) == ref
    assert run(_pipeline(golden_weights, voc_anchors, 4, lanes), batches) == ref


def test_tiling_with_progressive_decode(golden_weights, voc_anchors):
    files = _mixed()
    imgs = [files[2], files[1], files[0]]
    ref = _pipeline(golden_weights, voc_anchors, 15)
    ref.enable_tiling(2, 2)
    pipe = _pipeline(golden_weights, voc_anchors, 15)
    pipe.enable_tiling(2, 2)
    pipe.enable_progressive_jpeg_decode()
    got = DetectionPipeline.records(*pipe.collect(pipe.submit_images(imgs)))
    assert got == DetectionPipeline.records(*ref.collect(ref.submit_images([pil(f) for f in imgs])))


def test_letterbox_batch_device_takes_progressive_files(dog_u8):
    from oracle import preprocess_ref
    files = _mixed()
    out = preprocess.letterbox_batch_device(files + [dog_u8], IN_HW, gpu_progressive=True).cpu().numpy()
    for got, f in zip(out, files):
        np.testing.assert_array_equal(got, preprocess_ref.letterbox(pil(f), IN_HW))
    np.testing.assert_array_equal(out[-1], preprocess_ref.letterbox(dog_u8, IN_HW))


def _garbled():
    """A complete progressive file whose last scan holds 64 one bits (no Huffman code is all ones)."""
    victim = bytearray(prog(photo(240, 320, 3), "420"))
    last = bytes(victim).rindex(b"\xff\xda")
    start = last + 2 + int.from_bytes(victim[last + 2:last + 4], "big")
    victim[start + 100:start + 116] = b"\xff\x00" * 8
    return bytes(victim)


def test_corrupt_entropy_data_sets_status_and_spares_the_others(golden_weights, voc_anchors):
    good = [prog(photo(200, 300, 1), "420"), prog(photo(64, 80, 2), "444", restart_marker_blocks=2)]
    garbled = _garbled()
    got, status = preprocess.decode_progressive_jpeg_batch([good[0], garbled, good[1]], with_status=True)
    assert status[0, 0] == 0 and status[2, 0] == 0 and status[1, 0] != 0, status
    np.testing.assert_array_equal(got[0].cpu().numpy(), pil(good[0]))
    np.testing.assert_array_equal(got[2].cpu().numpy(), pil(good[1]))
    with pytest.raises(Exception, match="corrupt progressive JPEG data: image 1"):
        preprocess.decode_progressive_jpeg_batch([good[0], garbled])
    with pytest.raises(Exception, match="corrupt progressive JPEG data: image 0"):
        preprocess.letterbox_batch_device([garbled, good[0]], IN_HW, gpu_progressive=True)
    pipe = _pipeline(golden_weights, voc_anchors, 4)
    pipe.enable_progressive_jpeg_decode()
    t = pipe.submit_images([good[0], good[1], garbled])
    t2 = pipe.submit_images([good[1], good[0]])
    with pytest.raises(Exception, match="corrupt progressive JPEG data: image 2"):
        pipe.collect(t)
    ref = _pipeline(golden_weights, voc_anchors, 4)
    assert DetectionPipeline.records(*pipe.collect(t2)) == DetectionPipeline.records(*ref.collect(ref.submit_images([good[1], good[0]])))


def test_serve_gpu_progressive_keeps_its_lines(tmp_path, golden_weights):
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    files = _mixed()
    for i, f in enumerate(files):
        (d / f"{i}.{'png' if f[:4] == b'\x89PNG' else 'jpg'}").write_bytes(f)

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(d), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.7, 0.5, 2
    with open(tmp_path / "off.jsonl", "w") as fh:
        assert serve.serve(a, fh) == len(files)
    a.gpu_progressive = True
    with open(tmp_path / "on.jsonl", "w") as fh:
        assert serve.serve(a, fh) == len(files)
    lines = open(tmp_path / "on.jsonl").read()
    assert lines == open(tmp_path / "off.jsonl").read()
    assert len([json.loads(l) for l in lines.splitlines()]) == len(files)
    assert isinstance(serve.load_image(str(d / "1.jpg"), gpu_progressive=True), bytes)
    assert isinstance(serve.load_image(str(d / "1.jpg")), np.ndarray)
