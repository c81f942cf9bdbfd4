"""The image kernels' one-pass limits and libjpeg's 65500-pixel limit, without a GPU: the GPU suites' cases exceed every
launch, chunk and pass limit the csrc sources declare; the encoder's host entry points and the decoder's marker walker
refuse what PIL cannot write or read; and tests/render_ref.py states the renderer's clamps for records PIL cannot draw."""
import ctypes
import io
import math
import os
import re

import numpy as np
import pytest
from PIL import Image

from conftest import ROOT
from render_ref import COORD_LIMIT, clamped_coord, clamped_hundredths, render_ref
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import K2YError, last_error, lib
from k210_yolo_framework_b200.draw import draw_detections, label_font_size
from k210_yolo_framework_b200.helper import _COLORMAP, read_image
from k210_yolo_framework_b200.render import JPEG_MAX_DIMENSION, LabelAtlas, glyphs, jpeg_header, label_text

CSRC = os.path.join(ROOT, "k210_yolo_framework_b200", "csrc")
OVERSIZE = [(1, JPEG_MAX_DIMENSION + 1), (65535, 1)]


def read_constants(name, *names):
    """Integer constexpr values of a csrc file, with the constants their expressions name resolved."""
    src = open(os.path.join(CSRC, name)).read()

    def value(n):
        m = re.search(rf"constexpr[^;]*\b{n}\s*=\s*([^,;]+)", src)
        assert m, n
        return int(eval(re.sub(r"[A-Za-z_]\w*", lambda t: str(value(t.group(0))), m.group(1))))
    return {n: value(n) for n in names}


def oversize_jpeg(h, w):
    """A PIL file of min(h, 65500) x min(w, 65500) whose SOF0 says h x w: what PIL (libjpeg) refuses to read."""
    b = io.BytesIO()
    Image.fromarray(np.full((min(h, 65500), min(w, 65500), 3), 90, np.uint8)).save(b, "JPEG", quality=90)
    f = bytearray(b.getvalue())
    i = f.index(b"\xff\xc0")
    f[i + 5:i + 9] = h.to_bytes(2, "big") + w.to_bytes(2, "big")
    return bytes(f)


def entropy_bytes(f):
    """The unstuffed entropy-coded data of a single-scan JPEG file."""
    sos = f.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(f[sos + 2:sos + 4], "big")
    return f[start:-2].replace(b"\xff\x00", b"\xff")


def test_cases_exceed_every_one_pass_limit():
    """A change to one of these constants must come with cases that still cross it."""
    import test_gpu_jpeg_encode_limits as E
    import test_gpu_letterbox_limits as L
    import test_gpu_render_limits as R
    lb = read_constants("preprocess.cu", "LB_MAX_IMAGES", "LB_CHUNK")
    rd = read_constants("render.cu", "RENDER_MAX_IMAGES", "TILE_W", "TILE_H", "RENDER_THREADS")
    enc = read_constants("jpeg_encode.cu", "CHUNK_BYTES", "SCAN_THREADS")
    # letterbox: three launch groups, the last one partial; a pipeline batch over one group; extremes on both sides of the
    # first chunk boundary and in the scalar tail; a source of more than 2000 min/max chunks
    chunk, group = lb["LB_CHUNK"], lb["LB_MAX_IMAGES"]
    assert L.LB_CHUNK == chunk
    assert L.GROUP_BATCH > 2 * group and L.GROUP_BATCH % group and L.PIPE_BATCH > group
    nbytes = L.PLANT_HW[0] * L.PLANT_HW[1] * 3
    pos = L.plant_positions(nbytes)
    assert nbytes > chunk and nbytes % 16 and {0, nbytes - 1, chunk - 1, chunk, nbytes // 16 * 16} <= set(pos)
    assert max(h * w * 3 for h, w in L.GEOMETRY_SOURCES) // chunk > 2000
    # rendering: records on both sides of one and two passes, a full C x K block, two and three launch groups
    t = rd["RENDER_THREADS"]
    assert t == rd["TILE_W"] * rd["TILE_H"] == R.RENDER_THREADS
    assert {t - 1, t, t + 1, 2 * t, 2 * t + 1} <= set(R.RECORD_COUNTS)
    assert R.MANY[0] == R.MANY[1] * R.MANY[2] > 8 * t
    m = rd["RENDER_MAX_IMAGES"]
    assert any(m < n < 2 * m for n in R.IMAGE_COUNTS) and any(n > 2 * m for n in R.IMAGE_COUNTS)
    # TrueType label sizes 1..60, the largest mask spanning several tiles both ways
    sizes = [label_font_size(h) for h in R.FONT_HEIGHTS]
    assert min(sizes) == 1 and max(sizes) == 60 and len(set(sizes)) == len(sizes)
    from PIL import ImageFont
    font = ImageFont.truetype(io.BytesIO(ImageFont.load_default().font_bytes), size=max(sizes))
    mask, _, _ = glyphs(font, label_text(79, 100))
    assert mask.shape[1] > 4 * rd["TILE_W"] and mask.shape[0] > 4 * rd["TILE_H"]
    # encoder: entropy-coded data longer than one pass of the stuffing scan (PIL writes the bytes the GPU must write)
    b = io.BytesIO()
    Image.fromarray(E.big_noise()).save(b, "JPEG", quality=E.BIG_QUALITY)
    assert len(entropy_bytes(b.getvalue())) > enc["SCAN_THREADS"] * enc["CHUNK_BYTES"] == 1024 * 8192


@pytest.mark.parametrize("hw", OVERSIZE + [(JPEG_MAX_DIMENSION + 1, 1), (1, 65535)])
def test_encoder_entry_points_refuse_over_65500(hw):
    h, w = hw
    with pytest.raises(ValueError, match="65500"):
        jpeg_header(h, w, 75)
    with pytest.raises(K2YError):       # what the library's refusal has always raised
        jpeg_header(h, w, 75)
    n = ctypes.c_size_t()
    assert lib.k2y_jpeg_encode_header(h, w, 75, None, 0, ctypes.byref(n)) != 0 and "65500" in last_error()
    hws = np.array([[8, 8], [h, w]], np.int32)
    offs = np.zeros(2, np.int64)
    assert lib.k2y_jpeg_encode_plan(2, hws.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                    offs.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)), 75, None, 0, ctypes.byref(n)) != 0
    assert "image 1" in last_error() and "65500" in last_error()
    with pytest.raises(OSError):      # libjpeg's "Maximum supported image dimension is 65500 pixels"
        Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(io.BytesIO(), "JPEG")


def test_encoder_entry_points_take_65500():
    n = ctypes.c_size_t()
    for h, w in [(1, JPEG_MAX_DIMENSION), (JPEG_MAX_DIMENSION, JPEG_MAX_DIMENSION)]:
        assert jpeg_header(h, w, 75)[-14:-12] == b"\xff\xda"
        hws = np.array([[h, w]], np.int32)
        assert lib.k2y_jpeg_encode_plan(1, hws.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                        np.zeros(1, np.int64).ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)), 75, None, 0,
                                        ctypes.byref(n)) == 0


@pytest.mark.parametrize("hw", OVERSIZE)
def test_decoder_leaves_files_over_65500_to_pil(hw):
    f = oversize_jpeg(*hw)
    with pytest.raises(OSError):      # libjpeg reports "Maximum supported image dimension is 65500 pixels" on stderr
        read_image(io.BytesIO(f))
    h, w, gpu, reason = preprocess.inspect_jpeg(f)
    assert (h, w) == hw and not gpu and "65500" in reason
    assert not preprocess.gpu_decodable(f)
    lim = oversize_jpeg(min(hw[0], JPEG_MAX_DIMENSION), min(hw[1], JPEG_MAX_DIMENSION))
    assert preprocess.inspect_jpeg(lim)[2] and preprocess.gpu_decodable(lim)


def test_render_ref_states_the_kernel_clamps():
    inf, nan = float("inf"), float("nan")
    assert [clamped_coord(v) for v in [inf, -inf, nan, 1e30, -1e30, 12.5, -0.5, 2.49, -3.5]] == \
        [COORD_LIMIT, -COORD_LIMIT, -COORD_LIMIT, COORD_LIMIT, -COORD_LIMIT, 13, 0, 2, -3]
    assert [clamped_hundredths(s) for s in [nan, -0.5, 1.5, inf, -inf, 0.125, 1.0, 0.0]] == [0, 0, 100, 100, 0, 12, 100, 0]
    # a record PIL cannot format draws as its clamped twin, which PIL draws when its rings do not cross
    from test_gpu_render_limits import non_finite_records
    from test_render_host import no_crossing
    h, w = 200, 300
    img = np.random.default_rng(0).integers(0, 256, (h, w, 3), dtype=np.uint8)
    atlas = LabelAtlas(20, "missing.otf").host(h)
    drawn = 0
    for c, i, s, *box in non_finite_records(h, w):
        twin = (c, i, float(np.float32(clamped_hundredths(s) / 100))) + tuple(float(clamped_coord(v)) for v in box)
        ref = render_ref(img, [twin], _COLORMAP, atlas)
        assert np.array_equal(render_ref(img, [(c, i, s, *box)], _COLORMAP, atlas), ref)
        if all(math.isfinite(v) for v in twin[2:]) and no_crossing(twin, h, w):
            assert np.array_equal(np.array(draw_detections(img, [twin], _COLORMAP, font_path="missing.otf")), ref), twin
            drawn += 1
    assert drawn >= 8
