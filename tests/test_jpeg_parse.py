"""Host-side JPEG header parsing (k2y_jpeg_inspect / k2y_jpeg_plan): dimensions, sampling, classification and its reason,
malformed headers, descriptor-blob sizes and the C-ABI struct — CPU only."""
import ctypes
import io

import numpy as np
import pytest

from k210_yolo_framework_b200 import _lib, preprocess


def _img(h=37, w=53):
    return np.random.default_rng(h * w).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _pil(img, mode=None, **kw):
    from PIL import Image
    b = io.BytesIO()
    im = Image.fromarray(img)
    (im.convert(mode) if mode else im).save(b, "JPEG", **kw)
    return b.getvalue()


def _cv2(img, factor):
    import cv2
    ok, buf = cv2.imencode(".jpg", img[..., ::-1].copy(), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, factor)])
    assert ok
    return buf.tobytes()


def _info(data):
    info = _lib.JpegInfo()
    buf = np.frombuffer(data, np.uint8)
    rc = _lib.lib.k2y_jpeg_inspect(buf.ctypes.data, buf.size, ctypes.byref(info))
    return rc, info


def _sof(data):
    i = 2
    while True:
        assert data[i] == 0xFF
        m = data[i + 1]
        if 0xC0 <= m <= 0xC3:
            return i
        i += 2 + int.from_bytes(data[i + 2:i + 4], "big")


def test_struct_size():
    assert ctypes.sizeof(_lib.JpegInfo) == 16 * 4 + 64


@pytest.mark.parametrize("enc,comps,sampling", [
    (lambda im: _pil(im, subsampling=0), 3, [(1, 1), (1, 1), (1, 1)]),
    (lambda im: _pil(im, subsampling=1), 3, [(2, 1), (1, 1), (1, 1)]),
    (lambda im: _pil(im, subsampling=2), 3, [(2, 2), (1, 1), (1, 1)]),
    (lambda im: _cv2(im, "IMWRITE_JPEG_SAMPLING_FACTOR_440"), 3, [(1, 2), (1, 1), (1, 1)]),
    (lambda im: _cv2(im, "IMWRITE_JPEG_SAMPLING_FACTOR_411"), 3, [(4, 1), (1, 1), (1, 1)]),
    (lambda im: _pil(im, "L"), 1, [(1, 1)]),
    (lambda im: _pil(im, optimize=True, restart_marker_blocks=3), 3, [(2, 2), (1, 1), (1, 1)]),
])
def test_supported_layouts(enc, comps, sampling):
    data = enc(_img())
    rc, info = _info(data)
    assert rc == 0 and info.gpu_decodable == 1 and info.reason == b""
    assert (info.height, info.width, info.components, info.precision) == (37, 53, comps, 8)
    assert [(info.h_samp[c], info.v_samp[c]) for c in range(comps)] == sampling
    assert info.sof_marker in (0xC0, 0xC1) and data.rfind(b"\xff\xda", 0, info.entropy_offset) > 0
    assert preprocess.inspect_jpeg(data) == (37, 53, True, "")
    assert preprocess.gpu_decodable(data) and preprocess.gpu_decodable(bytearray(data)) and preprocess.gpu_decodable(memoryview(data))


def test_restart_interval_is_reported():
    assert _info(_pil(_img(), restart_marker_blocks=3))[1].restart_interval == 3
    assert _info(_pil(_img()))[1].restart_interval == 0


def test_valid_files_the_gpu_does_not_take():
    img = _img()
    prog = _pil(img, progressive=True)
    assert preprocess.inspect_jpeg(prog) == (37, 53, False, "progressive (SOF 0xC2)")
    assert preprocess.inspect_jpeg(_pil(img, "CMYK")) == (37, 53, False, "4 components (CMYK/YCCK)")
    base = bytearray(_pil(img))
    s = _sof(base)
    arith = bytearray(base)
    arith[s + 1] = 0xC9
    assert preprocess.inspect_jpeg(bytes(arith)) == (37, 53, False, "arithmetic coding (SOF 0xC9)")
    twelve = bytearray(base)
    twelve[s + 4] = 12
    assert preprocess.inspect_jpeg(bytes(twelve)) == (37, 53, False, "12-bit samples")
    lossless = bytearray(base)
    lossless[s + 1] = 0xC3
    assert preprocess.inspect_jpeg(bytes(lossless))[2:] == (False, "lossless (SOF 0xC3)")
    assert not preprocess.gpu_decodable(prog) and not preprocess.gpu_decodable(b"\x89PNG\r\n\x1a\n")


@pytest.mark.parametrize("cut", [3, 10, 25, 100, 300])
def test_truncated_headers_are_invalid(cut):
    data = _pil(_img())
    rc, _ = _info(data[:cut])
    assert rc == _lib.lib.k2y_jpeg_inspect(None, 0, None) == -1
    rc, _ = _info(data[:cut])
    assert rc == -1 and "k2y_jpeg_inspect" in _lib.last_error()
    with pytest.raises(_lib.K2YError):
        preprocess.inspect_jpeg(data[:cut])


def test_garbled_headers_name_the_marker():
    data = bytearray(_pil(_img()))
    s = _sof(data)
    bad = bytearray(data)
    bad[s + 2:s + 4] = b"\xff\xf0"        # SOF length past the end of the file
    assert _info(bytes(bad))[0] == -1 and "0xC0" in _lib.last_error()
    bad = bytearray(data)
    bad[s + 1] = 0xF3                     # a marker no decoder knows
    assert _info(bytes(bad))[0] == -1 and "unsupported marker 0xF3" in _lib.last_error()
    bad = bytearray(data)
    bad[s + 9] = 0                        # zero components
    assert _info(bytes(bad))[0] == -1 and "SOF" in _lib.last_error()
    assert _info(b"\x89PNG\r\n\x1a\n" + bytes(100))[0] == -1 and "no SOI" in _lib.last_error()


def test_plan_blob_sizes_and_rejects_non_gpu_files():
    img = _img()
    files = [np.frombuffer(_pil(img, subsampling=2), np.uint8), np.frombuffer(_pil(img, "L"), np.uint8),
             np.frombuffer(_pil(img, subsampling=0, restart_marker_blocks=1), np.uint8)]
    dst = np.array([0, 16, 32], np.int64)
    one = preprocess._jpeg_layout(files[:1], dst[:1], 0)[3]
    sizes = [preprocess._jpeg_plan([f], np.zeros(1, np.int64), dst[:1], None) for f in files]
    # header 96, 608 per image, 16 per restart segment (rounded up to 16 as a whole), 1424 per Huffman table
    mcus444 = 5 * 7
    assert sizes == [96 + 608 + 16 + 6 * 1424, 96 + 608 + 16 + 2 * 1424, 96 + 608 + 16 * mcus444 + 6 * 1424]
    assert one >= sizes[0] + files[0].size
    both = preprocess._jpeg_plan(files, np.zeros(3, np.int64), dst, None)
    assert both == 96 + 3 * 608 + 16 * (2 + mcus444) + 14 * 1424
    blob = np.zeros(both + 16, np.uint8)
    blob = blob[(-blob.ctypes.data) % 16:][:both]
    offs = np.array([0, 4096, 8192], np.int64)
    preprocess._jpeg_plan(files, offs, dst, blob)
    ws = ctypes.c_size_t()
    assert _lib.lib.k2y_jpeg_workspace_bytes(blob.ctypes.data, ctypes.byref(ws)) == 0 and ws.value > 0
    assert _lib.lib.k2y_jpeg_workspace_bytes(np.zeros(128, np.uint8).ctypes.data, ctypes.byref(ws)) == -1
    with pytest.raises(_lib.K2YError, match="not decodable on the GPU: progressive"):
        preprocess._jpeg_plan([np.frombuffer(_pil(img, progressive=True), np.uint8)], np.zeros(1, np.int64), dst[:1], None)


def test_layout_routes_files():
    from PIL import Image
    img = _img()
    png = io.BytesIO()
    Image.fromarray(img).save(png, "PNG")
    entries = [_pil(img), img, bytearray(_pil(img, progressive=True)), memoryview(png.getvalue())]
    lay = preprocess.BatchLayout(entries, (224, 320))
    assert [i for i, _ in lay.jpeg] == [0]
    assert lay.arrays[0] is None and lay.arrays[1] is img
    np.testing.assert_array_equal(lay.arrays[3], img)          # PNG decoded on the host
    assert lay.hw.tolist() == [[37, 53]] * 4
    assert lay.host_ranges() == [(int(lay.offsets[1]), int(lay.offsets[3] + 37 * 53 * 3))]
    assert lay.jpeg_plan[0][0] >= lay.nbytes and lay.jpeg_plan[0][0] % 16 == 0
    gaps = preprocess.BatchLayout([img, _pil(img), img, img], (224, 320))
    assert gaps.host_ranges() == [(0, 37 * 53 * 3), (int(gaps.offsets[2]), int(gaps.offsets[3] + 37 * 53 * 3))]
    for bad in ([b""], ["x.jpg"], [b"not an image"], [memoryview(np.zeros((4, 4), np.uint8)[:, ::2])]):
        with pytest.raises(ValueError):
            preprocess.BatchLayout(bad, (32, 32))


def test_truncated_file_goes_to_the_host_decoder():
    """A JPEG cut inside its entropy-coded data has valid headers but no EOI marker: the batch route hands it to the host
    decoder, which refuses it as PIL does (``ValueError`` before anything is enqueued), instead of decoding undefined pixels."""
    data = _pil(_img(64, 64))
    cut = data[:len(data) - 40]
    assert preprocess.inspect_jpeg(cut)[2] and not preprocess.gpu_decodable(cut)
    assert preprocess.gpu_decodable(data) and not preprocess.gpu_decodable(data + b"trailer")
    with pytest.raises(ValueError, match="image 1: cannot decode"):
        preprocess.BatchLayout([data, cut], (32, 32))
    lay = preprocess.BatchLayout([data, data + b"trailer"], (32, 32))   # appended data: decoded on the host, like PIL
    assert [i for i, _ in lay.jpeg] == [0] and lay.arrays[1] is not None


def test_oversubscribed_huffman_table_is_invalid():
    """Code lengths that cannot all be assigned (three 1-bit codes) are refused by the parser, as libjpeg refuses the file."""
    data = bytearray(_pil(_img()))
    i = data.index(b"\xff\xc4")
    assert data[i + 5] == 0 and data[i + 7] >= 3   # bits[1], bits[3] of the first (standard DC) table
    data[i + 5] = 3
    data[i + 7] -= 3                     # the same symbol count: the segment stays well-formed
    rc, _ = _info(bytes(data))
    assert rc == -1 and "more codes than its code lengths allow" in _lib.last_error()
    assert not preprocess.gpu_decodable(bytes(data))
    with pytest.raises(ValueError):
        preprocess.BatchLayout([bytes(data)], (32, 32))


def test_images_too_large_for_the_gpu_are_left_to_the_host():
    data = bytearray(_pil(_img()))
    s = _sof(data)
    data[s + 5:s + 9] = (40000).to_bytes(2, "big") + (40000).to_bytes(2, "big")    # 40000 x 40000
    h, w, ok, why = preprocess.inspect_jpeg(bytes(data))
    assert (h, w, ok) == (40000, 40000, False) and why.startswith("too large for the GPU decoder")
