"""Host-side PNG parsing and routing (k2y_png_inspect / k2y_png_plan, preprocess.BatchLayout(gpu_png=True)): which files the GPU
takes and the reason for the others, plan and workspace sizes, the staging layout beside GPU JPEGs, and evaluate_map's size
check.  No GPU needed."""
import ctypes
import io
import struct
import zlib

import numpy as np
import pytest

from png_cases import chunk, ihdr, make_png, pil_png, png_file, SIG
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import K2YError, check, lib

IN_HW = (224, 320)


def _rgb(w=6, h=4):
    return png_file(w, h, 2, 8, zlib.compress(bytes((1 + 3 * w) * h)))


def _plte(n=4):
    return bytes(range(3 * n))


def test_every_supported_kind_is_gpu_decodable():
    rng = np.random.default_rng(0)
    for color, depth in [(0, 1), (0, 2), (0, 4), (0, 8), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16), (6, 8), (6, 16)]:
        f = make_png(rng, 5, 3, color, depth)
        assert preprocess.inspect_png(f) == (3, 5, True, ""), (color, depth)
        assert preprocess.png_gpu_decodable(f) and not preprocess.gpu_decodable(f)


def _reason(data):
    return preprocess.inspect_png(data)[2:]


def test_routing_rules_and_reasons():
    z = zlib.compress(bytes(13 * 2))
    assert _reason(png_file(4, 2, 2, 8, z, interlace=1)) == (False, "interlaced (Adam7)")
    assert _reason(png_file(4, 2, 0, 16, zlib.compress(bytes(9 * 2)))) == (False, "16-bit greyscale")
    assert _reason(png_file(4, 2, 2, 8, z, before=chunk(b"acTL", bytes(8)))) == (False, "APNG (acTL chunk)")
    assert _reason(png_file(4, 2, 3, 8, zlib.compress(bytes(5 * 2)))) == (False, "palette image without PLTE")
    assert _reason(png_file(4, 2, 3, 8, zlib.compress(bytes(5 * 2)), plte=b"\x00" * 4)) == (False, "damaged PLTE chunk")
    assert _reason(png_file(4, 2, 2, 8, z, before=chunk(b"ABCD", b"x"))) == (False, "unknown critical chunk ABCD")
    bad_crc = bytearray(png_file(4, 2, 2, 8, z, before=chunk(b"tEXt", b"k\x00v")))
    bad_crc[bad_crc.index(b"tEXt") + 7] ^= 1
    assert _reason(bytes(bad_crc)) == (False, "CRC error in tEXt chunk")
    assert _reason(png_file(4, 2, 2, 8, z, split=[5], between=chunk(b"tEXt", b"k\x00v"))) == (False, "chunk between IDAT chunks")
    assert _reason(png_file(4, 2, 2, 8, z, iend=False)) == (False, "no IEND chunk")
    assert _reason(png_file(4, 2, 2, 8, b"\x78\xbb" + z[2:]))[0] is False          # FDICT
    assert _reason(png_file(4, 2, 2, 8, b"\x79\x9c" + z[2:]))[0] is False          # CM 9
    assert _reason(png_file(4, 2, 2, 8, b"\x88\x98" + z[2:]))[0] is False          # CINFO 8
    assert _reason(png_file(4, 2, 2, 8, b"\x78\x9d" + z[2:]))[0] is False          # FCHECK
    assert _reason(png_file(70000, 1, 0, 8, zlib.compress(bytes(70001)))) == (False, "more than 65535 rows or columns")
    # 60000 x 60000 RGBA16: 28.8 GB of filtered rows, which PIL opens once MAX_IMAGE_PIXELS is lifted
    assert _reason(png_file(60000, 60000, 6, 16, zlib.compress(b""))) == (False, "more than 2 GiB of filtered image data")
    assert _reason(png_file(16384, 16384, 6, 16, zlib.compress(b""))) == (False, "more than 2 GiB of filtered image data")
    just_under = np.frombuffer(png_file(16383, 16383, 6, 16, zlib.compress(b"")), np.uint8)    # 2^31 - 245752 bytes
    info = preprocess.PngInfo()          # the library's own verdict (PIL's pixel limit, checked in Python, would refuse it)
    check(lib.k2y_png_inspect(just_under.ctypes.data, just_under.size, ctypes.byref(info)))
    assert info.gpu_decodable == 1
    # ancillary chunks after the image data, a damaged IDAT CRC, tRNS on a palette: still the GPU's
    ok = bytearray(png_file(4, 2, 3, 8, zlib.compress(bytes(5 * 2)), plte=_plte(), before=chunk(b"tRNS", b"\x00"),
                            after=chunk(b"tEXt", b"a\x00b")))
    ok[ok.index(b"IDAT") + 4 + int.from_bytes(ok[ok.index(b"IDAT") - 4:ok.index(b"IDAT")], "big")] ^= 1
    assert _reason(bytes(ok)) == (True, "")


def test_decompression_bomb_limit_goes_to_pil(monkeypatch):
    from PIL import Image
    f = _rgb(60, 50)
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 2999)
    h, w, ok, why = preprocess.inspect_png(f)
    assert (h, w, ok) == (50, 60, False) and "decompression-bomb" in why
    assert not preprocess.png_gpu_decodable(f)


def test_malformed_headers_raise():
    with pytest.raises(K2YError, match="not a PNG"):
        preprocess.inspect_png(b"GIF89a" + bytes(40))
    bad = bytearray(_rgb())
    bad[20] ^= 1                           # IHDR CRC
    with pytest.raises(K2YError, match="IHDR"):
        preprocess.inspect_png(bytes(bad))
    with pytest.raises(K2YError, match="IHDR"):
        preprocess.inspect_png(SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 2, 3, 2, 0, 0, 0)) + chunk(b"IEND", b""))
    assert not preprocess.png_gpu_decodable(b"\x89PNG")


def test_plan_and_workspace_sizes():
    files = [np.frombuffer(make_png(np.random.default_rng(k), 7 + k, 3 + k, 2, 8, split=[3, 9]), np.uint8) for k in range(3)]
    dst = np.zeros(3, np.int64)
    one = preprocess._png_plan(files[:1], dst[:1], dst[:1], None)
    three = preprocess._png_plan(files, dst, dst, None)
    assert three > one > 0
    blob = np.zeros(three + 16, np.uint8)
    blob = blob[(-blob.ctypes.data) % 16:][:three]
    preprocess._png_plan(files, np.arange(3, dtype=np.int64) * 4096, dst, blob)
    ws = ctypes.c_size_t()
    check(lib.k2y_png_workspace_bytes(blob.ctypes.data, ctypes.byref(ws)))
    # per image: the zlib stream + 8 zero bytes and the filtered rows, each 16-byte aligned
    expect = 0
    for k, f in enumerate(files):
        info = preprocess.PngInfo()
        check(lib.k2y_png_inspect(f.ctypes.data, f.size, ctypes.byref(info)))
        raw = (3 + k) * (1 + 3 * (7 + k))
        # stream + 8 zero bytes, filtered rows, two int64 words, one chunk: its 32-byte record and raw uint16 symbols
        expect += -(-(info.stream_bytes + 8) // 16) * 16 + -(-raw // 16) * 16 + 16 + 32 + -(-2 * raw // 16) * 16
    assert ws.value == expect
    with pytest.raises(K2YError, match="not decodable on the GPU: interlaced"):
        preprocess._png_plan([np.frombuffer(png_file(4, 2, 2, 8, zlib.compress(bytes(26)), interlace=1), np.uint8)], dst[:1], dst[:1], None)


def _jpeg(img):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=90)
    return b.getvalue()


def test_layout_routes_pngs_only_when_asked():
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    png, jpg = pil_png(img), _jpeg(img)
    host_png = png_file(4, 2, 0, 16, zlib.compress(bytes(9 * 2)))
    images = [png, img, jpg, host_png, png]
    default = preprocess.BatchLayout(images, IN_HW)
    assert default.png == [] and default.png_plan is None and default.staged_end == default.jpeg_plan[3]
    assert [a is None for a in default.arrays] == [False, False, True, False, False]
    lay = preprocess.BatchLayout(images, IN_HW, gpu_png=True)
    assert [i for i, _ in lay.png] == [0, 4] and [i for i, _ in lay.jpeg] == [2]
    assert [a is None for a in lay.arrays] == [True, False, True, False, True]
    np.testing.assert_array_equal(lay.offsets, default.offsets)
    np.testing.assert_array_equal(lay.hw, default.hw)
    np.testing.assert_array_equal(lay.matrices, default.matrices)
    assert lay.host_ranges() == [(int(lay.offsets[1]), int(lay.offsets[1] + 37 * 53 * 3)),
                                 (int(lay.offsets[3]), int(lay.offsets[3] + 2 * 4 * 3))]
    # the PNGs and their blob lie behind the JPEGs' range, all 16-byte aligned, up to staged_end
    src, blob_at, blob_bytes, end = lay.png_plan
    assert src[0] >= lay.jpeg_plan[3] and src[0] % 16 == 0 and all(s % 16 == 0 for s in src) and blob_at % 16 == 0
    assert end == lay.staged_end == blob_at + blob_bytes
    np.testing.assert_array_equal(lay.png_dst, lay.offsets[[0, 4]])
    only_png = preprocess.BatchLayout([png, img], IN_HW, gpu_png=True)
    assert only_png.jpeg_plan is None and only_png.png_plan[0][0] == (only_png.nbytes + 15) // 16 * 16


def test_load_checked_takes_png_sizes_from_the_header(tmp_path):
    import evaluate_map
    rng = np.random.default_rng(2)
    p = tmp_path / "a.png"
    p.write_bytes(pil_png(rng.integers(0, 256, (21, 34, 3), dtype=np.uint8)))
    got = evaluate_map.load_checked(str(p), (21, 34), gpu_png=True)
    assert isinstance(got, bytes)
    assert evaluate_map.load_checked(str(p), (21, 34)).shape == (21, 34, 3)
    with pytest.raises(ValueError, match="differs"):
        evaluate_map.load_checked(str(p), (34, 21), gpu_png=True)


def test_serve_flag():
    import serve
    ap = serve.build_parser()
    assert ap.parse_args(["ck", "imgs"]).gpu_png is False
    assert ap.parse_args(["ck", "imgs", "--gpu_png"]).gpu_png is True
