"""Host-side progressive-JPEG parsing and routing (k2y_jpeg_progressive_inspect / _plan, BatchLayout(gpu_progressive=True)),
and tests/progressive_writer.py against PIL: which scripts the GPU takes, which are malformed (refused as libjpeg-turbo's
JERR_BAD_PROGRESSION refuses them, naming the scan) and which stay with PIL; the block-smoothing rule of jdcoefct.c as the
installed libjpeg-turbo applies it; blob sizes; the baseline entry points unchanged on progressive files."""
import ctypes
import io

import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import JpegProgressiveInfo, K2YError, lib
from k210_yolo_framework_b200.helper import read_image
from oracle import jpeg_ref as J
import progressive_writer as W

Q = [J.quality_table(J.STD_Q_LUMA, 90), J.quality_table(J.STD_Q_CHROMA, 90)]
FULL_DC = [((0, 1, 2), 0, 0, 0, 0)]
CHROMA_AC = [((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)]


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([127.5 + 127.5 * np.sin(rng.uniform(0.02, 0.2) * (xx + yy * rng.uniform(0, 1)) + c) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 10, base.shape), 0, 255).astype(np.uint8)


def pil_progressive(img, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=90, progressive=True, **kw)
    return b.getvalue()


def coefs_of(img, layout="420"):
    return J.pixels_to_coefs(img, layout, Q)


def written(script, img=None, layout="420", **kw):
    img = photo(37, 53, 1) if img is None else img
    coefs, samp = coefs_of(img, layout)
    return W.write_progressive(coefs, {0: Q[0], 1: Q[1]}, height=img.shape[0], width=img.shape[1], sampling=samp, script=script, **kw)


def info(data):
    buf = np.frombuffer(data, np.uint8)
    out = JpegProgressiveInfo()
    assert lib.k2y_jpeg_progressive_inspect(buf.ctypes.data, buf.size, ctypes.byref(out)) == 0
    return out


def patch_scan(data, index, ss=None, se=None, ah=None, al=None):
    """`data` with the parameters of its `index`-th SOS replaced."""
    d = bytearray(data)
    at = -1
    for _ in range(index + 1):
        at = bytes(d).index(b"\xff\xda", at + 1)
    end = at + 2 + int.from_bytes(d[at + 2:at + 4], "big")
    old_ah, old_al = d[end - 1] >> 4, d[end - 1] & 15
    d[end - 3] = d[end - 3] if ss is None else ss
    d[end - 2] = d[end - 2] if se is None else se
    d[end - 1] = ((old_ah if ah is None else ah) << 4) | (old_al if al is None else al)
    return bytes(d)


def test_pil_progressive_files_decode_in_four_levels_and_the_baseline_view_is_unchanged():
    img = photo(37, 53, 2)
    for kw in ({}, {"subsampling": 0}, {"subsampling": 1}, {"restart_marker_blocks": 1}, {"restart_marker_rows": 1}):
        f = pil_progressive(img, **kw)
        assert preprocess.inspect_jpeg_progressive(f) == (37, 53, True, "")
        assert preprocess.progressive_gpu_decodable(f)
        i = info(f)
        assert (i.scans, i.levels, i.sof_marker) == (10, 4, 0xC2)    # libjpeg's default script: four entropy launches
        assert preprocess.inspect_jpeg(f) == (37, 53, False, "progressive (SOF 0xC2)")
        assert not preprocess.gpu_decodable(f)
        with pytest.raises(K2YError, match="not decodable on the GPU: progressive"):
            preprocess._jpeg_plan([np.frombuffer(f, np.uint8)], np.zeros(1, np.int64), np.zeros(1, np.int64), None)
    grey = pil_progressive(img[..., 0])
    assert preprocess.inspect_jpeg_progressive(grey)[2] and info(grey).scans == 6


def test_baseline_and_other_files_are_not_for_the_progressive_decoder():
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(photo(9, 9, 1)).save(b, "JPEG")
    assert preprocess.inspect_jpeg_progressive(b.getvalue()) == (9, 9, False, "sequential (SOF 0xC0)")
    assert not preprocess.progressive_gpu_decodable(b.getvalue())
    b = io.BytesIO()
    Image.fromarray(photo(9, 9, 1)).save(b, "PNG")
    assert not preprocess.progressive_gpu_decodable(b.getvalue())
    with pytest.raises(K2YError, match="not a JPEG"):
        preprocess.inspect_jpeg_progressive(b.getvalue())
    f = pil_progressive(photo(9, 9, 1))
    assert preprocess.inspect_jpeg_progressive(f[:-2])[2:] == (False, "file ends before its EOI marker")
    assert not preprocess.progressive_gpu_decodable(f[:-2]) and not preprocess.progressive_gpu_decodable(f + b"\0")


@pytest.mark.parametrize("scan, change, what", [
    (0, dict(se=1), "scan 0 .* a DC scan with Se != 0"),
    (1, dict(ss=6, se=5), "scan 1 .* an AC scan with Ss > Se or Se > 63"),
    (1, dict(se=64), "scan 1 .* an AC scan with Ss > Se or Se > 63"),
    (5, dict(ah=2, al=0), "scan 5 .* a refinement with Al != Ah - 1"),
    (0, dict(al=14), "scan 0 .* Al > 13"),
])
def test_malformed_progressions_name_the_scan(scan, change, what):
    f = patch_scan(pil_progressive(photo(24, 40, 3)), scan, **change)
    with pytest.raises(K2YError, match=what):
        preprocess.inspect_jpeg_progressive(f)
    assert not preprocess.progressive_gpu_decodable(f)
    with pytest.raises(ValueError, match=what):
        preprocess._jpeg_layout([np.frombuffer(f, np.uint8)], np.zeros(1, np.int64), 0, preprocess._progressive_plan)


def test_an_ac_scan_of_two_components_is_malformed():
    with pytest.raises(K2YError, match="scan 1 .* an AC scan of more than one component"):
        preprocess.inspect_jpeg_progressive(written(FULL_DC + [((1, 2), 1, 63, 0, 0)]))


@pytest.mark.parametrize("script, reason", [
    ([((0,), 1, 63, 0, 0)] + FULL_DC + CHROMA_AC, "scan 0: AC of component 0 before its DC"),
    (FULL_DC + CHROMA_AC + [((0,), 1, 63, 0, 1), ((0,), 1, 63, 2, 1)], "scan 4: refinement Ah=2 of coefficient 1 of component 0"),
    (FULL_DC + CHROMA_AC + [((0,), 1, 63, 2, 1)], "scan 3: refinement Ah=2 of coefficient 1 of component 0"),
    (FULL_DC + CHROMA_AC + [((0,), 1, 63, 0, 0), ((0,), 5, 9, 0, 0)], "scan 4: coefficient 5 of component 0 sent twice"),
    (FULL_DC + FULL_DC + CHROMA_AC + [((0,), 1, 63, 0, 0)], "scan 1: coefficient 0 of component 0 sent twice"),
    (FULL_DC + CHROMA_AC + [((0,), 1, 63, 0, 1)], "block smoothing: coefficient 1 of component 0 known to bit 1"),
    (FULL_DC + CHROMA_AC + [((0,), 1, 8, 0, 0), ((0,), 10, 63, 0, 0)], "block smoothing: coefficient 9 of component 0 never sent"),
    (W.DEFAULT_SCRIPT_YCC[:5], "block smoothing: coefficient 1 of component 0 known to bit 2"),
])
def test_valid_scripts_left_to_pil_say_why(script, reason):
    f = written(script)
    read_image(io.BytesIO(f))      # PIL decodes them
    assert preprocess.inspect_jpeg_progressive(f) == (37, 53, False, reason)
    assert not preprocess.progressive_gpu_decodable(f)


@pytest.mark.parametrize("script", [
    FULL_DC + CHROMA_AC + [((0,), 1, 9, 0, 0)],                                                # 10..63 never sent
    FULL_DC + CHROMA_AC + [((0,), 1, 9, 0, 0), ((0,), 10, 63, 0, 2), ((0,), 10, 63, 2, 1)],   # 10..63 partly refined
    [((0,), 0, 0, 0, 0)],            # chroma never sent: its tables are not latched, so libjpeg does not smooth at all
])
def test_scripts_without_block_smoothing_are_gpu_decodable(script):
    assert preprocess.inspect_jpeg_progressive(written(script)) == (37, 53, True, "")


def test_dc_only_script_is_block_smoothed():
    f = written([((0, 1, 2), 0, 0, 0, 1), ((0, 1, 2), 0, 0, 1, 0)])
    assert preprocess.inspect_jpeg_progressive(f) == (37, 53, False, "block smoothing: coefficient 1 of component 0 never sent")


def test_writer_complete_scripts_equal_decode_coefs():
    """PIL's decode of the writer's files is the exact back end of the coefficients, for complete scripts in every layout,
    with restart intervals and both kinds of Huffman tables."""
    img = photo(37, 53, 4)
    for layout in ("420", "444", "422", "440", "411", "gray"):
        coefs, samp = coefs_of(img, layout)
        script = W.DEFAULT_SCRIPT_GREY if layout == "gray" else W.DEFAULT_SCRIPT_YCC
        qt = [Q[0]] + [Q[1]] * (len(coefs) - 1)
        ref = J.decode_coefs(coefs, qt, 37, 53, samp)
        for restart, huff in ((0, "optimal"), (1, "flat"), (5, "optimal")):
            f = W.write_progressive(coefs, {0: Q[0], 1: Q[1]}, height=37, width=53, sampling=samp, script=script, restart=restart,
                                    huffman=huff)
            np.testing.assert_array_equal(read_image(io.BytesIO(f)), ref, err_msg=f"{layout} {restart} {huff}")
            assert preprocess.inspect_jpeg_progressive(f)[2]


def test_writer_correction_bit_buffer_and_long_eob_runs():
    """Flat blocks with rare large coefficients: AC refinements buffer many correction bits behind EOB runs (forced out past
    jcphuff.c's limit), and runs cross thousands of blocks; restart intervals end them."""
    rng = np.random.default_rng(6)
    blocks = np.zeros((40, 60, 8, 8), np.int64)
    pick = rng.random((40, 60)) < 0.3
    blocks[pick, 0, 1] = rng.integers(-200, 200, int(pick.sum()))
    blocks[..., 0, 0] = rng.integers(-50, 50, (40, 60))
    q = np.full(64, 4, np.int64)
    script = [((0,), 0, 0, 0, 3), ((0,), 1, 63, 0, 4)] + [((0,), 1, 63, a + 1, a) for a in (3, 2, 1, 0)] + \
             [((0,), 0, 0, a + 1, a) for a in (2, 1, 0)]
    ref = J.decode_coefs([blocks], [q], 320, 480, [(1, 1)])
    for restart in (0, 13):
        f = W.write_progressive([blocks], {0: q}, height=320, width=480, sampling=[(1, 1)], script=script, restart=restart)
        np.testing.assert_array_equal(read_image(io.BytesIO(f)), ref)
        assert preprocess.inspect_jpeg_progressive(f)[2]


def test_block_smoothing_rule_follows_libjpeg():
    """jdcoefct.c smoothing_ok, as the installed libjpeg-turbo applies it: a luma coefficient in 1..9 left at Al = 1 makes PIL's
    pixels differ from the exact decode of the known bits (it smooths), one in 10..63 does not."""
    img = photo(64, 96, 7)
    coefs, samp = coefs_of(img, "420")
    qt = [Q[0], Q[1], Q[1]]
    for script, smooths in ((FULL_DC + CHROMA_AC + [((0,), 1, 63, 0, 1)], True),
                            (FULL_DC + CHROMA_AC + [((0,), 1, 9, 0, 0), ((0,), 10, 63, 0, 1)], False),
                            (FULL_DC + CHROMA_AC + [((0,), 1, 9, 0, 0)], False)):
        f = W.write_progressive(coefs, {0: Q[0], 1: Q[1]}, height=64, width=96, sampling=samp, script=script)
        known = J.decode_coefs(W.known_coefs(coefs, script, 3), qt, 64, 96, samp)
        assert np.array_equal(read_image(io.BytesIO(f)), known) != smooths
        assert preprocess.inspect_jpeg_progressive(f)[2] != smooths


def test_blob_sizes():
    """Header 368 bytes, 528 per image, 96 per scan, 32 per (scan, restart interval), 1424 per Huffman table (one per
    component of a DC first scan, one per AC scan, none for a DC refinement)."""
    f = pil_progressive(photo(37, 53, 1))                 # 10 scans: 11 tables; 4:2:0, 3x4 MCUs
    g = pil_progressive(photo(37, 53, 1), restart_marker_blocks=1)
    one = lambda files: preprocess._progressive_plan([np.frombuffer(x, np.uint8) for x in files], np.zeros(len(files), np.int64),
                                                      np.zeros(len(files), np.int64), None)
    assert one([f]) == 368 + 528 + 10 * 96 + 10 * 32 + 11 * 1424
    segs = 2 * 12 + 4 * 35 + 4 * 12      # a restart every MCU: 2 DC scans of 12 MCUs, 4 luma AC of 7 x 5, 4 chroma AC of 4 x 3
    assert one([g]) == 368 + 528 + 10 * 96 + segs * 32 + 11 * 1424
    assert one([f, g, f]) == 368 + 3 * 528 + 30 * 96 + (20 + segs) * 32 + 33 * 1424


def test_batch_layout_routes_progressive_files_behind_the_pngs():
    from PIL import Image
    img = photo(37, 53, 1)
    prog = pil_progressive(img)
    base = io.BytesIO()
    Image.fromarray(img).save(base, "JPEG")
    png = io.BytesIO()
    Image.fromarray(img).save(png, "PNG")
    files = [prog, base.getvalue(), png.getvalue(), img]
    off = preprocess.BatchLayout(files, (224, 320))
    assert off.progressive == [] and off.progressive_plan is None and off.arrays[0] is not None
    on = preprocess.BatchLayout(files, (224, 320), gpu_png=True, gpu_progressive=True)
    assert [i for i, _ in on.progressive] == [0] and [i for i, _ in on.jpeg] == [1] and [i for i, _ in on.png] == [2]
    assert on.arrays[0] is None and on.arrays[3] is not None
    assert on.progressive_plan[0][0] >= on.png_plan[3] and on.progressive_plan[0][0] % 16 == 0
    assert on.staged_end == on.progressive_plan[3]
    only = preprocess.BatchLayout([prog, img], (224, 320), gpu_progressive=True)
    assert only.jpeg_plan is None and only.png_plan is None and only.progressive_plan[0][0] == only.nbytes + (-only.nbytes) % 16


def test_serve_flag():
    import argparse
    import serve
    ap = argparse.ArgumentParser()
    serve.add_model_args(ap)
    assert ap.parse_args(["ck"]).gpu_progressive is False
    assert ap.parse_args(["ck", "--gpu_progressive"]).gpu_progressive is True
