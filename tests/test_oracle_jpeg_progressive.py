"""oracle/jpeg_progressive_ref.py against PIL on the crafted progressive files of tests/progressive_streams.py and against
the coefficients tests/progressive_writer.py encodes; the host-side plan of csrc/jpeg_progressive.cu: scan levels from the
coefficients a scan may write, and files with restart markers out of sequence left to PIL."""
import ctypes
import io

import numpy as np
import pytest

import progressive_streams as P
import progressive_writer as W
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import JpegProgressiveInfo, lib
from k210_yolo_framework_b200.helper import read_image
from oracle import jpeg_progressive_ref as R
from oracle import jpeg_ref as J

EXACT = dict(P.exact_cases())
RESYNC = dict(P.resync_cases())


@pytest.mark.parametrize("name", list(EXACT))
def test_oracle_equals_pil(name):
    d = EXACT[name]
    r = R.decode(d)
    assert r.restart_issues == [] and r.hit_end == []
    np.testing.assert_array_equal(J.decode_coefs(r.coefs, r.qt, r.height, r.width, r.sampling), read_image(io.BytesIO(d)))


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_cases_take_the_gpu_route(name):
    assert preprocess.inspect_jpeg_progressive(EXACT[name])[2:] == (True, "")


def test_oracle_gives_known_coefs_of_the_writer():
    img = P.photo(37, 53, 4)
    q = [J.quality_table(J.STD_Q_LUMA, 90), J.quality_table(J.STD_Q_CHROMA, 90)]
    scripts = [W.DEFAULT_SCRIPT_YCC, W.DEFAULT_SCRIPT_YCC[:5],
               [((0, 1, 2), 0, 0, 0, 2), ((0,), 1, 9, 0, 3), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0), ((0,), 10, 63, 0, 1),
                ((0,), 1, 9, 3, 2), ((0,), 1, 9, 2, 1), ((0,), 1, 9, 1, 0), ((0, 1, 2), 0, 0, 2, 1), ((0,), 10, 63, 1, 0)]]
    for layout in ("420", "444", "gray"):
        coefs, samp = J.pixels_to_coefs(img, layout, q)
        for si, script in enumerate(scripts):
            if layout == "gray":
                script = [(tuple(c for c in comps if c == 0), *rest) for comps, *rest in script if 0 in comps]
            for restart, huff in ((0, "optimal"), (5, "flat")):
                f = W.write_progressive(coefs, {0: q[0], 1: q[1]}, height=37, width=53, sampling=samp, script=script, restart=restart,
                                        huffman=huff)
                r = R.decode(f)
                assert r.restart_issues == [] and r.hit_end == []
                hmax, vmax = max(h for h, _ in samp), max(v for _, v in samp)
                for c, (got, want) in enumerate(zip(r.coefs, W.known_coefs(coefs, script, len(coefs)))):
                    # the blocks a component's own scans cover (MCU padding past them gets DC only)
                    dh, dw = -(-37 * samp[c][1] // vmax), -(-53 * samp[c][0] // hmax)
                    rows, cols = -(-dh // 8), -(-dw // 8)
                    np.testing.assert_array_equal(got[:rows, :cols].astype(np.int64), want[:rows, :cols],
                                                  err_msg=f"{layout} script {si} {restart} comp {c}")


@pytest.mark.parametrize("name", list(RESYNC))
def test_restart_markers_out_of_sequence_are_reported_and_left_to_pil(name):
    d = RESYNC[name]
    read_image(io.BytesIO(d))                       # PIL decodes them, resynchronising
    assert R.decode(d).restart_issues
    h, w, ok, why = preprocess.inspect_jpeg_progressive(d)
    assert not ok and ("RST" in why or "restart markers" in why), why
    assert not preprocess.progressive_gpu_decodable(d)


def test_in_sequence_files_have_no_restart_issues():
    img = P.photo(32, 64, 0)
    for kw in ({"restart_marker_blocks": 1}, {"restart_marker_rows": 1}, {}):
        d = P.pil_file(img, progressive=True, **kw)
        assert R.decode(d).restart_issues == []
        np.testing.assert_array_equal(R.decode_pixels(d), read_image(io.BytesIO(d)))


def scan_levels(data):
    """The level of each scan in the plan blob of one file."""
    buf = np.frombuffer(data, np.uint8)
    n = preprocess._progressive_plan([buf], np.zeros(1, np.int64), np.zeros(1, np.int64), None)
    blob = np.zeros(n + 16, np.uint8)
    at = (-blob.ctypes.data) % 16
    blob = blob[at:at + n]
    preprocess._progressive_plan([buf], np.zeros(1, np.int64), np.zeros(1, np.int64), blob)
    hdr = blob[:128].view(np.int32)
    nscan, nseg = int(hdr[2]), int(hdr[3])
    seg_off = int(blob[56:64].view(np.int64)[0])
    segs = blob[seg_off:seg_off + 32 * nseg].view(np.int32).reshape(nseg, 8)   # begin, end (int64), scan, first_mcu, mcus, level
    levels = {}
    for s in segs:
        levels.setdefault(int(s[4]), set()).add(int(s[7]))
    assert all(len(v) == 1 for v in levels.values())
    return [levels[k].pop() for k in range(nscan)]


def info(data):
    buf = np.frombuffer(data, np.uint8)
    out = JpegProgressiveInfo()
    assert lib.k2y_jpeg_progressive_inspect(buf.ctypes.data, buf.size, ctypes.byref(out)) == 0
    return out


def test_levels_follow_the_coefficients_a_scan_may_write():
    # libjpeg's default scripts: Y 6..63 first follows Y 1..5 first, which may write up to zig-zag 20
    f = P.pil_file(P.photo(37, 53, 2), progressive=True)
    assert scan_levels(f) == [0, 0, 0, 0, 1, 2, 1, 1, 1, 3] and info(f).levels == 4
    g = P.pil_file(P.photo(37, 53, 2)[..., 0], progressive=True)
    assert scan_levels(g) == [0, 0, 1, 2, 1, 3]
    # DC, Y 1..5 first, its refinement (may write zz6), Y 6..63 first: the last after the refinement
    assert scan_levels(EXACT["refine-stray-then-owner"]) == [0, 0, 1, 2]
    # DC, Y 6..63 first, Y 1..5 first (may write zz1..20): the stray after the owner
    assert scan_levels(EXACT["first-stray-after-owner"]) == [0, 0, 1]
    # a stray into a band a later scan refines: the refinement after the stray
    assert scan_levels(EXACT["stray-then-refined"]) == [0, 0, 1, 2]
    # bands that cannot reach each other stay concurrent: 1..5 may write to 20, 21..63 is apart; 6..20 follows both
    assert scan_levels(EXACT["dht-redefined-one-level"]) == [0, 0, 0, 1]
