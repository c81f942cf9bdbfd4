"""oracle/jpeg_ref.py against PIL on the CPU: every writer variant decodes in PIL to exactly the numpy back end's pixels, and
the back end's SIMD islow IDCT equals PIL's over more than 10^5 random extreme blocks (8-bit tables up to 255, 16-bit tables
up to 65535, coefficients up to +-32767), with libjpeg-turbo's default SIMD dispatch and with SSE2 forced, while its C path
(jidctint.c, what the GPU IDCT used to restate) gives other pixels on most of those blocks."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest

from jpeg_cases import extreme_cases, size_cases, sync_cases, write, writer_cases
from k210_yolo_framework_b200.helper import read_image
from oracle import jpeg_ref as J

GROUPS = {"writer": writer_cases, "sizes": size_cases, "extreme": extreme_cases, "sync": sync_cases}


def test_standard_tables_are_the_ones_pil_writes():
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.zeros((16, 16, 3), np.uint8)).save(b, "JPEG")
    d = b.getvalue()
    i = d.index(b"\xff\xc4")
    got = {}
    while d[i:i + 2] == b"\xff\xc4":
        ln = int.from_bytes(d[i + 2:i + 4], "big")
        s = d[i + 4:i + 2 + ln]
        k = 0
        while k < len(s):
            bits = list(s[k + 1:k + 17])
            got[(s[k] >> 4, s[k] & 15)] = (bits, list(s[k + 17:k + 17 + sum(bits)]))
            k += 17 + sum(bits)
        i += 2 + ln
    assert got == {(0, 0): J.STD_DC_LUMA, (1, 0): J.STD_AC_LUMA, (0, 1): J.STD_DC_CHROMA, (1, 1): J.STD_AC_CHROMA}


@pytest.mark.parametrize("group", list(GROUPS))
def test_written_files_decode_in_pil_to_the_back_end(group):
    for name, w in GROUPS[group]():
        ref = J.decode_coefs(w.coefs, w.qt, w.height, w.width, w.sampling)
        got = read_image(io.BytesIO(w.data))
        assert got.shape == ref.shape, name
        assert np.array_equal(got, ref), (name, int((got != ref).sum()))


def test_sync_cases_put_segment_ends_on_subsequence_boundaries():
    """The segment lengths the sync cases claim, from the writer's per-segment bit counts."""
    c = dict(sync_cases())
    padded = sorted({-(-b // 8) * 8 for b in c["sync-512k"].seg_bits})
    assert padded == [504, 512, 520, 1016, 1024, 1032, 1528, 1536, 1544]
    assert [-(-b // 8) * 8 for b in c["sync-window"].seg_bits] == [256 * 512 - 8, 256 * 512, 256 * 512 + 8, 2 * 256 * 512]
    assert set(c["sync-one-byte-segments"].seg_bits) >= {2}


def test_scan_out_of_frame_order_is_refused():
    """T.81 B.2.3: libjpeg-turbo refuses a scan that lists its components out of frame order; so does the marker walker
    (the file is malformed for inspect_jpeg and never routed to the GPU)."""
    from k210_yolo_framework_b200 import K2YError, preprocess
    for order in ([0, 2, 1], [1, 0, 2], [2, 1, 0]):
        w = write("444", seed=13, scan_order=order, tq=[0, 0, 0], hsel=[(0, 0)] * 3)   # same tables: only the order is wrong
        with pytest.raises(OSError):
            read_image(io.BytesIO(w.data))
        with pytest.raises(K2YError, match="out of frame order"):
            preprocess.inspect_jpeg(w.data)
        assert not preprocess.gpu_decodable(w.data)
    w = write("444", seed=13, ids=[9, 5, 1], tq=[0, 0, 0], hsel=[(0, 0)] * 3)   # descending ids in frame order are fine
    assert preprocess.inspect_jpeg(w.data)[2]


_DECODE = """
import io, sys
import numpy as np
from PIL import Image
files = np.load(sys.argv[1])
np.savez(sys.argv[2], **{k: np.asarray(Image.open(io.BytesIO(files[k].tobytes())).convert("L")) for k in files.files})
"""


@pytest.fixture(scope="module")
def extreme_files(tmp_path_factory):
    """16 grey files of 8000 blocks (128000 in all): DC-only and full extreme blocks, 8- and 16-bit tables (random per
    entry, or one value for the whole table), and the back end's pixels for each."""
    rng = np.random.default_rng(1)
    files, refs = {}, {}
    for i in range(16):
        wide = i % 4 >= 2
        q = rng.integers(1, 65536 if wide else 256, 64)
        if i % 8 < 2:
            q[:] = rng.integers(1, 65536 if wide else 256)
        w = J.grey_file(J.extreme_blocks(rng, 8000, "dc" if i % 2 == 0 else "full"), q, 1000, huffman="optimal")
        files[f"f{i}"] = np.frombuffer(w.data, np.uint8)
        refs[f"f{i}"] = J.decode_coefs(w.coefs, w.qt, w.height, w.width, w.sampling)[..., 0]
    d = tmp_path_factory.mktemp("jpeg_extreme")
    np.savez(d / "files.npz", **files)
    return d, refs


def _pil_in_subprocess(d, env):
    e = {k: v for k, v in os.environ.items() if not k.startswith("JSIMD_")}
    e.update(env)
    subprocess.run([sys.executable, "-c", _DECODE, str(d / "files.npz"), str(d / "out.npz")], env=e, check=True)
    return np.load(d / "out.npz")


def _blocks(img):
    return img.reshape(img.shape[0] // 8, 8, img.shape[1] // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


@pytest.mark.parametrize("env", [{}, {"JSIMD_FORCESSE2": "1"}], ids=["default", "sse2"])
def test_simd_idct_equals_pil_on_extreme_blocks(extreme_files, env):
    d, refs = extreme_files
    got = _pil_in_subprocess(d, env)
    for k, ref in refs.items():
        bad = np.any(_blocks(got[k]) != _blocks(ref), axis=(1, 2))
        assert not bad.any(), (k, int(bad.sum()))


def test_c_path_differs_on_extreme_blocks(extreme_files):
    """libjpeg-turbo's C IDCT (jidctint.c) differs from the SIMD one on these blocks: restating it is not PIL's contract."""
    d, refs = extreme_files
    got = _pil_in_subprocess(d, {"JSIMD_FORCENONE": "1"})
    for k, ref in refs.items():
        bad = np.any(_blocks(got[k]) != _blocks(ref), axis=(1, 2))
        assert bad.mean() > 0.5, (k, float(bad.mean()))
