"""GPU baseline-JPEG decode (csrc/jpeg.cu) on bitstreams libjpeg-turbo's compressor never writes, from oracle/jpeg_ref.py's
writer: every writer knob in each layout, odd sizes, restart segments and codewords on the Huffman kernel's 512-bit
subsequence and 256-subsequence window boundaries, out-of-range coefficients, and single-byte damage that still decodes
cleanly.  Each file must be GPU-decodable, decode with status 0, and give exactly PIL's pixels and the numpy back end's on
the written coefficients; each case runs alone (a failure names it) and all run once more in one batch."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from jpeg_cases import extreme_cases, photo, size_cases, sync_cases, writer_cases
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200.helper import read_image
from oracle import jpeg_ref as J

_CACHE = {}


def _cases():
    if not _CACHE:
        for name, w in writer_cases() + size_cases() + extreme_cases() + sync_cases():
            _CACHE[name] = w
    return _CACHE


NAMES = list(_cases())


def pil(data):
    return read_image(io.BytesIO(data))


def check(names):
    ws = [_cases()[n] for n in names]
    files = [w.data for w in ws]
    for n, f in zip(names, files):
        assert preprocess.gpu_decodable(f), n
    got, status = preprocess.decode_jpeg_batch(files, with_status=True)
    torch.cuda.synchronize()
    assert (status[:, 0] == 0).all(), [(n, int(s)) for n, s in zip(names, status[:, 0]) if s]
    for n, g, w in zip(names, got, ws):
        g = g.cpu().numpy()
        ref = J.decode_coefs(w.coefs, w.qt, w.height, w.width, w.sampling)
        p = pil(w.data)
        assert np.array_equal(p, ref), f"{n}: PIL and the back end differ"
        assert g.shape == ref.shape, (n, g.shape, ref.shape)
        if not np.array_equal(g, ref):
            bad = np.argwhere(g != ref)
            raise AssertionError(f"{n}: {len(bad)} bytes differ, first at {bad[0].tolist()}: {g[tuple(bad[0])]} vs {ref[tuple(bad[0])]}")


@pytest.mark.parametrize("name", NAMES)
def test_case_alone(name):
    check([name])


def test_all_cases_in_one_batch():
    check(NAMES)


def _damaged(n_tries=200):
    """Single-byte changes to the entropy data of a photo file without restart markers (no marker created or removed)."""
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(photo(120, 160, 5)).save(b, "JPEG", quality=92)
    src = b.getvalue()
    sos = src.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(src[sos + 2:sos + 4], "big")
    rng = np.random.default_rng(7)
    out = []
    for _ in range(n_tries):
        while True:
            i = int(rng.integers(start + 1, len(src) - 2))
            if src[i] != 0xFF and src[i - 1] != 0xFF:
                break
        v = int(rng.integers(0, 255))
        if v == src[i]:
            v ^= 1
        d = bytearray(src)
        d[i] = v
        out.append(bytes(d))
    return out


def test_damaged_complete_files_that_decode_cleanly_match_pil():
    """A damaged file whose entropy data still decodes without a bad code and with the right block count: the GPU calls it
    clean, so its pixels must be PIL's, whatever values its coefficients walked to."""
    files = _damaged()
    assert all(preprocess.gpu_decodable(f) for f in files)
    got, status = preprocess.decode_jpeg_batch(files, with_status=True)
    torch.cuda.synchronize()
    clean = [i for i in range(len(files)) if status[i, 0] == 0]
    assert len(clean) >= 3, len(clean)
    for i in clean:
        np.testing.assert_array_equal(got[i].cpu().numpy(), pil(files[i]), err_msg=f"variant {i}")


def test_files_through_letterbox_and_submit_images(golden_weights, voc_anchors):
    from oracle import preprocess_ref
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    c = _cases()
    damaged = _damaged(40)
    _, status = preprocess.decode_jpeg_batch(damaged, with_status=True)
    files = [c[n].data for n in ("extreme-colour-420", "extreme-dc-walk", "ids-desc-411", "sync-straddle", "dri3-440",
                                 "segments-420", "size-23x19-420")]
    files += [damaged[i] for i in range(len(damaged)) if status[i, 0] == 0][:1]
    hw = (224, 320)
    out = preprocess.letterbox_batch_device(files, hw).cpu().numpy()
    for i, f in enumerate(files):
        np.testing.assert_array_equal(out[i], preprocess_ref.letterbox(pil(f), hw), err_msg=f"file {i}")
    pipe = DetectionPipeline("yolo_mobilev1", hw, voc_anchors, 20, 0.75, 4, obj_thresh=0.7, iou_thresh=0.5)
    pipe.engine.set_weights(golden_weights)
    batches = [files[i:i + 4] for i in range(0, len(files), 4)]
    got = [DetectionPipeline.records(*pipe.collect(pipe.submit_images(b))) for b in batches]
    ref = [DetectionPipeline.records(*pipe.collect(pipe.submit_images([pil(f) for f in b]))) for b in batches]
    assert got == ref
