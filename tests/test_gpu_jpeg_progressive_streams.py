"""GPU JPEG decoders on bitstreams libjpeg-turbo's compressor never writes (tests/progressive_streams.py).  Progressive:
runs past a scan's band and every other crafted stream decode with status 0 to exactly PIL's pixels and the oracle's, each
case alone and all in one batch.  Restart markers out of sequence, in progressive files and in baseline ones: PIL's pixels
or a refusal naming the image, never status 0 with other pixels; also through letterbox and submit_images."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import progressive_streams as P
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200._lib import K2YError
from k210_yolo_framework_b200.helper import read_image
from k210_yolo_framework_b200.pipeline import DetectionPipeline
from oracle import jpeg_progressive_ref as R
from test_gpu_jpeg import _pipeline

EXACT = dict(P.exact_cases())
RESYNC = dict(P.resync_cases())
BASE = dict(P.baseline_resync_cases())


def pil(data):
    return read_image(io.BytesIO(data))


def check_exact(names):
    files = [EXACT[n] for n in names]
    for n, f in zip(names, files):
        assert preprocess.progressive_gpu_decodable(f), (n, preprocess.inspect_jpeg_progressive(f))
    got, status = preprocess.decode_progressive_jpeg_batch(files, with_status=True)
    torch.cuda.synchronize()
    assert (status[:, 0] == 0).all(), [(n, int(s)) for n, s in zip(names, status[:, 0]) if s]
    for n, g, f in zip(names, got, files):
        g, ref = g.cpu().numpy(), pil(f)
        np.testing.assert_array_equal(R.decode_pixels(f), ref, err_msg=f"{n}: the oracle and PIL differ")
        if not np.array_equal(g, ref):
            bad = np.argwhere(g != ref)
            raise AssertionError(f"{n}: {len(bad)} bytes differ, first at {bad[0].tolist()}: {g[tuple(bad[0])]} vs {ref[tuple(bad[0])]}")


@pytest.mark.parametrize("name", list(EXACT))
def test_case_alone(name):
    check_exact([name])


def test_all_cases_in_one_batch():
    check_exact(list(EXACT))


def test_all_cases_twice_in_one_batch_reversed():
    names = list(EXACT)
    check_exact(names + names[::-1])


@pytest.mark.parametrize("name", list(RESYNC))
def test_progressive_restart_markers_out_of_sequence_stay_with_pil(name):
    d = RESYNC[name]
    assert not preprocess.progressive_gpu_decodable(d)
    from oracle import preprocess_ref
    out = preprocess.letterbox_batch_device([d, EXACT["refine-stray-then-owner"]], (224, 320), gpu_progressive=True).cpu().numpy()
    np.testing.assert_array_equal(out[0], preprocess_ref.letterbox(pil(d), (224, 320)))


@pytest.mark.parametrize("name", list(BASE))
def test_baseline_restart_markers_out_of_sequence_give_pil_or_refuse(name):
    d = BASE[name]
    assert preprocess.gpu_decodable(d)
    got, status = preprocess.decode_jpeg_batch([d], with_status=True)
    torch.cuda.synchronize()
    same = np.array_equal(got[0].cpu().numpy(), pil(d))
    if name == "base-extra-trailing":
        assert status[0, 0] == 0 and same
    elif name not in ("base-rst-missing-last", "base-rst-without-dri"):
        assert status[0, 0] & 4, status[0]        # a marker between intervals out of sequence
    else:
        assert status[0, 0] != 0 or same, status[0]


def test_baseline_out_of_sequence_names_the_image():
    good = BASE["base-extra-trailing"]
    with pytest.raises(K2YError, match="image 1: restart marker out of sequence"):
        preprocess.decode_jpeg_batch([good, BASE["base-rst+1"], good])
    with pytest.raises(K2YError, match="image 0: restart marker out of sequence"):
        preprocess.letterbox_batch_device([BASE["base-rst-1"], good], (224, 320))


@pytest.mark.parametrize("lanes", [None, 2])
def test_misnumbered_restart_markers_through_submit_images(golden_weights, voc_anchors, lanes):
    """A progressive file with RST1 for RST0 goes to PIL and gives PIL's records; a baseline one raises naming the image,
    and the batches around it are unaffected."""
    prog_bad, base_bad = RESYNC["prog-rst+1"], BASE["base-rst+1"]
    good = [EXACT["strays-420"], EXACT["refine-stray-restart1"], BASE["base-extra-trailing"]]
    on = _pipeline(golden_weights, voc_anchors, 4, lanes)
    on.enable_progressive_jpeg_decode()
    ref = _pipeline(golden_weights, voc_anchors, 4, lanes)
    batch = [prog_bad] + good
    got = DetectionPipeline.records(*on.collect(on.submit_images(batch)))
    assert got == DetectionPipeline.records(*ref.collect(ref.submit_images([pil(f) for f in batch])))
    t = on.submit_images([good[0], base_bad])
    t2 = on.submit_images(good)
    with pytest.raises(K2YError, match="image 1: restart marker out of sequence"):
        on.collect(t)
    assert DetectionPipeline.records(*on.collect(t2)) == DetectionPipeline.records(*ref.collect(ref.submit_images([pil(f) for f in good])))
