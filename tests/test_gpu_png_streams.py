"""GPU PNG inflate (csrc/png.cu) against oracle/inflate_ref.py on the streams of tests/png_streams.py: every file gives the
pixels PIL gives with a zero error word, or a non-zero one where PIL refuses, and status words [1..3] (chunks, confirmed
chunks, the longest chunk's output or the serial decoder's bytes) equal ``chunk_status``.  test_oracle_inflate.py checks the
oracle against PIL itself on the same files."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import inflate_ref as I
import png_streams as S
from k210_yolo_framework_b200 import preprocess


def check(cases):
    files = [f for _, f in cases]
    got, status = preprocess.decode_png_batch(files, with_status=True)
    for i, (name, f) in enumerate(cases):
        exp = I.pixels_as_pil(f)
        if isinstance(exp, I.Refused):
            assert status[i, 0] != 0, (name, status[i])
        else:
            assert status[i, 0] == 0, (name, status[i])
            np.testing.assert_array_equal(got[i].cpu().numpy(), exp, err_msg=name)
        (w, h, c, d, _), _, idat = I.png_parts(f)
        want = I.chunk_status(b"".join(idat), h * (1 + I.row_bytes(w, c, d)))
        assert list(status[i, 1:]) == want, (name, list(status[i]), want)
    return status


def test_every_zlib_error_rule_in_three_places():
    check([(f"{rule} / {place}", f) for rule, place, f in S.error_rule_cases()])


def test_where_the_image_ends():
    check(S.image_end_cases())


def test_multi_chunk_streams_in_one_batch():
    st = check(S.multi_chunk_cases())
    assert len(set(st[:, 1].tolist())) >= 3        # images of different chunk counts share the batch
