"""Host packing of a ragged letterbox batch (preprocess.BatchLayout): offsets, alignment, descriptors — CPU only."""
import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess
from oracle import preprocess_ref


def _images():
    rng = np.random.default_rng(0)
    shapes = [(375, 500), (1, 1), (33, 61), (224, 320), (720, 1280), (100, 37)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    imgs.append(imgs[0][:, ::-1])          # a non-contiguous view packs like its copy
    return imgs


@pytest.mark.parametrize("in_hw", [(224, 320), (416, 416)])
def test_layout_offsets_alignment_and_matrices(in_hw):
    imgs = _images()
    lay = preprocess.BatchLayout(imgs, in_hw)
    sizes = [im.shape[0] * im.shape[1] * 3 for im in imgs]
    assert len(lay) == len(imgs) and lay.offsets.dtype == np.int64 and lay.hw.dtype == np.int32
    assert lay.offsets[0] == 0 and all(o % preprocess.ALIGN == 0 for o in lay.offsets)
    for i in range(1, len(imgs)):
        assert lay.offsets[i - 1] + sizes[i - 1] <= lay.offsets[i] < lay.offsets[i - 1] + sizes[i - 1] + preprocess.ALIGN
    assert lay.offsets[-1] + sizes[-1] <= lay.nbytes < lay.offsets[-1] + sizes[-1] + preprocess.ALIGN
    assert lay.hw.tolist() == [list(im.shape[:2]) for im in imgs]
    assert lay.matrices.shape == (len(imgs), 6) and lay.matrices.flags["C_CONTIGUOUS"]
    for m, im in zip(lay.matrices, imgs):
        _, _, inv = preprocess_ref.letterbox_params(im.shape[:2], in_hw)
        assert np.array_equal(m, inv[:2].reshape(-1))           # bit for bit: the host matrix is the reference value
    buf = np.full(lay.nbytes, 0xAB, np.uint8)
    lay.pack(imgs, buf)
    for im, off, n in zip(imgs, lay.offsets, sizes):
        assert np.array_equal(buf[off:off + n].reshape(im.shape), im)


def test_layout_rejects_bad_input():
    good = np.zeros((4, 4, 3), np.uint8)
    for bad in ([], (), None, [good.astype(np.int16)], [good[..., :2]], [good[..., 0]], [np.zeros((0, 4, 3), np.uint8)],
                [good, "x"]):
        with pytest.raises(ValueError):
            preprocess.BatchLayout(bad, (32, 32))
