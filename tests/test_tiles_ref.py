"""Tile windows (tiles.tile_windows against oracle/tiles_ref.py and against their defining properties), the merge oracle on
hand-made cases, and BatchLayout with tiling.  No GPU."""
import math

import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess, tiles
from oracle import tiles_ref

LENGTHS = [1, 2, 3, 4, 5, 7, 16, 33, 100, 224, 320, 375, 500, 719, 720, 1280, 4001]
COUNTS = [1, 2, 3, 4, 5, 8]
OVERLAPS = [0, 0.0, 0.1, 0.2, 0.25, 1 / 3, 0.5, 0.75, 0.9, 0.999]
GRID = [(L, k, f) for L in LENGTHS for k in COUNTS for f in OVERLAPS if L >= k]


def test_axis_tiles_properties():
    for L, k, f in GRID:
        t_all = tiles_ref.axis_tiles(L, k, f)
        starts, sizes = [a for a, _ in t_all], [t for _, t in t_all]
        t = sizes[0]
        assert len(t_all) == k and all(s == t for s in sizes), (L, k, f)
        assert 1 <= t <= L and starts[0] == 0 and starts[-1] + t == L, (L, k, f)
        assert all(0 <= a and a + t <= L for a in starts) and starts == sorted(starts), (L, k, f)
        covered = np.zeros(L, bool)
        for a in starts:
            covered[a:a + t] = True
        assert covered.all(), (L, k, f)
        if k == 1:
            assert t_all == [(0, L)]
        if t < L:
            need = math.floor(f * t)
            assert all(a + t - b >= need for a, b in zip(starts, starts[1:])), (L, k, f)


def test_product_windows_equal_the_oracle():
    for L, k, f in GRID:
        assert tiles.axis_tiles(L, k, f) == tiles_ref.axis_tiles(L, k, f), (L, k, f)
    for h, w, rows, cols, f in [(720, 1280, 3, 3, 0.2), (375, 500, 2, 2, 0.2), (224, 320, 1, 4, 0.5), (500, 333, 4, 1, 0.0),
                                (1, 1, 1, 1, 0.2), (3, 4, 3, 4, 0.9), (1080, 1920, 4, 4, 1 / 3)]:
        got = tiles.tile_windows(h, w, rows, cols, f)
        assert got.dtype == np.int32 and got.shape == (1 + rows * cols, 4)
        np.testing.assert_array_equal(got, tiles_ref.tile_windows(h, w, rows, cols, f))
        assert got[0].tolist() == [0, 0, h, w]
        assert got[1].tolist()[:2] == [0, 0] and (got[-1, 0] + got[-1, 2], got[-1, 1] + got[-1, 3]) == (h, w)
    # the documented example: three tiles of a 1280-pixel axis, a fifth shared
    assert tiles.axis_tiles(1280, 3, 0.2) == [(0, 493), (394, 493), (787, 493)]


@pytest.mark.parametrize("args", [(2, 5, 3, 1, 0.2), (5, 2, 1, 3, 0.2), (100, 100, 0, 1, 0.2), (100, 100, 1, 0, 0.2),
                                  (100, 100, 2, 2, 1.0), (100, 100, 2, 2, -0.1), (100, 100, 2, 2, 1.5)])
def test_bad_tilings_raise(args):
    with pytest.raises(ValueError):
        tiles.tile_windows(*args)
    with pytest.raises(ValueError):
        tiles_ref.tile_windows(*args)


def _rec(box, score, index):
    return tuple(np.float32(v) for v in box) + (np.float32(score), index)


def test_merge_duplicate_across_views_keeps_the_lower_view():
    # the same object seen by view 0 at (10, 20, 50, 60) and by view 2, whose origin is (5, 15), at (5, 5, 45, 45)
    out = tiles_ref.merge_class([[_rec((10, 20, 50, 60), 0.9, 7)], [], [_rec((5, 5, 45, 45), 0.9, 3)]], [(0, 0), (0, 0), (5, 15)],
                                nbox=1050, iou_thresh=0.5, max_per_class=30)
    assert [(r[5], float(r[4])) for r in out] == [(7, np.float32(0.9))]
    # a higher score in the tile wins, and carries the tile's view in its index and the shifted box
    out = tiles_ref.merge_class([[_rec((10, 20, 50, 60), 0.8, 7)], [], [_rec((5, 5, 45, 45), 0.9, 3)]], [(0, 0), (0, 0), (5, 15)],
                                1050, 0.5, 30)
    assert len(out) == 1 and out[0][5] == 2 * 1050 + 3 and [float(v) for v in out[0][:4]] == [10, 20, 50, 60]


def test_merge_cap_order_zero_area_and_empty():
    far = [_rec((100 * i, 0, 100 * i + 10, 10), 0.5 + 0.01 * i, i) for i in range(6)]
    out = tiles_ref.merge_class([far[:3], far[3:]], [(0, 0), (0, 0)], 1050, 0.5, max_per_class=4)
    assert [r[5] for r in out] == [1050 + 5, 1050 + 4, 1050 + 3, 2]          # score descending, the cap binds at 4
    # equal scores: view ascending, then index ascending
    tie = tiles_ref.merge_class([[_rec((0, 0, 10, 10), 0.5, 9), _rec((50, 0, 60, 10), 0.5, 4)], [_rec((100, 0, 110, 10), 0.5, 1)]],
                                [(0, 0), (0, 0)], 1050, 0.5, 30)
    assert [r[5] for r in tie] == [4, 9, 1051]
    # a zero-area box has IoU 0 with everything, itself included: both copies survive, and nothing suppresses them
    z = tiles_ref.merge_class([[_rec((5, 5, 5, 30), 0.9, 1)], [_rec((5, 5, 5, 30), 0.8, 1), _rec((0, 0, 40, 40), 0.7, 2)]], [(0, 0), (0, 0)],
                              1050, 0.0, 30)
    assert [r[5] for r in z] == [1, 1051, 1052]
    assert tiles_ref.merge_class([[], [], []], [(0, 0)] * 3, 1050, 0.5, 30) == []
    dets, counts = tiles_ref.merge_views(np.zeros((4, 2, 3), tiles_ref.DET), np.zeros((4, 2), np.int32), np.zeros((4, 2)), 2, 1050, 0.5)
    assert counts.tolist() == [[0, 0], [0, 0]] and dets.shape == (2, 2, 3)


def test_merge_shift_is_one_float32_add():
    y0 = 16777216.0   # 2^24: adding 1.0 in float32 rounds back to 2^24 (half to even)
    out = tiles_ref.merge_class([[], [_rec((1.0, 3.0, 2.5, 0.25), 0.9, 0)]], [(0, 0), (y0, 7)], 10, 0.5, 30)
    assert [float(v) for v in out[0][:4]] == [16777216.0, 10.0, 16777218.0, 7.25]


def test_batch_layout_with_tiling_keeps_the_per_image_fields():
    rng = np.random.default_rng(0)
    images = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in [(375, 500), (100, 37), (720, 1280), (33, 61)]]
    plain = preprocess.BatchLayout(images, (224, 320))
    tiled = preprocess.BatchLayout(images, (224, 320), tiling=(2, 3, 0.25))
    assert len(tiled) == len(plain) == 4 and tiled.views == 7 and plain.views == 1 and plain.windows is None
    np.testing.assert_array_equal(tiled.offsets, plain.offsets)
    np.testing.assert_array_equal(tiled.hw, plain.hw)
    np.testing.assert_array_equal(tiled.matrices, plain.matrices)
    assert tiled.nbytes == plain.nbytes
    assert tiled.windows.shape == (28, 4) and tiled.windows.dtype == np.int32 and tiled.view_matrices.shape == (28, 6)
    for i, im in enumerate(images):
        win = tiles_ref.tile_windows(im.shape[0], im.shape[1], 2, 3, 0.25)
        np.testing.assert_array_equal(tiled.windows[7 * i:7 * i + 7], win)
        for v, (y0, x0, th, tw) in enumerate(win):
            want = preprocess.letterbox_params((th, tw), (224, 320))[2][:2].reshape(-1)
            np.testing.assert_array_equal(tiled.view_matrices[7 * i + v], want)
    with pytest.raises(ValueError, match="tiling 4x1"):
        preprocess.BatchLayout([images[0], np.zeros((3, 50, 3), np.uint8)], (224, 320), tiling=(4, 1, 0.2))
