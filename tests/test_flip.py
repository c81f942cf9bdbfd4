"""Test-time flip without a GPU: the oracle's un-mirror of mirrored views (oracle/flip_ref.py) on hand-made records,
the view planning of tiles.plan_views, BatchLayout with flip, the --flip flag and the pipeline's refusals."""
import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess, tiles
from oracle import flip_ref
from oracle import tiles_merge_ref as ref

F = np.float32
NBOX = 1050


def _bits(v):
    return int(np.array(v, F).view(np.uint32))


def _merge(views, origins, sides, hw, mirrored, thr=0.5, K=30, **kw):
    return flip_ref.merge_class(views, origins, sides, hw, NBOX, thr, K, mirrored=mirrored, **kw)


# ---- the oracle's un-mirror -----------------------------------------------------------------------------------------------
def test_mirrored_record_swaps_and_reflects_the_x_fields():
    rec = (5., 10., 40., 30., 0.9, 7)                    # in the mirrored 100-wide window: x 10 .. 30
    out = _merge([[rec]], [(3, 20)], [0], [(50, 100)], [True])
    assert out == [(F(8), F(20 + 70), F(43), F(20 + 90), F(0.9), 7)]
    plain = _merge([[rec]], [(3, 20)], [0], [(50, 100)], None)
    assert plain[0][:4] == (F(8), F(30), F(43), F(50))


def test_tw_minus_tw_is_plus_zero_and_minus_zero_reflects_to_tw():
    rec = (0., -0.0, 10., 64., 0.9, 1)                   # xmax_m = tw, xmin_m = -0.0
    out = _merge([[rec]], [(0, 0)], [0], [(10, 64)], [True])
    y0, x0, y1, x1 = out[0][:4]
    assert _bits(x0) == 0 and x1 == F(64)               # fl(64 - 64) = +0.0, + 0 stays +0.0
    out = _merge([[rec]], [(-0.0, -0.0)], [0], [(10, 64)], [True])
    assert _bits(out[0][1]) == 0                        # +0.0 + -0.0 = +0.0


def test_nan_fields_come_back_as_the_canonical_nan():
    nan_payload = np.array(0xffc00123, np.uint32).view(F)    # negative, with a payload
    rec = (1., nan_payload, 2., 5., 0.9, 0)
    out = _merge([[rec]], [(0, 7)], [0], [(10, 20)], [True])
    assert _bits(out[0][3]) == 0x7fffffff               # xmax = tw - xmin_m + x0: NaN
    assert out[0][1] == F(20 - 5 + 7)


@pytest.mark.parametrize("border", [0.0, 2.0, 5.0])
@pytest.mark.parametrize("sides", range(16))
def test_side_bits_swap_for_a_mirrored_view(sides, border):
    th, tw = 60, 100
    swapped = flip_ref.swap_sides(sides)
    assert swapped & 5 == sides & 5 and bool(swapped & 2) == bool(sides & 8) and bool(swapped & 8) == bool(sides & 2)
    for rec in [(20., 1., 40., 30., 0.9, 0), (20., 70., 40., 99., 0.9, 1), (1., 40., 59., 60., 0.9, 2), (20., 3., 40., 97., 0.9, 3)]:
        got = len(_merge([[rec]], [(0, 0)], [sides], [(th, tw)], [True], border=border))
        assert got == (0 if ref.border_drops(rec, swapped, th, tw, border) else 1), (rec, sides)
        # the same record upright, in window coordinates, meets the window's own sides
        up = (rec[0], tw - rec[3], rec[2], tw - rec[1]) + rec[4:]
        assert got == len(_merge([[up]], [(0, 0)], [sides], [(th, tw)], [False], border=border))


def _scene(rng, m, th, tw):
    y, x = rng.integers(0, th - 10, m), rng.integers(0, tw - 10, m)
    h, w = rng.integers(1, 60, m), rng.integers(1, 80, m)
    s = rng.choice(F(np.linspace(0.1, 1.0, 7)), m)
    return [(F(y[j]), F(x[j]), F(min(th, y[j] + h[j])), F(min(tw, x[j] + w[j])), F(s[j]), int(j)) for j in range(m)]


@pytest.mark.parametrize("match,merge", [("iou", "suppress"), ("ios", "union")])
def test_a_scene_mirrored_about_the_window_centre_merges_as_upright(match, merge):
    """Integer boxes reflect exactly, so a tiling whose views are all mirrored gives the boxes of the upright tiling."""
    rng = np.random.default_rng(5)
    win = tiles.tile_windows(300, 400, 2, 2, 0.2)
    sides = tiles.view_sides(win, 300, 400).tolist()
    hw = [tuple(w[2:]) for w in win.tolist()]
    origins = [tuple(w[:2]) for w in win.tolist()]
    for trial in range(10):
        up = [_scene(rng, int(rng.integers(0, 12)), th, tw) for th, tw in hw]
        mir = [[(r[0], F(tw - r[3]), r[2], F(tw - r[1])) + r[4:] for r in recs] for recs, (th, tw) in zip(up, hw)]
        for border in (None, 3.0):
            want = _merge(up, origins, sides, hw, None, match=match, merge=merge, border=border)
            got = _merge(mir, origins, sides, hw, [True] * 5, match=match, merge=merge, border=border)
            assert np.array(got, object).tolist() == np.array(want, object).tolist(), (trial, border)


def test_mirrored_views_are_numbered_after_the_windows():
    """W = 2 windows: view 3 is window 1 mirrored; its record's index is 3 * nbox + index."""
    win = np.array([(0, 0, 100, 200), (0, 50, 100, 150)], np.int32)
    windows, mirror = tiles.mirror_views(win)
    assert windows.tolist() == win.tolist() * 2 and mirror.tolist() == [0, 0, 1, 1]
    rec = (10., 10., 20., 20., 0.9, 4)
    views = [[], [], [], [rec]]
    out = _merge(views, [tuple(w[:2]) for w in windows.tolist()], [0] * 4, [tuple(w[2:]) for w in windows.tolist()], mirror)
    assert out[0][5] == 3 * NBOX + 4 and out[0][1] == F(50 + 150 - 20)


def test_merge_views_block_form_takes_the_flags():
    rng = np.random.default_rng(2)
    N, C, K = 4, 2, 5
    dets = np.zeros((N, C, K), ref.DET)
    counts = rng.integers(0, K + 1, (N, C)).astype(np.int32)
    for g in range(N):
        for c in range(C):
            for k in range(K):
                dets[g, c, k] = (F(k), F(k + 1), F(k + 5), F(k + 9), F(0.9 - 0.1 * k), k)
    origins = np.array([(0, 0), (0, 0), (0, 30), (0, 30)], F)
    hw = np.array([(100, 100), (100, 100), (100, 70), (100, 70)], F)
    mirror = np.array([0, 1, 0, 1], np.int32)
    got, cnt = flip_ref.merge_views(dets, counts, origins, [0, 2, 4], NBOX, 0.5, view_hw=hw, mirrored=mirror)
    for b in range(2):
        for c in range(C):
            lists = [[tuple(dets[g, c, k]) for k in range(counts[g, c])] for g in (2 * b, 2 * b + 1)]
            want = flip_ref.merge_class(lists, origins[2 * b:2 * b + 2], [0, 0], hw[2 * b:2 * b + 2], NBOX, 0.5, K, mirrored=[0, 1])
            assert cnt[b, c] == len(want) and [tuple(r) for r in got[b, c, :len(want)]] == want


@pytest.mark.parametrize("match,merge,border", [("iou", "suppress", None), ("ios", "union", 3.0), ("iou", "union", 0.0)])
def test_no_mirrored_view_is_the_plain_merge(match, merge, border):
    """flip_ref without a mirrored view is tiles_merge_ref's merge, border drop included."""
    rng = np.random.default_rng(9)
    win = tiles.tile_windows(300, 400, 2, 2, 0.2)
    sides = tiles.view_sides(win, 300, 400).tolist()
    hw = [tuple(w[2:]) for w in win.tolist()]
    origins = [tuple(w[:2]) for w in win.tolist()]
    for trial in range(10):
        views = [_scene(rng, int(rng.integers(0, 12)), th, tw) for th, tw in hw]
        want = ref.merge_class(views, origins, sides, hw, NBOX, 0.5, 30, match, merge, border)
        for mirrored in (None, [0] * 5):
            got = _merge(views, origins, sides, hw, mirrored, match=match, merge=merge, border=border)
            assert np.array(got, object).tolist() == np.array(want, object).tolist(), trial


# ---- view planning --------------------------------------------------------------------------------------------------------
def test_plan_views_fixed_grids():
    assert tiles.plan_views(32, 30, 1024, None, True) == (None, 2, 16)
    assert tiles.plan_views(32, 30, 1024, ("grid", 2, 2, 0.2), False) == ((2, 2, 0.2), 5, 6)
    assert tiles.plan_views(32, 30, 1024, ("grid", 2, 2, 0.2), True) == ((2, 2, 0.2), 10, 3)
    assert tiles.plan_views(2, 30, 1024, None, True) == (None, 2, 1)
    with pytest.raises(ValueError):
        tiles.plan_views(1, 30, 1024, None, True)                          # 2 views, batch 1
    assert tiles.plan_views(32, 30, 1024, ("grid", 2, 3, 0.2), True)[1:] == (14, 2)
    with pytest.raises(ValueError):
        tiles.plan_views(64, 100, 1024, ("grid", 2, 3, 0.2), True)          # 14 x 100 > 1024
    assert tiles.plan_views(64, 100, 1024, ("grid", 2, 2, 0.2), False)[1:] == (5, 12)
    with pytest.raises(ValueError):
        tiles.plan_views(64, 600, 1024, None, True)                         # 2 x 600 > 1024


def test_plan_views_fixed_grid_over_the_batch():
    with pytest.raises(ValueError):
        tiles.plan_views(9, 30, 1024, ("grid", 2, 2, 0.2), True)            # 10 views, batch 9
    assert tiles.plan_views(10, 30, 1024, ("grid", 2, 2, 0.2), True)[1:] == (10, 1)


@pytest.mark.parametrize("batch,ipb,K,cap", [(3, 3, 30, 1), (6, 3, 30, 2), (9, 3, 30, 3), (32, 4, 30, 8), (64, 2, 100, 10),
                                            (32, 1, 30, 32), (40, 1, 30, 34)])
def test_plan_views_sized_grids_under_caps(batch, ipb, K, cap):
    size = ("size", (224, 320), 0.2, ipb)
    tiling, V, n = tiles.plan_views(batch, K, 1024, size, False)
    assert (tiling.max_views, V, n) == (cap, cap, ipb)
    if cap // 2 < 1:
        with pytest.raises(ValueError):
            tiles.plan_views(batch, K, 1024, size, True)
        return
    tiling, V, n = tiles.plan_views(batch, K, 1024, size, True)
    assert (tiling.max_views, V, n) == (cap // 2, cap // 2 * 2, ipb)
    for h, w in [(200, 300), (375, 500), (720, 1280), (3000, 4000)]:
        assert 2 * len(tiling.windows(h, w)) <= cap


# ---- BatchLayout ----------------------------------------------------------------------------------------------------------
IMAGES = [np.zeros((200, 300, 3), np.uint8), np.zeros((375, 500, 3), np.uint8), np.zeros((720, 1280, 3), np.uint8)]


def test_layout_with_flip_alone():
    lay = preprocess.BatchLayout(IMAGES, (224, 320), flip=True)
    hw = [im.shape[:2] for im in IMAGES]
    assert lay.views == 2 and lay.n_views == 6 and lay.view_counts.tolist() == [2, 2, 2]
    assert lay.view_offsets.tolist() == [0, 2, 4, 6] and lay.view_mirror.tolist() == [0, 1] * 3
    assert lay.windows.tolist() == [[0, 0, h, w] for h, w in hw for _ in range(2)]
    assert lay.view_sides.tolist() == [0] * 6 and lay.merge_table_at is None
    whole = preprocess.BatchLayout(IMAGES, (224, 320))
    assert np.array_equal(lay.view_matrices, np.repeat(whole.matrices, 2, axis=0))
    t = preprocess.BatchLayout(IMAGES, (224, 320), merge_table=True, flip=True)
    assert t.merge_table.tolist() == [0, 2, 4, 6] + [0] * 6 + [0, 1] * 3
    assert t.merge_table_at % preprocess.ALIGN == 0 and t.staged_end == t.merge_table_at + 4 * (4 + 6 + 6)


def test_layout_with_a_grid_and_flip():
    lay = preprocess.BatchLayout(IMAGES, (224, 320), tiling=(2, 2, 0.2), flip=True)
    assert lay.views == 10 and lay.view_offsets.tolist() == [0, 10, 20, 30]
    for b, (h, w) in enumerate(im.shape[:2] for im in IMAGES):
        win = tiles.tile_windows(h, w, 2, 2, 0.2)
        assert lay.windows[10 * b:10 * b + 10].tolist() == win.tolist() * 2
        assert lay.view_sides[10 * b:10 * b + 10].tolist() == tiles.view_sides(win, h, w).tolist() * 2
        assert lay.view_mirror[10 * b:10 * b + 10].tolist() == [0] * 5 + [1] * 5
    t = preprocess.BatchLayout(IMAGES, (224, 320), tiling=(2, 2, 0.2), merge_table=True, flip=True)
    assert t.merge_table.tolist() == lay.view_offsets.tolist() + lay.view_sides.tolist() + lay.view_mirror.tolist()
    assert t.staged_end == t.merge_table_at + 4 * (4 + 30 + 30)
    plain = preprocess.BatchLayout(IMAGES, (224, 320), tiling=(2, 2, 0.2), merge_table=True)
    assert plain.view_mirror is None and plain.merge_table.tolist() == plain.view_offsets.tolist() + plain.view_sides.tolist()


def test_layout_with_a_sized_tiling_and_flip():
    plan = tiles.SizedTiling((224, 320), 0.2, 5)
    lay = preprocess.BatchLayout(IMAGES, (224, 320), tiling=plan, merge_table=True, flip=True)
    assert lay.views is None and lay.view_counts.tolist() == [2, 10, 10] and lay.view_offsets.tolist() == [0, 2, 12, 22]
    assert lay.windows[:2].tolist() == [[0, 0, 200, 300]] * 2
    assert lay.windows[2:12].tolist() == tiles.tile_windows(375, 500, 2, 2, 0.2).tolist() * 2
    assert lay.view_mirror.tolist() == [0, 1] + ([0] * 5 + [1] * 5) * 2
    assert lay.merge_table.tolist() == lay.view_offsets.tolist() + lay.view_sides.tolist() + lay.view_mirror.tolist()


# ---- the flag and the refusals --------------------------------------------------------------------------------------------
def test_serve_flip_flag():
    import serve
    ap = serve.build_parser()
    assert ap.parse_args(["ck", "imgs"]).flip is False
    assert ap.parse_args(["ck", "imgs", "--flip"]).flip is True
    for extra in (["--tiles", "2", "2"], ["--tile_size", "224", "320", "--tile_images", "4"], ["--tile_match", "ios"],
                  ["--tile_merge", "union"], ["--tile_border", "2"], ["--tile_overlap", "0.3"]):
        ns = ap.parse_args(["ck", "imgs", "--flip"] + extra)
        assert ns.flip is True
        ns2 = ap.parse_args(["ck", "imgs"] + extra + ["--flip"])
        assert vars(ns) == vars(ns2)
    with pytest.raises(SystemExit):
        ap.parse_args(["ck", "imgs", "--flip", "--tile_size", "224", "320"])


class _Gather:
    K = 30


def _bare_pipeline(batch, grid, flip):
    """The view-planning state of a DetectionPipeline after an enable_tiling(grid) / enable_flip that succeeded, without the
    network and the device buffers, which a refused call must not reach."""
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    p = object.__new__(DetectionPipeline)
    p.batch, p.gather = batch, _Gather()
    p._grid, p._merge_options, p._flip = grid, dict(match="iou", merge="suppress", match_thresh=None, border=None), flip
    p._tiling, p._views, p._ipb = (None, 1, batch) if grid is None and not flip else tiles.plan_views(batch, 30, 1024, grid, flip)
    return p


def _state(p):
    return (p.images_per_batch, p._views, p._tiling, p._grid, p._flip, dict(p._merge_options))


@pytest.mark.parametrize("batch,grid,flip,call,kw", [
    (1, None, False, "flip", {}),                                                # 2 views, batch 1
    (9, None, True, "tiling", dict(rows=2, cols=2)),                             # 10 views, batch 9
    (9, ("grid", 2, 2, 0.2), False, "flip", {}),
    (64, ("grid", 5, 6, 0.2), False, "flip", {}),                                # 62 x 30 records > 1024
    (3, ("size", (224, 320), 0.2, 3), False, "flip", {}),                        # max_views 1: no flipped window fits
    (6, None, True, "tiling", dict(tile_size=(224, 320), images_per_batch=6)),   # max_views 1 again, flip first
    (6, None, False, "flip", dict(match="giou")),
    (6, ("grid", 1, 2, 0.2), False, "flip", dict(border=-1.0)),
])
def test_refusals_leave_the_pipeline_as_it_was(batch, grid, flip, call, kw):
    p = _bare_pipeline(batch, grid, flip)
    before = _state(p)
    with pytest.raises(ValueError):
        (p.enable_flip if call == "flip" else p.enable_tiling)(**kw)
    assert _state(p) == before
