"""Grids planned from a tile size (tiles.plan_grid / plan_windows against oracle/tiles_merge_ref.py and their defining
properties), the options of the merge of views on hand-made cases, BatchLayout with a SizedTiling and the serve.py flags.
No GPU."""
import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess, tiles
from oracle import tiles_merge_ref as ref
from oracle import tiles_ref

F = np.float32
NBOX = 1050
LENGTHS = [1, 2, 3, 7, 33, 100, 224, 225, 320, 375, 447, 448, 449, 500, 720, 1280, 3000, 4000]
TILES = [1, 2, 5, 100, 224, 320, 640]
OVERLAPS = [0, 0.0, 0.2, 0.25, 1 / 3, 0.5, 0.9]


def test_axis_count_equals_the_oracle_and_is_minimal():
    for L in LENGTHS:
        for T in TILES:
            if L > 500 and T < 5:
                continue            # the oracle walks k upwards one by one
            for f in OVERLAPS:
                k = tiles.axis_count(L, T, f)
                assert k == ref.axis_count(L, T, f), (L, T, f)
                t = tiles.axis_tiles(L, k, f)[0][1]
                assert 1 <= k <= L
                if L <= T:
                    assert k == 1
                elif t > T:                                   # no k reaches T: every pixel its own tile
                    assert k == L
                else:
                    assert k == 1 or tiles.axis_tiles(L, k - 1, f)[0][1] > T, (L, T, f)


@pytest.mark.parametrize("cap", [1, 2, 3, 5, 8, 10, 17, 34])
def test_plan_grid_equals_the_oracle_and_respects_the_cap(cap):
    for h in [1, 33, 224, 375, 500, 720, 1080, 3000]:
        for w in [1, 61, 320, 333, 640, 1280, 1920, 4000]:
            for tile_hw in [(224, 320), (320, 320), (100, 150), (640, 640)]:
                for f in (0.0, 0.2, 0.5):
                    rows, cols = tiles.plan_grid(h, w, tile_hw, f, cap)
                    assert (rows, cols) == ref.plan_grid(h, w, tile_hw, f, cap), (h, w, tile_hw, f, cap)
                    win = tiles.plan_windows(h, w, tile_hw, f, cap)
                    assert win.tolist() == ref.plan_windows(h, w, tile_hw, f, cap).tolist()
                    assert len(win) == tiles.view_count(rows, cols) <= cap
                    free_r, free_c = tiles.axis_count(h, tile_hw[0], f), tiles.axis_count(w, tile_hw[1], f)
                    assert rows <= free_r and cols <= free_c
                    if (rows, cols) == (free_r, free_c):               # the cap did not bind: tiles fit T unless L stopped it
                        t_h, t_w = win[-1, 2], win[-1, 3]
                        assert t_h <= tile_hw[0] or rows == h and t_h == 1
                        assert t_w <= tile_hw[1] or cols == w and t_w == 1
                    else:                                              # it did: one more tile on either axis breaks it
                        assert tiles.view_count(rows + 1, cols) > cap or rows + 1 > free_r
                        assert tiles.view_count(rows, cols + 1) > cap or cols + 1 > free_c
                    if rows * cols == 1:
                        assert win.tolist() == [[0, 0, h, w]]
                    else:
                        assert win.tolist() == tiles.tile_windows(h, w, rows, cols, f).tolist()


def test_plan_grid_examples():
    assert tiles.plan_grid(375, 500, (224, 320), 0.2, 10) == (2, 2)
    assert tiles.plan_grid(200, 300, (224, 320), 0.2, 10) == (1, 1)
    assert len(tiles.plan_windows(200, 300, (224, 320), 0.2, 10)) == 1          # fits one tile: the whole image only
    assert tiles.plan_grid(3000, 4000, (224, 320), 0.2, 10 ** 6) == (17, 16)
    assert tiles.plan_grid(3000, 4000, (224, 320), 0.2, 34) == (5, 6)           # capped from (17, 16): 31 views
    assert tiles.plan_grid(3000, 4000, (224, 320), 0.2, 2) == (1, 1)            # 1x2 would be 3 views
    assert tiles.plan_grid(720, 1280, (224, 320), 0.0, 5) == (2, 2)            # (4, 4) -> rows first on the tie
    with pytest.raises(ValueError):
        tiles.plan_grid(100, 100, (0, 320), 0.2, 5)
    with pytest.raises(ValueError):
        tiles.plan_grid(100, 100, (224, 320), 0.2, 0)
    with pytest.raises(ValueError):
        tiles.plan_grid(100, 100, (224, 320), 1.0, 5)


def test_view_sides():
    win = tiles.tile_windows(300, 400, 2, 2, 0.2)
    sides = tiles.view_sides(win, 300, 400)
    assert sides.tolist() == [0, 4 | 8, 4 | 2, 1 | 8, 1 | 2]
    assert sides.tolist() == ref.view_sides(win, 300, 400).tolist()
    mid = tiles.tile_windows(300, 400, 3, 3, 0.2)[5]
    assert tiles.view_sides(mid[None], 300, 400).tolist() == [15]


# ---- the merge options -------------------------------------------------------------------------------------------------
def _merge(views, thr=0.5, origins=None, sides=None, hw=None, K=30, **kw):
    V = len(views)
    origins = origins or [(0, 0)] * V
    sides = sides or [0] * V
    hw = hw or [(1000, 1000)] * V
    return ref.merge_class(views, origins, sides, hw, NBOX, thr, K, **kw)


def test_a_fragment_is_folded_by_ios_union_and_kept_by_iou_suppress():
    """A 100 x 100 object; the right tile (origin x 150) sees its left edge cut at x = 150 as a fragment of 100 x 50."""
    whole = (100., 100., 200., 200., 0.9, 7)            # view 0
    frag = (100., 0., 200., 50., 0.8, 3)                # view 1, window x from 150: image x 150 .. 200
    frag2 = (98., 0., 203., 52., 0.85, 4)               # a fragment a little larger than the object on three sides
    views = [[whole], [frag2, frag]]
    origins = [(0, 0), (0, 150)]
    plain = _merge(views, origins=origins)
    assert [r[5] for r in plain] == [7, NBOX + 4]       # IoU 0.478 with the whole box: the larger fragment stays
    folded = _merge(views, origins=origins, match="ios", merge="union")
    assert len(folded) == 1
    y0, x0, y1, x1, s, i = folded[0]
    assert (y0, x0, y1, x1) == (F(98), F(100), F(203), F(202)) and s == F(0.9) and i == 7
    sup = _merge(views, origins=origins, match="ios")
    assert [r[:4] for r in sup] == [(F(100), F(100), F(200), F(200))]


def test_union_uses_the_kept_box_only_not_the_growing_union():
    kept = (0., 0., 10., 10., 0.9, 0)
    a = (0., 8., 10., 18., 0.8, 1)                      # IoS with kept 0.2: no match
    b = (0., 1., 10., 11., 0.7, 2)                      # matches kept
    out = _merge([[kept, a, b]], thr=0.5, match="ios", merge="union")
    assert [r[5] for r in out] == [0, 1]
    assert out[0][:4] == (F(0), F(0), F(10), F(11))     # a was not folded although union(kept, b) reaches it


def test_a_kept_record_that_matched_nothing_is_its_suppress_record():
    rng = np.random.default_rng(1)
    recs = [tuple(F(v) for v in rng.uniform(0, 500, 4)) + (F(rng.uniform(0.1, 1)), int(j)) for j in range(40)]
    for match in ("iou", "ios"):
        sup = _merge([recs[:20], recs[20:]], thr=2.0, match=match)       # nothing exceeds 2: nothing matched
        uni = _merge([recs[:20], recs[20:]], thr=2.0, match=match, merge="union")
        assert np.array(sup, object).tolist() == np.array(uni, object).tolist() and len(sup) == 30


@pytest.mark.parametrize("side,box,dropped", [
    (1, (2., 50., 40., 90.), True), (1, (3., 50., 40., 90.), False), (1, (40., 50., 2.9, 90.), True),
    (2, (50., 2.5, 90., 40.), True), (2, (50., 3., 90., 40.), False),
    (4, (50., 50., 97.5, 90.), True), (4, (50., 50., 97., 90.), False), (4, (98., 50., 50., 90.), True),
    (8, (50., 50., 90., 197.1), True), (8, (50., 50., 90., 197.), False),
    (0, (0., 0., 100., 200.), False), (15, (10., 10., 20., 20.), False), (15, (10., 10., 20., 198.), True)])
def test_border_drop_on_each_side(side, box, dropped):
    """A 100 x 200 window, border 3: a side whose bit is clear (an image edge) never drops."""
    rec = box + (0.9, 5)
    assert ref.border_drops(rec, side, 100, 200, 3.0) == dropped
    out = _merge([[], [rec]], sides=[0, side], hw=[(500, 500), (100, 200)], border=3.0)
    assert len(out) == (0 if dropped else 1)
    assert len(_merge([[rec], []], sides=[side, 0], hw=[(100, 200), (500, 500)], border=None)) == 1


def test_border_drop_at_image_edges():
    """The 2x2 tiles of a 300 x 400 image: a box touching the image's outer edge in a corner tile stays, the same box at a
    tile's inner edge goes."""
    win = tiles.tile_windows(300, 400, 2, 2, 0.2)
    sides = tiles.view_sides(win, 300, 400)
    hw = [tuple(w[2:]) for w in win.tolist()]
    origins = [tuple(w[:2]) for w in win.tolist()]
    th, tw = hw[1]
    corner = (0., 0., 30., 30., 0.9, 1)                 # top-left of tile 1: image corner
    inner = (th - 30., tw - 30., th - 1., tw - 1., 0.8, 2)   # bottom-right of tile 1: inside the image
    views = [[], [corner, inner], [], [], []]
    out = _merge(views, origins=origins, sides=sides.tolist(), hw=hw, border=2.0)
    assert [r[5] for r in out] == [NBOX + 1]
    assert len(_merge(views, origins=origins, sides=sides.tolist(), hw=hw, border=0.5)) == 2


def test_zero_area_boxes_under_ios():
    line = (10., 10., 10., 50., 0.9, 0)                 # no height
    box = (0., 0., 100., 100., 0.8, 1)
    assert not ref.metric_gt(line[:4], box[:4], 0.0, "ios") and ref.metric_gt(line[:4], box[:4], -1.0, "ios")
    assert len(_merge([[line, box]], thr=0.0, match="ios")) == 2
    assert len(_merge([[line, box]], thr=-0.5, match="ios")) == 1     # 0 > -0.5: the zero-area metric matches


def test_ios_of_a_nested_box_is_one():
    inner = (10., 10., 20., 20.)
    outer = (0., 0., 100., 100.)
    assert ref.metric_gt(inner, outer, 0.999, "ios") and not ref.metric_gt(inner, outer, 1.0, "ios")
    assert not ref.metric_gt(inner, outer, 0.5, "iou")


def test_ties_order_by_view_then_index():
    a = (0., 0., 10., 10., 0.5, 9)
    b = (0., 0., 10., 10., 0.5, 2)
    c = (0., 0., 10., 11., 0.5, 4)
    out = _merge([[a], [b, c]], match="ios", merge="union")
    assert [(r[5], r[3]) for r in out] == [(9, F(11))]                 # view 0 wins the tie and folds both
    out = _merge([[], [c, b]], match="iou")
    assert [r[5] for r in out] == [NBOX + 2]                           # then the lower index


def test_union_orders_minus_zero_below_plus_zero():
    """-0.0 survives the shift only from an origin of -0.0 (-0.0 + +0.0 is +0.0), which k2y_merge_views_ex accepts."""
    kept = (0.0, 0.0, -0.0, -0.0, 0.9, 0)
    other = (-0.0, -0.0, 0.0, 0.0, 0.8, 1)
    origins = [(-0.0, -0.0)]
    out = _merge([[kept, other]], thr=-1.0, origins=origins, merge="union")     # zero areas: metric 0 > -1, every pair matches
    assert len(out) == 1 and [bool(np.signbit(v)) for v in out[0][:4]] == [True, True, False, False]
    out = _merge([[tuple(other[:4]) + (0.95, 2), kept]], thr=-1.0, origins=origins, merge="union")
    assert len(out) == 1 and out[0][5] == 2 and [bool(np.signbit(v)) for v in out[0][:4]] == [True, True, False, False]
    out = _merge([[kept]], thr=-1.0, origins=origins, merge="union")
    assert [bool(np.signbit(v)) for v in out[0][:4]] == [False, False, True, True]     # alone: its own fields


def test_union_skips_nan_fields():
    nan = F("nan")
    kept = (nan, 0., 10., 10., 0.9, 0)
    a = (2., -1., nan, 12., 0.8, 1)
    b = (nan, 1., nan, 5., 0.7, 2)
    out = _merge([[kept, a, b]], thr=-1.0, merge="union")
    y0, x0, y1, x1 = out[0][:4]
    assert (y0, x0, y1, x1) == (F(2), F(-1), F(10), F(12))
    alone = _merge([[kept]], thr=-1.0, merge="union")
    assert np.isnan(alone[0][0]) and alone[0][1:4] == (F(0), F(10), F(10))
    # a NaN coordinate never makes a border drop: fminf / fmaxf take the other field, a comparison with NaN is false
    assert not ref.border_drops((nan, nan, nan, nan), 15, 100, 100, 5.0)
    assert ref.border_drops((nan, 50., 1., 60.), 1, 100, 100, 5.0)


def test_defaults_equal_the_fixed_grid_merge():
    rng = np.random.default_rng(3)
    for trial in range(30):
        V = int(rng.integers(1, 8))
        views, origins = [], []
        for v in range(V):
            m = int(rng.integers(0, 12))
            y, x = rng.uniform(0, 300, m), rng.uniform(0, 300, m)
            h, w = rng.uniform(0, 150, m), rng.uniform(0, 150, m)
            s = rng.choice(F(np.linspace(0.1, 1.0, 7)), m)
            views.append([(F(y[j]), F(x[j]), F(y[j] + h[j]), F(x[j] + w[j]), F(s[j]), int(j)) for j in range(m)])
            origins.append((0, 0) if v == 0 else tuple(int(t) for t in rng.integers(0, 200, 2)))
        thr = float(rng.choice([0.0, 0.3, 0.5, 0.9]))
        want = tiles_ref.merge_class(views, origins, NBOX, thr, 30)
        got = ref.merge_class(views, origins, [0] * V, [(0, 0)] * V, NBOX, thr, 30)
        assert np.array(want, object).tolist() == np.array(got, object).tolist(), trial


# ---- BatchLayout and the flags ------------------------------------------------------------------------------------------
def test_layout_with_a_sized_tiling():
    images = [np.zeros((200, 300, 3), np.uint8), np.zeros((375, 500, 3), np.uint8), np.zeros((720, 1280, 3), np.uint8)]
    plan = tiles.SizedTiling((224, 320), 0.2, 10)
    lay = preprocess.BatchLayout(images, (224, 320), tiling=plan)
    assert lay.views is None and lay.view_counts.tolist() == [1, 5, 10] and lay.view_offsets.tolist() == [0, 1, 6, 16]
    assert lay.n_views == 16 and len(lay.view_matrices) == 16 and lay.merge_table_at is None
    assert lay.windows[:1].tolist() == [[0, 0, 200, 300]]
    assert lay.windows[1:6].tolist() == tiles.tile_windows(375, 500, 2, 2, 0.2).tolist()
    assert lay.windows[6:].tolist() == tiles.plan_windows(720, 1280, (224, 320), 0.2, 10).tolist()
    assert lay.view_sides.tolist() == np.concatenate([tiles.view_sides(lay.windows[a:b], h, w) for (a, b), (h, w) in
                                                      zip(zip(lay.view_offsets[:-1], lay.view_offsets[1:]), lay.hw)]).tolist()
    plain_end = lay.staged_end
    t = preprocess.BatchLayout(images, (224, 320), tiling=plan, merge_table=True)
    assert t.merge_table_at % preprocess.ALIGN == 0 and t.merge_table_at >= plain_end
    assert t.staged_end == t.merge_table_at + 4 * (4 + 16)
    assert t.merge_table.tolist() == lay.view_offsets.tolist() + lay.view_sides.tolist()
    fixed = preprocess.BatchLayout(images, (224, 320), tiling=(2, 2, 0.2))
    assert fixed.views == 5 and fixed.view_counts.tolist() == [5, 5, 5] and fixed.view_offsets.tolist() == [0, 5, 10, 15]


def test_serve_tile_flags():
    import serve
    ap = serve.build_parser()
    ns = ap.parse_args(["ck", "imgs", "--tile_size", "224", "320", "--tile_images", "4", "--tile_match", "ios", "--tile_merge",
                        "union", "--tile_border", "2.5"])
    assert ns.tile_size == [224, 320] and ns.tile_images == 4 and ns.tile_match == "ios" and ns.tile_merge == "union"
    assert ns.tile_border == 2.5 and ns.tiles is None
    ns = ap.parse_args(["ck", "imgs"])
    assert ns.tile_size is None and ns.tile_images is None and ns.tile_match == "iou" and ns.tile_merge == "suppress"
    assert ns.tile_border is None
    for bad in (["--tile_size", "224", "320"], ["--tile_images", "4"], ["--tiles", "2", "2", "--tile_size", "224", "320",
                                                                         "--tile_images", "4"], ["--tile_match", "giou"],
                ["--tile_merge", "wbf"]):
        with pytest.raises(SystemExit):
            ap.parse_args(["ck", "imgs"] + bad)
