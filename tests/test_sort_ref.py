"""oracle/sort_ref.py against the outside authorities, without a GPU: ``lsap`` equals scipy's linear_sum_assignment exactly, the
scalar Kalman form agrees with SORT's matrix-form filter, and ``Sort`` gives the ids and boxes of a literal matrix-form SORT;
plus the life-cycle rules, the refusals of ``enable_tracking`` and of ``serve.py --track`` on images."""
import math

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from oracle import sort_ref


def _same_assignment(c):
    a, b = linear_sum_assignment(c), sort_ref.lsap(c)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (c, a, b)


@pytest.mark.parametrize("kind", ["uniform", "integer"])
def test_lsap_equals_scipy_on_seeded_matrices(kind):
    rng = np.random.default_rng(1 if kind == "uniform" else 2)
    for _ in range(1500):
        nr, nc = (int(v) for v in rng.integers(1, 9, 2))
        c = rng.random((nr, nc)) if kind == "uniform" else rng.integers(0, 3, (nr, nc)).astype(np.float64)
        _same_assignment(c)
        _same_assignment(c.T)
        _same_assignment(-c)


def test_lsap_equals_scipy_on_degenerate_matrices():
    for shape in [(1, 1), (1, 7), (7, 1), (5, 5), (3, 8), (8, 3)]:
        _same_assignment(np.zeros(shape))
        _same_assignment(np.full(shape, 0.25))
        _same_assignment(-np.full(shape, 1.0))
    rng = np.random.default_rng(3)
    _same_assignment(rng.random((1, 9)))
    _same_assignment(rng.random((9, 1)))
    for shape in [(0, 0), (0, 4), (4, 0)]:
        r, c = sort_ref.lsap(np.zeros(shape))
        assert r.size == c.size == 0


def _rand_box(rng, scale=300.0):
    x1, y1 = rng.random(2) * scale
    w, h = 5 + rng.random(2) * 80
    return [float(x1), float(y1), float(x1 + w), float(y1 + h)]


def _close(a, b, rel=1e-9):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    ok = ~np.isnan(a)
    assert np.all(np.abs(a[ok] - b[ok]) <= rel * np.maximum(1.0, np.abs(b[ok]))), (a, b)


def test_scalar_kalman_agrees_with_the_matrix_filter():
    rng = np.random.default_rng(4)
    for seq in range(40):
        box = _rand_box(rng)
        s, m = sort_ref.ScalarKalman(box), sort_ref.MatrixKalman(box)
        for step in range(60):
            s.predict()
            m.predict()
            _close(s.state(), m.state())
            _close(s.box(), m.box())
            if rng.random() < 0.7:
                b = _rand_box(rng) if rng.random() < 0.2 else [v + rng.normal() * 3 for v in box]
                if b[2] - b[0] > 0 and b[3] - b[1] > 0:
                    box = b
                    s.update(box)
                    m.update(box)
                    _close(s.state(), m.state())


def test_vs_clamp_and_nan_prediction():
    for cls in (sort_ref.ScalarKalman, sort_ref.MatrixKalman):
        k = cls([0.0, 0.0, 100.0, 100.0])
        for w in (100.0, 100.0, 100.0, 60.0, 30.0, 10.0):     # the area shrinks fast: vs falls below -s
            k.predict()
            k.update([0.0, 0.0, w, w])
        x = k.state()
        assert x[6] + x[2] <= 0
        k.predict()
        assert k.state()[6] == 0.0
        if cls is sort_ref.ScalarKalman:        # vs *= 0.0 gives -0.0; the matrix product F x adds it to +0.0 terms
            assert math.copysign(1.0, k.state()[6]) == -1.0
    k = sort_ref.ScalarKalman([0.0, 0.0, math.inf, 10.0])     # an infinite box predicts NaN
    k.predict()
    assert any(v != v for v in k.box())
    t = sort_ref.Sort(1, 4, max_age=3, min_hits=0)
    ids, _ = t.update(0, np.array([[[0, 0, 10, np.inf], [0, 0, 10, 10], [0, 0, 0, 0], [0, 0, 0, 0]]], np.float32), [2])
    assert ids[0].tolist() == [1, 2, -1, -1] and len(t.tracks[0]) == 2
    t.update(1, np.zeros((1, 4, 4), np.float32), [0])
    assert [tr.id for tr in t.tracks[0]] == [2]          # the NaN prediction was deleted before association


def _scene(rng, n_frames, n_obj, size=400.0, duplicates=True):
    """Frames of one class: objects moving at constant speed that cross, vanish for a while (occlusion), appear and leave,
    each frame's records in random order with noise, a few zero-area records and (with `duplicates`) identical records, whose
    assignment ties only an exact restatement resolves alike."""
    objs = []
    for o in range(n_obj):
        start = int(rng.integers(0, n_frames // 2))
        objs.append(dict(start=start, end=start + int(rng.integers(3, n_frames)), p=rng.random(2) * size,
                         v=rng.normal(size=2) * 6, wh=10 + rng.random(2) * 60, gap=set(rng.integers(0, n_frames, 3).tolist())))
    frames = []
    for f in range(n_frames):
        recs = []
        for o in objs:
            if o["start"] <= f < o["end"] and f not in o["gap"]:
                c = o["p"] + o["v"] * (f - o["start"]) + rng.normal(size=2)
                x1, y1 = c - o["wh"] / 2
                recs.append([y1, x1, y1 + o["wh"][1], x1 + o["wh"][0]])
        if duplicates and rng.random() < 0.2 and recs:
            recs.append(list(recs[0]))
        if rng.random() < 0.1:
            recs.append([5.0, 5.0, 5.0, 9.0])
        rng.shuffle(recs)
        frames.append(np.array(recs, np.float32).reshape(-1, 4))
    return frames


def _block(frames_c, K):
    """One frame of C classes as (boxes [C, K, 4], counts [C])."""
    C = len(frames_c)
    boxes = np.zeros((C, K, 4), np.float32)
    counts = np.zeros(C, np.int32)
    for c, r in enumerate(frames_c):
        r = r[:K]
        boxes[c, :len(r)] = r
        counts[c] = len(r)
    return boxes, counts


@pytest.mark.parametrize("seed,max_age,min_hits,thresh", [(0, 1, 3, 0.3), (1, 3, 1, 0.3), (2, 0, 0, 0.1), (3, 5, 2, 0.5)])
def test_sort_ref_equals_matrix_sort(seed, max_age, min_hits, thresh):
    rng = np.random.default_rng(seed)
    frames = _scene(rng, 80, 14, duplicates=False)
    K = 24
    a, b = sort_ref.Sort(1, K, max_age, min_hits, thresh), sort_ref.MatrixSort(1, K, max_age, min_hits, thresh)
    reported = 0
    for f, recs in enumerate(frames):
        boxes, counts = _block([recs], K)
        ia, ba = a.update(f, boxes, counts)
        ib, bb = b.update(f, boxes, counts)
        assert np.array_equal(ia, ib), f
        np.testing.assert_allclose(ba, bb, rtol=1e-6)
        assert [t.id for t in a.tracks[0]] == [t.id + 1 for t in b.trackers[0]]
        for ta, tb in zip(a.tracks[0], b.trackers[0]):
            _close(ta.kf.box(), tb.kf.box())
            _close(ta.kf.state(), tb.kf.state())
        reported += int((ia >= 0).sum())
    assert reported > 100 and a.next_id > 14


@pytest.mark.parametrize("explicit", [sort_ref.Sort, sort_ref.MatrixSort])
def test_position_gaps_equal_explicit_empty_updates(explicit):
    rng = np.random.default_rng(5)
    frames = _scene(rng, 40, 8, duplicates=explicit is sort_ref.Sort)
    keep = [p for p in range(40) if p % 7 not in (3, 4)] + [60, 61]
    frames += [frames[-1]] * 22
    a, b = sort_ref.Sort(1, 16, 2, 1), explicit(1, 16, 2, 1)
    empty = np.zeros((1, 16, 4), np.float32)
    for p in range(62):
        boxes, counts = _block([frames[p]], 16)
        rb = b.update(p, boxes, counts) if p in keep else b.update(p, empty, [0])
        if p in keep:
            ra = a.update(p, boxes, counts)
            assert np.array_equal(ra[0], rb[0]), p
            np.testing.assert_allclose(ra[1], rb[1], rtol=1e-6)
    assert a.frame_count == b.frame_count == 62
    with pytest.raises(ValueError):
        a.update(61, empty, [0])


def _one(x, w=20.0):
    return np.array([[[10.0, x, 30.0, x + w]]], np.float32)


@pytest.mark.parametrize("cls", [sort_ref.Sort, sort_ref.MatrixSort])
def test_early_frames_report_and_later_births_wait_for_min_hits(cls):
    t = cls(2, 2, max_age=1, min_hits=2)
    blk = np.zeros((2, 2, 4), np.float32)
    blk[0, 0] = [10, 10, 30, 30]
    ids, _ = t.update(0, blk, [1, 0])
    assert ids[0, 0] == 1                               # frame_count 1 <= min_hits: a newborn is reported
    ids, _ = t.update(1, blk, [1, 0])
    assert ids[0, 0] == 1
    blk[1, 0] = [100, 100, 140, 150]
    ids, boxes = t.update(2, blk, [1, 1])
    assert ids[0, 0] == 1 and ids[1, 0] == -1 and boxes[1, 0].tolist() == [0, 0, 0, 0]   # born at frame 3: not yet
    ids, _ = t.update(3, blk, [1, 1])
    assert ids[1, 0] == -1                              # hit_streak 1 < 2
    ids, _ = t.update(4, blk, [1, 1])
    assert ids[1, 0] == 2


@pytest.mark.parametrize("cls", [sort_ref.Sort, sort_ref.MatrixSort])
def test_a_track_survives_max_age_missed_frames_and_no_more(cls):
    for max_age in (1, 3):
        t = cls(1, 1, max_age=max_age, min_hits=0)
        t.update(0, _one(10.0), [1])
        for p in range(1, max_age + 1):
            t.update(p, _one(10.0), [0])
        ids, _ = t.update(max_age + 1, _one(10.0), [1])
        assert ids[0, 0] == 1
        for p in range(max_age + 2, 2 * max_age + 3):
            t.update(p, _one(10.0), [0])
        ids, _ = t.update(2 * max_age + 3, _one(10.0), [1])
        assert ids[0, 0] == 2


def test_birth_order_sets_the_ids():
    for cls in (sort_ref.Sort, sort_ref.MatrixSort):
        t = cls(2, 3, max_age=1, min_hits=0, iou_thresh=0.3)
        blk = np.zeros((2, 3, 4), np.float32)
        blk[0, :2] = [[0, 0, 10, 10], [0, 6, 10, 16]]
        blk[1, 0] = [0, 0, 10, 10]
        ids, _ = t.update(0, blk, [2, 1])
        assert ids[0, :2].tolist() == [1, 2] and ids[1, 0] == 3          # class ascending, then record order
        # record 1 overlaps both tracks above the threshold, so the assignment runs: it takes track 1, record 0 takes track 2
        # with IoU 0 (a dropped match), record 2 no track.  Births: record 2 (untouched) first, then record 0 (dropped).
        blk[0, :3] = [[0, 40, 10, 50], [0, 3, 10, 13], [0, 100, 10, 110]]
        ids, _ = t.update(1, blk, [3, 0])
        assert ids[0].tolist() == [5, 1, 4]


class _Gather:
    def __init__(self, C, K):
        self.C, self.K = C, K


def test_enable_tracking_refusals_leave_the_pipeline_as_it_was():
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    p = object.__new__(DetectionPipeline)
    p.gather, p.device_index, p._track, p._track_n = _Gather(20, 30), 0, None, [None, None]
    for kw in (dict(max_age=34), dict(max_age=-1), dict(min_hits=-1), dict(iou_thresh=1.5), dict(max_age=1.5)):
        with pytest.raises(ValueError):
            p.enable_tracking(**kw)
        assert p._track is None and p._track_n == [None, None]
    p.gather = _Gather(80, 100)
    with pytest.raises(ValueError, match="max_age <= 9"):
        p.enable_tracking(max_age=10)
    assert p._track is None


def test_track_on_images_is_an_argparse_error(tmp_path):
    import serve
    (tmp_path / "imgs").mkdir()
    lst = tmp_path / "list.txt"
    lst.write_text("a.jpg\n")
    for images in (tmp_path / "imgs", lst):
        with pytest.raises(SystemExit):
            serve.build_parser().parse_args(["ck", str(images), "--track"])
        serve.build_parser().parse_args(["ck", str(images)])
