"""oracle/bytetrack_ref.py without a GPU: the reduced assignment reaches the optimum of lap's extended square problem, the block
filter agrees with the matrix filter (cho_factor / cho_solve), ``ByteTrack`` gives the ids and boxes of the literal matrix
form; plus the named behaviours of ByteTrack, the capacity bound and the refusals of the settings past it."""
import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from bytetrack_streams import crowded, stream
from oracle import bytetrack_ref as br
from oracle import sort_ref


# -- assignment ----------------------------------------------------------------------------------------------------------------
def _extended_optimum(c, thresh):
    """scipy's optimum of lap.lapjv's extend_cost square matrix with cost_limit = thresh."""
    nr, nc = c.shape
    n = nr + nc
    ext = np.full((n, n), thresh / 2.0)
    ext[nr:, nc:] = 0.0
    ext[:nr, :nc] = c
    r, k = linear_sum_assignment(ext)
    return ext[r, k].sum()


def test_reduced_assignment_reaches_the_extended_optimum():
    rng = np.random.default_rng(11)
    cases = []
    for _ in range(600):
        nr, nc = (int(v) for v in rng.integers(0, 8, 2))
        kind = int(rng.integers(0, 3))
        c = rng.random((nr, nc)) if kind == 0 else (rng.integers(0, 4, (nr, nc)) / 4.0 if kind == 1 else np.full((nr, nc), 0.5))
        cases.append((c, float(rng.choice([0.0, 0.3, 0.5, 0.8, 1.0]))))
    for c, thresh in cases:
        matches, ur, uc = br.assign(c.tolist(), c.shape[1], thresh)
        assert all(c[i, j] < thresh for i, j in matches)
        assert sorted(ur + [i for i, _ in matches]) == list(range(c.shape[0]))
        assert sorted(uc + [j for _, j in matches]) == list(range(c.shape[1]))
        assert [i for i, _ in matches] == sorted(i for i, _ in matches)
        got = sum(c[i, j] - thresh for i, j in matches) + (c.shape[0] + c.shape[1]) * thresh / 2.0
        assert got == pytest.approx(_extended_optimum(c, thresh), abs=1e-9), (c, thresh)


# -- the filter ----------------------------------------------------------------------------------------------------------------
def _det(x1, y1, w, h, score=0.9, k=0):
    return br._Det(x1, y1, x1 + w, y1 + h, score, k)


def test_block_filter_agrees_with_the_matrix_filter():
    rng = np.random.default_rng(4)
    kf = br.KalmanFilter()
    for _ in range(40):
        d = _det(*(rng.random(2) * 500), *(5 + rng.random(2) * 100))
        t = br._Track(d, 2)
        mean, cov = kf.initiate(br.STrack.tlwh_to_xyah(np.array(d.tlwh)))
        for step in range(30):
            lost = rng.random() < 0.2
            t.state = br.LOST if lost else br.TRACKED
            if lost:
                mean = mean.copy()
                mean[7] = 0
            t.predict()
            mean, cov = kf.predict(mean, cov)
            if rng.random() < 0.8:
                x1, y1 = np.array(t.tlbr()[:2]) + rng.normal(size=2) * 3
                d = _det(x1, y1, *(5 + rng.random(2) * 100))
                t.update(d, step)
                mean, cov = kf.update(mean, cov, br.STrack.tlwh_to_xyah(np.array(d.tlwh)))
            blk = np.zeros((8, 8))
            for b in range(4):
                blk[b, b], blk[b, 4 + b], blk[4 + b, b], blk[4 + b, 4 + b] = t.cov[b][0], t.cov[b][1], t.cov[b][1], t.cov[b][2]
            np.testing.assert_allclose(t.mean, mean, rtol=1e-12, atol=0)
            # P -= K S K' cancels, so the covariance is compared relative to its largest entry
            np.testing.assert_allclose(blk, cov, rtol=0, atol=1e-12 * np.abs(cov).max())


# -- the restatement against the literal form --------------------------------------------------------------------------------
def _both(cls_kw, frames, positions=None, C=None, K=None):
    C = C or frames[0][0].shape[0]
    K = K or frames[0][0].shape[1]
    a, m = br.ByteTrack(C, K, **cls_kw), br.MatrixByteTrack(C, K, **cls_kw)
    out = []
    for p, (b, c, s) in zip(positions or range(len(frames)), frames):
        ia, ba = a.update(p, b, c, s)
        im, bm = m.update(p, b, c, s)
        assert np.array_equal(ia, im), (p, np.argwhere(ia != im))
        np.testing.assert_allclose(ba, bm, rtol=1e-6, atol=1e-6)
        out.append((ia, ba))
    return a, out


@pytest.mark.parametrize("seed,C,K,kw", [
    (0, 3, 30, {}), (1, 3, 30, dict(track_buffer=0)), (2, 3, 30, dict(track_buffer=1, fuse_score=False)),
    (3, 2, 60, dict(track_thresh=0.6, match_thresh=0.9)), (4, 2, 100, dict(track_buffer=5))])
def test_bytetrack_equals_the_matrix_form(seed, C, K, kw):
    frames = stream(np.random.default_rng(seed), C, K, 60, n_obj=40 if K >= 60 else 12, track_thresh=kw.get("track_thresh", 0.5))
    _, out = _both(kw, frames)
    ids = np.stack([o[0] for o in out])
    assert (ids >= 0).sum() > 60


# -- named behaviours ----------------------------------------------------------------------------------------------------------
def _frame(boxes_scores, C=1, K=4):
    b = np.zeros((C, K, 4), np.float32)
    s = np.zeros((C, K), np.float32)
    c = np.zeros(C, np.int32)
    for k, (box, score) in enumerate(boxes_scores):
        b[0, k], s[0, k] = box, score
    c[0] = len(boxes_scores)
    return b, c, s


def _box(x, y=100.0, w=40.0, h=80.0):
    return [y, x, y + h, x + w]        # (ymin, xmin, ymax, xmax)


def test_low_score_records_carry_a_track_through_an_occlusion():
    scores = [0.9] * 5 + [0.3] * 3 + [0.9] * 4
    frames = [_frame([(_box(100.0 + 3 * f), s)]) for f, s in enumerate(scores)]
    _, out = _both({}, frames)
    ids = [int(o[0][0, 0]) for o in out]
    assert ids[0] == 1 and set(ids) == {1}
    # SORT, given the records a detector keeps above track_thresh, starts a new track after the occlusion
    s = sort_ref.Sort(1, 4, max_age=1, min_hits=1)
    sort_ids = []
    for p, (b, c, sc) in enumerate(frames):
        keep = np.array([c[0] if sc[0, 0] > 0.5 else 0], np.int32)
        sort_ids.append(int(s.update(p, b, keep)[0][0, 0]))
    assert sort_ids[0] != sort_ids[-1] and sort_ids[-1] >= 0


def test_first_frame_births_report_at_once_and_later_births_wait_a_frame():
    frames = [_frame([(_box(100.0), 0.9)]), _frame([(_box(100.0), 0.9), (_box(300.0), 0.9)]),
              _frame([(_box(100.0), 0.9), (_box(300.0), 0.9)])]
    _, out = _both({}, frames)
    assert out[0][0][0, 0] == 1
    assert out[1][0][0, 0] == 1 and out[1][0][0, 1] == -1
    assert out[2][0][0, 0] == 1 and out[2][0][0, 1] == 2


@pytest.mark.parametrize("B", [0, 1, 5])
def test_a_lost_track_is_refound_within_track_buffer_and_no_later(B):
    for missed, same in ((max(B, 1) if B else 1, True), (B + 1 if B else 2, False)):
        frames = [_frame([(_box(100.0), 0.9)])] * 3 + [_frame([])] * missed + [_frame([(_box(100.0), 0.9)])] * 2
        _, out = _both(dict(track_buffer=B), frames)
        assert out[0][0][0, 0] == 1
        last = int(out[-1][0][0, 0])
        assert (last == 1) == same, (B, missed, [int(o[0][0, 0]) for o in out])


def test_a_low_score_record_never_starts_a_track():
    frames = [_frame([(_box(100.0 + f), 0.3), (_box(300.0), 0.55)]) for f in range(6)]
    a, out = _both({}, frames)
    assert all((o[0] == -1).all() for o in out)
    assert a.next_id == 1 + 0 and not a.tracked[0] and not a.lost[0]
    frames = [_frame([(_box(300.0), 0.6)])] + frames
    a, out = _both({}, frames)
    assert out[0][0][0, 0] == 1 and a.next_id == 2


def test_duplicate_removal_keeps_the_longer_lived_track():
    frames = [_frame([(_box(100.0), 0.9)])] * 2 + [_frame([(_box(100.0), 0.9), (_box(102.0), 0.9)])] * 4 + \
        [_frame([(_box(101.0), 0.9)])] * 2
    a, out = _both({}, frames)
    live = [t.id for t in a.tracked[0] + a.lost[0]]
    assert 1 in live and 2 not in live
    assert all(int(o[0][0, 0]) in (1, -1) for o in out[-2:])


@pytest.mark.parametrize("cls", [br.ByteTrack, br.MatrixByteTrack])
def test_position_gaps_equal_explicit_empty_updates(cls):
    frames = stream(np.random.default_rng(5), 2, 30, 50)
    keep = [p for p in range(50) if p % 9 not in (3, 4, 5)]
    gapped = cls(2, 30, track_buffer=2)
    explicit = cls(2, 30, track_buffer=2)
    empty = (np.zeros((2, 30, 4), np.float32), np.zeros(2, np.int32), np.zeros((2, 30), np.float32))
    for p in range(50):
        if p in keep:
            a = gapped.update(p, *frames[p])
            b = explicit.update(p, *frames[p])
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        else:
            explicit.update(p, *empty)


def _live_peak(C, K, B, frames):
    """The most tracks one class holds within a frame: the live tracks before it plus its births."""
    t = br.ByteTrack(C, K, track_buffer=B)
    peak, before = 0, 0
    for p, f in enumerate(frames):
        ids_before = t.next_id
        t.update(p, *f)
        peak = max(peak, before + (t.next_id - ids_before))
        before = len(t.tracked[0]) + len(t.lost[0])
        assert before <= K * (max(B, 1) + 1)
    return peak


@pytest.mark.parametrize("B", [0, 1, 4, 30])
def test_the_crowded_stream_stays_within_the_bound(B):
    K = 20
    peak = _live_peak(2, K, B, crowded(2, K, 2 * max(B, 1) + 12))
    assert peak <= br.max_tracks(K, B)
    assert peak >= K * (max(B, 1) // 2 + 2)
    rnd = stream(np.random.default_rng(9), 1, K, 80, n_obj=30)
    assert _live_peak(1, K, B, rnd) <= br.max_tracks(K, B)


def test_settings_past_the_cap_are_refused():
    from k210_yolo_framework_b200.track import BYTETRACK_MAX_TRACKS_PER_CLASS, check_bytetrack_setting
    assert br.max_tracks(100, 30) == 3200 and br.max_tracks(30, 30) == 960 and br.max_tracks(30, 0) == 90
    check_bytetrack_setting(100, 0.5, 0.8, 38)
    with pytest.raises(ValueError, match="track_buffer <= 38"):
        check_bytetrack_setting(100, 0.5, 0.8, 39)
    assert br.max_tracks(100, 38) <= BYTETRACK_MAX_TRACKS_PER_CLASS < br.max_tracks(100, 39)
    for bad in (dict(track_thresh=1.5), dict(match_thresh=-0.1), dict(track_buffer=-1), dict(track_buffer=2.5)):
        kw = dict(track_thresh=0.5, match_thresh=0.8, track_buffer=30)
        kw.update(bad)
        with pytest.raises(ValueError):
            check_bytetrack_setting(30, **kw)


class _Gather:
    def __init__(self, C, K):
        self.C, self.K = C, K


def test_enable_tracking_refusals_leave_the_pipeline_as_it_was():
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    p = object.__new__(DetectionPipeline)
    p.gather, p.device_index, p._track, p._track_n = _Gather(80, 100), 0, None, [None, None]
    for kw in (dict(method="bytetrack", track_buffer=39), dict(method="bytetrack", track_thresh=2.0),
               dict(method="bytetrack", max_age=3), dict(method="bytetrack", iou_thresh=0.5), dict(track_buffer=10),
               dict(fuse_score=False), dict(method="deepsort")):
        with pytest.raises(ValueError):
            p.enable_tracking(**kw)
        assert p._track is None and p._track_n == [None, None]


def test_tracker_flags_parse():
    import serve
    a = serve.build_parser().parse_args(["ck", "v.avi", "--tracker", "bytetrack", "--track_thresh", "0.6", "--track_match", "0.9",
                                         "--track_buffer", "12", "--track_no_fuse_score"])
    assert (a.tracker, a.track_thresh, a.track_match, a.track_buffer, a.track_no_fuse_score) == ("bytetrack", 0.6, 0.9, 12, True)
    d = serve.build_parser().parse_args(["ck", "v.avi"])
    assert (d.tracker, d.track_thresh, d.track_match, d.track_buffer, d.track_no_fuse_score) == ("sort", 0.5, 0.8, 30, False)


def test_the_other_trackers_flags_are_argparse_errors(tmp_path):
    import evaluate_mot
    import serve
    for argv in (["--track_buffer", "10"], ["--track_no_fuse_score"], ["--tracker", "bytetrack", "--track_max_age", "3"],
                 ["--tracker", "bytetrack", "--track_iou", "0.5"]):
        with pytest.raises(SystemExit):
            serve.build_parser().parse_args(["ck", "v.avi"] + argv)
        with pytest.raises(SystemExit):
            evaluate_mot.build_parser().parse_args(["ck", str(tmp_path), "--person_class", "14"] + argv)
    evaluate_mot.build_parser().parse_args(["ck", str(tmp_path), "--person_class", "14", "--track_max_age", "3"])
