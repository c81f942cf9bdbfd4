"""oracle/ocsort_ref.py without a GPU: ``OcSort`` gives the ids and boxes of the literal matrix form bit for bit, each of
OC-SORT's mechanisms (ORU, OCM, OCR) and quirks changes the outcome where it should, the restated acos stays within 1 ulp of
math.acos, no stream passes the capacity bound, and the API and the command lines refuse what the tracker does not take."""
import copy
import math
import struct

import numpy as np
import pytest

from ocsort_streams import crowded, stream
from oracle import ocsort_ref as oc
from oracle import sort_ref


def _canonical(ids, boxes, frame):
    """ids and boxes with the outputs of identical records (same box and score) put in ascending id order.  Such records
    tie exactly in every cost, and the literal form's np.arccos, within 1 ulp of the restated acos but not always equal to
    it, can break the tie the other way in a later row; either record then carries the same track."""
    ids, boxes = ids.copy(), boxes.copy()
    b, counts, s = frame
    for c in range(ids.shape[0]):
        groups = {}
        for k in range(int(counts[c])):
            groups.setdefault(b[c, k].tobytes() + s[c, k].tobytes(), []).append(k)
        for ks in groups.values():
            if len(ks) > 1:
                order = sorted(ks, key=lambda k: ids[c, k])
                ids[c, ks], boxes[c, ks] = ids[c, order], boxes[c, order]
    return ids, boxes


def _both(kw, frames, positions=None):
    C, K = frames[0][0].shape[:2]
    a, m = oc.OcSort(C, K, **kw), oc.MatrixOcSort(C, K, **kw)
    out = []
    for p, (b, c, s) in zip(positions or range(len(frames)), frames):
        ia, ba = a.update(p, b, c, s)
        im, bm = m.update(p, b, c, s)
        ga, gm = (ia, ba), (im, bm)
        if not np.array_equal(ia, im):
            ga, gm = _canonical(ia, ba, (b, c, s)), _canonical(im, bm, (b, c, s))
        assert np.array_equal(ga[0], gm[0]), (p, np.argwhere(ga[0] != gm[0]))
        assert np.array_equal(ga[1].view(np.int32), gm[1].view(np.int32)), (p, np.argwhere(ga[1] != gm[1]))
        out.append((ia, ba))
    return a, out


@pytest.mark.parametrize("seed,C,K,kw", [
    (0, 3, 30, {}), (1, 3, 30, dict(use_byte=True)), (2, 2, 60, dict(delta_t=1, max_age=5)),
    (3, 2, 30, dict(delta_t=8, use_byte=True, max_age=3)), (4, 2, 40, dict(delta_t=5, min_hits=1, inertia=0.6)),
    (5, 1, 100, dict(use_byte=True, det_thresh=0.5, iou_thresh=0.2, max_age=8))])
def test_ocsort_equals_the_matrix_form(seed, C, K, kw):
    frames = stream(np.random.default_rng(seed), C, K, 60, n_obj=30 if K >= 60 else 12, max_age=kw.get("max_age", 30),
                    det_thresh=kw.get("det_thresh", 0.6))
    _, out = _both(kw, frames)
    assert (np.stack([o[0] for o in out]) >= 0).sum() > 40


@pytest.mark.parametrize("cls", [oc.OcSort, oc.MatrixOcSort])
def test_position_gaps_equal_explicit_empty_updates(cls):
    frames = stream(np.random.default_rng(6), 2, 30, 50, max_age=4)
    keep = [p for p in range(50) if p % 9 not in (3, 4, 5)]
    gapped, explicit = cls(2, 30, max_age=4, use_byte=True), cls(2, 30, max_age=4, use_byte=True)
    empty = (np.zeros((2, 30, 4), np.float32), np.zeros(2, np.int32), np.zeros((2, 30), np.float32))
    for p in range(50):
        if p in keep:
            a, b = gapped.update(p, *frames[p]), explicit.update(p, *frames[p])
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))
        else:
            explicit.update(p, *empty)


# -- hand-built cases ------------------------------------------------------------------------------------------------------------
def _frame(boxes_scores, K=4):
    b = np.zeros((1, K, 4), np.float32)
    s = np.zeros((1, K), np.float32)
    for k, (box, score) in enumerate(boxes_scores):
        b[0, k], s[0, k] = box, score
    return b, np.array([len(boxes_scores)], np.int32), s


def _box(x, y=100.0, w=40.0, h=80.0):
    return [y, x, y + h, x + w]        # (ymin, xmin, ymax, xmax)


def _det(x, y=100.0, w=40.0, h=80.0, s=0.9):
    return (float(np.float32(x)), float(np.float32(y)), float(np.float32(x + w)), float(np.float32(y + h)), float(np.float32(s)))


class _Matrix:
    """SORT's 7x7 filter with OC-SORT's z, run by hand."""

    def __init__(self, det):
        self.x = np.zeros(7)
        self.x[:4] = oc.to_z(det)
        self.P = sort_ref.MatrixKalman.P0.copy()

    def predict(self):
        F = sort_ref.MatrixKalman.F
        self.x, self.P = F @ self.x, F @ self.P @ F.T + sort_ref.MatrixKalman.Q

    def update(self, z):
        H, R = sort_ref.MatrixKalman.H, sort_ref.MatrixKalman.R
        S = H @ self.P @ H.T + R
        K = self.P @ H.T @ np.linalg.inv(S)
        self.x = self.x + K @ (np.asarray(z) - H @ self.x)
        I_KH = np.eye(7) - K @ H
        self.P = I_KH @ self.P @ I_KH.T + K @ R @ K.T


def test_oru_replays_the_virtual_path_and_applies_the_new_observation_twice():
    seen = [_det(100.0 + 6 * f) for f in range(5)]
    back = _det(100.0 + 6 * 9 + 6.0, y=104.0, w=42.0)              # frame 9, off the path it was on
    frames = [_frame([(_box(d[0], d[1], d[2] - d[0], d[3] - d[1]), 0.9)]) for d in seen] + [_frame([])] * 4 + \
        [_frame([(_box(back[0], back[1], back[2] - back[0], back[3] - back[1]), 0.9)])]
    a, out = _both(dict(min_hits=1), frames)
    assert int(out[-1][0][0, 0]) == 1
    got = np.array(a.tracks[0][0].kf.state())
    m = _Matrix(seen[0])
    for d in seen[1:]:
        m.predict()
        m.update(oc.to_z(d))
    m.predict()                                                     # frame 5: frozen after this predict
    z1, z2 = oc.to_z(seen[-1]), oc.to_z(back)
    w1, h1, w2, h2 = math.sqrt(z1[2] * z1[3]), math.sqrt(z1[2] / z1[3]), math.sqrt(z2[2] * z2[3]), math.sqrt(z2[2] / z2[3])
    gap = 5
    for i in range(1, gap + 1):
        w, h = w1 + i * (w2 - w1) / gap, h1 + i * (h2 - h1) / gap
        m.update([z1[0] + i * (z2[0] - z1[0]) / gap, z1[1] + i * (z2[1] - z1[1]) / gap, w * h, w / h])
        if i < gap:
            m.predict()
    once = m.x.copy()
    m.update(z2)                                                    # the real observation, on top
    np.testing.assert_allclose(got, m.x, rtol=1e-9, atol=1e-9)
    assert np.abs(once - m.x).max() > 1e-3                          # the second application moves the state
    plain = _Matrix(seen[0])                                        # no ORU: predict through the loss, update once
    for d in seen[1:]:
        plain.predict()
        plain.update(oc.to_z(d))
    for _ in range(5):
        plain.predict()
    plain.update(z2)
    assert np.abs(plain.x - got).max() > 1.0


def _predicted(t):
    """The box round 1 will see for track t in the next frame."""
    kf = copy.deepcopy(t.kf)
    kf.predict()
    return kf.box()


def test_ocm_direction_term_flips_an_assignment_iou_alone_decides_the_other_way():
    frames = [_frame([(_box(100.0 + 2 * f), 0.9)]) for f in range(8)]
    a, _ = _both(dict(delta_t=1), frames)
    x1, y1, x2, y2 = _predicted(a.tracks[0][0])
    side = _box(x1, y1 + 4.0, x2 - x1, y2 - y1)          # off the direction of motion: the larger IoU
    ahead = _box(x1 + 4.0, y1, x2 - x1, y2 - y1)         # along it
    pb = [x1, y1, x2, y2]
    assert sort_ref.iou([side[1], side[0], side[3], side[2]], pb) > sort_ref.iou([ahead[1], ahead[0], ahead[3], ahead[2]], pb)
    last = _frame([(side, 0.9), (ahead, 0.9)])
    ids = {}
    for inertia in (0.0, 0.6):
        _, out = _both(dict(delta_t=1, inertia=inertia), frames + [last])
        ids[inertia] = out[-1][0][0, :2].tolist()
    assert ids[0.0] == [1, -1]          # IoU alone: the record off the direction of motion
    assert ids[0.6] == [-1, 1]          # with the direction term: the one along it


def _drift_stream():
    """A track moving 15 px a frame for 6 frames, lost for 4, and back where it was last seen (record 1), with a record
    slightly overlapping its drifted prediction (record 0) and one far away (record 2)."""
    frames = [_frame([(_box(100.0 + 15 * f), 0.9)]) for f in range(6)] + [_frame([])] * 4
    return frames, [_box(280.0), _box(175.0), _box(1000.0)]


def test_ocr_refinds_a_track_whose_prediction_drifted_to_iou_zero():
    frames, (near, back, far) = _drift_stream()
    a, _ = _both(dict(min_hits=0), frames)
    pred = _predicted(a.tracks[0][0])
    assert sort_ref.iou([back[1], back[0], back[3], back[2]], pred) == 0.0
    assert 0.0 < sort_ref.iou([near[1], near[0], near[3], near[2]], pred) < 0.3
    _, out = _both(dict(min_hits=0), frames + [_frame([(near, 0.9), (back, 0.9), (far, 0.9)])])
    assert out[-1][0][0, :3].tolist() == [2, 1, 3]


def test_birth_order_becomes_sorted_once_ocrs_assignment_runs():
    frames, (near, back, far) = _drift_stream()
    # round 1 pairs the track with `near` and drops the pair (IoU < 0.3): the births would be [far, near]; OCR's
    # assignment takes `back` and sorts them, so `near` is born first
    _, out = _both(dict(min_hits=0), frames + [_frame([(near, 0.9), (back, 0.9), (far, 0.9)])])
    assert out[-1][0][0, 0] < out[-1][0][0, 2]
    # with nothing for OCR to take its assignment does not run, and the dropped record is born last
    _, out = _both(dict(min_hits=0), frames + [_frame([(near, 0.9), (_box(2000.0), 0.9), (far, 0.9)])])
    assert out[-1][0][0, 0] > out[-1][0][0, 2] > 0


def test_sum_of_sentinel_quirks_apply_at_negative_coordinates():
    for x, y, negative in ((-400.0, -300.0, True), (100.0, 100.0, False)):
        frames = [_frame([(_box(x + 3 * f, y), 0.9)]) for f in range(6)]
        a, out = _both(dict(min_hits=1), frames)
        t = a.tracks[0][0]
        assert (t.velocity is None) == negative         # last_observation never sums >= 0: no velocity
        rec = np.array(_box(x + 15, y), np.float32)
        if negative:                                    # the filter's state box, not the record's
            x1, y1, x2, y2 = t.kf.box()
            assert np.array_equal(out[-1][1][0, 0], np.array([y1, x1, y2, x2], np.float64).astype(np.float32))
            assert not np.array_equal(out[-1][1][0, 0], rec)
        else:
            assert np.array_equal(out[-1][1][0, 0], rec)


def test_k_previous_obs_falls_back_to_the_newest_observation():
    t = oc._Track(_det(0.0), 3)
    obs = {}
    for age, x in ((1, 10.0), (2, 20.0), (3, 30.0)):
        t.predict()
        t.update(_det(x))
        obs[age] = _det(x)
    t.predict()
    t.update(None)
    t.predict()                                         # age 5: ages 2, 3, 4 looked up, 2 first
    assert t.k_previous_obs() == _det(20.0) == tuple(oc.k_previous_obs(obs, 5, 3))
    t.update(None)
    t.predict()
    t.update(None)
    t.predict()                                         # age 7: ages 4, 5, 6 hold nothing: the newest, age 3's
    assert t.age == 7 and t.k_previous_obs() == _det(30.0) == tuple(oc.k_previous_obs(obs, 7, 3))
    assert tuple(oc.k_previous_obs({}, 7, 3)) == oc.SENTINEL == oc._Track(_det(0.0), 3).k_previous_obs()


# -- acos --------------------------------------------------------------------------------------------------------------------------
def _ulps(a, b):
    ia, ib = (struct.unpack("<q", struct.pack("<d", v))[0] for v in (a, b))
    ia, ib = (v if v >= 0 else -(v & 0x7fffffffffffffff) for v in (ia, ib))
    return abs(ia - ib)


def test_restated_acos_is_within_one_ulp_of_math_acos():
    edges = [-1.0, -0.0, 0.0, 1.0, 5e-324, -5e-324, 1e-300, -1e-300, 2.0 ** -57, -2.0 ** -57, 2.0 ** -56, 0.5, -0.5]
    edges += [float(np.nextafter(v, 0.0)) for v in (0.5, -0.5, 1.0, -1.0)] + [float(np.nextafter(v, 1.0)) for v in (0.5, -0.5)]
    sweep = edges + np.random.default_rng(3).uniform(-1.0, 1.0, 50000).tolist() + np.linspace(-1.0, 1.0, 20001).tolist()
    worst = max(_ulps(oc.acos(x), math.acos(x)) for x in sweep)
    assert worst <= 1
    assert oc.acos(1.0) == 0.0 and oc.acos(-1.0) == math.pi and oc.acos(0.0) == math.pi / 2.0


# -- capacity and refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [0, 1, 4, 30])
def test_no_stream_passes_the_bound(B):
    K = 20
    a = oc.OcSort(2, K, max_age=B)
    peak = 0
    for p, f in enumerate(crowded(2, K, B + 8)):
        a.update(p, *f)
        peak = max(peak, len(a.tracks[0]))
    assert peak == oc.max_tracks(K, B)                  # the crowded stream reaches the bound exactly
    for kw in ({}, dict(use_byte=True)):
        a = oc.OcSort(1, K, max_age=B, **kw)
        for p, f in enumerate(stream(np.random.default_rng(9), 1, K, 80, n_obj=30, max_age=B)):
            a.update(p, *f)
            assert len(a.tracks[0]) <= oc.max_tracks(K, B)


def test_settings_past_the_cap_are_refused():
    from k210_yolo_framework_b200.track import OCSORT_MAX_TRACKS_PER_CLASS, check_ocsort_setting
    assert oc.max_tracks(30, 30) == 930 and oc.max_tracks(100, 30) == 3100
    assert OCSORT_MAX_TRACKS_PER_CLASS == oc.MAX_TRACKS_PER_CLASS
    check_ocsort_setting(100, 0.6, 39, 3, 0.3, 3, 0.2)
    with pytest.raises(ValueError, match="max_age <= 39"):
        check_ocsort_setting(100, 0.6, 40, 3, 0.3, 3, 0.2)
    check_ocsort_setting(1, 0.6, 4095, 3, 0.3, 8, 0.2)
    for bad in (dict(det_thresh=1.5), dict(max_age=-1), dict(max_age=2.5), dict(min_hits=-1), dict(iou_thresh=-0.1),
                dict(delta_t=0), dict(delta_t=9), dict(delta_t=True), dict(inertia=1.5)):
        kw = dict(det_thresh=0.6, max_age=30, min_hits=3, iou_thresh=0.3, delta_t=3, inertia=0.2)
        kw.update(bad)
        with pytest.raises(ValueError):
            check_ocsort_setting(30, **kw)


class _Gather:
    def __init__(self, C, K):
        self.C, self.K = C, K


def test_enable_tracking_refusals_leave_the_pipeline_as_it_was():
    from k210_yolo_framework_b200.pipeline import DetectionPipeline
    p = object.__new__(DetectionPipeline)
    p.gather, p.device_index, p._track, p._track_n = _Gather(80, 100), 0, None, [None, None]
    for kw in (dict(method="ocsort", max_age=40), dict(method="ocsort", max_age=9, delta_t=9),
               dict(method="ocsort", max_age=9, track_buffer=10), dict(method="ocsort", max_age=9, fuse_score=False),
               dict(method="ocsort", max_age=9, inertia=2.0), dict(delta_t=5), dict(use_byte=True),
               dict(method="bytetrack", det_thresh=0.5), dict(method="bytetrack", inertia=0.3), dict(method="sort", max_age=10)):
        with pytest.raises(ValueError):
            p.enable_tracking(**kw)
        assert p._track is None and p._track_n == [None, None]


def test_tracker_flags_parse():
    import serve
    a = serve.build_parser().parse_args(["ck", "v.avi", "--tracker", "ocsort"])
    assert (a.track_max_age, a.track_min_hits, a.track_iou, a.track_det_thresh, a.track_delta_t, a.track_inertia,
            a.track_use_byte) == (30, 3, 0.3, 0.6, 3, 0.2, False)
    a = serve.build_parser().parse_args(["ck", "v.avi", "--tracker", "ocsort", "--track_max_age", "1", "--track_min_hits", "2",
                                         "--track_iou", "0.4", "--track_det_thresh", "0.5", "--track_delta_t", "5",
                                         "--track_inertia", "0.3", "--track_use_byte"])
    assert (a.track_max_age, a.track_min_hits, a.track_iou, a.track_det_thresh, a.track_delta_t, a.track_inertia,
            a.track_use_byte) == (1, 2, 0.4, 0.5, 5, 0.3, True)
    for argv in ([], ["--tracker", "bytetrack"]):
        d = serve.build_parser().parse_args(["ck", "v.avi"] + argv)
        assert (d.track_max_age, d.track_min_hits, d.track_iou) == (1, 3, 0.3)


def test_the_other_trackers_flags_are_argparse_errors(tmp_path):
    import evaluate_mot
    import serve
    for argv in (["--track_delta_t", "5"], ["--track_use_byte"], ["--tracker", "bytetrack", "--track_inertia", "0.5"],
                 ["--tracker", "bytetrack", "--track_det_thresh", "0.5"], ["--tracker", "ocsort", "--track_buffer", "10"],
                 ["--tracker", "ocsort", "--track_no_fuse_score"], ["--tracker", "ocsort", "--track_match", "0.5"]):
        with pytest.raises(SystemExit):
            serve.build_parser().parse_args(["ck", "v.avi"] + argv)
        with pytest.raises(SystemExit):
            evaluate_mot.build_parser().parse_args(["ck", str(tmp_path), "--person_class", "14"] + argv)
    a = evaluate_mot.build_parser().parse_args(["ck", str(tmp_path), "--person_class", "14", "--tracker", "ocsort",
                                                "--track_max_age", "3", "--track_use_byte"])
    assert (a.track_max_age, a.track_use_byte) == (3, True)
