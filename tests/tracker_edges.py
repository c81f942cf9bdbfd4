"""Frames that put a tracker's decision exactly on its threshold, for SORT (oracle/sort_ref.py), ByteTrack
(oracle/bytetrack_ref.py) and OC-SORT (oracle/ocsort_ref.py).  Each boundary case holds one float64 quantity equal to one
threshold, and names what moves the threshold to its neighbours:

* ``param``: the threshold is a setting; side -1 / +1 runs with np.nextafter(t, -inf / +inf) (an integer setting: t -/+ 1);
* ``score``: the threshold is fixed and the quantity is a float32 score; a side moves that score by one float32 step;
* ``const``: the threshold is a constant of the tracker (ByteTrack's 0.5 and 0.7); only the oracle's constant can move.

``flip`` is the side whose ids or boxes differ from those at t (tests/test_tracker_edges_ref.py proves it).  The boxes are
chosen so that the boxes the trackers compare are exact: zero-velocity tracks of square boxes predict their own box, 12 x 12
boxes shifted by 4 have an IoU of exactly 0.5 (SORT's IoU; ByteTrack's "+1" IoU with 11 x 11 boxes), and so on.

ByteTrack's duplicate threshold 0.15 has no exact case: its cost 1 - IoU is exact for IoU >= 0.5, so it could equal 0.15
only if the double 0.15 were a multiple of 2^-53, which it is not.

``EDGE_STREAMS`` are further frames at the trackers' edges that are not a single threshold (tie-heavy frames, OC-SORT's
delta_t, inertia and direction extremes), compared kernel against oracle only."""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

from oracle import bytetrack_ref, ocsort_ref, sort_ref


def frame(C, K, recs):
    """(boxes float32 [C, K, 4] (ymin, xmin, ymax, xmax), counts [C], scores float32 [C, K]) of {class: [(x1, y1, x2, y2,
    score)]}."""
    boxes = np.zeros((C, K, 4), np.float32)
    scores = np.zeros((C, K), np.float32)
    counts = np.zeros(C, np.int32)
    for c, rs in recs.items():
        for k, (x1, y1, x2, y2, s) in enumerate(rs):
            boxes[c, k] = [y1, x1, y2, x2]
            scores[c, k] = s
        counts[c] = len(rs)
    return boxes, counts, scores


def sq(x, y, side, s=0.9):
    """A square record of `side` at (x, y)."""
    return (x, y, x + side, y + side, s)


@dataclass
class Case:
    name: str
    tracker: str                    # "sort", "bytetrack" or "ocsort"
    C: int
    K: int
    kw: dict
    frames: list
    positions: list
    kind: str = "param"             # "param", "score" or "const"
    param: Optional[str] = None     # the setting ("param") or oracle constant ("const") that is the threshold
    t: float = 0.0                  # the threshold
    quantity: float = 0.0           # what meets it, computed with the oracle's helpers
    flip: int = 1
    score_at: tuple = ()            # (frame, class, record) of the score a "score" case moves


def neighbour(t, side):
    if side == 0:
        return t
    if isinstance(t, int):
        return t + side
    return float(np.nextafter(t, math.inf if side > 0 else -math.inf))


def variant(case: Case, side: int):
    """(kw, frames) of the case at `side`; None where the kernel cannot run it (a setting outside its range, or a
    constant of the tracker)."""
    if side == 0:
        return case.kw, case.frames
    if case.kind == "param":
        v = neighbour(case.t, side)
        if (v < 0) if isinstance(v, int) else not 0.0 <= v <= 1.0:        # frames >= 0; IoUs and scores in [0, 1]
            return None
        return dict(case.kw, **{case.param: v}), case.frames
    if case.kind == "score":
        f, c, k = case.score_at
        frames = [(b.copy(), n.copy(), s.copy()) for b, n, s in case.frames]
        s = frames[f][2]
        s[c, k] = np.nextafter(s[c, k], np.float32(math.inf if side > 0 else -math.inf))
        return case.kw, frames
    return None


def run_ref(tracker, C, K, kw, frames, positions):
    """The oracle's (ids [N, C, K], boxes [N, C, K, 4]) over the frames."""
    if tracker == "sort":
        t = sort_ref.Sort(C, K, **kw)
        out = [t.update(p, b, c) for p, (b, c, _) in zip(positions, frames)]
    else:
        t = (bytetrack_ref.ByteTrack if tracker == "bytetrack" else ocsort_ref.OcSort)(C, K, **kw)
        out = [t.update(p, *f) for p, f in zip(positions, frames)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def _xyxy(r):
    return list(r[:4])


# -- SORT ------------------------------------------------------------------------------------------------------------------------
def _sort_pred(birth):
    """The box a track born from `birth` (x1, y1, x2, y2) predicts in the next frame."""
    kf = sort_ref.ScalarKalman(birth)
    kf.predict()
    return kf.box()


def sort_cases():
    C, K = 2, 8
    F = lambda recs: frame(C, K, {1: recs})
    out = []
    a, b = sq(100, 100, 12), sq(104, 100, 12)
    q = sort_ref.iou(_xyxy(b), _sort_pred(_xyxy(a)))
    # the filter: a match of the assignment with iou < thresh is dropped (the record is born)
    out.append(Case("sort_filter_iou_half", "sort", C, K, dict(max_age=1, min_hits=0, iou_thresh=0.5), [F([a]), F([b])],
                    [0, 1], param="iou_thresh", t=0.5, quantity=q, flip=1))
    # the shortcut: when the entries with iou > thresh share no row and no column they are taken as they are.  At thresh
    # 0.5 the only such entry is (d0, t1) at 0.6, so d0 goes to t1; one step below, (d0, t0) at exactly 0.5 passes too,
    # the assignment runs and pairs d0 with t0 (0.5 + 7/17 against 0.6 + 0)
    t0, t1, d0, d1 = sq(100, 100, 12), sq(107, 100, 12), sq(104, 100, 12), sq(112, 100, 12)
    q = sort_ref.iou(_xyxy(d0), _sort_pred(_xyxy(t0)))
    out.append(Case("sort_shortcut_iou_half", "sort", C, K, dict(max_age=1, min_hits=0, iou_thresh=0.5),
                    [F([t0, t1]), F([d0, d1])], [0, 1], param="iou_thresh", t=0.5, quantity=q, flip=-1))
    far = sq(300, 100, 12)
    q = sort_ref.iou(_xyxy(far), _sort_pred(_xyxy(a)))
    out.append(Case("sort_iou_thresh_0", "sort", C, K, dict(max_age=1, min_hits=0, iou_thresh=0.0), [F([a]), F([far])],
                    [0, 1], param="iou_thresh", t=0.0, quantity=q, flip=1))
    q = sort_ref.iou(_xyxy(a), _sort_pred(_xyxy(a)))
    out.append(Case("sort_iou_thresh_1", "sort", C, K, dict(max_age=1, min_hits=0, iou_thresh=1.0), [F([a]), F([a])],
                    [0, 1], param="iou_thresh", t=1.0, quantity=q, flip=1))
    # reported when hit_streak >= min_hits: born at frame 4, the streak reaches 3 at frame 7
    fr = [F([]) for _ in range(4)] + [F([a]) for _ in range(4)]
    s = sort_ref.Sort(C, K, max_age=1, min_hits=3)
    for p, (bx, n, _) in enumerate(fr):
        s.update(p, bx, n)
    out.append(Case("sort_streak_is_min_hits", "sort", C, K, dict(max_age=1, min_hits=3, iou_thresh=0.3), fr, list(range(8)),
                    param="min_hits", t=3, quantity=s.tracks[1][0].hit_streak, flip=1))
    # reported when frame_count <= min_hits: born (streak 0) in the third update
    fr = [F([]), F([]), F([a])]
    s = sort_ref.Sort(C, K, max_age=1, min_hits=3)
    for p, (bx, n, _) in enumerate(fr):
        s.update(p, bx, n)
    out.append(Case("sort_frame_count_is_min_hits", "sort", C, K, dict(max_age=1, min_hits=3, iou_thresh=0.3), fr, [0, 1, 2],
                    param="min_hits", t=3, quantity=s.frame_count, flip=-1))
    # removed when time_since_update > max_age: missed for exactly max_age frames, then seen again
    fr = [F([a]), F([]), F([]), F([]), F([a])]
    s = sort_ref.Sort(C, K, max_age=3, min_hits=0)
    for p, (bx, n, _) in enumerate(fr[:-1]):
        s.update(p, bx, n)
    out.append(Case("sort_missed_max_age_frames", "sort", C, K, dict(max_age=3, min_hits=0, iou_thresh=0.3), fr,
                    list(range(5)), param="max_age", t=3, quantity=s.tracks[1][0].time_since_update, flip=-1))
    # a gap of max_age + 1 positions: max_age updates without detections
    s = sort_ref.Sort(C, K, max_age=3, min_hits=0)
    s.update(0, *F([a])[:2])
    for _ in range(4 - 0 - 1):              # what update(4) runs first: an update without detections per missing position
        s._empty_update()
    out.append(Case("sort_gap_max_age_plus_1", "sort", C, K, dict(max_age=3, min_hits=0, iou_thresh=0.3), [F([a]), F([a])],
                    [0, 4], param="max_age", t=3, quantity=s.tracks[1][0].time_since_update, flip=-1))
    return out


# -- ByteTrack -------------------------------------------------------------------------------------------------------------------
def _bt_det(r):
    return bytetrack_ref._Det(r[0], r[1], r[2], r[3], float(np.float32(r[4])), 0)


def bytetrack_cases():
    C, K = 2, 8
    F = lambda recs: frame(C, K, {1: recs})
    out = []
    a = sq(100, 100, 11)
    s6 = np.float32(0.6)
    # high when score > track_thresh, low when 0.1 < score < track_thresh: at equality neither
    out.append(Case("bytetrack_score_is_track_thresh", "bytetrack", C, K, dict(track_thresh=float(s6)),
                    [F([a]), F([a[:4] + (s6,)])], [0, 1], param="track_thresh", t=float(s6), quantity=float(s6), flip=1))
    # the low bound: float32(0.1) widened is above 0.1, the float32 below it is not
    lo = np.float32(0.1)
    out.append(Case("bytetrack_score_float32_0_1", "bytetrack", C, K, {}, [F([a]), F([a[:4] + (lo,)])], [0, 1],
                    kind="score", t=bytetrack_ref.LOW_THRESH, quantity=float(lo), flip=-1, score_at=(1, 1, 0)))
    # born when score >= det_thresh = track_thresh + 0.1: 0.4 + 0.1 is 0.5 exactly
    out.append(Case("bytetrack_score_is_det_thresh", "bytetrack", C, K, dict(track_thresh=0.4), [F([a[:4] + (0.5,)])], [0],
                    kind="score", t=0.4 + 0.1, quantity=float(np.float32(0.5)), flip=-1, score_at=(0, 1, 0)))
    # the second association keeps cost < 0.5: a low record at IoU 0.5 exactly
    b = sq(104, 100, 11, 0.3)
    tr = bytetrack_ref._Track(_bt_det(a), 1)
    tr.predict()
    q = 1.0 - bytetrack_ref.iou(tr.tlbr(), _bt_det(b).tlbr)
    out.append(Case("bytetrack_second_cost_0_5", "bytetrack", C, K, {}, [F([a]), F([b])], [0, 1], kind="const",
                    param="SECOND_THRESH", t=bytetrack_ref.SECOND_THRESH, quantity=q, flip=1))
    # round 1 keeps cost < match_thresh (plain cost)
    b = sq(104, 100, 11)
    q = 1.0 - bytetrack_ref.iou(tr.tlbr(), _bt_det(b).tlbr)
    out.append(Case("bytetrack_cost_is_match_thresh", "bytetrack", C, K, dict(match_thresh=q, fuse_score=False),
                    [F([a]), F([b])], [0, 1], param="match_thresh", t=q, quantity=q, flip=1))
    # the unconfirmed association keeps cost < 0.7: a track born in frame 2 (not activated), 12 x 12 boxes shifted by 7
    u, v = sq(100, 100, 12), sq(107, 100, 12)
    tu = bytetrack_ref._Track(_bt_det(u), 2)
    q = 1.0 - bytetrack_ref.iou(tu.tlbr(), _bt_det(v).tlbr)
    out.append(Case("bytetrack_unconfirmed_cost_0_7", "bytetrack", C, K, dict(fuse_score=False), [F([]), F([u]), F([v])],
                    [0, 1, 2], kind="const", param="UNCONFIRMED_THRESH", t=bytetrack_ref.UNCONFIRMED_THRESH, quantity=q,
                    flip=1))
    # a lost track is removed when frame_id - end_frame > track_buffer: lost for exactly track_buffer frames, then found
    fr = [F([a]), F([]), F([]), F([]), F([a])]
    bt = bytetrack_ref.ByteTrack(C, K, track_buffer=3)
    for p, f in enumerate(fr[:-1]):
        bt.update(p, *f)
    out.append(Case("bytetrack_lost_track_buffer_frames", "bytetrack", C, K, dict(track_buffer=3), fr, list(range(5)),
                    param="track_buffer", t=3, quantity=bt.frame_id - bt.lost[1][0].frame_id, flip=-1))
    return out


# -- OC-SORT ---------------------------------------------------------------------------------------------------------------------
def _moving(n, step=2.0, x0=100.0):
    """Records of a 12 x 12 box moving `step` along x for n frames."""
    return [sq(x0 + step * f, 100, 12) for f in range(n)]


def _oc_state(C, K, kw, frames):
    """The oracle after the frames, and its track of class 1 predicted for the next frame (a copy)."""
    t = ocsort_ref.OcSort(C, K, **kw)
    for p, f in enumerate(frames):
        t.update(p, *f)
    trk = copy.deepcopy(t.tracks[1][0])
    return trk, trk.predict()


def ocsort_cases():
    C, K = 2, 8
    F = lambda recs: frame(C, K, {1: recs})
    out = []
    a = sq(100, 100, 12)
    s6 = np.float32(0.6)
    # high (and born) when score > det_thresh
    out.append(Case("ocsort_score_is_det_thresh", "ocsort", C, K, dict(det_thresh=float(s6), min_hits=0),
                    [F([a[:4] + (s6,)])], [0], param="det_thresh", t=float(s6), quantity=float(s6), flip=-1))
    s5 = np.float32(0.55)
    out.append(Case("ocsort_byte_score_is_det_thresh", "ocsort", C, K, dict(det_thresh=float(s5), min_hits=0, use_byte=True),
                    [F([a]), F([a[:4] + (s5,)])], [0, 1], param="det_thresh", t=float(s5), quantity=float(s5), flip=1))
    lo = np.float32(0.1)
    out.append(Case("ocsort_byte_score_float32_0_1", "ocsort", C, K, dict(min_hits=0, use_byte=True),
                    [F([a]), F([a[:4] + (lo,)])], [0, 1], kind="score", t=ocsort_ref.LOW_THRESH, quantity=float(lo), flip=-1,
                    score_at=(1, 1, 0)))
    # round 1 at iou == iou_thresh on the predicted box: the record ahead of the track's prediction
    kw = dict(min_hits=0, iou_thresh=0.5)
    path = _moving(8)
    trk, pred = _oc_state(C, K, kw, [F([r]) for r in path])
    d = sq(100 + 2 * 8 + 3, 100, 12)
    q = ocsort_ref.iou(_xyxy(d), pred)
    out.append(Case("ocsort_round1_iou_is_thresh", "ocsort", C, K, dict(kw, iou_thresh=q), [F([r]) for r in path] + [F([d])],
                    list(range(9)), param="iou_thresh", t=q, quantity=q, flip=1))
    # round 3 (OCR) at iou == iou_thresh on the last observation: the record 4 behind it, away from the prediction
    d = sq(path[-1][0] - 4, 100, 12)
    q = ocsort_ref.iou(_xyxy(d), list(trk.last_obs[:4]))
    assert ocsort_ref.iou(_xyxy(d), pred) < 0.5
    out.append(Case("ocsort_ocr_iou_is_thresh", "ocsort", C, K, kw, [F([r]) for r in path] + [F([d])], list(range(9)),
                    param="iou_thresh", t=0.5, quantity=q, flip=-1))
    # removed when time_since_update > max_age
    fr = [F([a]), F([]), F([]), F([]), F([a])]
    oc = ocsort_ref.OcSort(C, K, max_age=3, min_hits=0)
    for p, f in enumerate(fr[:-1]):
        oc.update(p, *f)
    out.append(Case("ocsort_missed_max_age_frames", "ocsort", C, K, dict(max_age=3, min_hits=0), fr, list(range(5)),
                    param="max_age", t=3, quantity=oc.tracks[1][0].time_since_update, flip=-1))
    return out


def boundary_cases():
    return sort_cases() + bytetrack_cases() + ocsort_cases()


# -- edges that are not one threshold --------------------------------------------------------------------------------------------
def _tie_frames(C, K):
    """More than 32 identical tracks met by more than 32 identical and duplicated records: every assignment step a tie."""
    a, b = sq(100, 100, 12), sq(103, 100, 12)
    return [frame(C, K, {0: [a] * 40}), frame(C, K, {0: [a] * 40}), frame(C, K, {0: [a] * 20 + [b] * 25}),
            frame(C, K, {0: [b] * 45}), frame(C, K, {0: [a, b] * 23})]


def _direction_frames(C, K):
    """One object per class 0 that moves along x, turns back (exactly opposite), stops (zero displacement), is lost for a
    while and comes back; a second one that moves along y exactly parallel to itself."""
    fr = []
    x = 100.0
    for f in range(30):
        step = 4.0 if f < 10 else (-4.0 if f < 18 else 0.0)
        x += step
        recs = [] if 22 <= f < 25 else [sq(x, 100, 12, 0.9)]
        recs.append(sq(300, 100 + 3.0 * f, 10, 0.8))
        fr.append(frame(C, K, {0: recs}))
    return fr


EDGE_STREAMS = [
    ("sort_ties", "sort", dict(max_age=3, min_hits=0), _tie_frames),
    ("bytetrack_ties", "bytetrack", dict(track_buffer=3), _tie_frames),
    ("ocsort_ties", "ocsort", dict(max_age=3, min_hits=0), _tie_frames),
    ("ocsort_delta_t_1_inertia_0", "ocsort", dict(delta_t=1, inertia=0.0, min_hits=0, max_age=2), _direction_frames),
    ("ocsort_delta_t_8_inertia_1", "ocsort", dict(delta_t=8, inertia=1.0, min_hits=0, max_age=2), _direction_frames),
    ("ocsort_delta_t_3_expiry", "ocsort", dict(delta_t=3, min_hits=1, max_age=1), _direction_frames),
]
