"""SORT (Bewley et al., 2016, "Simple Online and Realtime Tracking") restated in plain Python: the rules the GPU tracker
(``k2y_track_update``, csrc/track.cu) follows bit for bit.  ``Sort.update`` of the published sort.py, with these choices:

* Per class.  A track belongs to one class and matches only records of its class; every class runs SORT on its own records.
  On single-class data this is SORT exactly.
* Detections.  A frame's records come in gather order (class ascending, then record order).  Each becomes the float64 box
  [x1, y1, x2, y2] = [xmin, ymin, xmax, ymax] (exact).  A record whose width x2 - x1 or height y2 - y1 is not > 0 is not a
  detection and gets no track.
* Kalman filter.  SORT's 7-state constant-velocity filter [cx, cy, s, r, vcx, vcy, vs] with its F, H, Q = diag(1, 1, 1, 1,
  .01, .01, 1e-4), R = diag(1, 1, 10, 10) and initial P = diag(10, 10, 10, 10, 1e4, 1e4, 1e4).  With these matrices P stays
  block-diagonal, blocks (cx, vcx), (cy, vcy), (s, vs) and (r), and S is diagonal, so the filter is exactly three 2-state
  filters and one scalar filter.  ``_predict2`` / ``_update2`` / ``_predict1`` / ``_update1`` state them with an explicit order
  of float64 operations and no fused multiply-add (filterpy's predict, P = F P F' + Q, and Joseph-form update,
  P = (I - K H) P (I - K H)' + K R K', written out per block); the GPU does the same operations in the same order.
* The filter's quirks, kept: before each predict vs *= 0.0 when vs + s <= 0 (a negative vs becomes -0.0); a track whose
  predicted box has a NaN is deleted before association; a box is w = sqrt(s r), h = s / w.
* IoU is SORT's ``iou_batch`` (no "+1"), with max and min propagating NaN as numpy's do.  One deviation: an IoU whose union
  is not > 0 counts as 0 (numpy would give NaN, which scipy's assignment refuses).
* Association is SORT's ``associate_detections_to_trackers``: when every row and column of (iou > thresh) has at most one
  entry and some entry is set, those pairs in row-major order; otherwise ``lsap(-iou)``; then a match with iou < thresh is
  dropped.  Unmatched detections are born in SORT's order: those no pair touched, ascending, then the dropped matches' in
  match order.
* ``lsap`` restates scipy's ``linear_sum_assignment`` (Crouse's shortest augmenting path as scipy implements it): transposed
  when there are more rows than columns, remaining columns scanned from a list filled in reverse order and shrunk by
  swap-with-last, a tie on path cost going to an unassigned column, the dual updates u[i] += minVal - d[col4row[i]] and
  v[j] -= minVal - d[j].  Its row and column arrays equal scipy's, ties included.
* Life cycle: SORT's hits, hit_streak, time_since_update and age.  A track is reported in a frame when
  time_since_update < 1 and (hit_streak >= min_hits or frame_count <= min_hits), frame_count counting the stream's updates.
  A track is removed when time_since_update > max_age.  Removal runs before the frame's births are appended; SORT appends
  first and deletes after, and since a newborn is never removed the track list, the assignment's column order, is the same.
* Ids: one counter per stream starting at 1, taken in birth order: frame, then class ascending, then birth order in the class.
* Dropped frames: a frame is identified by its position in the stream.  A jump of g > 1 positions first runs g - 1 updates
  without detections, as SORT called on each missing frame does.
* Output per record: a track id, or -1 when the record has no track or its track is not reported this frame; and for a record
  with an id, the track's post-update state box (ymin, xmin, ymax, xmax), float64 rounded to float32 (zeros elsewhere).

Capacity: at most K (max_age + 1) tracks of a class are alive after a frame (each frame updates or creates at most K), so
a class's list never exceeds that bound; the GPU tracker refuses a setting where it passes 1024.

``MatrixSort`` is a literal matrix-form SORT (numpy filter, ``iou_batch``, scipy assignment, per class): what the restatement
is checked against, and the host baseline the video benchmark times.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

# per block (cx, vcx), (cy, vcy), (s, vs): process noise of position and velocity, measurement noise; and of the scalar r
_QP, _QV, _R = (1.0, 1.0, 1.0), (0.01, 0.01, 1e-4), (1.0, 1.0, 10.0)
_QR, _RR = 1.0, 10.0
_P0, _V0 = 10.0, 10000.0


# -- scipy's linear_sum_assignment ---------------------------------------------------------------------------------------------
def lsap(cost) -> tuple:
    """(rows, cols) of scipy.optimize.linear_sum_assignment(cost), exactly (ties included)."""
    c = np.asarray(cost, np.float64)
    nr, nc = c.shape
    if nr == 0 or nc == 0:
        return np.empty(0, np.int64), np.empty(0, np.int64)
    transpose = nc < nr
    if transpose:
        c = c.T
        nr, nc = nc, nr
    c = c.tolist()
    u, v = [0.0] * nr, [0.0] * nc
    path, col4row, row4col = [-1] * nc, [-1] * nr, [-1] * nc
    for cur in range(nr):
        spc = [math.inf] * nc
        SR, SC = [False] * nr, [False] * nc
        remaining = [nc - it - 1 for it in range(nc)]
        num = nc
        i, sink, min_val = cur, -1, 0.0
        while sink == -1:
            index, lowest = -1, math.inf
            SR[i] = True
            for it in range(num):
                j = remaining[it]
                r = min_val + c[i][j] - u[i] - v[j]
                if r < spc[j]:
                    path[j] = i
                    spc[j] = r
                if spc[j] < lowest or (spc[j] == lowest and row4col[j] == -1):
                    lowest = spc[j]
                    index = it
            min_val = lowest
            j = remaining[index]
            if row4col[j] == -1:
                sink = j
            else:
                i = row4col[j]
            SC[j] = True
            num -= 1
            remaining[index] = remaining[num]
        u[cur] += min_val
        for i in range(nr):
            if SR[i] and i != cur:
                u[i] += min_val - spc[col4row[i]]
        for j in range(nc):
            if SC[j]:
                v[j] -= min_val - spc[j]
        j = sink
        while True:
            i = path[j]
            row4col[j] = i
            col4row[i], j = j, col4row[i]
            if i == cur:
                break
    if transpose:
        order = sorted(range(nr), key=lambda k: col4row[k])
        return np.array([col4row[k] for k in order], np.int64), np.array(order, np.int64)
    return np.arange(nr, dtype=np.int64), np.array(col4row, np.int64)


# -- the filter, in scalar form --------------------------------------------------------------------------------------------------
def _predict2(blk, qp, qv):
    """(p, v, a, b, d) of one 2-state block after x = F x, P = F P F' + Q."""
    p, v, a, b, d = blk
    t = b + d
    return [p + v, v, ((a + b) + t) + qp, t, d + qv]


def _update2(blk, z, R):
    """(p, v, a, b, d) after the Joseph-form update with measurement z of p and noise R."""
    p, v, a, b, d = blk
    y = z - p
    S = a + R
    k0, k1 = a / S, b / S
    c = 1.0 - k0
    m = b - k1 * a
    n = d - k1 * b
    rk0 = R * k0
    return [p + k0 * y, v + k1 * y, (c * a) * c + rk0 * k0, c * m + rk0 * k1, (n - k1 * m) + (R * k1) * k1]


def _predict1(blk, q):
    r, pr = blk
    return [r, pr + q]


def _update1(blk, z, R):
    r, pr = blk
    S = pr + R
    k = pr / S
    c = 1.0 - k
    return [r + k * (z - r), (c * pr) * c + (R * k) * k]


def to_z(box):
    """SORT's convert_bbox_to_z: [x1, y1, x2, y2] -> (cx, cy, s, r)."""
    w = box[2] - box[0]
    h = box[3] - box[1]
    return box[0] + w / 2.0, box[1] + h / 2.0, w * h, w / h


def to_box(cx, cy, s, r):
    """SORT's convert_x_to_bbox: -> [x1, y1, x2, y2]."""
    with np.errstate(all="ignore"):       # IEEE results (NaN, inf) where Python's math would raise
        w = float(np.sqrt(np.float64(s * r)))
        h = float(np.float64(s) / np.float64(w))
    return [cx - w / 2.0, cy - h / 2.0, cx + w / 2.0, cy + h / 2.0]


class ScalarKalman:
    """SORT's KalmanBoxTracker filter in block form: blocks[0..2] are (p, v, a, b, d) of cx, cy, s; rblk is (r, P_rr)."""

    def __init__(self, box):
        cx, cy, s, r = to_z(box)
        self.blocks = [[cx, 0.0, _P0, 0.0, _V0], [cy, 0.0, _P0, 0.0, _V0], [s, 0.0, _P0, 0.0, _V0]]
        self.rblk = [r, _P0]

    def predict(self):
        sb = self.blocks[2]
        if sb[1] + sb[0] <= 0:
            sb[1] *= 0.0
        self.blocks = [_predict2(b, _QP[k], _QV[k]) for k, b in enumerate(self.blocks)]
        self.rblk = _predict1(self.rblk, _QR)

    def update(self, box):
        z = to_z(box)
        self.blocks = [_update2(b, z[k], _R[k]) for k, b in enumerate(self.blocks)]
        self.rblk = _update1(self.rblk, z[3], _RR)

    def state(self):
        """x as SORT orders it: [cx, cy, s, r, vcx, vcy, vs]."""
        b = self.blocks
        return [b[0][0], b[1][0], b[2][0], self.rblk[0], b[0][1], b[1][1], b[2][1]]

    def box(self):
        b = self.blocks
        return to_box(b[0][0], b[1][0], b[2][0], self.rblk[0])


# -- SORT, per class, per record ------------------------------------------------------------------------------------------------
def _mx(a, b):
    return a if (a >= b or a != a) else b


def _mn(a, b):
    return a if (a <= b or a != a) else b


def iou(d, t) -> float:
    """SORT's iou_batch for one pair, 0 where the union is not > 0."""
    w = _mx(0.0, _mn(d[2], t[2]) - _mx(d[0], t[0]))
    h = _mx(0.0, _mn(d[3], t[3]) - _mx(d[1], t[1]))
    wh = w * h
    union = ((d[2] - d[0]) * (d[3] - d[1]) + (t[2] - t[0]) * (t[3] - t[1])) - wh
    return wh / union if union > 0 else 0.0


def associate(dets, trks, thresh):
    """SORT's associate_detections_to_trackers: (matches [(d, t)], detections to be born in birth order)."""
    D, T = len(dets), len(trks)
    if T == 0 or D == 0:
        return [], list(range(D))
    m = [[iou(d, t) for t in trks] for d in dets]
    above = [[v > thresh for v in row] for row in m]
    rows = [sum(r) for r in above]
    cols = [sum(above[i][j] for i in range(D)) for j in range(T)]
    if max(rows) == 1 and max(cols) == 1:
        pairs = [(i, j) for i in range(D) for j in range(T) if above[i][j]]
    else:
        r, c = lsap([[-v for v in row] for row in m])
        pairs = list(zip(r.tolist(), c.tolist()))
    touched = {i for i, _ in pairs}
    born = [i for i in range(D) if i not in touched]
    matches = []
    for i, j in pairs:
        if m[i][j] < thresh:
            born.append(i)
        else:
            matches.append((i, j))
    return matches, born


class _Track:
    __slots__ = ("kf", "id", "hits", "hit_streak", "time_since_update", "age")

    def __init__(self, box, kf_cls):
        self.kf = kf_cls(box)
        self.id = -1
        self.hits = self.hit_streak = self.time_since_update = self.age = 0


class Sort:
    """The tracker of one stream over C classes of at most K records.  ``update(position, boxes, counts)`` takes one frame:
    `boxes` float32 [C, K, 4] (ymin, xmin, ymax, xmax) and `counts` [C]; returns (ids int32 [C, K], boxes float32 [C, K, 4])."""

    kf_cls = ScalarKalman

    def __init__(self, C: int, K: int, max_age: int = 1, min_hits: int = 3, iou_thresh: float = 0.3):
        self.C, self.K = int(C), int(K)
        self.max_age, self.min_hits, self.iou_thresh = int(max_age), int(min_hits), float(iou_thresh)
        self.reset()

    def reset(self) -> None:
        self.tracks: List[List[_Track]] = [[] for _ in range(self.C)]
        self.frame_count = 0
        self.last_position: Optional[int] = None
        self.next_id = 1

    def _associate(self, dets, trk_boxes):
        return associate(dets, trk_boxes, self.iou_thresh)

    def _reported(self, t: _Track) -> bool:
        return t.time_since_update < 1 and (t.hit_streak >= self.min_hits or self.frame_count <= self.min_hits)

    def _predict(self, c: int) -> list:
        keep, boxes = [], []
        for t in self.tracks[c]:
            t.kf.predict()
            t.age += 1
            if t.time_since_update > 0:
                t.hit_streak = 0
            t.time_since_update += 1
            b = t.kf.box()
            if not any(v != v for v in b):
                keep.append(t)
                boxes.append(b)
        self.tracks[c] = keep
        return boxes

    def _remove_dead(self, c: int) -> None:
        self.tracks[c] = [t for t in self.tracks[c] if t.time_since_update <= self.max_age]

    def _empty_update(self) -> None:
        self.frame_count += 1
        for c in range(self.C):
            self._predict(c)
            self._remove_dead(c)

    def update(self, position: int, boxes, counts):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                self._empty_update()
        self.last_position = position
        self.frame_count += 1
        boxes = np.asarray(boxes, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)

        def emit(c, k, t):
            if self._reported(t):
                ids[c, k] = t.id
                x1, y1, x2, y2 = t.kf.box()
                out[c, k] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)

        for c in range(self.C):
            trk_boxes = self._predict(c)
            dets, det_k = [], []
            for k in range(int(counts[c])):
                ymin, xmin, ymax, xmax = (float(v) for v in boxes[c, k])
                if xmax - xmin > 0 and ymax - ymin > 0:
                    dets.append([xmin, ymin, xmax, ymax])
                    det_k.append(k)
            matches, born = self._associate(dets, trk_boxes)
            trks = self.tracks[c]
            for d, j in matches:
                t = trks[j]
                t.time_since_update = 0
                t.hits += 1
                t.hit_streak += 1
                t.kf.update(dets[d])
            for d, j in matches:
                emit(c, det_k[d], trks[j])
            self._remove_dead(c)
            for d in born:
                t = _Track(dets[d], self.kf_cls)
                t.id = self.next_id
                self.next_id += 1
                self.tracks[c].append(t)
                emit(c, det_k[d], t)
        return ids, out


# -- literal matrix-form SORT ---------------------------------------------------------------------------------------------------
class MatrixKalman:
    """SORT's KalmanBoxTracker filter as filterpy runs it: 7x7 matrices, predict P = F P F' + Q, Joseph-form update."""
    F = np.eye(7)
    F[0, 4] = F[1, 5] = F[2, 6] = 1.0
    H = np.eye(4, 7)
    R = np.diag([1.0, 1.0, 10.0, 10.0])
    Q = np.diag([1.0, 1.0, 1.0, 1.0, 0.01, 0.01, 1e-4])
    P0 = np.diag([10.0, 10.0, 10.0, 10.0, 1e4, 1e4, 1e4])

    def __init__(self, box):
        self.x = np.zeros((7, 1))
        self.x[:4, 0] = to_z(box)
        self.P = self.P0.copy()

    def predict(self):
        if self.x[6, 0] + self.x[2, 0] <= 0:
            self.x[6, 0] *= 0.0
        self.x = self.F @ self.x
        self.P = self.F @ self.P @ self.F.T + self.Q

    def update(self, box):
        z = np.array(to_z(box)).reshape(4, 1)
        y = z - self.H @ self.x
        PHT = self.P @ self.H.T
        S = self.H @ PHT + self.R
        K = PHT @ np.linalg.inv(S)
        self.x = self.x + K @ y
        I_KH = np.eye(7) - K @ self.H
        self.P = I_KH @ self.P @ I_KH.T + K @ self.R @ K.T

    def state(self):
        return self.x[:, 0].tolist()

    def box(self):
        x = self.x[:, 0]
        with np.errstate(invalid="ignore", divide="ignore"):
            w = np.sqrt(x[2] * x[3])
            h = x[2] / w
        return [x[0] - w / 2.0, x[1] - h / 2.0, x[0] + w / 2.0, x[1] + h / 2.0]


def iou_batch(bb_test, bb_gt):
    """SORT's iou_batch, with the union-not->-0 deviation."""
    bb_gt = np.expand_dims(bb_gt, 0)
    bb_test = np.expand_dims(bb_test, 1)
    xx1 = np.maximum(bb_test[..., 0], bb_gt[..., 0])
    yy1 = np.maximum(bb_test[..., 1], bb_gt[..., 1])
    xx2 = np.minimum(bb_test[..., 2], bb_gt[..., 2])
    yy2 = np.minimum(bb_test[..., 3], bb_gt[..., 3])
    w = np.maximum(0., xx2 - xx1)
    h = np.maximum(0., yy2 - yy1)
    wh = w * h
    union = ((bb_test[..., 2] - bb_test[..., 0]) * (bb_test[..., 3] - bb_test[..., 1])
             + (bb_gt[..., 2] - bb_gt[..., 0]) * (bb_gt[..., 3] - bb_gt[..., 1]) - wh)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(union > 0, wh / np.where(union > 0, union, 1.0), 0.0)


class MatrixTrack:
    """sort.py's KalmanBoxTracker over ``MatrixKalman``: predict / update / get_state and the life-cycle counters.  `id` is
    the stream's counter before the birth (0-based, as sort.py's class counter), reported as id + 1."""

    def __init__(self, bbox, id_):
        self.kf = MatrixKalman(bbox)
        self.time_since_update = 0
        self.id = id_
        self.hits = 0
        self.hit_streak = 0
        self.age = 0

    def update(self, bbox):
        self.time_since_update = 0
        self.hits += 1
        self.hit_streak += 1
        self.kf.update(bbox)

    def predict(self):
        self.kf.predict()
        self.age += 1
        if self.time_since_update > 0:
            self.hit_streak = 0
        self.time_since_update += 1
        return self.kf.box()

    def get_state(self):
        return self.kf.box()


def associate_detections_to_trackers(detections, trackers, iou_threshold=0.3):
    """sort.py's function, with ``iou_batch`` above and scipy's linear_sum_assignment."""
    from scipy.optimize import linear_sum_assignment
    if len(trackers) == 0:
        return np.empty((0, 2), dtype=int), np.arange(len(detections)), np.empty((0, 5), dtype=int)
    iou_matrix = iou_batch(detections, trackers)
    if min(iou_matrix.shape) > 0:
        a = (iou_matrix > iou_threshold).astype(np.int32)
        if a.sum(1).max() == 1 and a.sum(0).max() == 1:
            matched_indices = np.stack(np.where(a), axis=1)
        else:
            matched_indices = np.stack(linear_sum_assignment(-iou_matrix), axis=1)
    else:
        matched_indices = np.empty(shape=(0, 2), dtype=int)
    unmatched_detections = [d for d in range(len(detections)) if d not in matched_indices[:, 0]]
    unmatched_trackers = [t for t in range(len(trackers)) if t not in matched_indices[:, 1]]
    matches = []
    for m in matched_indices:
        if iou_matrix[m[0], m[1]] < iou_threshold:
            unmatched_detections.append(m[0])
            unmatched_trackers.append(m[1])
        else:
            matches.append(m.reshape(1, 2))
    matches = np.concatenate(matches, axis=0) if matches else np.empty((0, 2), dtype=int)
    return matches, np.array(unmatched_detections, dtype=int), np.array(unmatched_trackers, dtype=int)


class MatrixSort:
    """SORT as published, written independently of ``Sort``: sort.py's Sort.update loop run per class (predict every
    tracker, delete those predicting NaN, associate, update the matched, append the births, then walk the list in reverse
    to report and pop the dead), with ``MatrixTrack`` and ``associate_detections_to_trackers``.  Its own additions are
    only what a per-record output needs: each record remembers the tracker it updated or created, and is given that
    tracker's id + 1 and state box when the reverse walk reports it.  One difference from sort.py: a tracker is dropped
    before association only for a NaN in its predicted box, as sort.py's to_del does; sort.py's masked_invalid would also
    drop an infinite row from the matrix without dropping its tracker, which misaligns the two.  Same interface as ``Sort``."""

    def __init__(self, C: int, K: int, max_age: int = 1, min_hits: int = 3, iou_thresh: float = 0.3):
        self.C, self.K = int(C), int(K)
        self.max_age, self.min_hits, self.iou_threshold = int(max_age), int(min_hits), float(iou_thresh)
        self.reset()

    def reset(self) -> None:
        self.trackers: List[List[MatrixTrack]] = [[] for _ in range(self.C)]
        self.frame_count = 0
        self.count = 0
        self.last_position: Optional[int] = None

    def _update_class(self, c: int, dets: np.ndarray):
        """sort.py's Sort.update body for class c; returns ({det: tracker}, the trackers reported, by id())."""
        trackers = self.trackers[c]
        trks = np.zeros((len(trackers), 5))
        to_del = []
        for t, trk in enumerate(trks):
            pos = trackers[t].predict()
            trk[:] = [pos[0], pos[1], pos[2], pos[3], 0]
            if np.any(np.isnan(pos)):
                to_del.append(t)
        trks = np.delete(trks, to_del, axis=0)
        for t in reversed(to_del):
            trackers.pop(t)
        matched, unmatched_dets, unmatched_trks = associate_detections_to_trackers(dets, trks[:, :4], self.iou_threshold)
        owner = {}
        for m in matched:
            trackers[m[1]].update(dets[m[0], :])
            owner[int(m[0])] = trackers[m[1]]
        for i in unmatched_dets:
            trk = MatrixTrack(dets[i, :], self.count)
            self.count += 1
            trackers.append(trk)
            owner[int(i)] = trk
        reported = set()
        i = len(trackers)
        for trk in reversed(trackers):
            if trk.time_since_update < 1 and (trk.hit_streak >= self.min_hits or self.frame_count <= self.min_hits):
                reported.add(id(trk))
            i -= 1
            if trk.time_since_update > self.max_age:
                trackers.pop(i)
        return owner, reported

    def update(self, position: int, boxes, counts):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                self.frame_count += 1
                for c in range(self.C):
                    self._update_class(c, np.empty((0, 4)))
        self.last_position = position
        self.frame_count += 1
        boxes = np.asarray(boxes, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)
        for c in range(self.C):
            k_of = [k for k in range(int(counts[c]))
                    if float(boxes[c, k, 3]) - float(boxes[c, k, 1]) > 0 and float(boxes[c, k, 2]) - float(boxes[c, k, 0]) > 0]
            dets = boxes[c, k_of][:, [1, 0, 3, 2]].astype(np.float64).reshape(-1, 4)
            owner, reported = self._update_class(c, dets)
            for d, trk in owner.items():
                if id(trk) in reported:
                    x1, y1, x2, y2 = trk.get_state()
                    ids[c, k_of[d]] = trk.id + 1
                    out[c, k_of[d]] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)
        return ids, out
