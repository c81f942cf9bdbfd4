"""OC-SORT (Cao et al., CVPR 2023, "Observation-Centric SORT: Rethinking SORT for Robust Multi-Object Tracking") restated in
plain Python: the rules the GPU tracker (``k2y_ocsort_update``, csrc/ocsort.cu) follows bit for bit.  ``OCSort.update`` of the
published ocsort.py with its IoU association (GIoU, DIoU, CIoU and centre distance are not restated), written from the
published algorithm and code without a copy at hand to compare against; every rule the outcome depends on is listed below,
and where the published code leaves room the rule says so and states the choice.  What SORT already fixes is taken from
oracle/sort_ref.py and not repeated: the block-form filter (``_predict2`` / ``_update2`` / ``_predict1`` / ``_update1`` with
SORT's Q, R and P0, which OC-SORT's KalmanBoxTracker sets the same way), ``lsap`` standing in for lap's
``lapjv(extend_cost=True)``, ``iou`` (no "+1", 0 where the union is not > 0), the state box w = sqrt(s r), h = s / w, one
id counter per stream in (frame, class, birth) order, dropped frames run as updates without detections, and a track whose
predicted box has a NaN deleted before association.

* Setting: ``det_thresh`` 0.6, ``max_age`` 30, ``min_hits`` 3, ``iou_thresh`` 0.3, ``delta_t`` 3, ``inertia`` 0.2,
  ``use_byte`` False.  Per class and per stream, as SORT here.
* Detections, in record order.  Choice: a record is a detection only when its four coordinates are finite and its width
  and height are > 0 (SORT's filter, plus finiteness: a non-finite box gives a NaN direction term, which scipy's assignment
  refuses).  The float32 score is widened to float64.  High: score > det_thresh; with ``use_byte`` a record is low when
  0.1 < score < det_thresh.  A detection is the float64 (x1, y1, x2, y2, score).  Only high detections are born.
* Boxes: z = (cx, cy, w h, w / (h + 1e-6)) with cx = x1 + w / 2.0 (OC-SORT adds the 1e-6 SORT's z lacks).  Before the
  filter's predict the tracker sets vs *= 0.0 when vs + s <= 0 (SORT's quirk, kept; it belongs to the tracker's predict,
  and ORU's own predicts do not apply it).
* Per-track observations.  ``last_observation`` starts as the sentinel (-1, -1, -1, -1, -1); a newborn does not store its
  birth box there.  ``observations`` maps age to the detection; ``velocity`` is None until set.  k_previous_obs(age, delta_t)
  is the observation stored at age - dt for the first dt from delta_t down to 1, else the newest stored observation, else
  the sentinel.  The newest stored observation is always ``last_observation`` (both are set together, ages increase), so
  the restatement keeps a ring of delta_t (age, detection) slots indexed by age mod delta_t (the ages looked up, age -
  delta_t .. age - 1, fall in distinct slots, and an overwritten slot only held an age below them) and falls back to
  ``last_observation``.  On a matched update, first, when ``last_observation``'s five values summed left to right are >= 0
  (a quirk, kept: numpy's sum of five values is that loop), the velocity becomes speed_direction(previous, detection), with
  previous the observation at age - dt for the first dt from delta_t down to 1, else ``last_observation``; speed_direction is
  the unit (dy, dx) between the centres ((x1 + x2) / 2.0, (y1 + y2) / 2.0), norm sqrt(dy dy + dx dx) + 1e-6.  Then
  ``last_observation`` and observations[age] are set, hits and hit_streak count, time_since_update = 0, and the filter
  takes z.
* ORU, observation-centric re-update (the published KalmanFilterNew's freeze / unfreeze), the rule most likely to be
  questioned.  The filter keeps the history of what each update call was given (z or None, one entry per frame after the
  birth), and whether it is observed; a newborn is not.  An update without a detection of an observed filter freezes a
  copy of its state (x and P after that frame's predict, with the history up to it) and makes it unobserved.  The next
  update with a detection, when a frozen copy exists, restores it, and with box1 the last z in the history before the
  loss, box2 the new z, w = sqrt(s r) and h = sqrt(s / r) of each, gap the frames between the two, and d* = (box2 -
  box1) / gap for x, y, w and h, it runs for i = 1..gap an update with the virtual z (x1 + i dx, y1 + i dy, w h, w / h)
  (w = w1 + i dw, h = h1 + i dh), with the filter's own predict between the steps but not after the last.  Then the real
  update with box2 runs on top, as the published code does: the new observation is applied twice.  The restored history
  takes the virtual boxes in place of the lost frames, and the real z is not appended, so after a re-update "the last z in
  the history" is the last virtual box, (x1 + gap dx, ...), not box2: a second loss right after replays from there.
* Association round 1 (OCM, observation-centric momentum): rows are the high detections, columns the predicted tracks.
  iou[d][t] on the predicted box; angle[d][t] from v_t = the track's velocity or (0, 0) and u = the unit direction
  (same + 1e-6 norm) from the centre of k_previous_obs to the detection's centre: c = clip(v.x u.x + v.y u.y, -1, 1),
  angle = (pi / 2.0 - |acos(c)|) / pi, times 0 for a track whose k-previous observation is the sentinel (its score field
  < 0), then times ``inertia``, then times the detection's score.  When every row and column of (iou > iou_thresh) has at
  most one entry and some entry is set, those pairs in row-major order; otherwise lsap(-(iou + angle)).  A match with
  iou < iou_thresh is dropped.  Unmatched detections and tracks come in SORT's order: those no pair touched ascending, then
  the dropped pairs' in match order.
* Round 2 (BYTE, only with ``use_byte``), when low detections and unmatched tracks exist: low detections x the unmatched
  tracks' predicted boxes; when the largest IoU is > iou_thresh, lsap(-iou), skipping pairs with iou < iou_thresh; the
  unmatched tracks then become sorted ascending (np.setdiff1d).
* Round 3 (OCR, observation-centric recovery), when unmatched high detections and tracks both exist: those detections x the
  tracks' ``last_observation`` (the sentinel included, whose area is 0); when the largest IoU is > iou_thresh, lsap(-iou),
  skipping pairs with iou < iou_thresh; both lists then become sorted ascending, which decides the birth order and so the
  ids.
* Life cycle: the tracks still unmatched update without a detection; a track is removed when time_since_update >
  max_age (before the births are appended: the same lists, as in sort_ref); the unmatched high detections are born in
  list order.  A track is reported when time_since_update < 1 and (hit_streak >= min_hits or frame_count <= min_hits).
* Output per record: the id of the track the record updated (in any round) or created, when that track is reported, with
  OC-SORT's box: ``last_observation[:4]`` when its sum is >= 0 (normally the record's own box, exactly), else the
  filter's state box (a newborn reported while frame_count <= min_hits, or a box at negative coordinates), as float32
  (ymin, xmin, ymax, xmax); -1 and zeros elsewhere.
* acos.  ``math.acos`` / ``np.arccos`` are not guaranteed to give the GPU's result, so ``acos`` below is fdlibm's
  ``__ieee754_acos`` written out from its algorithm and published coefficients: only +, -, *, / and sqrt in a fixed order,
  and word manipulations (``struct`` here, ``__double_as_longlong`` / ``__hiloint2double`` on the GPU), so the direction term
  is the same on both sides, bit for bit.  It is within 1 ulp of ``math.acos``; the literal form's ``np.arccos`` is too, and
  may differ from it in the last bit, which can only swap which of two identical records carries a track.

Capacity.  Each record updates at most one track (the three rounds take disjoint tracks, and a record is high or low) or
is born, so each frame leaves at most K tracks of a class with time_since_update 0; a track lives while time_since_update
<= max_age, so at most K (max_age + 1) tracks of a class are alive after a frame, and, dead tracks removed before the
births, within one.  The GPU tracker refuses a setting past 4096 tracks per class (ByteTrack's cap): max_age 30 gives 930
at K = 30 and 3100 at K = 100.  delta_t sizes every track's ring of observations, 48 bytes a slot; it is capped at 8
(OC-SORT's default is 3), which keeps a track's state under 1 KB.

``MatrixOcSort`` is a literal form: numpy 7x7 filter matrices with filterpy's Joseph-form update, freeze / unfreeze with an
actual state copy and a ``history_obs`` list, ``np.arccos``, dict observations, and ocsort.py's lists and ``np.setdiff1d``;
the restatement is checked against it.
"""
from __future__ import annotations

import copy
import math
import struct
from typing import List, Optional

import numpy as np

from .sort_ref import _P0, _QP, _QR, _QV, _R, _RR, _V0, MatrixKalman, _predict1, _predict2, _update1, _update2, iou, lsap, \
    to_box

SENTINEL = (-1.0, -1.0, -1.0, -1.0, -1.0)
LOW_THRESH = 0.1
DELTA_T_MAX = 8
MAX_TRACKS_PER_CLASS = 4096


def max_tracks(K: int, max_age: int) -> int:
    """Tracks one class holds after a frame, and within one (module docstring, Capacity)."""
    return int(K) * (int(max_age) + 1)


# -- fdlibm's acos ---------------------------------------------------------------------------------------------------------------
_PI, _PIO2_HI, _PIO2_LO = 3.14159265358979311600e+00, 1.57079632679489655800e+00, 6.12323399573676603587e-17
_PS = (1.66666666666666657415e-01, -3.25565818622400915405e-01, 2.01212532134862925881e-01, -4.00555345006794114027e-02,
       7.91534994289814532176e-04, 3.47933107596021167570e-05)
_QS = (-2.40339491173441421878e+00, 2.02094576023350569471e+00, -6.88283971605453293030e-01, 7.70381505559019352791e-02)


def _words(x: float):
    """(high word as a signed int32, low word as uint32) of the double x."""
    u = struct.unpack("<Q", struct.pack("<d", x))[0]
    hi = u >> 32
    return (hi - (1 << 32) if hi & 0x80000000 else hi), u & 0xffffffff


def _hi_only(x: float) -> float:
    """x with its low word cleared."""
    u = struct.unpack("<Q", struct.pack("<d", x))[0]
    return struct.unpack("<d", struct.pack("<Q", u & 0xffffffff00000000))[0]


def _pq(z: float) -> float:
    p = z * (_PS[0] + z * (_PS[1] + z * (_PS[2] + z * (_PS[3] + z * (_PS[4] + z * _PS[5])))))
    q = 1.0 + z * (_QS[0] + z * (_QS[1] + z * (_QS[2] + z * _QS[3])))
    return p / q


def acos(x: float) -> float:
    """fdlibm's __ieee754_acos."""
    hx, lx = _words(x)
    ix = hx & 0x7fffffff
    if ix >= 0x3ff00000:                                    # |x| >= 1
        if ((ix - 0x3ff00000) | lx) == 0:
            return 0.0 if hx > 0 else _PI + 2.0 * _PIO2_LO
        return math.nan
    if ix < 0x3fe00000:                                     # |x| < 0.5
        if ix <= 0x3c600000:
            return _PIO2_HI + _PIO2_LO
        r = _pq(x * x)
        return _PIO2_HI - (x - (_PIO2_LO - x * r))
    if hx < 0:                                              # x <= -0.5
        z = (1.0 + x) * 0.5
        s = math.sqrt(z)
        r = _pq(z)
        w = r * s - _PIO2_LO
        return _PI - 2.0 * (s + w)
    z = (1.0 - x) * 0.5                                     # x >= 0.5
    s = math.sqrt(z)
    df = _hi_only(s)
    c = (z - df * df) / (s + df)
    r = _pq(z)
    w = r * s + c
    return 2.0 * (df + w)


# -- boxes and directions --------------------------------------------------------------------------------------------------------
def to_z(box):
    """OC-SORT's convert_bbox_to_z: [x1, y1, x2, y2, ...] -> (cx, cy, s, r)."""
    w = box[2] - box[0]
    h = box[3] - box[1]
    return box[0] + w / 2.0, box[1] + h / 2.0, w * h, w / (h + 1e-6)


def _sum5(o) -> float:
    return (((o[0] + o[1]) + o[2]) + o[3]) + o[4]


def speed_direction(b1, b2):
    """The unit (dy, dx) from the centre of b1 to that of b2."""
    cx1, cy1 = (b1[0] + b1[2]) / 2.0, (b1[1] + b1[3]) / 2.0
    cx2, cy2 = (b2[0] + b2[2]) / 2.0, (b2[1] + b2[3]) / 2.0
    dy, dx = cy2 - cy1, cx2 - cx1
    norm = math.sqrt(dy * dy + dx * dx) + 1e-6
    return dy / norm, dx / norm


def angle_term(det, prev, velocity, inertia: float) -> float:
    """Round 1's direction term of detection `det` for a track with k-previous observation `prev` and `velocity`."""
    vy, vx = velocity if velocity is not None else (0.0, 0.0)
    uy, ux = speed_direction(prev, det)
    c = vx * ux + vy * uy
    c = -1.0 if c < -1.0 else (1.0 if c > 1.0 else c)
    a = (math.pi / 2.0 - abs(acos(c))) / math.pi
    valid = 0.0 if prev[4] < 0 else 1.0
    return ((valid * a) * inertia) * det[4]


# -- the filter with ORU ---------------------------------------------------------------------------------------------------------
class OcKalman:
    """SORT's block filter (sort_ref) with OC-SORT's observation history and freeze / restore."""

    def __init__(self, box):
        cx, cy, s, r = to_z(box)
        self.blocks = [[cx, 0.0, _P0, 0.0, _V0], [cy, 0.0, _P0, 0.0, _V0], [s, 0.0, _P0, 0.0, _V0]]
        self.rblk = [r, _P0]
        self.observed = False
        self.frozen = None
        self.n_hist = 0             # update calls so far: the length of the published history_obs
        self.last_z = None          # the history's last z, and its index
        self.last_i = -1

    def predict(self):
        self.blocks = [_predict2(b, _QP[k], _QV[k]) for k, b in enumerate(self.blocks)]
        self.rblk = _predict1(self.rblk, _QR)

    def _update(self, z):
        self.blocks = [_update2(b, z[k], _R[k]) for k, b in enumerate(self.blocks)]
        self.rblk = _update1(self.rblk, z[3], _RR)

    def update(self, z):
        i = self.n_hist
        self.n_hist += 1
        if z is None:
            if self.observed:
                self.frozen = ([list(b) for b in self.blocks], list(self.rblk))
                self.observed = False
            return
        if not self.observed and self.frozen is not None:
            self.blocks, self.rblk = self.frozen
            self.frozen = None
            gap = i - self.last_i
            x1, y1, s1, r1 = self.last_z
            x2, y2, s2, r2 = z
            w1, h1 = math.sqrt(s1 * r1), math.sqrt(s1 / r1)
            w2, h2 = math.sqrt(s2 * r2), math.sqrt(s2 / r2)
            dx, dy, dw, dh = (x2 - x1) / gap, (y2 - y1) / gap, (w2 - w1) / gap, (h2 - h1) / gap
            for k in range(gap):
                f = float(k + 1)
                w, h = w1 + f * dw, h1 + f * dh
                vz = (x1 + f * dx, y1 + f * dy, w * h, w / h)
                self._update(vz)
                if k != gap - 1:
                    self.predict()
            self.last_z = vz
        else:
            self.last_z = z
        self.last_i = i
        self.observed = True
        self._update(z)

    def state(self):
        b = self.blocks
        return [b[0][0], b[1][0], b[2][0], self.rblk[0], b[0][1], b[1][1], b[2][1]]

    def box(self):
        b = self.blocks
        return to_box(b[0][0], b[1][0], b[2][0], self.rblk[0])


class _Track:
    __slots__ = ("kf", "id", "hits", "hit_streak", "time_since_update", "age", "last_obs", "ring", "velocity", "delta_t")

    def __init__(self, det, delta_t):
        self.kf = OcKalman(det)
        self.id = -1
        self.hits = self.hit_streak = self.time_since_update = self.age = 0
        self.last_obs = SENTINEL
        self.ring = [(-1, None)] * delta_t         # (age, detection) at slot age % delta_t
        self.velocity = None
        self.delta_t = delta_t

    def predict(self):
        sb = self.kf.blocks[2]
        if sb[1] + sb[0] <= 0:
            sb[1] *= 0.0
        self.kf.predict()
        self.age += 1
        if self.time_since_update > 0:
            self.hit_streak = 0
        self.time_since_update += 1
        return self.kf.box()

    def _stored(self, age):
        a, o = self.ring[age % self.delta_t]
        return o if a == age else None

    def k_previous_obs(self):
        for dt in range(self.delta_t, 0, -1):
            o = self._stored(self.age - dt)
            if o is not None:
                return o
        return self.last_obs

    def update(self, det):
        if det is None:
            self.kf.update(None)
            return
        if _sum5(self.last_obs) >= 0:
            self.velocity = speed_direction(self.k_previous_obs(), det)
        self.last_obs = det
        self.ring[self.age % self.delta_t] = (self.age, det)
        self.time_since_update = 0
        self.hits += 1
        self.hit_streak += 1
        self.kf.update(to_z(det))

    def out_box(self):
        return list(self.last_obs[:4]) if _sum5(self.last_obs) >= 0 else self.kf.box()


def detections(boxes_c, count, scores_c, det_thresh, use_byte):
    """(high, low) detections of one class's records: lists of ((x1, y1, x2, y2, score), record), record order."""
    high, low = [], []
    for k in range(int(count)):
        ymin, xmin, ymax, xmax = (float(v) for v in boxes_c[k])
        if not all(math.isfinite(v) for v in (ymin, xmin, ymax, xmax)) or not (xmax - xmin > 0 and ymax - ymin > 0):
            continue
        s = float(scores_c[k])
        if s > det_thresh:
            high.append(((xmin, ymin, xmax, ymax, s), k))
        elif use_byte and LOW_THRESH < s < det_thresh:
            low.append(((xmin, ymin, xmax, ymax, s), k))
    return high, low


def associate(dets, trk_boxes, prevs, velocities, thresh, inertia):
    """Round 1: (matches [(d, t)], unmatched detections, unmatched tracks), each in OC-SORT's order."""
    D, T = len(dets), len(trk_boxes)
    if T == 0:
        return [], list(range(D)), []
    if D == 0:
        return [], [], list(range(T))
    m = [[iou(d, t) for t in trk_boxes] for d in dets]
    above = [[v > thresh for v in row] for row in m]
    rows = [sum(r) for r in above]
    cols = [sum(above[i][j] for i in range(D)) for j in range(T)]
    if max(rows) == 1 and max(cols) == 1:
        pairs = [(i, j) for i in range(D) for j in range(T) if above[i][j]]
    else:
        cost = [[-(m[i][j] + angle_term(dets[i], prevs[j], velocities[j], inertia)) for j in range(T)] for i in range(D)]
        r, c = lsap(cost)
        pairs = list(zip(r.tolist(), c.tolist()))
    td, tt = {i for i, _ in pairs}, {j for _, j in pairs}
    ud, ut = [i for i in range(D) if i not in td], [j for j in range(T) if j not in tt]
    matches = []
    for i, j in pairs:
        if m[i][j] < thresh:
            ud.append(i)
            ut.append(j)
        else:
            matches.append((i, j))
    return matches, ud, ut


def _rematch(dets, boxes, thresh):
    """Rounds 2 and 3: the pairs (d, t) of lsap(-iou) with iou >= thresh when the largest iou is > thresh, else None."""
    m = [[iou(d, b) for b in boxes] for d in dets]
    if not max(max(row) for row in m) > thresh:
        return None
    r, c = lsap([[-v for v in row] for row in m])
    return [(i, j) for i, j in zip(r.tolist(), c.tolist()) if not m[i][j] < thresh]


class OcSort:
    """OC-SORT of one stream over C classes of at most K records.  ``update(position, boxes, counts, scores)`` takes one frame:
    `boxes` float32 [C, K, 4] (ymin, xmin, ymax, xmax), `counts` [C] and `scores` float32 [C, K]; returns (ids int32 [C, K],
    boxes float32 [C, K, 4])."""

    def __init__(self, C: int, K: int, det_thresh: float = 0.6, max_age: int = 30, min_hits: int = 3,
                 iou_thresh: float = 0.3, delta_t: int = 3, inertia: float = 0.2, use_byte: bool = False):
        self.C, self.K = int(C), int(K)
        self.det_thresh, self.max_age, self.min_hits = float(det_thresh), int(max_age), int(min_hits)
        self.iou_thresh, self.delta_t, self.inertia, self.use_byte = float(iou_thresh), int(delta_t), float(inertia), bool(use_byte)
        self.reset()

    def reset(self) -> None:
        self.tracks: List[List[_Track]] = [[] for _ in range(self.C)]
        self.frame_count = 0
        self.last_position: Optional[int] = None
        self.next_id = 1

    def _reported(self, t: _Track) -> bool:
        return t.time_since_update < 1 and (t.hit_streak >= self.min_hits or self.frame_count <= self.min_hits)

    def _step(self, c: int, high, low) -> dict:
        """One frame of class c; returns {record: track}."""
        trks, boxes = [], []
        for t in self.tracks[c]:
            b = t.predict()
            if not any(v != v for v in b):
                trks.append(t)
                boxes.append(b)
        self.tracks[c] = trks
        dets = [d for d, _ in high]
        owner = {}
        matches, ud, ut = associate(dets, boxes, [t.k_previous_obs() for t in trks], [t.velocity for t in trks],
                                    self.iou_thresh, self.inertia)
        for i, j in matches:
            trks[j].update(dets[i])
            owner[high[i][1]] = trks[j]
        if self.use_byte and low and ut:
            pairs = _rematch([d for d, _ in low], [boxes[j] for j in ut], self.iou_thresh)
            if pairs is not None:
                for i, j in pairs:
                    trks[ut[j]].update(low[i][0])
                    owner[low[i][1]] = trks[ut[j]]
                gone = {ut[j] for _, j in pairs}
                ut = sorted(j for j in ut if j not in gone)
        if ud and ut:
            pairs = _rematch([dets[i] for i in ud], [trks[j].last_obs for j in ut], self.iou_thresh)
            if pairs is not None:
                for i, j in pairs:
                    trks[ut[j]].update(dets[ud[i]])
                    owner[high[ud[i]][1]] = trks[ut[j]]
                gd, gt = {ud[i] for i, _ in pairs}, {ut[j] for _, j in pairs}
                ud = sorted(i for i in ud if i not in gd)
                ut = sorted(j for j in ut if j not in gt)
        for j in ut:
            trks[j].update(None)
        self.tracks[c] = [t for t in trks if t.time_since_update <= self.max_age]
        for i in ud:
            t = _Track(dets[i], self.delta_t)
            t.id = self.next_id
            self.next_id += 1
            self.tracks[c].append(t)
            owner[high[i][1]] = t
        return owner

    def update(self, position: int, boxes, counts, scores):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                self.frame_count += 1
                for c in range(self.C):
                    self._step(c, [], [])
        self.last_position = position
        self.frame_count += 1
        boxes = np.asarray(boxes, np.float32)
        scores = np.asarray(scores, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)
        for c in range(self.C):
            high, low = detections(boxes[c], counts[c], scores[c], self.det_thresh, self.use_byte)
            for k, t in self._step(c, high, low).items():
                if self._reported(t):
                    x1, y1, x2, y2 = t.out_box()
                    ids[c, k] = t.id
                    out[c, k] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)
        return ids, out


# -- literal matrix form -------------------------------------------------------------------------------------------------------
class KalmanFilterNew:
    """The published KalmanFilterNew as OC-SORT's KalmanBoxTracker uses it: filterpy's 7x7 predict and Joseph-form update,
    the observation history, and freeze / unfreeze with a copy of the whole state."""
    F, H, R, Q, P0 = MatrixKalman.F, MatrixKalman.H, MatrixKalman.R, MatrixKalman.Q, MatrixKalman.P0

    def __init__(self, z):
        self.x = np.zeros((7, 1))
        self.x[:4] = z
        self.P = self.P0.copy()
        self.observed = False
        self.attr_saved = None
        self.history_obs = []

    def predict(self):
        self.x = self.F @ self.x
        self.P = self.F @ self.P @ self.F.T + self.Q

    def freeze(self):
        self.attr_saved = copy.deepcopy(self.__dict__)

    def unfreeze(self):
        if self.attr_saved is not None:
            new_history = copy.deepcopy(self.history_obs)
            self.__dict__ = self.attr_saved
            self.history_obs = self.history_obs[:-1]
            occur = [int(d is None) for d in new_history]
            indices = np.where(np.array(occur) == 0)[0]
            index1, index2 = indices[-2], indices[-1]
            x1, y1, s1, r1 = new_history[index1]
            w1, h1 = np.sqrt(s1 * r1), np.sqrt(s1 / r1)
            x2, y2, s2, r2 = new_history[index2]
            w2, h2 = np.sqrt(s2 * r2), np.sqrt(s2 / r2)
            time_gap = index2 - index1
            dx, dy = (x2 - x1) / time_gap, (y2 - y1) / time_gap
            dw, dh = (w2 - w1) / time_gap, (h2 - h1) / time_gap
            for i in range(index2 - index1):
                x, y = x1 + (i + 1) * dx, y1 + (i + 1) * dy
                w, h = w1 + (i + 1) * dw, h1 + (i + 1) * dh
                s, r = w * h, w / h
                self.update(np.array([x, y, s, r]).reshape((4, 1)))
                if not i == (index2 - index1 - 1):
                    self.predict()

    def update(self, z):
        self.history_obs.append(z)
        if z is None:
            if self.observed:
                self.freeze()
            self.observed = False
            return
        if not self.observed:
            self.unfreeze()
        self.observed = True
        y = z - self.H @ self.x
        PHT = self.P @ self.H.T
        S = self.H @ PHT + self.R
        K = PHT @ np.linalg.inv(S)
        self.x = self.x + K @ y
        I_KH = np.eye(7) - K @ self.H
        self.P = I_KH @ self.P @ I_KH.T + K @ self.R @ K.T


def convert_bbox_to_z(bbox):
    w = bbox[2] - bbox[0]
    h = bbox[3] - bbox[1]
    x = bbox[0] + w / 2.
    y = bbox[1] + h / 2.
    s = w * h
    r = w / float(h + 1e-6)
    return np.array([x, y, s, r]).reshape((4, 1))


def convert_x_to_bbox(x):
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.sqrt(x[2] * x[3])
        h = x[2] / w
    return np.array([x[0] - w / 2., x[1] - h / 2., x[0] + w / 2., x[1] + h / 2.]).reshape((1, 4))


def k_previous_obs(observations, cur_age, k):
    if len(observations) == 0:
        return [-1, -1, -1, -1, -1]
    for i in range(k):
        dt = k - i
        if cur_age - dt in observations:
            return observations[cur_age - dt]
    max_age = max(observations.keys())
    return observations[max_age]


def matrix_speed_direction(bbox1, bbox2):
    cx1, cy1 = (bbox1[0] + bbox1[2]) / 2.0, (bbox1[1] + bbox1[3]) / 2.0
    cx2, cy2 = (bbox2[0] + bbox2[2]) / 2.0, (bbox2[1] + bbox2[3]) / 2.0
    speed = np.array([cy2 - cy1, cx2 - cx1])
    norm = np.sqrt((cy2 - cy1) ** 2 + (cx2 - cx1) ** 2) + 1e-6
    return speed / norm


class KalmanBoxTracker:
    """ocsort.py's KalmanBoxTracker; `counter` is the stream's id counter (a list)."""

    def __init__(self, bbox, counter, delta_t=3):
        self.kf = KalmanFilterNew(convert_bbox_to_z(bbox))
        self.time_since_update = 0
        self.id = counter[0]
        counter[0] += 1
        self.hits = 0
        self.hit_streak = 0
        self.age = 0
        self.last_observation = np.array([-1, -1, -1, -1, -1])
        self.observations = dict()
        self.velocity = None
        self.delta_t = delta_t

    def update(self, bbox):
        if bbox is not None:
            if self.last_observation.sum() >= 0:
                previous_box = None
                for i in range(self.delta_t):
                    dt = self.delta_t - i
                    if self.age - dt in self.observations:
                        previous_box = self.observations[self.age - dt]
                        break
                if previous_box is None:
                    previous_box = self.last_observation
                self.velocity = matrix_speed_direction(previous_box, bbox)
            self.last_observation = bbox
            self.observations[self.age] = bbox
            self.time_since_update = 0
            self.hits += 1
            self.hit_streak += 1
            self.kf.update(convert_bbox_to_z(bbox))
        else:
            self.kf.update(bbox)

    def predict(self):
        if (self.kf.x[6] + self.kf.x[2]) <= 0:
            self.kf.x[6] *= 0.0
        self.kf.predict()
        self.age += 1
        if self.time_since_update > 0:
            self.hit_streak = 0
        self.time_since_update += 1
        return convert_x_to_bbox(self.kf.x)

    def get_state(self):
        return convert_x_to_bbox(self.kf.x)


def iou_batch(bb_test, bb_gt):
    from .sort_ref import iou_batch as sort_iou_batch
    return sort_iou_batch(np.asarray(bb_test)[:, :4], np.asarray(bb_gt)[:, :4])


def speed_direction_batch(dets, tracks):
    tracks = tracks[..., np.newaxis]
    CX1, CY1 = (dets[:, 0] + dets[:, 2]) / 2.0, (dets[:, 1] + dets[:, 3]) / 2.0
    CX2, CY2 = (tracks[:, 0] + tracks[:, 2]) / 2.0, (tracks[:, 1] + tracks[:, 3]) / 2.0
    dx = CX1 - CX2
    dy = CY1 - CY2
    norm = np.sqrt(dx ** 2 + dy ** 2) + 1e-6
    dx = dx / norm
    dy = dy / norm
    return dy, dx


def linear_assignment(cost_matrix):
    from scipy.optimize import linear_sum_assignment
    x, y = linear_sum_assignment(cost_matrix)
    return np.array(list(zip(x, y)))


def matrix_associate(detections, trackers, iou_threshold, velocities, previous_obs, vdc_weight):
    """ocsort.py's association.associate."""
    if len(trackers) == 0:
        return np.empty((0, 2), dtype=int), np.arange(len(detections)), np.empty((0, 5), dtype=int)
    Y, X = speed_direction_batch(detections, previous_obs)
    inertia_Y, inertia_X = velocities[:, 0], velocities[:, 1]
    inertia_Y = np.repeat(inertia_Y[:, np.newaxis], Y.shape[1], axis=1)
    inertia_X = np.repeat(inertia_X[:, np.newaxis], X.shape[1], axis=1)
    diff_angle_cos = inertia_X * X + inertia_Y * Y
    diff_angle_cos = np.clip(diff_angle_cos, a_min=-1, a_max=1)
    diff_angle = np.arccos(diff_angle_cos)
    diff_angle = (np.pi / 2.0 - np.abs(diff_angle)) / np.pi
    valid_mask = np.ones(previous_obs.shape[0])
    valid_mask[np.where(previous_obs[:, 4] < 0)] = 0
    iou_matrix = iou_batch(detections, trackers)
    scores = np.repeat(detections[:, -1][:, np.newaxis], trackers.shape[0], axis=1)
    valid_mask = np.repeat(valid_mask[:, np.newaxis], X.shape[1], axis=1)
    angle_diff_cost = (valid_mask * diff_angle) * vdc_weight
    angle_diff_cost = angle_diff_cost.T
    angle_diff_cost = angle_diff_cost * scores
    if min(iou_matrix.shape) > 0:
        a = (iou_matrix > iou_threshold).astype(np.int32)
        if a.sum(1).max() == 1 and a.sum(0).max() == 1:
            matched_indices = np.stack(np.where(a), axis=1)
        else:
            matched_indices = linear_assignment(-(iou_matrix + angle_diff_cost))
    else:
        matched_indices = np.empty(shape=(0, 2))
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
    return matches, np.array(unmatched_detections), np.array(unmatched_trackers)


class OCSortClass:
    """ocsort.py's OCSort.update for one class, on detections (x1, y1, x2, y2, score) with their records; returns ({record:
    tracker}, the trackers reported, by id())."""

    def __init__(self, det_thresh, max_age, min_hits, iou_threshold, delta_t, inertia, use_byte, counter):
        self.max_age, self.min_hits, self.iou_threshold = max_age, min_hits, iou_threshold
        self.trackers = []
        self.frame_count = 0
        self.det_thresh, self.delta_t, self.inertia, self.use_byte = det_thresh, delta_t, inertia, use_byte
        self.counter = counter

    def update(self, dets_all, recs):
        self.frame_count += 1
        scores = dets_all[:, 4]
        inds_low = scores > LOW_THRESH
        inds_high = scores < self.det_thresh
        inds_second = np.logical_and(inds_low, inds_high)
        dets_second, recs_second = dets_all[inds_second], recs[inds_second]
        remain_inds = scores > self.det_thresh
        dets, recs = dets_all[remain_inds], recs[remain_inds]
        owner = {}
        trks = np.zeros((len(self.trackers), 5))
        to_del = []
        for t, trk in enumerate(trks):
            pos = self.trackers[t].predict()[0]
            trk[:] = [pos[0], pos[1], pos[2], pos[3], 0]
            if np.any(np.isnan(pos)):
                to_del.append(t)
        trks = np.delete(trks, to_del, axis=0)          # sort_ref's choice: only a NaN row goes, with its tracker
        for t in reversed(to_del):
            self.trackers.pop(t)
        velocities = np.array([trk.velocity if trk.velocity is not None else np.array((0, 0)) for trk in self.trackers])
        last_boxes = np.array([trk.last_observation for trk in self.trackers])
        k_observations = np.array([k_previous_obs(trk.observations, trk.age, self.delta_t) for trk in self.trackers])
        matched, unmatched_dets, unmatched_trks = matrix_associate(dets, trks, self.iou_threshold, velocities, k_observations,
                                                                   self.inertia)
        for m in matched:
            self.trackers[m[1]].update(dets[m[0], :])
            owner[int(recs[m[0]])] = self.trackers[m[1]]
        if self.use_byte and len(dets_second) > 0 and unmatched_trks.shape[0] > 0:
            u_trks = trks[unmatched_trks]
            iou_left = np.array(iou_batch(dets_second, u_trks))
            if iou_left.max() > self.iou_threshold:
                matched_indices = linear_assignment(-iou_left)
                to_remove_trk_indices = []
                for m in matched_indices:
                    det_ind, trk_ind = m[0], unmatched_trks[m[1]]
                    if iou_left[m[0], m[1]] < self.iou_threshold:
                        continue
                    self.trackers[trk_ind].update(dets_second[det_ind, :])
                    owner[int(recs_second[det_ind])] = self.trackers[trk_ind]
                    to_remove_trk_indices.append(trk_ind)
                unmatched_trks = np.setdiff1d(unmatched_trks, np.array(to_remove_trk_indices))
        if unmatched_dets.shape[0] > 0 and unmatched_trks.shape[0] > 0:
            left_dets = dets[unmatched_dets]
            left_trks = last_boxes[unmatched_trks]
            iou_left = np.array(iou_batch(left_dets, left_trks))
            if iou_left.max() > self.iou_threshold:
                rematched_indices = linear_assignment(-iou_left)
                to_remove_det_indices = []
                to_remove_trk_indices = []
                for m in rematched_indices:
                    det_ind, trk_ind = unmatched_dets[m[0]], unmatched_trks[m[1]]
                    if iou_left[m[0], m[1]] < self.iou_threshold:
                        continue
                    self.trackers[trk_ind].update(dets[det_ind, :])
                    owner[int(recs[det_ind])] = self.trackers[trk_ind]
                    to_remove_det_indices.append(det_ind)
                    to_remove_trk_indices.append(trk_ind)
                unmatched_dets = np.setdiff1d(unmatched_dets, np.array(to_remove_det_indices))
                unmatched_trks = np.setdiff1d(unmatched_trks, np.array(to_remove_trk_indices))
        for m in unmatched_trks:
            self.trackers[m].update(None)
        for i in unmatched_dets:
            trk = KalmanBoxTracker(dets[i, :], self.counter, delta_t=self.delta_t)
            self.trackers.append(trk)
            owner[int(recs[i])] = trk
        reported = {}
        i = len(self.trackers)
        for trk in reversed(self.trackers):
            if trk.last_observation.sum() < 0:
                d = trk.get_state()[0]
            else:
                d = trk.last_observation[:4]
            if (trk.time_since_update < 1) and (trk.hit_streak >= self.min_hits or self.frame_count <= self.min_hits):
                reported[id(trk)] = d
            i -= 1
            if trk.time_since_update > self.max_age:
                self.trackers.pop(i)
        return owner, reported


class MatrixOcSort:
    """The literal form, one ``OCSortClass`` per class sharing the stream's id counter.  Same interface as ``OcSort``."""

    def __init__(self, C: int, K: int, det_thresh: float = 0.6, max_age: int = 30, min_hits: int = 3,
                 iou_thresh: float = 0.3, delta_t: int = 3, inertia: float = 0.2, use_byte: bool = False):
        self.C, self.K = int(C), int(K)
        self.setting = (float(det_thresh), int(max_age), int(min_hits), float(iou_thresh), int(delta_t), float(inertia),
                        bool(use_byte))
        self.reset()

    def reset(self) -> None:
        self.counter = [0]
        self.trackers = [OCSortClass(*self.setting, self.counter) for _ in range(self.C)]
        self.last_position: Optional[int] = None

    def update(self, position: int, boxes, counts, scores):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                for tr in self.trackers:
                    tr.update(np.empty((0, 5)), np.empty(0, np.int64))
        self.last_position = position
        boxes = np.asarray(boxes, np.float32)
        scores = np.asarray(scores, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)
        for c, tr in enumerate(self.trackers):
            b = boxes[c, :int(counts[c])].astype(np.float64)
            ok = np.isfinite(b).all(1) & (b[:, 3] - b[:, 1] > 0) & (b[:, 2] - b[:, 0] > 0)
            recs = np.nonzero(ok)[0]
            dets = np.concatenate([b[recs][:, [1, 0, 3, 2]], scores[c, recs].astype(np.float64)[:, None]], axis=1)
            owner, reported = tr.update(dets, recs)
            for rec, t in owner.items():
                if id(t) in reported:
                    x1, y1, x2, y2 = (float(v) for v in reported[id(t)])
                    ids[c, rec] = t.id + 1
                    out[c, rec] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)
        return ids, out
