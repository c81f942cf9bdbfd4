"""ByteTrack (Zhang et al., ECCV 2022, "ByteTrack: Multi-Object Tracking by Associating Every Detection Box") restated in
plain Python: the rules the GPU tracker (``k2y_bytetrack_update``, csrc/bytetrack.cu) follows bit for bit.  ``BYTETracker.update``
with these rules and choices:

* Setting: ``track_thresh`` (0.5), ``match_thresh`` (0.8), ``track_buffer`` (30 frames) and ``fuse_score`` (True; ByteTrack's
  --mot20 turns it off), named as on ByteTrack's command line.  Fixed as in ByteTrack: the low-score bound 0.1, the second
  association's threshold 0.5, the unconfirmed association's 0.7, the duplicate threshold 0.15, and det_thresh =
  track_thresh + 0.1.  Choice: ``track_buffer`` is a number of frames (max_time_lost), not scaled by frame rate / 30.
* Per class and per stream, as oracle/sort_ref.py: each class runs its own ByteTrack; one id counter per stream, from 1, an id
  taken at every birth in (frame, class, birth order) order (a re-activated track keeps its id; as in ByteTrack, tracks that
  are never confirmed leave gaps); a jump of g > 1 positions first runs g - 1 updates without detections; ``frame_id``
  counts the updates.
* Detections, in record order.  Choice: a record is a detection only when its four coordinates are finite and its width and
  height are > 0.  High: score > track_thresh; low: 0.1 < score < track_thresh (choice: the float32 score widened to
  float64 against float64 thresholds).  tlwh = (x1, y1, x2 - x1, y2 - y1); a detection's tlbr is (x1, y1, w + x1, h + y1).
* Kalman filter: ByteTrack's constant-velocity filter on (x, y, a, h) with w_p = 1/20, w_v = 1/160.  P stays
  block-diagonal and S diagonal, so it is exactly four 2-state blocks (p, v, P_pp, P_pv, P_vv) of x, y, a and h, written
  out in float64 with the operation order below and no fused multiply-add:
  - initiate from z = (x1 + w/2, y1 + h/2, w/h, h): mean (z, 0), P = diag(std^2), std = (2 w_p) h for x, y, h and 1e-2
    for a; velocity (10 w_v) h and 1e-5;
  - predict: q = w_p h and w_v h (1e-2, 1e-5 for a) with h the mean's before the predict; p += v; P = F P F' + Q;
  - update: R std w_p h (1e-1 for a) with h the predicted mean's; S = P_pp + R; the gain is the Cholesky solve, k =
    (P_p. / sqrt(S)) / sqrt(S); mean += k y; P -= k S k';
  - a track's tlwh is (x - w/2, y - h/2, w, h), w = a h, its tlbr (x1, y1, w + x1, h + y1);
  - quirk, kept: a track not in state Tracked has its h velocity set to 0 before each predict.
* IoU is cython_bbox's ``bbox_overlaps`` (tracks as its boxes, detections as its query boxes): the "+1" areas, iw tested
  > 0 before ih, min / max as Cython's (the second operand when it compares below / above the first).  Choice: an IoU whose
  union is not > 0 counts as 0.  Cost is 1 - IoU; with fuse_score 1 - (1 - cost) * score.
* Assignment: ByteTrack calls lap.lapjv(cost, extend_cost=True, cost_limit=thresh).  Choice: ``lsap(min(cost - thresh, 0))``
  (sort_ref.lsap, scipy's algorithm, ties included; rows are tracks, so it transposes when tracks outnumber detections),
  keeping the pairs with cost < thresh, in row order; unmatched rows and columns ascending.  Its optimum is that of lap's
  extended (T + D) square problem (a pair costs cost - thresh against leaving both sides out); only ties may go another way.
* One frame, per class, in BYTETracker.update's list orders (they are the assignment's row orders, so they decide ties):
  1. tracked splits into unconfirmed (not activated) and active; pool = active + lost; every pool track is predicted
     (unconfirmed tracks are not: a quirk, kept);
  2. pool x high detections (fused cost, match_thresh): a matched Tracked track is updated, a matched Lost track is
     re-activated (updated, Tracked, activated, keeps its id and start frame);
  3. the pool's unmatched rows in state Tracked x low detections (plain cost, 0.5), same rule; those still unmatched
     become Lost;
  4. unconfirmed x the high detections left from 2 (fused cost, 0.7): matched tracks are updated and activated, the others
     removed;
  5. each high detection left from 4 with score >= det_thresh is born: a new id, Tracked, activated only when frame_id == 1;
  6. the lost tracks from before this frame with frame_id - end_frame > track_buffer are removed;
  7. tracked = (old tracked still Tracked) + births + re-activated; lost = (old lost still Lost, not removed) + newly lost
     (ByteTrack's joint_stracks / sub_stracks, which come to these orders);
  8. duplicates: every (tracked, lost) pair with 1 - IoU < 0.15 on their current means drops the one with the shorter
     frame_id - start_frame, a tie dropping the tracked one; a dropped track just disappears.
* Output per record: a track id when the track it updated, re-activated or created in this frame ends the frame in tracked
  and activated, with that track's tlbr as float32 (ymin, xmin, ymax, xmax); -1 and zeros elsewhere.  A low-score record can
  keep a track alive and carry its id, but never starts one.

Capacity.  After frame f a class's live tracks (tracked and lost) have end_frame in [f - max(B, 1), f], B = track_buffer:
every tracked track was updated or born in f, and a lost one ended at most max(B, 1) frames back (one newly lost at f - 1
survives f even with B = 0, since step 6 sees only the lost of before the frame).  Each frame ends at most K tracks, one
per detection, so at most K (max(B, 1) + 1) are alive after a frame; within a frame the births (at most K) come before the
removal of step 6, so the storage must hold ``max_tracks(K, B)`` = K (max(B, 1) + 2).  The GPU tracker refuses a setting
past 4096.  The bound is safe, not tight: only a frame-1 birth or a track confirmed by a record in a later frame can become
lost, so a record that starts a track cannot also keep an old one alive, and the most crowded streams the tests build (K
new boxes every second frame, confirmed in the next one and then lost) reach about K (B / 2 + 2) tracks.  A tighter bound is
not derived here, so the cap stays about twice what such streams need (track_buffer <= 38 at K = 100).

``MatrixByteTrack`` is a literal matrix form: numpy 8x8 filter matrices with scipy's cho_factor / cho_solve and STrack
objects in Python lists the way BYTETracker.update keeps them; the restatement is checked against it.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

from .sort_ref import lsap

W_P, W_V = 1.0 / 20, 1.0 / 160
LOW_THRESH, SECOND_THRESH, UNCONFIRMED_THRESH, DUPLICATE_THRESH = 0.1, 0.5, 0.7, 0.15
TRACKED, LOST, REMOVED = 1, 2, 3


def max_tracks(K: int, track_buffer: int) -> int:
    """Tracks one class may hold within a frame (module docstring, Capacity)."""
    return int(K) * (max(int(track_buffer), 1) + 2)


# -- assignment ----------------------------------------------------------------------------------------------------------------
def assign(cost, nc, thresh):
    """(matches [(row, col)] in row order, unmatched rows, unmatched cols) of lap.lapjv(cost, extend_cost=True,
    cost_limit=thresh) as restated for the rows of `cost` over nc columns: lsap(min(cost - thresh, 0)), pairs with
    cost < thresh kept."""
    nr = len(cost)
    if nr == 0 or nc == 0:
        return [], list(range(nr)), list(range(nc))
    r, c = lsap([[min(v - thresh, 0.0) for v in row] for row in cost])
    matches = [(i, j) for i, j in zip(r.tolist(), c.tolist()) if cost[i][j] < thresh]
    mr, mc = {i for i, _ in matches}, {j for _, j in matches}
    return matches, [i for i in range(nr) if i not in mr], [j for j in range(nc) if j not in mc]


# -- IoU ------------------------------------------------------------------------------------------------------------------------
def _cmin(a, b):
    return b if b < a else a


def _cmax(a, b):
    return b if b > a else a


def iou(a, b) -> float:
    """cython_bbox.bbox_overlaps of box a (a track's tlbr) and query box b (a detection's), 0 where the union is not > 0."""
    iw = (_cmin(a[2], b[2]) - _cmax(a[0], b[0])) + 1.0
    if iw > 0:
        ih = (_cmin(a[3], b[3]) - _cmax(a[1], b[1])) + 1.0
        if ih > 0:
            inter = iw * ih
            ua = (((a[2] - a[0]) + 1.0) * ((a[3] - a[1]) + 1.0) + ((b[2] - b[0]) + 1.0) * ((b[3] - b[1]) + 1.0)) - inter
            return inter / ua if ua > 0 else 0.0
    return 0.0


def fused(cost, score):
    return 1.0 - (1.0 - cost) * score


# -- the filter, in block form ------------------------------------------------------------------------------------------------
class _Track:
    __slots__ = ("mean", "cov", "id", "state", "activated", "frame_id", "start_frame", "rec")

    def __init__(self, det, frame_id):
        x1, y1, w, h = det.tlwh
        self.mean = [x1 + w / 2.0, y1 + h / 2.0, w / h, h, 0.0, 0.0, 0.0, 0.0]
        sp, sv = (2.0 * W_P) * h, (10.0 * W_V) * h
        self.cov = [[sp * sp, 0.0, sv * sv], [sp * sp, 0.0, sv * sv], [1e-2 * 1e-2, 0.0, 1e-5 * 1e-5], [sp * sp, 0.0, sv * sv]]
        self.id = -1
        self.state = TRACKED
        self.activated = frame_id == 1
        self.frame_id = self.start_frame = frame_id
        self.rec = det.k

    def predict(self):
        m = self.mean
        if self.state != TRACKED:
            m[7] = 0.0
        qp, qv = W_P * m[3], W_V * m[3]
        Qp, Qv = [qp * qp, qp * qp, 1e-2 * 1e-2, qp * qp], [qv * qv, qv * qv, 1e-5 * 1e-5, qv * qv]
        for b in range(4):
            a, pv, d = self.cov[b]
            t = pv + d
            m[b] = m[b] + m[4 + b]
            self.cov[b] = [((a + pv) + t) + Qp[b], t, d + Qv[b]]

    def update(self, det, frame_id):
        x1, y1, w, h = det.tlwh
        z = [x1 + w / 2.0, y1 + h / 2.0, w / h, h]
        m = self.mean
        r = W_P * m[3]
        R = [r * r, r * r, 1e-1 * 1e-1, r * r]
        for b in range(4):
            a, pv, d = self.cov[b]
            S = a + R[b]
            L = math.sqrt(S)
            k0, k1 = (a / L) / L, (pv / L) / L
            y = z[b] - m[b]
            m[b] = m[b] + k0 * y
            m[4 + b] = m[4 + b] + k1 * y
            ks0, ks1 = k0 * S, k1 * S
            self.cov[b] = [a - ks0 * k0, pv - ks0 * k1, d - ks1 * k1]
        self.frame_id = frame_id
        self.state = TRACKED
        self.activated = True
        self.rec = det.k

    def tlbr(self):
        x, y, a, h = self.mean[:4]
        w = a * h
        x1, y1 = x - w / 2.0, y - h / 2.0
        return [x1, y1, w + x1, h + y1]


class _Det:
    __slots__ = ("tlwh", "tlbr", "score", "k")

    def __init__(self, xmin, ymin, xmax, ymax, score, k):
        w, h = xmax - xmin, ymax - ymin
        self.tlwh = (xmin, ymin, w, h)
        self.tlbr = [xmin, ymin, w + xmin, h + ymin]
        self.score, self.k = score, k


def detections(boxes_c, count, scores_c, track_thresh):
    """(high, low) detections of one class's records (``_Det``, record order)."""
    high, low = [], []
    for k in range(int(count)):
        ymin, xmin, ymax, xmax = (float(v) for v in boxes_c[k])
        if not all(math.isfinite(v) for v in (ymin, xmin, ymax, xmax)) or not (xmax - xmin > 0 and ymax - ymin > 0):
            continue
        s = float(scores_c[k])
        if s > track_thresh:
            high.append(_Det(xmin, ymin, xmax, ymax, s, k))
        elif LOW_THRESH < s < track_thresh:
            low.append(_Det(xmin, ymin, xmax, ymax, s, k))
    return high, low


class ByteTrack:
    """ByteTrack of one stream over C classes of at most K records.  ``update(position, boxes, counts, scores)`` takes one
    frame: `boxes` float32 [C, K, 4] (ymin, xmin, ymax, xmax), `counts` [C] and `scores` float32 [C, K]; returns (ids int32
    [C, K], boxes float32 [C, K, 4])."""

    def __init__(self, C: int, K: int, track_thresh: float = 0.5, match_thresh: float = 0.8, track_buffer: int = 30,
                 fuse_score: bool = True):
        self.C, self.K = int(C), int(K)
        self.track_thresh, self.match_thresh = float(track_thresh), float(match_thresh)
        self.track_buffer, self.fuse_score = int(track_buffer), bool(fuse_score)
        self.det_thresh = self.track_thresh + 0.1
        self.reset()

    def reset(self) -> None:
        self.tracked: List[List[_Track]] = [[] for _ in range(self.C)]
        self.lost: List[List[_Track]] = [[] for _ in range(self.C)]
        self.frame_id = 0
        self.last_position: Optional[int] = None
        self.next_id = 1

    def _costs(self, trks, dets, fuse):
        boxes = [t.tlbr() for t in trks]
        return [[fused(1.0 - iou(b, d.tlbr), d.score) if fuse else 1.0 - iou(b, d.tlbr) for d in dets] for b in boxes]

    def _step(self, c: int, high, low) -> None:
        f, B = self.frame_id, self.track_buffer
        tracked, lost = self.tracked[c], self.lost[c]
        unconfirmed = [t for t in tracked if not t.activated]
        pool = [t for t in tracked if t.activated] + lost
        for t in pool:
            t.predict()
        matches, u_rows, u_high = assign(self._costs(pool, high, self.fuse_score), len(high), self.match_thresh)
        for i, j in matches:
            pool[i].update(high[j], f)                # a Lost track is re-activated: Tracked, activated, same id
        rest = [pool[i] for i in u_rows if pool[i].state == TRACKED]
        matches, u_rest, _ = assign(self._costs(rest, low, False), len(low), SECOND_THRESH)
        for i, j in matches:
            rest[i].update(low[j], f)
        for i in u_rest:
            rest[i].state = LOST
        left = [high[j] for j in u_high]
        matches, u_unc, u_left = assign(self._costs(unconfirmed, left, self.fuse_score), len(left), UNCONFIRMED_THRESH)
        for i, j in matches:
            unconfirmed[i].update(left[j], f)
        for i in u_unc:
            unconfirmed[i].state = REMOVED
        born = [_Track(left[j], f) for j in u_left if left[j].score >= self.det_thresh]
        for t in born:
            t.id = self.next_id
            self.next_id += 1
        new_tracked = [t for t in tracked if t.state == TRACKED] + born + [t for t in lost if t.state == TRACKED]
        new_lost = [t for t in lost if t.state == LOST and not f - t.frame_id > B] + [t for t in tracked if t.state == LOST]
        drop_t, drop_l = set(), set()
        lboxes = [t.tlbr() for t in new_lost]
        for p, a in enumerate(new_tracked):
            ba = a.tlbr()
            for q, b in enumerate(new_lost):
                if 1.0 - iou(ba, lboxes[q]) < DUPLICATE_THRESH:
                    if a.frame_id - a.start_frame > b.frame_id - b.start_frame:
                        drop_l.add(q)
                    else:
                        drop_t.add(p)
        self.tracked[c] = [t for p, t in enumerate(new_tracked) if p not in drop_t]
        self.lost[c] = [t for q, t in enumerate(new_lost) if q not in drop_l]

    def update(self, position: int, boxes, counts, scores):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                self.frame_id += 1
                for c in range(self.C):
                    self._step(c, [], [])
        self.last_position = position
        self.frame_id += 1
        boxes = np.asarray(boxes, np.float32)
        scores = np.asarray(scores, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)
        for c in range(self.C):
            high, low = detections(boxes[c], counts[c], scores[c], self.track_thresh)
            self._step(c, high, low)
            for t in self.tracked[c]:
                if t.activated:
                    x1, y1, x2, y2 = t.tlbr()
                    ids[c, t.rec] = t.id
                    out[c, t.rec] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)
        return ids, out


# -- literal matrix form -------------------------------------------------------------------------------------------------------
class KalmanFilter:
    """ByteTrack's KalmanFilter (DeepSORT's): 8x8 matrices, the Cholesky solve of scipy."""

    def __init__(self):
        ndim, dt = 4, 1.0
        self._motion_mat = np.eye(2 * ndim, 2 * ndim)
        for i in range(ndim):
            self._motion_mat[i, ndim + i] = dt
        self._update_mat = np.eye(ndim, 2 * ndim)
        self._std_weight_position = 1.0 / 20
        self._std_weight_velocity = 1.0 / 160

    def initiate(self, measurement):
        mean_pos = measurement
        mean_vel = np.zeros_like(mean_pos)
        mean = np.r_[mean_pos, mean_vel]
        std = [2 * self._std_weight_position * measurement[3], 2 * self._std_weight_position * measurement[3], 1e-2,
               2 * self._std_weight_position * measurement[3], 10 * self._std_weight_velocity * measurement[3],
               10 * self._std_weight_velocity * measurement[3], 1e-5, 10 * self._std_weight_velocity * measurement[3]]
        return mean, np.diag(np.square(std))

    def predict(self, mean, covariance):
        std_pos = [self._std_weight_position * mean[3], self._std_weight_position * mean[3], 1e-2,
                   self._std_weight_position * mean[3]]
        std_vel = [self._std_weight_velocity * mean[3], self._std_weight_velocity * mean[3], 1e-5,
                   self._std_weight_velocity * mean[3]]
        motion_cov = np.diag(np.square(np.r_[std_pos, std_vel]))
        mean = np.dot(mean, self._motion_mat.T)
        covariance = np.linalg.multi_dot((self._motion_mat, covariance, self._motion_mat.T)) + motion_cov
        return mean, covariance

    def project(self, mean, covariance):
        std = [self._std_weight_position * mean[3], self._std_weight_position * mean[3], 1e-1,
               self._std_weight_position * mean[3]]
        innovation_cov = np.diag(np.square(std))
        mean = np.dot(self._update_mat, mean)
        covariance = np.linalg.multi_dot((self._update_mat, covariance, self._update_mat.T))
        return mean, covariance + innovation_cov

    def update(self, mean, covariance, measurement):
        import scipy.linalg
        projected_mean, projected_cov = self.project(mean, covariance)
        chol_factor, lower = scipy.linalg.cho_factor(projected_cov, lower=True, check_finite=False)
        kalman_gain = scipy.linalg.cho_solve((chol_factor, lower), np.dot(covariance, self._update_mat.T).T,
                                             check_finite=False).T
        innovation = measurement - projected_mean
        new_mean = mean + np.dot(innovation, kalman_gain.T)
        new_covariance = covariance - np.linalg.multi_dot((kalman_gain, projected_cov, kalman_gain.T))
        return new_mean, new_covariance


class STrack:
    """ByteTrack's STrack: a detection until ``activate``, then a track.  `counter` is the stream's id counter (a list)."""
    shared_kalman = KalmanFilter()

    def __init__(self, tlwh, score, rec):
        self._tlwh = np.asarray(tlwh, dtype=np.float64)
        self.kalman_filter = None
        self.mean, self.covariance = None, None
        self.is_activated = False
        self.score = score
        self.rec = rec
        self.state = TRACKED
        self.track_id = 0
        self.frame_id = self.start_frame = 0

    @staticmethod
    def multi_predict(stracks):
        for st in stracks:
            mean_state = st.mean.copy()
            if st.state != TRACKED:
                mean_state[7] = 0
            st.mean, st.covariance = STrack.shared_kalman.predict(mean_state, st.covariance)

    def activate(self, kalman_filter, frame_id, counter):
        self.kalman_filter = kalman_filter
        self.track_id = counter[0]
        counter[0] += 1
        self.mean, self.covariance = self.kalman_filter.initiate(self.tlwh_to_xyah(self._tlwh))
        self.state = TRACKED
        if frame_id == 1:
            self.is_activated = True
        self.frame_id = frame_id
        self.start_frame = frame_id

    def re_activate(self, new_track, frame_id):
        self.mean, self.covariance = self.kalman_filter.update(self.mean, self.covariance, self.tlwh_to_xyah(new_track.tlwh))
        self.state = TRACKED
        self.is_activated = True
        self.frame_id = frame_id
        self.score = new_track.score

    def update(self, new_track, frame_id):
        self.frame_id = frame_id
        self.mean, self.covariance = self.kalman_filter.update(self.mean, self.covariance, self.tlwh_to_xyah(new_track.tlwh))
        self.state = TRACKED
        self.is_activated = True
        self.score = new_track.score

    @property
    def end_frame(self):
        return self.frame_id

    @property
    def tlwh(self):
        if self.mean is None:
            return self._tlwh.copy()
        ret = self.mean[:4].copy()
        ret[2] *= ret[3]
        ret[:2] -= ret[2:] / 2
        return ret

    @property
    def tlbr(self):
        ret = self.tlwh.copy()
        ret[2:] += ret[:2]
        return ret

    @staticmethod
    def tlwh_to_xyah(tlwh):
        ret = np.asarray(tlwh).copy()
        ret[:2] += ret[2:] / 2
        ret[2] /= ret[3]
        return ret

    @staticmethod
    def tlbr_to_tlwh(tlbr):
        ret = np.asarray(tlbr).copy()
        ret[2:] -= ret[:2]
        return ret


def bbox_ious(boxes, query_boxes):
    """cython_bbox.bbox_overlaps, vectorised, with the union-not->-0 choice."""
    boxes, query_boxes = np.asarray(boxes, np.float64).reshape(-1, 4), np.asarray(query_boxes, np.float64).reshape(-1, 4)
    a, b = boxes[:, None, :], query_boxes[None, :, :]
    iw = np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]) + 1
    ih = np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]) + 1
    box_area = (b[..., 2] - b[..., 0] + 1) * (b[..., 3] - b[..., 1] + 1)
    ua = (a[..., 2] - a[..., 0] + 1) * (a[..., 3] - a[..., 1] + 1) + box_area - iw * ih
    ok = (iw > 0) & (ih > 0) & (ua > 0)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return np.where(ok, iw * ih / np.where(ok, ua, 1.0), 0.0)


def iou_distance(atracks, btracks):
    atlbrs = [t.tlbr for t in atracks]
    btlbrs = [t.tlbr for t in btracks]
    ious = np.zeros((len(atlbrs), len(btlbrs)), dtype=np.float64)
    if ious.size:
        ious = bbox_ious(np.ascontiguousarray(atlbrs), np.ascontiguousarray(btlbrs))
    return 1 - ious


def fuse_score(cost_matrix, detections):
    if cost_matrix.size == 0:
        return cost_matrix
    iou_sim = 1 - cost_matrix
    det_scores = np.expand_dims(np.array([det.score for det in detections]), axis=0).repeat(cost_matrix.shape[0], axis=0)
    return 1 - iou_sim * det_scores


def linear_assignment(cost_matrix, thresh):
    """matching.linear_assignment with lap.lapjv replaced by scipy on min(cost - thresh, 0) (the module docstring's choice)."""
    from scipy.optimize import linear_sum_assignment
    if cost_matrix.size == 0:
        return np.empty((0, 2), dtype=int), tuple(range(cost_matrix.shape[0])), tuple(range(cost_matrix.shape[1]))
    r, c = linear_sum_assignment(np.minimum(cost_matrix - thresh, 0.0))
    x = np.full(cost_matrix.shape[0], -1)
    y = np.full(cost_matrix.shape[1], -1)
    for i, j in zip(r, c):
        if cost_matrix[i, j] < thresh:
            x[i], y[j] = j, i
    matches = np.asarray([[ix, mx] for ix, mx in enumerate(x) if mx >= 0])
    return matches, np.where(x < 0)[0], np.where(y < 0)[0]


def joint_stracks(tlista, tlistb):
    exists, res = {}, []
    for t in tlista:
        exists[t.track_id] = 1
        res.append(t)
    for t in tlistb:
        if not exists.get(t.track_id, 0):
            exists[t.track_id] = 1
            res.append(t)
    return res


def sub_stracks(tlista, tlistb):
    stracks = {t.track_id: t for t in tlista}
    for t in tlistb:
        if stracks.get(t.track_id, 0):
            del stracks[t.track_id]
    return list(stracks.values())


def remove_duplicate_stracks(stracksa, stracksb):
    pdist = iou_distance(stracksa, stracksb)
    pairs = np.where(pdist < DUPLICATE_THRESH)
    dupa, dupb = [], []
    for p, q in zip(*pairs):
        timep = stracksa[p].frame_id - stracksa[p].start_frame
        timeq = stracksb[q].frame_id - stracksb[q].start_frame
        if timep > timeq:
            dupb.append(q)
        else:
            dupa.append(p)
    return [t for i, t in enumerate(stracksa) if i not in dupa], [t for i, t in enumerate(stracksb) if i not in dupb]


class BYTETracker:
    """BYTETracker.update for one class; `owner` maps each record to the track it updated or created this frame."""

    def __init__(self, track_thresh, match_thresh, track_buffer, fuse, counter):
        self.tracked_stracks, self.lost_stracks, self.removed_stracks = [], [], []
        self.frame_id = 0
        self.track_thresh, self.match_thresh, self.fuse = track_thresh, match_thresh, fuse
        self.det_thresh = track_thresh + 0.1
        self.max_time_lost = track_buffer
        self.kalman_filter = KalmanFilter()
        self.counter = counter

    def update(self, bboxes, scores, recs):
        self.frame_id += 1
        activated_starcks, refind_stracks, lost_stracks, removed_stracks = [], [], [], []
        owner = {}
        remain_inds = scores > self.track_thresh
        inds_low = scores > LOW_THRESH
        inds_high = scores < self.track_thresh
        inds_second = np.logical_and(inds_low, inds_high)
        detections = [STrack(STrack.tlbr_to_tlwh(b), s, r) for b, s, r in
                      zip(bboxes[remain_inds], scores[remain_inds], recs[remain_inds])]
        unconfirmed, tracked_stracks = [], []
        for track in self.tracked_stracks:
            (tracked_stracks if track.is_activated else unconfirmed).append(track)
        strack_pool = joint_stracks(tracked_stracks, self.lost_stracks)
        STrack.multi_predict(strack_pool)
        dists = iou_distance(strack_pool, detections)
        if self.fuse:
            dists = fuse_score(dists, detections)
        matches, u_track, u_detection = linear_assignment(dists, thresh=self.match_thresh)
        for itracked, idet in matches:
            track, det = strack_pool[itracked], detections[idet]
            owner[det.rec] = track
            if track.state == TRACKED:
                track.update(det, self.frame_id)
                activated_starcks.append(track)
            else:
                track.re_activate(det, self.frame_id)
                refind_stracks.append(track)
        detections_second = [STrack(STrack.tlbr_to_tlwh(b), s, r) for b, s, r in
                             zip(bboxes[inds_second], scores[inds_second], recs[inds_second])]
        r_tracked_stracks = [strack_pool[i] for i in u_track if strack_pool[i].state == TRACKED]
        dists = iou_distance(r_tracked_stracks, detections_second)
        matches, u_track, _ = linear_assignment(dists, thresh=SECOND_THRESH)
        for itracked, idet in matches:
            track, det = r_tracked_stracks[itracked], detections_second[idet]
            owner[det.rec] = track
            if track.state == TRACKED:
                track.update(det, self.frame_id)
                activated_starcks.append(track)
            else:
                track.re_activate(det, self.frame_id)
                refind_stracks.append(track)
        for it in u_track:
            track = r_tracked_stracks[it]
            if not track.state == LOST:
                track.state = LOST
                lost_stracks.append(track)
        detections = [detections[i] for i in u_detection]
        dists = iou_distance(unconfirmed, detections)
        if self.fuse:
            dists = fuse_score(dists, detections)
        matches, u_unconfirmed, u_detection = linear_assignment(dists, thresh=UNCONFIRMED_THRESH)
        for itracked, idet in matches:
            unconfirmed[itracked].update(detections[idet], self.frame_id)
            owner[detections[idet].rec] = unconfirmed[itracked]
            activated_starcks.append(unconfirmed[itracked])
        for it in u_unconfirmed:
            track = unconfirmed[it]
            track.state = REMOVED
            removed_stracks.append(track)
        for inew in u_detection:
            track = detections[inew]
            if track.score < self.det_thresh:
                continue
            track.activate(self.kalman_filter, self.frame_id, self.counter)
            owner[track.rec] = track
            activated_starcks.append(track)
        for track in self.lost_stracks:
            if self.frame_id - track.end_frame > self.max_time_lost:
                track.state = REMOVED
                removed_stracks.append(track)
        self.tracked_stracks = [t for t in self.tracked_stracks if t.state == TRACKED]
        self.tracked_stracks = joint_stracks(self.tracked_stracks, activated_starcks)
        self.tracked_stracks = joint_stracks(self.tracked_stracks, refind_stracks)
        self.lost_stracks = sub_stracks(self.lost_stracks, self.tracked_stracks)
        self.lost_stracks.extend(lost_stracks)
        self.lost_stracks = sub_stracks(self.lost_stracks, self.removed_stracks + removed_stracks)
        self.removed_stracks.extend(removed_stracks)
        self.tracked_stracks, self.lost_stracks = remove_duplicate_stracks(self.tracked_stracks, self.lost_stracks)
        output = [t for t in self.tracked_stracks if t.is_activated]
        return owner, output


class MatrixByteTrack:
    """The literal form, one ``BYTETracker`` per class sharing the stream's id counter.  Same interface as ``ByteTrack``."""

    def __init__(self, C: int, K: int, track_thresh: float = 0.5, match_thresh: float = 0.8, track_buffer: int = 30,
                 fuse_score: bool = True):
        self.C, self.K = int(C), int(K)
        self.setting = (float(track_thresh), float(match_thresh), int(track_buffer), bool(fuse_score))
        self.reset()

    def reset(self) -> None:
        self.counter = [1]
        self.trackers = [BYTETracker(*self.setting, self.counter) for _ in range(self.C)]
        self.last_position: Optional[int] = None

    def update(self, position: int, boxes, counts, scores):
        position = int(position)
        if self.last_position is not None:
            if position <= self.last_position:
                raise ValueError(f"frame position {position} does not follow {self.last_position}")
            for _ in range(position - self.last_position - 1):
                for tr in self.trackers:
                    tr.update(np.empty((0, 4)), np.empty(0), np.empty(0, np.int64))
        self.last_position = position
        boxes = np.asarray(boxes, np.float32)
        scores = np.asarray(scores, np.float32)
        ids = np.full((self.C, self.K), -1, np.int32)
        out = np.zeros((self.C, self.K, 4), np.float32)
        for c, tr in enumerate(self.trackers):
            b = boxes[c, :int(counts[c])].astype(np.float64)
            ok = np.isfinite(b).all(1) & (b[:, 3] - b[:, 1] > 0) & (b[:, 2] - b[:, 0] > 0)
            recs = np.nonzero(ok)[0]
            owner, output = tr.update(b[recs][:, [1, 0, 3, 2]], scores[c, recs].astype(np.float64), recs)
            shown = {id(t) for t in output}
            for rec, t in owner.items():
                if id(t) in shown:
                    x1, y1, x2, y2 = t.tlbr
                    ids[c, rec] = t.track_id
                    out[c, rec] = np.array([y1, x1, y2, x2], np.float64).astype(np.float32)
        return ids, out
