"""MOTChallenge tracking evaluation (CLEAR MOT and identity metrics), restated in plain Python — TEST INFRASTRUCTURE ONLY.

This module defines the protocol that ``k210_yolo_framework_b200.evaluate.MotEval`` (csrc/evaluate_mot.cu) implements on
the GPU: integer counts equal, float64 sums equal bit for bit.  The rules follow TrackEval's ``MotChallenge2DBox``
preprocessing and its ``CLEAR`` and ``Identity`` metrics as far as they are known from TrackEval's published code; they
have NOT been compared with TrackEval itself, which is not available here.

Inputs
  * Ground truth: float64 rows [n, 8] (frame, id, left, top, w, h, conf, class).  A MOT16/17/20 ``gt/gt.txt`` row is
    (frame, id, left, top, w, h, conf, class, visibility); a MOT15 row (frame, id, left, top, w, h, conf, x, y, z) has no
    class and is read as class 1 (``k210_yolo_framework_b200.evaluate.load_mot_gt`` reads both).  Frames run 1..seqLength.
  * Tracker rows: float64 [n, 7] (frame, id, left, top, w, h, conf), made from the pipeline's tracks by ``tracker_rows``:
    for frame position p, each record of the person class with a track id >= 0 gives frame = p + 1, id = the track id,
    left = float64(xmin) + 1, top = float64(ymin) + 1, w = float64(xmax) - float64(xmin), h = float64(ymax) -
    float64(ymin) (the track box of ``DetectionPipeline.tracks``, (ymin, xmin, ymax, xmax); MOTChallenge pixels start at
    1) and conf = the record's score.  Rows keep record order within a frame; that order is the column order of every
    assignment below.  Ground-truth rows keep file order within a frame; that order is the row order.
  * Refusals (ValueError naming the sequence and frame): a gt or tracker frame that is not an integer in 1..seqLength; an
    id that appears twice in one frame, in gt or in tracker rows; for MOT16/17/20 a gt class outside 1..13.

IoU (TrackEval's box IoU, float64): x2 = left + w, y2 = top + h; intersection = max(min(x2) - max(x1), 0) * max(min(y2) -
max(y1), 0); area = (x2 - x1) * (y2 - y1) of the corners; union = area1 + area2 - intersection.  With eps = 2^-52
(np.finfo(float).eps): intersection = 0 where either area is <= eps or the union is <= eps, and union = 1 where it is
<= eps.  ``lsap`` is ``oracle.sort_ref.lsap``, scipy's linear_sum_assignment ties included.

Preprocessing (MOT16/17/20; for MOT15 only the conf filter applies)
  * Distractor removal, per frame with both gt and tracker rows: S = IoU of all the frame's gt rows (any class, any conf)
    against its tracker rows; S = 0 where S < 0.5 - eps; rows, cols = lsap(-S), keeping pairs with S > eps; every tracker
    row paired with a gt row of a distractor class (2, 7, 8, 12; MOT20 adds 6) is removed.
  * Then only the gt rows with conf != 0 and class 1 are kept.

CLEAR MOT (threshold 0.5).  An effective frame has at least one gt row and one tracker row after preprocessing.  A frame
without gt rows adds its tracker rows to FP; one with gt rows but no tracker rows adds them to FN and to each gt id's
present count.  Neither changes the "previous timestep" state (TrackEval's ``continue``).  In an effective frame: score =
1000 * [tracker id == the tracker matched to this gt id at the last effective frame] + IoU, 0 where IoU < 0.5 - eps;
lsap(-score), keeping pairs with score > eps.  A match is an IDSW when its gt id's last earlier match (at any frame) was to
a different tracker id.  TP += matches, FN += gt - matches, FP += tracker - matches; the frame's IoU sum runs left to right
in row order and MOTP_sum adds the frame sums left to right in frame order.  Frag: per gt id, the effective frames where
it is matched and was not matched at the previous effective frame; Frag = sum of (count - 1) over ids with count > 0.
MT / PT / ML from each gt id's matched / present ratio: MT > 0.8, PT >= 0.2 and not MT, ML every other id with a kept row.
MOTA = (TP - FP - IDSW) / max(1, TP + FN), MOTP = MOTP_sum / max(1, TP), Rcll = TP / max(1, TP + FN),
Prcn = TP / max(1, TP + FP).

Identity.  A potential match is a (gt id, tracker id) pair with IoU >= 0.5 in a frame after preprocessing; their counts
over the sequence weigh a bipartite graph.  IDTP is the weight of a maximum-weight matching of gt ids to tracker ids.
This equals TrackEval's square (G + T)^2 cost through scipy: there every assignment's cost is sum(gt rows) + sum(tracker
rows) - 2 * (the counts of the matched pairs), so the least cost is reached exactly at a maximum-weight matching.  The
value is unique, only the matching may differ between exact solvers; ``identity`` solves each connected component of the
graph with ``lsap``.  IDFN = sum(gt rows) - IDTP, IDFP = sum(tracker rows) - IDTP, IDR = IDTP / max(1, IDTP + IDFN),
IDP = IDTP / max(1, IDTP + IDFP), IDF1 = IDTP / max(1, IDTP + IDFP / 2 + IDFN / 2).

Over several sequences the integer fields are summed, MOTP_sum is summed in sequence order, and the ratios recomputed.

Two facts the GPU relies on, both checked by the tests:
  * Isolated positives: in a frame whose positive-score pairs share no row and no column, every optimal assignment takes
    exactly those pairs, whatever the continuity bonus (a score is positive exactly where IoU >= 0.5 - eps), so no lsap
    is needed there.
  * Rounds: solve every effective frame with the bonus from the previous round's matches of its predecessor, starting
    from "no matches"; re-solve only frames whose predecessor changed; stop when nothing changes.  After round r the
    first r effective frames equal the sequential result (by induction along the frames), so the fixed point exists, is
    unique and is the sequential result.  ``clear_pairs_by_rounds`` does this; ``clear_pairs`` is the sequential loop.

``evaluate_literal`` is the same protocol written independently with numpy and scipy, in TrackEval's form: per-frame masked
matrices, ``scipy.optimize.linear_sum_assignment`` and the square identity matrix.  The restatement is checked against it.
"""
from __future__ import annotations

from collections import Counter
from typing import Dict, List, Sequence

import numpy as np

from oracle.sort_ref import lsap

EPS = float(np.finfo(float).eps)
BENCHMARKS = ("MOT15", "MOT16", "MOT17", "MOT20")
INT_FIELDS = ("TP", "FP", "FN", "IDSW", "Frag", "MT", "PT", "ML", "IDTP", "IDFP", "IDFN", "gt_rows", "tracker_rows")


def distractor_classes(benchmark: str) -> tuple:
    return (2, 6, 7, 8, 12) if benchmark == "MOT20" else (2, 7, 8, 12)


# -- inputs ---------------------------------------------------------------------------------------------------------------------
def tracker_rows(positions, ids, boxes, dets, counts, person_class: int) -> np.ndarray:
    """float64 [n, 7] (frame, id, left, top, w, h, conf) of host blocks: positions [N], ids int32 [N, C, K], boxes float32
    [N, C, K, 4] (ymin, xmin, ymax, xmax), dets int32 [N, C, K, 6] (the score is word 4), counts [N, C]."""
    ids, boxes, counts = np.asarray(ids), np.asarray(boxes, np.float32), np.asarray(counts)
    score = np.ascontiguousarray(np.asarray(dets, np.int32)[..., 4]).view(np.float32)
    out = []
    for n, p in enumerate(positions):
        for k in range(int(counts[n, person_class])):
            t = int(ids[n, person_class, k])
            if t < 0:
                continue
            y0, x0, y1, x1 = (float(v) for v in boxes[n, person_class, k])
            out.append([int(p) + 1, t, x0 + 1.0, y0 + 1.0, x1 - x0, y1 - y0, float(score[n, person_class, k])])
    return np.array(out, np.float64).reshape(-1, 7)


def check_rows(name: str, gt, trk, seq_length: int, benchmark: str = "MOT17") -> None:
    """The refusals: ValueError naming the sequence and frame."""
    if benchmark not in BENCHMARKS:
        raise ValueError(f"benchmark {benchmark!r} is not one of {BENCHMARKS}")
    for what, rows in (("gt", np.asarray(gt, np.float64)), ("tracker", np.asarray(trk, np.float64))):
        seen = set()
        for r in rows.tolist():
            f = r[0]
            if not (f == int(f) and 1 <= f <= seq_length):
                raise ValueError(f"{name}: {what} frame {f:g} is outside 1..{seq_length}")
            if (f, r[1]) in seen:
                raise ValueError(f"{name}: {what} id {r[1]:g} appears twice in frame {int(f)}")
            seen.add((f, r[1]))
            if what == "gt" and benchmark != "MOT15" and not (r[7] == int(r[7]) and 1 <= r[7] <= 13):
                raise ValueError(f"{name}: gt class {r[7]:g} in frame {int(f)} is outside 1..13")


# -- the restatement ------------------------------------------------------------------------------------------------------------
def iou(a, b) -> float:
    """TrackEval's box IoU of two (left, top, w, h) boxes, with its guards."""
    ax2, ay2, bx2, by2 = a[0] + a[2], a[1] + a[3], b[0] + b[2], b[1] + b[3]
    inter = max(min(ax2, bx2) - max(a[0], b[0]), 0.0) * max(min(ay2, by2) - max(a[1], b[1]), 0.0)
    area1 = (ax2 - a[0]) * (ay2 - a[1])
    area2 = (bx2 - b[0]) * (by2 - b[1])
    union = area1 + area2 - inter
    if area1 <= EPS or area2 <= EPS or union <= EPS:
        inter = 0.0
    if union <= EPS:
        union = 1.0
    return inter / union


def iou_matrix(ga, ta) -> List[List[float]]:
    return [[iou(g, t) for t in ta] for g in ga]


def isolated(score) -> bool:
    """True when the positive entries share no row and no column."""
    rows = [sum(v > 0 for v in r) for r in score]
    cols = [sum(r[j] > 0 for r in score) for j in range(len(score[0]))] if score else []
    return max(rows + [0]) <= 1 and max(cols + [0]) <= 1


def assign(score, shortcut: bool = True) -> list:
    """(row, col) pairs of lsap(-score) with score > eps, rows ascending; with `shortcut`, the positive entries directly
    when they are isolated."""
    if not score or not score[0]:
        return []
    if shortcut and isolated(score):
        return [(i, j) for i, r in enumerate(score) for j, v in enumerate(r) if v > 0]
    rows, cols = lsap([[-v for v in r] for r in score])
    return [(i, j) for i, j in zip(rows.tolist(), cols.tolist()) if score[i][j] > EPS]


class Frame:
    """One frame after preprocessing: gt ids and boxes, tracker ids and boxes, and S = IoU of the two (rows x cols)."""
    __slots__ = ("gids", "tids", "S")

    def __init__(self, gids, tids, S):
        self.gids, self.tids, self.S = gids, tids, S


def preprocess(gt, trk, seq_length: int, benchmark: str = "MOT17") -> List[Frame]:
    gt, trk = np.asarray(gt, np.float64).reshape(-1, 8), np.asarray(trk, np.float64).reshape(-1, 7)
    distract = distractor_classes(benchmark)
    by_g, by_t = [[] for _ in range(seq_length + 1)], [[] for _ in range(seq_length + 1)]
    for r in gt.tolist():
        by_g[int(r[0])].append(r)
    for r in trk.tolist():
        by_t[int(r[0])].append(r)
    frames = []
    for f in range(1, seq_length + 1):
        g, t = by_g[f], by_t[f]
        if benchmark != "MOT15" and g and t:
            S = iou_matrix([r[2:6] for r in g], [r[2:6] for r in t])
            S = [[v if v >= 0.5 - EPS else 0.0 for v in r] for r in S]
            removed = {j for i, j in assign(S, shortcut=False) if int(g[i][7]) in distract}
            t = [r for j, r in enumerate(t) if j not in removed]
        if benchmark != "MOT15":
            g = [r for r in g if r[6] != 0 and r[7] == 1]
        else:
            g = [r for r in g if r[6] != 0]
        frames.append(Frame([int(r[1]) for r in g], [int(r[1]) for r in t], iou_matrix([r[2:6] for r in g], [r[2:6] for r in t])))
    return frames


def clear_score(fr: Frame, prev: Dict[int, int]):
    """The CLEAR score of an effective frame given the gt id -> tracker id matches of the last effective frame."""
    return [[(1000.0 + s if prev.get(g) == t else s) if s >= 0.5 - EPS else 0.0 for t, s in zip(fr.tids, row)]
            for g, row in zip(fr.gids, fr.S)]


def _pairs_to_map(fr: Frame, pairs) -> Dict[int, int]:
    return {fr.gids[i]: fr.tids[j] for i, j in pairs}


def clear_pairs(frames: Sequence[Frame]) -> list:
    """The sequential loop: each effective frame's matched (row, col) pairs (None for the other frames)."""
    prev, out = {}, []
    for fr in frames:
        if not fr.gids or not fr.tids:
            out.append(None)
            continue
        pairs = assign(clear_score(fr, prev), shortcut=False)
        prev = _pairs_to_map(fr, pairs)
        out.append(pairs)
    return out


def clear_pairs_by_rounds(frames: Sequence[Frame]):
    """(pairs as ``clear_pairs``, rounds): every effective frame solved from its predecessor's matches of the previous
    round, starting from no matches; only frames whose predecessor changed are solved again, frames of isolated positives
    never; stops when nothing changed."""
    eff = [k for k, fr in enumerate(frames) if fr.gids and fr.tids]
    pred = {eff[n]: eff[n - 1] for n in range(1, len(eff))}
    fixed = {k for k in eff if isolated(clear_score(frames[k], {}))}
    state = {k: assign(clear_score(frames[k], {})) for k in eff}
    changed, rounds = set(eff), 1 if eff else 0
    while True:
        todo = [k for k in eff if k in pred and pred[k] in changed and k not in fixed]
        if not todo:
            break
        rounds += 1
        new = {k: assign(clear_score(frames[k], _pairs_to_map(frames[pred[k]], state[pred[k]]))) for k in todo}
        changed = {k for k in todo if new[k] != state[k]}
        state.update(new)
    return [state.get(k) for k in range(len(frames))], rounds


def clear_counts(frames: Sequence[Frame], pairs: Sequence) -> dict:
    """CLEAR's counts and MOTP_sum from each effective frame's final pairs."""
    TP = FP = FN = IDSW = 0
    motp = 0.0
    present, matched, frag = Counter(), Counter(), Counter()
    last: Dict[int, int] = {}
    prev: Dict[int, int] = {}
    for fr, pr in zip(frames, pairs):
        if not fr.gids:
            FP += len(fr.tids)
            continue
        present.update(fr.gids)
        if not fr.tids:
            FN += len(fr.gids)
            continue
        s = 0.0
        for i, j in pr:
            g, t = fr.gids[i], fr.tids[j]
            if g in last and last[g] != t:
                IDSW += 1
            if g not in prev:
                frag[g] += 1
            matched[g] += 1
            s += fr.S[i][j]
        for i, j in pr:
            last[fr.gids[i]] = fr.tids[j]
        prev = _pairs_to_map(fr, pr)
        TP += len(pr)
        FN += len(fr.gids) - len(pr)
        FP += len(fr.tids) - len(pr)
        motp += s
    ratio = [matched[g] / present[g] for g in present]
    MT = sum(r > 0.8 for r in ratio)
    PT = sum(r >= 0.2 for r in ratio) - MT
    return dict(TP=TP, FP=FP, FN=FN, IDSW=IDSW, Frag=sum(c - 1 for c in frag.values() if c > 0), MT=MT, PT=PT,
                ML=len(present) - MT - PT, MOTP_sum=motp)


def potential_matches(frames: Sequence[Frame]) -> Counter:
    return Counter((fr.gids[i], fr.tids[j]) for fr in frames for i, row in enumerate(fr.S) for j, s in enumerate(row)
                   if s >= 0.5)


def identity(frames: Sequence[Frame]) -> int:
    """IDTP: a maximum-weight matching of the potential-match counts, solved per connected component with ``lsap``."""
    counts = potential_matches(frames)
    adj: Dict[tuple, set] = {}
    for g, t in counts:
        adj.setdefault(("g", g), set()).add(("t", t))
        adj.setdefault(("t", t), set()).add(("g", g))
    seen, idtp = set(), 0
    for start in sorted(adj):
        if start in seen:
            continue
        comp, stack = [], [start]
        seen.add(start)
        while stack:
            v = stack.pop()
            comp.append(v)
            for w in adj[v]:
                if w not in seen:
                    seen.add(w)
                    stack.append(w)
        gs = sorted(v[1] for v in comp if v[0] == "g")
        ts = sorted(v[1] for v in comp if v[0] == "t")
        rows, cols = lsap([[-float(counts.get((g, t), 0)) for t in ts] for g in gs])
        idtp += sum(counts.get((gs[i], ts[j]), 0) for i, j in zip(rows.tolist(), cols.tolist()))
    return idtp


def finish(d: dict) -> dict:
    """Adds the ratios to a dict of the counts and MOTP_sum."""
    TP, FP, FN, IDSW = d["TP"], d["FP"], d["FN"], d["IDSW"]
    IDTP, IDFP, IDFN = d["IDTP"], d["IDFP"], d["IDFN"]
    d = dict(d)
    d["MOTA"] = (TP - FP - IDSW) / max(1, TP + FN)
    d["MOTP"] = d["MOTP_sum"] / max(1, TP)
    d["Rcll"] = TP / max(1, TP + FN)
    d["Prcn"] = TP / max(1, TP + FP)
    d["IDR"] = IDTP / max(1, IDTP + IDFN)
    d["IDP"] = IDTP / max(1, IDTP + IDFP)
    d["IDF1"] = IDTP / max(1, IDTP + 0.5 * IDFP + 0.5 * IDFN)
    return d


def evaluate(name: str, gt, trk, seq_length: int, benchmark: str = "MOT17", by_rounds: bool = False) -> dict:
    """Every field of one sequence (the sequential CLEAR loop, or with `by_rounds` the rounds, whose count is added)."""
    check_rows(name, gt, trk, seq_length, benchmark)
    frames = preprocess(gt, trk, seq_length, benchmark)
    if by_rounds:
        pairs, rounds = clear_pairs_by_rounds(frames)
    else:
        pairs, rounds = clear_pairs(frames), None
    d = clear_counts(frames, pairs)
    n_gt, n_trk = sum(len(fr.gids) for fr in frames), sum(len(fr.tids) for fr in frames)
    d["IDTP"] = identity(frames)
    d.update(IDFN=n_gt - d["IDTP"], IDFP=n_trk - d["IDTP"], gt_rows=n_gt, tracker_rows=n_trk)
    d = finish(d)
    if by_rounds:
        d["rounds"] = rounds
    return d


def combine(results: Sequence[dict]) -> dict:
    """The fields over several sequences: integer fields summed, MOTP_sum summed in sequence order, ratios recomputed."""
    d = {k: sum(r[k] for r in results) for k in INT_FIELDS}
    s = 0.0
    for r in results:
        s += r["MOTP_sum"]
    d["MOTP_sum"] = s
    return finish(d)


# -- the literal form -----------------------------------------------------------------------------------------------------------
def box_ious(b1, b2) -> np.ndarray:
    """TrackEval's _calculate_box_ious for xywh boxes, vectorised."""
    b1, b2 = np.array(b1, np.float64).reshape(-1, 4), np.array(b2, np.float64).reshape(-1, 4)
    b1[:, 2] = b1[:, 0] + b1[:, 2]
    b1[:, 3] = b1[:, 1] + b1[:, 3]
    b2[:, 2] = b2[:, 0] + b2[:, 2]
    b2[:, 3] = b2[:, 1] + b2[:, 3]
    mn = np.minimum(b1[:, None, :], b2[None, :, :])
    mx = np.maximum(b1[:, None, :], b2[None, :, :])
    inter = np.maximum(mn[..., 2] - mx[..., 0], 0) * np.maximum(mn[..., 3] - mx[..., 1], 0)
    a1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    a2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    union = a1[:, None] + a2[None, :] - inter
    inter[a1 <= 0 + EPS, :] = 0
    inter[:, a2 <= 0 + EPS] = 0
    inter[union <= 0 + EPS] = 0
    union[union <= 0 + EPS] = 1
    return inter / union


def evaluate_literal(gt, trk, seq_length: int, benchmark: str = "MOT17") -> dict:
    """The protocol in TrackEval's matrix form with numpy and scipy, written apart from the restatement above."""
    from scipy.optimize import linear_sum_assignment
    gt, trk = np.asarray(gt, np.float64).reshape(-1, 8), np.asarray(trk, np.float64).reshape(-1, 7)
    distract = np.array(distractor_classes(benchmark))
    g_ids, t_ids, sims = [], [], []
    for f in range(1, seq_length + 1):
        gm, tm = gt[:, 0] == f, trk[:, 0] == f
        gi, gb, gc, gz = gt[gm, 1].astype(int), gt[gm, 2:6], gt[gm, 7].astype(int), gt[gm, 6]
        ti, tb = trk[tm, 1].astype(int), trk[tm, 2:6]
        sim = box_ious(gb, tb)
        remove = np.array([], int)
        if benchmark != "MOT15" and len(gi) and len(ti):
            ms = sim.copy()
            ms[ms < 0.5 - EPS] = 0
            r, c = linear_sum_assignment(-ms)
            ok = ms[r, c] > 0 + EPS
            r, c = r[ok], c[ok]
            remove = c[np.isin(gc[r], distract)]
        ti, sim = np.delete(ti, remove), np.delete(sim, remove, axis=1)
        keep = (gz != 0) & (gc == 1) if benchmark != "MOT15" else gz != 0
        g_ids.append(gi[keep])
        t_ids.append(ti)
        sims.append(sim[keep])
    ug = np.unique(np.concatenate(g_ids + [np.zeros(0, int)]))
    ut = np.unique(np.concatenate(t_ids + [np.zeros(0, int)]))
    g_ids = [np.searchsorted(ug, x) for x in g_ids]
    t_ids = [np.searchsorted(ut, x) for x in t_ids]
    G, T = len(ug), len(ut)
    # CLEAR
    res = dict(TP=0, FP=0, FN=0, IDSW=0, MOTP_sum=0.0)
    gt_id_count, matched_count, frag_count = np.zeros(G), np.zeros(G), np.zeros(G)
    prev_tracker = np.full(G, np.nan)
    prev_ts = np.full(G, np.nan)
    for gi, ti, sim in zip(g_ids, t_ids, sims):
        if len(gi) == 0:
            res["FP"] += len(ti)
            continue
        if len(ti) == 0:
            res["FN"] += len(gi)
            gt_id_count[gi] += 1
            continue
        gt_id_count[gi] += 1
        score = 1000 * (ti[None, :] == prev_ts[gi[:, None]]) + sim
        score[sim < 0.5 - EPS] = 0
        r, c = linear_sum_assignment(-score)
        ok = score[r, c] > 0 + EPS
        r, c = r[ok], c[ok]
        mg, mt = gi[r], ti[c]
        pm = prev_tracker[mg]
        res["IDSW"] += int(np.sum(np.logical_not(np.isnan(pm)) & np.not_equal(mt, pm)))
        matched_count[mg] += 1
        not_prev = np.isnan(prev_ts)
        prev_tracker[mg] = mt
        prev_ts[:] = np.nan
        prev_ts[mg] = mt
        frag_count += np.logical_and(not_prev, np.logical_not(np.isnan(prev_ts)))
        res["TP"] += len(mg)
        res["FN"] += len(gi) - len(mg)
        res["FP"] += len(ti) - len(mg)
        if len(mg):
            res["MOTP_sum"] += sum(sim[r, c])
    ratio = matched_count[gt_id_count > 0] / gt_id_count[gt_id_count > 0]
    res["MT"] = int(np.sum(np.greater(ratio, 0.8)))
    res["PT"] = int(np.sum(np.greater_equal(ratio, 0.2))) - res["MT"]
    res["ML"] = G - res["MT"] - res["PT"]
    res["Frag"] = int(np.sum(np.subtract(frag_count[frag_count > 0], 1)))
    # Identity, TrackEval's square matrix
    pot = np.zeros((G, T))
    gcount, tcount = np.zeros(G), np.zeros(T)
    for gi, ti, sim in zip(g_ids, t_ids, sims):
        a, b = np.nonzero(np.greater_equal(sim, 0.5))
        np.add.at(pot, (gi[a], ti[b]), 1)
        gcount[gi] += 1
        tcount[ti] += 1
    fp = np.zeros((G + T, G + T))
    fn = np.zeros((G + T, G + T))
    fp[G:, :T] = 1e10
    fn[:G, T:] = 1e10
    for g in range(G):
        fn[g, :T] = gcount[g]
        fn[g, T + g] = gcount[g]
    for t in range(T):
        fp[:G, t] = tcount[t]
        fp[t + G, t] = tcount[t]
    fn[:G, :T] -= pot
    fp[:G, :T] -= pot
    r, c = linear_sum_assignment(fn + fp)
    IDFN = int(fn[r, c].sum())
    IDFP = int(fp[r, c].sum())
    res.update(IDTP=int(gcount.sum()) - IDFN, IDFN=IDFN, IDFP=IDFP, gt_rows=int(gcount.sum()), tracker_rows=int(tcount.sum()))
    return finish(res)
