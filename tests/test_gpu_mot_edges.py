"""The GPU MOT evaluator against oracle/mot_ref.py (CLEAR MOT, identity) and oracle/mot_hota_ref.py (HOTA), exactly, at its
edges: IoUs exactly at CLEAR's 0.5 - eps and HOTA's alpha - eps and one step below, tracker ids 0 and 2^22 - 1 and on both
sides of a 32-id word of the HOTA bitmap; frames of 512 gt rows and 512 tracker rows that overlap ambiguously, so that
distractor removal, CLEAR and HOTA each solve a 512 x 512 assignment; and a sequence of 1500 gt ids and 1500 tracker ids,
so that the identity metrics' assignment (IDTP) is one dense 1500 x 1500 solve in global memory."""
import math

import numpy as np
import pytest

from mot_sequences import blocks
from oracle import mot_hota_ref, mot_ref
from test_gpu_mot import PERSON
from test_gpu_mot import _check as _check_clear
from test_gpu_mot_hota import _check as _check_hota

EPS = mot_ref.EPS
MAX_ID = 1 << 22


# tracker boxes (left, width) as float32 records give them, and the gt width whose IoU with them is about t: the union
# rounds to 2 in both, the intersection is w - 0.5 in the first and w in the second
GEOMETRIES = [((0.5, 1.5), lambda t: 2.0 * t + 0.5), ((0.0, 2.0), lambda t: 2.0 * t)]


def _pair_for(target):
    """(gt width w, tracker (left, width)) such that the gt box (0, top, w, 1) and the tracker box have an IoU of exactly
    `target`."""
    for trk, guess in GEOMETRIES:
        w = guess(target)
        for c in [w] + [float(v) for v in np.nextafter(w, [math.inf, -math.inf])]:
            if mot_ref.iou((0.0, 0.0, c, 1.0), (trk[0], 0.0, trk[1], 1.0)) == target:
                return c, trk
    raise AssertionError(f"no gt width gives IoU {target!r}")


def _targets():
    half_m = 0.5 - EPS
    t = [half_m, float(np.nextafter(half_m, 0)), 0.5, float(np.nextafter(0.5, 0))]
    for a in (mot_hota_ref.ALPHAS[0], mot_hota_ref.ALPHAS[4], mot_hota_ref.ALPHAS[12], mot_hota_ref.ALPHAS[17]):
        t += [a - EPS, float(np.nextafter(a - EPS, 0)), a]
    return t


IDS = [0, MAX_ID - 1, 31, 32, 63, 64, 1023, 1024, MAX_ID - 32, MAX_ID - 33, 5, 6, 7, 8, 9, 10, 11, 12, 13]


def _boundary_sequence(L=6):
    """(gt, frames): per frame one gt / tracker pair at each target IoU, each pair in its own row band; tracker ids at the
    edges of the id range, rotated between frames so that some matches switch ids."""
    targets = _targets()
    assert len(IDS) >= len(targets)
    pairs = [_pair_for(t) for t in targets]
    gt, frames = [], []
    for f in range(1, L + 1):
        recs = []
        for k, (w, (left, tw)) in enumerate(pairs):
            top = 10.0 * k
            gt.append([f, k + 1, 0.0, top, w, 1.0, 1, 1])
            tid = IDS[(k + (f // 3)) % len(targets)]
            # tracker (ymin, xmin, ymax, xmax): left = xmin + 1, top = ymin + 1
            recs.append((tid, (top - 1.0, left - 1.0, top, left - 1.0 + tw), 0.5))
        frames.append(recs)
    return np.array(gt, np.float64), frames


def _crowd_sequence(rng, L=3, n=512):
    """Frames of n gt rows and n tracker rows packed along one line, every box overlapping several others at IoUs around
    0.5.  In all but the last frame a tenth of the gt rows are of distractor classes, so distractor removal solves n x n;
    the last frame has none, so CLEAR and HOTA keep all n x n rows."""
    gt, frames = [], []
    for f in range(1, L + 1):
        recs = []
        for i in range(n):
            x, y = 6.0 * i, 100.0 + 3.0 * (i % 4)
            cls = 1 if f == L or rng.random() < 0.9 else int(rng.choice([2, 7, 8, 12]))
            gt.append([f, i + 1, x, y, 24.0, 60.0, 1, cls])
            j = rng.integers(-4, 5, 2)
            recs.append((int(rng.integers(0, MAX_ID)) if i % 7 == 0 else 100 + (i + f * (i % 5 == 0)) % n,
                         (y - 1.0 + j[1], x - 1.0 + j[0], y - 1.0 + j[1] + 60.0, x - 1.0 + j[0] + 24.0), 0.5))
        ids = [r[0] for r in recs]
        seen = set()
        for k, t in enumerate(ids):                     # one id once per frame
            while t in seen:
                t = (t + 1) % MAX_ID
            seen.add(t)
            recs[k] = (t,) + recs[k][1:]
        frames.append(recs)
    return np.array(gt, np.float64), frames


def _identity_sequence(rng, L=199, rows=15):
    """rows objects side by side for L frames.  Each gt id lasts two frames (frames 2k - 1, 2k) and each tracker id two
    frames out of phase with them (2k, 2k + 1), so every row is one chain of potential matches through the sequence:
    (L + 1) / 2 gt ids and as many tracker ids per row, 1500 of each at the defaults."""
    gt, frames = [], []
    for f in range(1, L + 1):
        recs = []
        for r in range(rows):
            x, y = 100.0 * r, 200.0
            gt.append([f, (f - 1) // 2 * rows + r + 1, x, y, 40.0, 100.0, 1, 1])
            j = rng.integers(-4, 5, 4)
            recs.append((f // 2 * rows + r, (y - 1.0 + j[1], x - 1.0 + j[0], y - 1.0 + j[1] + 100.0 + j[3],
                                             x - 1.0 + j[0] + 40.0 + j[2]), 0.5))
        frames.append(recs)
    return np.array(gt, np.float64), frames


def _run(seqs, K, benchmark="MOT17"):
    """MotEval's result over seqs [(name, gt, frames, L)] and the oracles' CLEAR / identity and HOTA results."""
    import torch
    from k210_yolo_framework_b200.evaluate import MotEval
    ev = MotEval(benchmark, device=0)
    clear, hota = {}, {}
    for name, gt, frames, L in seqs:
        ev.add_sequence(name, gt, L)
    for name, gt, frames, L in seqs:
        ids, boxes, dets, counts = blocks(frames, K=K, rng=np.random.default_rng(1))
        trk = mot_ref.tracker_rows(range(L), ids, boxes, dets, counts, PERSON)
        clear[name] = mot_ref.evaluate(name, gt, trk, L, benchmark, by_rounds=True)
        hota[name] = mot_hota_ref.evaluate_hota(name, gt, trk, L, benchmark)
        blk = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (ids, boxes, dets, counts)]
        ev.update(name, range(L), *blk, PERSON)
    return ev.result(), clear, hota


def test_the_boundary_sequence_is_on_its_boundaries():
    """Each target IoU is met exactly, and CLEAR counts the rows at 0.5 - eps and not those one step below (CPU)."""
    gt, frames = _boundary_sequence()
    for t in _targets():
        w, (left, tw) = _pair_for(t)
        assert mot_ref.iou((0.0, 0.0, w, 1.0), (left, 0.0, tw, 1.0)) == t
    ids, boxes, dets, counts = blocks(frames, K=32, rng=np.random.default_rng(1))
    trk = mot_ref.tracker_rows(range(len(frames)), ids, boxes, dets, counts, PERSON)
    r = mot_ref.evaluate("b", gt, trk, len(frames))
    below = sum(t < 0.5 - EPS for t in _targets())
    n = len(_targets())
    assert r["FP"] == r["FN"] == below * len(frames) and r["TP"] == (n - below) * len(frames) and r["IDSW"] > 0


@pytest.mark.gpu
def test_ious_at_the_thresholds_and_ids_at_the_edges():
    gt, frames = _boundary_sequence()
    res, clear, hota = _run([("b", gt, frames, len(frames))], K=32)
    _check_clear(res, clear)
    _check_hota(res, hota)


def test_the_crowd_and_identity_sequences_reach_their_sizes():
    """The last crowd frame keeps 512 gt rows and 512 tracker rows whose positive entries share rows and columns, so CLEAR
    and HOTA cannot take the isolated-pairs shortcut; the identity sequence has 1500 gt ids and 1500 tracker ids (CPU)."""
    gt, frames = _crowd_sequence(np.random.default_rng(3))
    ids, boxes, dets, counts = blocks(frames, K=520, rng=np.random.default_rng(1))
    trk = mot_ref.tracker_rows(range(len(frames)), ids, boxes, dets, counts, PERSON)
    last = mot_ref.preprocess(gt, trk, len(frames))[-1]
    assert len(last.gids) == len(last.tids) == 512
    assert not mot_ref.isolated(mot_ref.clear_score(last, {}))
    assert len(set(gt[gt[:, 7] != 1, 0].tolist())) == len(frames) - 1      # distractors in every other frame
    gt, frames = _identity_sequence(np.random.default_rng(4))
    ids, boxes, dets, counts = blocks(frames, K=32, rng=np.random.default_rng(1))
    trk = mot_ref.tracker_rows(range(len(frames)), ids, boxes, dets, counts, PERSON)
    assert len(set(gt[:, 1].tolist())) == len(set(trk[:, 1].tolist())) == 1500
    assert mot_ref.evaluate("i", gt, trk, len(frames))["TP"] == len(gt)


@pytest.mark.gpu
def test_frames_of_512_rows_each_side():
    gt, frames = _crowd_sequence(np.random.default_rng(3))
    res, clear, hota = _run([("c", gt, frames, len(frames))], K=520)
    _check_clear(res, clear)
    _check_hota(res, hota)
    assert res["solved"]["c"] > 0


@pytest.mark.gpu
def test_identity_metrics_of_1500_gt_ids_by_1500_tracker_ids():
    gt, frames = _identity_sequence(np.random.default_rng(4))
    res, clear, hota = _run([("i", gt, frames, len(frames))], K=32)
    _check_clear(res, clear)
    _check_hota(res, hota)
    r = clear["i"]
    assert 0 < r["IDTP"] < r["TP"] and r["IDFP"] > 0 and r["IDFN"] > 0
